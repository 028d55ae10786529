"""Rate of the device report writer (smr_format_reports) on the benchmark workload: bench.py's seeded reads against the 8 stand-in
databases, aligned once on the GPU, then formatted per output kind.  Prints one JSON line:
  * per format (sam, blast, fastx+other, denovo, all): device time of the call (CUDA events: layout, size pass, scans, write pass),
    the H2D of text + results and the D2H of the output, the call's wall time, output MB/s and reads/s;
  * the host formatters of hostio (format_sam_rows / format_blast_rows, one Python row at a time) on a subset;
  * with --reference, the reference binary's report stage ("done Reports in" of its log) on a subset of the same reads.
Run on the GPU:  python tools/bench_reports.py --reads 1000000"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from sortmerna_b200 import api, hostio  # noqa: E402

FORMATS = {"sam": dict(sam=True), "blast": dict(blast="1 cigar qcov qstrand"), "fastx_other": dict(fastx=True, other=True),
           "denovo": dict(denovo=(0.97, 0.97)),
           "all": dict(sam=True, blast="1 cigar qcov qstrand", fastx=True, other=True, denovo=(0.97, 0.97))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reads", type=int, default=20_000, help="subset for the Python hostio formatters")
    ap.add_argument("--reference", type=int, default=0, help="reads of the subset the reference binary formats (0: skip)")
    args = ap.parse_args()
    out = dict(card=bench.card(0), reads=args.reads)
    with tempfile.TemporaryDirectory(prefix="smr_bench_rpt_") as work:
        fastas, idx_dir, prefixes, refs, stats, _ = bench.load_databases(work)
        pool = bench.DbPool(refs)
        reads = bench._gen_reads_numpy(pool, args.reads, bench.GEN_SEED + 4242)
        fq = os.path.join(work, "reads.fq")
        bench.write_fastq(fq, reads)
        text = open(fq, "rb").read()
        ms = bench.minimal_scores(stats, fastas, args.reads)
        g = json.load(open(os.path.join(ROOT, "sortmerna_b200", "gumbel_defaults.json")))["gumbel"]
        al = api.Aligner(0)
        al.set_params(api.default_params())
        bench.load_resident_index(al, "files", fastas, prefixes, refs, ms, stats)
        gum = []
        for k, f in enumerate(fastas):
            lam, K = g[os.path.basename(f)]["lambda_"], g[os.path.basename(f)]["K"]
            gum.append((lam, K))
            al.set_report_scoring(k, lam, K, *hostio.evalue_params(stats[k], K, args.reads * bench.READ_LEN, args.reads))
        n = al.upload_fastx(text)
        al.run_resident(with_stats=True)
        res = al.download()
        out["aligned"] = int(res["res"]["is_hit"].sum())
        out["text_mb"] = len(text) / 1e6
        fm = {}
        for name, kw in FORMATS.items():
            al.format_reports(res, None, **kw)   # warm-up: buffers, module load
            dev, wall = [], []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                s = al.format_reports(res, None, **kw)
                wall.append(time.perf_counter() - t0)
                dev.append(al.report_timings())
            nb = sum(len(x) for x in s["sam"] + s["blast"]) + len(s["aligned"]) + len(s["other"]) + len(s["denovo"])
            dms = float(np.median([t["device_ms"] for t in dev]))
            w = float(np.median(wall))
            fm[name] = dict(out_mb=nb / 1e6, device_ms=dms, h2d_ms=float(np.median([t["h2d_ms"] for t in dev])),
                            d2h_ms=float(np.median([t["d2h_ms"] for t in dev])), call_wall_ms=w * 1e3,
                            device_mb_s=nb / 1e6 / (dms / 1e3), wall_mb_s=nb / 1e6 / w, wall_reads_s=n / w)
        out["writer"] = fm
        # Python host formatters on a subset
        m = args.host_reads
        sub = hostio.pack_reads([f"@{i:09d}" for i in range(m)], [bytes(np.frombuffer(b"ACGT", np.uint8)[reads[i]]) for i in range(m)],
                                [b"I" * bench.READ_LEN] * m)
        slots = res["slots"]
        r_res, r_alns, r_st = res["res"][:m], res["alns"][:m * slots], res["stats"][:m * slots]
        t0 = time.perf_counter()
        rows = hostio.format_sam_rows(sub, refs, r_res, r_alns, res["cigar"], slots)
        t_sam = time.perf_counter() - t0
        evp = [hostio.evalue_params(st, K, args.reads * bench.READ_LEN, args.reads) for st, (_, K) in zip(stats, gum)]
        t0 = time.perf_counter()
        hostio.format_blast_rows(sub, refs, r_res, r_alns, res["cigar"], slots, r_st, gum, evp)
        t_blast = time.perf_counter() - t0
        out["hostio"] = dict(reads=m, sam_rows=len(rows), sam_reads_s=m / t_sam, blast_reads_s=m / t_blast)
        al.close()
        if args.reference:
            from oracle import ora
            if not os.path.exists(ora.REF_BIN):
                out["reference"] = "not built"
            else:
                ref_idx = bench.reference_index_dir(work, fastas)
                k = args.reference
                fq2 = os.path.join(work, "ref_reads.fq")
                bench.write_fastq(fq2, reads[:k])
                r = ora.run_reference(fastas, fq2, os.path.join(work, "ref"), extra=["-sam", "-blast", "1 cigar qcov qstrand", "-fastx", "-other"],
                                      threads=os.cpu_count() or 8, idx_dir=ref_idx)
                mt = re.search(r"done Reports in ([0-9.eE+-]+) sec", r["stdout"])
                sec = float(mt.group(1)) if mt else None
                out["reference"] = dict(reads=k, threads=os.cpu_count(), report_stage_s=sec, reads_s=k / sec if sec else None)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
