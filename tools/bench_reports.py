"""Rate of the device report writer (smr_format_reports) on the benchmark workload: bench.py's seeded reads against the 8 stand-in
databases, aligned once on the GPU, then formatted per output kind.  Prints one JSON line:
  * per format (sam, blast, fastx+other, denovo, all): device time of the call (CUDA events: layout, size pass, scans, write pass),
    the H2D of text + results and the D2H of the output, the call's wall time, output MB/s and reads/s;
  * the host formatters of hostio (format_sam_rows / format_blast_rows, one Python row at a time) on a subset;
  * with --reference, the reference binary's report stage ("done Reports in" of its log) on a subset of the same reads;
  * with --gzip, per format the gzip call (smr_format_reports_gz, the -zip-out output) next to the plain call on the same reads: the
    compressed bytes, the call wall times, the sizes Python's zlib makes of the same streams at levels 1 and 6, and the gz call's
    device span minus the plain call's (compress_span_ms: the encoder's kernels plus the host work inside the span -- chunk plan,
    the read-back of the chunk sizes, the byte-size scan, the uploads).  For "all", the encoder's kernels alone under torch.profiler
    (one run of its own): device time per kernel, their sum and its input GB/s;
  * with --pairwise, only BLAST: tabular rows (smr_format_reports, '1 cigar qcov qstrand') and pairwise rows (-blast 0,
    smr_format_blast_pairwise) of the same results, each plain and gzip: output MB, device time, H2D / D2H and the call's wall time.
Run on the GPU:  python tools/bench_reports.py --reads 1000000 [--gzip | --pairwise]"""
import argparse
import json
import os
import re
import sys
import tempfile
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from sortmerna_b200 import api, hostio  # noqa: E402

FORMATS = {"sam": dict(sam=True), "blast": dict(blast="1 cigar qcov qstrand"), "fastx_other": dict(fastx=True, other=True),
           "denovo": dict(denovo=(0.97, 0.97)),
           "all": dict(sam=True, blast="1 cigar qcov qstrand", fastx=True, other=True, denovo=(0.97, 0.97))}


def pairwise_leg(al, res, n, reps):
    """tabular and pairwise BLAST of the same results, plain and gzip (medians over reps calls after one warm-up)"""
    calls = {"blast_tabular": lambda gz: al.format_reports(res, None, gzip=gz, **FORMATS["blast"])["blast"],
             "blast_pairwise": lambda gz: al.format_blast_pairwise(res, None, gzip=gz)}
    out = {}
    for name, call in calls.items():
        for gz in (False, True):
            call(gz)
            dev, wall = [], []
            for _ in range(reps):
                t0 = time.perf_counter()
                s = call(gz)
                wall.append(time.perf_counter() - t0)
                dev.append(al.report_timings())
            nb = sum(len(x) for x in s)
            med = {k: float(np.median([t[k] for t in dev])) for k in ("device_ms", "h2d_ms", "d2h_ms")}
            w = float(np.median(wall))
            out[name + ("_gz" if gz else "")] = dict(out_mb=nb / 1e6, **med, call_wall_ms=w * 1e3, device_mb_s=nb / 1e6 / (med["device_ms"] / 1e3),
                                                     wall_reads_s=n / w)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reads", type=int, default=20_000, help="subset for the Python hostio formatters")
    ap.add_argument("--reference", type=int, default=0, help="reads of the subset the reference binary formats (0: skip)")
    ap.add_argument("--gzip", action="store_true", help="also time the gzip (-zip-out) call of every format")
    ap.add_argument("--pairwise", action="store_true", help="only tabular and pairwise BLAST (-blast 0), each plain and gzip")
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
        if args.pairwise:
            out["blast"] = pairwise_leg(al, res, n, args.reps)
            al.close()
            print(json.dumps(out))
            return
        def timed(kw, gz):
            al.format_reports(res, None, gzip=gz, **kw)   # warm-up: buffers, module load
            dev, wall = [], []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                s = al.format_reports(res, None, gzip=gz, **kw)
                wall.append(time.perf_counter() - t0)
                dev.append(al.report_timings())
            med = {k: float(np.median([t[k] for t in dev])) for k in ("device_ms", "h2d_ms", "d2h_ms")}
            return s, med, float(np.median(wall))

        def streams(s):
            return dict(sam=b"".join(s["sam"]), blast=b"".join(s["blast"]), aligned=s["aligned"], other=s["other"], denovo=s["denovo"])

        fm, zl = {}, {}
        for name, kw in FORMATS.items():
            s, med, w = timed(kw, False)
            nb = sum(len(x) for x in streams(s).values())
            fm[name] = dict(out_mb=nb / 1e6, device_ms=med["device_ms"], h2d_ms=med["h2d_ms"], d2h_ms=med["d2h_ms"], call_wall_ms=w * 1e3,
                            device_mb_s=nb / 1e6 / (med["device_ms"] / 1e3), wall_mb_s=nb / 1e6 / w, wall_reads_s=n / w)
            if args.gzip:
                if name == "all":   # zlib of every stream kind once; a format's size is the sum over the kinds it writes
                    for k, v in streams(s).items():
                        zl[k] = (len(zlib.compress(v, 1)), len(zlib.compress(v, 6)))
                g, gmed, gw = timed(kw, True)
                gb = sum(len(x) for x in g["sam"] + g["blast"]) + len(g["aligned"]) + len(g["other"]) + len(g["denovo"])
                comp = gmed["device_ms"] - med["device_ms"]
                fm[name]["gzip"] = dict(out_mb=gb / 1e6, ratio=gb / nb if nb else None, device_ms=gmed["device_ms"], compress_span_ms=comp,
                                        compress_span_in_gb_s=nb / 1e9 / (comp / 1e3) if comp > 0 else None, h2d_ms=gmed["h2d_ms"],
                                        d2h_ms=gmed["d2h_ms"], call_wall_ms=gw * 1e3, plain_call_wall_ms=w * 1e3)
        if args.gzip:
            for name in fm:
                kinds = [k for k, v in streams(al.format_reports(res, None, **FORMATS[name])).items() if v]
                fm[name]["gzip"]["zlib1_mb"] = sum(zl[k][0] for k in kinds) / 1e6
                fm[name]["gzip"]["zlib6_mb"] = sum(zl[k][1] for k in kinds) / 1e6
        if args.gzip:   # the encoder's kernels alone, in a profiled run of their own
            import torch
            from torch.profiler import ProfilerActivity, profile
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                al.format_reports(res, None, gzip=True, **FORMATS["all"])
                torch.cuda.synchronize()
            kern = {}
            for ev in prof.key_averages():
                if "def_" in ev.key or "inf_crc" in ev.key:
                    t_us = getattr(ev, "device_time_total", None)
                    kern[ev.key.split("(")[0].replace("smr::", "")] = (t_us if t_us is not None else ev.cuda_time_total) / 1e3
            tot = sum(kern.values())
            fm["all"]["gzip"].update(kernels_ms=kern, compress_kernels_ms=tot,
                                     compress_kernels_in_gb_s=fm["all"]["out_mb"] / 1e3 / (tot / 1e3) if tot > 0 else None)
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
