"""Rate of the device OTU map (smr_otu_begin / smr_otu_add / smr_otu_finish) on the benchmark workload: bench.py's seeded reads against
the 8 stand-in databases, aligned once on the GPU, then the OTU map at -id / -coverage (0.97 / 0.97 by default).  Prints one JSON line:
  * device time of smr_otu_add (CUDA events: layout, rule, compaction, append) and its H2D of text + results; device time of
    smr_otu_finish (sort, sizes, scan, write, D2H); the wall time of begin + add + finish; the map's lines, entries and bytes;
  * the denovo leg: device time of smr_denovo_stats (per-read counters and totals, CUDA events) per 1 M reads;
  * with --reference N, the reference binary's OTU stage ("OTU groups processing done in" of its log) and its denovo_stats pass
    ("done Denovo stats in") on the first N reads, at -threads 1.
Run on the GPU:  python tools/bench_otu.py --reads 1000000 --reference 20000"""
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
from sortmerna_b200 import api  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--id", type=float, default=0.97)
    ap.add_argument("--coverage", type=float, default=0.97)
    ap.add_argument("--reference", type=int, default=0, help="reads of the subset the reference binary maps (0: skip)")
    args = ap.parse_args()
    out = dict(card=bench.card(0), reads=args.reads, min_id=args.id, min_cov=args.coverage)
    with tempfile.TemporaryDirectory(prefix="smr_bench_otu_") as work:
        fastas, idx_dir, prefixes, refs, stats, _ = bench.load_databases(work)
        pool = bench.DbPool(refs)
        reads = bench._gen_reads_numpy(pool, args.reads, bench.GEN_SEED + 4242)
        fq = os.path.join(work, "reads.fq")
        bench.write_fastq(fq, reads)
        text = open(fq, "rb").read()
        ms = bench.minimal_scores(stats, fastas, args.reads)
        al = api.Aligner(0)
        al.set_params(api.default_params())
        bench.load_resident_index(al, "files", fastas, prefixes, refs, ms, stats)
        al.upload_fastx(text)
        al.run_resident(with_stats=True)
        res = al.download()
        out["aligned"] = int(res["res"]["is_hit"].sum())
        runs = []
        for rep in range(args.reps + 1):   # the first run is a warm-up: buffers, module load
            t0 = time.perf_counter()
            al.otu_begin(args.id, args.coverage)
            al.otu_add(res, None)
            m = al.otu_finish()
            wall = time.perf_counter() - t0
            if rep:
                runs.append((al.otu_timings(), wall))
        med = lambda f: float(np.median([f(t, w) for t, w in runs]))   # noqa: E731
        out["otu"] = dict(total_otu=m["total_otu"], n_yid_ycov=m["n_yid_ycov"], out_mb=len(m["text"]) / 1e6,
                          add_h2d_ms=med(lambda t, w: t["add_h2d_ms"]), add_device_ms=med(lambda t, w: t["add_device_ms"]),
                          finish_ms=med(lambda t, w: t["finish_ms"]), wall_ms=med(lambda t, w: w * 1e3))
        out["otu"]["device_ms_per_1m_reads"] = (out["otu"]["add_device_ms"] + out["otu"]["finish_ms"]) * 1e6 / args.reads
        dn = []
        for rep in range(args.reps + 1):
            t0 = time.perf_counter()
            _, tot = al.denovo_stats(res, None, args.id, args.coverage)
            wall = time.perf_counter() - t0
            if rep:
                dn.append((al.report_timings(), wall))
        dmed = lambda f: float(np.median([f(t, w) for t, w in dn]))   # noqa: E731
        out["denovo"] = dict(totals=tot, h2d_ms=dmed(lambda t, w: t["h2d_ms"]), device_ms=dmed(lambda t, w: t["device_ms"]),
                             d2h_ms=dmed(lambda t, w: t["d2h_ms"]), wall_ms=dmed(lambda t, w: w * 1e3))
        out["denovo"]["device_ms_per_1m_reads"] = out["denovo"]["device_ms"] * 1e6 / args.reads
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
                r = ora.run_reference(fastas, fq2, os.path.join(work, "ref"), extra=["-otu_map", "-id", str(args.id), "-coverage", str(args.coverage)],
                                      threads=1, idx_dir=ref_idx)
                mt = re.search(r"OTU groups processing done in ([0-9.eE+-]+) sec", r["stdout"])
                sec = float(mt.group(1)) if mt else None
                mo = re.search(r"Total OTUs = (\d+)", r["log"])
                md = re.search(r"done Denovo stats in ([0-9.eE+-]+) sec", r["stdout"])
                dsec = float(md.group(1)) if md else None
                out["reference"] = dict(reads=k, threads=1, otu_stage_s=sec, reads_s=k / sec if sec else None,
                                        total_otu=int(mo.group(1)) if mo else None, denovo_stats_s=dsec,
                                        denovo_reads_s=k / dsec if dsec else None)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
