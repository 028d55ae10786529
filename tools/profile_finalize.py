"""Device time of each finalize-stage kernel on the benchmark workload, from torch.profiler (CUDA activities).

run_impl times the whole finalize stage as one span (smr_last_timings final_ms); this splits it per kernel.  The databases,
indexes and reads are made the way bench.py makes them (8 seeded stand-in databases indexed on the device, synthetic 150 bp
reads).  The batch is uploaded once and run_resident() runs it --warmup times untraced, then --runs times under the profiler.
Prints one JSON line: the mean ms per run of every kernel whose name matches --match, plus the library's own final_ms.
Usage: python tools/profile_finalize.py [--reads 1000000] [--runs 3]   (needs a GPU; SMR_LIB_PATH selects another build)"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--match", default="finalize,traceback,final_jobs", help="comma-separated substrings of the kernel names to report")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from sortmerna_b200 import api

    work = tempfile.TemporaryDirectory(prefix="smr_prof_")
    fastas, idx_dir, prefixes, refs, stats, built = bench.load_databases(work.name)
    ms = bench.minimal_scores(stats, fastas, 10_000_000)
    al = api.Aligner(0)
    al.set_params(api.default_params())
    bench.load_resident_index(al, "device", fastas, prefixes, refs, ms, stats)
    n = args.reads
    reads = bench.gen_reads(bench.DbPool(refs), n, bench.GEN_SEED)
    off = np.arange(n + 1, dtype=np.uint64) * bench.READ_LEN
    al.upload(np.ascontiguousarray(reads.reshape(-1)), off)
    for _ in range(args.warmup):
        al.run_resident()
    torch.cuda.synchronize()
    final_ms = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.runs):
            al.run_resident()
            final_ms.append(al.timings()["final_ms"])
        torch.cuda.synchronize()
    keys = [k for k in args.match.split(",") if k]
    per_kernel = {}
    for ev in prof.key_averages():
        if any(k in ev.key for k in keys):
            t_us = getattr(ev, "device_time_total", None)
            if t_us is None:
                t_us = ev.cuda_time_total
            name = ev.key.split("(")[0].replace("smr::", "")
            per_kernel[name] = {"ms_per_run": t_us / 1000.0 / args.runs, "launches_per_run": ev.count / args.runs}
    out = {"reads": n, "runs": args.runs, "device": torch.cuda.get_device_name(0), "kernels": per_kernel,
           "final_ms_span": float(np.mean(final_ms)), "num_aligned": int(al.download()["counters"]["num_aligned"])}
    try:
        import subprocess
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                                            text=True, timeout=20).stdout.strip()
    except Exception:
        pass
    print(json.dumps(out))
    al.close()


if __name__ == "__main__":
    main()
