"""The index budget (smr_set_index_budget) on bench.py's workload: the 8 seeded stand-in databases built on the device, synthetic
150 bp reads, with the budget off and at about 1/2, 1/4 and 1/8 of the parts' search arrays (never below the largest part), at
1 M and 4 M reads per batch.  Per leg: the groups, the kernel time and the index upload time per batch (CUDA events inside the C ABI),
end-to-end reads/s (upload, run, download, host clock) and the device memory the context holds (torch.cuda.mem_get_info against the
free memory before it was made).  Every budgeted leg checks that its results equal the unbudgeted leg's.  Prints one JSON line with
the card name and power limit.
Run on the GPU:  python tools/bench_index_budget.py --batches 1000000 4000000 --steps 3"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from sortmerna_b200 import api  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1_000_000, 4_000_000])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--fractions", type=float, nargs="+", default=[0.5, 0.25, 0.125])
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    out = {"card": card(), "legs": []}
    with tempfile.TemporaryDirectory(prefix="smr_budget_bench_") as work:
        fastas, idx_dir, prefixes, refs, stats, _ = bench.load_databases(work)
        pool = bench.DbPool(refs)
        for n in args.batches:
            ms = bench.minimal_scores(stats, fastas, n * args.steps)
            batches = [np.ascontiguousarray(bench.gen_reads(pool, n, bench.GEN_SEED + k).reshape(-1)) for k in range(args.steps)]
            off = np.arange(n + 1, dtype=np.uint64) * bench.READ_LEN
            torch.cuda.empty_cache()
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            al = api.Aligner(0)
            al.set_params(api.default_params())
            bench.load_resident_index(al, "device", fastas, prefixes, refs, ms, stats)
            total = al.index_residency()["largest_group_bytes"]
            base = None
            for frac in [0.0] + args.fractions:
                budget = 0 if frac == 0 else int(total * frac)
                try:
                    al.set_index_budget(budget)
                except api.SmrError as e:   # a part larger than this fraction: run at the largest part instead
                    budget = int(str(e).split("its search arrays take ")[1].split(" ")[0])
                    al.set_index_budget(budget)
                al.align(batches[0], off)                      # warm-up: arenas, the index arena and the groups' host copies
                k_ms = up_us = 0.0
                t0 = time.time()
                for c in batches:
                    o = al.align(c, off)
                    k_ms += o["timings"]["total_ms"]
                    up_us += al.index_residency()["last_upload_us"]
                e2e = n * len(batches) / (time.time() - t0)
                torch.cuda.synchronize()
                used = free0 - torch.cuda.mem_get_info()[0]
                r = al.index_residency()
                if base is None:
                    base = o
                else:
                    same = all(np.array_equal(o[k], base[k]) for k in ("res", "alns", "cigar", "matched")) and o["counters"] == base["counters"]
                    assert same, f"budget {budget}: results differ from the run without a budget"
                out["legs"].append(dict(reads_per_batch=n, budget=budget, groups=r["groups"], largest_group_bytes=r["largest_group_bytes"],
                                        device_search_bytes=r["device_search_bytes"], host_bytes=r["host_bytes"],
                                        kernel_ms_per_batch=round(k_ms / len(batches), 2), upload_ms_per_batch=round(up_us / 1000 / len(batches), 2),
                                        e2e_reads_per_s=round(e2e), device_bytes_used=int(used), index_search_bytes=total))
                print(json.dumps(out["legs"][-1]), file=sys.stderr)
            al.close()
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
