"""Candidate-kernel time on a Smith-Waterman-heavy workload, the regime of real rRNA databases where a read wins votes in many
references: one seeded database of near-copies -- groups of 30-50 copies of a random ancestor, each copy at 0.2-1 % substitutions --
and 150 bp reads drawn from it at 1 % substitutions, random strand.  Many copies then tie at the top vote counts, so a read makes
about 19 Smith-Waterman calls (440 k cells; the CPU oracle on 200 reads) and the scorer warps, not the planners, bound the candidate
kernel.  (Copies at 1-3 % give 1-6 calls per read: the read's own copy out-votes the others and the `best` countdown ends the call.)
bench.py's stand-ins (5 % / 15 % divergence) are the opposite regime.

Prints one JSON line: the card, the per-step kernel times (median over the steps; CUDA events inside the C ABI), and the
Smith-Waterman calls and cells per read.  The library is the tree's build, or SMR_LIB_PATH.
Run on the GPU:  python tools/bench_heavy.py --reads 200000 --steps 5"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from sortmerna_b200 import api, hostio  # noqa: E402
from tools import stage_data  # noqa: E402

SEED = 20261016
GUMBEL_OF = "silva-bac-16s-id90.fasta"    # Gumbel parameters of the database the copies resemble (16S, ~1.4 kb)


def write_database(path, groups, length, div=(0.002, 0.01)):
    rng = np.random.default_rng(SEED)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    with open(path, "wb") as f:
        n = 0
        for g in range(groups):
            root = rng.integers(0, 4, length, dtype=np.uint8)
            for _ in range(int(rng.integers(30, 51))):
                hit = rng.random(length) < rng.uniform(*div)
                s = np.where(hit, (root + rng.integers(1, 4, length, dtype=np.uint8)) & 3, root).astype(np.uint8)
                f.write(b">heavy_%06d\n" % n + acgt[s].tobytes() + b"\n")
                n += 1
    return n


def gen_reads(refs, n, seed, err=0.01):
    rng = np.random.default_rng(seed)
    cat, off = refs.cat, refs.off.astype(np.int64)
    k = rng.integers(0, refs.n, n)
    st = off[k] + rng.integers(0, off[k + 1] - off[k] - bench.READ_LEN + 1)
    r = cat[st[:, None] + np.arange(bench.READ_LEN)[None, :]]
    sub = rng.random(r.shape) < err
    r = np.where(sub, rng.integers(0, 4, r.shape, dtype=np.uint8), r).astype(np.uint8)
    flip = (rng.random(n) < 0.5)[:, None]
    return np.ascontiguousarray(np.where(flip, (3 - r)[:, ::-1], r))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=200_000, help="reads per step")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--groups", type=int, default=100)
    ap.add_argument("--length", type=int, default=1400)
    args = ap.parse_args()
    out = dict(card=bench.card(0), reads_per_step=args.reads, steps=args.steps, lib=os.environ.get("SMR_LIB_PATH", "tree"))
    with tempfile.TemporaryDirectory(prefix="smr_bench_heavy_") as work:
        fasta = os.path.join(work, "heavy.fasta")
        out["references"] = write_database(fasta, args.groups, args.length)
        idx_dir, _ = stage_data.ensure_indexes([fasta], os.path.join(work, "idx"))
        prefix = hostio.find_index_prefixes(idx_dir)[os.path.basename(fasta)]
        refs = hostio.load_references(fasta)
        st = hostio.parse_stats(prefix)
        g = json.load(open(os.path.join(ROOT, "sortmerna_b200", "gumbel_defaults.json")))["gumbel"][GUMBEL_OF]
        ntot = args.reads * args.steps
        ms = hostio.minimal_score(st, g["lambda_"], g["K"], ntot * bench.READ_LEN, ntot)
        al = api.Aligner(0)
        al.set_params(api.default_params())
        if al.build_index_device(0, fasta, refs, ms, (18, 9, 3), st.lnwin) != 1:
            raise SystemExit("expected a single-part index")
        off = np.arange(args.reads + 1, dtype=np.uint64) * bench.READ_LEN
        batches = [gen_reads(refs, args.reads, SEED + 1 + s).reshape(-1) for s in range(args.steps)]
        al.upload(batches[0], off)
        for _ in range(args.warmup):
            al.run_resident()
            al.download()
        t = {k: [] for k in ("seed_ms", "lis_ms", "final_ms", "total_ms")}
        cnt = None
        aligned = 0
        for s in range(args.steps):
            al.upload(batches[s], off)
            al.run_resident()
            tm = al.timings()
            for k in t:
                t[k].append(tm[k])
            res = al.download()
            aligned += int(res["res"]["is_hit"].sum())
            c = np.array([res["counters"][k] for k in api.CNT_NAMES], dtype=np.int64)
            cnt = c if cnt is None else cnt + c
        al.close()
    c = dict(zip(api.CNT_NAMES, (int(x) for x in cnt)))
    nr = args.reads * args.steps
    out["kernel_ms_per_step"] = {"seed": float(np.median(t["seed_ms"])), "candidates_sw": float(np.median(t["lis_ms"])),
                                 "finalize": float(np.median(t["final_ms"])), "total": float(np.median(t["total_ms"]))}
    out["candidates_sw_ms_runs"] = [round(x, 2) for x in t["lis_ms"]]
    out["per_read"] = {"sw_calls": c["sw_calls"] / nr, "sw_cells": c["sw_cells"] / nr, "lis_calls": c["lis_calls"] / nr,
                       "pos_entries": c["pos_entries"] / nr, "aligned": aligned / nr}
    out["counters"] = {k: c[k] for k in ("sw_calls", "sw_cells", "lis_calls", "pos_entries")}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
