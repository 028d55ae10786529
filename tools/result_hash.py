"""SHA-256 over everything smr_align_batch returns for N reads of the synthetic bench workload (8 databases, device-built
indexes): two builds of the library (SMR_LIB_PATH) that print the same line returned bit-identical results.
Usage: python tools/result_hash.py [N]   (needs a GPU)"""
import hashlib
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from sortmerna_b200 import api  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000
    work = tempfile.TemporaryDirectory(prefix="smr_hash_")
    fastas, idx_dir, prefixes, refs, stats, built = bench.load_databases(work.name)
    ms = bench.minimal_scores(stats, fastas, 10_000_000)
    al = api.Aligner(0)
    al.set_params(api.default_params())
    bench.load_resident_index(al, "device", fastas, prefixes, refs, ms, stats)
    reads = bench.gen_reads(bench.DbPool(refs), n, bench.GEN_SEED + 99)
    off = (np.arange(n + 1, dtype=np.uint64) * bench.READ_LEN)
    got = al.align(np.ascontiguousarray(reads.reshape(-1)), off)
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(got["res"]).tobytes())
    a = got["alns"]
    for f in sorted(a.dtype.names):
        if f != "cigar_off":                       # where a CIGAR lies in the pool depends on the order the warps finished in
            h.update(np.ascontiguousarray(a[f]).tobytes())
    ln = a["cigar_len"].astype(np.int64); of = a["cigar_off"].astype(np.int64)
    tot = int(ln.sum())
    start = np.repeat(of - (np.cumsum(ln) - ln), ln)     # CIGAR words gathered in alignment-slot order
    h.update(np.ascontiguousarray(got["cigar"][start + np.arange(tot)]).tobytes())
    c = got.get("counters", {})
    print("result_hash", n, h.hexdigest(), "aligned", int(got["res"]["is_hit"].sum()),
          {k: int(c[k]) for k in ("sw_calls", "sw_cells", "lis_calls", "pos_entries") if k in c})
    al.close()


if __name__ == "__main__":
    main()
