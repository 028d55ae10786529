"""Shared by the pairwise BLAST tests: the fixtures of tests/golden/blast_pairwise/ (make_blast_pairwise_golden.py), the inputs that
reproduce them, and the comparison of two aligned.blast texts."""
import gzip
import json
import os

import numpy as np

from conftest import GOLDEN
from helpers import params_kwargs_from_args

CASES = json.load(open(os.path.join(GOLDEN, "blast_pairwise.json")))


def expected(case: str) -> bytes:
    """the reference binary's aligned.blast of the case"""
    return gzip.open(os.path.join(GOLDEN, "blast_pairwise", case + ".blast.gz"), "rb").read()


def inputs(case: str, golden_idx_dir: str) -> dict:
    """reads, references, index prefixes, parameters and the E-value inputs of the case, in --ref order"""
    from sortmerna_b200 import hostio
    c = CASES[case]
    pre = hostio.find_index_prefixes(golden_idx_dir)
    prefixes = [pre[d] for d in c["dbs"]]
    stats = [hostio.parse_stats(p) for p in prefixes]
    reads = os.path.join(GOLDEN, c["reads"])
    batch = hostio.load_reads(reads)
    tot = int(np.diff(batch.off.astype(np.int64)).sum())
    gumbel = list(zip(c["lambda_"], c["K"]))
    return dict(reads=reads, text=open(reads, "rb").read(), batch=batch, prefixes=prefixes, stats=stats,
                refs=[hostio.load_references(os.path.join(GOLDEN, d)) for d in c["dbs"]], minimal_score=c["minimal_score"],
                params=params_kwargs_from_args(c["args"]), gumbel=gumbel,
                ev_params=[hostio.evalue_params(st, k, tot, batch.n) for st, (_, k) in zip(stats, gumbel)])


def assert_pairwise_equal(ours: bytes, theirs: bytes, evalue_rtol: float = 1.2e-2):
    """Byte for byte, except the E-value of each Score line: the reference computes it from the full-precision Gumbel lambda / K,
    while aligned.log, and so the fixtures, hold 6 digits of them (exp(-lambda * S) moves by up to ~1e-3 relative), and it prints 3
    significant digits: there the tolerance is one unit of the last printed digit."""
    a, b = ours.split(b"\n"), theirs.split(b"\n")
    assert len(a) == len(b), (len(a), len(b))
    for k, (x, y) in enumerate(zip(a, b)):
        if x == y:
            continue
        assert x.startswith(b"Score: ") and y.startswith(b"Score: "), (k, x, y)
        fx, fy = x.split(b"\t"), y.split(b"\t")
        assert len(fx) == len(fy) == 3 and fx[0] == fy[0] and fx[2] == fy[2], (k, x, y)
        ex, ey = float(fx[1].split(b" ")[1]), float(fy[1].split(b" ")[1])
        assert abs(ex - ey) <= evalue_rtol * abs(ey) + 1e-300, (k, x, y)
