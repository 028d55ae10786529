"""hostio.otu_map, the plain-Python restatement of the reference's OTU map (fill_otu_map2 / OtuMap::write, otumap.cpp:84-281), on the
oracle's results against what the reference binary wrote (tests/golden/otu_map.json, made by tests/golden/make_otu_golden.py), and
the rounding of fill_otu_map2 (* 0.001) against that of denovo_stats_run (/ 1000.0) at thresholds where the two differ."""
import json
import math
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import params_kwargs_from_args
from oracle import ora
from sortmerna_b200 import hostio

CASES = ["default", "best3", "rev_only", "loose", "none", "parts", "merged"]
# k in 0..1000 for which k * 0.001 is above k / 1000.0 (one ulp): a threshold just above k / 1000.0 separates the two roundings
SPLIT_K = [k for k in range(1001) if k * 0.001 != k / 1000.0]


def load_otu(case):
    with open(os.path.join(GOLDEN, "otu_map.json")) as f:
        return json.load(f)[case]


def oracle_run(golden, golden_parts, case):
    """(results, stats, refs_by_index) of the oracle for a case of otu_map.json"""
    c = load_otu(case)
    b = golden["batch"]
    args = [a for a in c["args"] if a not in ("-m", "0.5")]
    prm = ora.default_params(**params_kwargs_from_args(args))
    ms = c["minimal_score"]
    if case == "parts":
        oix, inum, parts, refs, mss = [], [], [], [], []
        for k, g in enumerate(golden_parts):
            for p in range(g["stats"].num_parts):
                oix.append(ora.OracleIndex(g["prefix"], p, g["stats"].lnwin)); inum.append(k); parts.append(p)
                refs.append(g["part_refs"][p]); mss.append(ms[k])
        out = ora.align(oix, inum, parts, 2, refs, mss, [18, 9, 3] * len(oix), prm, b, nthreads=2)
        by_index = [g["part_refs"] for g in golden_parts]
    elif case == "merged":   # db_bac.fasta as index 0 and as index 1
        oix = [ora.OracleIndex(golden["prefixes"][1], 0, golden["stats"][1].lnwin) for _ in range(2)]
        by_index = [golden["refs"][1], golden["refs"][1]]
        out = ora.align(oix, [0, 1], [0, 0], 2, by_index, ms, [18, 9, 3] * 2, prm, b, nthreads=2)
    else:
        oix = [ora.OracleIndex(p, 0, s.lnwin) for p, s in zip(golden["prefixes"], golden["stats"])]
        by_index = golden["refs"]
        out = ora.align(oix, [0, 1], [0, 0], 2, by_index, ms, [18, 9, 3] * 2, prm, b, nthreads=2)
    st = hostio.host_aln_stats(b, by_index, out["res"], out["alns"], out["cigar"], out["slots"])
    return c, out, st, by_index


@pytest.mark.parametrize("case", CASES)
def test_otu_map_matches_reference(golden, golden_parts, case):
    c, out, st, by_index = oracle_run(golden, golden_parts, case)
    m = hostio.otu_map(by_index, golden["batch"].headers, out["res"], out["alns"], out["slots"], st, c["min_id"], c["min_cov"])
    assert m["n_yid_ycov"] == c["n_yid_ycov"] and m["total_otu"] == c["total_otu"]
    if c["otu_map"] is None:   # the reference writes no file when nothing passes
        assert m["n_yid_ycov"] == 0 and m["text"] == b""
    else:
        assert m["text"].decode() == c["otu_map"]
    if case == "merged":   # lines gather reads of both indexes
        assert any(len(ln.split("\t")) != len(set(ln.split("\t"))) for ln in c["otu_map"].split("\n"))


def _entries(by_index, out, st, min_id, min_cov, scale):
    """(read, slot) of every entry, with the OTU rounding given by scale(x) -- restated from the counters of hostio.denovo_classes"""
    slots = out["slots"]
    cls = hostio.denovo_classes(out["res"], out["alns"], slots, st, min_id, min_cov)
    got = []
    for r in np.nonzero(cls[:, 0] > 0)[0]:
        for a in range(int(out["res"]["n_align"][r])):
            al, s = out["alns"][r * slots + a], st[r * slots + a]
            idv = int(s["n_match_denovo"]) / (int(s["n_miss"]) + int(s["n_gap"]) + int(s["n_match"]))
            cov = abs(int(al["read_end1"]) - int(al["read_begin1"]) + 1) / int(al["readlen"])
            if scale(idv) >= min_id and scale(cov) >= min_cov:
                got.append((int(r), a))
    return got


def test_rounding_boundary(golden, golden_parts):
    """Thresholds nextafter(k / 1000, 1) for k of the 144-value set: an alignment rounded to exactly k / 1000 fails denovo_stats_run's
    test but passes fill_otu_map2's, and joins the map when another alignment of its read makes it count.  hostio.otu_map must take
    those entries, and the golden reads must hold some."""
    c, out, st, by_index = oracle_run(golden, golden_parts, "loose")
    slots = out["slots"]
    ids = set()
    for r in range(out["res"].shape[0]):
        if int(out["res"]["n_align"][r]) > 1:
            for a in range(int(out["res"]["n_align"][r])):
                s = st[r * slots + a]
                ids.add(math.floor(int(s["n_match_denovo"]) / (int(s["n_miss"]) + int(s["n_gap"]) + int(s["n_match"])) * 1000.0 + 0.5))
    ks = sorted(set(SPLIT_K) & ids)
    assert ks, "no alignment of the golden reads rounds to a k of the 144-value set"
    seen = 0
    for k in ks:
        t = math.nextafter(k / 1000.0, 1.0)
        m = hostio.otu_map(by_index, golden["batch"].headers, out["res"], out["alns"], slots, st, t, 0.0)
        otu = _entries(by_index, out, st, t, 0.0, lambda x: math.floor(x * 1000.0 + 0.5) * 0.001)
        div = _entries(by_index, out, st, t, 0.0, lambda x: math.floor(x * 1000.0 + 0.5) / 1000.0)
        assert m["n_yid_ycov"] == len(otu)
        assert set(div) <= set(otu)
        seen += len(otu) - len(div)
    assert seen > 0, "no threshold separated the two roundings"
