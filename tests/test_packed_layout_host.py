"""The packed result layout on the host (no GPU needed): smr_pack_kvdb_blobs_packed on packed copies of the oracle's results gives the
bytes smr_pack_kvdb_blobs gives on the strided ones, for every golden case, all alignments (case_all) included, and for the option
sets of tests/golden/kvdb_blobs.json the committed digests of the reference's serializer.  api.unpack_alns / api.pack_alns
round-trip."""
import hashlib
import json
import os
import struct

import numpy as np
import pytest

from conftest import GOLDEN, case_names, load_case
from helpers import params_kwargs_from_args
from sortmerna_b200 import api, hostio


def _oracle(golden, case):
    from oracle import ora
    exp = load_case(case)
    kw = params_kwargs_from_args(exp["args"])
    oix = [ora.OracleIndex(p, 0, s.lnwin) for p, s in zip(golden["prefixes"], golden["stats"])]
    out = ora.align(oix, [0, 1], [0, 0], 2, golden["refs"], exp["log"]["minimal_score"], [18, 9, 3, 18, 9, 3], ora.default_params(**kw),
                    golden["batch"], nthreads=4)
    return out, kw.get("num_alignments", 1)


def _blobs(out, na, denovo=None):
    buf, off = api.pack_kvdb_blobs(out, na, denovo)
    return [bytes(buf[int(off[r]):int(off[r + 1])]) for r in range(out["res"].shape[0])]


def _digest(blobs):
    return hashlib.sha256(b"".join(struct.pack("<Q", len(b)) + b for b in blobs)).hexdigest()


@pytest.mark.parametrize("case", case_names())
def test_packed_blobs_equal_strided(golden, case):
    out, na = _oracle(golden, case)
    p = api.pack_alns(out)
    assert p["slots"] == 0 and p["alns"].shape[0] == int(out["res"]["n_align"].sum())
    strided = _blobs(out, na)
    assert _blobs(p, na) == strided
    gold = json.load(open(os.path.join(GOLDEN, "kvdb_blobs.json")))
    if f"{case}|None" in gold:
        assert _digest(strided) == gold[f"{case}|None"]["sha256"]
    if case == "all":
        assert int(out["res"]["n_align"].max()) >= 100   # a read past the default stride of 16
    if case == "best3":   # with the denovo counters of the reference's denovo_stats pass (kvdb_blobs.json "None|best3")
        dn = json.load(open(os.path.join(GOLDEN, "denovo.json")))["best3"]
        st = hostio.host_aln_stats(golden["batch"], golden["refs"], out["res"], out["alns"], out["cigar"], out["slots"])
        d4 = hostio.denovo_classes(out["res"], out["alns"], out["slots"], st, dn["min_id"], dn["min_cov"])
        assert _digest(_blobs(p, na, d4)) == gold["None|best3"]["sha256"]


def test_packed_blobs_empty_batch():
    res = np.zeros(3, api.RESULT_DTYPE)
    out = dict(res=res, alns=np.zeros(0, api.ALN_DTYPE), cigar=np.zeros(0, np.uint32), slots=0, aln_off=np.zeros(4, np.uint64))
    buf, off = api.pack_kvdb_blobs(out, 0)
    assert buf.size == 0 and off.tolist() == [0, 0, 0, 0]


def test_unpack_round_trip():
    rng = np.random.default_rng(5)
    n, slots = 200, 7
    res = np.zeros(n, api.RESULT_DTYPE)
    res["n_align"] = rng.integers(0, slots + 1, n)
    res["n_align"][:5] = 0
    alns = np.zeros(n * slots, api.ALN_DTYPE)
    stats = np.zeros(n * slots, api.STATS_DTYPE)
    for r in range(n):
        for k in range(int(res["n_align"][r])):
            alns[r * slots + k]["ref_num"] = 1000 * r + k + 1
            alns[r * slots + k]["score1"] = k + 1
            stats[r * slots + k]["n_match"] = 7 * r + k
    out = dict(res=res, alns=alns, stats=stats, cigar=np.zeros(0, np.uint32), slots=slots)
    p = api.pack_alns(out)
    assert p["aln_off"].tolist() == [0] + np.cumsum(res["n_align"]).tolist()
    assert p["alns"]["ref_num"].tolist() == [1000 * r + k + 1 for r in range(n) for k in range(int(res["n_align"][r]))]
    for s in (slots, slots + 3):
        u = api.unpack_alns(p, s)
        assert u["slots"] == s and "aln_off" not in u
        assert np.array_equal(u["alns"].reshape(n, s)[:, :slots], alns.reshape(n, slots))
        assert np.array_equal(u["stats"].reshape(n, s)[:, :slots], stats.reshape(n, slots))
        assert not u["alns"].reshape(n, s)[:, slots:].view(np.uint8).any()
        back = api.pack_alns(u)
        assert np.array_equal(back["alns"], p["alns"]) and np.array_equal(back["stats"], p["stats"])
    with pytest.raises(ValueError):
        api.unpack_alns(p, int(res["n_align"].max()) - 1)
