"""The denovo_stats pass on the device (smr_denovo_stats, sortmerna_b200/csrc/smr_otu.cuh): per-read counters against
hostio.denovo_classes, totals against the reference's (tests/golden/denovo.json), paired batches against an extended host restatement
and the reference binary, batches, resident text, the KVDB blobs and the refusals."""
import ctypes as C
import hashlib
import json
import math
import os
import re
import shutil
import struct
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, load_denovo
from helpers import params_kwargs_from_args
from integration_common import REF_DIR
from sortmerna_b200 import api, hostio

pytestmark = pytest.mark.gpu

READS = os.path.join(GOLDEN, "reads_mix.fq")
_OPEN = []


@pytest.fixture(autouse=True)
def _close_contexts():
    yield
    while _OPEN:
        _OPEN.pop().close()


def _aligner(golden, args, ms):
    a = api.Aligner(0)
    _OPEN.append(a)
    a.set_params(api.default_params(**params_kwargs_from_args(args)))
    for k in range(2):
        a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], ms[k], (18, 9, 3), golden["stats"][k].lnwin)
    return a


def _case(golden, case):
    c = load_denovo()[case]
    a = _aligner(golden, c["args"], c["minimal_score"])
    b = golden["batch"]
    return a, c, a.align(b.cat, b.off, with_stats=True)


def _text():
    return open(READS, "rb").read()


def _host(out, mid, mcov, **kw):
    return hostio.denovo_classes(out["res"], out["alns"], out["slots"], out["stats"], mid, mcov, **kw)


@pytest.mark.parametrize("case", ["default", "best3", "rev_only", "loose"])
def test_golden_cases(golden, case):
    """per-read counters equal hostio.denovo_classes on the same results; totals equal what the reference counted"""
    a, c, out = _case(golden, case)
    per_read, tot = a.denovo_stats(out, _text(), c["min_id"], c["min_cov"])
    assert np.array_equal(per_read, _host(out, c["min_id"], c["min_cov"]))
    assert [tot[k] for k in api.DENOVO_TOTALS] == c["counts"]
    assert tot["num_denovo"] == c["total_denovo"]
    t = a.report_timings()
    assert t["device_ms"] > 0


def test_threshold_edges(golden):
    """thresholds at nextafter(k / 1000, +-1) around rounded %id and %cov values the golden alignments take"""
    a, c, out = _case(golden, "loose")
    text = _text()
    slots, st, alns = out["slots"], out["stats"], out["alns"]
    ids, covs = set(), set()
    for r in range(out["res"].shape[0]):
        for k in range(int(out["res"]["n_align"][r])):
            s, al = st[r * slots + k], alns[r * slots + k]
            ids.add(math.floor(int(s["n_match_denovo"]) / (int(s["n_miss"]) + int(s["n_gap"]) + int(s["n_match"])) * 1000.0 + 0.5))
            covs.add(math.floor(abs(int(al["read_end1"]) - int(al["read_begin1"]) + 1) / int(al["readlen"]) * 1000.0 + 0.5))
    ks = sorted(ids)[::max(1, len(ids) // 6)][:6]
    kc = sorted(covs)[::max(1, len(covs) // 6)][:6]
    th = [(math.nextafter(k / 1000.0, d), 0.0) for k in ks for d in (0.0, 2.0)] + [(0.0, math.nextafter(k / 1000.0, d)) for k in kc for d in (0.0, 2.0)]
    for mid, mcov in th:
        per_read, tot = a.denovo_stats(out, text, mid, mcov)
        want = _host(out, mid, mcov)
        assert np.array_equal(per_read, want), (mid, mcov)
        assert [tot[k] for k in api.DENOVO_TOTALS] == want.sum(axis=0).tolist()


def test_batches_and_resident_text(golden):
    """three batches give the totals of one; the resident text gives what the text passed gives"""
    a, c, _ = _case(golden, "best3")
    text = _text()
    lines = text.split(b"\n")
    recs = [b"\n".join(lines[i:i + 4]) + b"\n" for i in range(0, len(lines) - 3, 4)]
    cut = [0, len(recs) // 3, 2 * len(recs) // 3, len(recs)]
    a.upload_fastx(text)
    a.run_resident(with_stats=True)
    whole = a.download()
    one_r, one = a.denovo_stats(whole, None, c["min_id"], c["min_cov"])
    passed_r, passed = a.denovo_stats(whole, text, c["min_id"], c["min_cov"])
    assert np.array_equal(one_r, passed_r) and one == passed
    sums, rows = dict.fromkeys(api.DENOVO_TOTALS, 0), []
    for i in range(3):
        t = b"".join(recs[cut[i]:cut[i + 1]])
        a.upload_fastx(t)
        a.run_resident(with_stats=True)
        pr, tot = a.denovo_stats(a.download(), None, c["min_id"], c["min_cov"])
        rows.append(pr)
        for k in sums:
            sums[k] += tot[k]
    assert sums == one and np.array_equal(np.concatenate(rows), one_r)


def test_kvdb_blobs_with_device_counters(golden):
    """blobs packed with the device's counters equal those packed with hostio.denovo_classes, and the committed digest"""
    a, c, out = _case(golden, "best3")
    per_read, _ = a.denovo_stats(out, _text(), c["min_id"], c["min_cov"])
    buf_d, off_d = api.pack_kvdb_blobs(out, 3, per_read)
    buf_h, off_h = api.pack_kvdb_blobs(out, 3, _host(out, c["min_id"], c["min_cov"]))
    assert np.array_equal(off_d, off_h) and np.array_equal(buf_d, buf_h)
    g = json.load(open(os.path.join(GOLDEN, "kvdb_blobs.json")))["None|best3"]
    blobs = [bytes(buf_d[int(off_d[r]):int(off_d[r + 1])]) for r in range(out["res"].shape[0])]
    assert hashlib.sha256(b"".join(struct.pack("<Q", len(b)) + b for b in blobs)).hexdigest() == g["sha256"]


def _paired_text(odd=False, empty=True):
    """the golden mates interleaved; empty: an empty second mate in the first 10 pairs; odd: one more record without its mate"""
    lines = _text().split(b"\n")
    recs = [lines[i:i + 4] for i in range(0, len(lines) - 3, 4) if lines[i].startswith(b"@") and len(lines[i + 1]) >= 18]
    recs = recs[: len(recs) // 2 * 2]
    for k in range(0, 20 if empty else 0, 2):
        recs[k + 1] = [recs[k + 1][0], b"", b"+", b""]
    if odd:
        recs.append(recs[0])
    return b"".join(b"\n".join(r) + b"\n" for r in recs), np.array([len(r[1]) for r in recs])


def _paired_run(golden, text, ms):
    a = _aligner(golden, [], ms)
    a.upload_fastx(text)
    a.run_resident(with_stats=True)
    out = a.download()
    return a, out, a.denovo_stats(out, None, 0.97, 0.97, paired=True)


@pytest.mark.parametrize("odd", [False, True])
def test_paired_empty_second_mate(golden, odd):
    """a pair whose second mate is empty contributes nothing, though its first mate aligns, and so does a last record without its
    mate -- against the extended host restatement"""
    text, lens = _paired_text(odd)
    a, out, (per_read, tot) = _paired_run(golden, text, load_denovo()["default"]["minimal_score"])
    want = _host(out, 0.97, 0.97, paired=True, seq_lens=lens)
    assert np.array_equal(per_read, want) and [tot[k] for k in api.DENOVO_TOTALS] == want.sum(axis=0).tolist()
    single, _ = a.denovo_stats(out, None, 0.97, 0.97)
    skipped = [k for k in range(0, 20, 2) if single[k].sum() > 0]
    assert skipped and all(per_read[k].sum() == 0 for k in skipped)
    if odd:
        assert per_read[-1].sum() == 0 and single[-1].sum() > 0


@pytest.mark.parametrize("odd", [False, True])
def test_paired_against_reference_binary(golden, golden_idx_dir, odd):
    """totals of the reference binary's -paired_in run (-threads 1) on the golden mates interleaved, odd: with one more record
    without its mate, which the reference skips.  The mates hold no read shorter than a seed: such a read, an empty
    one included, sets off a quirk of the reference's paired read feed (integration_common.golden_mates), so the empty-mate rule is
    checked against the host restatement alone"""
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_ref")):
        pytest.skip("oracle/_ref/sortmerna_ref not built (oracle/Makefile.ref)")
    from oracle import ora
    text, lens = _paired_text(odd, empty=False)
    d = tempfile.mkdtemp(prefix="smr_dn_ref_")
    try:
        p = os.path.join(d, "pe.fq")
        open(p, "wb").write(text)
        r = ora.run_reference([os.path.join(GOLDEN, "db_arc.fasta"), os.path.join(GOLDEN, "db_bac.fasta")], p, os.path.join(d, "ref"),
                              extra=["-paired_in", "-otu_map", "-de_novo_otu", "-fastx"], threads=1, idx_dir=golden_idx_dir)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    m = re.search(r"num_yid_ycov: (\d+)\s+num_yid_ncov: (\d+)\s+num_nid_ycov: (\d+)\s+num_denovo: (\d+)", r["stdout"])
    a, out, (per_read, tot) = _paired_run(golden, text, ora.parse_log(r["log"])["minimal_score"])
    assert np.array_equal(per_read, _host(out, 0.97, 0.97, paired=True, seq_lens=lens))
    assert [tot[k] for k in api.DENOVO_TOTALS] == [int(x) for x in m.groups()]


def test_refusals(golden):
    a, c, out = _case(golden, "default")
    text = _text()
    L, h = a.L, a.h
    noo = dict(out)
    del noo["stats"]
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):   # stats required
        a.denovo_stats(noo, text)
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):   # record count
        a.denovo_stats(out, text[: len(text) // 2].rsplit(b"\n@", 1)[0] + b"\n")
    bad = dict(out, alns=out["alns"].copy())
    r = int(np.nonzero(out["res"]["n_align"] > 0)[0][0])
    bad["alns"]["readlen"][r * out["slots"]] += 1
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):   # readlen against the record
        a.denovo_stats(bad, text)
    tot = np.zeros(4, np.uint64)
    o = api.DenovoOpts(0.97, 0.97, 0)
    L.smr_denovo_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                   C.c_void_p, C.c_void_p]
    assert L.smr_denovo_stats(h, C.cast(C.byref(o), C.c_void_p), None, 0, None, None, None, 0, None, None) == 2   # no totals
    assert L.smr_denovo_stats(h, None, None, 0, None, None, None, 0, None, api._ptr(tot)) == 2                     # no opts
    # the context still works
    per_read, t = a.denovo_stats(out, text, c["min_id"], c["min_cov"])
    assert [t[k] for k in api.DENOVO_TOTALS] == c["counts"]
