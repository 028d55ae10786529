"""The OTU map on the device (smr_otu_begin / smr_otu_add / smr_otu_finish, sortmerna_b200/csrc/smr_otu.cuh): otu_map.txt and the two
OTU numbers of aligned.log against the reference binary's stored output (tests/golden/otu_map.json), hostio.otu_map on the same results
and, where it is built, the reference binary itself."""
import ctypes as C
import gzip
import math
import os
import shutil
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import params_kwargs_from_args
from integration_common import REF_DIR
from sortmerna_b200 import api, hostio
from test_otu_map_host import CASES, SPLIT_K, load_otu

pytestmark = pytest.mark.gpu

READS = os.path.join(GOLDEN, "reads_mix.fq")
_OPEN = []


@pytest.fixture(autouse=True)
def _close_contexts():
    """a failing test must not leave its context (and its device memory) to the next"""
    yield
    while _OPEN:
        _OPEN.pop().close()


@pytest.fixture(scope="module")
def otu_setups(golden, golden_parts):
    """per case of otu_map.json: how to load its indexes -- [(index_num, part, prefix, refs, lnwin)], refs_by_index"""
    out = {}
    for case in CASES:
        if case == "parts":
            loads = [(k, p, g["prefix"], g["part_refs"][p], g["stats"].lnwin) for k, g in enumerate(golden_parts) for p in range(g["stats"].num_parts)]
            out[case] = (loads, [g["part_refs"] for g in golden_parts])
        elif case == "merged":   # db_bac.fasta as index 0 and as index 1
            loads = [(k, 0, golden["prefixes"][1], golden["refs"][1], golden["stats"][1].lnwin) for k in range(2)]
            out[case] = (loads, [golden["refs"][1]] * 2)
        else:
            loads = [(k, 0, golden["prefixes"][k], golden["refs"][k], golden["stats"][k].lnwin) for k in range(2)]
            out[case] = (loads, golden["refs"])
    return out


def _aligner(otu_setups, case, **kw):
    c = load_otu(case)
    a = api.Aligner(0)
    _OPEN.append(a)
    a.set_params(api.default_params(**{**params_kwargs_from_args([x for x in c["args"] if x not in ("-m", "0.5")]), **kw}))
    loads, by_index = otu_setups[case]
    for (k, p, prefix, refs, lnwin) in loads:
        a.load_index_part(k, p, prefix, refs, c["minimal_score"][k], (18, 9, 3), lnwin)
    for k, r in enumerate(by_index):
        a.refs_by_index[k] = r
    return a, c, by_index


def _text():
    return open(READS, "rb").read()


def _otu(a, out, text, min_id, min_cov):
    a.otu_begin(min_id, min_cov)
    a.otu_add(out, text)
    return a.otu_finish()


@pytest.mark.parametrize("case", CASES)
def test_golden_cases(golden, otu_setups, case):
    """otu_map.txt byte-identical to the reference's, Total OTUs and n_yid_ycov equal; no map where the reference wrote none"""
    a, c, _ = _aligner(otu_setups, case)
    b = golden["batch"]
    out = a.align(b.cat, b.off, with_stats=True)
    m = _otu(a, out, _text(), c["min_id"], c["min_cov"])
    assert m["total_otu"] == c["total_otu"] and m["n_yid_ycov"] == c["n_yid_ycov"]
    assert m["text"] == (c["otu_map"].encode() if c["otu_map"] is not None else b"")


@pytest.mark.parametrize("case", ["default", "best3", "loose", "parts", "merged"])
def test_equals_host(golden, otu_setups, case):
    """byte-identical to hostio.otu_map on the same results, at the case's thresholds and at nextafter(k / 1000, 1) for k where
    fill_otu_map2's * 0.001 and denovo_stats_run's / 1000.0 differ"""
    a, c, by_index = _aligner(otu_setups, case)
    b = golden["batch"]
    out = a.align(b.cat, b.off, with_stats=True)
    text = _text()
    thresholds = [(c["min_id"], c["min_cov"]), (0.0, 0.0)]
    thresholds += [(math.nextafter(k / 1000.0, 1.0), 0.0) for k in SPLIT_K if 850 <= k <= 1000]
    thresholds += [(0.0, math.nextafter(k / 1000.0, 1.0)) for k in SPLIT_K if 850 <= k <= 1000][::3]
    for mid, mcov in thresholds:
        m = _otu(a, out, text, mid, mcov)
        h = hostio.otu_map(by_index, b.headers, out["res"], out["alns"], out["slots"], out["stats"], mid, mcov)
        assert m == h, (mid, mcov)


def test_multi_batch_equals_one_batch(golden, otu_setups, tmp_path):
    """ReportWriter(otu_map=...): the golden reads in 3 batches write the otu_map.txt one batch writes, and the reference's"""
    a, c, _ = _aligner(otu_setups, "best3")
    lines = _text().split(b"\n")
    recs = [b"\n".join(lines[i:i + 4]) + b"\n" for i in range(0, len(lines) - 3, 4)]
    cut = [0, len(recs) // 3, 2 * len(recs) // 3, len(recs)]
    res = {}
    for name, pieces in (("one", [recs]), ("three", [recs[cut[i]:cut[i + 1]] for i in range(3)])):
        w = api.ReportWriter(str(tmp_path / name), a, otu_map=(c["min_id"], c["min_cov"]), fastx=True)
        for p in pieces:
            text = b"".join(p)
            a.upload_fastx(text)
            a.run_resident(with_stats=True)
            w.write(a.download(), text)
        files = {os.path.basename(f): open(f, "rb").read() for f in w.close()}
        res[name] = (files, w.total_otu, w.n_yid_ycov)
    assert sorted(res["one"][0]) == ["aligned.fq", "otu_map.txt"]
    assert res["three"] == res["one"]
    assert res["one"][0]["otu_map.txt"] == c["otu_map"].encode()
    assert (res["one"][1], res["one"][2]) == (c["total_otu"], c["n_yid_ycov"])


def test_no_file_when_nothing_passes(golden, otu_setups, tmp_path):
    a, c, _ = _aligner(otu_setups, "none")
    b = golden["batch"]
    w = api.ReportWriter(str(tmp_path), a, otu_map=(c["min_id"], c["min_cov"]))
    w.write(a.align(b.cat, b.off, with_stats=True), _text())
    assert w.close() == [] and not os.path.exists(tmp_path / "otu_map.txt")
    assert (w.total_otu, w.n_yid_ycov) == (0, 0)


@pytest.mark.parametrize("source", ["fastx", "fastx_gz"])
def test_resident_text(golden, otu_setups, source):
    """the resident text of upload_fastx / upload_fastx_gz gives what the text passed in gives"""
    a, c, _ = _aligner(otu_setups, "loose")
    text = _text()
    if source == "fastx":
        a.upload_fastx(text)
    else:
        a.upload_fastx_gz(gzip.compress(text, 6))
    a.run_resident(with_stats=True)
    out = a.download()
    resident = _otu(a, out, None, c["min_id"], c["min_cov"])
    passed = _otu(a, out, text, c["min_id"], c["min_cov"])
    assert resident == passed and resident["text"] == c["otu_map"].encode()


def _fasta_multiline(fq: bytes) -> bytes:
    lines = fq.split(b"\n")
    out = []
    for i in range(0, len(lines) - 3, 4):
        s = lines[i + 1]
        out.append(b">" + lines[i][1:] + b" some description\n" + b"".join(s[k:k + 60] + b"\n" for k in range(0, len(s), 60)))
    return b"".join(out)


@pytest.mark.parametrize("shape", ["fastq", "fasta_multiline"])
def test_against_reference_binary(golden, golden_idx_dir, shape):
    """otu_map.txt byte-identical to the reference binary's (-threads 1) on the same reads against both golden databases"""
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_ref")):
        pytest.skip("oracle/_ref/sortmerna_ref not built (oracle/Makefile.ref)")
    from oracle import ora
    d = tempfile.mkdtemp(prefix="smr_otu_ref_")
    try:
        text = _text() if shape == "fastq" else _fasta_multiline(_text())
        reads = os.path.join(d, "reads." + ("fq" if shape == "fastq" else "fasta"))
        open(reads, "wb").write(text)
        fastas = [os.path.join(GOLDEN, "db_arc.fasta"), os.path.join(GOLDEN, "db_bac.fasta")]
        r = ora.run_reference(fastas, reads, os.path.join(d, "ref"), extra=["-fastx", "-otu_map", "-num_alignments", "2", "-id", "0.9", "-coverage", "0.8"],
                              threads=1, idx_dir=golden_idx_dir)
        want = open(os.path.join(r["out_dir"], "otu_map.txt"), "rb").read()
        log = ora.parse_log(r["log"])
        a = api.Aligner(0)
        _OPEN.append(a)
        a.set_params(api.default_params(num_alignments=2))
        for k in range(2):
            a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], log["minimal_score"][k], (18, 9, 3), golden["stats"][k].lnwin)
        a.upload_fastx(text)
        a.run_resident(with_stats=True)
        m = _otu(a, a.download(), None, 0.9, 0.8)
        assert m["text"] == want and len(want) > 1000
        assert f"Total OTUs = {m['total_otu']}" in r["log"]
    finally:
        shutil.rmtree(d, ignore_errors=True)


def test_refusals(golden, otu_setups, tmp_path):
    a, c, _ = _aligner(otu_setups, "default")
    b = golden["batch"]
    out = a.align(b.cat, b.off, with_stats=True)
    text = _text()
    # no begin yet
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):
        a.otu_add(out, text)
    # a part without smr_set_report_refs
    o = api.OtuOpts(0.97, 0.97, 0, 0)
    assert a.L.smr_otu_begin(a.h, C.byref(o)) == 2
    # paired batches
    for kw in ({"paired_in": True}, {"paired_out": True}):
        with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED"):
            a.otu_begin(0.97, 0.97, **kw)
    with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED"):
        api.ReportWriter(str(tmp_path), a, otu_map=(0.97, 0.97), paired_in=True)
    # too small an output buffer: SMR_ERR_CAPACITY with the counts; the accumulator is kept and a retry succeeds
    a.otu_begin(c["min_id"], c["min_cov"])
    a.otu_add(out, text)
    counts = np.zeros(3, np.uint64)
    small = np.zeros(16, np.uint8)
    assert a.L.smr_otu_finish(a.h, api._ptr(small), C.c_uint64(small.size), api._ptr(counts)) == 5
    assert counts.tolist() == [len(c["otu_map"]), c["total_otu"], c["n_yid_ycov"]]
    assert a.otu_finish()["text"] == c["otu_map"].encode()
    # a part loaded between begin and finish
    a.otu_begin(c["min_id"], c["min_cov"])
    a.otu_add(out, text)
    a.load_index_part(2, 0, golden["prefixes"][0], golden["refs"][0], c["minimal_score"][0], (18, 9, 3), golden["stats"][0].lnwin)
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):
        a.otu_add(out, text)
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):
        a.otu_finish()
    # -no-best
    n = api.Aligner(0)
    _OPEN.append(n)
    n.set_params(api.default_params(is_best=0, num_alignments=2))
    n.load_index_part(0, 0, golden["prefixes"][0], golden["refs"][0], c["minimal_score"][0], (18, 9, 3), golden["stats"][0].lnwin)
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):
        n.otu_begin()
