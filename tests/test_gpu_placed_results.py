"""Results placed on the device (smr_place_results, smr_download_placed and the _placed report calls): the placed arrays equal what
smr_download_results writes, byte for byte, on every golden case, under an index budget of several groups and with scratch-overflow
retries; every _placed report call gives the streams of its host-array twin; and the refusals."""
import gzip
import os
import shutil
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, case_names, load_case
from helpers import params_kwargs_from_args
from integration_common import golden_mates
from sortmerna_b200 import api, hostio

pytestmark = pytest.mark.gpu

TEXT = os.path.join(GOLDEN, "reads_mix.fq")


def _aligner(golden, ms, **kw):
    al = api.Aligner(0)
    al.set_params(api.default_params(**kw))
    for k in range(2):
        al.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], ms[k], (18, 9, 3), golden["stats"][k].lnwin)
    return al


def _assert_placed_equals_download(al):
    """run_resident(with_stats) + place() against download() of the same run, byte for byte; returns the placed results"""
    info = al.place()
    want = al.download()
    got = al.download_placed(with_stats=True)
    assert got["slots"] == want["slots"] == info["slots"]
    for k in ("res", "alns", "cigar", "stats"):
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), k
    assert info["counters"] == want["counters"]
    assert np.array_equal(info["matched"], want["matched"])
    assert info["n_alns"] == want["alns"].size and info["cigar_words"] == want["cigar"].size
    return got


def _run(al, stats=True):
    al.set_place_stats(stats)
    al.run_resident(with_stats=stats)


@pytest.mark.parametrize("name", case_names())
def test_placed_equals_download_on_golden_cases(golden, name):
    exp = load_case(name)
    al = _aligner(golden, exp["log"]["minimal_score"], **params_kwargs_from_args(exp["args"]))
    try:
        if al.params.num_alignments == 0:
            al.set_aln_slots(1)   # place() grows the stride to what the library names and runs the batch again
        al.upload_fastx(open(TEXT, "rb").read())
        al.set_place_stats(True)
        al.run_resident()
        first = al.place()
        _run(al)   # the stride is final now: the host download of the same run has its stats buffer at that stride
        got = _assert_placed_equals_download(al)
        if name == "all":
            assert first["slots"] > 1 and int(got["res"]["n_align"].max()) > 1
        assert first["counters"]["num_aligned"] == exp["log"]["passing"]
    finally:
        al.close()


def test_download_after_a_placement_that_grew_the_stride(golden):
    """run_resident(with_stats=True) at stride 1, place() growing the stride and running the batch again, then download() of that
    run with its stats: the host stats buffer follows the stride"""
    exp = load_case("all")
    al = _aligner(golden, exp["log"]["minimal_score"], **params_kwargs_from_args(exp["args"]))
    try:
        al.set_aln_slots(1)
        al.upload_fastx(open(TEXT, "rb").read())
        _run(al)
        info = al.place()
        assert info["slots"] > 1
        want = al.download()
        got = al.download_placed(with_stats=True)
        assert want["stats"].size == got["stats"].size == info["n_alns"]
        for k in ("res", "alns", "cigar", "stats"):
            assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), k
        assert info["counters"] == want["counters"]
    finally:
        al.close()


def test_placed_under_an_index_budget(golden):
    exp = load_case("default")
    al = _aligner(golden, exp["log"]["minimal_score"])
    try:
        total = al.index_residency()["device_search_bytes"]
        al.set_index_budget(total - 1)
        assert al.index_residency()["groups"] == 2
        al.upload_fastx(open(TEXT, "rb").read())
        _run(al)
        _assert_placed_equals_download(al)
    finally:
        al.close()


# -- reads that overflow their seed-lane scratch at scale 1: the exact 18-mer core between the flanks of references that hold every
# one-edit variant of it (more ids in one window than the 128 of the per-lane buffer), among ordinary reads
L = 18
ACGT = np.frombuffer(b"ACGT", np.uint8)


def _variants(core):
    out = set()
    for i in range(L):
        for b in range(4):
            if b != core[i]:
                v = core.copy(); v[i] = b; out.add(v.tobytes())
            out.add(np.concatenate([core[:i], [b], core[i:]]).astype(np.uint8).tobytes())
        out.add(np.concatenate([core[:i], core[i + 1:]]).astype(np.uint8).tobytes())
    out.discard(core.tobytes())
    return [np.frombuffer(v, np.uint8) for v in sorted(out)]


def _overflow_inputs(d):
    rng = np.random.default_rng(20261018)
    core = rng.integers(0, 4, L, dtype=np.uint8)
    refs, flanks = [], []
    for v in _variants(core):
        for c in range(4):
            a, b = rng.integers(0, 4, 60, dtype=np.uint8), rng.integers(0, 4, 60, dtype=np.uint8)
            a[-1], b[0] = (c + 1) & 3, c
            s = np.concatenate([a, v, b])
            if core.tobytes() not in s.tobytes():
                refs.append(s)
                flanks.append((a, b))
    plain = [rng.integers(0, 4, 2000, dtype=np.uint8) for _ in range(20)]
    fasta = os.path.join(d, "neigh.fasta")
    with open(fasta, "wb") as f:
        for k, s in enumerate(refs + plain):
            f.write(b">n%05d\n" % k + ACGT[s].tobytes() + b"\n")
    reads = []
    for k in range(300):
        p = plain[k % 20]
        o = int(rng.integers(0, p.size - 150))
        s = p[o:o + 150].copy()
        s[rng.integers(0, 150, 2)] = rng.integers(0, 4, 2)
        reads.append(s)
    for k in rng.choice(len(flanks), 6, replace=False):
        a, b = flanks[k]
        reads.insert(int(rng.integers(0, len(reads))), np.concatenate([a, core, b[:72]]))
    fq = os.path.join(d, "reads.fq")
    with open(fq, "wb") as f:
        for i, s in enumerate(reads):
            f.write(b"@q%d\n" % i + ACGT[s].tobytes() + b"\n+\n" + b"I" * s.size + b"\n")
    return fasta, fq


def test_placed_with_scratch_overflow_retries(capfd):
    d = tempfile.mkdtemp(prefix="smr_place_ovf_")
    al = api.Aligner(0)
    try:
        fasta, fq = _overflow_inputs(d)
        al.set_params(api.default_params())
        al.build_index_device(0, fasta, hostio.load_references(fasta), 60)
        al.upload_fastx(open(fq, "rb").read())
        os.environ["SMR_VERBOSE"] = "1"
        try:
            _run(al)
            capfd.readouterr()
            got = _assert_placed_equals_download(al)
        finally:
            del os.environ["SMR_VERBOSE"]
        err = capfd.readouterr().err
        assert "reads overflowed their scratch at scale 1" in err, err[-2000:]
        assert int(got["res"]["is_hit"].sum()) > 0
    finally:
        al.close()
        shutil.rmtree(d, ignore_errors=True)


def test_placed_with_scratch_overflow_retries_in_sub_batches(monkeypatch, capfd):
    """the same reads with sub-batches of 2 slots: the retries run as several batches, and the placement writes their CIGARs in the
    order the download does"""
    d = tempfile.mkdtemp(prefix="smr_place_ovf_")
    monkeypatch.setenv("SMR_RETRY_SLOTS", "2")   # read when the context is made
    al = api.Aligner(0)
    try:
        fasta, fq = _overflow_inputs(d)
        al.set_params(api.default_params())
        al.build_index_device(0, fasta, hostio.load_references(fasta), 60)
        al.upload_fastx(open(fq, "rb").read())
        monkeypatch.setenv("SMR_VERBOSE", "1")
        _run(al)
        capfd.readouterr()
        al.place()
        placed = capfd.readouterr().err
        got = _assert_placed_equals_download(al)   # place() finds the placement made; download() retries the same reads
        downloaded = capfd.readouterr().err
        monkeypatch.delenv("SMR_VERBOSE")
        line = "reads overflowed their scratch at scale 1: retrying"
        assert placed.count(line) > 1 and downloaded.count(line) == placed.count(line), placed[-2000:]
        assert int(got["res"]["is_hit"].sum()) > 0
    finally:
        al.close()
        shutil.rmtree(d, ignore_errors=True)


# -- the report side: each _placed call against its host-array twin
GUMBEL = [(0.594908, 0.326193), (0.600371, 0.328947)]


def _scored(golden, ms, **kw):
    al = _aligner(golden, ms, **kw)
    tot = int(np.diff(golden["batch"].off.astype(np.int64)).sum())
    for k, (lam, K) in enumerate(GUMBEL):
        al.set_report_scoring(k, lam, K, *hostio.evalue_params(golden["stats"][k], K, tot, golden["batch"].n))
    return al


def _both(al, fn, **kw):
    """fn(out, **kw) with the host arrays of download() and fn(None, **kw) with the placed results"""
    al.place()
    out = al.download()
    return fn(out, **kw), fn(None, **kw)


@pytest.mark.parametrize("gz", [False, True])
def test_placed_reports_equal_host_arrays(golden, gz):
    exp = load_case("default")
    al = _scored(golden, exp["log"]["minimal_score"])
    try:
        al.upload_fastx(open(TEXT, "rb").read())
        _run(al)
        opts = api.report_opts(sam=True, blast="1 cigar qcov qstrand", fastx=True, other=True, denovo=(0.9, 0.9))
        a, b = _both(al, al.format_reports, opts=opts, gzip=gz)
        assert a == b and a["sam"][0] and a["blast"][1] and a["aligned"] and a["other"]
        if gz:
            assert gzip.decompress(a["sam"][0]).count(b"\n") > 0
        a, b = _both(al, al.format_blast_pairwise, gzip=gz)
        assert a == b and a[0]
        a, b = _both(al, al.denovo_stats, min_id=0.9, min_cov=0.9)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[1]["n_yid_ycov"] > 0
        al.otu_begin(0.9, 0.9)
        n_host = al.otu_add(al.download())
        host_map = al.otu_finish()
        al.otu_begin(0.9, 0.9)
        assert al.otu_add(None) == n_host > 0
        assert al.otu_finish() == host_map
    finally:
        al.close()


@pytest.mark.parametrize("extra", [dict(paired_in=True), dict(out2=True), dict(sout=True), dict(paired_in=True, out2=True)])
def test_placed_read_files_on_a_mate_stream(golden, tmp_path, extra):
    exp = load_case("default")
    al = _scored(golden, exp["log"]["minimal_score"])
    try:
        r1, r2 = golden_mates(str(tmp_path))
        n = 0
        for _ in al.stream_mates(r1, r2, batch_bytes=20000, piece_bytes=4096):
            _run(al)
            opts = api.report_opts(fastx=True, other=True, sam=True, denovo=(0.9, 0.9), **extra)
            a, b = _both(al, al.format_reports, opts=opts)
            assert a == b
            a, b = _both(al, al.denovo_stats, min_id=0.9, min_cov=0.9, paired=True)
            assert np.array_equal(a[0], b[0]) and a[1] == b[1]
            n += 1
        assert n >= 3
    finally:
        al.close()


def test_refusals(golden):
    exp = load_case("default")
    al = _aligner(golden, exp["log"]["minimal_score"])
    text = open(TEXT, "rb").read()
    opts = api.report_opts(fastx=True)
    try:
        al.upload_fastx(text)
        with pytest.raises(api.SmrError, match="SMR_ERR_ARG.*not been run"):   # nothing run yet
            al.place()
        al.set_place_stats(False)
        al.run_resident()
        with pytest.raises(api.SmrError, match="SMR_ERR_ARG.*no placed results"):   # run, not placed
            al.format_reports(None, opts=opts)
        al.place()
        assert al.format_reports(None, opts=opts)["aligned"]
        with pytest.raises(api.SmrError, match="SMR_ERR_ARG.*no smr_aln_stats"):   # SAM reads stats this placement lacks
            al.format_reports(None, opts=api.report_opts(sam=True))
        al.run_resident()   # a new run: the placement of the earlier one is refused
        with pytest.raises(api.SmrError, match="SMR_ERR_ARG.*no placed results"):
            al.format_reports(None, opts=opts)
        al.place()
        al.upload_fastx(text)   # a new batch
        with pytest.raises(api.SmrError, match="SMR_ERR_ARG.*no placed results"):
            al.denovo_stats(None)
        with pytest.raises(api.SmrError, match="SMR_ERR_ARG.*no placed results"):
            al.format_blast_pairwise(None)
        al.set_aln_layout("packed")
        al.run_resident()
        with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED.*strided layout only"):
            al.place()
        with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED.*strided layout only"):
            al.format_reports(None, opts=opts)
    finally:
        al.close()
