"""Packed results placed on the device (smr_place_results_packed, Aligner.place_packed): the first run stays on the device, the reads
that outgrow its stride run again and stay there too, and one count pass, two scans and a warp-per-read scatter place every read.
Checked here:
- every golden case, and case_all at first-run strides 1, 2 and 16: the placement equals api.pack_alns of the strided download at
  the grown stride, byte for byte;
- the near-copy database (up to about 1,600 alignments per read) in sub-batches, reads that overflow their scratch as well as the
  stride, and an index budget of two groups: equal to the oracle, the strided results and the run without a budget;
- every packed _placed report call against its host-array twin;
- the contracts: one placement per run, a packed download that copies it, invalidation, the refusals;
- api.run_files at -num_alignments 0, which runs packed: its files equal what ReportWriter writes from the strided results."""
import ctypes as C
import os
import re
import shutil
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, case_names, load_case
from helpers import assert_same_results, params_kwargs_from_args
from integration_common import golden_mates
from sortmerna_b200 import api, hostio
from test_gpu_packed_results import MS, both_overflow_inputs, near_copy_inputs, near_copy_oracle

pytestmark = pytest.mark.gpu

READS = os.path.join(GOLDEN, "reads_mix.fq")
BLAST = "1 cigar qcov qstrand"
RERUN = re.compile(r"packed results: (\d+) reads stored more than (\d+) alignments and were run again at their own count in (\d+) sub-batches")
GUMBEL = [(0.594908, 0.326193), (0.600371, 0.328947)]

_OPEN = []


@pytest.fixture(autouse=True)
def _close_contexts():
    yield
    while _OPEN:
        _OPEN.pop().close()


def _golden_aligner(golden, exp, layout="strided", slots=None, track=True):
    a = api.Aligner(0)
    if track:
        _OPEN.append(a)
    a.set_params(api.default_params(**params_kwargs_from_args(exp["args"])))
    tot = int(np.diff(golden["batch"].off.astype(np.int64)).sum())
    for k in range(2):
        a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], exp["log"]["minimal_score"][k], (18, 9, 3), golden["stats"][k].lnwin)
        a.set_report_scoring(k, *GUMBEL[k], *hostio.evalue_params(golden["stats"][k], GUMBEL[k][1], tot, golden["batch"].n))
    a.set_aln_layout(layout)
    if slots:
        a.set_aln_slots(slots)
    return a


def _placed(a, cat=None, off=None, text=None):
    """upload, run_resident, place_packed, download_placed: (the placed arrays, place_packed's dict)"""
    if text is not None:
        a.upload_fastx(text)
    else:
        a.upload(cat, off)
    a.run_resident(with_stats=True)
    info = a.place_packed()
    return a.download_placed(with_stats=True), info


def _words(out):
    """the CIGAR words of every alignment of a packed result, in its order"""
    a = out["alns"]
    n = a["cigar_len"].astype(np.int64)
    at = np.repeat(a["cigar_off"].astype(np.int64) - np.concatenate([[0], np.cumsum(n)[:-1]]), n) + np.arange(int(n.sum()))
    return np.asarray(out["cigar"])[at]


def assert_placed_equals_strided(p, info, s, what):
    """the packed placement against the strided download at its grown stride, packed by api.pack_alns: results, stats and aln_off
    byte for byte, the alignments byte for byte but for cigar_off, and the same CIGAR words per alignment.  The placement's CIGARs
    are compacted in read order; the strided download's follow read order too, except that the reads a scratch-overflow retry ran
    come after the others."""
    q = api.pack_alns(s)
    assert p["slots"] == 0 and info["slots"] == 0, what
    for k in ("res", "stats", "aln_off"):
        assert np.asarray(p[k]).tobytes() == np.asarray(q[k]).tobytes(), (what, k)
    x, y = p["alns"].copy(), q["alns"].copy()
    n = x["cigar_len"].astype(np.uint64)
    assert x["cigar_off"].tolist() == np.concatenate([[0], np.cumsum(n)[:-1]]).astype(np.uint64).tolist(), what   # read order
    x["cigar_off"] = y["cigar_off"] = 0
    assert x.tobytes() == y.tobytes(), (what, "alns")
    assert p["cigar"].size == int(n.sum()) and np.array_equal(p["cigar"], _words(q)), (what, "cigar")
    assert info["n_alns"] == p["alns"].shape[0] and info["cigar_words"] == p["cigar"].size, what
    assert info["counters"]["num_aligned"] == s["counters"]["num_aligned"], what
    assert info["matched"].tolist() == s["matched"].tolist(), what


# ---- 1. golden cases ----
@pytest.mark.parametrize("case", case_names())
def test_golden_cases_placed_equal_strided(golden, case):
    exp = load_case(case)
    b = golden["batch"]
    s = _golden_aligner(golden, exp).align(b.cat, b.off, with_stats=True)
    p, info = _placed(_golden_aligner(golden, exp, "packed"), b.cat, b.off)
    assert_placed_equals_strided(p, info, s, case)
    assert info["counters"]["num_aligned"] == exp["log"]["passing"]


@pytest.mark.parametrize("stride", [1, 2, 16])
def test_case_all_first_strides_placed_equal_strided(golden, stride, capfd, monkeypatch):
    exp = load_case("all")
    b = golden["batch"]
    s = _golden_aligner(golden, exp).align(b.cat, b.off, with_stats=True)
    monkeypatch.setenv("SMR_VERBOSE", "1")
    capfd.readouterr()
    p, info = _placed(_golden_aligner(golden, exp, "packed", stride), b.cat, b.off)
    runs = RERUN.findall(capfd.readouterr().err)
    assert len(runs) == 1 and int(runs[0][0]) == int((s["res"]["n_align"] > stride).sum()) > 0 and int(runs[0][1]) == stride
    assert_placed_equals_strided(p, info, s, f"stride {stride}")
    assert info["place_ms"] > 0


# ---- 2. near copies, both overflows, an index budget ----
@pytest.fixture(scope="module")
def near_copies():
    d = tempfile.mkdtemp(prefix="smr_placed_packed_")
    yield near_copy_inputs(d)
    shutil.rmtree(d, ignore_errors=True)


@pytest.fixture(scope="module")
def near_oracle(near_copies):
    return near_copy_oracle(near_copies)


def _near_aligner(nc, layout):
    a = api.Aligner(0)
    _OPEN.append(a)
    a.set_params(api.default_params(num_alignments=0))
    a.load_index_part(0, 0, nc["prefix"], nc["refs"], MS, (18, 9, 3), nc["stats"].lnwin)
    a.set_aln_layout(layout)
    return a


def test_near_copies_placed_equal_oracle_and_strided(near_copies, near_oracle, capfd, monkeypatch):
    nc, b = near_copies, near_copies["batch"]
    cnt = near_oracle["res"]["n_align"]
    s = _near_aligner(nc, "strided").align(b.cat, b.off, with_stats=True)
    monkeypatch.setenv("SMR_VERBOSE", "1")
    monkeypatch.setenv("SMR_RETRY_SLOTS", "1000")   # read at smr_init: sub-batches of the small group, the large group's reads alone
    capfd.readouterr()
    p, info = _placed(_near_aligner(nc, "packed"), b.cat, b.off)
    runs = RERUN.findall(capfd.readouterr().err)
    assert len(runs) == 1 and int(runs[0][0]) == int((cnt > 16).sum()) and int(runs[0][2]) >= int((cnt > 1000).sum()) + 2
    assert int(p["res"]["n_align"].max()) >= 1500
    assert_same_results(api.unpack_alns(p, near_oracle["slots"]), near_oracle, "near copies")
    assert info["matched"].tolist() == near_oracle["matched"].tolist()
    assert info["counters"]["num_aligned"] == near_oracle["counters"]["num_aligned"]
    assert_placed_equals_strided(p, info, s, "near copies")


def test_scratch_and_slot_overflow_placed_equal_oracle(tmp_path, capfd, monkeypatch):
    nc = both_overflow_inputs(str(tmp_path))
    want = near_copy_oracle(nc)
    b = nc["batch"]
    monkeypatch.setenv("SMR_VERBOSE", "1")
    capfd.readouterr()
    p, info = _placed(_near_aligner(nc, "packed"), b.cat, b.off)
    err = capfd.readouterr().err
    assert "overflowed their scratch" in err and RERUN.search(err)
    assert_same_results(api.unpack_alns(p, want["slots"]), want, "scratch and slots")
    assert info["matched"].tolist() == want["matched"].tolist()
    assert info["counters"]["num_aligned"] == want["counters"]["num_aligned"]
    # the packed download of the same aligner equals the placement
    d = _near_aligner(nc, "packed").align(b.cat, b.off, with_stats=True)
    for k in ("res", "alns", "stats", "cigar", "aln_off"):
        assert np.asarray(p[k]).tobytes() == np.asarray(d[k]).tobytes(), k


def test_placed_under_an_index_budget(golden):
    exp = load_case("all")
    b = golden["batch"]
    want, winfo = _placed(_golden_aligner(golden, exp, "packed", 4), b.cat, b.off)
    a = _golden_aligner(golden, exp, "packed", 4)
    a.set_index_budget(a.index_residency()["device_search_bytes"] - 1)
    assert a.index_residency()["groups"] == 2
    got, ginfo = _placed(a, b.cat, b.off)
    for k in ("res", "alns", "stats", "cigar", "aln_off"):
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), k
    assert ginfo["counters"]["num_aligned"] == winfo["counters"]["num_aligned"] and ginfo["matched"].tolist() == winfo["matched"].tolist()


# ---- 3. every packed _placed call against its host-array twin ----
def _twins(a, text, opts):
    """the _placed calls after place_packed() against the same calls given the packed download of the same run"""
    a.place_packed()
    out = a.download()
    assert out["slots"] == 0
    for gz in (False, True):
        x, y = a.format_reports(None, opts=opts, gzip=gz), a.format_reports(out, text, opts=opts, gzip=gz)
        assert x == y, (gz, "format_reports")
        buf, so = a.format_placed_into(opts, np.zeros(16, np.uint8), gz)   # grown to the size the library names
        groups = a.report_groups()
        assert api.Aligner._report_streams(buf, so, len(groups), api.num_out_of(opts), groups) == y, (gz, "format_placed_into")
    po = api.report_opts(blast="0", paired_in=opts.paired_in, mates=opts.mates)
    for gz in (False, True):
        assert a.format_blast_pairwise(None, opts=po, gzip=gz) == a.format_blast_pairwise(out, text, opts=po, gzip=gz), gz
    paired = bool(opts.paired_in or opts.mates)
    dx, dy = a.denovo_stats(None, min_id=0.9, min_cov=0.9, paired=paired), a.denovo_stats(out, text, 0.9, 0.9, paired=paired)
    assert np.array_equal(dx[0], dy[0]) and dx[1] == dy[1]
    assert a.denovo_stats(None, min_id=0.9, min_cov=0.9, paired=paired, per_read=False) == (None, dy[1])
    feed = "two_files" if opts.mates else "one_file" if opts.paired_in else None
    a.otu_begin(0.9, 0.9, paired_in=bool(opts.paired_in), feed=feed)
    n_host = a.otu_add(out, text)
    host_map = a.otu_finish()
    a.otu_begin(0.9, 0.9, paired_in=bool(opts.paired_in), feed=feed)
    assert a.otu_add(None) == n_host
    assert a.otu_finish() == host_map
    return out


def test_placed_reports_equal_host_arrays_case_all(golden):
    exp = load_case("all")
    a = _golden_aligner(golden, exp, "packed", 4)
    text = open(READS, "rb").read()
    a.upload_fastx(text)
    a.run_resident(with_stats=True)
    out = _twins(a, text, api.report_opts(sam=True, blast=BLAST, fastx=True, other=True, denovo=(0.9, 0.9)))
    assert int(out["res"]["n_align"].max()) > 4
    a.upload_fastx(text)
    a.run_resident(with_stats=True)
    a.place_packed()
    r = a.format_reports(None, sam=True)
    assert sum(g.count(b"\n") for g in r["sam"]) == 5497


def test_placed_reports_on_a_mate_stream(golden, tmp_path):
    exp = load_case("all")
    a = _golden_aligner(golden, exp, "packed", 2)
    r1, r2 = golden_mates(str(tmp_path))
    n = 0
    for _ in a.stream_mates(r1, r2, batch_bytes=40000, piece_bytes=1 << 16):
        a.run_resident(with_stats=True)
        text = a.resident_text()
        for extra in (dict(paired_in=True, out2=True), dict(sout=True)):
            _twins(a, text, api.report_opts(sam=True, fastx=True, other=True, denovo=(0.9, 0.9), mates=True, **extra))
        n += 1
    assert n >= 2


# ---- 4. contracts ----
def test_contracts(golden, capfd, monkeypatch):
    exp = load_case("all")
    b = golden["batch"]
    text = open(READS, "rb").read()
    a = _golden_aligner(golden, exp, "packed", 2)
    L, h = a.L, a.h
    L.smr_place_results_packed.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    a.upload_fastx(text)
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG.*not been run"):
        a.place_packed()
    monkeypatch.setenv("SMR_VERBOSE", "1")
    a.run_resident(with_stats=True)
    capfd.readouterr()
    i1 = a.place_packed()
    i2 = a.place_packed()   # places nothing, adds the same counters
    assert {k: v for k, v in i1.items() if k not in ("matched", "place_ms")} == {k: v for k, v in i2.items() if k not in ("matched", "place_ms")}
    assert i1["matched"].tolist() == i2["matched"].tolist()
    d = a.download()         # copies the placement
    assert len(RERUN.findall(capfd.readouterr().err)) == 1
    p = a.download_placed(with_stats=True)
    for k in ("res", "alns", "stats", "cigar", "aln_off"):
        assert np.asarray(p[k]).tobytes() == np.asarray(d[k]).tobytes(), k
    assert d["counters"] == i1["counters"]
    # a packed download first: the placement it made serves the _placed calls, and place_packed() re-runs nothing
    a.run_resident(with_stats=True)
    capfd.readouterr()
    d2 = a.download()
    assert a.format_reports(None, sam=True) == a.format_reports(d2, text, sam=True)
    a.place_packed()
    assert len(RERUN.findall(capfd.readouterr().err)) == 1
    monkeypatch.delenv("SMR_VERBOSE")
    # a new run, then a new batch: the placement of the earlier run is refused
    a.run_resident(with_stats=True)
    with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED.*no placed results.*strided layout only"):
        a.format_reports(None, fastx=True)
    a.otu_begin(0.9, 0.9)
    with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED.*no placed results"):
        a.otu_add(None)
    a.place_packed()
    a.upload_fastx(text)
    with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED.*no placed results"):
        a.denovo_stats(None)
    with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED.*no placed results"):
        a.format_blast_pairwise(None)
    with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED.*strided layout only"):   # smr_place_results stays strided
        a.place()
    # the strided layout: smr_place_results_packed is refused, naming smr_place_results; a packed placement is not a strided one
    a.set_aln_layout("strided")
    a.upload(b.cat, b.off)
    a.run_resident(with_stats=True)
    assert L.smr_place_results_packed(h, None, 0, None, None) == 2
    assert b"smr_place_results" in L.smr_last_error(h)
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG.*no placed results"):
        a.format_reports(None, fastx=True)


# ---- 5. the run driver ----
def _write_fastq(path, batch):
    acgt = np.frombuffer(b"ACGT", np.uint8)
    with open(path, "wb") as f:
        for k in range(batch.n):
            s = acgt[batch.cat[int(batch.off[k]):int(batch.off[k + 1])]].tobytes()
            f.write(b"@r%d\n" % k + s + b"\n+\n" + b"I" * len(s) + b"\n")


def test_run_files_all_alignments_runs_packed(near_copies, tmp_path):
    nc = near_copies
    fq = str(tmp_path / "reads.fq")
    _write_fastq(fq, nc["batch"])
    lam, K = 0.6, 0.33
    kw = dict(gumbel=[(lam, K)], minimal_score=[MS], sam=True, blast="1", fastx=True, other=True, cmd="x ")
    out = {}
    for k, bb in (("one", 1 << 30), ("three", os.path.getsize(fq) // 3 + 1)):
        r = api.run_files([nc["fasta"]], fq, str(tmp_path / k), api.default_params(num_alignments=0), batch_bytes=bb, piece_bytes=4096, **kw)
        assert r["layout"] == "packed" and r["reads"] == nc["batch"].n
        assert r["batches"] == 1 if k == "one" else r["batches"] >= 3
        out[k] = {os.path.basename(p): open(p, "rb").read() for p in r["paths"] if not p.endswith("aligned.log")}
    assert out["three"] == out["one"]
    # what ReportWriter writes from the strided results at the grown stride, over the same reads and the same device-built index
    st, seqs = hostio.fasta_index_stats(nc["fasta"], 18, 3072.0)
    al = api.Aligner(0)
    _OPEN.append(al)
    al.set_params(api.default_params(num_alignments=0))
    counts = al.read_counts(fq)
    al.build_index_device(0, nc["fasta"], hostio.split_by_parts(hostio.load_references(nc["fasta"]), st), MS, (18, 9, 3), 18, 1, 10000, 3072.0)
    al.set_report_scoring(0, lam, K, *hostio.evalue_params(st, K, counts["length"], counts["reads"]))
    w = api.ReportWriter(str(tmp_path / "strided"), al, sam_header=hostio.sam_header_of(list(seqs), "x ", False), sam=True, blast="1",
                         fastx=True, other=True)
    text = open(fq, "rb").read()
    s = al.align(nc["batch"].cat, nc["batch"].off, with_stats=True)
    assert s["slots"] >= 1500
    w.write(s, text)
    want = {os.path.basename(p): open(p, "rb").read() for p in w.close()}
    assert sorted(want) == sorted(out["one"])
    for fn in want:
        assert out["one"][fn] == want[fn], fn
    assert want["aligned.sam"].count(b"\n") > 10000
    # strided parameters keep the strided driver
    r = api.run_files([nc["fasta"]], fq, str(tmp_path / "n1"), api.default_params(num_alignments=1), **kw)
    assert r["layout"] == "strided"
