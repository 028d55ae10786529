"""Pairwise BLAST rows (-blast 0) on the device (smr_format_blast_pairwise[_gz], Aligner.format_blast_pairwise, ReportWriter with
blast="0"): against the reference binary's stored output (tests/golden/blast_pairwise/), the host restatement
hostio.format_blast_pairwise_rows on the device's own results, and, where it is built, the reference binary itself."""
import ctypes as C
import gzip
import os

import numpy as np
import pytest

from conftest import GOLDEN
from integration_common import REF_DIR, golden_mates
from pairwise_common import CASES, assert_pairwise_equal, expected, inputs
from sortmerna_b200 import api, hostio

pytestmark = pytest.mark.gpu

_OPEN = []


@pytest.fixture(autouse=True)
def _close_contexts():
    """a failing test must not leave its context (and its device memory) to the next"""
    yield
    while _OPEN:
        _OPEN.pop().close()


def _aligner(x):
    a = api.Aligner(0)
    _OPEN.append(a)
    a.set_params(api.default_params(**x["params"]))
    for k, (p, st) in enumerate(zip(x["prefixes"], x["stats"])):
        a.load_index_part(k, 0, p, x["refs"][k], x["minimal_score"][k], (18, 9, 3), st.lnwin)
        a.set_report_scoring(k, *x["gumbel"][k], *x["ev_params"][k])
    return a


def _case(case, golden_idx_dir, with_stats=True):
    x = inputs(case, golden_idx_dir)
    a = _aligner(x)
    b = x["batch"]
    return x, a, a.align(b.cat, b.off, with_stats=with_stats)


@pytest.mark.parametrize("case", sorted(CASES))
def test_fixture_and_host_restatement(golden_idx_dir, case):
    """the device's rows equal the reference's (E-values to their last printed digit), and hostio's on the device's own results byte
    for byte; stats are not needed"""
    x, a, out = _case(case, golden_idx_dir, with_stats=False)
    got = a.format_blast_pairwise(out, x["text"])
    assert len(got) == len(x["prefixes"])
    host = hostio.format_blast_pairwise_rows(x["batch"], x["refs"], out["res"], out["alns"], out["cigar"], out["slots"], x["gumbel"],
                                             x["ev_params"])
    assert b"".join(got) == "".join(host).encode()
    assert_pairwise_equal(b"".join(got), expected(case))
    # the resident text gives the same bytes
    a.upload_fastx(x["text"])
    a.run_resident(with_stats=False)
    assert a.format_blast_pairwise(a.download(), None) == got


def test_gzip_members_inflate_to_the_plain_bytes(golden_idx_dir):
    x, a, out = _case("best3_both", golden_idx_dir)
    plain = a.format_blast_pairwise(out, x["text"])
    z = a.format_blast_pairwise(out, x["text"], gzip=True)
    assert all(len(p) > 1000 for p in plain)
    assert [gzip.decompress(m) for m in z] == plain
    assert all(m[:2] == b"\x1f\x8b" for m in z)


def test_capacity_retry(golden_idx_dir):
    """too small a buffer: SMR_ERR_CAPACITY with the sizes in stream_off; a retry with them succeeds"""
    x, a, out = _case("default", golden_idx_dir)
    want = a.format_blast_pairwise(out, x["text"])
    o = api.report_opts(blast="0")
    txt = np.frombuffer(x["text"], np.uint8)
    cig = np.ascontiguousarray(out["cigar"], np.uint32)
    for fn, gz in ((a.L.smr_format_blast_pairwise, False), (a.L.smr_format_blast_pairwise_gz, True)):
        so = np.zeros(2, np.uint64)
        args = [a.h, C.cast(C.byref(o), C.c_void_p), api._ptr(txt), txt.size, api._ptr(out["res"]), api._ptr(out["alns"]), api._ptr(cig),
                cig.size, None, x["batch"].n]
        small = np.zeros(16, np.uint8)
        assert fn(*args, api._ptr(small), small.size, api._ptr(so)) == 5
        need = int(so[-1])
        assert need > 16 and so[0] == 0
        buf = np.zeros(need, np.uint8)
        assert fn(*args, api._ptr(buf), buf.size, api._ptr(so)) == 0
        data = bytes(buf[:int(so[1])])
        assert (gzip.decompress(data) if gz else data) == want[0]


def test_refusals(golden_idx_dir):
    x, a, out = _case("default", golden_idx_dir)
    t = x["text"]
    for kw in (dict(blast="0 cigar"), dict(blast="1"), dict(blast="0", sam=True), dict(blast="0", fastx=True), dict(blast="0", other=True),
               dict(blast="0", denovo=(0.97, 0.97)), dict(blast="0", paired_in=True, paired_out=True)):
        with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):
            a.format_blast_pairwise(out, t, opts=api.report_opts(**kw))
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):
        a.format_blast_pairwise(out, t, opts=api.report_opts())   # -blast not given
    with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED.*smr_format_blast_pairwise"):
        a.format_reports(out, t, blast="0")
    # a CIGAR that runs past its reference
    bad = dict(out, alns=out["alns"].copy())
    k = int(np.nonzero(out["res"]["n_align"])[0][0]) * out["slots"]
    bad["alns"][k]["ref_begin1"] = 1 << 20
    with pytest.raises(api.SmrError, match="runs past its read or its reference"):
        a.format_blast_pairwise(bad, t)
    assert b"".join(a.format_blast_pairwise(out, t)) == b"".join(a.format_blast_pairwise(out, t, paired_in=False))


def test_report_writer_three_batches_equal_one(golden_idx_dir, tmp_path):
    """ReportWriter with blast="0": the golden reads in 3 batches write the files one batch writes; SAM and aligned.fq still come from
    format_reports"""
    x, a, _ = _case("best3_both", golden_idx_dir)
    lines = x["text"].split(b"\n")
    recs = [b"\n".join(lines[i:i + 4]) + b"\n" for i in range(0, len(lines) - 3, 4)]
    cut = [0, len(recs) // 3, 2 * len(recs) // 3, len(recs)]
    res = {}
    for name, pieces in (("one", [recs]), ("three", [recs[cut[i]:cut[i + 1]] for i in range(3)])):
        for zip_out in (False, True):
            w = api.ReportWriter(str(tmp_path / f"{name}{int(zip_out)}"), a, sam_header="@HD\n", zip_out=zip_out, sam=True, blast="0", fastx=True)
            for p in pieces:
                text = b"".join(p)
                a.upload_fastx(text)
                a.run_resident(with_stats=True)
                w.write(a.download(), text)
            res[name, zip_out] = {os.path.basename(f).replace(".gz", ""): (gzip.open if zip_out else open)(f, "rb").read() for f in w.close()}
    assert sorted(res["one", False]) == ["aligned.blast", "aligned.fq", "aligned.sam"]
    for key in res:
        assert res[key] == res["one", False], key
    assert_pairwise_equal(res["one", False]["aligned.blast"], expected("best3_both"))


# ---- against the reference binary ----
def _need_ref():
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_ref")):
        pytest.skip("oracle/_ref/sortmerna_ref not built (oracle/Makefile.ref)")


def _fasta_multiline(fq: bytes) -> bytes:
    lines = fq.split(b"\n")
    out = []
    for i in range(0, len(lines) - 3, 4):
        s = lines[i + 1]
        out.append(b">" + lines[i][1:] + b"\n" + b"".join(s[k:k + 60] + b"\n" for k in range(0, len(s), 60)))
    return b"".join(out)


def _reference(d, reads, idx_dir, extra):
    from oracle import ora
    r = ora.run_reference([os.path.join(GOLDEN, "db_bac.fasta")], reads, os.path.join(d, "ref"), extra=list(extra), threads=1, idx_dir=idx_dir)
    files = {}
    for fn in os.listdir(r["out_dir"]):
        p = os.path.join(r["out_dir"], fn)
        files[fn.replace(".gz", "")] = gzip.open(p, "rb").read() if fn.endswith(".gz") else open(p, "rb").read()
    return files, ora.parse_log(r["log"])


def _writer_aligner(golden, log, reads):
    """db_bac.fasta loaded as the reference ran it: its minimal score, and its E-value inputs from the reference's count of the reads"""
    al = api.Aligner(0)
    _OPEN.append(al)
    al.set_params(api.default_params())
    al.load_index_part(0, 0, golden["prefixes"][1], golden["refs"][1], log["minimal_score"][0], (18, 9, 3), golden["stats"][1].lnwin)
    c = al.read_counts(reads)   # as the reference counts them: for a multi-line FASTA not the true length (test_gpu_stream)
    al.set_report_scoring(0, log["lambda_"][0], log["K"][0], *hostio.evalue_params(golden["stats"][1], log["K"][0], c["length"], c["reads"]))
    return al


def _sam_rows(b):
    return b"".join(ln + b"\n" for ln in b.split(b"\n") if ln and not ln.startswith(b"@"))


@pytest.mark.parametrize("shape", ["fastq", "fasta_multiline", "fastq_gz_zip_out", "paired_in", "mates"])
def test_against_reference_binary(golden, golden_idx_dir, tmp_path, shape):
    """aligned.blast of -blast 0 (and aligned.sam) through ReportWriter equal the reference binary's at -threads 1 on the same reads
    against the golden bacterial slice"""
    _need_ref()
    d = str(tmp_path)
    text = open(os.path.join(GOLDEN, "reads_mix.fq"), "rb").read()
    reads, extra, kw, zip_out = os.path.join(GOLDEN, "reads_mix.fq"), [], {}, False
    if shape == "fasta_multiline":
        text = _fasta_multiline(text)
        reads = os.path.join(d, "reads.fasta")
        open(reads, "wb").write(text)
    elif shape == "fastq_gz_zip_out":
        reads = os.path.join(d, "reads.fastq.gz")
        with gzip.open(reads, "wb", compresslevel=6) as f:
            f.write(text)
        extra, zip_out = ["-zip-out", "1"], True
    elif shape in ("paired_in", "mates"):
        reads = golden_mates(d)
        recs = [open(p, "rb").read().split(b"\n") for p in reads]
        text = b"".join(b"\n".join(recs[j][i:i + 4]) + b"\n" for i in range(0, len(recs[0]) - 3, 4) for j in (0, 1))
        if shape == "paired_in":
            extra, kw = ["-paired_in"], dict(paired_in=True)
    ref, log = _reference(d, reads, golden_idx_dir, ["-blast", "0", "-sam"] + extra)
    al = _writer_aligner(golden, log, reads)
    w = api.ReportWriter(os.path.join(d, "ours"), al, zip_out=zip_out, sam=True, blast="0", **kw)
    if shape == "mates":
        for _ in al.stream_mates(reads[0], reads[1], batch_bytes=len(text) // 3 + 1, piece_bytes=8192):
            al.run_resident(with_stats=True)
            w.write(al.download(), None)
    else:
        if zip_out:
            al.upload_fastx_gz(open(reads, "rb").read())
        else:
            al.upload_fastx(text)
        al.run_resident(with_stats=True)
        w.write(al.download(), None)
    ours = {os.path.basename(p).replace(".gz", ""): (gzip.open if zip_out else open)(p, "rb").read() for p in w.close()}
    assert _sam_rows(ours["aligned.sam"]) == _sam_rows(ref["aligned.sam"])
    assert ours["aligned.blast"].count(b"Sequence ID: ") == _sam_rows(ref["aligned.sam"]).count(b"\n") > 100
    assert_pairwise_equal(ours["aligned.blast"], ref["aligned.blast"])


def test_print_all_reads_writes_no_null_rows(golden, golden_idx_dir, tmp_path):
    """-print_all_reads 1: the reference writes no row for a read without alignments, in aligned.sam (ReportSam::append returns
    first) or in tabular aligned.blast (the null row sits inside the loop over the read's alignments) -- the writer, which has no
    such option, writes the same files"""
    _need_ref()
    d = str(tmp_path)
    reads = os.path.join(GOLDEN, "reads_mix.fq")
    text = open(reads, "rb").read()
    ref, log = _reference(d, reads, golden_idx_dir, ["-blast", "1 cigar qcov qstrand", "-sam", "-print_all_reads", "1"])
    al = _writer_aligner(golden, log, reads)
    w = api.ReportWriter(os.path.join(d, "ours"), al, sam=True, blast="1 cigar qcov qstrand")
    al.upload_fastx(text)
    al.run_resident(with_stats=True)
    out = al.download()
    w.write(out, None)
    ours = {os.path.basename(p): open(p, "rb").read() for p in w.close()}
    assert int((out["res"]["n_align"] == 0).sum()) > 10
    assert _sam_rows(ours["aligned.sam"]) == _sam_rows(ref["aligned.sam"])
    x, y = ours["aligned.blast"].decode().split("\n"), ref["aligned.blast"].decode().split("\n")
    assert len(x) == len(y) > 100
    for u, v in zip(x, y):   # every column but the E-value byte for byte (see pairwise_common.assert_pairwise_equal)
        fu, fv = u.split("\t"), v.split("\t")
        assert fu[:10] == fv[:10] and fu[11:] == fv[11:], (u, v)
        if len(fu) > 10:
            assert abs(float(fu[10]) - float(fv[10])) <= 1.2e-2 * abs(float(fv[10])) + 1e-300, (u, v)
