"""The report writer on the device (smr_format_reports, sortmerna_b200/csrc/smr_report.cuh): SAM / BLAST rows and the aligned / other /
aligned_denovo read files of a batch, against the reference binary's stored output, the host formatters of hostio and, where it is
built, the reference binary itself."""
import gzip
import os
import shutil
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, case_names, load_case, load_denovo
from helpers import params_kwargs_from_args, strip_seq
from integration_common import REF_DIR, golden_mates
from sortmerna_b200 import api, hostio

pytestmark = pytest.mark.gpu

READS = os.path.join(GOLDEN, "reads_mix.fq")
BLAST = "1 cigar qcov qstrand"


_OPEN = []


def _new_aligner():
    a = api.Aligner(0)
    _OPEN.append(a)
    return a


@pytest.fixture(autouse=True)
def _close_contexts():
    """a failing test must not leave its context (and its device memory) to the next"""
    yield
    while _OPEN:
        _OPEN.pop().close()


def _text():
    return open(READS, "rb").read()


def _aligner(golden, exp, parts=None):
    a = _new_aligner()
    a.set_params(api.default_params(**params_kwargs_from_args(exp["args"] if parts is None else [])))   # case_parts: -m only splits the index
    tot = int(np.diff(golden["batch"].off.astype(np.int64)).sum())
    for k in range(2):
        if parts is None:
            a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], exp["log"]["minimal_score"][k], (18, 9, 3), golden["stats"][k].lnwin)
            st = golden["stats"][k]
        else:
            g = parts[k]
            for p in range(g["stats"].num_parts):
                a.load_index_part(k, p, g["prefix"], g["part_refs"][p], exp["log"]["minimal_score"][k], (18, 9, 3), g["stats"].lnwin)
            a.refs_by_index[k] = g["part_refs"]
            st = g["stats"]
        lam, K = exp["log"]["lambda_"][k], exp["log"]["K"][k]
        a.set_report_scoring(k, lam, K, *hostio.evalue_params(st, K, tot, golden["batch"].n))
    return a


def _rows(b):
    return b.decode().split("\n")[:-1] if b else []


def _assert_blast_in_order(ours, theirs, evalue_rtol=1.2e-2):
    """helpers.assert_blast_rows_equal, in order: every column identical except the E-value (the goldens hold 6 digits of lambda / K)"""
    assert len(ours) == len(theirs)
    for x, y in zip(ours, theirs):
        fx, fy = x.split("\t"), y.split("\t")
        assert fx[:10] == fy[:10] and fx[11:] == fy[11:], (x, y)
        assert abs(float(fx[10]) - float(fy[10])) <= evalue_rtol * abs(float(fy[10])) + 1e-300, (x, y)


@pytest.mark.parametrize("case", case_names() + ["parts"])
def test_golden_cases_in_order(golden, golden_parts, case):
    """SAM and BLAST rows of every golden case equal the reference's, in the reference's order"""
    exp = load_case(case)
    a = _aligner(golden, exp, golden_parts if case == "parts" else None)
    b = golden["batch"]
    out = a.align(b.cat, b.off, with_stats=True)
    s = a.format_reports(out, _text(), sam=True, blast=BLAST)
    sam = [r for g in s["sam"] for r in _rows(g)]
    if case != "default":
        sam = strip_seq(sam)
    assert sam == exp["sam"]
    _assert_blast_in_order([r for g in s["blast"] for r in _rows(g)], exp["blast"])
    a.close()


@pytest.mark.parametrize("case", ["default", "rev_only", "scores", "best3", "all"])
def test_equals_host_formatters(golden, case):
    """byte-identical to hostio.format_sam_rows / format_blast_rows on the same results and the same lambda / K, regrouped by
    (index, part).  hostio reverses QUAL per minus-strand row; the reference (and the writer) reverse the read's quality in place, so
    with several minus-strand rows of one read and group they differ in QUAL only -- compared without SEQ / QUAL there."""
    exp = load_case(case)
    a = _aligner(golden, exp)
    b = golden["batch"]
    out = a.align(b.cat, b.off, with_stats=True)
    s = a.format_reports(out, _text(), sam=True, blast=BLAST)
    slots = out["slots"]
    keys = [(int(out["alns"][r * slots + k]["index_num"]), int(out["alns"][r * slots + k]["part"]))
            for r in range(b.n) for k in range(int(out["res"]["n_align"][r]))]
    order = sorted(range(len(keys)), key=lambda i: keys[i])
    sam_h = hostio.format_sam_rows(b, golden["refs"], out["res"], out["alns"], out["cigar"], slots)
    tot = int(np.diff(b.off.astype(np.int64)).sum())
    gum = list(zip(exp["log"]["lambda_"], exp["log"]["K"]))
    evp = [hostio.evalue_params(st, k, tot, b.n) for st, (_, k) in zip(golden["stats"], gum)]
    blast_h = hostio.format_blast_rows(b, golden["refs"], out["res"], out["alns"], out["cigar"], slots, out["stats"], gum, evp)
    sam_g = [r for g in s["sam"] for r in _rows(g)]
    want = [sam_h[i] for i in order]
    if case in ("best3", "all"):
        sam_g, want = strip_seq(sam_g), strip_seq(want)
    assert sam_g == want
    assert [r for g in s["blast"] for r in _rows(g)] == [blast_h[i] for i in order]
    a.close()


def test_bench_workload_sam_digest():
    """the 20,000-read sample of the benchmark workload: the writer's SAM rows hash to what the reference binary printed"""
    import json
    from test_gpu_bundled_sets import rows_digest, workload
    from tools import stage_data
    exp = json.load(open(os.path.join(GOLDEN, "bench_workload.json")))
    with tempfile.TemporaryDirectory(prefix="smr_rpt_wl_") as d:
        fastas, reads, kw = workload(d)
        idx_dir, _ = stage_data.ensure_indexes(fastas, os.path.join(d, "idx"), **kw)
        pre = hostio.find_index_prefixes(idx_dir)
        al = _new_aligner()
        al.set_params(api.default_params())
        for k, f in enumerate(fastas):
            p = pre[os.path.basename(f)]
            al.load_index_part(k, 0, p, hostio.load_references(f), exp["minimal_score"][k], (18, 9, 3), hostio.parse_stats(p).lnwin)
        n = al.upload_fastx(open(reads, "rb").read())
        al.run_resident(with_stats=True)
        out = al.download()
        s = al.format_reports(out, None, sam=True)
        al.close()
    rows = [r for g in s["sam"] for r in _rows(g)]
    assert n == exp["reads"] and len(rows) == exp["sam_rows"]
    assert rows_digest(rows) == exp["sam_sha256"]


# ---- against the reference binary ----
def _need_ref():
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_ref")):
        pytest.skip("oracle/_ref/sortmerna_ref not built (oracle/Makefile.ref)")


def _reference(d, fasta, reads, idx_dir, extra):
    from oracle import ora
    r = ora.run_reference([fasta], reads, os.path.join(d, "ref"), extra=["-sam", "-fastx", "-other"] + list(extra), threads=1, idx_dir=idx_dir)
    files = {}
    for fn in os.listdir(r["out_dir"]):
        p = os.path.join(r["out_dir"], fn)
        data = gzip.open(p, "rb").read() if fn.endswith(".gz") else open(p, "rb").read()
        files[fn[:-3] if fn.endswith(".gz") else fn] = data
    return files, ora.parse_log(r["log"])


def _fasta_multiline(fq: bytes) -> bytes:
    lines = fq.split(b"\n")
    out = []
    for i in range(0, len(lines) - 3, 4):
        s = lines[i + 1]
        out.append(b">" + lines[i][1:] + b"\n" + b"".join(s[k:k + 60] + b"\n" for k in range(0, len(s), 60)))
    return b"".join(out)


@pytest.mark.parametrize("shape", ["fastq", "paired_in", "paired_out", "fasta_multiline", "fastq_gz"])
def test_against_reference_binary(golden, golden_idx_dir, shape):
    """aligned.sam body rows, aligned.* and other.* byte-identical to the reference binary (-threads 1) on the same reads against the
    golden bacterial slice"""
    _need_ref()
    fasta = os.path.join(GOLDEN, "db_bac.fasta")
    d = tempfile.mkdtemp(prefix="smr_rpt_ref_")
    try:
        extra, opts = [], {}
        if shape in ("paired_in", "paired_out"):
            m = golden_mates(d)
            reads = m
            recs = [open(p, "rb").read().split(b"\n") for p in m]
            text = b"".join(b"\n".join(recs[j][i:i + 4]) + b"\n" for i in range(0, len(recs[0]) - 3, 4) for j in (0, 1))
            extra, opts = ["-" + shape], {shape: True}
        elif shape == "fasta_multiline":
            text = _fasta_multiline(_text())
            reads = os.path.join(d, "reads.fasta")
            open(reads, "wb").write(text)
        else:
            text = _text()
            reads = READS
            if shape == "fastq_gz":
                reads = os.path.join(d, "reads.fastq.gz")
                with gzip.open(reads, "wb", compresslevel=6) as f:
                    f.write(text)
        ref, log = _reference(d, fasta, reads, golden_idx_dir, extra)
        al = _new_aligner()
        al.set_params(api.default_params())
        al.load_index_part(0, 0, golden["prefixes"][1], golden["refs"][1], log["minimal_score"][0], (18, 9, 3), golden["stats"][1].lnwin)
        if shape == "fastq_gz":
            al.upload_fastx_gz(open(reads, "rb").read())
            text = None
        else:
            al.upload_fastx(text)
        al.run_resident(with_stats=True)
        out = al.download()
        s = al.format_reports(out, text, sam=True, fastx=True, other=True, **opts)
        al.close()
        ext = "fa" if shape == "fasta_multiline" else "fq"
        assert s["sam"][0] == b"".join(ln + b"\n" for ln in ref["aligned.sam"].split(b"\n") if ln and not ln.startswith(b"@"))
        assert s["aligned"] == ref["aligned." + ext]
        assert s["other"] == ref["other." + ext]
        assert len(s["aligned"]) > 1000 and len(s["other"]) > 100
    finally:
        shutil.rmtree(d, ignore_errors=True)


@pytest.mark.parametrize("case", ["default", "best3", "rev_only", "loose"])
def test_denovo_reads(golden, case):
    """aligned_denovo: the reads of tests/golden/denovo.json, classified on the device from n_match_denovo, -id and -coverage"""
    dn = load_denovo()[case]
    a = _new_aligner()
    a.set_params(api.default_params(**params_kwargs_from_args(dn["args"])))
    for k in range(2):
        a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], dn["minimal_score"][k], (18, 9, 3), golden["stats"][k].lnwin)
    b = golden["batch"]
    out = a.align(b.cat, b.off, with_stats=True)
    s = a.format_reports(out, _text(), denovo=(dn["min_id"], dn["min_cov"]))
    lines = s["denovo"].split(b"\n")
    ids = sorted(hostio.seq_id(lines[i].decode()) for i in range(0, len(lines) - 1, 4))
    assert ids == dn["denovo_reads"]
    a.close()


def test_multi_batch_equals_one_batch(golden, tmp_path):
    """ReportWriter: the golden reads in 3 batches write the files one batch writes, byte for byte"""
    exp = load_case("best3")
    lines = _text().split(b"\n")
    recs = [b"\n".join(lines[i:i + 4]) + b"\n" for i in range(0, len(lines) - 3, 4)]
    cut = [0, len(recs) // 3, 2 * len(recs) // 3, len(recs)]
    a = _aligner(golden, exp)
    res = {}
    for name, pieces in (("one", [recs]), ("three", [recs[cut[i]:cut[i + 1]] for i in range(3)])):
        w = api.ReportWriter(str(tmp_path / name), a, sam_header=hostio.sam_header(golden["prefixes"], "sortmerna"), sam=True, blast=BLAST,
                             fastx=True, other=True, denovo=(0.97, 0.97))
        for p in pieces:
            text = b"".join(p)
            a.upload_fastx(text)
            a.run_resident(with_stats=True)
            w.write(a.download(), text)
        res[name] = {os.path.basename(f): open(f, "rb").read() for f in w.close()}
    assert sorted(res["one"]) == ["aligned.blast", "aligned.fq", "aligned.sam", "aligned_denovo.fq", "other.fq"]
    for fn in res["one"]:
        assert res["three"][fn] == res["one"][fn], fn
    assert res["one"]["aligned.sam"].count(b"\n") > 1000
    a.close()


def test_refusals(golden):
    exp = load_case("default")
    a = _aligner(golden, exp)
    b = golden["batch"]
    out = a.align(b.cat, b.off, with_stats=True)
    text = _text()
    short = b"\n".join(text.split(b"\n")[4:])   # one record fewer than the results
    with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):
        a.format_reports(out, short, sam=True)
    with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED"):
        a.format_reports(out, text, sam=True, out2=True)
    with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED"):
        a.format_reports(out, text, blast="0")
    # too small an output buffer: SMR_ERR_CAPACITY with the sizes; a retry with them succeeds
    import ctypes as C
    o = api.report_opts(sam=True, fastx=True)
    a._upload_report_refs()
    G = len(a.report_groups())
    so = np.zeros(2 * G + 4, np.uint64)
    txt = np.frombuffer(text, np.uint8)
    cig = np.ascontiguousarray(out["cigar"], np.uint32)
    small = np.zeros(16, np.uint8)
    args = [a.h, C.cast(C.byref(o), C.c_void_p), api._ptr(txt), txt.size, api._ptr(out["res"]), api._ptr(out["alns"]), api._ptr(cig), cig.size,
            api._ptr(out["stats"]), b.n]
    assert a.L.smr_format_reports(*args, api._ptr(small), small.size, api._ptr(so)) == 5
    need = int(so[-1])
    assert need > 16 and so[G] > 0 and so[2 * G + 1] > so[2 * G]
    buf = np.zeros(need, np.uint8)
    assert a.L.smr_format_reports(*args, api._ptr(buf), buf.size, api._ptr(so)) == 0
    s = a.format_reports(out, text, sam=True, fastx=True)
    assert bytes(buf[:int(so[G])]) == b"".join(s["sam"]) and bytes(buf[int(so[2 * G]):int(so[2 * G + 1])]) == s["aligned"]
    a.close()
