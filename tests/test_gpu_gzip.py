"""gzip on the device (smr_gzip / smr_format_reports_gz, sortmerna_b200/csrc/smr_deflate.cuh): the device writes the bytes the host run
of the same encoder (tests/deflate_check.cpp) writes, every member decompresses to its input, the report streams and ReportWriter's
-zip-out files decompress to the plain writer's output, and, where it is built, to the reference binary's -zip-out files."""
import gzip
import os
import shutil
import subprocess
import tempfile
import zlib

import numpy as np
import pytest

from conftest import GOLDEN, load_case
from helpers import params_kwargs_from_args
from integration_common import REF_DIR
from sortmerna_b200 import api, hostio
from test_deflate_host import ROOT, corpus

pytestmark = pytest.mark.gpu

READS = os.path.join(GOLDEN, "reads_mix.fq")
BLAST = "1 cigar qcov qstrand"
_OPEN = []


@pytest.fixture(autouse=True)
def _close_contexts():
    yield
    while _OPEN:
        _OPEN.pop().close()


def _new_aligner():
    a = api.Aligner(0)
    _OPEN.append(a)
    return a


@pytest.fixture(scope="module")
def deflate_check(tmp_path_factory):
    e = str(tmp_path_factory.mktemp("deflate") / "deflate_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "deflate_check.cpp"), "-o", e])
    return e


def _host_gzip(exe, data: bytes) -> bytes:
    with tempfile.TemporaryDirectory(prefix="smr_gz_") as d:
        open(os.path.join(d, "in"), "wb").write(data)
        subprocess.check_call([exe, os.path.join(d, "in"), os.path.join(d, "out")], stdout=subprocess.DEVNULL)
        return open(os.path.join(d, "out"), "rb").read()


def _big_fastq(nbytes: int) -> bytes:
    """seeded FASTQ of 150-nt reads with varied qualities, about nbytes long"""
    rng = np.random.default_rng(99)
    n = nbytes // 315 + 1
    rec = np.empty((n, 315), np.uint8)
    ids = np.char.zfill(np.arange(n).astype("S9"), 9)
    rec[:, 0] = ord("@"); rec[:, 1:10] = np.frombuffer(ids.tobytes(), np.uint8).reshape(n, 9); rec[:, 10] = 10
    rec[:, 11:161] = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, (n, 150))]
    rec[:, 161] = 10; rec[:, 162] = ord("+"); rec[:, 163] = 10
    rec[:, 164:314] = rng.integers(35, 74, (n, 150)).astype(np.uint8)
    rec[:, 314] = 10
    return rec.tobytes()


def test_gzip_equals_host_encoder(deflate_check):
    a = _new_aligner()
    for name, data in list(corpus().items()) + [("fastq_300mb", _big_fastq(300 << 20))]:
        got = a.gzip(data)
        assert got == _host_gzip(deflate_check, data), name
        assert zlib.decompress(got, 31) == data, name
        assert a.gzip(data) == got, name


def _run(a, text):
    a.upload_fastx(text)
    a.run_resident(with_stats=True)
    return a.download()


def _golden_aligner(golden, case="default"):
    exp = load_case(case)
    a = _new_aligner()
    a.set_params(api.default_params(**params_kwargs_from_args(exp["args"])))
    tot = int(np.diff(golden["batch"].off.astype(np.int64)).sum())
    for k in range(2):
        a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], exp["log"]["minimal_score"][k], (18, 9, 3), golden["stats"][k].lnwin)
        lam, K = exp["log"]["lambda_"][k], exp["log"]["K"][k]
        a.set_report_scoring(k, lam, K, *hostio.evalue_params(golden["stats"][k], K, tot, golden["batch"].n))
    return a


def _records(text):
    lines = text.split(b"\n")
    return [b"\n".join(lines[i:i + 4]) + b"\n" for i in range(0, len(lines) - 3, 4)]


@pytest.mark.parametrize("shape", ["all", "best3", "paired_in", "paired_out"])
def test_format_reports_gz_streams(golden, shape):
    """every gz stream is one member that decompresses to the plain call's stream; empty streams stay empty"""
    a = _golden_aligner(golden, "best3" if shape == "best3" else "default")
    recs = _records(open(READS, "rb").read())
    text = b"".join(recs[:len(recs) // 2 * 2])
    out = _run(a, text)
    kw = dict(sam=True, blast=BLAST, fastx=True, other=True, denovo=(0.97, 0.97))
    if shape.startswith("paired"):
        kw[shape] = True
    plain = a.format_reports(out, None, **kw)
    gz = a.format_reports(out, None, gzip=True, **kw)
    pairs = list(zip(plain["sam"] + plain["blast"], gz["sam"] + gz["blast"])) + [(plain[k], gz[k]) for k in ("aligned", "other", "denovo")]
    for p, g in pairs:
        if not p:
            assert g == b""
            continue
        assert g[:4] == b"\x1f\x8b\x08\x00" and zlib.decompress(g, 31) == p
        d = zlib.decompressobj(31)
        d.decompress(g)
        assert d.eof and d.unused_data == b""   # exactly one member
    assert sum(len(p) > 0 for p, _ in pairs) >= 5
    assert a.report_timings()["device_ms"] > 0


def test_capacity_retry_gives_identical_bytes(golden):
    import ctypes as C
    a = _golden_aligner(golden)
    text = open(READS, "rb").read()
    out = _run(a, text)
    o = api.report_opts(sam=True, fastx=True, other=True)
    a._upload_report_refs()
    G = len(a.report_groups())
    cig = np.ascontiguousarray(out["cigar"], np.uint32)
    args = [a.h, C.cast(C.byref(o), C.c_void_p), None, 0, api._ptr(out["res"]), api._ptr(out["alns"]), api._ptr(cig), cig.size,
            api._ptr(out["stats"]), out["res"].shape[0]]
    a.L.smr_format_reports_gz.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                          C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
    so = np.zeros(2 * G + 4, np.uint64)
    small = np.zeros(16, np.uint8)
    assert a.L.smr_format_reports_gz(*args, api._ptr(small), small.size, api._ptr(so)) == 5
    need = int(so[-1])
    so2 = np.zeros_like(so)
    buf = np.zeros(need, np.uint8)
    assert a.L.smr_format_reports_gz(*args, api._ptr(buf), buf.size, api._ptr(so2)) == 0
    assert np.array_equal(so, so2)
    s = a.format_reports(out, None, gzip=True, sam=True, fastx=True, other=True)
    assert bytes(buf) == b"".join(s["sam"] + s["blast"]) + s["aligned"] + s["other"] + s["denovo"]
    plain = a.format_reports(out, None, sam=True, fastx=True, other=True)
    assert zlib.decompress(s["aligned"], 31) == plain["aligned"]


def test_streams_survive_a_smaller_earlier_call(golden):
    """a gz call that writes nothing leaves the context's output buffer at 8 + 1 + 256 = 265 bytes; a following call whose streams
    total 258..264 bytes must still compress the streams it wrote, not a fresh buffer"""
    lines = open(READS, "rb").read().split(b"\n")
    seq, qual = lines[1][:100], lines[3][:100]
    head = lines[0] + b"_" * (260 - (len(lines[0]) + 1 + 2 * 101 + 2))
    text = head + b"\n" + seq + b"\n+\n" + qual + b"\n"
    assert len(text) == 260
    ref = _golden_aligner(golden)
    plain = ref.format_reports(_run(ref, text), text, fastx=True, other=True)
    assert len(plain["aligned"]) + len(plain["other"]) == 260
    a = _golden_aligner(golden)
    out = _run(a, text)
    nothing = a.format_reports(out, text, gzip=True)
    assert all(x == b"" for x in nothing["sam"] + nothing["blast"]) and nothing["aligned"] == nothing["other"] == b""
    gz = a.format_reports(out, text, gzip=True, fastx=True, other=True)
    for k in ("aligned", "other"):
        assert (zlib.decompress(gz[k], 31) if gz[k] else b"") == plain[k], k


def _gzip_t(path):
    subprocess.check_call(["gzip", "-t", path])


def test_report_writer_zip_out(golden, tmp_path):
    """3 batches with zip_out: the reference's names with .gz, each decompressing to the plain one-batch file; gzip -t passes; a file
    with nothing in it is one empty member"""
    a = _golden_aligner(golden, "best3")
    recs = _records(open(READS, "rb").read())
    cut = [0, len(recs) // 3, 2 * len(recs) // 3, len(recs)]
    head = hostio.sam_header(golden["prefixes"], "sortmerna")
    kw = dict(sam=True, blast=BLAST, fastx=True, other=True, denovo=(0.0, 0.0))   # every aligned read passes -id 0 -coverage 0: an empty aligned_denovo
    res = {}
    for name, pieces, z in (("plain", [recs], False), ("gz", [recs[cut[i]:cut[i + 1]] for i in range(3)], True)):
        w = api.ReportWriter(str(tmp_path / name), a, sam_header=head, zip_out=z, **kw)
        for p in pieces:
            text = b"".join(p)
            w.write(_run(a, text), text)
        res[name] = {os.path.basename(f): f for f in w.close()}
    assert sorted(res["gz"]) == sorted(f + ".gz" for f in res["plain"])
    assert sorted(res["plain"]) == ["aligned.blast", "aligned.fq", "aligned.sam", "aligned_denovo.fq", "other.fq"]
    for fn, path in res["plain"].items():
        gzp = res["gz"][fn + ".gz"]
        _gzip_t(gzp)
        assert gzip.open(gzp, "rb").read() == open(path, "rb").read(), fn
    assert open(res["plain"]["aligned_denovo.fq"], "rb").read() == b""
    assert open(res["gz"]["aligned_denovo.fq.gz"], "rb").read() == a.gzip(b"")
    # round trip: aligned.fq.gz through the device's own inflate gives the plain file's text
    a.upload_fastx_gz(open(res["gz"]["aligned.fq.gz"], "rb").read())
    assert a.resident_text() == open(res["plain"]["aligned.fq"], "rb").read()


def _need_ref():
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_ref")):
        pytest.skip("oracle/_ref/sortmerna_ref not built (oracle/Makefile.ref)")


@pytest.mark.parametrize("shape", ["fastq_gz_default", "fastq_zip_out_1"])
def test_against_reference_binary(golden, golden_idx_dir, shape):
    """the reference's -zip-out files (its default for .fastq.gz input, and -zip-out 1 on FASTQ): the same file names, the same
    decompressed contents"""
    _need_ref()
    from oracle import ora
    fasta = os.path.join(GOLDEN, "db_bac.fasta")
    d = tempfile.mkdtemp(prefix="smr_gz_ref_")
    try:
        text = open(READS, "rb").read()
        reads, extra = READS, ["-zip-out", "1"]
        if shape == "fastq_gz_default":
            reads, extra = os.path.join(d, "reads.fastq.gz"), []
            with gzip.open(reads, "wb", compresslevel=6) as f:
                f.write(text)
        r = ora.run_reference([fasta], reads, os.path.join(d, "ref"), extra=["-sam", "-fastx", "-other"] + extra, threads=1, idx_dir=golden_idx_dir)
        ref = {fn: gzip.open(os.path.join(r["out_dir"], fn), "rb").read() for fn in os.listdir(r["out_dir"]) if fn != "aligned.log"}
        log = ora.parse_log(r["log"])
        al = _new_aligner()
        al.set_params(api.default_params())
        al.load_index_part(0, 0, golden["prefixes"][1], golden["refs"][1], log["minimal_score"][0], (18, 9, 3), golden["stats"][1].lnwin)
        head = b"".join(ln + b"\n" for ln in ref["aligned.sam.gz"].split(b"\n") if ln.startswith(b"@")).decode()
        w = api.ReportWriter(os.path.join(d, "ours"), al, sam_header=head, zip_out=True, sam=True, fastx=True, other=True)
        if shape == "fastq_gz_default":
            al.upload_fastx_gz(open(reads, "rb").read())
            al.run_resident(with_stats=True)
            w.write(al.download(), None)
        else:
            w.write(_run(al, text), text)
        ours = {os.path.basename(f): gzip.open(f, "rb").read() for f in w.close()}
        assert sorted(ours) == sorted(ref) == ["aligned.fq.gz", "aligned.sam.gz", "other.fq.gz"]
        for fn in ref:
            assert ours[fn] == ref[fn], fn
        assert len(ref["aligned.fq.gz"]) > 1000
    finally:
        shutil.rmtree(d, ignore_errors=True)
