"""aligned.bam on the device (smr_format_bam_placed, smr_bam_header, run_files(bam=True), -bam): it decodes to aligned.sam.  The BAM
streams decode, group by group, to the SAM rows of the same placement, and the from-spec encoder of tests/bam_spec.py applied to
those rows gives the records byte for byte; the header's dictionary is the (id, length) of every reference in --ref order; the
BGZF framing holds on multi-block streams; the contracts; and the files run_files and the command line write."""
import ctypes as C
import gzip
import json
import os
import re

import numpy as np
import pytest

import bam_spec
from conftest import GOLDEN, case_names, load_case
from helpers import params_kwargs_from_args
from integration_common import golden_mates
from sortmerna_b200 import __main__ as cli
from sortmerna_b200 import api, hostio

pytestmark = pytest.mark.gpu

READS = os.path.join(GOLDEN, "reads_mix.fq")
REFS = [os.path.join(GOLDEN, "db_arc.fasta"), os.path.join(GOLDEN, "db_bac.fasta")]
GUMBEL = [(0.594908, 0.326193), (0.600371, 0.328947)]
_OPEN = []


@pytest.fixture(autouse=True)
def _close_contexts():
    yield
    while _OPEN:
        _OPEN.pop().close()


def _aligner(golden, exp=None, layout="strided", slots=None, parts=None):
    a = api.Aligner(0)
    _OPEN.append(a)
    a.set_params(api.default_params(**params_kwargs_from_args(exp["args"] if exp else [])))
    ms = exp["log"]["minimal_score"] if exp else load_case("default")["log"]["minimal_score"]
    for k in range(2):
        if parts is None:
            a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], ms[k], (18, 9, 3), golden["stats"][k].lnwin)
        else:
            for p in range(parts[k]["stats"].num_parts):
                a.load_index_part(k, p, parts[k]["prefix"], parts[k]["part_refs"][p], ms[k], (18, 9, 3), parts[k]["stats"].lnwin)
            a.refs_by_index[k] = parts[k]["part_refs"]
    a.set_aln_layout(layout)
    if slots:
        a.set_aln_slots(slots)
    return a


def _run_and_place(a, text):
    a.upload_fastx(text)
    a.set_place_stats(True)
    a.run_resident()
    return a.place_packed() if a.layout == "packed" else a.place()


def _groups(a):
    """per report group: (names of its references, refID base)"""
    out, base = [], 0
    for (i, p) in a.report_groups():
        r = a.refs_by_index[i]
        ids = list((r[p] if isinstance(r, (list, tuple)) else r).ids)
        out.append((ids, base))
        base += len(ids)
    return out


def _rows(b: bytes) -> list:
    return b.decode().splitlines()


def assert_bam_is_sam(a, opts=None, what=""):
    """the placed batch's BAM streams against its SAM streams: decoded rows equal, and encoded rows equal the records; returns the
    BAM streams"""
    o = opts if opts is not None else api.report_opts(sam=True)
    sbuf, sso = a.format_placed_into(o, np.zeros(1 << 20, np.uint8))
    bbuf, bso = a.format_placed_into(o, np.zeros(1 << 16, np.uint8), bam=True)
    grp = _groups(a)
    names = [n for ids, _ in grp for n in ids]
    assert bso.size == len(grp) + 1
    streams = []
    for g, (ids, base) in enumerate(grp):
        sam = _rows(bytes(sbuf[int(sso[g]):int(sso[g + 1])]))
        stream = bytes(bbuf[int(bso[g]):int(bso[g + 1])])
        streams.append(stream)
        recs = bam_spec.split_records(bam_spec.check_stream(stream))
        assert [bam_spec.decode_record(r, names) for r in recs] == sam, (what, g)
        first = {}
        for k, n in enumerate(ids):
            first.setdefault(n, k)
        assert [bam_spec.encode_row(row, base + first[row.split("\t")[2]]) for row in sam] == recs, (what, g)
    return streams


# ---- 1. golden cases ----
@pytest.mark.parametrize("case", case_names())
def test_golden_cases_strided(golden, case):
    exp = load_case(case)
    a = _aligner(golden, exp)
    _run_and_place(a, open(READS, "rb").read())
    streams = assert_bam_is_sam(a, what=case)
    assert sum(len(s) for s in streams) > 0


@pytest.mark.parametrize("stride", [1, 16])
def test_case_all_packed(golden, stride):
    a = _aligner(golden, load_case("all"), "packed", stride)
    _run_and_place(a, open(READS, "rb").read())
    assert_bam_is_sam(a, what=f"packed {stride}")


# ---- 2. the header ----
def _header(a, sq):
    seqs = [x for f in REFS for x in hostio.fasta_index_stats(f)[1]]
    text = hostio.sam_header_of(seqs, "x -bam ", sq)
    got_text, refs, recs = bam_spec.decode_file(a.bam_header(text.encode()) + bam_spec.EOF_BLOCK)
    assert got_text == text and recs == []
    assert refs == [(s, int(n)) for s, n in seqs]
    return refs


@pytest.mark.parametrize("parts", [False, True])
def test_header_dictionary(golden, golden_parts, parts):
    a = _aligner(golden, parts=golden_parts if parts else None)
    if parts:
        assert len(a.report_groups()) > 2
    for sq in (False, True):
        refs = _header(a, sq)
    # every record's refID names its SAM RNAME: checked by decode_record over the same dictionary
    _run_and_place(a, open(READS, "rb").read())
    assert [n for ids, _ in _groups(a) for n in ids] == [n for n, _ in refs]
    assert_bam_is_sam(a, what="parts" if parts else "two groups")


def test_header_needs_report_refs(golden):
    a = _aligner(golden)
    a.refs_by_index.clear()
    with pytest.raises(api.SmrError):
        a.bam_header(b"@HD\n")
    L = a.L
    out, nb = np.zeros(1 << 16, np.uint8), np.zeros(1, np.uint64)
    L.smr_bam_header.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
    assert L.smr_bam_header(a.h, None, 0, api._ptr(out), out.size, api._ptr(nb)) == 2
    assert b"smr_set_report_refs" in L.smr_last_error(a.h)


# ---- 3. multi-block streams ----
def test_bench_workload_sample(tmp_path):
    from test_gpu_bundled_sets import workload
    from tools import stage_data
    fastas, reads, kw = workload(str(tmp_path))
    idx_dir, _ = stage_data.ensure_indexes(fastas, str(tmp_path / "idx"), **kw)
    pre = hostio.find_index_prefixes(idx_dir)
    a = api.Aligner(0)
    _OPEN.append(a)
    a.set_params(api.default_params())
    ms = json.load(open(os.path.join(GOLDEN, "bench_workload.json")))["minimal_score"]
    for k, f in enumerate(fastas):
        p = pre[os.path.basename(f)]
        a.load_index_part(k, 0, p, hostio.load_references(f), ms[k], (18, 9, 3), hostio.parse_stats(p).lnwin)
    _run_and_place(a, open(reads, "rb").read())
    streams = assert_bam_is_sam(a, what="bench sample")
    assert max(len(bam_spec.members(s)) for s in streams) >= 3


def test_incompressible_quality_lines(golden):
    """the golden reads with random quality lines: the blocks hardly compress, and every member stays within 64 KiB"""
    rng = np.random.default_rng(5)
    lines = open(READS, "rb").read().split(b"\n")
    for i in range(3, len(lines), 4):
        lines[i] = bytes(rng.integers(33, 127, len(lines[i]), dtype=np.uint8))
    a = _aligner(golden, load_case("all"), "packed", 16)
    _run_and_place(a, b"\n".join(lines))
    streams = assert_bam_is_sam(a, what="random quality")
    ms = [m for s in streams for m, _ in bam_spec.members(s)]
    assert len(ms) >= 3 and max(len(m) for m in ms) <= 65536


# ---- 4. contracts ----
def _call(a, opts, cap=1 << 24):
    L = a.L
    a._upload_report_refs()
    out, so = np.zeros(cap, np.uint8), np.zeros(len(a.report_groups()) + 1, np.uint64)
    L.smr_format_bam_placed.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    rc = L.smr_format_bam_placed(a.h, C.cast(C.byref(opts), C.c_void_p), api._ptr(out), cap, api._ptr(so))
    return rc, L.smr_last_error(a.h).decode(), out, so


def test_contracts(golden):
    text = open(READS, "rb").read()
    a = _aligner(golden)
    a.upload_fastx(text)
    a.run_resident()
    rc, msg, _, _ = _call(a, api.report_opts(sam=True))
    assert rc == 2 and "no placed results" in msg
    a.place()   # without stats
    rc, msg, _, _ = _call(a, api.report_opts(sam=True))
    assert rc == 2 and "smr_aln_stats" in msg
    _run_and_place(a, text)
    for bad in (api.report_opts(), api.report_opts(sam=True, blast="1"), api.report_opts(sam=True, fastx=True),
                api.report_opts(sam=True, other=True), api.report_opts(sam=True, denovo=(0.9, 0.9))):
        rc, msg, _, _ = _call(a, bad)
        assert rc == 2 and "SAM alone" in msg
    # capacity: the sizes, then the same bytes
    rc0, _, big, so0 = _call(a, api.report_opts(sam=True))
    assert rc0 == 0 and int(so0[-1]) > 1000
    rc, _, _, so = _call(a, api.report_opts(sam=True), cap=100)
    assert rc == 5 and so.tolist() == so0.tolist()
    rc, _, again, so = _call(a, api.report_opts(sam=True), cap=int(so0[-1]))
    assert rc == 0 and bytes(again[:int(so[-1])]) == bytes(big[:int(so0[-1])])
    # the packed layout without a packed placement
    p = _aligner(golden, layout="packed")
    p.upload_fastx(text)
    p.set_place_stats(True)
    p.run_resident()
    rc, msg, _, _ = _call(p, api.report_opts(sam=True))
    assert rc == 4 and "packed" in msg


def test_qname_and_quality_refused(golden):
    recs = open(READS, "rb").read().split(b"\n")
    aligned = {row.split("\t")[0] for row in load_case("default")["sam"]}
    name_at = next(i for i in range(0, len(recs) - 3, 4) if recs[i][1:].split(b" ")[0].decode() in aligned)   # a read with a row
    a = _aligner(golden)
    long_name = list(recs)
    long_name[name_at] = b"@" + b"n" * 255 + b" tail"
    _run_and_place(a, b"\n".join(long_name))
    with pytest.raises(api.SmrError, match=r"SMR_ERR_ARG.*BAM: read %d of the batch has a QNAME longer than 254 bytes" % (name_at // 4)):
        a.format_placed_into(api.report_opts(sam=True), np.zeros(1 << 16, np.uint8), bam=True)
    ok = list(recs)
    ok[name_at] = b"@" + b"n" * 254
    _run_and_place(a, b"\n".join(ok))
    assert_bam_is_sam(a, what="254-byte QNAME")
    bad_q = list(recs)
    bad_q[name_at + 3] = b"\x7f" + bad_q[name_at + 3][1:]
    _run_and_place(a, b"\n".join(bad_q))
    with pytest.raises(api.SmrError, match=r"BAM: read %d of the batch has a quality byte outside" % (name_at // 4)):
        a.format_placed_into(api.report_opts(sam=True), np.zeros(1 << 16, np.uint8), bam=True)
    short_q = list(recs)
    short_q[name_at + 3] = short_q[name_at + 3][:-1]
    _run_and_place(a, b"\n".join(short_q))
    with pytest.raises(api.SmrError, match=r"BAM: read %d of the batch has a quality line whose length differs" % (name_at // 4)):
        a.format_placed_into(api.report_opts(sam=True), np.zeros(1 << 16, np.uint8), bam=True)


def test_mate_stream_batch(golden, tmp_path):
    m1, m2 = golden_mates(str(tmp_path))
    a = _aligner(golden)
    a.set_place_stats(True)
    n = 0
    for _ in a.stream_mates(m1, m2, batch_bytes=20000, piece_bytes=4096):
        a.run_resident()
        a.place()
        assert_bam_is_sam(a, api.report_opts(sam=True, paired_in=True), what="mates")
        n += 1
    assert n >= 2


# ---- 5. run_files and the command line ----
def assert_bam_file_is_sam(d):
    sam = open(os.path.join(d, "aligned.sam"), "rb").read().decode()
    text, refs, recs = bam_spec.decode_file(open(os.path.join(d, "aligned.bam"), "rb").read())
    head = "".join(line + "\n" for line in sam.splitlines() if line.startswith("@"))
    assert text == head
    body = [line for line in sam.splitlines() if not line.startswith("@")]
    assert [bam_spec.decode_record(r, [n for n, _ in refs]) for r in recs] == body
    return len(body)


KW = dict(gumbel=GUMBEL, minimal_score=[37, 36], cmd="x ", sam=True, bam=True)


@pytest.mark.parametrize("leg", ["single", "mates", "budget", "sq"])
def test_run_files(tmp_path, leg):
    reads = golden_mates(str(tmp_path)) if leg == "mates" else READS
    kw = dict(KW, paired_in=leg == "mates", sq=leg == "sq")
    if leg == "budget":   # one byte short of both indexes: two groups
        a = api.Aligner(0)
        _OPEN.append(a)
        for k, f in enumerate(REFS):
            st, _ = hostio.fasta_index_stats(f)
            a.build_index_device(k, f, hostio.split_by_parts(hostio.load_references(f), st), 36)
        kw["index_budget"] = a.index_residency()["device_search_bytes"] - 1
    r = api.run_files(REFS, reads, str(tmp_path / "out"), **kw)
    assert os.path.join(str(tmp_path / "out"), "aligned.bam") in r["paths"]
    assert assert_bam_file_is_sam(str(tmp_path / "out")) > 100


def test_run_files_zip_out_leaves_bam(tmp_path):
    r = api.run_files(REFS, READS, str(tmp_path / "z"), **dict(KW, zip_out=True))
    names = sorted(os.path.basename(p) for p in r["paths"])
    assert "aligned.bam" in names and "aligned.sam.gz" in names
    sam = gzip.open(str(tmp_path / "z" / "aligned.sam.gz")).read()
    (tmp_path / "z" / "aligned.sam").write_bytes(sam)
    assert assert_bam_file_is_sam(str(tmp_path / "z")) > 100


def test_run_files_packed_and_batches(tmp_path):
    from test_gpu_packed_results import MS, near_copy_inputs
    from test_gpu_placed_packed import _write_fastq
    nc = near_copy_inputs(str(tmp_path))
    fq = str(tmp_path / "reads.fq")
    _write_fastq(fq, nc["batch"])
    out = {}
    for k, bb in (("one", 1 << 30), ("three", os.path.getsize(fq) // 3 + 1)):
        r = api.run_files([nc["fasta"]], fq, str(tmp_path / k), api.default_params(num_alignments=0), gumbel=[(0.6, 0.33)],
                          minimal_score=[MS], sam=True, bam=True, cmd="x ", batch_bytes=bb, piece_bytes=4096)
        assert r["layout"] == "packed" and (r["batches"] == 1 if k == "one" else r["batches"] >= 3)
        assert assert_bam_file_is_sam(str(tmp_path / k)) > 10000
        out[k] = bam_spec.decode_file(open(str(tmp_path / k / "aligned.bam"), "rb").read())
    assert out["three"] == out["one"]   # the same header and records; the blocks differ, since no block spans two batches


def test_run_files_bam_without_sam(tmp_path):
    kw = dict(KW)
    r1 = api.run_files(REFS, READS, str(tmp_path / "a"), **kw)
    kw["sam"] = False
    r2 = api.run_files(REFS, READS, str(tmp_path / "b"), **kw)
    assert sorted(os.path.basename(p) for p in r2["paths"]) == ["aligned.bam", "aligned.log"]
    assert open(str(tmp_path / "a" / "aligned.bam"), "rb").read() == open(str(tmp_path / "b" / "aligned.bam"), "rb").read()
    assert r1["num_aligned"] == r2["num_aligned"]


def test_command_line(tmp_path):
    args = [a for r in REFS for a in ("-ref", r)] + ["-reads", READS, "-workdir", str(tmp_path), "-sam", "-bam", "-SQ"]
    for lam, K in GUMBEL:
        args += ["-gumbel", f"{lam},{K}"]
    assert cli.main(args) == 0
    d = str(tmp_path / "out")
    assert assert_bam_file_is_sam(d) > 100
    text = bam_spec.decode_file(open(os.path.join(d, "aligned.bam"), "rb").read())[0]
    assert re.search(r"@PG\tID:sortmerna\tVN:1.0\tCL:python -m sortmerna_b200 .*-bam -SQ .*\n", text)
