"""The coordinate-sorted aligned.bam and aligned.bam.bai on the device (smr_bam_sort_*, run_files(bam_sorted=True), -bam_sorted).
The sorted records are a stable sort by coordinate key of the unsorted smr_format_bam_placed records, so they decode to aligned.sam's
rows sorted the same way; the header is aligned.sam's with SO:coordinate; the records do not depend on the batching or the windows;
the index equals the from-spec writer of tests/bai_spec.py and answers region queries as brute force does; the contracts; the files
run_files and the command line write."""
import ctypes as C
import io
import os
import re
import struct

import numpy as np
import pytest

import bai_spec
import bam_spec
from conftest import GOLDEN, case_names, load_case
from integration_common import golden_mates
from summary_common import _STAMP
from sortmerna_b200 import __main__ as cli
from sortmerna_b200 import api, hostio
from test_gpu_bam import KW, READS, REFS, _OPEN, _aligner, _close_contexts, _groups, _run_and_place  # noqa: F401

pytestmark = pytest.mark.gpu


def _unsorted(a, opts):
    """the placed batch's records of smr_format_bam_placed, in the unsorted file's order"""
    buf, so = a.format_placed_into(opts, np.zeros(1 << 16, np.uint8), bam=True)
    return bam_spec.split_records(b"".join(bam_spec.check_stream(bytes(buf[int(so[g]):int(so[g + 1])])) for g in range(so.size - 1)))


def _stable_sorted(recs):
    return sorted(recs, key=lambda r: bai_spec.sort_key(*struct.unpack_from("<ii", r, 4), struct.unpack_from("<H", r, 18)[0]))


def _finish(a, runs, window, text=b"@HD\tVN:1.0\tSO:coordinate\n"):
    """the sorted file and its index from the runs (bytes of bam_sort_add, in order)"""
    head = a.bam_header(text)
    out = io.BytesIO()
    starts = np.cumsum([0] + [len(r) for r in runs])[:-1]
    bai = a.bam_sort_finish(io.BytesIO(b"".join(runs)), starts, out, len(head), window)
    return head + out.getvalue() + bam_spec.EOF_BLOCK, bai


def _check_file(data, bai, n_ref, regions=0, seed=1):
    """the file's framing, the BAI against the from-spec writer over the decoded file, and region queries: returns the records"""
    ms = bam_spec.members(data)
    assert all(len(m) <= 65536 for m, _ in ms)
    got = bai_spec.file_records(data)
    laid = [bai_spec.fields(r)[:4] + (vb, ve) for r, vb, ve in got]
    assert bai == bai_spec.write_bai(n_ref, laid)
    ix = bai_spec.parse_bai(bai)
    rng = np.random.default_rng(seed)
    lens = [r[1] for r in bam_spec.decode_file(data)[1]]
    qs = []
    for ref, ln in enumerate(lens):
        qs += [(ref, 0, ln)]
        if regions:
            qs += [(ref, *sorted(int(x) for x in rng.integers(0, ln + 1, 2))) for _ in range(regions)]
            qs += [(ref, b, min(ln, b + w)) for b in range(0, ln, 16384) for w in (1, 16384, 131072)]
    for ref, beg, end in qs:
        end = max(end, beg + 1)
        assert bai_spec.query(ix, laid, ref, beg, end) == bai_spec.brute(laid, ref, beg, end), (ref, beg, end)
    return [r for r, _, _ in got]


def assert_sorted_is_sam(a, opts=None, window=1 << 30, what=""):
    o = opts if opts is not None else api.report_opts(sam=True)
    sbuf, sso = a.format_placed_into(o, np.zeros(1 << 20, np.uint8))
    rows = bytes(sbuf[:int(sso[len(a.report_groups())])]).decode().splitlines()
    unsorted = _unsorted(a, o)
    a.bam_sort_begin()
    buf, nb = a.bam_sort_add(o, np.zeros(16, np.uint8))
    run = bytes(buf[:nb])
    want = _stable_sorted(unsorted)
    assert bam_spec.split_records(run) == want, what
    names = [n for ids, _ in _groups(a) for n in ids]
    text = "@HD\tVN:1.0\tSO:coordinate\n@PG\tID:x\n"
    data, bai = _finish(a, [run], window, text.encode())
    got_text, refs, recs = bam_spec.decode_file(data)
    assert got_text == text and [n for n, _ in refs] == names and recs == want
    keyed = sorted(range(len(rows)), key=lambda i: bai_spec.sort_key(names.index(rows[i].split("\t")[2]), int(rows[i].split("\t")[3]) - 1,
                                                                      int(rows[i].split("\t")[1])))
    decoded = [bam_spec.decode_record(r, names) for r in recs]
    # rows of one reference name in two groups map to the first; the golden references have unique names
    assert decoded == [rows[i] for i in keyed], what
    _check_file(data, bai, len(names))
    return recs


# ---- 1. one batch ----
@pytest.mark.parametrize("case", case_names())
def test_golden_cases_strided(golden, case):
    a = _aligner(golden, load_case(case))
    _run_and_place(a, open(READS, "rb").read())
    assert_sorted_is_sam(a, what=case)


@pytest.mark.parametrize("stride", [1, 16])
def test_case_all_packed(golden, stride):
    a = _aligner(golden, load_case("all"), "packed", stride)
    _run_and_place(a, open(READS, "rb").read())
    assert len(assert_sorted_is_sam(a, window=65536, what=f"packed {stride}")) > 1000


# ---- 2. runs and windows ----
def _stream_sorted(a, reads, batch_bytes, window):
    opts = api.report_opts(sam=True)
    a.bam_sort_begin()
    runs, unsorted, buf = [], [], np.zeros(16, np.uint8)
    for _ in a.stream_fastx(reads, batch_bytes=batch_bytes, piece_bytes=1 << 16):
        a.run_resident()
        a.place_packed() if a.layout == "packed" else a.place()
        unsorted += _unsorted(a, opts)
        buf, nb = a.bam_sort_add(opts, buf)
        runs.append(bytes(buf[:nb]))
    data, bai = _finish(a, runs, window)
    return data, bai, runs, unsorted


def _invariance(a, reads, n_ref):
    size = os.path.getsize(reads)
    out = {}
    for batches, window in ((1, 1 << 40), (3, 65536), (3, 1 << 20), (5, 300000)):
        data, bai, runs, unsorted = _stream_sorted(a, reads, size + 1 if batches == 1 else size // batches + 1, window)
        assert len(runs) >= batches
        assert a.bam_sort_seconds["windows"] >= (2 if window == 65536 else 1)
        out[(batches, window)] = _check_file(data, bai, n_ref)
        assert out[(batches, window)] == _stable_sorted(unsorted)
    first = next(iter(out.values()))
    assert all(v == first for v in out.values()) and len(first) > 1000


def test_invariance_bench_sample(tmp_path):
    from test_gpu_bundled_sets import workload
    from tools import stage_data
    import json
    fastas, reads, kw = workload(str(tmp_path))
    idx_dir, _ = stage_data.ensure_indexes(fastas, str(tmp_path / "idx"), **kw)
    pre = hostio.find_index_prefixes(idx_dir)
    a = api.Aligner(0)
    _OPEN.append(a)
    a.set_params(api.default_params())
    a.set_place_stats(True)
    ms = json.load(open(os.path.join(GOLDEN, "bench_workload.json")))["minimal_score"]
    n_ref = 0
    for k, f in enumerate(fastas):
        p = pre[os.path.basename(f)]
        refs = hostio.load_references(f)
        n_ref += refs.n
        a.load_index_part(k, 0, p, refs, ms[k], (18, 9, 3), hostio.parse_stats(p).lnwin)
    _invariance(a, reads, n_ref)


def test_invariance_near_copies_packed(tmp_path):
    from test_gpu_packed_results import MS, near_copy_inputs
    from test_gpu_placed_packed import _write_fastq
    nc = near_copy_inputs(str(tmp_path))
    fq = str(tmp_path / "reads.fq")
    _write_fastq(fq, nc["batch"])
    a = api.Aligner(0)
    _OPEN.append(a)
    a.set_params(api.default_params(num_alignments=0))
    a.set_place_stats(True)
    refs = hostio.load_references(nc["fasta"])
    st, _ = hostio.fasta_index_stats(nc["fasta"])
    a.build_index_device(0, nc["fasta"], hostio.split_by_parts(refs, st), MS)
    a.set_aln_layout("packed")
    _invariance(a, fq, refs.n)


# ---- 3. the index on a reference with bins at levels 3-5 ----
def _boundary_inputs(d):
    """two seeded references (200 kb and 60 kb) and a third no read comes from; reads of 100-300 nt drawn across 16 kb and 128 kb
    boundaries and at random, on both strands"""
    rng = np.random.default_rng(2024)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    seqs = [acgt[rng.integers(0, 4, n)].tobytes() for n in (200000, 60000, 5000)]
    fasta = os.path.join(d, "bnd.fasta")
    with open(fasta, "wb") as f:
        for k, s in enumerate(seqs):
            f.write(b">ref%d\n" % k + b"\n".join(s[i:i + 80] for i in range(0, len(s), 80)) + b"\n")
    comp = bytes.maketrans(b"ACGT", b"TGCA")
    fq = os.path.join(d, "bnd.fq")
    with open(fq, "wb") as f:
        for i in range(3000):
            k = 0 if i % 4 else 1
            L = int(rng.integers(100, 301))
            n = len(seqs[k])
            if i % 3 == 0:
                b = int(rng.choice([16384 * j for j in range(1, n // 16384 + 1)])) - int(rng.integers(1, L))
            elif i % 3 == 1 and k == 0:
                b = 131072 - int(rng.integers(1, L))
            else:
                b = int(rng.integers(0, n - L))
            b = max(0, min(b, n - L))
            s = seqs[k][b:b + L]
            if rng.random() < 0.5:
                s = s.translate(comp)[::-1]
            f.write(b"@q%d\n%s\n+\n%s\n" % (i, s, b"I" * L))
    return fasta, fq


def test_index_on_boundaries(tmp_path):
    fasta, fq = _boundary_inputs(str(tmp_path))
    d = str(tmp_path / "out")
    r = api.run_files([fasta], fq, d, gumbel=[(0.6, 0.33)], minimal_score=[150], cmd="x ", sam=True, bam_sorted=True,
                      batch_bytes=os.path.getsize(fq) // 3 + 1, piece_bytes=1 << 16)
    assert r["batches"] >= 3 and r["num_aligned"] > 2500
    data = open(os.path.join(d, "aligned.bam"), "rb").read()
    bai = open(os.path.join(d, "aligned.bam.bai"), "rb").read()
    recs = _check_file(data, bai, 3, regions=200, seed=7)
    bins = {bai_spec.fields(x)[3] for x in recs}
    assert any(73 <= b < 585 for b in bins) and any(585 <= b < 4681 for b in bins) and any(b >= 4681 for b in bins)
    ix = bai_spec.parse_bai(bai)
    assert len(ix[0]["intv"]) >= 12 and ix[2] == dict(bins={}, intv=[])
    assert_file_is_sam(d)


# ---- 4. contracts ----
def _fn(a, name, *types):
    f = getattr(a.L, name)
    f.argtypes = [C.c_void_p] + list(types)
    return f


def _err(a):
    return a.L.smr_last_error(a.h).decode()


def test_contracts(golden):
    V, U = C.c_void_p, C.c_uint64
    text = open(READS, "rb").read()
    a = _aligner(golden)
    _run_and_place(a, text)
    opts = api.report_opts(sam=True)
    add = _fn(a, "smr_bam_sort_add_placed", V, V, U, V)
    plan = _fn(a, "smr_bam_sort_plan", U, U, V, U, V)
    win = _fn(a, "smr_bam_sort_window", U, V, U, V, U, V)
    idx = _fn(a, "smr_bam_sort_index", V, U, V)
    nb = np.zeros(1, np.uint64)
    o = C.cast(C.byref(opts), V)
    # no open accumulator
    assert add(a.h, o, None, 0, api._ptr(nb)) == 2 and "smr_bam_sort_begin" in _err(a)
    assert plan(a.h, 1 << 20, 0, None, 0, api._ptr(nb)) == 2
    assert idx(a.h, None, 0, api._ptr(nb)) == 2
    a.bam_sort_begin()
    # add: the size, the accumulator unchanged, the same bytes on retry, one append
    assert add(a.h, o, None, 0, api._ptr(nb)) == 5
    size = int(nb[0])
    small = np.zeros(size - 1, np.uint8)
    assert add(a.h, o, api._ptr(small), small.size, api._ptr(nb)) == 5 and int(nb[0]) == size
    buf = np.zeros(size, np.uint8)
    assert add(a.h, o, api._ptr(buf), size, api._ptr(nb)) == 0
    run = bytes(buf)
    assert bam_spec.split_records(run) == _stable_sorted(_unsorted(a, opts))
    # index before plan; window before plan
    assert idx(a.h, None, 0, api._ptr(nb)) == 2 and "smr_bam_sort_plan" in _err(a)
    # plan: capacity names the windows
    assert plan(a.h, 30000, 100, None, 0, api._ptr(nb)) == 5
    nw = int(nb[0])
    assert nw >= 3
    rg = np.zeros(nw * 2, np.uint64)
    assert plan(a.h, 30000, 100, api._ptr(rg), rg.size, api._ptr(nb)) == 0 and int(nb[0]) == nw
    assert rg[0] == 0 and rg[-1] == size and all(rg[2 * w + 1] == rg[2 * w + 2] for w in range(nw - 1))   # one run: consecutive ranges
    stage = np.frombuffer(run, np.uint8)
    out = np.zeros(1 << 20, np.uint8)
    # a window out of order, a wrong length, a wrong block_size
    assert win(a.h, 1, api._ptr(stage[int(rg[2]):]), int(rg[3] - rg[2]), api._ptr(out), out.size, api._ptr(nb)) == 2 and "order" in _err(a)
    w0 = stage[:int(rg[1])].copy()
    assert win(a.h, 0, api._ptr(w0), w0.size - 1, api._ptr(out), out.size, api._ptr(nb)) == 2 and "staged" in _err(a)
    bad = w0.copy()
    bad[0] ^= 1
    assert win(a.h, 0, api._ptr(bad), bad.size, api._ptr(out), out.size, api._ptr(nb)) == 2 and "block_size" in _err(a)
    # window capacity: the size, then the same bytes
    assert win(a.h, 0, api._ptr(w0), w0.size, api._ptr(out), 10, api._ptr(nb)) == 5
    need = int(nb[0])
    assert win(a.h, 0, api._ptr(w0), w0.size, api._ptr(out), need, api._ptr(nb)) == 0 and int(nb[0]) == need
    blocks0 = bytes(out[:need])
    assert idx(a.h, None, 0, api._ptr(nb)) == 2 and "last window" in _err(a)
    # an index part's report ids set again after begin
    a._report_refs.clear()
    a._upload_report_refs()
    assert win(a.h, 1, api._ptr(stage[int(rg[2]):]), int(rg[3] - rg[2]), api._ptr(out), out.size, api._ptr(nb)) == 2
    assert "begin the sorted BAM again" in _err(a)
    # begin again discards the open accumulator: a whole file from one run, window 0 as before
    a.bam_sort_begin()
    buf2, nb2 = a.bam_sort_add(opts, np.zeros(16, np.uint8))
    assert bytes(buf2[:nb2]) == run
    data, bai = _finish(a, [run], 30000)
    head = a.bam_header(b"@HD\tVN:1.0\tSO:coordinate\n")
    assert data[len(head):len(head) + need] == blocks0   # window 0's blocks do not depend on where the window lands
    assert _check_file(data, bai, len([n for ids, _ in _groups(a) for n in ids])) == bam_spec.split_records(run)


def test_no_alignments(golden):
    """a run with no alignments: the header, the EOF block and an index of empty references"""
    a = _aligner(golden)
    _run_and_place(a, b"@x\n" + b"A" * 60 + b"\n+\n" + b"I" * 60 + b"\n")
    a.bam_sort_begin()
    buf, nb = a.bam_sort_add(api.report_opts(sam=True), np.zeros(16, np.uint8))
    assert nb == 0
    data, bai = _finish(a, [b""], 1 << 20)
    n_ref = len([n for ids, _ in _groups(a) for n in ids])
    assert bam_spec.decode_file(data)[2] == []
    assert bai == b"BAI\1" + struct.pack("<i", n_ref) + struct.pack("<ii", 0, 0) * n_ref + struct.pack("<Q", 0)


# ---- 5. run_files and the command line ----
def assert_file_is_sam(d):
    sam = open(os.path.join(d, "aligned.sam"), "rb").read().decode()
    data = open(os.path.join(d, "aligned.bam"), "rb").read()
    text, refs, recs = bam_spec.decode_file(data)
    head = "".join(line + "\n" for line in sam.splitlines() if line.startswith("@"))
    assert "\tSO:unsorted\n" in head and text == head.replace("\tSO:unsorted\n", "\tSO:coordinate\n", 1)
    names = [n for n, _ in refs]
    body = [line for line in sam.splitlines() if not line.startswith("@")]
    key = [bai_spec.sort_key(names.index(f[2]), int(f[3]) - 1, int(f[1])) for f in (row.split("\t") for row in body)]
    want = [body[i] for i in sorted(range(len(body)), key=lambda i: key[i])]
    assert [bam_spec.decode_record(r, names) for r in recs] == want
    _check_file(data, open(os.path.join(d, "aligned.bam.bai"), "rb").read(), len(refs), regions=20)
    return len(body)


def _same_other_files(d1, d2):
    """every file but aligned.bam and its index byte for byte; aligned.log apart from its timestamp, which the runs' clock writes"""
    n1 = sorted(f for f in os.listdir(d1) if not f.startswith("aligned.bam"))
    n2 = sorted(f for f in os.listdir(d2) if not f.startswith("aligned.bam"))
    assert n1 == n2 and "aligned.log" in n1
    for f in n1:
        a, b = (open(os.path.join(d, f), "rb").read() for d in (d1, d2))
        if f == "aligned.log":
            a, b = ([ln for ln in x.decode().split("\n") if not _STAMP.match(ln)] for x in (a, b))
        assert a == b, f


@pytest.mark.parametrize("leg", ["single", "mates", "budget", "packed", "sq", "zip_out", "no_sam"])
def test_run_files(tmp_path, leg):
    reads = golden_mates(str(tmp_path)) if leg == "mates" else READS
    kw = dict(KW, paired_in=leg == "mates", sq=leg == "sq", zip_out=leg == "zip_out")
    kw.pop("bam")
    if leg == "budget":   # one byte short of both indexes: two groups
        a = api.Aligner(0)
        _OPEN.append(a)
        for k, f in enumerate(REFS):
            st, _ = hostio.fasta_index_stats(f)
            a.build_index_device(k, f, hostio.split_by_parts(hostio.load_references(f), st), 36)
        kw["index_budget"] = a.index_residency()["device_search_bytes"] - 1
    if leg == "packed":
        kw["params"] = api.default_params(num_alignments=0)
    base = api.run_files(REFS, reads, str(tmp_path / "base"), **kw)
    r = api.run_files(REFS, reads, str(tmp_path / "sorted"), bam_sorted=True, **dict(kw, sam=True))
    d = str(tmp_path / "sorted")
    assert {"aligned.bam", "aligned.bam.bai"} <= {os.path.basename(p) for p in r["paths"]}
    assert "bam_sort" in r["seconds"] and "bam_sort" not in base["seconds"]
    assert not [f for f in os.listdir(d) if f.startswith(".part")]
    if leg == "zip_out":
        import gzip
        (tmp_path / "sorted" / "aligned.sam").write_bytes(gzip.open(os.path.join(d, "aligned.sam.gz")).read())
    assert assert_file_is_sam(d) > 100
    if leg == "zip_out":
        os.unlink(os.path.join(d, "aligned.sam"))
    if leg == "no_sam":   # without -sam: only the BAM files and the log
        r2 = api.run_files(REFS, reads, str(tmp_path / "nosam"), bam_sorted=True, **dict(kw, sam=False))
        assert sorted(os.path.basename(p) for p in r2["paths"]) == ["aligned.bam", "aligned.bam.bai", "aligned.log"]
        for f in ("aligned.bam", "aligned.bam.bai"):
            assert open(os.path.join(d, f), "rb").read() == open(str(tmp_path / "nosam" / f), "rb").read()
    else:
        _same_other_files(str(tmp_path / "base"), d)


def test_command_line(tmp_path):
    args = [a for r in REFS for a in ("-ref", r)] + ["-reads", READS, "-workdir", str(tmp_path), "-sam", "-bam_sorted", "-SQ"]
    for lam, K in KW["gumbel"]:
        args += ["-gumbel", f"{lam},{K}"]
    assert cli.main(args) == 0
    d = str(tmp_path / "out")
    assert os.path.exists(os.path.join(d, "aligned.bam.bai"))
    assert assert_file_is_sam(d) > 100
    text = bam_spec.decode_file(open(os.path.join(d, "aligned.bam"), "rb").read())[0]
    assert re.search(r"@HD\tVN:1.0\tSO:coordinate\n", text)
    assert re.search(r"@PG\tID:sortmerna\tVN:1.0\tCL:python -m sortmerna_b200 .*-bam_sorted -SQ .*\n", text)
