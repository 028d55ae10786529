"""The packed result layout (smr_set_aln_layout(SMR_ALNS_PACKED)) on the GPU.  Read r's alignments follow the reads before it with no
stride; a run stores at most the stride per read, and the reads that accept more are run again at their own count in batches of
their own.  Checked here:
- every golden case, packed against strided on the same batch (api.unpack_alns), with no read run again;
- case_all (up to 100 alignments per read) with a first-pass stride of 1, 2 and 16: reads run again (SMR_VERBOSE), results equal the
  oracle's, SAM rows equal the reference's;
- a seeded near-copy database where reads store up to about 1,600 alignments: results equal the oracle's and strided at the grown
  stride, with SMR_RETRY_SLOTS small enough to split the re-run into sub-batches and run some reads alone;
- reads that overflow their scratch as well as the stride: results equal the oracle's;
- the report side, packed against strided byte for byte, and against the reference binary;
- the contracts of the packed calls."""
import ctypes as C
import gzip
import os
import re
import shutil
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, case_names, load_case
from helpers import assert_same_results, params_kwargs_from_args, strip_seq
from integration_common import REF_DIR, golden_mates
from sortmerna_b200 import api, hostio

pytestmark = pytest.mark.gpu

READS = os.path.join(GOLDEN, "reads_mix.fq")
BLAST = "1 cigar qcov qstrand"
WORK = ("num_short", "sw_calls", "sw_cells", "windows", "trie_nodes", "buckets", "bucket_entries", "pos_entries", "lis_calls")
RERUN = re.compile(r"packed results: (\d+) reads stored more than (\d+) alignments and were run again at their own count in (\d+) sub-batches "
                   r"\(largest count (\d+)\)")

_OPEN = []


@pytest.fixture(autouse=True)
def _close_contexts():
    """a failing test must not leave its context (and its device memory) to the next"""
    yield
    while _OPEN:
        _OPEN.pop().close()


def _ora():
    from oracle import ora
    return ora


def _aligner(golden, exp, layout="strided", slots=None, track=True):
    """track: closed after the test (a module fixture's aligner is not)"""
    a = api.Aligner(0)
    if track:
        _OPEN.append(a)
    a.set_params(api.default_params(**params_kwargs_from_args(exp["args"])))
    tot = int(np.diff(golden["batch"].off.astype(np.int64)).sum())
    for k in range(2):
        a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], exp["log"]["minimal_score"][k], (18, 9, 3), golden["stats"][k].lnwin)
        a.set_report_scoring(k, exp["log"]["lambda_"][k], exp["log"]["K"][k], *hostio.evalue_params(golden["stats"][k], exp["log"]["K"][k], tot, golden["batch"].n))
    a.set_aln_layout(layout)
    if slots:
        a.set_aln_slots(slots)
    return a


def _text():
    return open(READS, "rb").read()


def _rows(b):
    return b.decode().split("\n")[:-1] if b else []


def _cigars(out, slots):
    """the CIGAR words of every stored alignment, in (read, slot) order"""
    res, alns, cig = out["res"], out["alns"], out["cigar"]
    return [cig[int(alns[r * slots + k]["cigar_off"]):][:int(alns[r * slots + k]["cigar_len"])].tolist()
            for r in range(res.shape[0]) for k in range(int(res["n_align"][r]))]


def assert_packed_equals_strided(p, s, what, counters=True):
    """a packed result against a strided one of the same batch: results, alignments (CIGAR offsets aside), CIGAR words per alignment,
    stats, Readstats counters and matched; the work counters too when no read was run again"""
    slots = s["slots"]
    assert p["slots"] == 0 and p["aln_off"].tolist() == [0] + np.cumsum(p["res"]["n_align"]).tolist()
    assert p["alns"].shape[0] == int(p["res"]["n_align"].sum())
    u = api.unpack_alns(p, slots)
    assert np.array_equal(u["res"], s["res"]), what
    keep = [f for f in api.ALN_DTYPE.names if f != "cigar_off"]
    assert np.array_equal(u["alns"][keep], s["alns"][keep]), what
    assert _cigars(u, slots) == _cigars(s, slots), what
    if s.get("stats") is not None:
        assert np.array_equal(u["stats"], s["stats"]), what
    assert p["matched"].tolist() == s["matched"].tolist(), what
    assert p["counters"]["num_aligned"] == s["counters"]["num_aligned"], what
    if counters:
        assert {k: p["counters"][k] for k in WORK} == {k: s["counters"][k] for k in WORK}, what


def _reruns(err):
    m = RERUN.findall(err)
    return [tuple(int(x) for x in t) for t in m]


# ---- 1. every golden case, packed against strided ----
@pytest.mark.parametrize("case", case_names())
def test_golden_cases_packed_equal_strided(golden, case, capfd, monkeypatch):
    exp = load_case(case)
    b = golden["batch"]
    s = _aligner(golden, exp).align(b.cat, b.off, with_stats=True)   # the all-alignments cases grow the stride
    monkeypatch.setenv("SMR_VERBOSE", "1")
    capfd.readouterr()
    p = _aligner(golden, exp, "packed", s["slots"]).align(b.cat, b.off, with_stats=True)
    assert not _reruns(capfd.readouterr().err)        # the first run's stride was enough for every read
    assert_packed_equals_strided(p, s, case)
    if case == "all":
        assert s["slots"] >= 100 and int(p["res"]["n_align"].max()) >= 100


# ---- 2. case_all with a small first-pass stride ----
@pytest.fixture(scope="module")
def all_oracle(golden):
    ora = _ora()
    exp = load_case("all")
    oix = [ora.OracleIndex(p, 0, s.lnwin) for p, s in zip(golden["prefixes"], golden["stats"])]
    return ora.align(oix, [0, 1], [0, 0], 2, golden["refs"], exp["log"]["minimal_score"], [18, 9, 3, 18, 9, 3],
                     ora.default_params(**params_kwargs_from_args(exp["args"])), golden["batch"], nthreads=4)


@pytest.mark.parametrize("stride", [1, 2, 16])
def test_case_all_reruns_equal_oracle_and_reference(golden, all_oracle, stride, capfd, monkeypatch):
    exp = load_case("all")
    b = golden["batch"]
    monkeypatch.setenv("SMR_VERBOSE", "1")
    capfd.readouterr()
    a = _aligner(golden, exp, "packed", stride)
    p = a.align(b.cat, b.off, with_stats=True)
    runs = _reruns(capfd.readouterr().err)
    n_over = int((all_oracle["res"]["n_align"] > stride).sum())
    assert runs and runs[-1][0] == n_over > 0 and runs[-1][1] == stride
    assert runs[-1][3] == int(all_oracle["res"]["n_align"].max())
    assert_same_results(api.unpack_alns(p, all_oracle["slots"]), all_oracle, f"stride {stride}")
    assert p["matched"].tolist() == all_oracle["matched"].tolist()
    assert p["counters"]["num_aligned"] == all_oracle["counters"]["num_aligned"] == exp["log"]["passing"]
    s = a.format_reports(p, _text(), sam=True)
    sam = strip_seq([r for g in s["sam"] for r in _rows(g)])
    assert len(sam) == len(exp["sam"]) == 5497 and sam == exp["sam"]


# ---- 3 / 4. a near-copy database: over a thousand alignments per read; scratch overflow on top ----
SEED = 20261018
MS = 120


def _near_copies(rng, groups, length):
    """groups: copies per group; each group = copies of one random ancestor at 0.2-1 % substitutions"""
    out = []
    for n in groups:
        root = rng.integers(0, 4, length, dtype=np.uint8)
        for _ in range(n):
            hit = rng.random(length) < rng.uniform(0.002, 0.01)
            out.append(np.where(hit, (root + rng.integers(1, 4, length, dtype=np.uint8)) & 3, root).astype(np.uint8))
    return out


def _reads_from(rng, refs, picks, read_len=150, err=0.01):
    out = []
    for k in picks:
        s = refs[k]
        p = int(rng.integers(0, s.size - read_len + 1))
        r = s[p:p + read_len].copy()
        hit = rng.random(read_len) < err
        r[hit] = (r[hit] + rng.integers(1, 4, int(hit.sum()), dtype=np.uint8)) & 3
        out.append((3 - r)[::-1].copy() if rng.random() < 0.5 else r)
    return out


def near_copy_inputs(d):
    """One group of 2,000 copies and one of 200 copies of a 300 nt ancestor; 12 reads from each group and 4 random reads.  A read of
    the large group stores 950-1,600 alignments, one of the small group 100-170; the oracle needs a few seconds for them.  The
    database and its index go to d."""
    rng = np.random.default_rng(SEED)
    refs = _near_copies(rng, (2000, 200), 300)
    reads = _reads_from(rng, refs, list(rng.integers(0, 2000, 12)) + list(rng.integers(2000, 2200, 12)))
    reads += [rng.integers(0, 4, 150, dtype=np.uint8) for _ in range(4)]
    order = rng.permutation(len(reads))
    reads = [reads[i] for i in order]
    acgt = np.frombuffer(b"ACGT", np.uint8)
    fasta = os.path.join(d, "copies.fasta")
    with open(fasta, "wb") as f:
        for k, s in enumerate(refs):
            f.write(b">copy_%05d\n" % k + acgt[s].tobytes() + b"\n")
    prefix = os.path.join(d, "copies")
    api.build_index(fasta, prefix)
    batch = hostio.pack_reads([b"r%d" % k for k in range(len(reads))], [acgt[r].tobytes() for r in reads])
    return dict(fasta=fasta, prefix=prefix, refs=hostio.load_references(fasta), stats=hostio.parse_stats(prefix), batch=batch)


def near_copy_oracle(nc):
    ora = _ora()
    oix = [ora.OracleIndex(nc["prefix"], 0, nc["stats"].lnwin)]
    return ora.align(oix, [0], [0], 1, [nc["refs"]], [MS], [18, 9, 3], ora.default_params(num_alignments=0), nc["batch"], nthreads=4)


@pytest.fixture(scope="module")
def near_copies():
    d = tempfile.mkdtemp(prefix="smr_packed_")
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


def test_near_copies_equal_oracle_and_strided(near_copies, near_oracle, capfd, monkeypatch):
    nc = near_copies
    cnt = near_oracle["res"]["n_align"]
    assert int(cnt.max()) >= 1500 and int(((cnt > 100) & (cnt < 400)).sum()) >= 6 and int((cnt == 0).sum()) >= 4
    b = nc["batch"]
    s = _near_aligner(nc, "strided").align(b.cat, b.off, with_stats=True)
    monkeypatch.setenv("SMR_VERBOSE", "1")
    monkeypatch.setenv("SMR_RETRY_SLOTS", "1000")   # read at smr_init: sub-batches of the small group, the large group's reads alone
    capfd.readouterr()
    p = _near_aligner(nc, "packed").align(b.cat, b.off, with_stats=True)
    runs = _reruns(capfd.readouterr().err)
    assert runs and runs[-1][0] == int((cnt > 16).sum()) and runs[-1][3] == int(cnt.max())
    big = int((cnt > 1000).sum())
    assert runs[-1][2] >= big + 2          # every read of the large group alone, the small group's in a few sub-batches
    assert_same_results(api.unpack_alns(p, near_oracle["slots"]), near_oracle, "near copies")
    assert p["matched"].tolist() == near_oracle["matched"].tolist()
    assert p["counters"]["num_aligned"] == near_oracle["counters"]["num_aligned"]
    assert_packed_equals_strided(p, s, "near copies", counters=False)


L = 18


def core_variants(core):
    """every one-edit variant of an 18 nt core: substitutions, insertions (19-mers) and deletions (17-mers)"""
    out = set()
    for i in range(L):
        for b in range(4):
            if b != core[i]:
                v = core.copy(); v[i] = b; out.add(v.tobytes())
            out.add(np.concatenate([core[:i], [b], core[i:]]).astype(np.uint8).tobytes())
        out.add(np.concatenate([core[:i], core[i + 1:]]).astype(np.uint8).tobytes())
    out.discard(core.tobytes())
    return [np.frombuffer(v, np.uint8) for v in sorted(out)]


def both_overflow_inputs(d):
    """200 near copies of a 300 nt ancestor, and four references per one-edit variant of an 18 nt core between random 60 nt flanks
    that differ in the base next to the variant (as test_gpu_overflow_retry.py builds its seed-lane case): a window on the core hits
    more ids than a seed lane holds at scale 1.  Reads: 8 from the copies with the core written over 18 of their bases (they overflow
    the seed lane and then store 100-170 alignments), 8 plain ones from the copies."""
    rng = np.random.default_rng(SEED + 1)
    refs = _near_copies(rng, (200,), 300)
    core = rng.integers(0, 4, L, dtype=np.uint8)
    for v in core_variants(core):
        for c in range(4):
            a, b = rng.integers(0, 4, 60, dtype=np.uint8), rng.integers(0, 4, 60, dtype=np.uint8)
            a[-1], b[0] = (c + 1) & 3, c
            x = np.concatenate([a, v, b]).astype(np.uint8)
            if core.tobytes() not in x.tobytes():
                refs.append(x)
    reads = []
    for k, r in enumerate(_reads_from(rng, refs[:200], list(rng.integers(0, 200, 16)))):
        if k % 2 == 0:
            r = r.copy(); r[72:72 + L] = core   # a window of the first seed pass (skip 18)
        reads.append(r)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    fasta = os.path.join(d, "both.fasta")
    with open(fasta, "wb") as f:
        for k, x in enumerate(refs):
            f.write(b">ref_%05d\n" % k + acgt[x].tobytes() + b"\n")
    prefix = os.path.join(d, "both")
    api.build_index(fasta, prefix)
    batch = hostio.pack_reads([b"r%d" % k for k in range(len(reads))], [acgt[r].tobytes() for r in reads])
    return dict(fasta=fasta, prefix=prefix, refs=hostio.load_references(fasta), stats=hostio.parse_stats(prefix), batch=batch)


def test_scratch_and_slot_overflow_equal_oracle(tmp_path, capfd, monkeypatch):
    """reads that overflow their scratch and store more alignments than the stride: retried at 8x with room for the stride, then
    run again at their exact count"""
    nc = both_overflow_inputs(str(tmp_path))
    want = near_copy_oracle(nc)
    cnt = want["res"]["n_align"]
    assert int((cnt > 16).sum()) >= 8
    monkeypatch.setenv("SMR_VERBOSE", "1")
    capfd.readouterr()
    b = nc["batch"]
    p = _near_aligner(nc, "packed").align(b.cat, b.off, with_stats=True)
    err = capfd.readouterr().err
    assert "overflowed their scratch" in err
    runs = _reruns(err)
    assert runs and runs[-1][0] == int((cnt > 16).sum()) and runs[-1][3] == int(cnt.max())
    assert_same_results(api.unpack_alns(p, want["slots"]), want, "scratch and slots")
    assert p["matched"].tolist() == want["matched"].tolist()
    assert p["counters"]["num_aligned"] == want["counters"]["num_aligned"]


def test_near_copies_first_stride_covers_small_group(near_copies, near_oracle, capfd, monkeypatch):
    """a first-pass stride between the groups: only the large group's reads are run again for their count"""
    nc = near_copies
    cnt = near_oracle["res"]["n_align"]
    monkeypatch.setenv("SMR_VERBOSE", "1")
    capfd.readouterr()
    a = _near_aligner(nc, "packed")
    a.set_aln_slots(600)
    b = nc["batch"]
    p = a.align(b.cat, b.off, with_stats=True)
    runs = _reruns(capfd.readouterr().err)
    assert runs and runs[-1][0] == int((cnt > 600).sum())
    assert_same_results(api.unpack_alns(p, near_oracle["slots"]), near_oracle, "near copies, stride 600")


# ---- 5. report side ----
@pytest.fixture(scope="module")
def all_pair(golden):
    """case_all's batch, strided at its grown stride and packed from a first-pass stride of 4"""
    exp = load_case("all")
    b = golden["batch"]
    sa = _aligner(golden, exp, track=False)
    s = sa.align(b.cat, b.off, with_stats=True)
    pa = _aligner(golden, exp, "packed", 4, track=False)
    p = pa.align(b.cat, b.off, with_stats=True)
    yield sa, s, pa, p
    sa.close()
    pa.close()


def test_reports_packed_equal_strided(all_pair):
    sa, s, pa, p = all_pair
    t = _text()
    for kw in (dict(sam=True, blast=BLAST), dict(fastx=True, other=True, denovo=(0.97, 0.97))):
        for gz in (False, True):
            x, y = pa.format_reports(p, t, gzip=gz, **kw), sa.format_reports(s, t, gzip=gz, **kw)
            assert x == y, (kw, gz)
    x = sa.format_reports(s, t, sam=True)["sam"]
    assert sum(len(_rows(g)) for g in x) == 5497
    for gz in (False, True):
        assert pa.format_blast_pairwise(p, t, gzip=gz) == sa.format_blast_pairwise(s, t, gzip=gz)
    for a, o in ((pa, p), (sa, s)):
        a.otu_begin(0.9, 0.9)
        assert a.otu_add(o, t) > 0
    mp, ms = pa.otu_finish(), sa.otu_finish()
    assert mp == ms and mp["n_yid_ycov"] > 0
    dp, ds = pa.denovo_stats(p, t, 0.9, 0.9), sa.denovo_stats(s, t, 0.9, 0.9)
    assert np.array_equal(dp[0], ds[0]) and dp[1] == ds[1]
    bp, bs = api.pack_kvdb_blobs(p, 0, dp[0]), api.pack_kvdb_blobs(s, 0, ds[0])
    assert bp[0].tobytes() == bs[0].tobytes() and np.array_equal(bp[1], bs[1])


def _writer_run(golden, d, layout, reads, log):
    al = api.Aligner(0)
    _OPEN.append(al)
    al.set_params(api.default_params(num_alignments=0))
    al.load_index_part(0, 0, golden["prefixes"][1], golden["refs"][1], log["minimal_score"][0], (18, 9, 3), golden["stats"][1].lnwin)
    al.set_aln_layout(layout)
    al.set_aln_slots(2 if layout == "packed" else 256)   # download() does not grow a strided stride
    w = api.ReportWriter(d, al, sam=True, fastx=True, other=True, out2=True, denovo=(0.9, 0.9))
    for _ in al.stream_mates(reads[0], reads[1], batch_bytes=40000, piece_bytes=1 << 16):
        al.run_resident(with_stats=True)
        w.write(al.download(), None)
    paths = w.close()
    return {os.path.basename(p): open(p, "rb").read() for p in paths}


def test_report_writer_mates_packed_equal_strided(golden, tmp_path):
    reads = golden_mates(str(tmp_path))
    log = dict(minimal_score=[load_case("all")["log"]["minimal_score"][1]])
    x = _writer_run(golden, str(tmp_path / "packed"), "packed", reads, log)
    y = _writer_run(golden, str(tmp_path / "strided"), "strided", reads, log)
    assert x == y and len(x["aligned.sam"]) > 10000 and "aligned_fwd.fq" in x


def test_report_writer_packed_against_reference_binary(golden, golden_idx_dir):
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_ref")):
        pytest.skip("oracle/_ref/sortmerna_ref not built (oracle/Makefile.ref)")
    from oracle import ora
    fasta = os.path.join(GOLDEN, "db_bac.fasta")
    d = tempfile.mkdtemp(prefix="smr_packed_ref_")
    try:
        extra = ["-num_alignments", "0", "-sam", "-blast", BLAST, "-fastx", "-other", "-otu_map", "-de_novo_otu"]
        r = ora.run_reference([fasta], READS, os.path.join(d, "ref"), extra=extra, threads=1, idx_dir=golden_idx_dir)
        log = ora.parse_log(r["log"])
        ref = {fn: open(os.path.join(r["out_dir"], fn), "rb").read() for fn in os.listdir(r["out_dir"]) if fn != "aligned.log"}
        al = api.Aligner(0)
        _OPEN.append(al)
        al.set_params(api.default_params(num_alignments=0))
        al.load_index_part(0, 0, golden["prefixes"][1], golden["refs"][1], log["minimal_score"][0], (18, 9, 3), golden["stats"][1].lnwin)
        b = golden["batch"]
        tot = int(np.diff(b.off.astype(np.int64)).sum())
        al.set_report_scoring(0, log["lambda_"][0], log["K"][0], *hostio.evalue_params(golden["stats"][1], log["K"][0], tot, b.n))
        al.set_aln_layout("packed")
        al.set_aln_slots(2)
        head = b"".join(ln + b"\n" for ln in ref["aligned.sam"].split(b"\n") if ln.startswith(b"@")).decode()
        w = api.ReportWriter(os.path.join(d, "ours"), al, sam_header=head, otu_map=(0.97, 0.97), sam=True, blast=BLAST, fastx=True, other=True,
                             denovo=(0.97, 0.97))
        t = _text()
        al.upload_fastx(t)
        al.run_resident(with_stats=True)
        out = al.download()
        assert int(out["res"]["n_align"].max()) > 2
        w.write(out, None)
        ours = {os.path.basename(p): open(p, "rb").read() for p in w.close()}
        assert sorted(ours) == sorted(ref)
        for fn in ref:
            if fn == "aligned.blast":   # the E-value: the goldens' lambda / K have 6 digits (helpers.assert_blast_rows_equal)
                assert len(ours[fn].split(b"\n")) == len(ref[fn].split(b"\n"))
                assert [ln.split(b"\t")[:10] + ln.split(b"\t")[11:] for ln in ours[fn].split(b"\n")] == \
                       [ln.split(b"\t")[:10] + ln.split(b"\t")[11:] for ln in ref[fn].split(b"\n")]
            else:
                assert ours[fn] == ref[fn], fn
    finally:
        shutil.rmtree(d, ignore_errors=True)


# ---- 6. contracts ----
def test_packed_contracts(golden, all_pair, capfd, monkeypatch):
    _, s, pa, p = all_pair
    L, h = pa.L, pa.h
    b = golden["batch"]
    n, total, words = b.n, p["alns"].shape[0], p["cigar"].size
    cat, off = np.ascontiguousarray(b.cat, np.uint8), np.ascontiguousarray(b.off, np.uint64)

    def call(cap, wcap):
        res = np.zeros(n, api.RESULT_DTYPE)
        alns = np.zeros(max(cap, 1), api.ALN_DTYPE)
        st = np.zeros(max(cap, 1), api.STATS_DTYPE)
        pool = np.zeros(max(wcap, 1), np.uint32)
        cnt = np.zeros(api.CNT_FIXED + 2, np.uint64)
        used, wused = C.c_uint64(0), C.c_uint64(0)
        rc = L.smr_align_batch_packed(h, api._ptr(cat), api._ptr(off), C.c_uint32(n), api._ptr(res), api._ptr(alns), C.c_uint64(cap),
                                      C.byref(used), api._ptr(st), api._ptr(pool), C.c_uint64(wcap), C.byref(wused), api._ptr(cnt),
                                      C.c_uint32(cnt.size))
        return rc, used.value, wused.value, res, alns[:used.value], st[:used.value], pool[:wused.value], cnt

    monkeypatch.setenv("SMR_VERBOSE", "1")
    capfd.readouterr()
    rc, used, wused, *_ = call(total - 1, words)          # a short aln_cap: both sizes exact
    assert rc == 5 and used == total and wused == words
    assert b"aln_cap" in L.smr_last_error(h)
    # the batch is resident and run: a download into arrays that large only copies what the failed call placed
    res = np.zeros(n, api.RESULT_DTYPE)
    alns, st = np.zeros(total, api.ALN_DTYPE), np.zeros(total, api.STATS_DTYPE)
    pool, cnt = np.zeros(words, np.uint32), np.zeros(api.CNT_FIXED + 2, np.uint64)
    used, wused = C.c_uint64(0), C.c_uint64(0)
    assert L.smr_download_results_packed(h, api._ptr(res), api._ptr(alns), C.c_uint64(total), C.byref(used), api._ptr(st), api._ptr(pool),
                                         C.c_uint64(words), C.byref(wused), api._ptr(cnt), C.c_uint32(cnt.size)) == 0
    assert len(_reruns(capfd.readouterr().err)) == 1    # the reads were run again once, for the failed call
    assert np.array_equal(res, p["res"]) and alns.tobytes() == p["alns"].tobytes() and st.tobytes() == p["stats"].tobytes()
    assert pool.tobytes() == p["cigar"].tobytes() and cnt[0] == p["counters"]["num_aligned"]
    # the Aligner keeps the sizes the library named: its next align makes one call and runs the reads again once
    assert pa._packed_sizes[0] >= total and pa._packed_sizes[1] >= words
    again = pa.align(b.cat, b.off, with_stats=True)
    assert len(_reruns(capfd.readouterr().err)) == 1
    assert again["alns"].tobytes() == p["alns"].tobytes()
    monkeypatch.delenv("SMR_VERBOSE")
    rc, used, wused, *_ = call(total, words - 1)          # a short CIGAR pool
    assert rc == 5 and used == total and wused == words
    rc, used, wused, res, alns, st, pool, cnt = call(total, words)
    assert rc == 0 and (used, wused) == (total, words)
    assert np.array_equal(res, p["res"]) and alns.tobytes() == p["alns"].tobytes() and st.tobytes() == p["stats"].tobytes()
    assert pool.tobytes() == p["cigar"].tobytes()
    # downloading twice gives the same results; the resident batch stays
    pa.upload(b.cat, b.off)
    pa.run_resident(with_stats=True)
    d1, d2 = pa.download(), pa.download()
    for k in ("res", "alns", "stats", "cigar", "aln_off"):
        assert np.array_equal(d1[k], d2[k]) and np.array_equal(d1[k], p[k]), k
    assert {k: d1["counters"][k] for k in WORK} == {k: d2["counters"][k] for k in WORK}
    # the strided entry points and the stats buffer are refused in the packed layout, naming the packed call
    res = np.zeros(n, api.RESULT_DTYPE)
    alns = np.zeros(n * 4, api.ALN_DTYPE)
    pool = np.zeros(1 << 16, np.uint32)
    cnt = np.zeros(api.CNT_FIXED + 2, np.uint64)
    assert L.smr_align_batch(h, api._ptr(cat), api._ptr(off), C.c_uint32(n), api._ptr(res), api._ptr(alns), api._ptr(pool), C.c_uint64(pool.size),
                             None, api._ptr(cnt), C.c_uint32(cnt.size)) == 2
    assert b"smr_align_batch_packed" in L.smr_last_error(h)
    assert L.smr_download_results(h, api._ptr(res), api._ptr(alns), api._ptr(pool), C.c_uint64(pool.size), None, api._ptr(cnt), C.c_uint32(cnt.size)) == 2
    assert b"smr_download_results_packed" in L.smr_last_error(h)
    assert L.smr_set_stats_buffer(h, api._ptr(np.zeros(8, api.STATS_DTYPE))) == 2
    assert L.smr_set_stats_buffer(h, None) == 0        # clearing a buffer set in the strided layout is allowed
    assert L.smr_set_aln_layout(h, C.c_uint32(2)) == 2
    with pytest.raises(KeyError):
        pa.set_aln_layout("banded")
    # align_files formats a packed result through its strided equivalent
    rows_p = api.align_files(pa, b)["sam"]
    # strided results again after switching back
    pa.set_aln_layout("strided")
    again = pa.align(b.cat, b.off, with_stats=True)
    assert_packed_equals_strided(p, again, "strided after packed", counters=False)
    assert api.align_files(pa, b)["sam"] == rows_p and len(rows_p) > 1000
    pa.set_aln_layout("packed")
