"""The index budget (smr_set_index_budget) on the GPU: a batch run over resident groups of index parts must give what the
all-resident run gives, bit for bit, while the device holds no more of the parts' search arrays than the budget.  Checked here:
- every golden case, each part its own group and groups of two, in the strided and the packed layout, and against expected.json;
- case_parts (2 indexes x 3 parts) with group boundaries inside an index and across indexes;
- the bench workload against its 8 databases and set4_mates, with one group per database where the sizes allow, against the stored
  SAM digests;
- scratch-overflow retries under a budget, and all alignments (-num_alignments 0) with reads that outgrow the stride in one group and
  keep accepting in later ones;
- the report side after a budgeted run;
- device memory: the residency counters, the drop of free memory while loading 8 databases under a quarter budget, and device-built
  parts equal under a budget;
- the refusals and the settings: a part larger than the budget, budget 0, a budget changed between runs."""
import ctypes as C
import os
import re
import shutil
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, case_names, load_case
from helpers import params_kwargs_from_args, strip_seq
from sortmerna_b200 import api, hostio
from test_gpu_packed_results import both_overflow_inputs, near_copy_inputs, MS

pytestmark = pytest.mark.gpu

READS = os.path.join(GOLDEN, "reads_mix.fq")
_OPEN = []


@pytest.fixture(autouse=True)
def _close_contexts():
    yield
    while _OPEN:
        _OPEN.pop().close()


def _new(params):
    a = api.Aligner(0)
    _OPEN.append(a)
    a.set_params(params)
    return a


def _nbytes(a, slot, which):
    nb = C.c_uint64(0)
    assert a.L.smr_debug_index_array(a.h, C.c_uint32(slot), C.c_uint32(which), C.c_void_p(0), C.c_uint64(0), C.byref(nb)) == 0
    return int(nb.value)


def part_bytes(a):
    """the search-array bytes of every loaded part, as the library lays them out: flookup, ftext, fid, pos_off, pos, each with 64
    bytes of slack at a multiple of 256 bytes"""
    r = lambda b: (b + 64 + 255) // 256 * 256
    out = []
    for s in range(len(a.parts)):
        e = _nbytes(a, s, 1) // 8
        out.append(r(_nbytes(a, s, 0)) + r((e + 7) // 8 * 8 * 4) + r(e * 4) + r(_nbytes(a, s, 2)) + r(_nbytes(a, s, 3)))
    return out


def groups_of(sizes, budget):
    """the groups the library forms: consecutive parts, greedily, each within the budget"""
    gs = []
    for s in sizes:
        if not gs or sum(gs[-1]) + s > budget:
            gs.append([])
        gs[-1].append(s)
    return gs


def budget_for(sizes, per):
    """a budget that puts `per` consecutive parts in each group, where the sizes allow it (never less than the largest part)"""
    return max([max(sizes)] + [sum(sizes[i:i + per]) for i in range(0, len(sizes), per)])


def set_budget(a, sizes, budget):
    a.set_index_budget(budget)
    r = a.index_residency()
    want = groups_of(sizes, budget) if budget else [sizes]
    assert r["groups"] == len(want) and r["largest_group_bytes"] == max(sum(g) for g in want)
    return len(want)


# the candidate kernel's work counters: a read whose seed scratch overflows in a later group has had its candidate work in the
# earlier groups counted before it is retried (DESIGN 5f); without a budget every part is seeded first and the read never gets there
CANDIDATE_WORK = ("sw_calls", "sw_cells", "pos_entries", "lis_calls", "spec_calls", "spec_cells", "spec_pairs", "slow_pairs", "rounds_a",
                  "rounds_b", "w1_cnt")


def assert_same(x, y, what, seed_overflow=False):
    """results, alignments, CIGAR words, stats, matched and every counter (the dbg_ / cyc_ clock counters are 0 without
    instrumentation); seed_overflow: reads overflowed their seed scratch, and the candidate work may be counted more often, never less"""
    if seed_overflow:
        x, y = dict(x), dict(y)
        xc, yc = dict(x["counters"]), dict(y["counters"])
        for k in CANDIDATE_WORK:
            assert xc.pop(k) >= yc.pop(k), (what, k)
        x["counters"], y["counters"] = xc, yc
    for k in ("res", "alns", "cigar", "matched"):
        assert np.array_equal(x[k], y[k]), (what, k)
    if "stats" in y or "stats" in x:
        assert np.array_equal(x["stats"], y["stats"]), (what, "stats")
    if "aln_off" in y:
        assert np.array_equal(x["aln_off"], y["aln_off"]), (what, "aln_off")
    assert x["slots"] == y["slots"]
    assert x["counters"] == y["counters"], (what, {k: (x["counters"][k], y["counters"][k]) for k in x["counters"] if x["counters"][k] != y["counters"][k]})


def _golden_aligner(golden, exp, layout="strided", slots=None):
    a = _new(api.default_params(**params_kwargs_from_args(exp["args"])))
    tot = int(np.diff(golden["batch"].off.astype(np.int64)).sum())
    for k in range(2):
        a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], exp["log"]["minimal_score"][k], (18, 9, 3), golden["stats"][k].lnwin)
        a.set_report_scoring(k, exp["log"]["lambda_"][k], exp["log"]["K"][k], *hostio.evalue_params(golden["stats"][k], exp["log"]["K"][k], tot, golden["batch"].n))
    a.set_aln_layout(layout)
    if slots:
        a.set_aln_slots(slots)
    return a


# ---- 1. every golden case ----
@pytest.mark.parametrize("layout", ["strided", "packed"])
@pytest.mark.parametrize("case", case_names())
def test_golden_cases(golden, case, layout, capfd, monkeypatch):
    exp = load_case(case)
    monkeypatch.setenv("SMR_VERBOSE", "1")
    b = golden["batch"]
    base = _golden_aligner(golden, exp).align(b.cat, b.off, with_stats=True)   # (the all-alignments cases grow the stride)
    slots = base["slots"] if layout == "packed" else None
    want = _golden_aligner(golden, exp, layout, slots).align(b.cat, b.off, with_stats=True) if layout == "packed" else base
    a = _golden_aligner(golden, exp, layout, slots)
    sizes = part_bytes(a)
    for per in (1, 2):
        ng = set_budget(a, sizes, budget_for(sizes, per))
        assert ng == (2 if per == 1 else 1)
        capfd.readouterr()
        got = a.align(b.cat, b.off, with_stats=True)
        seed_ovf = ng > 1 and re.search(r"causes so far: lane [1-9]|region [1-9]|overflowed their scratch at scale", capfd.readouterr().err) is not None
        assert_same(got, want, (case, layout, per), seed_ovf)
        if layout == "strided":
            rows = hostio.format_sam_rows(b, golden["refs"], got["res"], got["alns"], got["cigar"], got["slots"])
            assert sorted(rows if case == "default" else strip_seq(rows)) == sorted(exp["sam"])
            assert got["counters"]["num_aligned"] == exp["log"]["passing"]
    r = a.index_residency()
    assert r["uploads"] >= 2 and r["upload_bytes"] >= sum(sizes)


# ---- 2. case_parts: 2 indexes x 3 parts ----
def test_multipart_groups(golden, golden_parts):
    exp = load_case("parts")
    b = golden["batch"]

    def load():
        a = _new(api.default_params())
        for k, g in enumerate(golden_parts):
            for p in range(g["stats"].num_parts):
                a.load_index_part(k, p, g["prefix"], g["part_refs"][p], exp["log"]["minimal_score"][k], (18, 9, 3), g["stats"].lnwin)
        return a

    want = load().align(b.cat, b.off, with_stats=True)
    a = load()
    sizes = part_bytes(a)
    assert len(sizes) == 6
    by_index = [g["part_refs"] for g in golden_parts]
    seen = set()
    # one part per group; pairs (0-1, 2-3 across the indexes, 4-5); and (when the sizes allow) groups that cut an index after 2 parts
    for budget in (max(sizes), budget_for(sizes, 2), budget_for(sizes, 3), max(sizes[0] + sizes[1], sizes[2] + sizes[3], sizes[4] + sizes[5])):
        gs = groups_of(sizes, budget)
        seen.add(tuple(len(g) for g in gs))
        set_budget(a, sizes, budget)
        got = a.align(b.cat, b.off, with_stats=True)
        assert_same(got, want, ("parts", budget))
        rows = strip_seq(hostio.format_sam_rows(b, by_index, got["res"], got["alns"], got["cigar"], got["slots"]))
        assert sorted(rows) == sorted(exp["sam"])
    cuts = [np.cumsum(s)[:-1].tolist() for s in seen]
    assert any(any(c % 3 for c in cs) for cs in cuts), seen          # a group boundary inside an index
    assert any(3 not in cs and len(cs) > 0 for cs in cuts), seen      # a group across the two indexes


# ---- 3. bench workload and set4_mates against their stored digests ----
@pytest.mark.parametrize("case", ["bench_workload", "set4_mates"])
def test_bundled_sets_one_group_per_database(case):
    import json
    import test_gpu_bundled_sets as bs
    from tools import stage_data
    exp = json.load(open(os.path.join(GOLDEN, case + ".json")))
    with tempfile.TemporaryDirectory(prefix="smr_budget_") as d:
        fastas, reads, kw = bs.CASES[case](d)
        idx_dir, _ = stage_data.ensure_indexes(fastas, os.path.join(d, "idx"), **kw)
        pre = hostio.find_index_prefixes(idx_dir)
        refs = [hostio.load_references(f) for f in fastas]
        a = _new(api.default_params())
        for k, f in enumerate(fastas):
            p = pre[os.path.basename(f)]
            a.load_index_part(k, 0, p, refs[k], exp["minimal_score"][k], (18, 9, 3), hostio.parse_stats(p).lnwin)
        batch = hostio.load_reads(reads)
        want = a.align(batch.cat, batch.off)
        sizes = part_bytes(a)
        ng = set_budget(a, sizes, max(sizes))
        assert ng >= 4, [len(g) for g in groups_of(sizes, max(sizes))]
        got = a.align(batch.cat, batch.off)
        r = a.index_residency()
        assert r["device_search_bytes"] <= max(sizes) and r["last_upload_us"] > 0
    assert_same(got, want, case)
    rows = hostio.format_sam_rows(batch, refs, got["res"], got["alns"], got["cigar"], got["slots"])
    assert len(rows) == exp["sam_rows"] and bs.rows_digest(rows) == exp["sam_sha256"]
    assert int(got["res"]["is_hit"].sum()) == exp["passing"]


# ---- 4. scratch-overflow retries under a budget ----
def _twice(nc, params, layout="strided"):
    """the database loaded as two indexes: every read that aligns aligns in both groups"""
    a = _new(params)
    for k in range(2):
        a.load_index_part(k, 0, nc["prefix"], nc["refs"], MS, (18, 9, 3), nc["stats"].lnwin)
    a.set_aln_layout(layout)
    return a


def test_scratch_overflow_retries(tmp_path, capfd, monkeypatch):
    nc = both_overflow_inputs(str(tmp_path))
    b = nc["batch"]
    monkeypatch.setenv("SMR_CHUNK_READS", "32")   # read at smr_init
    monkeypatch.setenv("SMR_VERBOSE", "1")
    for layout in ("strided", "packed"):
        prm = api.default_params(num_alignments=0)
        capfd.readouterr()
        want = _twice(nc, prm, layout).align(b.cat, b.off, with_stats=True)
        assert "overflowed their scratch" in capfd.readouterr().err
        a = _twice(nc, prm, layout)
        a.set_aln_slots(want["slots"] or 16)
        sizes = part_bytes(a)
        assert set_budget(a, sizes, max(sizes)) == 2
        got = a.align(b.cat, b.off, with_stats=True)
        assert "overflowed their scratch" in capfd.readouterr().err
        assert_same(got, want, layout)
        r = a.index_residency()
        assert r["uploads"] >= 4   # the first run's two groups and the retry's


# ---- 5. all alignments: reads outgrow the stride in one group and keep accepting in the next ----
@pytest.fixture(scope="module")
def near_copies():
    d = tempfile.mkdtemp(prefix="smr_budget_nc_")
    yield near_copy_inputs(d)
    shutil.rmtree(d, ignore_errors=True)


def test_all_alignments_packed(near_copies, capfd, monkeypatch):
    nc = near_copies
    b = nc["batch"]
    prm = api.default_params(num_alignments=0)
    want = _twice(nc, prm, "packed").align(b.cat, b.off, with_stats=True)
    cnt = want["res"]["n_align"]
    assert int(cnt.max()) >= 3000   # two groups of the large near-copy group's alignments
    a = _twice(nc, prm, "packed")
    sizes = part_bytes(a)
    assert set_budget(a, sizes, max(sizes)) == 2
    got = a.align(b.cat, b.off, with_stats=True)
    assert_same(got, want, "packed")


def test_all_alignments_strided_slots_needed(near_copies):
    nc = near_copies
    b = nc["batch"]
    prm = api.default_params(num_alignments=0)

    def needed(budgeted):
        a = _twice(nc, prm)
        if budgeted:
            sizes = part_bytes(a)
            assert set_budget(a, sizes, max(sizes)) == 2
        cat, off = np.ascontiguousarray(b.cat, np.uint8), np.ascontiguousarray(b.off, np.uint64)
        slots, res, alns, pool, cap, counters = a._outputs(b.n)
        used = C.c_uint64(0)
        rc = a.L.smr_align_batch(a.h, api._ptr(cat), api._ptr(off), C.c_uint32(b.n), api._ptr(res), api._ptr(alns), api._ptr(pool),
                                 C.c_uint64(cap), C.byref(used), api._ptr(counters), C.c_uint32(counters.size))
        assert rc == 5
        return int(a.L.smr_aln_slots_needed(a.h)), a.align(b.cat, b.off)

    n0, out0 = needed(False)
    n1, out1 = needed(True)
    assert n0 == n1 > 3000 and out1["slots"] == out0["slots"]
    assert_same(out1, out0, "strided at the grown stride")


# ---- 6. the report side after a budgeted run ----
def test_reports_after_budgeted_run(golden):
    exp = load_case("default")
    b = golden["batch"]
    t = open(READS, "rb").read()
    s_al = _golden_aligner(golden, exp)
    s = s_al.align(b.cat, b.off, with_stats=True)
    p_al = _golden_aligner(golden, exp)
    sizes = part_bytes(p_al)
    assert set_budget(p_al, sizes, max(sizes)) == 2
    p = p_al.align(b.cat, b.off, with_stats=True)
    for kw in (dict(sam=True, blast="1 cigar qcov qstrand"), dict(fastx=True, other=True, denovo=(0.97, 0.97))):
        for gz in (False, True):
            assert p_al.format_reports(p, t, gzip=gz, **kw) == s_al.format_reports(s, t, gzip=gz, **kw), (kw, gz)
    for gz in (False, True):
        assert p_al.format_blast_pairwise(p, t, gzip=gz) == s_al.format_blast_pairwise(s, t, gzip=gz)
    for a, o in ((p_al, p), (s_al, s)):
        a.otu_begin(0.9, 0.9)
        assert a.otu_add(o, t) > 0
    assert p_al.otu_finish() == s_al.otu_finish()
    dp, ds = p_al.denovo_stats(p, t, 0.9, 0.9), s_al.denovo_stats(s, t, 0.9, 0.9)
    assert np.array_equal(dp[0], ds[0]) and dp[1] == ds[1]


# ---- 7. memory ----
def test_device_memory_while_loading_8_databases():
    import torch
    from tools import synth_databases
    with tempfile.TemporaryDirectory(prefix="smr_budget_mem_") as d:
        fastas = synth_databases.write(os.path.join(d, "db"))

        def load(budget):
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            a = _new(api.default_params())
            a.set_index_budget(budget)
            for k, f in enumerate(fastas):
                a.build_index_device(k, f)
            torch.cuda.synchronize()
            return a, free0 - torch.cuda.mem_get_info()[0]

        full, drop_full = load(0)
        sizes = part_bytes(full)
        refseq = sum(_nbytes(full, s, 4) + _nbytes(full, s, 5) for s in range(len(sizes)))
        info_full = full.index_info()
        full.close(); _OPEN.remove(full)
        budget = max(sum(sizes) // 4, max(sizes))   # (a quarter, unless one database alone is larger)
        a, drop = load(budget)
        r = a.index_residency()
    assert r["device_search_bytes"] == 0 and r["host_bytes"] == sum(sizes) and r["groups"] == len(groups_of(sizes, budget)) >= 3
    slack = 256 << 20   # the allocator's granularity and the context's own small buffers
    assert drop <= budget + refseq + slack, (drop, budget, refseq)
    assert drop < drop_full - sum(sizes) // 2, (drop, drop_full)
    assert a.index_info()["hbm_bytes"] < info_full["hbm_bytes"] - sum(sizes) // 2


def test_device_build_under_budget_equals_unbudgeted():
    fasta = os.path.join(GOLDEN, "db_bac.fasta")
    a = _new(api.default_params())
    n = a.build_index_device(0, fasta, max_mb=0.5)
    assert n >= 3
    sizes = part_bytes(a)
    c = _new(api.default_params())
    c.set_index_budget(max(sizes))
    assert c.build_index_device(0, fasta, max_mb=0.5) == n
    r = c.index_residency()
    assert r["groups"] == len(groups_of(sizes, max(sizes))) > 1 and r["device_search_bytes"] == 0 and r["host_bytes"] == sum(sizes)
    for s in range(n):
        for which in ("flookup", "flist", "pos_off", "pos", "refseq", "ref_off"):
            assert np.array_equal(c.index_array(s, which), a.index_array(s, which)), (s, which)


# ---- 8. refusals and settings ----
def test_part_larger_than_budget_is_refused(golden):
    exp = load_case("default")
    a = _golden_aligner(golden, exp)
    sizes = part_bytes(a)
    with pytest.raises(api.SmrError) as e:
        a.set_index_budget(min(sizes) - 1)
    assert "SMR_ERR_CAPACITY" in str(e.value) or "5" in str(e.value)
    assert str(max(sizes)) in str(e.value) or str(min(sizes)) in str(e.value)
    assert a.index_residency()["groups"] == 1   # the budget is unchanged
    c = _new(api.default_params())
    c.set_index_budget(sizes[0] - 1)
    with pytest.raises(api.SmrError) as e:
        c.load_index_part(0, 0, golden["prefixes"][0], golden["refs"][0], exp["log"]["minimal_score"][0], (18, 9, 3), golden["stats"][0].lnwin)
    assert re.search(r"index 0 part 0: its search arrays take %d bytes" % sizes[0], str(e.value)), str(e.value)
    assert len(c.index_info()) and c.index_info()["parts"] == 0


def test_budget_changes_between_runs(golden):
    exp = load_case("best3")
    b = golden["batch"]
    a = _golden_aligner(golden, exp)
    want = a.align(b.cat, b.off, with_stats=True)
    sizes = part_bytes(a)
    info0 = a.index_info()
    a.set_index_budget(max(sizes))
    assert_same(a.align(b.cat, b.off, with_stats=True), want, "budget")
    r = a.index_residency()
    assert r["device_search_bytes"] == max(sizes) and r["host_bytes"] == sum(sizes) and r["last_upload_us"] > 0
    a.set_index_budget(0)
    assert_same(a.align(b.cat, b.off, with_stats=True), want, "budget 0")
    r = a.index_residency()
    assert r["groups"] == 1 and r["device_search_bytes"] == sum(sizes) and r["host_bytes"] == 0 and r["last_upload_us"] == 0
    assert a.index_info() == info0
    a.set_index_budget(sum(sizes))   # everything fits in one group: resident, as without a budget
    assert_same(a.align(b.cat, b.off, with_stats=True), want, "one group")
    assert a.index_residency()["host_bytes"] == 0
    a.set_index_budget(max(sizes))
    a.upload(b.cat, b.off)
    a.run_resident()
    assert_same(a.download(), a.align(b.cat, b.off), "resident path")
