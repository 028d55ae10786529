"""The scratch-overflow retry against the oracle.  Every read first runs with fixed scratch; a read that outgrows it is flagged,
dropped, and run again on its own with 8x the scratch (then 64x, 512x).  The hardest reads get their answer there: many seed ids
in one window (lane), many seed hits for the read (region), a candidate with more (refpos, readpos) pairs than the pair buffer
(pairs), a traceback band or CIGAR too large for the traceback arena (trace), a full device CIGAR pool (cigar).

The inputs are generated here from a seed and reach the production caps with real reads: one-edit variants of one 18-mer core
(lane), substitution variants of six more cores, all six in one read (region), a periodic reference (pairs), long reads with a
net indel imbalance or many indels (trace, one of them twice: 64x) and many 1 kb reads with ~30 indels (cigar), between ordinary
150 bp reads that must not be flagged and reads drawn from a swarm of near-copies (a dense database).  The CPU tests check with
the oracle that the inputs pass the lane, region, trace and cigar caps and that one read needs 64x; the GPU tests compare every
path with the oracle and count the causes the library logs (SMR_VERBOSE), so that a retry path that is never reached -- pairs
included -- fails the module instead of passing it.  A second batch of indel-rich reads needs more CIGAR words than the host pool
Aligner allocates by default: the library names the size and the Aligner grows the pool."""
import gzip
import os
import re
import shutil
import tempfile

import numpy as np
import pytest

from helpers import assert_same_results
from sortmerna_b200 import api, hostio

SEED = 20261016
L = 18                      # seed length (-L)
LANE_CAP = 128              # kLaneHitCap: ids of one window at scale 1
PAIR_CAP = 4096             # pair_cap at scale 1 (x8 per retry)
TRACE_DIR_CAP = 32768       # traceback direction matrix at scale 1, bytes (x8 per retry)
TRACE_CIG_CAP = 128         # CIGAR operations of one traceback at scale 1 (x8 per retry)
MS = 60                     # minimal SW score of every index (any threshold serves kernel-vs-oracle)
ACGT = np.frombuffer(b"ACGT", np.uint8)

# -------------------------------------------------------------------------------------------------------------------------
# inputs
# -------------------------------------------------------------------------------------------------------------------------


def _rand(rng, n):
    return rng.integers(0, 4, n, dtype=np.uint8)


def _mutate(rng, s, rate):
    hit = rng.random(s.size) < rate
    return np.where(hit, (s + rng.integers(1, 4, s.size, dtype=np.uint8)) & 3, s).astype(np.uint8)


def swarm_refs(rng):
    """tools/bench_heavy.write_database at 3-5 % divergence: 4 groups of 30-50 copies of a 1400 bp ancestor"""
    out = []
    for g in range(4):
        root = _rand(rng, 1400)
        for _ in range(int(rng.integers(30, 51))):
            out.append(_mutate(rng, root, rng.uniform(0.03, 0.05)))
    return out


def core_variants(core):
    """every one-edit variant of the core: substitutions, insertions (19-mers) and deletions (17-mers)"""
    out = set()
    for i in range(L):
        for b in range(4):
            if b != core[i]:
                v = core.copy(); v[i] = b; out.add(v.tobytes())
            out.add(np.concatenate([core[:i], [b], core[i:]]).astype(np.uint8).tobytes())
        out.add(np.concatenate([core[:i], core[i + 1:]]).astype(np.uint8).tobytes())
    out.discard(core.tobytes())
    return [np.frombuffer(v, np.uint8) for v in sorted(out)]


def neighbourhood_refs(rng, core, flank=60):
    """four references per variant of the core, between random flanks that differ in the base next to the variant (the index
    keeps (L+1)-mers: each is an id of its own), none holding the core itself; returns (refs, flanks)"""
    refs, flanks = [], []
    for v in core_variants(core):
        for c in range(4):
            a, b = _rand(rng, flank), _rand(rng, flank)
            a[-1], b[0] = (c + 1) & 3, c
            s = np.concatenate([a, v, b])
            if core.tobytes() not in s.tobytes():
                refs.append(s)
                flanks.append((a, b))
    return refs, flanks


def region_refs(rng, cores, flank=60):
    """two references per substitution variant of each core (fewer ids per window than the lane buffer holds)"""
    refs = []
    for core in cores:
        for v in core_variants(core):
            if v.size != L:
                continue
            for c in range(2):
                a, b = _rand(rng, flank), _rand(rng, flank)
                a[-1], b[0] = (c + 1) & 3, c
                s = np.concatenate([a, v, b])
                if core.tobytes() not in s.tobytes():
                    refs.append(s)
    return refs


def repeat_ref(rng, length=2000, period=7, mutations=2):
    """a periodic reference with a few point substitutions"""
    unit = _rand(rng, period)
    s = np.resize(unit, length).astype(np.uint8)
    for p in rng.choice(np.arange(200, length - 200), mutations, replace=False):
        s[p] = (s[p] + 1) & 3
    return s


def _indels(rng, s, n_ins, n_del, lo=20):
    """n_ins single-base insertions and n_del single-base deletions at distinct positions >= lo from both ends"""
    pos = np.sort(rng.choice(np.arange(lo, s.size - lo), n_ins + n_del, replace=False))
    kind = rng.permutation(np.array([1] * n_ins + [0] * n_del))
    out, last = [], 0
    for p, k in zip(pos, kind):
        out.append(s[last:p])
        if k:
            out.append(_rand(rng, 1))
            last = p
        else:
            last = p + 1
    out.append(s[last:])
    return np.concatenate(out).astype(np.uint8)


def _alternating_indels(rng, s, n, lo=20):
    """n single-base indels, insertions and deletions alternating (the band stays narrow), evenly spread"""
    pos = np.linspace(lo, s.size - lo, n).astype(int)
    out, last = [], 0
    for k, p in enumerate(pos):
        out.append(s[last:p])
        if k % 2 == 0:
            out.append(_rand(rng, 1)); last = p
        else:
            last = p + 1
    out.append(s[last:])
    return np.concatenate(out).astype(np.uint8)


def _strand(rng, s):
    return (3 - s)[::-1].copy() if rng.random() < 0.5 else s


def make_inputs(workdir):
    """Writes the database FASTAs and returns dict(fastas={name: path}, reads=[(name, seq bytes)], kinds=[kind per read])."""
    rng = np.random.default_rng(SEED)
    core = _rand(rng, L)
    swarm = swarm_refs(rng)
    neigh, flanks = neighbourhood_refs(rng, core)
    cores = [_rand(rng, L) for _ in range(6)]
    many = region_refs(rng, cores)
    rep = repeat_ref(rng)
    plain = [_rand(rng, 2000) for _ in range(40)]
    dbs = {"swarm": [("swarm_%04d" % k, s) for k, s in enumerate(swarm)] + [("repeat_0", rep)],
           "neigh": [("neigh_%04d" % k, s) for k, s in enumerate(neigh)] + [("region_%04d" % k, s) for k, s in enumerate(many)] + [("plain_%04d" % k, s) for k, s in enumerate(plain)]}
    fastas = {}
    for name, recs in dbs.items():
        p = os.path.join(workdir, name + ".fasta")
        with open(p, "wb") as f:
            for rid, s in recs:
                f.write(b">" + rid.encode() + b"\n" + ACGT[s].tobytes() + b"\n")
        fastas[name] = p
    reads = []   # (kind, 0-3 codes or bytes with N)

    def plain_slice(n):
        k = int(rng.integers(len(plain)))
        p = int(rng.integers(0, plain[k].size - n + 1))
        return plain[k][p:p + n].copy()

    for _ in range(400):                                    # ordinary: 1 % substitutions, some N, some no hit at all
        s = _rand(rng, 150) if rng.random() < 0.1 else _mutate(rng, plain_slice(150), 0.01)
        s = ACGT[_strand(rng, s)].copy()
        if rng.random() < 0.1:
            s[rng.integers(0, s.size, int(rng.integers(1, 4)))] = ord("N")
        reads.append(("plain", s.tobytes()))
    for _ in range(60):                                     # swarm: a near-copy of many references
        c = swarm[int(rng.integers(len(swarm)))]
        p = int(rng.integers(0, c.size - 150 + 1))
        reads.append(("swarm", ACGT[_strand(rng, _mutate(rng, c[p:p + 150], 0.01))].tobytes()))
    for _ in range(6):                                      # six cores at window positions, ~80 ids each (region)
        s = _rand(rng, 150)
        for k, p in enumerate(range(0, 121, 24)):
            s[p:p + L] = cores[(k + _) % 6]
        reads.append(("region", ACGT[s].tobytes()))
    for k in rng.choice(len(neigh), 8, replace=False):      # the exact core between the flanks of one variant (lane)
        a, b = flanks[k]
        reads.append(("neigh", ACGT[np.concatenate([a, core, b[:72]])].tobytes()))   # the core at 60, a window position
    for n in (400,):                                        # a periodic read: ~22 pass-1 windows x ~280 positions of one id (pairs)
        p = int(rng.integers(0, rep.size - n + 1))          # (longer ones work too, but the planner takes seconds per read)
        reads.append(("repeat", ACGT[rep[p:p + n]].tobytes()))
    for n, d in ((600, 12), (800, 16), (1000, 20), (1200, 14), (1500, 10), (700, -14), (900, -18)):   # net indel imbalance (trace: direction matrix)
        s = plain_slice(n + max(d, 0))
        s = _indels(rng, s, max(-d, 0), max(d, 0))
        reads.append(("band", ACGT[_strand(rng, s)].tobytes()))
    for n, k in ((1000, 70), (1300, 80), (1500, 90)):         # many indels (trace: more than 128 CIGAR operations)
        reads.append(("ops", ACGT[_strand(rng, _alternating_indels(rng, plain_slice(n), k))].tobytes()))
    for _ in range(420):                                    # 1 kb, 25-35 indels: under 128 operations, but ~65 CIGAR words each (cigar)
        reads.append(("pool", ACGT[_strand(rng, _alternating_indels(rng, plain_slice(1000), int(rng.integers(25, 36))))].tobytes()))
    s = plain_slice(1540)                                   # 1.5 kb with a net 40-nt deletion: band 41, too wide for 8x (64x)
    s = np.concatenate([s[:700], s[740:]])
    reads.append(("x64", ACGT[_strand(rng, s)].tobytes()))
    order = rng.permutation(len(reads))                     # interleaved: the retry's index remapping matters
    reads = [reads[i] for i in order]
    # the CIGAR-heavy batch: 1 kb reads with 40-60 indels (81-121 CIGAR operations: ~100 words each, twice the 48 words per read
    # of the Aligner's default host pool) with the many-indel reads above (retried) and a few ordinary reads between them
    heavy = [("heavy", ACGT[_strand(rng, _alternating_indels(rng, plain_slice(1000), int(rng.integers(40, 61))))].tobytes()) for _ in range(200)]
    heavy += [x for x in reads if x[0] == "ops"] + [x for x in reads if x[0] == "plain"][:20]
    heavy = [heavy[i] for i in rng.permutation(len(heavy))]
    return dict(fastas=fastas, reads=[(f"r{i}_{k}", s) for i, (k, s) in enumerate(reads)], kinds=[k for k, _ in reads],
                heavy=[(f"h{i}_{k}", s) for i, (k, s) in enumerate(heavy)], heavy_kinds=[k for k, _ in heavy])


def fastq_text(reads):
    return b"".join(b"@" + n.encode() + b"\n" + s + b"\n+\n" + b"I" * len(s) + b"\n" for n, s in reads)


@pytest.fixture(scope="module")
def inputs():
    d = tempfile.mkdtemp(prefix="smr_ovf_")
    try:
        inp = make_inputs(d)
        idx = {}
        for name, fasta in inp["fastas"].items():
            prefix = os.path.join(d, "idx_" + name)
            api.build_index(fasta, prefix)
            st = hostio.parse_stats(prefix)
            assert st.num_parts == 1
            idx[name] = dict(prefix=prefix, refs=hostio.load_references(fasta))
        inp["idx"] = idx
        inp["batch"] = hostio.pack_reads([">" + n for n, _ in inp["reads"]], [s for _, s in inp["reads"]])
        inp["text"] = fastq_text(inp["reads"])
        inp["heavy_batch"] = hostio.pack_reads([">" + n for n, _ in inp["heavy"]], [s for _, s in inp["heavy"]])
        yield inp
    finally:
        shutil.rmtree(d, ignore_errors=True)


def _ora():
    from oracle import ora  # the checker; never imported by the product
    return ora


_ORACLE = {}


def oracle_run(inputs, names, batch="batch", **kw):
    """ora.align of a batch on the index files `names` (cached per call signature), with a pool large enough for all"""
    key = (batch, tuple(names), tuple(sorted(kw.items())))
    if key not in _ORACLE:
        ora = _ora()
        ix = [ora.OracleIndex(inputs["idx"][n]["prefix"], 0, L) for n in names]
        b = inputs[batch]
        slots = kw.get("num_alignments", 1) or 16
        _ORACLE[key] = ora.align(ix, list(range(len(names))), [0] * len(names), len(names), [inputs["idx"][n]["refs"] for n in names],
                                 [MS] * len(names), [18, 9, 3] * len(names), ora.default_params(**kw), b,
                                 nthreads=max(1, min(16, os.cpu_count() or 1)), cigar_cap=int(b.off[-1]) // 2 * slots + 65536)
        for x in ix:
            x.close()
    return _ORACLE[key]


# -------------------------------------------------------------------------------------------------------------------------
# preconditions (CPU): the inputs pass the production caps
# -------------------------------------------------------------------------------------------------------------------------


def _windows03(seq):
    s = hostio.encode_nt(seq)
    return np.where(s > 3, 0, s).astype(np.uint8), bool((s > 3).any())


def test_inputs_pass_the_seed_caps(inputs):
    """the core reads have a window with more ids than the per-lane buffer; the region reads have more than 2*len+32 hits in one
    part, in windows that fit the lane buffer (all windows of the forward strand: the reverse strand has none)"""
    ora = _ora()
    both = {n: ora.OracleIndex(inputs["idx"][n]["prefix"], 0, L) for n in ("swarm", "neigh")}
    lane, region = [], []
    for (name, s), kind in zip(inputs["reads"], inputs["kinds"]):
        q, _ = _windows03(s)
        if kind == "neigh":
            lane.append(len(both["neigh"].seed_window(q, 60)[0]))
        if kind == "region":
            ids = [len(both["neigh"].seed_window(q, p)[0]) for p in range(0, q.size - L + 1, 3)]
            region.append((sum(ids), max(ids)))
    assert len(lane) == 8 and min(lane) > LANE_CAP and max(lane) <= 8 * LANE_CAP, lane
    assert len(region) == 6 and all(2 * 150 + 32 < n <= 8 * (2 * 150 + 32) and m <= LANE_CAP for n, m in region), region


def _band(a):
    rl = int(a["ref_end1"]) - int(a["ref_begin1"]) + 1
    ql = int(a["read_end1"]) - int(a["read_begin1"]) + 1
    return abs(rl - ql) + 1, ql


def _trace_bytes(a):
    band, ql = _band(a)
    return (2 * band + 1) * ql * 3 + 8


def test_inputs_pass_the_traceback_and_cigar_caps(inputs):
    """From the oracle's stored alignments: direction matrices and CIGARs larger than the scale-1 traceback arena, one direction
    matrix larger than the 8x arena (a second retry, 64x), and more CIGAR words than the device pool of the batch holds."""
    want = oracle_run(inputs, ["swarm", "neigh"])
    res, alns, kinds = want["res"], want["alns"], inputs["kinds"]
    n = res.size
    hit = np.nonzero(res["n_align"] > 0)[0]
    dir_over = [r for r in hit if _trace_bytes(alns[r]) > TRACE_DIR_CAP]
    ops_over = [r for r in hit if alns[r]["cigar_len"] > TRACE_CIG_CAP and _trace_bytes(alns[r]) <= TRACE_DIR_CAP]
    x64 = [r for r in hit if _trace_bytes(alns[r]) > 8 * TRACE_DIR_CAP]
    assert len(dir_over) >= 5 and {kinds[r] for r in dir_over} >= {"band", "x64"}, dir_over
    assert len(ops_over) >= 2 and {kinds[r] for r in ops_over} == {"ops"}, ops_over
    assert len(x64) == 1 and kinds[x64[0]] == "x64" and _trace_bytes(alns[x64[0]]) <= 64 * TRACE_DIR_CAP
    assert _band(alns[x64[0]])[0] == 41
    # the device CIGAR pool of the batch (24 words per read and slot + 4096) holds less than the reads that reach it need
    fits = [r for r in hit if _trace_bytes(alns[r]) <= TRACE_DIR_CAP and alns[r]["cigar_len"] <= TRACE_CIG_CAP]
    assert sum(int(alns[r]["cigar_len"]) for r in fits) > 24 * n + 4096
    pool = [r for r in hit if kinds[r] == "pool"]
    assert len(pool) >= 300 and all(40 < alns[r]["cigar_len"] <= TRACE_CIG_CAP for r in pool)
    # and the ordinary reads align, none of them near a cap
    plain = [r for r in range(n) if kinds[r] == "plain"]
    assert sum(res["n_align"][r] > 0 for r in plain) > 300
    assert all(_trace_bytes(alns[r]) <= TRACE_DIR_CAP and alns[r]["cigar_len"] <= 32 for r in plain if res["n_align"][r])


def test_heavy_batch_needs_a_larger_host_pool(inputs):
    """From the oracle: the CIGAR-heavy batch needs more words than the Aligner's default host pool (48 per read + 4096), and
    some of its reads have more CIGAR operations than the scale-1 traceback arena holds (they are retried)."""
    want = oracle_run(inputs, ["neigh"], batch="heavy_batch")
    n, kinds, alns = want["res"].size, inputs["heavy_kinds"], want["alns"]
    assert int(want["res"]["n_align"].sum()) >= n - 10
    assert want["cigar"].size > 48 * n + 4096, (want["cigar"].size, 48 * n + 4096)
    heavy = [r for r in range(n) if kinds[r] == "heavy" and want["res"]["n_align"][r]]
    assert len(heavy) >= 190 and all(80 < alns[r]["cigar_len"] <= TRACE_CIG_CAP for r in heavy)
    assert sum(alns[r]["cigar_len"] > TRACE_CIG_CAP for r in range(n) if kinds[r] == "ops") == 3


# -------------------------------------------------------------------------------------------------------------------------
# GPU: every path against the oracle
# -------------------------------------------------------------------------------------------------------------------------

CAUSES = ("lane", "region", "pairs", "trace", "cigar", "err")
WORK_COUNTERS = ("num_aligned", "num_short", "sw_calls", "sw_cells", "pos_entries", "lis_calls")   # the counters the reference reports
_LOG = re.compile(r"\[smr\] (\d+) reads overflowed their scratch at scale (\d+): retrying with scale (\d+) "
                  r"\(causes so far: lane (\d+) region (\d+) pairs (\d+) trace (\d+) cigar (\d+) err (\d+)\)")


def _aligner(inputs, names, **kw):
    a = api.Aligner(0)
    a.set_params(api.default_params(**kw))
    for k, n in enumerate(names):
        a.load_index_part(k, 0, inputs["idx"][n]["prefix"], inputs["idx"][n]["refs"], MS, (18, 9, 3), L)
    return a


def _collect(capfd):
    """the retry lines the library wrote to stderr since the last call: (causes, scales retried to).  The causes are counted per
    context, so the largest line is the total of the context so far."""
    err = capfd.readouterr().err
    best, scales = dict.fromkeys(CAUSES, 0), set()
    for m in _LOG.finditer(err):
        scales.add(int(m.group(3)))
        c = dict(zip(CAUSES, map(int, m.groups()[3:])))
        if sum(c.values()) > sum(best.values()):
            best = c
    return best, scales


def _check(inputs, got, want, names, what):
    assert_same_results(got, want, what)
    assert got["matched"].tolist() == want["matched"].tolist(), what
    assert got["counters"]["num_aligned"] == want["counters"]["num_aligned"], what
    assert got["counters"]["num_short"] == want["counters"]["num_short_last"], what
    refs = [inputs["idx"][n]["refs"] for n in names]
    st = hostio.host_aln_stats(inputs["batch"], refs, got["res"], got["alns"], got["cigar"], got["slots"])
    slots = got["slots"]
    live = np.zeros(got["res"].size * slots, bool)
    for r in range(got["res"].size):
        live[r * slots:r * slots + int(got["res"]["n_align"][r])] = True
    for f in st.dtype.names:
        assert np.array_equal(got["stats"][f][live], st[f][live]), (what, f)


OPTION_SETS = {
    "default": {},
    "best3": dict(num_alignments=3),
    "all": dict(num_alignments=0),
    "full_search": dict(is_full_search=1),
    "scores": dict(match=2, mismatch=-4, gap_open=6, gap_ext=3, score_N=-2),   # a scoring set of tests/fuzz_common.py
}


@pytest.mark.gpu
@pytest.mark.parametrize("opts", list(OPTION_SETS))
def test_host_path_retry_equals_oracle(inputs, opts, monkeypatch, capfd):
    kw = OPTION_SETS[opts]
    names = ["swarm", "neigh"]
    monkeypatch.setenv("SMR_VERBOSE", "1")
    capfd.readouterr()
    a = _aligner(inputs, names, **kw)
    b = inputs["batch"]
    got = a.align(b.cat, b.off, with_stats=True)
    a.close()
    causes, _ = _collect(capfd)
    assert sum(causes.values()) > 0, (opts, "no read overflowed its scratch")
    _check(inputs, got, oracle_run(inputs, names, **kw), names, opts)


@pytest.mark.gpu
def test_retry_across_chunks_equals_oracle(inputs, monkeypatch, capfd):
    """SMR_CHUNK_READS=64: the flagged reads of a retry come from many chunks"""
    names = ["swarm", "neigh"]
    monkeypatch.setenv("SMR_VERBOSE", "1")
    monkeypatch.setenv("SMR_CHUNK_READS", "64")
    capfd.readouterr()
    a = _aligner(inputs, names)
    b = inputs["batch"]
    got = a.align(b.cat, b.off, with_stats=True)
    a.close()
    _collect(capfd)
    _check(inputs, got, oracle_run(inputs, names), names, "chunks of 64")


@pytest.mark.gpu
def test_retry_with_one_index_file_each(inputs, monkeypatch, capfd):
    """each database on its own index file, then both: reads_matched_per_db of every database across a retry"""
    monkeypatch.setenv("SMR_VERBOSE", "1")
    b = inputs["batch"]
    for names in (["swarm"], ["neigh"], ["neigh", "swarm"]):
        capfd.readouterr()
        a = _aligner(inputs, names)
        got = a.align(b.cat, b.off, with_stats=True)
        a.close()
        _collect(capfd)
        _check(inputs, got, oracle_run(inputs, names), names, str(names))


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["batch", "fastx", "fastx_gz"])
def test_resident_path_retry_keeps_the_batch_and_its_results(inputs, source, monkeypatch, capfd):
    """upload / upload_fastx / upload_fastx_gz, run_resident + download == the host path; then, without uploading again, the
    resident batch is the one uploaded (layout, report text), a second download with no run between gives the same answer, and
    so does a second run + download"""
    names = ["swarm", "neigh"]
    monkeypatch.setenv("SMR_VERBOSE", "1")
    capfd.readouterr()
    a = _aligner(inputs, names)
    b, text = inputs["batch"], inputs["text"]
    host = a.align(b.cat, b.off, with_stats=True)
    if source == "batch":
        a.upload(b.cat, b.off)
    elif source == "fastx":
        assert a.upload_fastx(text) == b.n
    else:
        assert a.upload_fastx_gz(gzip.compress(text, 6)) == b.n
    before = a.resident_layout(with_headers=source != "batch")
    a.run_resident(with_stats=True)
    first = a.download()
    causes, _ = _collect(capfd)
    assert sum(causes.values()) > 0, "no read overflowed its scratch"
    assert_same_results(first, host, source + " first download")
    assert np.array_equal(first["stats"], host["stats"]) and first["matched"].tolist() == host["matched"].tolist()
    after = a.resident_layout(with_headers=source != "batch")
    for x, y, what in zip(before, after, ("header offsets", "read offsets", "sequences")):
        assert (x is None and y is None) or np.array_equal(x, y), what
    assert np.array_equal(after[1], b.off) and np.array_equal(after[2], b.cat)
    if source != "batch":
        assert a.resident_text() == text
        assert a.format_reports(first, None, sam=True, fastx=True, other=True) == a.format_reports(first, text, sam=True, fastx=True, other=True)
    again = a.download()   # the retry ran in a batch of its own: the device results of the run are still there
    assert_same_results(again, first, source + " download again")
    assert np.array_equal(again["stats"], first["stats"]) and again["matched"].tolist() == first["matched"].tolist()
    assert np.array_equal(again["cigar"], first["cigar"])
    assert {k: again["counters"][k] for k in WORK_COUNTERS} == {k: first["counters"][k] for k in WORK_COUNTERS}
    a.run_resident(with_stats=True)
    second = a.download()
    assert_same_results(second, first, source + " second download")
    assert np.array_equal(second["stats"], first["stats"]) and second["matched"].tolist() == first["matched"].tolist()
    assert second["counters"]["num_aligned"] == first["counters"]["num_aligned"]
    a.close()


@pytest.mark.gpu
def test_every_cause_is_retried(inputs, monkeypatch, capfd):
    """One call over the batch: every overflow cause occurs and is retried, no read fails its traceback, and one read goes
    through a second retry (64x); the results equal the oracle's."""
    names = ["swarm", "neigh"]
    monkeypatch.setenv("SMR_VERBOSE", "1")
    capfd.readouterr()
    a = _aligner(inputs, names)
    b = inputs["batch"]
    got = a.align(b.cat, b.off, with_stats=True)
    a.close()
    causes, scales = _collect(capfd)
    print("overflow causes retried:", causes, "scales:", sorted(scales))
    assert all(causes[k] > 0 for k in ("lane", "region", "pairs", "trace", "cigar")), causes
    assert causes["err"] == 0, causes
    assert scales == {8, 64}, scales
    _check(inputs, got, oracle_run(inputs, names), names, "causes")


def _align_batch_raw(a, b, cap):
    """smr_align_batch into a host pool of `cap` words: (status, *cigar_used)"""
    slots, res, alns, _, _, counters = a._outputs(b.n)
    pool = np.zeros(max(cap, 1), np.uint32)
    used = api.C.c_uint64(0)
    rc = a.L.smr_align_batch(a.h, api._ptr(b.cat), api._ptr(b.off), api.C.c_uint32(b.n), api._ptr(res), api._ptr(alns), api._ptr(pool),
                             api.C.c_uint64(cap), api.C.byref(used), api._ptr(counters), api.C.c_uint32(counters.size))
    return rc, int(used.value)


@pytest.mark.gpu
def test_host_pool_too_small_names_the_size(inputs, monkeypatch, capfd):
    """The CIGAR-heavy batch in a host pool too small: SMR_ERR_CAPACITY with *cigar_used = the words the successful call uses,
    counted across the retry of the reads that overflow the traceback arena and the device pool.  align() and download() grow the
    pool from it and return what the oracle returns."""
    names = ["neigh"]
    monkeypatch.setenv("SMR_VERBOSE", "1")
    b = inputs["heavy_batch"]
    want = oracle_run(inputs, names, batch="heavy_batch")
    a = _aligner(inputs, names)
    capfd.readouterr()
    rc, need = _align_batch_raw(a, b, 1000)
    causes, scales = _collect(capfd)
    assert rc == 5 and "cigar pool too small" in a.L.smr_last_error(a.h).decode()
    assert causes["trace"] > 0 and causes["cigar"] > 0 and 8 in scales, causes
    assert need == want["cigar"].size > 48 * b.n + 4096, (need, want["cigar"].size)
    assert _align_batch_raw(a, b, need - 1) == (5, need)
    assert _align_batch_raw(a, b, need) == (0, need)
    got = a.align(b.cat, b.off, with_stats=True)
    assert got["cigar"].size == need
    assert_same_results(got, want, "heavy, align")
    assert got["matched"].tolist() == want["matched"].tolist()
    assert got["counters"]["num_aligned"] == want["counters"]["num_aligned"]
    a.upload(b.cat, b.off)
    a.run_resident(with_stats=True)
    res = a.download()
    assert res["cigar"].size == need
    assert_same_results(res, got, "heavy, download")
    assert np.array_equal(res["stats"], got["stats"]) and res["matched"].tolist() == got["matched"].tolist()
    a.close()


def _download_raw(a, n, cap):
    """smr_download_results of the resident batch into a host pool of `cap` words: ((status, *cigar_used), the result dict)"""
    slots, res, alns, _, _, counters = a._outputs(n)
    pool = np.zeros(max(cap, 1), np.uint32)
    used = api.C.c_uint64(0)
    rc = a.L.smr_download_results(a.h, api._ptr(res), api._ptr(alns), api._ptr(pool), api.C.c_uint64(cap), api.C.byref(used),
                                  api._ptr(counters), api.C.c_uint32(counters.size))
    return (rc, int(used.value)), a._pack(res, alns, pool, int(used.value), counters, slots)


@pytest.mark.gpu
def test_download_again_into_a_larger_pool(inputs, monkeypatch, capfd):
    """One run of the CIGAR-heavy batch, then three downloads with no run between: a host pool too small names the words needed
    (counted across the retry, which every download runs again), and the download into a pool of that size equals align()."""
    names = ["neigh"]
    monkeypatch.setenv("SMR_VERBOSE", "1")
    b = inputs["heavy_batch"]
    a = _aligner(inputs, names)
    want = a.align(b.cat, b.off)
    need = want["cigar"].size
    a.upload(b.cat, b.off)
    a.run_resident()
    capfd.readouterr()
    assert _download_raw(a, b.n, 1000)[0] == (5, need)
    assert _download_raw(a, b.n, need - 1)[0] == (5, need)
    status, got = _download_raw(a, b.n, need)
    causes, scales = _collect(capfd)
    assert status == (0, need)
    assert causes["trace"] > 0 and 8 in scales, causes
    assert_same_results(got, want, "heavy, third download")   # (which reads fill the device CIGAR pool first, and so are retried,
    assert got["matched"].tolist() == want["matched"].tolist()   # varies from run to run: so does the order of the host pool)
    assert got["counters"]["num_aligned"] == want["counters"]["num_aligned"]
    a.close()
