"""The candidate kernel scores alignments, and the finalize stage locates stored ones over a dense job list, two per warp pass
with the packed 16-bit kernel.  These tests check it against the oracle: through smr_debug_ssw, which runs consecutive pairs
(2i, 2i + 1) through the packed score pass and the packed locate and marks any disagreement with the s32 kernel, and end to
end through smr_align_batch."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, load_case
from helpers import assert_same_results
from sortmerna_b200 import api, hostio

pytestmark = pytest.mark.gpu


def _ora():
    from oracle import ora  # the checker; never imported by the product
    return ora


@pytest.fixture(scope="module")
def aligner(golden):
    a = api.Aligner(0)
    a.set_params(api.default_params())
    exp = load_case("default")
    for k in range(2):
        a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], exp["log"]["minimal_score"][k], (18, 9, 3), golden["stats"][k].lnwin)
    yield a
    a.close()


def _mutate(rng, t, qlen, err):
    p = int(rng.integers(0, t.size - qlen + 1))
    q = t[p:p + qlen].copy()
    m = rng.random(q.size) < err
    q[m] = rng.integers(0, 4, int(m.sum()))
    return q


def _check_pairs(aligner, ora, pairs, scores, filters=0):
    match, mis, sn, go, ge = scores
    aligner.set_params(api.default_params(match=match, mismatch=mis, score_N=sn, gap_open=go, gap_ext=ge))
    try:
        qs, ts = [p[0] for p in pairs], [p[1] for p in pairs]
        q_off = np.zeros(len(qs) + 1, np.uint64); np.cumsum([x.size for x in qs], out=q_off[1:])
        t_off = np.zeros(len(ts) + 1, np.uint64); np.cumsum([x.size for x in ts], out=t_off[1:])
        out, cig = aligner.debug_ssw(np.concatenate(qs), q_off, np.concatenate(ts), t_off, filters=filters, cigar_cap=1024)
    finally:
        aligner.set_params(api.default_params())
    mat = ora.score_matrix(match, mis, sn)
    for k, (q, t) in enumerate(zip(qs, ts)):
        rc, eo, ec = ora.ssw_align(q.astype(np.int8), t.astype(np.int8), mat, go, ge, filters)
        assert rc == 0
        assert out[k, 0] not in (-12345, -12347), (k, out[k])
        assert out[k, 0] == eo[0] and out[k, 2] == eo[2] and out[k, 4] == eo[4], (k, out[k], eo)
        if eo[0] >= filters and eo[0] > 0:
            assert out[k, 1] == eo[1] and out[k, 3] == eo[3] and out[k, 5] == eo[5], (k, out[k], eo)
            assert cig[k, :eo[5]].tolist() == ec.tolist(), k
    return out


def test_pair_halves_of_different_shapes():
    """Consecutive pairs whose queries and windows differ in length (one half ends long before the other), with N on both sides."""
    ora = _ora()
    a = api.Aligner(0)
    try:
        rng = np.random.default_rng(5)
        pairs = []
        for it in range(400):
            qlen = int(rng.integers(20, 60)) if it % 2 else int(rng.integers(120, 256))
            t = rng.integers(0, 4, qlen + int(rng.integers(0, 200 if it % 3 else 5))).astype(np.uint8)
            q = _mutate(rng, t, qlen, float(rng.choice([0.0, 0.03, 0.15])))
            if it % 4 == 0:
                q[rng.integers(0, q.size, 2)] = 4
                t[rng.integers(0, t.size, 3)] = 4
            pairs.append((q, t))
        for scores in [(2, -3, -3, 5, 2), (1, -1, -1, 2, 1)]:
            _check_pairs(a, ora, pairs, scores, filters=1)
    finally:
        a.close()


def test_tandem_repeats_tie_break():
    """Periodic queries and windows: many cells reach the best score, so the column-then-row tie-break decides both end points."""
    ora = _ora()
    a = api.Aligner(0)
    try:
        rng = np.random.default_rng(11)
        pairs = []
        for it in range(240):
            unit = rng.integers(0, 4, int(rng.integers(1, 7))).astype(np.uint8)
            q = np.tile(unit, 300)[: int(rng.integers(18, 200))]
            t = np.tile(unit, 500)[: q.size + int(rng.integers(0, 250))]
            if it % 3 == 0:
                q = q.copy(); q[int(rng.integers(0, q.size))] = (q[0] + 1) % 4
            if it % 5 == 0:
                t = t.copy(); t[int(rng.integers(0, t.size))] = 4
            pairs.append((q, t))
        for scores in [(2, -3, -3, 5, 2), (2, -7, -7, 3, 1)]:
            _check_pairs(a, ora, pairs, scores, filters=1)
    finally:
        a.close()


def test_query_rows_at_the_packed_limit():
    """Queries of 256 rows (packed) next to queries of 257 rows (s32 row blocks), in both halves of a pair."""
    ora = _ora()
    a = api.Aligner(0)
    try:
        rng = np.random.default_rng(17)
        pairs = []
        for it in range(64):
            qlen = 256 if (it // 2) % 2 == 0 else 257
            if it % 7 == 3:
                qlen = 255
            t = rng.integers(0, 4, qlen + int(rng.integers(0, 60))).astype(np.uint8)
            pairs.append((_mutate(rng, t, qlen, 0.02), t))
        _check_pairs(a, ora, pairs, (2, -3, -3, 5, 2), filters=1)
    finally:
        a.close()


def test_scores_at_the_16bit_limit():
    """A large match score: best scores just below and just above the 32,000 the packed kernel accepts (m * match)."""
    ora = _ora()
    a = api.Aligner(0)
    try:
        rng = np.random.default_rng(23)
        pairs = []
        for it in range(48):
            qlen = [250, 251, 252, 254, 256][it % 5]   # 127 * 251 = 31,877 <= 32,000 < 127 * 252 = 32,004
            t = rng.integers(0, 4, qlen + int(rng.integers(0, 40))).astype(np.uint8)
            pairs.append((_mutate(rng, t, qlen, 0.0 if it % 3 == 0 else 0.01), t))
        out = _check_pairs(a, ora, pairs, (127, -3, -3, 5, 2), filters=1)
        assert (out[:, 0] > 32000).any() and ((out[:, 0] > 30000) & (out[:, 0] <= 32000)).any()
    finally:
        a.close()


def _golden_batch(n):
    h, s, q = hostio.read_fastx(os.path.join(GOLDEN, "reads_mix.fq"), n)
    return hostio.pack_reads(h, s, q)


def _align_both(aligner, golden, batch, **kw):
    ora = _ora()
    exp = load_case("default")
    aligner.set_params(api.default_params(**kw))
    try:
        got = aligner.align(batch.cat, batch.off)
    finally:
        aligner.set_params(api.default_params())
    oix = [ora.OracleIndex(p, 0, s.lnwin) for p, s in zip(golden["prefixes"], golden["stats"])]
    want = ora.align(oix, [0, 1], [0, 0], 2, golden["refs"], exp["log"]["minimal_score"], [18, 9, 3, 18, 9, 3], ora.default_params(**kw), batch,
                     nthreads=4)
    assert_same_results(got, want, str(kw))
    ln = got["alns"]["cigar_len"].astype(np.int64); of = got["alns"]["cigar_off"].astype(np.int64)
    for r in range(got["res"].size):
        for k in range(int(got["res"]["n_align"][r])):
            i = r * got["slots"] + k
            j = r * want["slots"] + k
            assert got["cigar"][of[i]:of[i] + ln[i]].tolist() == want["cigar"][int(want["alns"]["cigar_off"][j]):int(want["alns"]["cigar_off"][j]) +
                                                                                 int(want["alns"]["cigar_len"][j])].tolist(), (r, k)
    return got


def test_align_odd_number_of_stored_alignments(aligner, golden):
    """End to end: batches whose stored alignments leave one job without a partner in the last packed pass."""
    odd = 0
    for n in (1, 3, 7, 20, 61, 200):
        got = _align_both(aligner, golden, _golden_batch(n))
        odd += int(got["res"]["n_align"].sum()) % 2
    assert odd > 0


def test_align_all_alignments(aligner, golden):
    """End to end with -num_alignments 0: every accepted alignment of a read is stored and finalized."""
    got = _align_both(aligner, golden, golden["batch"], num_alignments=0)
    assert int(got["res"]["n_align"].max()) > 1
