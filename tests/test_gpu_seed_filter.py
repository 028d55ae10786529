"""The seed kernel's streaming screen (half_screen) against the oracle's trie walk, window by window, on a database built so
that the screen lets through many entries that do not match.

coop_stream (smr_seed.cuh) buffers the entries that pass the screen, classifies them exactly when the buffer fills, keeps only
the matches and replays them once enough are buffered.  The database is one sequence and its near copies: copies with two
substitutions one to three bases apart (their entries pass the screen for the windows that span both, and are two edits
away), copies with one substitution and exact copies (matches).  The windows are every window of slices of the sequence and
of the same slices with pairs of nearby substitutions, searched through the forward and the mirror lists, with and without
--full_search.  A host model of the stream (same rounds, lists, chunks and
buffer thresholds) shows that the windows reach:
  * classify passes that find only non-matches;
  * a window whose 0-error exit is replayed in a later flush than its first survivors;
  * a window whose ids repeat across two flushes (de-duplication across flushes);
  * survivors that do not match in the forward lists and in the mirror lists."""
import os
import shutil
import tempfile

import numpy as np
import pytest

from sortmerna_b200 import api, hostio

CAP = 1024        # ids per window kept by the kernel; no window here comes near it
ROUND = 32        # windows searched together by one warp
ACC_CAP, ACC_STEP = 384, 256   # kAccCap, kAccStep of coop_stream
M32 = 0xFFFFFFFF


def _char_bits(a, b):
    return ((1 << (2 * b)) - 1) & ~((1 << (2 * a)) - 1)


def _screen(P, T, pw):
    h = pw // 2
    x = T ^ P
    return (((x & _char_bits(0, h)) == 0) | ((x & _char_bits(h, pw)) == 0) | (((T ^ (P >> 2)) & _char_bits(h, pw - 1)) == 0)
            | (((T ^ ((P << 2) & M32)) & _char_bits(h + 1, pw + 1)) == 0))


def _within_one_edit(P, T, pw):
    m9, m8 = ((1 << (2 * pw)) - 1) & 0x55555555, ((1 << (2 * (pw - 1))) - 1) & 0x55555555
    x, y, z = T ^ P, T ^ (P >> 2), (T >> 2) ^ P
    A9, B8, C9 = (x | (x >> 1)) & m9, (y | (y >> 1)) & m8, (z | (z >> 1)) & m9
    a8, a9 = (A9 & m8) | (1 << (2 * (pw - 1))), A9 | (1 << (2 * pw))
    low = lambda v: v & (~v + np.uint64(1))   # lowest set bit (v != 0)
    return ((A9 & ((A9 + np.uint64(M32)) & np.uint64(M32))) == 0) | (B8 < low(a8)) | (C9 < low(a9))   # A9 - 1, mod 2^32


def _rev_chars(v, pw):
    return sum(((v >> (2 * (pw - 1 - i))) & 3) << (2 * i) for i in range(pw))


def stream_model(flookup, flist, keys, pw):
    """Survivors of coop_stream for windows with 9-mer keys (keyf, keyr), in stream order, one warp per ROUND windows:
    dicts {win, dir, id, match, exact, cls, flush} -- cls: the classify pass that judged it, flush: the flush that replays it
    (or would, had it matched; None for the non-matches after the last flush of their round); and the list of (survivors,
    matches) of every classify pass"""
    text = flist[:, 0].astype(np.uint64)
    out, passes = [], []
    npass = nflush = 0
    for w0 in range(0, len(keys), ROUND):
        chunks = []
        for d in (0, 1):
            for lane, (kf, kr) in enumerate(keys[w0:w0 + ROUND]):
                off, cnt = (int(flookup[kf, 0]), int(flookup[kf, 1])) if d == 0 else (int(flookup[kr, 2]), int(flookup[kr, 3]))
                P = _rev_chars(kr, pw) if d == 0 else kf
                for g in range(off >> 3, (off + cnt + 7) >> 3):
                    i = np.arange(max(8 * g, off), min(8 * g + 8, off + cnt))
                    T = text[i]
                    s = _screen(np.uint64(P), T, pw)
                    m = _within_one_edit(np.uint64(P), T, pw)
                    ex = (T & np.uint64((1 << (2 * pw)) - 1)) == np.uint64(P)
                    chunks.append([dict(win=w0 + lane, dir=d, id=int(flist[j, 1]), match=bool(mm), exact=bool(e))
                                   for j, ss, mm, e in zip(i, s, m, ex) if ss])
        buf, ncls = [], 0
        for e0 in range(0, len(chunks), ROUND):
            last = e0 + ROUND >= len(chunks)
            for c in chunks[e0:e0 + ROUND]:
                buf += c
            if len(buf) > ncls and (len(buf) > ACC_CAP - ACC_STEP or last):
                new = buf[ncls:]
                for s in new:
                    s["cls"] = npass
                passes.append((len(new), sum(s["match"] for s in new)))
                npass += 1
                buf = buf[:ncls] + [s for s in new if s["match"]]
                ncls = len(buf)
            out += [s for c in chunks[e0:e0 + ROUND] for s in c]
            if buf and (len(buf) > ACC_CAP - ACC_STEP or last):
                for s in out:
                    s.setdefault("flush", nflush)
                nflush += 1
                buf, ncls = [], 0
        for s in out:
            s.setdefault("flush", None)
    return out, passes


def _near_copies(rng, length=90):
    base = rng.integers(0, 4, length, dtype=np.uint8)
    seqs = [base.copy(), base.copy()]
    for k in range(800):
        s = base.copy()
        if k < 600:   # two substitutions one to three bases apart: two edits from the windows that span both
            a = int(rng.integers(0, length - 4))
            at = np.array([a, a + int(rng.integers(1, 4))])
        else:         # one substitution: matches
            at = rng.choice(length, 1)
        s[at] = (s[at] + rng.integers(1, 4, at.size, dtype=np.uint8)) & 3
        seqs.append(s)
    return base, seqs


def make_db(d):
    """(FASTA, index prefix, reads) of the near copies, written and indexed under d"""
    from tools import stage_data
    base, seqs = _near_copies(np.random.default_rng(20261017))
    fasta = os.path.join(d, "near_copies2.fasta")
    acgt = np.frombuffer(b"ACGT", np.uint8)
    with open(fasta, "wb") as f:
        f.write(b"".join(b">s%d\n%s\n" % (i, acgt[s].tobytes()) for i, s in enumerate(seqs)))
    idx_dir, _ = stage_data.ensure_indexes([fasta], os.path.join(d, "idx"))
    prefix = hostio.find_index_prefixes(idx_dir)[os.path.basename(fasta)]
    # the windows: every window of three slices of the sequence, and of the same slices with two substitutions two bases apart
    # every 18 bases (windows with hundreds of survivors in their lists and no match)
    reads = [base[a:a + 60].copy() for a in (0, 15, 30)]
    for r in reads[:3]:
        m = r.copy()
        at = np.concatenate([np.arange(5, m.size, 18), np.arange(7, m.size, 18)])
        m[at] = (m[at] + 1) & 3
        reads.append(m)
    return fasta, prefix, reads


@pytest.fixture(scope="module")
def db():
    d = tempfile.mkdtemp(prefix="smr_seed_filter_")
    yield make_db(d)
    shutil.rmtree(d, ignore_errors=True)


def windows(reads):
    cat = np.concatenate(reads)
    off = np.zeros(len(reads) + 1, np.uint64)
    np.cumsum([r.size for r in reads], out=off[1:])
    wr = np.array([r for r, s in enumerate(reads) for _ in range(s.size - 18 + 1)], np.uint32)
    wp = np.array([p for s in reads for p in range(s.size - 18 + 1)], np.uint32)
    keys = []
    for r, p in zip(wr, wp):
        v = int("".join("%d" % c for c in reads[r][p:p + 18]), 4)
        keys.append((v >> 18, v & ((1 << 18) - 1)))
    return cat, off, wr, wp, keys


def check_coverage(flookup, flist, keys, zero):
    """the parts of coop_stream these windows reach, by the host model; zero[k]: the oracle's 0-error flag of window k"""
    sv, passes = stream_model(flookup, flist, keys, 9)
    assert sum(1 for n, m in passes if n > 0 and m == 0) >= 1, "a classify pass that finds only non-matches"
    assert any(n > ACC_CAP - ACC_STEP and m < n for n, m in passes), "a full buffer of survivors, some of them non-matches"
    by_win = {}
    for s in sv:
        by_win.setdefault(s["win"], []).append(s)
    late_zero = any(zero[w] and ss[0]["flush"] < next(s["flush"] for s in ss if s["exact"] and s["match"])
                    for w, ss in by_win.items() if any(s["exact"] for s in ss))
    assert late_zero, "a window whose 0-error exit comes in a later flush than its first survivors"
    across = any(len({s["flush"] for s in ss if s["match"] and s["id"] == i}) > 1
                 for ss in by_win.values() for i in {s["id"] for s in ss if s["match"]})
    assert across, "an id of one window matched in two flushes"
    for d in (0, 1):
        assert any(s["dir"] == d and not s["match"] for s in sv), ("survivors that do not match", d)
        assert any(s["dir"] == d and s["match"] for s in sv), ("matches", d)


@pytest.mark.gpu
def test_seed_screen_matches_oracle(db):
    from oracle import ora
    fasta, prefix, reads = db
    refs = hostio.load_references(fasta)
    lnwin = hostio.parse_stats(prefix).lnwin
    al = api.Aligner(0)
    oix = ora.OracleIndex(prefix, 0, lnwin)
    try:
        al.set_params(api.default_params())
        al.load_index_part(0, 0, prefix, refs, 0, (18, 9, 3), lnwin)
        cat, off, wr, wp, keys = windows(reads)
        for full in (0, 1):
            al.set_params(api.default_params(is_full_search=full))
            want = [oix.seed_window(reads[int(wr[k])], int(wp[k]), full_search=bool(full)) for k in range(wr.size)]
            if full == 0:
                check_coverage(al.index_array(0, "flookup"), al.index_array(0, "flist"), keys, [z for _, z in want])
            ids, counts, zero = al.debug_seed_windows(0, cat, off, wr, wp, cap=CAP)
            for k, (eids, ez) in enumerate(want):
                assert counts[k] == eids.size, (full, k, counts[k], eids.size)
                assert ids[k, :eids.size].tolist() == eids.tolist(), (full, k)
                assert bool(zero[k]) == ez, (full, k)
    finally:
        al.close()
        oix.close()
