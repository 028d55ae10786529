"""The seed kernel's entry stream (coop_stream, smr_seed.cuh) against the oracle's trie walk, window by window, on indexes
whose lists are long: ids in order, their number and the 0-error flag, through the cooperative stream and through the
per-lane sequential scan, with and without --full_search.

The stream reads the entry texts in aligned chunks of eight and loads the ids of matching entries only when it flushes its
buffer of matches, so the windows are chosen to reach every part of that:
  * windows of reads drawn from the databases themselves, whose lists run to hundreds of entries;
  * lists starting at every residue mod 8 of the text array, in both directions;
  * windows with more than 8 ids, which spill past the ids kept in shared memory;
  * rounds of 32 windows with more matching entries than one flush can hold: a database of a few hundred copies of one
    sequence, each with one or two substitutions, so that every lane of a round streams long lists of matching entries."""
import os
import tempfile

import numpy as np
import pytest

from sortmerna_b200 import api, hostio

pytestmark = pytest.mark.gpu

CAP = 1024           # ids per window kept by the kernel; no window here comes near it
ROUND = 32           # windows searched together by one warp
FLUSH_CAP = 384      # matching entries one flush of coop_stream can hold (kAccCap)


def _near_copies(rng, n=300, length=220):
    base = rng.integers(0, 4, length, dtype=np.uint8)
    seqs = [base.copy()]
    for _ in range(n):
        s = base.copy()
        at = rng.choice(length, int(rng.integers(1, 3)), replace=False)
        s[at] = (s[at] + rng.integers(1, 4, at.size, dtype=np.uint8)) & 3
        seqs.append(s)
    return seqs


def _write_fasta(path, seqs):
    acgt = np.frombuffer(b"ACGT", np.uint8)
    with open(path, "wb") as f:
        f.write(b"".join(b">s%d\n%s\n" % (i, acgt[s].tobytes()) for i, s in enumerate(seqs)))


def make_databases(d):
    """FASTA paths: the bac-16s stand-in (1.4 kb sequences in clades of 50) and the 5S stand-in (119 nt), both reduced, then
    the near copies of one sequence"""
    from tools import synth_databases
    fastas = []
    for k, scale in ((0, 0.2), (6, 0.1)):
        _, seqs = synth_databases.database(k, scale)
        p = os.path.join(d, synth_databases.file_name(k))
        with open(p, "wb") as f:
            f.write(b"".join(b">s%d\n%s\n" % (i, s) for i, s in enumerate(seqs)))
        fastas.append(p)
    fastas.append(os.path.join(d, "near_copies.fasta"))
    _write_fasta(fastas[-1], _near_copies(np.random.default_rng(20261015)))
    return fastas


@pytest.fixture(scope="module")
def setup():
    from oracle import ora
    from tools import stage_data
    d = tempfile.mkdtemp(prefix="smr_seed_stream_")
    fastas = make_databases(d)
    idx_dir, _ = stage_data.ensure_indexes(fastas, os.path.join(d, "idx"))
    pre = hostio.find_index_prefixes(idx_dir)
    al = api.Aligner(0)
    al.set_params(api.default_params())
    dbs = []
    for k, f in enumerate(fastas):
        p = pre[os.path.basename(f)]
        refs = hostio.load_references(f)
        al.load_index_part(k, 0, p, refs, 0, (18, 9, 3), hostio.parse_stats(p).lnwin)
        dbs.append(dict(refs=refs, oix=ora.OracleIndex(p, 0, hostio.parse_stats(p).lnwin)))
    yield al, dbs
    al.close()
    for db in dbs:
        db["oix"].close()
    import shutil
    shutil.rmtree(d, ignore_errors=True)


def sample_reads(refs, rng, n, length):
    """n slices of the database's own sequences (all windows of a slice are searched: list starts of every residue), every
    other one with 3 % substitutions so that windows without an exact match in the database are searched as well"""
    out = []
    for i in range(n):
        k = int(rng.integers(0, refs.n))
        a, b = int(refs.off[k]), int(refs.off[k + 1])
        ln = min(length, b - a)
        st = a + int(rng.integers(0, b - a - ln + 1))
        s = np.minimum(refs.cat[st:st + ln], 3).astype(np.uint8)
        if i % 2:
            sub = rng.random(ln) < 0.03
            s[sub] = (s[sub] + rng.integers(1, 4, int(sub.sum()), dtype=np.uint8)) & 3
        out.append(s)
    return out


def windows(reads):
    cat = np.concatenate(reads)
    off = np.zeros(len(reads) + 1, np.uint64)
    np.cumsum([r.size for r in reads], out=off[1:])
    wr = np.array([r for r, s in enumerate(reads) for _ in range(s.size - 18 + 1)], np.uint32)
    wp = np.array([p for s in reads for p in range(s.size - 18 + 1)], np.uint32)
    return cat, off, wr, wp


def list_rows(lk, reads, wr, wp):
    """{offF, cntF} and {offR, cntR} of every window: the lookup rows (lk) of its two 9-mer halves"""
    v = np.array([int("".join("%d" % c for c in reads[r][p:p + 18]), 4) for r, p in zip(wr, wp)], np.int64)
    f, r = lk[v >> 18], lk[v & ((1 << 18) - 1)]
    return f[:, :2], r[:, 2:]


@pytest.mark.parametrize("slot", [0, 1, 2])
def test_seed_stream_matches_oracle(setup, slot):
    al, dbs = setup
    db = dbs[slot]
    rng = np.random.default_rng(100 + slot)
    reads = sample_reads(db["refs"], rng, 12, 300)
    cat, off, wr, wp = windows(reads)
    fl, rl = list_rows(al.index_array(slot, "flookup"), reads, wr, wp)
    for lists in (fl, rl):
        live = lists[:, 1] > 0
        assert set((lists[live, 0] % 8).tolist()) == set(range(8)), "list starts of every residue mod 8"
    if slot < 2:
        assert max(fl[:, 1].max(), rl[:, 1].max()) >= 200, "lists of hundreds of entries"
    per_search = {}
    for full in (0, 1):
        al.set_params(api.default_params(is_full_search=full))
        want = [db["oix"].seed_window(reads[int(wr[k])], int(wp[k]), full_search=bool(full)) for k in range(wr.size)]
        for fallback in (False, True):
            ids, counts, zero = al.debug_seed_windows(slot, cat, off, wr, wp, cap=CAP, fallback_path=fallback)
            for k, (eids, ez) in enumerate(want):
                assert counts[k] == eids.size, (full, fallback, k, counts[k], eids.size)
                assert ids[k, :eids.size].tolist() == eids.tolist(), (full, fallback, k)
                assert bool(zero[k]) == ez, (full, fallback, k)
        per_search[full] = np.array([e.size for e, _ in want])
    al.set_params(api.default_params())
    n = per_search[1]
    assert n.max() > 8, "windows with more ids than the shared-memory slots"
    if slot == 2:
        rounds = n[:n.size // ROUND * ROUND].reshape(-1, ROUND).sum(axis=1)
        # the ids of a window are distinct matching entries, so a round with more ids than a flush holds flushes mid-round
        assert rounds.max() > FLUSH_CAP, rounds.max()
