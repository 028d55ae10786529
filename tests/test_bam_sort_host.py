"""The coordinate-sorted aligned.bam on the CPU: the -bam_sorted option of the command line, the from-spec BAI writer and region
query of tests/bai_spec.py against brute force on synthetic files (with windows and block boundaries), and the sorted BAM's helpers
of smr_fmt.h printed by tests/bamsort_check.cpp."""
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

import bai_spec
import bam_spec
from sortmerna_b200 import __main__ as cli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ARC, BAC, READS = (os.path.join(GOLDEN, n) for n in ("db_arc.fasta", "db_bac.fasta", "reads_mix.fq"))
G = ["-gumbel", "0.59,0.32", "-gumbel", "0.60,0.33"]


def _args(*a):
    return cli.parse_args(["-ref", ARC, "-ref", BAC, "-reads", READS, "-workdir", "/w"] + G + list(a))


# ---- the command line ----
def test_bam_sorted_option():
    k = _args("-bam_sorted")
    assert k["bam_sorted"] and k["bam"] and not k["sam"] and k["blast"] is None   # an output format: no default BLAST
    assert not _args()["bam_sorted"] and not _args("-bam")["bam_sorted"]
    both, one = _args("-bam", "-bam_sorted"), _args("-bam_sorted")
    assert bytes(both.pop("params")) == bytes(one.pop("params")) and both == one
    assert _args("-bam_sorted", "-num_alignments", "0")["params"].num_alignments == 0
    with pytest.raises(cli.UsageError, match="given twice"):
        _args("-bam_sorted", "-bam_sorted")
    assert _args("-bam_sorted", "-zip-out", "1")["zip_out"]   # zip_out leaves aligned.bam and its index alone (run_files)


def test_bam_sorted_help_line():
    lines = cli.HELP.splitlines()
    i = next(k for k, s in enumerate(lines) if s.strip().startswith("-bam"))
    assert "-bam_sorted" in lines[i] and "-bam_sorted" in lines[i + 1] and "aligned.bam.bai" in lines[i + 1]
    assert "not a reference option" in lines[i + 1]


# ---- the from-spec BAI against brute force ----
def _bgzf(data: bytes) -> bytes:
    """one BGZF member of data (<= 65,280 bytes), compressed by zlib"""
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    body = c.compress(data) + c.flush()
    size = 18 + len(body) + 8
    head = b"\x1f\x8b\x08\x04\0\0\0\0\0\xff" + struct.pack("<HccHH", 6, b"B", b"C", 2, size - 1)
    return head + body + struct.pack("<II", zlib.crc32(data), len(data))


def _synthetic_file(rng, n: int, ref_len: int, window: int):
    """a sorted BAM of n records over two references of ref_len bases, the records cut into windows of at most `window` bytes and
    each window into BGZF blocks of 65,280 bytes: (file bytes, [(refID, pos, end, bin, vbeg, vend)] from the layout itself)"""
    names = ["chrA", "chrB"]
    rows = []
    for i in range(n):
        ref = int(rng.integers(0, 2))
        pos = int(rng.integers(0, ref_len - 2))
        room = ref_len - pos
        kind = rng.random()
        span = int(rng.integers(1, 300)) if kind < 0.6 else int(rng.integers(1, 20000)) if kind < 0.9 else int(rng.integers(1, 200000))
        span = min(span, room)
        m = min(span, int(rng.integers(1, 120)))
        cigar = f"{m}M" if m == span else f"{m}M{span - m}D"
        seq = "".join("ACGT"[x] for x in rng.integers(0, 4, m))
        flag = 16 if rng.random() < 0.5 else 0
        rows.append((ref, pos, flag, i, f"r{i}\t{flag}\t{names[ref]}\t{pos + 1}\t255\t{cigar}\t*\t0\t0\t{seq}\t*\tAS:i:{m}\tNM:i:0"))
    rows.sort(key=lambda r: (bai_spec.sort_key(r[0], r[1], r[2]), r[3]))
    recs = [bam_spec.encode_row(r[4], r[0]) for r in rows]
    text = b"@HD\tVN:1.0\tSO:coordinate\n"
    head = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", 2)
    for nm in names:
        head += struct.pack("<i", len(nm) + 1) + nm.encode() + b"\0" + struct.pack("<i", ref_len)
    out = bytearray(b"".join(_bgzf(head[k:k + bam_spec.BLOCK]) for k in range(0, len(head), bam_spec.BLOCK)))
    laid = []
    k = 0
    while k < len(recs):   # greedy windows of whole records
        j, size = k + 1, len(recs[k])
        while j < len(recs) and size + len(recs[j]) <= window:
            size += len(recs[j])
            j += 1
        data = b"".join(recs[k:j])
        blocks = [data[b:b + bam_spec.BLOCK] for b in range(0, len(data), bam_spec.BLOCK)]
        coff = [len(out)]
        for b in blocks:
            out += _bgzf(b)
            coff.append(len(out))
        at = 0
        for r in recs[k:j]:
            e = at + len(r)
            vb = coff[at // bam_spec.BLOCK] << 16 | at % bam_spec.BLOCK
            ve = coff[-1] << 16 if e == len(data) else coff[e // bam_spec.BLOCK] << 16 | e % bam_spec.BLOCK
            f = bai_spec.fields(r)
            laid.append((f[0], f[1], f[2], f[3], vb, ve))
            at = e
        k = j
    out += bam_spec.EOF_BLOCK
    return bytes(out), laid, recs


@pytest.mark.parametrize("window", [20000, 200000, 1 << 30])
def test_spec_bai_against_brute_force(window):
    rng = np.random.default_rng(window % 1000)
    data, laid, recs = _synthetic_file(rng, 3000, 300000, window)
    got = bai_spec.file_records(data)   # the virtual offsets read back from the file itself
    assert [r for r, _, _ in got] == recs
    assert [(vb, ve) for _, vb, ve in got] == [(x[4], x[5]) for x in laid]
    assert all(x[3] == bam_spec.reg2bin(x[1], x[2]) for x in laid)
    assert {x[3] for x in laid if 73 <= x[3] < 585} and len({x[3] for x in laid if 585 <= x[3] < 4681}) >= 2   # 128 kb and 16 kb bins
    bai = bai_spec.write_bai(2, laid)
    ix = bai_spec.parse_bai(bai)
    assert all(len(r["intv"]) >= 15 for r in ix)
    for r in range(2):   # the pseudo-bin: first vbeg, last vend, mapped count
        mine = [x for x in laid if x[0] == r]
        (b0, e0), (nm, nu) = ix[r]["bins"][bai_spec.PSEUDO_BIN]
        assert (b0, e0, nm, nu) == (mine[0][4], mine[-1][5], len(mine), 0)
    regions = [(int(rng.integers(0, 2)), *sorted(int(x) for x in rng.integers(0, 300001, 2))) for _ in range(300)]
    regions += [(r, b, b + w) for r in range(2) for b in range(0, 300000, 16384) for w in (1, 16384, 131072)]
    regions += [(r, 0, 300000) for r in range(2)] + [(r, 131071, 131073) for r in range(2)]
    n_hit = 0
    for ref, beg, end in regions:
        if end <= beg:
            end = beg + 1
        want = bai_spec.brute(laid, ref, beg, end)
        assert bai_spec.query(ix, laid, ref, beg, end) == want, (ref, beg, end)
        n_hit += len(want)
    assert n_hit > 1000


def test_spec_bai_empty_references():
    bai = bai_spec.write_bai(3, [])
    assert bai == b"BAI\1" + struct.pack("<i", 3) + struct.pack("<ii", 0, 0) * 3 + struct.pack("<Q", 0)
    assert bai_spec.parse_bai(bai) == [dict(bins={}, intv=[])] * 3


def test_spec_chunks_merge_in_one_block():
    """two runs of one bin split by another bin's record merge when the second starts in the block where the first ends"""
    recs = [(0, 10, 20, 4681, 0 << 16 | 100, 0 << 16 | 200), (0, 11, 20000, 585, 0 << 16 | 200, 0 << 16 | 300),
            (0, 12, 30, 4681, 0 << 16 | 300, 5 << 16 | 0), (0, 13, 30, 4681, 5 << 16 | 0, 5 << 16 | 50),
            (0, 14, 20000, 585, 5 << 16 | 50, 9 << 16 | 10), (0, 15, 30, 4681, 9 << 16 | 10, 9 << 16 | 90)]
    ix = bai_spec.parse_bai(bai_spec.write_bai(1, recs))[0]
    assert ix["bins"][4681] == [(100, 5 << 16 | 50), (9 << 16 | 10, 9 << 16 | 90)]
    assert ix["bins"][585] == [(200, 300), (5 << 16 | 50, 9 << 16 | 10)]
    assert ix["intv"] == [100, 200]


# ---- the helpers of smr_fmt.h ----
def test_field_helpers(tmp_path):
    exe = str(tmp_path / "bamsort_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "bamsort_check.cpp"), "-o", exe])
    n = {"key": 0, "voff": 0, "merge": 0}
    for line in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines():
        f = line.split()
        n[f[0]] += 1
        v = [int(x) for x in f[1:]]
        if f[0] == "key":
            assert v[3] == bai_spec.sort_key(v[0], v[1], v[2]), line
        elif f[0] == "voff":
            assert v[2] == v[0] << 16 | v[1] and v[2] >> 16 == v[0], line
        else:
            assert v[2] == (v[0] >> 16 == v[1] >> 16), line
    assert n == {"key": 120, "voff": 20, "merge": 64}
    keys = sorted([(bai_spec.sort_key(r, p, f), (r, p, f)) for r in (0, 1) for p in (-1, 0, 5) for f in (0, 16)])
    assert [k[1] for k in keys] == sorted([(r, p, f) for r in (0, 1) for p in (-1, 0, 5) for f in (0, 16)])
