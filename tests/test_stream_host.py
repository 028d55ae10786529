"""The read stream's two passes on the CPU (tests/stream_check.cpp runs the functions the kernels use): the resumable gzip inflate,
pushed in pieces, against zlib; and the count pass against a plain restatement of the reference's count_reads_parallel."""
import gzip
import json
import os
import subprocess
import zlib

import pytest

import inflate_cases
from sortmerna_b200 import hostio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("stream")
    e = str(d / "stream_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "stream_check.cpp"), "-o", e])
    return e


def inflate(exe, tmp_path, gz, piece):
    src, dst = tmp_path / "in.gz", tmp_path / "out.bin"
    src.write_bytes(gz)
    p = subprocess.run([exe, "inflate", str(src), str(dst), str(piece)], capture_output=True, text=True)
    return p.returncode, p.stdout.strip(), (dst.read_bytes() if p.returncode == 0 else b"")


def test_pieces_equal_zlib(exe, tmp_path):
    for name, gz, want in inflate_cases.cases(1500):
        for piece in ((17,) if len(gz) < 40000 else ()) + (1024, 65536, len(gz) + 1):
            rc, msg, got = inflate(exe, tmp_path, gz, piece)
            assert rc == 0, (name, piece, msg)
            assert got == want, (name, piece, msg)


def test_one_byte_pieces(exe, tmp_path):
    txt = inflate_cases.fastq_text(40, seed=7)
    for gz in (gzip.compress(txt, 6), gzip.compress(txt[:900], 1) + gzip.compress(txt[900:], 9)):
        rc, msg, got = inflate(exe, tmp_path, gz, 1)
        assert rc == 0 and got == txt, msg


def stored_and_fixed():
    txt = inflate_cases.fastq_text(300, seed=8)
    co = zlib.compressobj(6, zlib.DEFLATED, 31, 9, zlib.Z_FIXED)
    fixed = co.compress(txt) + co.flush()
    return txt, gzip.compress(txt, 0), fixed


def test_piece_ends_at_every_kind_of_place(exe, tmp_path):
    """A piece ends inside a gzip header, inside a trailer, exactly between members, inside a stored block and inside a Z_FIXED
    block: every cut of the first piece is tried."""
    txt, stored, fixed = stored_and_fixed()
    a, b = gzip.compress(txt[:5000], 6), gzip.compress(txt[5000:], 6)
    two = a + b
    for gz, cuts in ((two, [3, 9, len(a) - 6, len(a) - 1, len(a), len(a) + 5]), (stored, [7, 100, 5000, len(stored) - 3]),
                     (fixed, [20, 777, len(fixed) // 2, len(fixed) - 4])):
        for cut in cuts:
            src, dst = tmp_path / "in.gz", tmp_path / "out.bin"
            # pushing `cut` bytes first and then the rest is the same as pieces of `cut` for the first two pieces
            src.write_bytes(gz)
            p = subprocess.run([exe, "inflate", str(src), str(dst), str(cut)], capture_output=True, text=True)
            assert p.returncode == 0, (cut, p.stdout)
            assert dst.read_bytes() == txt, cut


def test_bad_input_is_refused(exe, tmp_path):
    for name, gz in inflate_cases.bad_cases():
        for piece in (1024, 65536, len(gz) + 1):
            rc, msg, _ = inflate(exe, tmp_path, gz, piece)
            assert rc == 1 and msg.startswith("error"), (name, piece, msg)
            # refused no later than the push that ends the file
            assert int(msg.split()[3]) <= (len(gz) - 1) // piece, (name, piece, msg)
    # a file that is no gzip member is refused at its first push, not held until the end
    for piece in (4, 17, 1024):
        rc, msg, _ = inflate(exe, tmp_path, b"@r\nACGT\n+\nIIII\n" * 4000, piece)
        assert rc == 1 and msg.split()[3] == "0", (piece, msg)
    # bytes after the last member that are no member are ignored, in whatever pieces they come
    txt = inflate_cases.fastq_text(50, seed=15)
    for piece in (5, 100, 100000):
        rc, msg, got = inflate(exe, tmp_path, gzip.compress(txt) + b"trailing garbage" * 10, piece)
        assert rc == 0 and got == txt, (piece, msg)


def ref_count(data: bytes, state=None, lines=None):
    """count_reads_parallel of readfeed.cpp:1486-1663 at one split, byte by byte."""
    lines = lines or (4 if data[:1] == b"@" else 2)
    st = state or {"reads": 0, "length": 0, "min_len": 0, "max_len": 0}
    pos, seqlen = 0, 0
    for c in data:
        if c == 10:
            if pos == 1:
                st["reads"] += 1
                st["length"] += seqlen
                st["max_len"] = max(st["max_len"], seqlen)
                if st["min_len"] == 0 or seqlen < st["min_len"]:
                    st["min_len"] = seqlen
                seqlen = 0
            pos = (pos + 1) % lines
        elif pos == 1:
            seqlen += 1
    return st


def ref_count_run(files):
    """count_reads_parallel over the -reads files of one run, [(bytes, is_gz)]: the line cycle of the first file for all; a gzip
    file updates the run's minimum read by read (readfeed.cpp:1522), a flat file is counted alone and merged (readfeed.cpp:1647-1657)"""
    lines = 4 if files[0][0][:1] == b"@" else 2
    st = {"reads": 0, "length": 0, "min_len": 0, "max_len": 0}
    for data, gz in files:
        one = ref_count(data, dict(st) if gz else None, lines)
        if gz:
            st = one
            continue
        st["reads"] += one["reads"]
        st["length"] += one["length"]
        st["max_len"] = max(st["max_len"], one["max_len"])
        if st["min_len"] == 0 or 0 < one["min_len"] < st["min_len"]:
            st["min_len"] = one["min_len"]
    return st


def count(exe, tmp_path, data, piece):
    src = tmp_path / "in.txt"
    src.write_bytes(data)
    out = subprocess.run([exe, "count", str(src), "x", str(piece)], capture_output=True, text=True, check=True).stdout.split()
    return dict(zip(("reads", "length", "min_len", "max_len"), map(int, out)))


def count_inputs():
    fq = inflate_cases.fastq_text(200, seed=9)
    return {
        "fastq": fq,
        "crlf": fq.replace(b"\n", b"\r\n"),
        "no_final_newline": fq.rstrip(b"\n"),
        "multiline_fasta": b"".join(b">r%d\nACGTACGT\nTTGA\nC\n" % i for i in range(50)) + b">last\nACG\n",
        "empty_seq_lines": b">a\nACGT\n>b\n\n>c\nAC\n>d\nACGTA\n>e\n\n>f\nA\n",
        "empty_last": b">a\nACGT\n>b\n\n",
        "fasta": b"".join(b">s%d\n%s\n" % (i, b"ACGT" * (i % 7 + 1)) for i in range(300)),
    }


def test_count_model_equals_count_reads_parallel(exe, tmp_path):
    for name, data in count_inputs().items():
        want = ref_count(data)
        for piece in (1, 17, 1024, 65536, len(data)):
            assert count(exe, tmp_path, data, piece) == want, (name, piece)


def test_golden_counts_give_every_minimal_score(exe, tmp_path):
    data = open(os.path.join(GOLDEN, "reads_mix.fq"), "rb").read()
    c = count(exe, tmp_path, data, 4096)
    assert c == ref_count(data)
    pre = hostio.find_index_prefixes(os.path.join(GOLDEN, "idx"))
    stats = [hostio.parse_stats(pre[n]) for n in ("db_arc.fasta", "db_bac.fasta")]
    cases = sorted(d for d in os.listdir(GOLDEN) if d.startswith("case_"))
    assert cases
    for case in cases:
        log = json.load(open(os.path.join(GOLDEN, case, "expected.json")))["log"]
        assert log["total_reads"] == c["reads"], case
        for k, ms in enumerate(log["minimal_score"]):
            assert hostio.minimal_score(stats[k], log["lambda_"][k], log["K"][k], c["length"], c["reads"]) == ms, case
