"""BAM on the CPU: the -bam option of the command line, the BGZF framing of smr_deflate.h run serially by tests/bgzf_check.cpp (the
steps the kernels perform, so its bytes are the device's), and BAM's field helpers of smr_fmt.h, each against tests/bam_spec.py,
which follows the SAM/BAM specification."""
import gzip
import os
import subprocess
import zlib

import numpy as np
import pytest

import bam_spec
from sortmerna_b200 import __main__ as cli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ARC, BAC, READS = (os.path.join(GOLDEN, n) for n in ("db_arc.fasta", "db_bac.fasta", "reads_mix.fq"))
G = ["-gumbel", "0.59,0.32", "-gumbel", "0.60,0.33"]


def _args(*a):
    return cli.parse_args(["-ref", ARC, "-ref", BAC, "-reads", READS, "-workdir", "/w"] + G + list(a))


# ---- the command line ----
def test_bam_option():
    k = _args("-bam")
    assert k["bam"] and not k["sam"] and k["blast"] is None   # an output format: no default BLAST
    assert not _args()["bam"] and _args()["blast"] == "1"
    assert _args("-sam", "-bam")["sam"] and _args("-sam", "-bam")["bam"]
    assert _args("-bam", "-num_alignments", "0")["params"].num_alignments == 0
    with pytest.raises(cli.UsageError, match=r"'-num_alignments' needs an output format \(-blast, -sam or -fastx\)"):
        _args("-num_alignments", "0", "-otu_map")
    with pytest.raises(cli.UsageError, match="given twice"):
        _args("-bam", "-bam")
    assert _args("-bam", "-zip-out", "1")["zip_out"]   # zip_out leaves aligned.bam alone (run_files)


def test_bam_help_line():
    line = [s for s in cli.HELP.splitlines() if s.strip().startswith("-bam")]
    assert len(line) == 1 and "aligned.bam" in line[0] and "not a reference option" in line[0]
    assert cli.HELP.index(" reports") < cli.HELP.index(line[0]) < cli.HELP.index(" alignment")


# ---- BGZF framing ----
@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    e = str(tmp_path_factory.mktemp("bgzf") / "bgzf_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "bgzf_check.cpp"), "-o", e])
    return e


def _blocks(exe, tmp_path, data: bytes):
    src, dst = tmp_path / "in.bin", tmp_path / "out.bgzf"
    src.write_bytes(data)
    p = subprocess.run([exe, "blocks", str(src), str(dst)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    f = p.stdout.split()
    return dst.read_bytes(), dict(blocks=int(f[4]), max_member=int(f[6]), bound=int(f[8]))


def _inputs():
    rng = np.random.default_rng(11)
    acgt = lambda n: np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes()  # noqa: E731
    B = bam_spec.BLOCK
    return {
        "empty": b"", "one_byte": b"\x01",
        "block_minus_1": acgt(B - 1), "block": acgt(B), "block_plus_1": acgt(B + 1),
        "random_3_blocks": rng.integers(0, 256, 3 * B + 777, dtype=np.uint8).tobytes(),
        "run": b"\0" * (5 * B),
        "reads": open(READS, "rb").read(),
    }


@pytest.mark.parametrize("name", list(_inputs()))
def test_bgzf_framing(exe, tmp_path, name):
    data = _inputs()[name]
    out, info = _blocks(exe, tmp_path, data)
    assert info["blocks"] == -(-len(data) // bam_spec.BLOCK)
    assert bam_spec.check_stream(out) == data   # BC, BSIZE, <= 64 KiB, ISIZE, CRC; each member alone; full blocks but the last
    assert gzip.decompress(out + bam_spec.EOF_BLOCK) == data
    ms = bam_spec.members(out)
    assert len(ms) == info["blocks"] and max((len(m) for m, _ in ms), default=0) == info["max_member"] <= info["bound"] <= 65536
    if name == "empty":
        assert out == b""


def test_bgzf_bound_is_reached_by_incompressible_blocks(exe, tmp_path):
    """both chunks of a full block of random bytes fall back to stored blocks: the member is exactly kBgzfMaxMember"""
    data = np.random.default_rng(3).integers(0, 256, 2 * bam_spec.BLOCK, dtype=np.uint8).tobytes()
    out, info = _blocks(exe, tmp_path, data)
    assert info["bound"] == 18 + (5 + 32768 + 5) + (5 + bam_spec.BLOCK - 32768) + 8 == 65321
    assert [len(m) for m, _ in bam_spec.members(out)] == [info["bound"]] * 2


def test_eof_block():
    m = bam_spec.members(bam_spec.EOF_BLOCK)
    assert len(m) == 1 and m[0][1] == b"" and len(bam_spec.EOF_BLOCK) == 28
    assert zlib.decompress(bam_spec.EOF_BLOCK, 31) == b""
    from sortmerna_b200 import api
    assert api.BGZF_EOF == bam_spec.EOF_BLOCK


# ---- field helpers ----
def test_field_helpers(exe):
    out = subprocess.run([exe, "fields"], capture_output=True, text=True, check=True).stdout.splitlines()
    n = {"bin": 0, "nt4": 0, "int": 0}
    for line in out:
        f = line.split()
        n[f[0]] += 1
        if f[0] == "bin":
            assert int(f[3]) == bam_spec.reg2bin(int(f[1]), int(f[2])), line
        elif f[0] == "nt4":
            assert int(f[2]) == bam_spec.NT16.index(f[1]), line
        else:
            t = bam_spec.int_tag("AS", int(f[1]))
            assert (int(f[2]), f[3]) == (len(t) - 3, chr(t[2])), line
    assert n["bin"] > 50 and n["nt4"] == 5 and n["int"] == 7


def test_spec_encoder_round_trip():
    """the encoder and the decoder of bam_spec agree on rows of both strands, soft clips, FASTA and FASTQ, and tags of every width"""
    names = ["ref_a", "ref_b"]
    rows = ["r1\t0\tref_b\t1\t255\t3S10M1I4M2D5M2S\t*\t0\t0\tACGTNACGTACGTACGTACGTACGT\t" + "I" * 25 + "\tAS:i:300\tNM:i:3",
            "r2\t16\tref_a\t70000\t255\t7M\t*\t0\t0\tACGTACG\t*\tAS:i:14\tNM:i:0",
            "q\t0\tref_a\t16384\t255\t5M\t*\t0\t0\tACGTA\t!#~+5\tAS:i:70000\tNM:i:255"]
    for row in rows:
        rid = names.index(row.split("\t")[2])
        assert bam_spec.decode_record(bam_spec.encode_row(row, rid), names) == row
