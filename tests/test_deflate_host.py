"""The gzip encoder of sortmerna_b200/csrc/smr_deflate.h run on the CPU (tests/deflate_check.cpp drives the same MATCH / PARSE / CODE /
WRITE / PLACE steps the kernels perform, serially, so it writes the device's bytes): zlib and the project's own inflate logic
(tests/inflate_check.cpp) must read every output back, and the output must stay within reach of zlib's level 1."""
import json
import os
import subprocess
import zlib

import numpy as np
import pytest

import inflate_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CHUNK = 32768   # kDefChunk


def sam_text() -> bytes:
    """the SAM rows of every golden case, joined"""
    rows = []
    for d in sorted(os.listdir(GOLDEN)):
        p = os.path.join(GOLDEN, d, "expected.json")
        if d.startswith("case_") and os.path.exists(p):
            rows += json.load(open(p))["sam"]
    return "".join(r + "\n" for r in rows).encode()


def corpus():
    rng = np.random.default_rng(7)
    acgt = lambda n: np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes()  # noqa: E731
    read = lambda name: open(os.path.join(GOLDEN, name), "rb").read()  # noqa: E731
    return {
        "empty": b"", "one_byte": b"A",
        "chunk_minus_1": acgt(CHUNK - 1), "chunk": acgt(CHUNK), "chunk_plus_1": acgt(CHUNK + 1),
        "random": rng.integers(0, 256, 3 * CHUNK + 123, dtype=np.uint8).tobytes(),
        "run": b"A" * 100_000,
        "reads_mix_fq": read("reads_mix.fq"), "db_arc_fasta": read("db_arc.fasta"), "db_bac_fasta": read("db_bac.fasta"),
        "sam_rows": sam_text(),
        "fastq_multi_mb": inflate_cases.fastq_text(16000, seed=11),
    }


@pytest.fixture(scope="module")
def exes(tmp_path_factory):
    d = tmp_path_factory.mktemp("deflate")
    out = {}
    for name in ("deflate_check", "inflate_check"):
        out[name] = str(d / name)
        subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", name + ".cpp"), "-o", out[name]])
    return out


def deflate(exe, tmp_path, data: bytes):
    src, dst = tmp_path / "in.bin", tmp_path / "out.gz"
    src.write_bytes(data)
    p = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    f = p.stdout.split()
    return dst.read_bytes(), dict(chunks=int(f[4]), stored=int(f[6]))


@pytest.fixture(scope="module")
def encoded(exes, tmp_path_factory):
    d = tmp_path_factory.mktemp("enc")
    return {k: (v,) + deflate(exes["deflate_check"], d, v) for k, v in corpus().items()}


def test_zlib_reads_every_output(encoded):
    for name, (data, gz, _) in encoded.items():
        assert gz[:4] == b"\x1f\x8b\x08\x00" and gz[9] == 3, name
        assert zlib.decompress(gz, 31) == data, name


def test_own_inflate_reads_every_output(exes, encoded, tmp_path):
    for name, (data, gz, _) in encoded.items():
        if not data:
            continue   # inflate_check refuses a member shorter than a header and trailer: the empty member is zlib's own bytes
        (tmp_path / "in.gz").write_bytes(gz)
        p = subprocess.run([exes["inflate_check"], str(tmp_path / "in.gz"), str(tmp_path / "out.bin"), "4096"], capture_output=True, text=True)
        assert p.returncode == 0, (name, p.stdout)
        assert (tmp_path / "out.bin").read_bytes() == data, name


def test_forms(encoded):
    """random bytes take the stored form; a run codes as distance-1 matches of 258; chunking follows kDefChunk"""
    assert encoded["empty"][1] == bytes.fromhex("1f8b0800000000000003030000000000" "00000000")
    assert encoded["random"][2] == dict(chunks=4, stored=4)
    assert len(encoded["random"][1]) == len(encoded["random"][0]) + 10 + 8 + 4 * 5 + 3 * 5
    assert encoded["chunk"][2]["chunks"] == 1 and encoded["chunk_plus_1"][2]["chunks"] == 2
    run = encoded["run"][1]
    assert len(run) < 400 and encoded["run"][2]["stored"] == 0


def test_deterministic(exes, encoded, tmp_path):
    data, gz, _ = encoded["fastq_multi_mb"]
    assert deflate(exes["deflate_check"], tmp_path, data)[0] == gz


@pytest.mark.parametrize("name", ["reads_mix_fq", "sam_rows"])
def test_size_within_zlib_level1(encoded, name):
    data, gz, _ = encoded[name]
    assert len(gz) <= 1.15 * len(zlib.compress(data, 1)), (len(gz), len(zlib.compress(data, 1)), len(zlib.compress(data, 6)))
