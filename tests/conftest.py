import gzip
import json
import lzma
import os
import shutil
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


def unpack_index(src, d):
    """A stored golden index into d: .gz and .xz members decompressed (xz where gzip would exceed 1 MB), the rest copied."""
    for fn in os.listdir(src):
        if fn.endswith((".gz", ".xz")):
            with (gzip.open if fn.endswith(".gz") else lzma.open)(os.path.join(src, fn), "rb") as fi, open(os.path.join(d, fn[:-3]), "wb") as fo:
                shutil.copyfileobj(fi, fo)
        else:
            shutil.copy(os.path.join(src, fn), d)


@pytest.fixture(scope="session")
def golden_idx_dir():
    """The reference-built index of the two golden database slices, gunzipped into a temp dir."""
    d = tempfile.mkdtemp(prefix="smr_idx_")
    unpack_index(os.path.join(GOLDEN, "idx"), d)
    yield d
    shutil.rmtree(d, ignore_errors=True)


@pytest.fixture(scope="session")
def golden(golden_idx_dir):
    """Inputs of the golden cases: references, reads, index prefixes (in --ref order: arc, bac)."""
    from sortmerna_b200 import hostio
    refs = [hostio.load_references(os.path.join(GOLDEN, "db_arc.fasta")), hostio.load_references(os.path.join(GOLDEN, "db_bac.fasta"))]
    pre = hostio.find_index_prefixes(golden_idx_dir)
    prefixes = [pre["db_arc.fasta"], pre["db_bac.fasta"]]
    stats = [hostio.parse_stats(p) for p in prefixes]
    batch = hostio.load_reads(os.path.join(GOLDEN, "reads_mix.fq"))
    return dict(refs=refs, prefixes=prefixes, stats=stats, batch=batch)


def load_case(name):
    with open(os.path.join(GOLDEN, "case_" + name, "expected.json")) as f:
        return json.load(f)


def load_denovo():
    with open(os.path.join(GOLDEN, "denovo.json")) as f:
        return json.load(f)


MULTIPART_CASES = ("parts",)   # golden cases whose index LAYOUT differs (tests/golden/make_golden.py EXTRA_INDEX_CASES)


def case_names():
    return sorted(d[5:] for d in os.listdir(GOLDEN) if d.startswith("case_") and d[5:] not in MULTIPART_CASES)


@pytest.fixture(scope="session")
def golden_parts():
    """The two golden database slices indexed in 3 parts each (smr_build_index with -m 0.5, proven equal to the reference's
    builder in tests/test_index_builder.py), with the per-part references."""
    from sortmerna_b200 import api, hostio
    d = tempfile.mkdtemp(prefix="smr_idx_parts_")
    out = []
    for name in ("db_arc.fasta", "db_bac.fasta"):
        fasta = os.path.join(GOLDEN, name)
        prefix = os.path.join(d, name)
        api.build_index(fasta, prefix, max_mb=0.5)
        st = hostio.parse_stats(prefix)
        out.append(dict(prefix=prefix, stats=st, part_refs=hostio.split_by_parts(hostio.load_references(fasta), st)))
    yield out
    shutil.rmtree(d, ignore_errors=True)


@pytest.fixture(scope="session")
def golden_t0():
    """BASELINE config 1: the 1.5 kb read of data/test_read.fasta vs data/test_ref.fasta (single-line copies), with the
    reference's own index and output (tests/golden/t0/, made by make_golden.make_t0)."""
    from sortmerna_b200 import hostio
    d = tempfile.mkdtemp(prefix="smr_idx_t0_")
    unpack_index(os.path.join(GOLDEN, "t0", "idx"), d)
    refs = hostio.load_references(os.path.join(GOLDEN, "t0", "db_t0.fasta"))
    prefix = hostio.find_index_prefixes(d)["db_t0.fasta"]
    batch = hostio.load_reads(os.path.join(GOLDEN, "t0", "reads_t0.fasta"))
    with open(os.path.join(GOLDEN, "t0", "expected.json")) as f:
        exp = json.load(f)
    yield dict(refs=refs, prefix=prefix, stats=hostio.parse_stats(prefix), batch=batch, exp=exp)
    shutil.rmtree(d, ignore_errors=True)
