"""The report writer's number formatting (sortmerna_b200/csrc/smr_fmt.h, the same code the kernels run) compiled for the CPU by
tests/report_fmt_check.cpp and compared with the C library's printf: "%.3g" of the %id / E-value / %qcov columns, "%u" / "%d"."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    e = str(tmp_path_factory.mktemp("fmt") / "report_fmt_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", os.path.join(ROOT, "tests", "report_fmt_check.cpp"), "-o", e])
    return e


@pytest.mark.parametrize("mode", [["ratios"], ["random", "10000000", "20261015"], ["bounds"], ["special"]],
                         ids=["ratios", "random", "bounds", "special"])
def test_g3_equals_printf(exe, mode):
    p = subprocess.run([exe] + mode, capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-2000:]
    assert p.stdout.startswith("ok ") and int(p.stdout.split()[1]) > 1000


def test_sam_header(tmp_path):
    """hostio.sam_header reads the sequence table of the .stats files (report_sam.cpp:154-205)"""
    import sys
    sys.path.insert(0, ROOT)
    from conftest import GOLDEN, unpack_index
    from sortmerna_b200 import hostio
    unpack_index(os.path.join(GOLDEN, "idx"), str(tmp_path))
    pre = hostio.find_index_prefixes(str(tmp_path))
    prefixes = [pre["db_arc.fasta"], pre["db_bac.fasta"]]
    h = hostio.sam_header(prefixes, "sortmerna -ref a -reads b", sq=True).split("\n")
    refs = [hostio.load_references(os.path.join(GOLDEN, n)) for n in ("db_arc.fasta", "db_bac.fasta")]
    want = [f"@SQ\tSN:{i}\tLN:{int(r.off[k + 1] - r.off[k])}" for r in refs for k, i in enumerate(r.ids)]
    assert h[0] == "@HD\tVN:1.0\tSO:unsorted" and h[1:-2] == want and h[-2] == "@PG\tID:sortmerna\tVN:1.0\tCL:sortmerna -ref a -reads b"
    assert hostio.sam_header(prefixes, "x").count("\n") == 2
