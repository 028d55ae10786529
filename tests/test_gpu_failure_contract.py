"""What a failed call of the C ABI returns and leaves behind: the status, the full smr_last_error text, the outputs the header
documents as written on failure, and a context that still aligns as a fresh one does."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN, load_case
from helpers import assert_same_results
from sortmerna_b200 import api
from sortmerna_b200.api import _ptr

pytestmark = pytest.mark.gpu

SMR_ERR_ARG, SMR_ERR_INDEX, SMR_ERR_CAPACITY = 2, 3, 5


def _load_index(a, golden, k):
    a.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], load_case("default")["log"]["minimal_score"][k], (18, 9, 3),
                      golden["stats"][k].lnwin)


def _load_truncated_index(a, golden, k):
    """smr_load_index_part of golden index k (part 0) with its kmer file cut to half its size; returns the status"""
    pre = golden["prefixes"][k]
    bufs = [np.fromfile(pre + ext + "_0.dat", dtype=np.uint8) for ext in (".kmer", ".bursttrie", ".pos")]
    bufs[0] = bufs[0][: bufs[0].size // 2].copy()
    refs = golden["refs"][k]
    cat = np.ascontiguousarray(refs.cat, np.uint8)
    off = np.ascontiguousarray(refs.off, np.uint64)
    sk = (C.c_uint32 * 3)(18, 9, 3)
    return a.L.smr_load_index_part(a.h, C.c_uint32(k), C.c_uint32(0), _ptr(bufs[0]), C.c_size_t(bufs[0].size), _ptr(bufs[1]),
                                   C.c_size_t(bufs[1].size), _ptr(bufs[2]), C.c_size_t(bufs[2].size), _ptr(cat), _ptr(off),
                                   C.c_uint32(refs.n), C.c_uint32(golden["stats"][k].lnwin), C.c_uint32(load_case("default")["log"]["minimal_score"][k]), sk)


def _aligner(golden, params=True, indexes=(0, 1)):
    a = api.Aligner(0)
    if params:
        a.set_params(api.default_params())
    for k in indexes:
        _load_index(a, golden, k)
    return a


def _err(a):
    return a.L.smr_last_error(a.h).decode()


@pytest.fixture(scope="module")
def fresh(golden):
    """the golden batch aligned on a fresh context with the default parameters"""
    a = _aligner(golden)
    b = golden["batch"]
    out = a.align(b.cat, b.off)
    a.close()
    return out


def _assert_usable(a, golden, fresh, what):
    a.set_params(api.default_params())
    b = golden["batch"]
    assert_same_results(fresh, a.align(b.cat, b.off), f"one align after {what}")


def test_gzip_cap_too_small(golden, fresh):
    a = _aligner(golden)
    with open(os.path.join(GOLDEN, "reads_mix.fq"), "rb") as f:
        data = f.read()
    size = len(a.gzip(data))
    buf = np.frombuffer(data, np.uint8)
    o = np.zeros(16, np.uint8)
    nb = C.c_uint64(0)
    rc = a.L.smr_gzip(a.h, _ptr(buf), buf.size, _ptr(o), o.size, C.cast(C.byref(nb), C.c_void_p))
    assert rc == SMR_ERR_CAPACITY
    assert _err(a) == "output buffer too small: stream_off holds the compressed sizes"
    assert nb.value == size
    _assert_usable(a, golden, fresh, "smr_gzip")
    a.close()


def test_all_alignments_stride_too_small(golden, fresh):
    """num_alignments = 0 with a stride of one slot: reads of the golden batch store more than one alignment"""
    a = _aligner(golden)
    a.set_params(api.default_params(num_alignments=0))
    a.set_aln_slots(1)
    b = golden["batch"]
    cat, off = np.ascontiguousarray(b.cat, np.uint8), np.ascontiguousarray(b.off, np.uint64)
    slots, res, alns, pool, cap, counters = a._outputs(b.n)
    assert slots == 1
    used = C.c_uint64(12345)
    rc = a.L.smr_align_batch(a.h, _ptr(cat), _ptr(off), C.c_uint32(b.n), _ptr(res), _ptr(alns), _ptr(pool), C.c_uint64(cap), C.byref(used),
                             _ptr(counters), C.c_uint32(counters.size))
    assert rc == SMR_ERR_CAPACITY
    need = int(a.L.smr_aln_slots_needed(a.h))
    assert need > 1
    assert _err(a) == (f"all-alignments mode: a read stored {need} alignments, the result stride is 1 (smr_set_aln_slots({need}) or more, "
                       "then call again)")
    assert used.value == 0   # written on failure too
    _assert_usable(a, golden, fresh, "the all-alignments stride error")
    a.close()


def test_upload_fastx_bad_first_byte(golden, fresh):
    a = _aligner(golden)
    buf = np.frombuffer(b"ACGTACGT\nACGT\n", np.uint8)
    n = C.c_uint32(7)
    rc = a.L.smr_upload_fastx(a.h, _ptr(buf), C.c_uint64(buf.size), C.byref(n))
    assert rc == SMR_ERR_ARG
    assert _err(a) == "reads text must start with '@' (FASTQ) or '>' (FASTA)"
    assert n.value == 0
    _assert_usable(a, golden, fresh, "smr_upload_fastx")
    a.close()


def test_run_resident_without_params(golden, fresh):
    a = _aligner(golden, params=False)
    b = golden["batch"]
    a.upload(b.cat, b.off)
    assert a.L.smr_run_resident(a.h) == SMR_ERR_ARG
    assert _err(a) == "smr_set_params not called"
    _assert_usable(a, golden, fresh, "smr_run_resident")
    a.close()


def test_load_truncated_index_part(golden, fresh):
    a = _aligner(golden, indexes=(0,))
    before = a.index_info()
    assert _load_truncated_index(a, golden, 1) == SMR_ERR_INDEX
    assert _err(a) == "kmer file too short"
    assert a.index_info() == before
    _load_index(a, golden, 1)
    _assert_usable(a, golden, fresh, "smr_load_index_part")
    a.close()
