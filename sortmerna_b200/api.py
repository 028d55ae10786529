"""ctypes binding of libsmr_b200.so (include/smr_b200.h) and a host-side driver that mirrors the
reference's `align()` call (src/sortmerna/processor.cpp:173-285): load every (index, part) given
with --ref, then push batches of reads through the GPU hot path.

There is NO CPU fallback: importing this module without the built extension, or creating an
`Aligner` without a CUDA device, raises.  (The CPU oracle lives under oracle/ and is test
infrastructure; nothing here imports it.)
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import hostio

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SMR_LIB_PATH") or os.path.join(HERE, "libsmr_b200.so")  # override: kernel-variant experiments only

STATUS = {0: "SMR_OK", 1: "SMR_ERR_CUDA", 2: "SMR_ERR_ARG", 3: "SMR_ERR_INDEX", 4: "SMR_ERR_UNSUPPORTED",
          5: "SMR_ERR_CAPACITY", 6: "SMR_ERR_NO_DEVICE"}

# every symbol include/smr_b200.h declares
SYMBOLS = ["smr_init", "smr_destroy", "smr_last_error", "smr_device_count", "smr_load_index_part",
           "smr_set_minimal_score", "smr_set_params", "smr_index_info", "smr_align_batch", "smr_upload_batch",
           "smr_run_resident", "smr_download_results", "smr_last_timings", "smr_debug_seed_windows", "smr_debug_ssw",
           "smr_debug_dpx_peak", "smr_set_stats_buffer", "smr_build_index", "smr_upload_fastx", "smr_resident_layout", "smr_pack_kvdb_blobs",
           "smr_set_aln_slots", "smr_aln_slots", "smr_aln_slots_needed", "smr_upload_fastx_gz", "smr_resident_text", "smr_debug_inflate",
           "smr_build_index_device", "smr_debug_index_array", "smr_set_instrumentation", "smr_set_report_refs", "smr_set_report_scoring",
           "smr_format_reports", "smr_last_report_timings", "smr_otu_begin", "smr_otu_add", "smr_otu_finish", "smr_last_otu_timings",
           "smr_format_reports_gz", "smr_gzip", "smr_stream_begin", "smr_stream_push", "smr_stream_next", "smr_stream_counts",
           "smr_stream_push_mate", "smr_format_blast_pairwise", "smr_format_blast_pairwise_gz",
           "smr_denovo_stats", "smr_set_aln_layout", "smr_align_batch_packed", "smr_download_results_packed", "smr_pack_kvdb_blobs_packed",
           "smr_set_index_budget", "smr_index_residency", "smr_set_place_stats", "smr_place_results", "smr_download_placed",
           "smr_last_place_timing", "smr_format_reports_placed", "smr_format_reports_placed_gz", "smr_format_blast_pairwise_placed",
           "smr_format_blast_pairwise_placed_gz", "smr_otu_add_placed", "smr_denovo_stats_placed",
           "smr_place_results_packed", "smr_format_bam_placed", "smr_bam_header", "smr_bam_sort_begin", "smr_bam_sort_add_placed",
           "smr_bam_sort_plan", "smr_bam_sort_window", "smr_bam_sort_index"]

# the BGZF end-of-file marker (SAMv1 4.1.2): an empty BGZF block, written once at the end of a BAM file
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
# the coordinate-sorted aligned.bam (Aligner.bam_sort_*): the bytes of records run_files compresses per window, and the BGZF bounds
# (smr_deflate.h: kBgzfBlock input bytes per block, at most kBgzfMaxMember bytes per member)
BAM_SORT_WINDOW = 256 << 20
BGZF_BLOCK, BAM_MAX_MEMBER = 65280, 65321

# smr_set_aln_layout: strided, nreads * slots alignments; packed, read r's n_align alignments from the sum of the counts before it
ALN_LAYOUTS = {"strided": 0, "packed": 1}

CNT_NAMES = ("num_aligned", "num_short", "sw_calls", "sw_cells", "windows", "trie_nodes", "buckets",
             "bucket_entries", "pos_entries", "lis_calls", "dbg_max_read_cycles", "dbg_sum_read_cycles", "dbg_lis_kernel_cycles",
             "cyc_vote", "cyc_order", "cyc_group", "cyc_plan", "cyc_wait", "cyc_replay", "spec_calls", "spec_cells", "spec_pairs", "slow_pairs",
             "sc_wait", "sc_load", "sc_sw", "sc_pub", "rounds_a", "rounds_b", "w1_cyc", "w1_cnt", "dbg_max_read_busy_cycles")
CNT_FIXED = 32


class Params(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "match", "mismatch", "score_N", "gap_open", "gap_ext", "num_seeds", "min_lis", "edges",
        "edges_is_percent", "num_alignments", "is_best", "is_forward", "is_reverse", "is_full_search",
        "minoccur")]


def default_params(**kw) -> Params:
    """Runopts::validate defaults (src/sortmerna/options.cpp:1684-1738)."""
    p = Params(match=2, mismatch=-3, score_N=-3, gap_open=5, gap_ext=2, num_seeds=2, min_lis=2, edges=4,
               edges_is_percent=0, num_alignments=1, is_best=1, is_forward=1, is_reverse=1, is_full_search=0,
               minoccur=0)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


RESULT_DTYPE = np.dtype([("lastIndex", "<u4"), ("lastPart", "<u4"), ("hit_seeds", "<u4"), ("min_index", "<u4"),
                         ("max_index", "<u4"), ("n_align", "<u4"), ("max_SW_count", "<u2"), ("is_done", "u1"),
                         ("is_hit", "u1")])
ALN_DTYPE = np.dtype([("cigar_off", "<u4"), ("cigar_len", "<u4"), ("ref_num", "<u4"), ("ref_begin1", "<i4"),
                      ("ref_end1", "<i4"), ("read_begin1", "<i4"), ("read_end1", "<i4"), ("readlen", "<u4"),
                      ("score1", "<u2"), ("part", "<u2"), ("index_num", "<u2"), ("strand", "u1"), ("pad", "u1")])

STATS_DTYPE = np.dtype([("n_miss", "<u4"), ("n_gap", "<u4"), ("n_match", "<u4"), ("n_match_denovo", "<u4")])

BLAST_COLS = {"cigar": 1, "qcov": 2, "qstrand": 3}


class ReportOpts(C.Structure):
    """smr_report_opts (include/smr_b200.h)"""
    _fields_ = [("sam", C.c_int32), ("blast", C.c_int32), ("blast_format", C.c_int32), ("blast_cols", C.c_int32 * 4), ("fastx", C.c_int32),
                ("other", C.c_int32), ("denovo", C.c_int32), ("min_id", C.c_double), ("min_cov", C.c_double), ("paired_in", C.c_int32),
                ("paired_out", C.c_int32), ("out2", C.c_int32), ("sout", C.c_int32), ("mates", C.c_int32)]


def report_opts(sam=False, blast=None, fastx=False, other=False, denovo=None, paired_in=False, paired_out=False, out2=False, sout=False,
                mates=False) -> ReportOpts:
    """blast: None, or the value of the reference's -blast option ('1 cigar qcov qstrand'; '0' = pairwise, written by
    format_blast_pairwise and refused by format_reports);
    denovo: None, or (min_id, min_cov) = the reference's -id / -coverage; mates: records 2k and 2k+1 come from two mate files
    (implied for the resident batch of stream_mates)."""
    o = ReportOpts(sam=int(bool(sam)), fastx=int(bool(fastx)), other=int(bool(other)), paired_in=int(bool(paired_in)),
                   paired_out=int(bool(paired_out)), out2=int(bool(out2)), sout=int(bool(sout)), mates=int(bool(mates)))
    if blast is not None:
        f = str(blast).split()
        o.blast, o.blast_format = 1, int(f[0])
        for k, c in enumerate(f[1:]):
            o.blast_cols[k] = BLAST_COLS[c]
    if denovo is not None:
        o.denovo, o.min_id, o.min_cov = 1, float(denovo[0]), float(denovo[1])
    return o


class OtuOpts(C.Structure):
    """smr_otu_opts (include/smr_b200.h)"""
    _fields_ = [("min_id", C.c_double), ("min_cov", C.c_double), ("paired_in", C.c_int32), ("paired_out", C.c_int32), ("feed", C.c_int32)]


# smr_otu_opts.feed: which records of a paired run the OTU map looks at (SMR_OTU_ONE_FILE: every record of one interleaved file;
# SMR_OTU_TWO_FILES: the first file's records 2k of two mate files)
OTU_FEEDS = {None: 0, "one_file": 1, "two_files": 2}


class DenovoOpts(C.Structure):
    """smr_denovo_opts (include/smr_b200.h)"""
    _fields_ = [("min_id", C.c_double), ("min_cov", C.c_double), ("paired", C.c_int32)]


DENOVO_TOTALS = ("n_yid_ycov", "n_yid_ncov", "n_nid_ycov", "num_denovo")


def num_out_of(o: ReportOpts) -> int:
    """files per kind of read file (ReportFxBase::set_num_out, report_fx_base.cpp:165-171)"""
    return 4 if o.out2 and o.sout else 2 if o.out2 or o.sout else 1


def fx_suffixes(o: ReportOpts) -> list:
    """the name suffixes of a kind's num_out files, in stream order (report_fx_base.cpp:73-90)"""
    n = num_out_of(o)
    if n == 4:
        return ["_paired_fwd", "_paired_rev", "_singleton_fwd", "_singleton_rev"]
    if n == 2:
        return ["_fwd", "_rev"] if o.out2 else ["_paired", "_singleton"]
    return [""]


_lib = None


def load_library():
    """Load the extension; raises if it has not been built (no silent fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(nvcc, sm_90a). There is no CPU fallback for the alignment hot path.")
        L = C.CDLL(LIB_PATH)
        L.smr_last_error.restype = C.c_char_p
        L.smr_last_error.argtypes = [C.c_void_p]
        L.smr_init.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.smr_destroy.argtypes = [C.c_void_p]
        L.smr_destroy.restype = None
        L.smr_aln_slots.restype = C.c_uint32
        L.smr_aln_slots.argtypes = [C.c_void_p]
        L.smr_aln_slots_needed.restype = C.c_uint32
        L.smr_aln_slots_needed.argtypes = [C.c_void_p]
        L.smr_set_aln_slots.argtypes = [C.c_void_p, C.c_uint32]
        L.smr_set_instrumentation.argtypes = [C.c_void_p, C.c_int]
        L.smr_stream_begin.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64]
        L.smr_stream_push.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int]
        L.smr_stream_next.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_int)]
        L.smr_stream_counts.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.smr_stream_push_mate.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_int]
        L.smr_set_index_budget.argtypes = [C.c_void_p, C.c_uint64]
        L.smr_index_residency.argtypes = [C.c_void_p, C.c_void_p]
        for name in SYMBOLS:
            getattr(L, name)  # AttributeError if the build is stale
        _lib = L
    return _lib


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


def build_index(fasta: str, out_prefix: str, lnwin: int = 18, interval: int = 1, max_pos: int = 10000, max_mb: float = 3072.0,
                threads: int = 0) -> dict:
    """smr_build_index: the native stand-in for the reference's `build_index` (indexdb.cpp:1119-2095).  Host code only (no GPU
    needed); writes <out_prefix>.{kmer,bursttrie,pos}_P.dat + .stats.  Defaults = the reference's (-L 18 -interval 1 -max_pos 10000 -m 3072)."""
    L = load_library()
    L.smr_build_index.argtypes = [C.c_char_p, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, C.c_uint32, C.POINTER(C.c_uint64),
                                  C.c_char_p, C.c_size_t]
    rep = (C.c_uint64 * 6)()
    err = C.create_string_buffer(1024)
    rc = L.smr_build_index(os.fsencode(fasta), os.fsencode(out_prefix), lnwin, interval, max_pos, float(max_mb), threads, rep, err, len(err))
    if rc != 0:
        raise SmrError(f"smr_build_index({fasta}): {err.value.decode(errors='replace')}")
    return dict(zip(("parts", "numseq", "windows", "unique_lmers", "trie_nodes", "bytes_written"), (int(x) for x in rep)))


def pack_kvdb_blobs(out: dict, num_alignments: int, denovo: np.ndarray | None = None):
    """smr_pack_kvdb_blobs: Read::toBinString() of every read of a result dict (align() / download() / the oracle's), as
    (blob bytes, offsets[nreads+1]).  denovo: optional (nreads, 4) uint32 counters of hostio.denovo_classes.  A packed result
    (slots == 0) goes through smr_pack_kvdb_blobs_packed."""
    L = load_library()
    res, alns, cig, slots = out["res"], out["alns"], np.ascontiguousarray(out["cigar"], np.uint32), int(out["slots"])
    n = res.shape[0]
    off = np.zeros(n + 1, np.uint64)
    dn = np.ascontiguousarray(denovo, np.uint32) if denovo is not None else None
    fn, name = (L.smr_pack_kvdb_blobs_packed, "smr_pack_kvdb_blobs_packed") if slots == 0 else (L.smr_pack_kvdb_blobs, "smr_pack_kvdb_blobs")
    args = [_ptr(res), _ptr(alns) if alns.size else C.c_void_p(0), _ptr(cig) if cig.size else C.c_void_p(0), C.c_uint32(n)]
    args += ([] if slots == 0 else [C.c_uint32(slots)]) + [C.c_int32(num_alignments), _ptr(dn) if dn is not None else C.c_void_p(0)]
    rc = fn(*args, C.c_void_p(0), C.c_uint64(0), _ptr(off))
    if rc != 0:
        raise SmrError(f"{name}: {STATUS.get(rc, rc)}")
    buf = np.zeros(int(off[n]), np.uint8)
    rc = fn(*args, _ptr(buf) if buf.size else C.c_void_p(0), C.c_uint64(buf.size), _ptr(off))
    if rc != 0:
        raise SmrError(f"{name}: {STATUS.get(rc, rc)}")
    return buf, off


def unpack_alns(out: dict, slots: int) -> dict:
    """The strided equivalent of a packed result (slots == 0) at stride `slots` (at least its largest n_align): "alns" and "stats"
    with read r's alignments at r * slots, "slots" = slots, "aln_off" dropped; the rest is shared with `out`."""
    res = out["res"]
    n, cnt = res.shape[0], res["n_align"].astype(np.int64)
    if cnt.size and int(cnt.max()) > slots:
        raise ValueError(f"unpack_alns: a read stores {int(cnt.max())} alignments, more than {slots} slots")
    off = np.asarray(out["aln_off"], np.int64)
    read = np.repeat(np.arange(n, dtype=np.int64), cnt)
    dst = read * slots + (np.arange(int(off[-1]) if off.size else 0, dtype=np.int64) - off[:-1][read])
    u = {k: v for k, v in out.items() if k != "aln_off"}
    u["alns"] = np.zeros(n * slots, ALN_DTYPE)
    u["alns"][dst] = out["alns"]
    if out.get("stats") is not None:
        u["stats"] = np.zeros(n * slots, STATS_DTYPE)
        u["stats"][dst] = out["stats"]
    u["slots"] = slots
    return u


def pack_alns(out: dict) -> dict:
    """The packed equivalent of a strided result: the inverse of unpack_alns."""
    res, slots = out["res"], int(out["slots"])
    cnt = res["n_align"].astype(np.int64)
    read = np.repeat(np.arange(res.shape[0], dtype=np.int64), cnt)
    off = np.zeros(res.shape[0] + 1, np.uint64)
    np.cumsum(cnt, out=off[1:])
    src = read * slots + (np.arange(int(off[-1]), dtype=np.int64) - off[:-1].astype(np.int64)[read])
    p = dict(out)
    p["alns"] = out["alns"][src].copy()
    if out.get("stats") is not None:
        p["stats"] = out["stats"][src].copy()
    p["slots"], p["aln_off"] = 0, off
    return p


class SmrError(RuntimeError):
    pass


class Aligner:
    """One GPU context.  Mirrors the objects `align()` receives: Index (+References, Refstats) via
    load_index_part, Runopts via set_params, Readfeed batches via align()."""

    def __init__(self, device: int = 0):
        self.L = load_library()
        self.h = C.c_void_p()
        rc = self.L.smr_init(device, C.byref(self.h))
        if rc != 0:
            raise SmrError(f"smr_init(device={device}) failed: {STATUS.get(rc, rc)} -- a CUDA device is required; "
                           "there is no CPU fallback")
        self.params = None
        self.n_index_files = 0
        self.refs_by_index = {}
        self.parts = []          # loaded (index_num, part)
        self.layout = "strided"  # set_aln_layout
        self._packed_sizes = (0, 0)   # packed layout: the largest alignment count and CIGAR words named so far (_packed_call)
        self._stats_packed = False
        self._report_refs = set()
        self._keep = []

    def _check(self, rc, what):
        if rc != 0:
            raise SmrError(f"{what}: {STATUS.get(rc, rc)}: {self.L.smr_last_error(self.h).decode()}")

    def close(self):
        if self.h:
            self.L.smr_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_params(self, params: Params):
        self.params = params
        self._check(self.L.smr_set_params(self.h, C.byref(params)), "smr_set_params")

    def set_instrumentation(self, on: bool):
        """smr_set_instrumentation: the instrumented instantiations of the seed and candidate kernels (seed-side counters and the
        cycle shares in `counters`); default off."""
        self._check(self.L.smr_set_instrumentation(self.h, C.c_int(1 if on else 0)), "smr_set_instrumentation")

    def set_aln_slots(self, slots: int):
        """smr_set_aln_slots: stride of the result layout in the all-alignments mode (num_alignments == 0); in the packed layout, the
        stride of the first run (reads that store more run again at their own count)."""
        self._check(self.L.smr_set_aln_slots(self.h, C.c_uint32(slots)), "smr_set_aln_slots")

    def set_aln_layout(self, layout: str):
        """smr_set_aln_layout: "strided" (default) or "packed".  Packed: align() / download() return "alns" and "stats" holding each
        read's n_align alignments one read after another, "aln_off" (uint64, nreads + 1) where each read's start, and slots = 0;
        format_reports / otu_add / denovo_stats / pack_kvdb_blobs take such results as they are, unpack_alns turns them strided."""
        self._check(self.L.smr_set_aln_layout(self.h, C.c_uint32(ALN_LAYOUTS[layout])), "smr_set_aln_layout")
        self.layout = layout

    def _packed_call(self, fn, name, head, n, with_stats):
        """smr_align_batch_packed / smr_download_results_packed.  The alignment array and the CIGAR pool start at the largest sizes
        the library named on this Aligner (grow-only, as the strided stride is kept), and after SMR_ERR_CAPACITY they grow to the
        sizes it names and the results are downloaded again (smr_download_results_packed: the batch is resident and run, and the
        library keeps the placed results of its run, so that call only copies)."""
        cap, words = self._packed_sizes
        cap, words = max(cap, n, 1), max(words, 48 * max(n, 1) + 4096)
        while True:
            res = np.zeros(n, RESULT_DTYPE)
            alns = np.zeros(cap, ALN_DTYPE)
            stats = np.zeros(cap, STATS_DTYPE) if with_stats else None
            pool = np.zeros(words, np.uint32)
            counters = np.zeros(CNT_FIXED + max(1, self.n_index_files), np.uint64)
            used, wused = C.c_uint64(0), C.c_uint64(0)
            rc = fn(*head, _ptr(res), _ptr(alns), C.c_uint64(cap), C.byref(used), _ptr(stats) if with_stats else C.c_void_p(0), _ptr(pool),
                    C.c_uint64(words), C.byref(wused), _ptr(counters), C.c_uint32(counters.size))
            if rc == 5 and (used.value > cap or wused.value > words):
                cap, words = max(cap, used.value), max(words, wused.value)
                self._packed_sizes = (cap, words)
                fn, name, head = self.L.smr_download_results_packed, "smr_download_results_packed", [self.h]
                continue
            break
        self._check(rc, name)
        out = self._pack(res, alns[:used.value], pool, wused.value, counters, 0)
        out["aln_off"] = np.zeros(n + 1, np.uint64)
        np.cumsum(res["n_align"], out=out["aln_off"][1:])
        if with_stats:
            out["stats"] = stats[:used.value]
        return out

    def load_index_part(self, index_num: int, part: int, prefix: str, refs: hostio.References, minimal_score: int,
                        skiplengths=(18, 9, 3), lnwin: int = 18):
        sfx = f"_{part}.dat"
        bufs = [np.fromfile(prefix + ext + sfx, dtype=np.uint8) for ext in (".kmer", ".bursttrie", ".pos")]
        sk = (C.c_uint32 * 3)(*skiplengths)
        cat = np.ascontiguousarray(refs.cat, np.uint8)
        off = np.ascontiguousarray(refs.off, np.uint64)
        rc = self.L.smr_load_index_part(self.h, C.c_uint32(index_num), C.c_uint32(part),
                                        _ptr(bufs[0]), C.c_size_t(bufs[0].size), _ptr(bufs[1]), C.c_size_t(bufs[1].size),
                                        _ptr(bufs[2]), C.c_size_t(bufs[2].size), _ptr(cat), _ptr(off), C.c_uint32(refs.n),
                                        C.c_uint32(lnwin), C.c_uint32(minimal_score), sk)
        self._check(rc, f"smr_load_index_part({prefix})")
        self.n_index_files = max(self.n_index_files, index_num + 1)
        self.refs_by_index[index_num] = refs
        self.parts.append((index_num, part))

    def build_index_device(self, index_num: int, fasta: str, refs=None, minimal_score: int = 0, skiplengths=(18, 9, 3), lnwin: int = 18,
                           interval: int = 1, max_pos: int = 10000, max_mb: float = 3072.0) -> int:
        """smr_build_index_device: the index of `fasta` built on the device and kept resident (every part); returns the number of
        parts.  refs: what the result formatters use for this index (a References, or the per-part list of hostio.split_by_parts)."""
        sk = (C.c_uint32 * 3)(*skiplengths)
        nparts = C.c_uint32(0)
        rep = (C.c_uint64 * 6)()
        self.L.smr_build_index_device.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, C.c_void_p, C.c_uint32,
                                                  C.c_void_p, C.c_void_p]
        rc = self.L.smr_build_index_device(self.h, index_num, os.fsencode(fasta), lnwin, interval, max_pos, float(max_mb), C.cast(sk, C.c_void_p), minimal_score,
                                           C.cast(C.byref(nparts), C.c_void_p), C.cast(rep, C.c_void_p))
        self._check(rc, f"smr_build_index_device({fasta})")
        self.n_index_files = max(self.n_index_files, index_num + 1)
        if refs is not None:
            self.refs_by_index[index_num] = refs
        self.parts += [(index_num, p) for p in range(int(nparts.value))]
        self.last_build_report = dict(zip(("parts", "numseq", "windows", "unique_lmers", "trie_nodes", "hbm_bytes"), (int(x) for x in rep)))
        return int(nparts.value)

    def index_array(self, slot: int, which: str) -> np.ndarray:
        """smr_debug_index_array: a resident array of loaded part `slot` (flookup u32x4 rows, flist {text,id}, pos_off, pos {pos,seq}, refseq, ref_off)."""
        k = ("flookup", "flist", "pos_off", "pos", "refseq", "ref_off").index(which)
        nb = C.c_uint64(0)
        self._check(self.L.smr_debug_index_array(self.h, C.c_uint32(slot), C.c_uint32(k), C.c_void_p(0), C.c_uint64(0), C.byref(nb)), "smr_debug_index_array")
        out = np.zeros(int(nb.value), np.uint8)
        if out.size:
            self._check(self.L.smr_debug_index_array(self.h, C.c_uint32(slot), C.c_uint32(k), _ptr(out), C.c_uint64(out.size), C.byref(nb)), "smr_debug_index_array")
        if which == "refseq":
            return out
        a = out.view(np.uint32)
        return a.reshape(-1, {"flookup": 4, "flist": 2, "pos": 2}.get(which, 1)) if which in ("flookup", "flist", "pos") else a

    def set_minimal_score(self, index_num: int, score: int):
        self._check(self.L.smr_set_minimal_score(self.h, C.c_uint32(index_num), C.c_uint32(score)), "smr_set_minimal_score")

    def index_info(self):
        out = np.zeros(6, np.uint64)
        self._check(self.L.smr_index_info(self.h, _ptr(out)), "smr_index_info")
        return dict(zip(("parts", "hbm_bytes", "nodes", "entries", "ids", "positions"), map(int, out)))

    def set_index_budget(self, nbytes: int):
        """smr_set_index_budget: at most `nbytes` of the parts' search arrays on the device (0: no limit).  Parts beyond it are
        held in pinned host memory and each run uploads them group by group; results are those of a run without a budget."""
        self._check(self.L.smr_set_index_budget(self.h, int(nbytes)), "smr_set_index_budget")

    def index_residency(self) -> dict:
        """smr_index_residency: the groups of the next run, the bytes of the largest, the search-array bytes on the device and in
        pinned host memory, the group uploads and their bytes since the context was made, and the last run's upload time (us)."""
        out = np.zeros(7, np.uint64)
        self._check(self.L.smr_index_residency(self.h, _ptr(out)), "smr_index_residency")
        return dict(zip(("groups", "largest_group_bytes", "device_search_bytes", "host_bytes", "uploads", "upload_bytes", "last_upload_us"),
                        map(int, out)))

    def _outputs(self, n, reuse=False, cigar_words=0):
        """result buffers of n reads; the CIGAR pool holds 48 words per alignment slot, or cigar_words if that is more"""
        slots = int(self.L.smr_aln_slots(self.h))   # num_alignments, or the stride of the all-alignments mode (0)
        if reuse:   # the same host buffers for every call of this shape (a streaming caller consumes a batch before the next)
            key = (n, slots, self.n_index_files, cigar_words)
            if getattr(self, "_out_key", None) != key:
                self._out_key, self._out_bufs = key, self._outputs(n, cigar_words=cigar_words)
            bufs = self._out_bufs
            bufs[5][:] = 0
            return bufs
        res = np.zeros(n, RESULT_DTYPE)
        alns = np.zeros(n * slots, ALN_DTYPE)
        cap = max(48 * n * slots + 4096, cigar_words)
        pool = np.zeros(cap, np.uint32)
        counters = np.zeros(CNT_FIXED + max(1, self.n_index_files), np.uint64)
        return slots, res, alns, pool, cap, counters

    def _pack(self, res, alns, pool, used, counters, slots):
        cnt = {k: int(counters[i]) for i, k in enumerate(CNT_NAMES)}
        return dict(res=res, alns=alns, cigar=pool[: used], matched=counters[CNT_FIXED:].copy(), counters=cnt,
                    slots=slots, timings=self.timings())

    def align(self, cat: np.ndarray, off: np.ndarray, with_stats: bool = False, reuse_outputs: bool = False):
        """smr_align_batch: host buffers in, host results out (H2D and D2H inside the call).
        with_stats: also return calc_miss_gap_match per stored alignment (out["stats"], computed on the GPU).
        reuse_outputs: write into the result buffers of the previous call of the same shape (valid until the next call)
        instead of allocating ~260 B/read of fresh zeroed host memory per call."""
        cat = np.ascontiguousarray(cat, np.uint8)
        off = np.ascontiguousarray(off, np.uint64)
        n = off.size - 1
        if self.layout == "packed":
            return self._packed_call(self.L.smr_align_batch_packed, "smr_align_batch_packed", [self.h, _ptr(cat), _ptr(off), C.c_uint32(n)], n, with_stats)
        words = 0
        while True:
            slots, res, alns, pool, cap, counters = self._outputs(n, reuse_outputs, words)
            stats = np.zeros(n * slots, STATS_DTYPE) if with_stats else None
            self._check(self.L.smr_set_stats_buffer(self.h, _ptr(stats) if with_stats else C.c_void_p(0)), "smr_set_stats_buffer")
            used = C.c_uint64(0)
            rc = self.L.smr_align_batch(self.h, _ptr(cat), _ptr(off), C.c_uint32(n), _ptr(res), _ptr(alns), _ptr(pool),
                                        C.c_uint64(cap), C.byref(used), _ptr(counters), C.c_uint32(counters.size))
            need = int(self.L.smr_aln_slots_needed(self.h)) if rc == 5 and self.params.num_alignments == 0 else 0
            if need > slots:   # all-alignments mode: the library names the stride this batch needs; allocate and run again
                self.set_aln_slots(need)
                continue
            if rc == 5 and used.value > cap:   # the CIGAR pool: the library names the words this batch needs
                words = used.value
                continue
            break
        self._check(rc, "smr_align_batch")
        self.L.smr_set_stats_buffer(self.h, C.c_void_p(0))
        out = self._pack(res, alns, pool, used.value, counters, slots)
        if with_stats:
            out["stats"] = stats
        return out

    def upload(self, cat: np.ndarray, off: np.ndarray):
        cat = np.ascontiguousarray(cat, np.uint8)
        off = np.ascontiguousarray(off, np.uint64)
        self._n_resident = off.size - 1
        self._check(self.L.smr_upload_batch(self.h, _ptr(cat), _ptr(off), C.c_uint32(off.size - 1)), "smr_upload_batch")

    def upload_fastx(self, text: bytes) -> int:
        """smr_upload_fastx: the bytes of an uncompressed FASTA / FASTQ file; record split and 0-4 encoding run on the device.
        Returns the number of reads; continue with run_resident() / download()."""
        n = C.c_uint32(0)
        buf = np.frombuffer(text, dtype=np.uint8)
        self._check(self.L.smr_upload_fastx(self.h, _ptr(buf), C.c_uint64(buf.size), C.byref(n)), "smr_upload_fastx")
        self._n_resident = int(n.value)
        return self._n_resident

    def upload_fastx_gz(self, gz: bytes) -> int:
        """smr_upload_fastx_gz: the bytes of a .fastq.gz / .fasta.gz; gzip inflate, record split and 0-4 encoding run on the device."""
        n = C.c_uint32(0)
        buf = np.frombuffer(gz, dtype=np.uint8)
        self._check(self.L.smr_upload_fastx_gz(self.h, _ptr(buf), C.c_uint64(buf.size), C.byref(n)), "smr_upload_fastx_gz")
        self._n_resident = int(n.value)
        return self._n_resident

    def resident_text(self) -> bytes:
        """smr_resident_text: the (inflated) text behind the resident batch; header offsets of resident_layout() index it."""
        nb = C.c_uint64(0)
        self._check(self.L.smr_resident_text(self.h, C.c_void_p(0), C.c_uint64(0), C.byref(nb)), "smr_resident_text")
        out = np.zeros(int(nb.value), np.uint8)
        if out.size:
            self._check(self.L.smr_resident_text(self.h, _ptr(out), C.c_uint64(out.size), C.byref(nb)), "smr_resident_text")
        return out.tobytes()

    def debug_inflate(self, gz: bytes, chunk_bytes: int = 65536, cap: int = 0):
        """smr_debug_inflate: (inflated bytes, {spans, candidates, device_us, h2d_us})."""
        buf = np.frombuffer(gz, dtype=np.uint8)
        nb = C.c_uint64(0)
        info = (C.c_uint32 * 4)()
        self._check(self.L.smr_debug_inflate(self.h, _ptr(buf), C.c_uint64(buf.size), C.c_uint64(chunk_bytes), C.c_void_p(0), C.c_uint64(0), C.byref(nb), info),
                    "smr_debug_inflate")
        out = np.zeros(int(nb.value), np.uint8)
        if out.size:   # the inflated text is still in the context's buffer
            nb2 = C.c_uint64(0)
            self.L.smr_resident_text.restype = C.c_int
            self._check(self.L.smr_debug_inflate(self.h, _ptr(buf), C.c_uint64(buf.size), C.c_uint64(chunk_bytes), _ptr(out), C.c_uint64(out.size), C.byref(nb2), info),
                        "smr_debug_inflate")
        return out.tobytes(), {"spans": info[0], "candidates": info[1], "device_us": info[2], "h2d_us": info[3]}

    # -- read stream (smr_stream_*): files of any size, pushed from disk piece by piece --
    STREAM_GZ, STREAM_COUNT_ONLY, STREAM_NEXT_FILE, STREAM_MATES = 1, 2, 4, 8

    def _push_file(self, path: str, piece_bytes: int, mate: int = 0):
        """Pushes the file at `path` into the open stream, piece by piece (mate 1 / 2 of a mate stream: smr_stream_push_mate);
        yields after every push."""
        with open(path, "rb") as f:
            piece = f.read(piece_bytes)
            while True:
                nxt = f.read(piece_bytes) if piece else b""
                buf = np.frombuffer(piece, dtype=np.uint8)
                args = (_ptr(buf) if buf.size else C.c_void_p(0), C.c_uint64(buf.size), C.c_int(0 if nxt else 1))
                if mate:
                    self._check(self.L.smr_stream_push_mate(self.h, C.c_uint32(mate), *args), "smr_stream_push_mate")
                else:
                    self._check(self.L.smr_stream_push(self.h, *args), "smr_stream_push")
                yield
                if not nxt:
                    return
                piece = nxt

    @staticmethod
    def _is_gz(path: str) -> bool:
        with open(path, "rb") as f:
            return f.read(2) == b"\x1f\x8b"

    def read_counts(self, path_or_paths, piece_bytes: int = 256 << 20) -> dict:
        """The reference's first pass over the reads files (Readfeed::count_reads_parallel, readfeed.cpp:1486-1663) on the device:
        {"reads", "length", "min_len", "max_len"} = num_reads_tot, length_all, min_read_len, max_read_len -- the figures
        hostio.minimal_score and hostio.evalue_params take.  gzip files are recognised by their magic bytes; several files (mates)
        are counted one after another as the reference counts the -reads files of one run (SMR_STREAM_NEXT_FILE)."""
        paths = [path_or_paths] if isinstance(path_or_paths, (str, os.PathLike)) else list(path_or_paths)
        for k, p in enumerate(paths):
            flags = self.STREAM_COUNT_ONLY | (self.STREAM_GZ if self._is_gz(p) else 0) | (self.STREAM_NEXT_FILE if k else 0)
            self._check(self.L.smr_stream_begin(self.h, C.c_uint32(flags), C.c_uint64(0)), "smr_stream_begin")
            for _ in self._push_file(p, piece_bytes):
                pass
        return self.stream_counts()

    def stream_fastx(self, path: str, batch_bytes: int = 256 << 20, piece_bytes: int = 256 << 20):
        """Streams a FASTA / FASTQ file (plain or gzip, by its magic bytes) through the device in record-aligned batches of at
        most batch_bytes of text (one longer record makes a batch alone).  Yields the read count of each batch once it is
        resident: run run_resident() / download() / ReportWriter.write(out) inside the loop.  The file is read piece_bytes at a
        time and is never held whole in host memory."""
        flags = self.STREAM_GZ if self._is_gz(path) else 0
        self._check(self.L.smr_stream_begin(self.h, C.c_uint32(flags), C.c_uint64(batch_bytes)), "smr_stream_begin")
        for _ in self._push_file(path, piece_bytes):
            yield from self._drain()
        yield from self._drain()

    def _drain(self):
        """the batches the open stream can make now: yields the read count of each once it is resident"""
        n, done = C.c_uint32(0), C.c_int(0)
        while True:
            self._check(self.L.smr_stream_next(self.h, C.byref(n), C.byref(done)), "smr_stream_next")
            if n.value == 0:
                return
            self._n_resident = int(n.value)
            yield int(n.value)

    def stream_mates(self, path1: str, path2: str, batch_bytes: int = 256 << 20, piece_bytes: int = 256 << 20):
        """Streams two mate files (the reference's -reads R1 -reads R2; plain or gzip by their magic bytes, both alike) through the
        device as pairs: every batch is k whole pairs interleaved (records 2k and 2k+1 are record k of each file) in at most
        batch_bytes of text, or one longer pair alone.  Yields the read count (2k) of each batch once it is resident, as
        stream_fastx; format_reports / ReportWriter.write(out) route it as mates.  Each round pushes one piece of each file that
        has not ended, then takes the batches that are ready.  Files that differ in record count or format raise SmrError."""
        gz = [self._is_gz(p) for p in (path1, path2)]
        if gz[0] != gz[1]:
            raise SmrError(f"stream_mates: {path1 if gz[0] else path2} is gzip and {path2 if gz[0] else path1} is not")
        flags = self.STREAM_MATES | (self.STREAM_GZ if gz[0] else 0)
        self._check(self.L.smr_stream_begin(self.h, C.c_uint32(flags), C.c_uint64(batch_bytes)), "smr_stream_begin")
        feeds = [self._push_file(path1, piece_bytes, 1), self._push_file(path2, piece_bytes, 2)]
        while feeds:
            feeds = [f for f in feeds if next(f, StopIteration) is not StopIteration]
            yield from self._drain()

    def stream_counts(self) -> dict:
        """smr_stream_counts of the open stream: the count_reads_parallel figures of what was pushed so far."""
        out = (C.c_uint64 * 4)()
        self._check(self.L.smr_stream_counts(self.h, out), "smr_stream_counts")
        return dict(zip(("reads", "length", "min_len", "max_len"), (int(v) for v in out)))

    def resident_layout(self, with_headers: bool = True, with_seq: bool = True):
        """smr_resident_layout: (header offsets in the uploaded text, read offsets, concatenated 0-4 codes) of the resident batch."""
        n = self._n_resident
        hdr = np.zeros(n, np.uint64) if with_headers else None
        off = np.zeros(n + 1, np.uint64)
        self._check(self.L.smr_resident_layout(self.h, _ptr(hdr) if with_headers and n else C.c_void_p(0), _ptr(off), C.c_void_p(0), C.c_uint64(0)),
                    "smr_resident_layout")
        seq = None
        if with_seq:
            seq = np.zeros(int(off[n]), np.uint8)
            if seq.size:
                self._check(self.L.smr_resident_layout(self.h, C.c_void_p(0), C.c_void_p(0), _ptr(seq), C.c_uint64(seq.size)), "smr_resident_layout")
        return hdr, off, seq

    def run_resident(self, with_stats: bool = False):
        """with_stats: download() also returns calc_miss_gap_match per stored alignment (out["stats"])"""
        n = self._n_resident
        if self.layout == "packed":   # the device computes the stats in this layout; download() copies them
            self._stats_packed = with_stats
            self._check(self.L.smr_run_resident(self.h), "smr_run_resident")
            return
        self._stats = np.zeros(n * int(self.L.smr_aln_slots(self.h)), STATS_DTYPE) if with_stats else None
        self._check(self.L.smr_set_stats_buffer(self.h, _ptr(self._stats) if with_stats else C.c_void_p(0)), "smr_set_stats_buffer")
        self._check(self.L.smr_run_resident(self.h), "smr_run_resident")

    def download(self):
        """smr_download_results: the results of the last run_resident(); may be called again without running again"""
        n = self._n_resident
        if self.layout == "packed":
            return self._packed_call(self.L.smr_download_results_packed, "smr_download_results_packed", [self.h], n, self._stats_packed)
        stats = getattr(self, "_stats", None)   # sized at the stride in effect, which the library writes them at
        stats = np.zeros(n * int(self.L.smr_aln_slots(self.h)), STATS_DTYPE) if stats is not None else None
        self._check(self.L.smr_set_stats_buffer(self.h, _ptr(stats) if stats is not None else C.c_void_p(0)), "smr_set_stats_buffer")
        words = 0
        while True:
            slots, res, alns, pool, cap, counters = self._outputs(n, cigar_words=words)
            used = C.c_uint64(0)
            rc = self.L.smr_download_results(self.h, _ptr(res), _ptr(alns), _ptr(pool), C.c_uint64(cap), C.byref(used),
                                             _ptr(counters), C.c_uint32(counters.size))
            if rc == 5 and used.value > cap:   # the CIGAR pool: the library names the words needed; download again into a larger one
                words = used.value
                continue
            break
        self.L.smr_set_stats_buffer(self.h, C.c_void_p(0))
        self._check(rc, "smr_download_results")
        out = self._pack(res, alns, pool, used.value, counters, slots)
        if stats is not None:
            out["stats"] = stats
        return out

    # ---- results placed on the device (smr_place_results; the report calls with out=None read them) ----
    def set_place_stats(self, on: bool):
        """smr_set_place_stats: later runs compute the smr_aln_stats a placement keeps (SAM, tabular BLAST, aligned_denovo, the OTU
        map and the denovo statistics read them); default off."""
        self._check(self.L.smr_set_place_stats(self.h, C.c_int(1 if on else 0)), "smr_set_place_stats")

    def place(self) -> dict:
        """smr_place_results: the results of the last run_resident() placed on the device in the strided layout (the packed layout
        is place_packed()), its scratch-overflow
        retries included; format_reports / format_blast_pairwise / otu_add / denovo_stats / ReportWriter.write with out=None read
        them there.  In the all-alignments mode (num_alignments 0) a read that stores more alignments than the stride makes the
        stride grow to what the library names and the batch run again, as align() does.  Returns {"nreads", "slots", "n_alns",
        "cigar_words", "counters" (by name, as download()), "matched" (reads_matched_per_db), "place_ms" (device time of the
        placement passes)}."""
        while True:
            rc, info = self._place("smr_place_results")
            slots = int(self.L.smr_aln_slots(self.h))
            need = int(self.L.smr_aln_slots_needed(self.h)) if rc == 5 and self.params.num_alignments == 0 else 0
            if need > slots:   # run again as run_resident() does, with a host stats buffer at the new stride if it had one
                self.set_aln_slots(need)
                self.run_resident(with_stats=getattr(self, "_stats", None) is not None)
                continue
            break
        self._check(rc, "smr_place_results")
        info["slots"] = slots
        self.placed_info = info
        return info

    def place_packed(self) -> dict:
        """smr_place_results_packed: the results of the last run_resident() in the packed layout placed on the device, as download()
        returns them there: the reads that stored more alignments than the first run's stride run again at their own count, and
        the reads that overflowed their scratch at a larger scale, then every read placed in read order.  format_reports /
        format_blast_pairwise / format_placed_into / otu_add / denovo_stats / ReportWriter.write with out=None read them there, and
        a later download() copies them.  Returns the dict place() returns, with "slots" = 0 and "n_alns" = the sum of n_align."""
        rc, info = self._place("smr_place_results_packed")
        self._check(rc, "smr_place_results_packed")
        self.placed_info = info
        return info

    def _place(self, fn: str):
        """smr_place_results[_packed] (`fn`): its status and the dict place() returns, with "slots" = 0"""
        f = getattr(self.L, fn)
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        self.L.smr_last_place_timing.argtypes = [C.c_void_p, C.c_void_p]
        counters = np.zeros(CNT_FIXED + max(1, self.n_index_files), np.uint64)
        n_alns, words, ms = C.c_uint64(0), C.c_uint64(0), C.c_double(0)
        rc = f(self.h, _ptr(counters), counters.size, C.cast(C.byref(n_alns), C.c_void_p), C.cast(C.byref(words), C.c_void_p))
        self.L.smr_last_place_timing(self.h, C.cast(C.byref(ms), C.c_void_p))
        return rc, dict(nreads=self._n_resident, slots=0, n_alns=int(n_alns.value), cigar_words=int(words.value),
                        counters={k: int(counters[i]) for i, k in enumerate(CNT_NAMES)}, matched=counters[CNT_FIXED:].copy(), place_ms=ms.value)

    def download_placed(self, with_stats: bool = False) -> dict:
        """smr_download_placed: the placed arrays on the host, in the form download() returns ("res", "alns", "cigar", "slots", and
        "stats" with with_stats; packed, "alns" / "stats" of sum n_align entries, "aln_off" and slots = 0); the counters are those
        place() / place_packed() returned."""
        n = self._n_resident
        n_alns, words = C.c_uint64(0), C.c_uint64(0)
        fn = self.L.smr_place_results_packed if self.layout == "packed" else self.L.smr_place_results
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        self._check(fn(self.h, None, 0, C.cast(C.byref(n_alns), C.c_void_p), C.cast(C.byref(words), C.c_void_p)),
                    "smr_place_results_packed" if self.layout == "packed" else "smr_place_results")
        slots = 0 if self.layout == "packed" else int(self.L.smr_aln_slots(self.h))
        res, alns = np.zeros(n, RESULT_DTYPE), np.zeros(int(n_alns.value), ALN_DTYPE)
        stats = np.zeros(int(n_alns.value), STATS_DTYPE) if with_stats else None
        pool = np.zeros(max(1, words.value), np.uint32)
        self.L.smr_download_placed.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
        self._check(self.L.smr_download_placed(self.h, _ptr(res), _ptr(alns), _ptr(stats) if with_stats else None, _ptr(pool), pool.size),
                    "smr_download_placed")
        out = dict(res=res, alns=alns, cigar=pool[:words.value], slots=slots)
        if with_stats:
            out["stats"] = stats
        if self.layout == "packed":
            out["aln_off"] = np.zeros(n + 1, np.uint64)
            np.cumsum(res["n_align"], out=out["aln_off"][1:])
        return out

    def format_placed_into(self, opts: ReportOpts, buf: np.ndarray, gzip: bool = False, pairwise: bool = False, bam: bool = False):
        """smr_format_reports_placed[_gz] (pairwise: smr_format_blast_pairwise_placed[_gz]; bam: smr_format_bam_placed, one BGZF
        stream of BAM records per report_groups() entry, opts = report_opts(sam=True, ...)) into `buf` (a uint8 array, grown when the
        streams do not fit): returns (buf, stream offsets).  The streams stay in buf, for a caller that writes them out as they are."""
        if opts.sam or opts.blast:
            self._upload_report_refs()
        G = len(self.report_groups())
        so = np.zeros(G + 1 if pairwise or bam else 2 * G + 3 * num_out_of(opts) + 1, np.uint64)
        name = "smr_format_bam_placed" if bam else \
            ("smr_format_blast_pairwise_placed" if pairwise else "smr_format_reports_placed") + ("_gz" if gzip else "")
        fn = getattr(self.L, name)
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        rc = fn(self.h, C.cast(C.byref(opts), C.c_void_p), _ptr(buf), buf.size, _ptr(so))
        if rc == 5 and int(so[-1]) > buf.size:   # SMR_ERR_CAPACITY: so names the size; grow and run again
            buf = np.empty(int(so[-1]) + (int(so[-1]) >> 3), np.uint8)
            rc = fn(self.h, C.cast(C.byref(opts), C.c_void_p), _ptr(buf), buf.size, _ptr(so))
        self._check(rc, name)
        return buf, so

    # ---- report writer (smr_format_reports) ----
    def report_groups(self) -> list:
        """the loaded (index, part)s in the order of the SAM / BLAST streams"""
        return sorted(set(self.parts))

    def _upload_report_refs(self):
        for (i, p) in self.report_groups():
            if (i, p) in self._report_refs:
                continue
            refs = self.refs_by_index.get(i)
            if refs is None:
                raise SmrError(f"no reference ids for index {i}: pass refs to load_index_part / build_index_device")
            r = refs[p] if isinstance(refs, (list, tuple)) else refs
            names = [x.encode() for x in r.ids]
            off = np.zeros(len(names) + 1, np.uint64)
            np.cumsum([len(x) for x in names], out=off[1:])
            cat = np.frombuffer(b"".join(names) or b"\0", np.uint8)
            self._check(self.L.smr_set_report_refs(self.h, C.c_uint32(i), C.c_uint32(p), _ptr(cat), _ptr(off), C.c_uint32(len(names))),
                        "smr_set_report_refs")
            self._report_refs.add((i, p))

    def set_report_scoring(self, index_num: int, lam: float, K: float, full_ref: int, full_read: int):
        """smr_set_report_scoring: Gumbel lambda / K and the corrected sizes (hostio.evalue_params) the BLAST E-values of index_num use"""
        self._check(self.L.smr_set_report_scoring(self.h, C.c_uint32(index_num), C.c_double(lam), C.c_double(K), C.c_uint64(int(full_ref)),
                                                  C.c_uint64(int(full_read))), "smr_set_report_scoring")

    def gzip(self, data: bytes) -> bytes:
        """smr_gzip: `data` compressed on the device into one gzip member (an empty member for empty data)"""
        buf = np.frombuffer(data, np.uint8)
        cap = buf.size + (buf.size >> 6) + 1024   # the stored fallback bounds a member: 10 bytes per 32 KB chunk, 18 around
        o = np.zeros(cap, np.uint8)
        nb = C.c_uint64(0)
        self.L.smr_gzip.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
        self._check(self.L.smr_gzip(self.h, _ptr(buf) if buf.size else None, buf.size, _ptr(o), o.size, C.cast(C.byref(nb), C.c_void_p)), "smr_gzip")
        return o[:nb.value].tobytes()

    def bam_header(self, text: bytes) -> bytes:
        """smr_bam_header: the BAM header of the loaded indexes, with `text` (the SAM header) as its text, as BGZF blocks"""
        self._upload_report_refs()
        buf = np.frombuffer(text, np.uint8)
        nb = C.c_uint64(0)
        self.L.smr_bam_header.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
        o = np.zeros(buf.size + (buf.size >> 6) + 4096, np.uint8)
        rc = self.L.smr_bam_header(self.h, _ptr(buf) if buf.size else None, buf.size, _ptr(o), o.size, C.cast(C.byref(nb), C.c_void_p))
        if rc == 5 and nb.value > o.size:   # SMR_ERR_CAPACITY: nb names the size (the reference names make it grow)
            o = np.zeros(nb.value, np.uint8)
            rc = self.L.smr_bam_header(self.h, _ptr(buf) if buf.size else None, buf.size, _ptr(o), o.size, C.cast(C.byref(nb), C.c_void_p))
        self._check(rc, "smr_bam_header")
        return o[:nb.value].tobytes()

    # ---- coordinate-sorted BAM (smr_bam_sort_*) ----
    def bam_sort_begin(self):
        """smr_bam_sort_begin: opens the accumulator of a coordinate-sorted aligned.bam (again: the open one is discarded)"""
        self._upload_report_refs()
        self._check(self.L.smr_bam_sort_begin(self.h), "smr_bam_sort_begin")

    def bam_sort_add(self, opts: ReportOpts, buf: np.ndarray):
        """smr_bam_sort_add_placed: the placed batch's BAM records (opts = report_opts(sam=True, ...)) sorted into one run,
        uncompressed, into `buf` (a uint8 array, grown when the run does not fit) -> (buf, nbytes).  The caller keeps the runs (for
        bam_sort_finish); the accumulator keeps their keys and sizes."""
        nb = C.c_uint64(0)
        fn = self.L.smr_bam_sort_add_placed
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        rc = fn(self.h, C.cast(C.byref(opts), C.c_void_p), _ptr(buf), buf.size, C.cast(C.byref(nb), C.c_void_p))
        if rc == 5 and nb.value > buf.size:   # SMR_ERR_CAPACITY: nb names the size; grow and run again
            buf = np.empty(nb.value + (nb.value >> 3), np.uint8)
            rc = fn(self.h, C.cast(C.byref(opts), C.c_void_p), _ptr(buf), buf.size, C.cast(C.byref(nb), C.c_void_p))
        self._check(rc, "smr_bam_sort_add_placed")
        return buf, nb.value

    def bam_sort_finish(self, runs, run_starts, out, header_bytes: int, window_bytes: int = BAM_SORT_WINDOW) -> bytes:
        """The end of a sorted aligned.bam: smr_bam_sort_plan, then every window (smr_bam_sort_window) with its ranges read from
        `runs` (a binary file holding the runs of bam_sort_add, run r from byte run_starts[r]) and its BGZF blocks written to `out`
        (a binary file, after the header_bytes of the header blocks), then smr_bam_sort_index.  Returns the BAI bytes; the caller
        writes the EOF block.  self.bam_sort_seconds: plan, read (the runs file), upload, device (gather, compress, index pass),
        d2h, write, index, and windows."""
        import time
        sec = dict.fromkeys(("plan", "read", "upload", "device", "d2h", "write", "index"), 0.0)
        t0 = time.perf_counter()
        R = len(run_starts)
        nw, ranges = C.c_uint64(0), np.zeros(0, np.uint64)
        plan = self.L.smr_bam_sort_plan
        plan.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
        rc = plan(self.h, window_bytes, header_bytes, None, 0, C.cast(C.byref(nw), C.c_void_p))
        if rc == 5:   # SMR_ERR_CAPACITY: nw names the windows
            ranges = np.zeros(nw.value * R * 2, np.uint64)
            rc = plan(self.h, window_bytes, header_bytes, _ptr(ranges), ranges.size, C.cast(C.byref(nw), C.c_void_p))
        self._check(rc, "smr_bam_sort_plan")
        n_win = nw.value
        ranges = ranges.reshape(n_win, R, 2) if n_win else np.zeros((0, R, 2), np.uint64)
        sec["plan"] = time.perf_counter() - t0
        win = self.L.smr_bam_sort_window
        win.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
        staged, ob = np.empty(0, np.uint8), np.empty(0, np.uint8)
        for w in range(n_win):
            t0 = time.perf_counter()
            n = int((ranges[w, :, 1] - ranges[w, :, 0]).sum())
            if staged.size < n:
                staged = np.empty(n, np.uint8)
            mv, at = memoryview(staged), 0
            for r in range(R):
                lo, hi = int(ranges[w, r, 0]), int(ranges[w, r, 1])
                if hi > lo:
                    runs.seek(int(run_starts[r]) + lo)
                    if runs.readinto(mv[at:at + hi - lo]) != hi - lo:
                        raise SmrError(f"bam_sort_finish: the runs file ends inside run {r}")
                    at += hi - lo
            t1 = time.perf_counter()
            cap = -(-n // BGZF_BLOCK) * BAM_MAX_MEMBER + 64   # the stored fallback bounds every member
            if ob.size < cap:
                ob = np.empty(cap, np.uint8)
            nb = C.c_uint64(0)
            self._check(win(self.h, w, _ptr(staged), n, _ptr(ob), ob.size, C.cast(C.byref(nb), C.c_void_p)), "smr_bam_sort_window")
            tm = self.report_timings()
            t2 = time.perf_counter()
            out.write(memoryview(ob)[:nb.value])
            sec["read"] += t1 - t0
            sec["upload"] += tm["h2d_ms"] / 1e3
            sec["device"] += tm["device_ms"] / 1e3
            sec["d2h"] += tm["d2h_ms"] / 1e3
            sec["write"] += time.perf_counter() - t2
        t0 = time.perf_counter()
        idx = self.L.smr_bam_sort_index
        idx.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        nb, bai = C.c_uint64(0), np.zeros(0, np.uint8)
        rc = idx(self.h, None, 0, C.cast(C.byref(nb), C.c_void_p))
        if rc == 5:   # SMR_ERR_CAPACITY: nb names the size
            bai = np.zeros(nb.value, np.uint8)
            rc = idx(self.h, _ptr(bai), bai.size, C.cast(C.byref(nb), C.c_void_p))
        self._check(rc, "smr_bam_sort_index")
        sec["index"] = time.perf_counter() - t0
        sec["windows"] = n_win
        self.bam_sort_seconds = sec
        return bai[:nb.value].tobytes()

    def format_reports(self, out: dict, text: bytes | None = None, opts: ReportOpts | None = None, gzip: bool = False, **kw) -> dict:
        """smr_format_reports: the report streams of one batch as bytes.  out = what align(with_stats=True) / download(with_stats=True)
        returned for it; text = the batch's FASTA / FASTQ bytes (None: the resident text of upload_fastx[_gz]); opts = report_opts(...)
        or its keyword arguments.  Returns {"sam": [bytes per group], "blast": [...], "aligned": bytes, "other": bytes, "denovo": bytes,
        "groups": report_groups()}; with out2 or sout, "aligned" / "other" / "denovo" are tuples of the num_out files (2, or 4 with
        both) in the reference's order (_fwd, _rev | _paired, _singleton | _paired_fwd, _paired_rev, _singleton_fwd, _singleton_rev).
        gzip: smr_format_reports_gz, every non-empty stream as one gzip member (empty ones stay b"").
        out=None: the results place() or place_packed() placed on the device and the resident text (smr_format_reports_placed[_gz]);
        text must be None."""
        o = opts if opts is not None else report_opts(**kw)
        if o.sam or o.blast:
            self._upload_report_refs()
        groups = self.report_groups()
        G = len(groups)
        num_out = num_out_of(o)
        if out is None:
            if text is not None:
                raise ValueError("format_reports: the placed results go with the resident text (text=None)")
            buf, so = self.format_placed_into(o, self._report_buffer(), gzip)
            self._report_buf = buf
            return self._report_streams(buf, so, G, num_out, groups)
        res, alns = out["res"], out["alns"]
        cig = np.ascontiguousarray(out["cigar"], np.uint32)
        st = out.get("stats")
        txt = np.frombuffer(text, np.uint8) if text is not None else None
        so = np.zeros(2 * G + 3 * num_out + 1, np.uint64)
        fn = self.L.smr_format_reports_gz if gzip else self.L.smr_format_reports
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                       C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
        args = [self.h, C.cast(C.byref(o), C.c_void_p), _ptr(txt) if txt is not None and txt.size else None, txt.size if txt is not None else 0,
                _ptr(res), _ptr(alns), _ptr(cig) if cig.size else None, cig.size, _ptr(st) if st is not None else None, res.shape[0]]
        buf = getattr(self, "_report_buf", None)
        if buf is None:
            buf = np.zeros(1 << 20, np.uint8)
        rc = fn(*args, _ptr(buf), buf.size, _ptr(so))
        if rc == 5 and int(so[-1]) > buf.size:   # SMR_ERR_CAPACITY: so names the size; grow and run again
            buf = np.zeros(int(so[-1]) + (int(so[-1]) >> 3), np.uint8)
            rc = fn(*args, _ptr(buf), buf.size, _ptr(so))
        self._check(rc, "smr_format_reports_gz" if gzip else "smr_format_reports")
        self._report_buf = buf
        return self._report_streams(buf, so, G, num_out, groups)

    def _report_buffer(self) -> np.ndarray:
        buf = getattr(self, "_report_buf", None)
        return buf if buf is not None else np.zeros(1 << 20, np.uint8)

    @staticmethod
    def _report_streams(buf, so, G, num_out, groups) -> dict:
        b = [bytes(buf[int(so[k]):int(so[k + 1])]) for k in range(so.size - 1)]
        fx = [b[2 * G + j * num_out:2 * G + (j + 1) * num_out] for j in range(3)]
        fx = [f[0] for f in fx] if num_out == 1 else [tuple(f) for f in fx]
        return dict(sam=b[:G], blast=b[G:2 * G], aligned=fx[0], other=fx[1], denovo=fx[2], groups=groups)

    def format_blast_pairwise(self, out: dict, text: bytes | None = None, opts: ReportOpts | None = None, gzip: bool = False, **kw) -> list:
        """smr_format_blast_pairwise: the pairwise BLAST rows (-blast 0) of one batch, as a list of bytes, one per report_groups() entry.
        out / text as for format_reports; opts = report_opts(blast="0", ...) or its keyword arguments (blast defaults to "0"; only
        paired_in / paired_out / mates matter besides).  gzip: smr_format_blast_pairwise_gz, every non-empty stream as one gzip member.
        out=None: the placed results and the resident text (smr_format_blast_pairwise_placed[_gz]), as format_reports."""
        if opts is None:
            kw.setdefault("blast", "0")
            opts = report_opts(**kw)
        self._upload_report_refs()
        G = len(self.report_groups())
        if out is None:
            if text is not None:
                raise ValueError("format_blast_pairwise: the placed results go with the resident text (text=None)")
            buf, so = self.format_placed_into(opts, self._report_buffer(), gzip, pairwise=True)
            self._report_buf = buf
            return [bytes(buf[int(so[k]):int(so[k + 1])]) for k in range(G)]
        res, alns = out["res"], out["alns"]
        cig = np.ascontiguousarray(out["cigar"], np.uint32)
        st = out.get("stats")
        txt = np.frombuffer(text, np.uint8) if text is not None else None
        so = np.zeros(G + 1, np.uint64)
        fn = self.L.smr_format_blast_pairwise_gz if gzip else self.L.smr_format_blast_pairwise
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                       C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
        args = [self.h, C.cast(C.byref(opts), C.c_void_p), _ptr(txt) if txt is not None and txt.size else None, txt.size if txt is not None else 0,
                _ptr(res), _ptr(alns), _ptr(cig) if cig.size else None, cig.size, _ptr(st) if st is not None else None, res.shape[0]]
        buf = getattr(self, "_report_buf", None)
        if buf is None:
            buf = np.zeros(1 << 20, np.uint8)
        rc = fn(*args, _ptr(buf), buf.size, _ptr(so))
        if rc == 5 and int(so[-1]) > buf.size:   # SMR_ERR_CAPACITY: so names the size; grow and run again
            buf = np.zeros(int(so[-1]) + (int(so[-1]) >> 3), np.uint8)
            rc = fn(*args, _ptr(buf), buf.size, _ptr(so))
        self._check(rc, "smr_format_blast_pairwise_gz" if gzip else "smr_format_blast_pairwise")
        self._report_buf = buf
        return [bytes(buf[int(so[k]):int(so[k + 1])]) for k in range(G)]

    # ---- OTU map (smr_otu_begin / smr_otu_add / smr_otu_finish) ----
    def otu_begin(self, min_id: float = 0.97, min_cov: float = 0.97, paired_in: bool = False, paired_out: bool = False, feed=None):
        """smr_otu_begin: open (or reset) the OTU map of this context; -id / -coverage as the reference's -otu_map defaults them.
        feed: None (single-end; paired_in / paired_out are refused), "one_file" (one interleaved paired file: every record) or
        "two_files" (two mate files, as stream_mates batches them: records 2k, the first file's, alone)"""
        self._upload_report_refs()
        o = OtuOpts(float(min_id), float(min_cov), int(bool(paired_in)), int(bool(paired_out)), OTU_FEEDS[feed] if feed in OTU_FEEDS else int(feed))
        self._check(self.L.smr_otu_begin(self.h, C.byref(o)), "smr_otu_begin")

    def otu_add(self, out: dict, text: bytes | None = None) -> int:
        """smr_otu_add: one batch (out and text as for format_reports; out needs "stats"); returns the entries it added.
        out=None: the placed results and the resident text (smr_otu_add_placed)."""
        n = C.c_uint64(0)
        if out is None:
            if text is not None:
                raise ValueError("otu_add: the placed results go with the resident text (text=None)")
            self.L.smr_otu_add_placed.argtypes = [C.c_void_p, C.c_void_p]
            self._check(self.L.smr_otu_add_placed(self.h, C.cast(C.byref(n), C.c_void_p)), "smr_otu_add_placed")
            return int(n.value)
        res, alns, st = out["res"], out["alns"], out.get("stats")
        txt = np.frombuffer(text, np.uint8) if text is not None else None
        self.L.smr_otu_add.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        rc = self.L.smr_otu_add(self.h, _ptr(txt) if txt is not None and txt.size else None, txt.size if txt is not None else 0, _ptr(res), _ptr(alns),
                                _ptr(st) if st is not None else None, res.shape[0], C.cast(C.byref(n), C.c_void_p))
        self._check(rc, "smr_otu_add")
        return int(n.value)

    def otu_finish(self) -> dict:
        """smr_otu_finish: {"text": the bytes of otu_map.txt, "total_otu": lines, "n_yid_ycov": entries}"""
        counts = np.zeros(3, np.uint64)
        buf = getattr(self, "_otu_buf", None)
        if buf is None:
            buf = np.zeros(1 << 16, np.uint8)
        rc = self.L.smr_otu_finish(self.h, _ptr(buf), C.c_uint64(buf.size), _ptr(counts))
        if rc == 5 and int(counts[0]) > buf.size:   # SMR_ERR_CAPACITY: counts[0] names the size; grow and run again
            buf = np.zeros(int(counts[0]) + (int(counts[0]) >> 3), np.uint8)
            rc = self.L.smr_otu_finish(self.h, _ptr(buf), C.c_uint64(buf.size), _ptr(counts))
        self._check(rc, "smr_otu_finish")
        self._otu_buf = buf
        return dict(text=bytes(buf[:int(counts[0])]), total_otu=int(counts[1]), n_yid_ycov=int(counts[2]))

    def denovo_stats(self, out: dict, text: bytes | None = None, min_id: float = 0.97, min_cov: float = 0.97, paired: bool = False,
                     per_read: bool = True):
        """smr_denovo_stats: the reference's denovo_stats pass over one batch (out and text as for format_reports; out needs "stats").
        Returns (per_read, totals): per_read an (nreads, 4) uint32 array of {c_yid_ycov, n_yid_ncov, n_nid_ycov, n_denovo} per read
        (pack_kvdb_blobs' denovo), totals {"n_yid_ycov", "n_yid_ncov", "n_nid_ycov", "num_denovo"} of this batch.  paired: records
        2k and 2k+1 are mates (implied for the resident batch of stream_mates).  out=None: the placed results and the resident text
        (smr_denovo_stats_placed).  per_read=False: the totals alone (per_read is returned as None)."""
        tot = np.zeros(4, np.uint64)
        o = DenovoOpts(float(min_id), float(min_cov), int(bool(paired)))
        if out is None:
            if text is not None:
                raise ValueError("denovo_stats: the placed results go with the resident text (text=None)")
            pr = np.zeros((self._n_resident, 4), np.uint32) if per_read else None
            self.L.smr_denovo_stats_placed.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
            self._check(self.L.smr_denovo_stats_placed(self.h, C.cast(C.byref(o), C.c_void_p), _ptr(pr) if pr is not None and pr.size else None,
                                                       _ptr(tot)), "smr_denovo_stats_placed")
            return pr, dict(zip(DENOVO_TOTALS, (int(v) for v in tot)))
        res, alns, st = out["res"], out["alns"], out.get("stats")
        txt = np.frombuffer(text, np.uint8) if text is not None else None
        n = res.shape[0]
        pr = np.zeros((n, 4), np.uint32) if per_read else None
        self.L.smr_denovo_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                            C.c_void_p, C.c_void_p]
        rc = self.L.smr_denovo_stats(self.h, C.cast(C.byref(o), C.c_void_p), _ptr(txt) if txt is not None and txt.size else None,
                                     txt.size if txt is not None else 0, _ptr(res), _ptr(alns), _ptr(st) if st is not None else None, n,
                                     _ptr(pr) if pr is not None and n else None, _ptr(tot))
        self._check(rc, "smr_denovo_stats")
        return pr, dict(zip(DENOVO_TOTALS, (int(v) for v in tot)))

    def otu_timings(self):
        out = np.zeros(3, np.float64)
        self._check(self.L.smr_last_otu_timings(self.h, _ptr(out)), "smr_last_otu_timings")
        return dict(add_h2d_ms=out[0], add_device_ms=out[1], finish_ms=out[2])

    def report_timings(self):
        out = np.zeros(3, np.float64)
        self._check(self.L.smr_last_report_timings(self.h, _ptr(out)), "smr_last_report_timings")
        return dict(h2d_ms=out[0], device_ms=out[1], d2h_ms=out[2])

    def timings(self):
        out = np.zeros(8, np.float64)
        self.L.smr_last_timings(self.h, _ptr(out))
        return dict(total_ms=out[0], seed_ms=out[1], lis_ms=out[2], final_ms=out[3], h2d_ms=out[4], d2h_ms=out[5],
                    launches=int(out[6]), decode_ms=out[7])

    def dpx_peak(self) -> float:
        """measured dependent-free DPX thread-ops/s (1e9/s) on this device"""
        v = C.c_double(0)
        self._check(self.L.smr_debug_dpx_peak(self.h, C.byref(v)), "smr_debug_dpx_peak")
        return v.value

    # ---- unit-test entry points ----
    def debug_seed_windows(self, part_slot, cat03, off, win_read, win_pos, cap=64, fallback_path=False):
        cat03 = np.ascontiguousarray(cat03, np.uint8)
        off = np.ascontiguousarray(off, np.uint64)
        win_read = np.ascontiguousarray(win_read, np.uint32)
        win_pos = np.ascontiguousarray(win_pos, np.uint32)
        nwin = win_read.size
        ids = np.zeros(nwin * cap, np.uint32)
        counts = np.zeros(nwin, np.uint32)
        zero = np.zeros(nwin, np.uint8)
        rc = self.L.smr_debug_seed_windows(self.h, C.c_uint32(part_slot), _ptr(cat03), _ptr(off), C.c_uint32(off.size - 1),
                                           _ptr(win_read), _ptr(win_pos), C.c_uint32(nwin), _ptr(ids),
                                           C.c_uint32(cap | (0x80000000 if fallback_path else 0)), _ptr(counts), _ptr(zero))
        self._check(rc, "smr_debug_seed_windows")
        return ids.reshape(nwin, cap), counts, zero

    def debug_ssw(self, q_cat, q_off, t_cat, t_off, filters=0, cigar_cap=256):
        q_cat = np.ascontiguousarray(q_cat, np.uint8)
        t_cat = np.ascontiguousarray(t_cat, np.uint8)
        q_off = np.ascontiguousarray(q_off, np.uint64)
        t_off = np.ascontiguousarray(t_off, np.uint64)
        n = q_off.size - 1
        out = np.zeros(n * 6, np.int32)
        cig = np.zeros(n * cigar_cap, np.uint32)
        rc = self.L.smr_debug_ssw(self.h, _ptr(q_cat), _ptr(q_off), _ptr(t_cat), _ptr(t_off), C.c_uint32(n),
                                  C.c_uint32(filters), _ptr(out), _ptr(cig), C.c_uint32(cigar_cap))
        self._check(rc, "smr_debug_ssw")
        return out.reshape(n, 6), cig.reshape(n, cigar_cap)


class ReportWriter:
    """The reference's report files from batches of one read file: aligned.sam (header + rows), aligned.blast, aligned.<ext>,
    other.<ext>, aligned_denovo.<ext> under out_dir (<ext> = fq for FASTQ input, fa for FASTA, report_fx_base.cpp:94).  Every stream of
    every batch is appended to a part file of its own; close() concatenates them in the reference's order (all SAM rows of (index, part)
    group 0, then group 1, ...), so that feeding a file in several batches writes what one batch writes.
    sam_header: the text before the SAM rows (hostio.sam_header); opts: report_opts(...) keyword arguments.
    otu_map: (min_id, min_cov) = the reference's -otu_map -id -coverage: close() also writes otu_map.txt (none when no alignment
    passes, as the reference) and sets total_otu (its lines, "Total OTUs" of aligned.log) and n_yid_ycov (its entries).  For
    single-end reads the entries are aligned.log's "passing %id and %coverage" figure too; that figure is the n_yid_ycov total of the
    denovo_stats pass (denovo_counts), which for two mate files counts both files while the map holds the first file's reads only.
    otu_feed: for a paired run with otu_map, "one_file" (one interleaved file, -paired_in / -paired_out: every record) or
    "two_files" (stream_mates batches: the first file's reads); without it a paired otu_map is refused (SMR_ERR_UNSUPPORTED).
    summary: writes aligned.log at close() (hostio.summary_log, always plain): a dict of summary_log's inputs the library does not
    know -- cmd, refs, reads, gumbel, minimal_score, and optionally lnwin, skiplengths, threads, sq, pid, timestamp and counts
    (Aligner.read_counts(reads); counted at close() when absent).  The writer sums num_aligned and reads_matched_per_db over the
    batches it is given, and with denovo or otu_map on runs the denovo_stats pass (Aligner.denovo_stats) on every batch, its totals
    in denovo_counts.
    zip_out: the reference's -zip-out (its default for gzip input): every report file is written gzip-compressed on the device under
    its name with ".gz" appended, as members appended batch by batch (a multi-member file, as the reference's merge makes); a file
    with no member gets one empty member.  otu_map.txt stays plain, as the reference writes it.
    out2 / sout (opts): each read file is split as the reference's -out2 / -sout split it, aligned_fwd.fq / aligned_rev.fq,
    aligned_paired.fq / aligned_singleton.fq, or aligned_paired_fwd.fq ... aligned_singleton_rev.fq with both, and likewise other.*
    and aligned_denovo.*; batches of stream_mates are mates without further options (mates=True for a batch passed as text).
    blast="0": aligned.blast holds the pairwise rows (format_blast_pairwise); the other files are written as with any other blast."""

    def __init__(self, out_dir: str, aligner: Aligner, sam_header: str = "", otu_map=None, zip_out: bool = False, otu_feed=None,
                 summary: dict | None = None, **opts):
        self.dir, self.al, self.header, self.zip_out = out_dir, aligner, sam_header, zip_out
        self.opts = report_opts(**opts)
        self.otu_map, self.total_otu, self.n_yid_ycov = otu_map, None, None
        if otu_feed not in OTU_FEEDS:
            raise ValueError(f"otu_feed: {otu_feed!r} is not one of {list(OTU_FEEDS)}")
        self.otu_feed = otu_feed
        if otu_map is not None:
            aligner.otu_begin(otu_map[0], otu_map[1], paired_in=self.opts.paired_in, paired_out=self.opts.paired_out, feed=otu_feed)
        self.summary = summary
        self.num_aligned, self.reads_matched_per_db = 0, None
        self.denovo_counts = dict.fromkeys(DENOVO_TOTALS, 0) if summary is not None and (otu_map is not None or self.opts.denovo) else None
        self.ext = None
        self._parts = {}
        os.makedirs(out_dir, exist_ok=True)

    def _append(self, key, data):
        fh = self._parts.get(key)
        if fh is None:
            fh = self._parts[key] = open(os.path.join(self.dir, f".part_{key}"), "w+b")
        fh.write(data)

    def write(self, out: dict | None = None, text: bytes | None = None) -> dict:
        """format one batch (see Aligner.format_reports) and append its streams; returns them.  out=None: the results the last
        Aligner.place() or Aligner.place_packed() placed on the device, with the resident text (their counters are the ones it
        returned)."""
        if out is None and text is not None:
            raise ValueError("ReportWriter.write: the placed results go with the resident text (text=None)")
        if self.ext is None:
            first = text[:1] if text is not None else self.al.resident_text()[:1]
            self.ext = "fq" if first == b"@" else "fa"
        o = self.opts
        pairwise = bool(o.blast) and o.blast_format == 0
        if pairwise:   # the other files without BLAST, the BLAST streams from the pairwise writer
            rest = ReportOpts.from_buffer_copy(o)
            rest.blast = 0
            s = self.al.format_reports(out, text, opts=rest, gzip=self.zip_out)
            po = report_opts(blast="0", paired_in=o.paired_in, paired_out=o.paired_out, mates=o.mates)
            s["blast"] = self.al.format_blast_pairwise(out, text, opts=po, gzip=self.zip_out)
        else:
            s = self.al.format_reports(out, text, opts=o, gzip=self.zip_out)
        for g, (rows_sam, rows_blast) in enumerate(zip(s["sam"], s["blast"])):
            self._append(f"sam_{g}", rows_sam)
            self._append(f"blast_{g}", rows_blast)
        for k in ("aligned", "other", "denovo"):
            for j, data in enumerate(s[k] if isinstance(s[k], tuple) else (s[k],)):
                self._append(f"{k}_{j}", data)
        if self.otu_map is not None:
            self.al.otu_add(out, text)
        if self.summary is not None:
            c = out if out is not None else self.al.placed_info
            self.num_aligned += c["counters"]["num_aligned"]
            m = np.asarray(c["matched"][:max(1, self.al.n_index_files)], np.uint64)
            self.reads_matched_per_db = m.copy() if self.reads_matched_per_db is None else self.reads_matched_per_db + m
        if self.denovo_counts is not None:
            mid, mcov = self.otu_map if self.otu_map is not None else (o.min_id, o.min_cov)
            paired = bool(o.paired_in or o.paired_out or o.mates) or self.otu_feed is not None
            _, t = self.al.denovo_stats(out, text, mid, mcov, paired=paired)
            for k, v in t.items():
                self.denovo_counts[k] += v
        return s

    def close(self) -> list:
        """write the files; returns their paths"""
        o, ext, groups = self.opts, self.ext or "fq", self.al.report_groups()
        files = []
        head = self.header.encode()
        if o.sam:
            files.append(("aligned.sam", [f"sam_{g}" for g in range(len(groups))], self.al.gzip(head) if self.zip_out and head else head))
        if o.blast:
            files.append(("aligned.blast", [f"blast_{g}" for g in range(len(groups))], b""))
        for flag, name, key in ((o.fastx, "aligned", "aligned"), (o.other, "other", "other"), (o.denovo, "aligned_denovo", "denovo")):
            if flag:
                files += [(f"{name}{sfx}.{ext}", [f"{key}_{j}"], b"") for j, sfx in enumerate(fx_suffixes(o))]
        paths = []
        for name, keys, head in files:
            path = os.path.join(self.dir, name + (".gz" if self.zip_out else ""))
            with open(path, "wb") as f:
                f.write(head)
                for k in keys:
                    fh = self._parts.get(k)
                    if fh is not None:
                        fh.seek(0)
                        while True:
                            chunk = fh.read(1 << 24)
                            if not chunk:
                                break
                            f.write(chunk)
                if self.zip_out and f.tell() == 0:
                    f.write(self.al.gzip(b""))
            paths.append(path)
        if self.otu_map is not None:
            m = self.al.otu_finish()
            self.total_otu, self.n_yid_ycov = m["total_otu"], m["n_yid_ycov"]
            if m["n_yid_ycov"] > 0:
                path = os.path.join(self.dir, "otu_map.txt")
                with open(path, "wb") as f:
                    f.write(m["text"])
                paths.append(path)
        if self.summary is not None:
            paths.append(self._write_summary())
        for k, fh in self._parts.items():
            fh.close()
            os.unlink(os.path.join(self.dir, f".part_{k}"))
        self._parts = {}
        return paths


    def _write_summary(self) -> str:
        """aligned.log from the summary inputs and what the batches gave (the reference writes it with a plain ofstream, even
        under -zip-out)"""
        kw = dict(self.summary)
        counts = kw.pop("counts", None) or self.al.read_counts(kw["reads"])
        nidx = len(kw["refs"])
        matched = self.reads_matched_per_db if self.reads_matched_per_db is not None else np.zeros(nidx, np.uint64)
        dn = self.denovo_counts
        text = hostio.summary_log(
            total_reads=counts["reads"], all_reads_len=counts["length"], min_len=counts["min_len"], max_len=counts["max_len"],
            num_aligned=self.num_aligned, reads_matched_per_db=[int(x) for x in matched[:nidx]], params=kw.pop("params", getattr(self.al, "params", None)),
            denovo=dn["num_denovo"] if self.opts.denovo else None,
            otu=(dn["n_yid_ycov"], self.total_otu) if self.otu_map is not None else None, **kw)
        path = os.path.join(self.dir, "aligned.log")
        with open(path, "wb") as f:
            f.write(text.encode())
        return path


def align_files(aligner: Aligner, batch: hostio.ReadBatch):
    """Convenience: align a parsed read batch and return results + SAM rows."""
    out = aligner.align(batch.cat, batch.off)
    refs = [aligner.refs_by_index[i] for i in range(aligner.n_index_files)]
    s = out if out["slots"] else unpack_alns(out, max(1, int(out["res"]["n_align"].max(initial=0))))   # the host formatter is strided
    out["sam"] = hostio.format_sam_rows(batch, refs, s["res"], s["alns"], s["cigar"], s["slots"])
    return out


def _reads_ext(path: str) -> str:
    """the read files' extension: fq for FASTQ input, fa for FASTA (report_fx_base.cpp:94), from the first byte of the reads"""
    import gzip
    with open(path, "rb") as f:
        gz = f.read(2) == b"\x1f\x8b"
    with (gzip.open(path, "rb") if gz else open(path, "rb")) as f:
        return "fq" if f.read(1) == b"@" else "fa"


class _FileWriter:
    """The writer thread of run_files: appends the streams of one batch to their files while the caller makes the next batch.
    Jobs are (buf, so, [(stream index, file handle)], release); release() hands buf back to the caller's pool once written."""

    def __init__(self):
        import queue
        import threading
        self.q = queue.Queue()
        self.wait_s = self.write_s = 0.0
        self.error = None
        self.th = threading.Thread(target=self._loop, daemon=True)
        self.th.start()

    def _loop(self):
        import time
        while True:
            t0 = time.perf_counter()
            job = self.q.get()
            t1 = time.perf_counter()
            self.wait_s += t1 - t0
            if job is None:
                return
            buf, so, dest, release = job
            try:
                if self.error is None:
                    mv = memoryview(buf)
                    for k, fh in dest:
                        a, b = int(so[k]), int(so[k + 1])
                        if b > a:
                            fh.write(mv[a:b])
            except BaseException as e:   # re-raised by the caller at the next put() or close()
                self.error = e
            finally:
                release()
            self.write_s += time.perf_counter() - t1

    def put(self, job):
        if self.error is not None:
            raise self.error
        self.q.put(job)

    def close(self):
        self.q.put(None)
        self.th.join()
        if self.error is not None:
            raise self.error


def run_files(refs, reads, out_dir, params: Params | None = None, *, gumbel, minimal_score=None, evalue: float = 1.0, sam: bool = False,
              sq: bool = False, blast=None, fastx: bool = False, other: bool = False, denovo=None, otu_map=None, paired_in: bool = False,
              paired_out: bool = False, out2: bool = False, sout: bool = False, zip_out: bool = False, bam: bool = False, bam_sorted: bool = False,
              lnwin: int = 18, interval: int = 1,
              max_pos: int = 10000, max_mb: float = 3072.0, skiplengths=None, index_budget: int = 0, batch_bytes: int = 256 << 20,
              piece_bytes: int = 256 << 20, cmd: str = "", threads: int = 1, device: int = 0) -> dict:
    """The reference's run from read files to its out/ directory, in one call: refs = the -ref FASTA files, reads = one reads file
    or two mate files (plain or gzip), out_dir = where the report files go, under the reference's names.
      1. the count pass over the reads (Aligner.read_counts);
      2. per reference: the index statistics from the FASTA (hostio.fasta_index_stats), the minimal score (hostio.minimal_score at
         E-value `evalue`, unless minimal_score[k] is given) and the E-value sizes, and the index built on the device
         (Aligner.build_index_device: lnwin, interval, max_pos, max_mb, skiplengths[k] = -passes); index_budget > 0 bounds its device
         memory (Aligner.set_index_budget);
      3. the reads streamed through the device (stream_fastx, or stream_mates for two files) in batches of batch_bytes of text, each
         run, placed on the device (Aligner.place) and formatted from there (the _placed calls), with the OTU map and the denovo
         statistics added from the placed results too.  With params.num_alignments == 0 (all alignments) the batches run in the
         packed layout and are placed with Aligner.place_packed: device memory follows the alignments stored, and only the reads
         that store more than the first run's stride run again, where the strided layout would size every read by the largest
         count of the batch;
      4. otu_map.txt and aligned.log (hostio.summary_log; cmd / threads / sq are what it prints).
    gumbel[k] = (lambda, K) of refs[k]: the library does not compute them (the reference's ALP).  params: an api.Params (default
    default_params()).  Report options as report_opts / ReportWriter take them: sam, sq (-SQ), blast ("1 cigar qcov qstrand", "0"),
    fastx, other, denovo = (min_id, min_cov) for aligned_denovo.*, otu_map = (min_id, min_cov), paired_in / paired_out / out2 / sout,
    zip_out (every report file gzip-compressed on the device, ".gz" appended; otu_map.txt and aligned.log stay plain).  bam: also
    aligned.bam, the rows of aligned.sam (with or without sam) as BAM records in BGZF blocks written on the device
    (Aligner.bam_header, format_placed_into(bam=True)) and the BGZF EOF block; it is BGZF whatever zip_out says.  bam_sorted (implies
    bam): aligned.bam sorted by coordinate, with SO:coordinate in its header, and its index aligned.bam.bai: each batch's records go
    as one sorted run (Aligner.bam_sort_add) to the part file .part_bamsort, and after the stream Aligner.bam_sort_finish writes the
    sorted records in windows of BAM_SORT_WINDOW bytes (seconds["bam_sort"]).
    Files are written by a writer thread while the caller's thread makes, runs and formats the next batch (the library calls release
    the GIL); two output buffers alternate between them, and the streams go from those buffers to the files without a copy.  The
    read files and the SAM / BLAST rows of the first (index, part) group are appended to their final files as they come.  With
    several groups the rows of the other groups go to part files first and are appended at the end, as the reference's order (every
    row of group 0, then of group 1, ...) requires: those bytes are written twice.
    Returns {"reads", "batches", "num_aligned", "minimal_score", "paths", "layout" ("strided" or "packed"), "seconds": per stage}: count, index, stream (the whole
    streamed pass: from the first batch until every report file is complete and closed, the part files appended), produce (batch
    production: push, inflate, cut, decode), run, place, format (the report calls, the OTU map and the denovo statistics), writer
    (the writer thread's busy time), writer_wait (its idle time), caller_wait (the caller waiting for a free output buffer), parts
    (appending the part files of the groups after the first, and closing the files), finish (otu_map.txt and aligned.log)."""
    import shutil
    import threading
    import time
    refs, reads = [os.fspath(r) for r in refs], [os.fspath(r) for r in ([reads] if isinstance(reads, (str, os.PathLike)) else reads)]
    if len(reads) not in (1, 2):
        raise ValueError("run_files: one reads file, or two mate files")
    if len(gumbel) != len(refs) or (minimal_score is not None and len(minimal_score) != len(refs)):
        raise ValueError("run_files: gumbel (and minimal_score) take one entry per reference")
    params = params if params is not None else default_params()
    mates = len(reads) == 2
    o = report_opts(sam=sam, blast=blast, fastx=fastx, other=other, denovo=denovo, paired_in=paired_in, paired_out=paired_out,
                    out2=out2, sout=sout)
    pairwise = bool(o.blast) and o.blast_format == 0
    rest = ReportOpts.from_buffer_copy(o)
    if pairwise:
        rest.blast = 0
    pw_opts = report_opts(blast="0", paired_in=paired_in, paired_out=paired_out)
    bam_opts = report_opts(sam=True, paired_in=paired_in, paired_out=paired_out)
    bam = bam or bam_sorted
    feed = "two_files" if mates else "one_file" if (paired_in or paired_out) else None
    with_denovo = otu_map is not None or o.denovo
    sec = dict.fromkeys(("count", "index", "stream", "produce", "run", "place", "format", "writer", "writer_wait", "caller_wait", "parts",
                         "finish"), 0.0)
    if bam_sorted:
        sec["bam_sort"] = 0.0
    os.makedirs(out_dir, exist_ok=True)
    al = Aligner(device)
    files, parts = {}, {}
    writer = None
    try:
        al.set_params(params)
        t0 = time.perf_counter()
        counts = al.read_counts(reads if mates else reads[0], piece_bytes)
        sec["count"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        stats, seqs = zip(*[hostio.fasta_index_stats(f, lnwin, max_mb) for f in refs])
        ms = list(minimal_score) if minimal_score is not None else \
            [hostio.minimal_score(st, lam, K, counts["length"], counts["reads"], evalue) for st, (lam, K) in zip(stats, gumbel)]
        sk = list(skiplengths) if skiplengths is not None else [(lnwin, lnwin // 2, 3)] * len(refs)
        if index_budget:
            al.set_index_budget(index_budget)
        for k, f in enumerate(refs):
            al.build_index_device(k, f, hostio.split_by_parts(hostio.load_references(f), stats[k]), int(ms[k]), tuple(sk[k]), lnwin, interval,
                                  max_pos, max_mb)
            if o.blast:
                lam, K = gumbel[k]
                al.set_report_scoring(k, lam, K, *hostio.evalue_params(stats[k], K, counts["length"], counts["reads"]))
        al.set_place_stats(bool(o.sam or bam or o.blast or o.denovo or otu_map is not None))
        layout = "packed" if params.num_alignments == 0 else "strided"
        al.set_aln_layout(layout)
        place = al.place_packed if layout == "packed" else al.place
        if otu_map is not None:
            al.otu_begin(otu_map[0], otu_map[1], paired_in=paired_in, paired_out=paired_out, feed=feed)
        sec["index"] = time.perf_counter() - t0
        # the files: every stream of a batch -> (file, or a part file for the SAM / BLAST rows of groups after the first)
        G = len(al.report_groups())
        ext, gz = _reads_ext(reads[0]), ".gz" if zip_out else ""

        def open_file(name):
            files[name] = open(os.path.join(out_dir, name + gz), "wb")
            return files[name]

        def part_file(key):
            parts[key] = open(os.path.join(out_dir, f".part_{key}"), "w+b")
            return parts[key]

        dest, pw_dest, bam_dest = [], [], []
        head = hostio.sam_header_of([x for s in seqs for x in s], cmd, sq).encode()
        if o.sam:
            fh = open_file("aligned.sam")
            fh.write(al.gzip(head) if zip_out else head)
            dest += [(g, fh if g == 0 else part_file(f"sam_{g}")) for g in range(G)]
        run_starts, bam_header_bytes = [], 0
        if bam_sorted:   # the batches' sorted runs go to a part file; the windows are written after the stream
            fh = files["aligned.bam"] = open(os.path.join(out_dir, "aligned.bam"), "wb")
            hb = al.bam_header(head.replace(b"\tSO:unsorted\n", b"\tSO:coordinate\n", 1))
            fh.write(hb)
            bam_header_bytes = len(hb)
            files["aligned.bam.bai"] = open(os.path.join(out_dir, "aligned.bam.bai"), "wb")
            bam_dest = [(0, part_file("bamsort"))]
            al.bam_sort_begin()
        elif bam:
            fh = files["aligned.bam"] = open(os.path.join(out_dir, "aligned.bam"), "wb")
            fh.write(al.bam_header(head))
            bam_dest = [(g, fh if g == 0 else part_file(f"bam_{g}")) for g in range(G)]
        if o.blast:
            fh = open_file("aligned.blast")
            (pw_dest if pairwise else dest).extend((g + (0 if pairwise else G), fh if g == 0 else part_file(f"blast_{g}")) for g in range(G))
        num_out = num_out_of(o)
        for j, (flag, name) in enumerate(((o.fastx, "aligned"), (o.other, "other"), (o.denovo, "aligned_denovo"))):
            if flag:
                dest += [(2 * G + j * num_out + i, open_file(f"{name}{sfx}.{ext}")) for i, sfx in enumerate(fx_suffixes(o))]
        # two sets of output buffers (one buffer for each report call of a batch) alternate between this thread and the writer
        free = [[np.zeros(1 << 20, np.uint8), np.zeros(1 << 16, np.uint8), np.zeros(1 << 16, np.uint8)] for _ in range(2)]
        cv = threading.Condition()

        def release(slot):
            def f():
                with cv:
                    free.append(slot)
                    cv.notify()
            return f

        writer = _FileWriter()
        n_reads, num_aligned, n_batches = 0, 0, 0
        run_end = 0   # bytes of the runs in .part_bamsort so far
        matched = np.zeros(max(1, len(refs)), np.uint64)
        dn = dict.fromkeys(DENOVO_TOTALS, 0)
        dn_min, dn_paired = otu_map or denovo or (0, 0), bool(paired_in or paired_out) or feed is not None
        gen = al.stream_mates(reads[0], reads[1], batch_bytes, piece_bytes) if mates else al.stream_fastx(reads[0], batch_bytes, piece_bytes)
        t_stream = t0 = time.perf_counter()
        for n in gen:
            t1 = time.perf_counter()
            sec["produce"] += t1 - t0
            al.run_resident()
            t2 = time.perf_counter()
            info = place()
            t3 = time.perf_counter()
            n_reads += n
            n_batches += 1
            num_aligned += info["counters"]["num_aligned"]
            matched += np.asarray(info["matched"][:matched.size], np.uint64)
            with cv:
                while not free:
                    cv.wait()
                slot = free.pop()
            t4 = time.perf_counter()
            jobs = []
            if dest:
                slot[0], so = al.format_placed_into(rest, slot[0], zip_out)
                jobs.append((slot[0], so, dest))
            if pw_dest:
                slot[1], so = al.format_placed_into(pw_opts, slot[1], zip_out, pairwise=True)
                jobs.append((slot[1], so, pw_dest))
            if bam_sorted:
                slot[2], nb = al.bam_sort_add(bam_opts, slot[2])
                run_starts.append(run_end)
                run_end += nb
                jobs.append((slot[2], np.array([0, nb], np.uint64), bam_dest))
            elif bam_dest:
                slot[2], so = al.format_placed_into(bam_opts, slot[2], bam=True)
                jobs.append((slot[2], so, bam_dest))
            if otu_map is not None:
                al.otu_add(None)
            if with_denovo:
                for k, v in al.denovo_stats(None, None, dn_min[0], dn_min[1], dn_paired, per_read=False)[1].items():
                    dn[k] += v
            done = release(slot)
            if not jobs:
                done()
            for i, (buf, so, d) in enumerate(jobs):
                writer.put((buf, so, d, done if i + 1 == len(jobs) else (lambda: None)))
            t0 = time.perf_counter()
            sec["run"] += t2 - t1
            sec["place"] += t3 - t2
            sec["caller_wait"] += t4 - t3
            sec["format"] += t0 - t4
        sec["produce"] += time.perf_counter() - t0
        writer.close()
        sec["writer"], sec["writer_wait"] = writer.write_s, writer.wait_s
        writer = None
        t1 = time.perf_counter()
        for kind, name in (("sam", "aligned.sam"), ("blast", "aligned.blast"), ("bam", "aligned.bam")):
            for g in range(1, G):
                fh = parts.get(f"{kind}_{g}")
                if fh is not None:
                    fh.seek(0)
                    shutil.copyfileobj(fh, files[name], 1 << 24)
        if bam_sorted:
            t2 = time.perf_counter()
            runs = parts["bamsort"]
            runs.flush()
            bai = al.bam_sort_finish(runs, run_starts, files["aligned.bam"], bam_header_bytes)
            files["aligned.bam.bai"].write(bai)
            sec["bam_sort"] = time.perf_counter() - t2
        if bam:
            files["aligned.bam"].write(BGZF_EOF)
        paths = []
        for name, fh in files.items():
            if zip_out and fh.tell() == 0:   # never aligned.bam: it holds its header
                fh.write(al.gzip(b""))
            fh.close()
            paths.append(fh.name)
        t0 = time.perf_counter()
        sec["parts"] = t0 - t1
        sec["stream"] = t0 - t_stream
        total_otu = None
        if otu_map is not None:
            m = al.otu_finish()
            total_otu = m["total_otu"]
            if m["n_yid_ycov"] > 0:
                path = os.path.join(out_dir, "otu_map.txt")
                with open(path, "wb") as f:
                    f.write(m["text"])
                paths.append(path)
        log = hostio.summary_log(cmd=cmd, refs=refs, reads=reads, total_reads=counts["reads"], num_aligned=num_aligned,
                                 min_len=counts["min_len"], max_len=counts["max_len"], all_reads_len=counts["length"],
                                 reads_matched_per_db=[int(x) for x in matched[:len(refs)]], gumbel=list(gumbel), minimal_score=[int(x) for x in ms],
                                 lnwin=lnwin, skiplengths=sk, params=params, threads=threads, sq=sq,
                                 denovo=dn["num_denovo"] if o.denovo else None, otu=(dn["n_yid_ycov"], total_otu) if otu_map is not None else None)
        path = os.path.join(out_dir, "aligned.log")
        with open(path, "wb") as f:
            f.write(log.encode())
        paths.append(path)
        sec["finish"] = time.perf_counter() - t0
        return dict(reads=n_reads, batches=n_batches, num_aligned=num_aligned, paths=paths, seconds=sec, minimal_score=[int(x) for x in ms],
                    layout=layout)
    finally:
        if writer is not None:
            try:
                writer.close()
            except BaseException:
                pass
        for fh in list(files.values()) + list(parts.values()):
            fh.close()
        for key in parts:
            try:
                os.unlink(os.path.join(out_dir, f".part_{key}"))
            except OSError:
                pass
        al.close()
