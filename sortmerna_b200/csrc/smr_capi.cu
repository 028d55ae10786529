// C ABI of libsmr_b200.so (include/smr_b200.h): context, index residency, batch driver.
// Host side of the seam that replaces align() (src/sortmerna/processor.cpp:173-285).
#include "../../include/smr_b200.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "smr_decode.cuh"
#include "smr_report.cuh"
#include "smr_otu.cuh"
#include "smr_bamsort.cuh"
#include "smr_inflate.cuh"
#include "smr_stream.cuh"
#include "smr_deflate.cuh"
#include "smr_build.h"
#include "smr_build_dev.cuh"
#include "smr_final.cuh"
#include "smr_place.cuh"
#include "smr_index.h"

using namespace smr;

namespace {

// Device memory (DevBuf) or page-locked host memory (PinBuf), freed by its destructor.  Move-only: the buffers live in vectors.
template <bool kPinned>
struct Buf {
  void* p = nullptr; size_t cap = 0;
  Buf() = default;
  Buf(Buf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  Buf& operator=(Buf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }   // o frees what this held
  ~Buf() { reset(); }
  void reset() {
    if (p) { if (kPinned) cudaFreeHost(p); else cudaFree(p); }
    p = nullptr; cap = 0;
  }
  // exactly `bytes`, contents undefined; what the buffer held is freed first
  cudaError_t alloc(size_t bytes) {
    reset();
    const cudaError_t e = kPinned ? cudaHostAlloc(&p, bytes, cudaHostAllocDefault) : cudaMalloc(&p, bytes);
    if (e == cudaSuccess) cap = bytes; else p = nullptr;
    return e;
  }
};
using DevBuf = Buf<false>;
using PinBuf = Buf<true>;   // host staging (page-locked once; pageable vectors cost a page-fault pass + a bounce copy per batch)

// The search arrays of a part -- flookup, ftext, fid, pos_off, pos, what the seed and candidate kernels read -- lie one after the
// other in one buffer, each at a multiple of 256 bytes: the part's own device buffer, its pinned host copy and its place in the
// index arena of a budgeted run (smr_set_index_budget) have the same layout, so that moving a part is one copy.
constexpr int kSearchArrays = 5;

struct Part {
  DevIndex d{};
  std::vector<DevBuf> owned;   // the device arrays behind refseq, ref_off and rnames (part_array)
  size_t search_len[kSearchArrays] = {};   // bytes of each search array, 64 bytes of zero slack included
  DevBuf search;               // the part's own device copy of its search arrays (alloc_search); empty while the host holds them
  PinBuf host;                 // the pinned host copy of its search arrays, while an index budget runs the batch over several groups
  size_t bytes = 0, n_nodes = 0, n_entries = 0, n_ids = 0, n_pos = 0, n_refseq = 0;
  const char* rnames = nullptr; const uint64_t* rname_off = nullptr; uint32_t n_rnames = 0; bool has_rnames = false;   // smr_set_report_refs
  std::vector<std::string> h_rnames;   // host copy of the same ids: the OTU map ranks them (smr_otu_begin)
};

// device times of one run (CUDA events, ms) and its kernel launches (smr_last_timings)
struct RunTimes {
  double total = 0, seed = 0, lis = 0, final = 0; uint64_t launches = 0;
  RunTimes& operator+=(const RunTimes& o) { total += o.total; seed += o.seed; lis += o.lis; final += o.final; launches += o.launches; return *this; }
};

// One batch of reads on the device, the seed scratch sized from it, and what a run of it leaves for a download.  The context's
// resident batch is one; a scratch-overflow retry runs the flagged reads as another.  Move-only: the buffers free themselves.
struct Batch {
  uint32_t nreads = 0, max_len = 0; uint64_t total_nt = 0;
  uint32_t scale = 1;                // scratch scale (1 = fast path; 8x per retry)
  bool from_text = false;            // decoded from text on the device (smr_upload_fastx[_gz]): its header offsets are known
  std::vector<uint32_t> off32;       // host copy of seq_off
  DevBuf seq04, seq_off, pk_off, pk03, pk03alt, has_n;
  DevBuf hits, hit_cnt, cost, bins; size_t hits_stride = 0; uint32_t cnt_stride = 0;
  DevBuf state, flags, hit_db, aln_work, out_aln, aln_stats, cigar_pool, scalars, counters; uint64_t cigar_cap_dev = 0;
  std::vector<uint32_t> base;        // packed arenas: read r stores at [base[r], base[r + 1]) (empty: r * slots_of, the strided arenas)
  DevBuf aln_base;                   // device copy of base
  uint32_t run_slots = 0;            // the stride of its last run (0: not run)
  uint64_t run_id = 0;               // which run of the context its results are (0: not run)
  bool run_stats = false;            // its last run computed the stats
  RunTimes run;
};

// What a read stream's inflate carries from one round to the next (smr_inflate.h): where to resume, the open member's CRC-32 and
// length, the members seen so far, and the last 32 KB of output (win; win2 is the scratch that replaces it).
struct InfStream { InfResume at; InfCarry carry; uint32_t members = 0; bool have_window = false; DevBuf win, win2; };

// One file of a read stream: the compressed bytes not inflated yet (gz) and the text not made into a batch yet.
struct StreamSide {
  bool eof = false;
  std::vector<uint8_t> tail;   // gz: the pushed bytes from the byte of the resume point on (inf.at.bit counts from tail[0])
  InfStream inf;
  DevBuf text;                 // pending text: [off, n) is not in a batch yet
  uint64_t off = 0, n = 0, pushed = 0;
  char first = 0;              // the file's first byte: '@' = FASTQ
  bool have_first = false;
};

// The read stream of a context (smr_stream_begin .. smr_stream_next): one file, or two mate files (SMR_STREAM_MATES) whose
// records k are paired.  Their buffers belong to it; its scratch outlives it (close_stream).
struct ReadStream {
  bool open = false, gz = false, count_only = false, mates = false;
  uint64_t batch_bytes = 0;
  StreamSide side[2];          // side[1]: mate 2 of a mate stream
  CountState counts;
  struct Scratch { DevBuf rc, cut, mflag, mend[2]; } scr;   // count-pass partials, batch cut; mate stream: record flags, record ends per mate
};

// The device words that the text passes hand to the host, one buffer.  Each group belongs to the function named, which zeroes it.
struct TextWords {
  uint32_t nrec, seq_bytes, err;   // text_layout: records, sequence bytes, decode error bits
  uint32_t pk_words, max_len;      // upload_fastx_impl: packed words of the batch, its longest read
  uint32_t rpt_err;                // rpt_prologue: the report side's error bits (RptArgs::err)
  uint32_t rpt_bad;                // format_reports_impl, BAM: the first read BAM cannot hold
};

}  // namespace

struct smr_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  smr_params prm{};
  bool have_params = false;
  std::vector<Part> parts;
  // the index budget (smr_set_index_budget): what the parts' search arrays may take on the device; 0 = no limit
  struct {
    uint64_t budget = 0;
    DevBuf arena;                              // the resident group of a run over several groups (at most `budget` bytes)
    uint64_t uploads = 0, upload_bytes = 0;    // group uploads into the arena since smr_init, and their bytes
    double t_upload = 0;                       // ms of group uploads in the resident batch's last run and the retries of its download
  } ib;
  uint32_t n_index_files = 0;
  int sm_count = 132;
  uint32_t chunk_reads = 1u << 20;
  uint32_t need_slots = 0;       // set with SMR_ERR_CAPACITY in all-alignments mode: the stride the batch needs
  uint32_t all_slots = 16;       // stride of the result layout when num_alignments == 0 (smr_set_aln_slots)
  uint32_t layout = SMR_ALNS_STRIDED;   // smr_set_aln_layout
  uint64_t retry_slots = 1u << 24;      // slot budget of one sub-batch of reads run again (rerun_flagged)
  uint64_t runs_made = 0;               // numbers the runs (Batch::run_id)
  // The results of the resident batch's last run placed on the device (place: smr_place_results in the strided layout,
  // smr_place_results_packed and the packed downloads in the packed one), kept until the batch is run again or replaced; the
  // report-side _placed calls read them there, and a packed download retried for capacity, or repeated, copies them.
  struct Placed {
    uint64_t run_id = 0;   // Batch::run_id of the run they come from; 0 = none
    uint32_t nreads = 0, slots = 0; bool stats = false;
    bool packed = false;   // placed in the packed layout: n_alns alignments, read r's from aln_off[r]; slots = the first run's stride
    bool trace = false;    // packed: a run met a trace back error (each call that reads the placement fails with SMR_ERR_INDEX)
    uint64_t cig_words = 0, n_alns = 0;
    DevBuf res, aln, st, cig, cnt;                     // the placed arrays, the counters (ncnt u64)
    DevBuf words, off, nal, aoff, src, runs, scal, fsel, fout;   // scratch: CIGAR words and offsets, rows and aln_off per read, each read's
                                                                 // source run, the run table, flagged reads (scan, bits, list)
    std::vector<uint64_t> cnt_host;                    // what smr_place_results[_packed] adds to the caller's counters
    double t_place = 0;                                // ms of the placement passes (CUDA events), retries and re-runs excluded
    RunTimes t_run;                                    // the first run and its re-runs
  } pl;
  bool place_stats = false;   // smr_set_place_stats: every run computes the smr_aln_stats a placement keeps
  uint32_t lis_ctas_per_sm = kLisMinCtas;   // persistent CTAs of the candidate kernel per SM (matches its __launch_bounds__)

  // the resident batch and the text it was decoded from (smr_upload_*, smr_stream_next); clear_resident empties it
  struct Resident {
    Batch b;
    DevBuf text, hdroff;      // the text (smr_upload_fastx[_gz], a stream's batch) and each record's header offset in it (smr_decode.cuh)
    uint64_t text_bytes = 0;  // 0: no text behind the batch
    bool mates = false;       // the batch came from a mate stream: records 2k and 2k+1 are mates
  } res;
  // scratch of a run that no later call reads, sized by the scale of the run (setup_arenas)
  // (kept: a run over several groups of parts, the kOvfSlots bits held back between groups, group_flags_kernel)
  struct { DevBuf parts, seed_ctr, lis, lis_epochs, lis_queue, lis_done, lis_rows, lis_dbg, fin, lane_hits, tb, tb_jobs, fin_list, kept; } run;
  smr_aln_stats* host_stats = nullptr;   // optional output of the report arithmetic
  // page-locked staging of a download (download_impl) and of the host read layout (read_layout, upload_fastx_impl)
  struct { PinBuf state, flags, hitdb, outaln, stats, cigar, off32, pkoff; std::vector<uint64_t> coff; } h;
  // the line layout of the last text (text_layout, newline_index), read by the decode, the read stream and the report writer; cnt
  // holds the per-chunk newline counts, and then the decode's per-record packed-word counts; words holds the TextWords
  struct { DevBuf cnt, words, nl, hdr, sb, rec, spos; } tx;
  DevBuf cub_tmp;   // cub scratch of the text layout, the report writer and the OTU map
  // gz inflate scratch (inflate_round, smr_inflate.cuh) and what the last round found
  struct { DevBuf gz, cand, res, sym, win, ids, off, cnt, moff, mem, poff, plen, pcrc; uint32_t spans = 0, candidates = 0; } inf;
  ReadStream rs;
  double t_inflate = 0, t_decode = 0;
  bool instr = false;         // smr_set_instrumentation: seed kernel counts windows / lists / entries, candidate kernel accounts its phases (clock64)
  uint64_t flag_hist[6] = {0, 0, 0, 0, 0, 0};  // overflow causes seen so far (seed lane / seed region / pairs / trace / cigar / error)
  // report writer (smr_report.cuh): scoring tables per index_num (smr_set_report_scoring), scratch (rpt_prologue, format_reports_impl)
  struct RptScore { bool set = false; DevBuf ev, bits; };
  std::vector<RptScore> rpt_score;
  struct { DevBuf text, line, recs, res, aln, cig, st, flags, keys, keys2, vals, rows, first, sz, off, bsz, boff, fxsz, fxoff, grp, so, out, aoff, sread; } r;
  double t_rpt[3] = {0, 0, 0};
  struct { DevBuf in, chunk, m, freq, codes, hdr, info, scratch, poff, plen, crc, dst, trl, ghdr, out; } z;   // gzip deflate (gzip_streams, smr_deflate.cuh)
  uint64_t parts_gen = 0;   // bumped whenever a part is loaded or its report ids are set: an open OTU map refuses to go on after that
  // OTU map accumulator (smr_otu.cuh), smr_otu_begin .. smr_otu_finish
  struct Otu {
    bool active = false; uint64_t gen = 0; double min_id = 0, min_cov = 0; uint32_t feed = 0;
    std::vector<RptGroup> groups; uint32_t gbits = 0, kbits = 0;
    DevBuf rank, rank_off, grp, key, ent, pool, flag, pos, nsz, noff, vals, skey, sidx, size, off, out, scal;
    uint64_t n = 0, pool_bytes = 0;
    double t[3] = {0, 0, 0};
  } otu;
  struct { DevBuf read, tot; } dn;   // smr_denovo_stats: per-read counters, totals
  // coordinate-sorted BAM (smr_bamsort.cuh), smr_bam_sort_begin .. smr_bam_sort_index
  struct BamSort {
    bool active = false, planned = false; uint64_t gen = 0;
    std::vector<uint64_t> lin_off;                 // the linear index table: reference k's 16 kb windows at [lin_off[k], lin_off[k + 1])
    std::vector<uint64_t> run_rec, run_bytes;      // each run's first record (accumulator order) and first byte, and the totals
    DevBuf key, size;                              // the accumulator: each record's key and size, run after run (12 B per record)
    DevBuf ord, bkey, sbkey, bperm, ssz, soff, doff, gat;   // scratch of add
    DevBuf pperm, pkey, psz, pdoff, csz, coff;                // plan: the sorted order and the offsets of both orders
    DevBuf runs, adj, stage, win, wsoff, vb, ve, rb, head, pid, piece, bso, lin, linoff, err;   // window
    std::vector<uint64_t> pdoff_h;                 // plan: the byte offset of each record in sorted order, and the total
    std::vector<uint64_t> win_rec;                 // plan: each window's first record in sorted order, and the total
    std::vector<uint64_t> ranges_h;                // plan: each window's [lo, hi) of each run, as smr_bam_sort_plan returns them
    uint64_t header_bytes = 0, next = 0, coffset = 0;   // window: the next one, and the compressed offset of its first block
    std::vector<BamPiece> pieces;                  // window: the chunk pieces of the windows so far, in file order
  } bs;
  // timings
  std::vector<cudaEvent_t> ev;
  RunTimes t_run;   // the last run, and the retries of its download
  double t_h2d = 0, t_d2h = 0;
};

namespace {

// A failed call inside the library: the status and the smr_last_error text its entry point returns (SMR_CATCH).  Not a
// std::exception, so that only its own catch clause takes it.
struct Failure { int code; std::string msg; };
[[noreturn]] void fail(int code, std::string msg) { throw Failure{code, std::move(msg)}; }

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) fail(SMR_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
  } while (0)

// runs f when it leaves its scope, by return or by a throw
template <class F>
struct OnExit { F f; ~OnExit() { f(); } };
template <class F>
OnExit<F> on_exit(F f) { return OnExit<F>{f}; }

// alignment slots per read in every flat result array: num_alignments, or the stride set for "all alignments" (0)
uint32_t slots_of(const smr_ctx* ctx) { return ctx->prm.num_alignments > 0 ? (uint32_t)ctx->prm.num_alignments : std::max(1u, ctx->all_slots); }

bool packed(const smr_ctx* ctx) { return ctx->layout == SMR_ALNS_PACKED; }

// the result slots of a batch: strided, nreads * slots_of; packed, its stored alignments (the sum of n_align).  dev: results
// is the placement's device array, whose count the placement keeps.
uint64_t result_slots(const smr_ctx* ctx, const smr_read_result* results, uint32_t nreads, bool dev = false) {
  if (!packed(ctx)) return (uint64_t)nreads * slots_of(ctx);
  if (dev) return ctx->pl.n_alns;
  uint64_t n = 0;
  for (uint32_t r = 0; r < nreads; ++r) n += results[r].n_align;
  return n;
}

// slots of the reads [c0, c1) of a run's batch
uint64_t batch_slots(const smr_ctx* ctx, const Batch& b, uint32_t c0, uint32_t c1) {
  return b.base.empty() ? (uint64_t)(c1 - c0) * slots_of(ctx) : b.base[c1] - b.base[c0];
}

// grow-only: at least `bytes`; what the buffer held is not kept
template <class T = void, bool kPinned>
T* ensure(Buf<kPinned>& b, size_t bytes) {
  if (bytes > b.cap || !b.p) CK(b.alloc(bytes + bytes / 8 + 256));
  return (T*)b.p;
}

// grow-only as ensure, keeping the first `keep` bytes
void ensure_keep(smr_ctx* ctx, DevBuf& b, size_t bytes, size_t keep) {
  if (bytes <= b.cap && b.p) return;
  DevBuf n;
  CK(n.alloc(bytes + bytes / 8 + 256));
  if (keep) {
    CK(cudaMemcpyAsync(n.p, b.p, keep, cudaMemcpyDeviceToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  b = std::move(n);   // n frees the old buffer
}

// n items from the host to b (grown as needed), queued on the context's stream
template <class T>
void upload_async(smr_ctx* ctx, DevBuf& b, const T* src, size_t n) {
  ensure(b, n * sizeof(T) + 16);
  if (n) CK(cudaMemcpyAsync(b.p, src, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
}

// the context's first n events (created on first use), for the timings of one function: none is held across a call that takes its own
cudaEvent_t* events(smr_ctx* ctx, size_t n) {
  for (cudaEvent_t e; ctx->ev.size() < n; ctx->ev.push_back(e)) CK(cudaEventCreate(&e));
  return ctx->ev.data();
}

double elapsed_ms(cudaEvent_t a, cudaEvent_t b) { float ms = 0; cudaEventElapsedTime(&ms, a, b); return ms; }

// a device array of the part: n items, copied from src (host) or else zero, and 64 zero bytes of slack past the end; counted in pt.bytes
template <class T>
T* part_array(smr_ctx* ctx, Part& pt, size_t n, const void* src) {
  const size_t bytes = n * sizeof(T);
  DevBuf b;
  CK(b.alloc(bytes + 64));
  CK(cudaMemsetAsync(b.p, 0, bytes + 64, ctx->stream));
  if (src && bytes) CK(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  T* out = (T*)b.p;
  pt.bytes += bytes + 64;
  pt.owned.push_back(std::move(b));
  return out;
}

// ---------------------------------------------------------------------------------------------------------------------
// search arrays and the index budget
// ---------------------------------------------------------------------------------------------------------------------
// where search array k starts in the part's search buffer; search_at(pt, kSearchArrays) is the buffer's size
size_t search_at(const Part& pt, int k) {
  size_t at = 0;
  for (int j = 0; j < k; ++j) at += (pt.search_len[j] + 255) & ~(size_t)255;
  return at;
}
size_t search_bytes(const Part& pt) { return search_at(pt, kSearchArrays); }

// points d's search arrays into a buffer of the part's layout (null: none)
void set_search_ptrs(DevIndex& d, const Part& pt, const uint8_t* base) {
  auto at = [&](int k) { return base ? (const void*)(base + search_at(pt, k)) : nullptr; };
  d.flookup = (const uint4*)at(0); d.ftext = (const uint32_t*)at(1); d.fid = (const uint32_t*)at(2);
  d.pos_off = (const uint32_t*)at(3); d.pos = (const uint2*)at(4);
}

std::string part_name(const Part& pt) { return "index " + std::to_string(pt.d.index_num) + " part " + std::to_string(pt.d.part); }

// fails if the part's search arrays alone pass the index budget
void check_budget(const smr_ctx* ctx, const Part& pt, uint64_t budget) {
  if (budget && search_bytes(pt) > budget)
    fail(SMR_ERR_CAPACITY, part_name(pt) + ": its search arrays take " + std::to_string(search_bytes(pt)) + " bytes, more than the index budget of " +
                               std::to_string(budget) + " bytes");
}

// The part's own device buffer for search arrays of len[k] bytes each (64 bytes of zero slack are added), zeroed; points pt.d at it.
// pt.bytes counts len[k] + 64 for each.  A part larger than the index budget fails first.  Returns the buffer.
uint8_t* alloc_search(smr_ctx* ctx, Part& pt, const size_t (&len)[kSearchArrays]) {
  for (int k = 0; k < kSearchArrays; ++k) { pt.search_len[k] = len[k] + 64; pt.bytes += len[k] + 64; }
  check_budget(ctx, pt, ctx->ib.budget);
  CK(pt.search.alloc(search_bytes(pt)));
  CK(cudaMemsetAsync(pt.search.p, 0, search_bytes(pt), ctx->stream));
  set_search_ptrs(pt.d, pt, (const uint8_t*)pt.search.p);
  return (uint8_t*)pt.search.p;
}

// the search arrays of the part to its pinned host copy; its device copy is freed
void search_to_host(smr_ctx* ctx, Part& pt) {
  if (!pt.search.p) return;
  CK(pt.host.alloc(search_bytes(pt)));   // a failed pinned allocation is SMR_ERR_CUDA: the part stays on the device
  CK(cudaMemcpyAsync(pt.host.p, pt.search.p, search_bytes(pt), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  pt.search.reset();
  set_search_ptrs(pt.d, pt, nullptr);
}

// the search arrays of the part back to its own device buffer; its host copy is freed
void search_to_device(smr_ctx* ctx, Part& pt) {
  if (pt.search.p) return;
  CK(pt.search.alloc(search_bytes(pt)));
  CK(cudaMemcpyAsync(pt.search.p, pt.host.p, search_bytes(pt), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  pt.host.reset();
  set_search_ptrs(pt.d, pt, (const uint8_t*)pt.search.p);
}

// consecutive parts [first, first + n) run together; `bytes` of search arrays
struct IndexGroup { uint32_t first, n; uint64_t bytes; };

// The groups of the next run: consecutive parts in load order, each group within the budget (no budget: one group).
std::vector<IndexGroup> index_groups(const smr_ctx* ctx) {
  std::vector<IndexGroup> gs;
  for (uint32_t i = 0; i < ctx->parts.size(); ++i) {
    const uint64_t b = search_bytes(ctx->parts[i]);
    if (gs.empty() || (ctx->ib.budget && gs.back().bytes + b > ctx->ib.budget)) gs.push_back(IndexGroup{i, 0, 0});
    gs.back().n += 1; gs.back().bytes += b;
  }
  return gs;
}

// where part i of group gr lies in the index arena: after the group's parts before it
size_t arena_at(const smr_ctx* ctx, const IndexGroup& gr, uint32_t i) {
  size_t at = 0;
  for (uint32_t j = gr.first; j < i; ++j) at += search_bytes(ctx->parts[j]);
  return at;
}

uint32_t max_group_parts(const smr_ctx* ctx) {
  uint32_t m = 1;
  for (const IndexGroup& g : index_groups(ctx)) m = std::max(m, g.n);
  return m;
}

// Puts the search arrays where the budget wants them: one group, every part on the device in its own buffer and no arena; several
// groups, every part on the host (the arena is sized by the run).  Returns the groups.
std::vector<IndexGroup> apply_budget(smr_ctx* ctx) {
  for (const Part& pt : ctx->parts) check_budget(ctx, pt, ctx->ib.budget);
  const std::vector<IndexGroup> gs = index_groups(ctx);
  if (gs.size() <= 1) {
    ctx->ib.arena.reset();
    for (Part& pt : ctx->parts) search_to_device(ctx, pt);
  } else {
    for (Part& pt : ctx->parts) search_to_host(ctx, pt);
  }
  return gs;
}

// a loaded part joins the context's part list; under an index budget that now needs several groups, every part's search arrays go
// to the host, so that loading too stays within the budget plus the part being loaded
void add_part(smr_ctx* ctx, Part&& pt) {
  if (ctx->parts.size() >= 0xFFFF) fail(SMR_ERR_UNSUPPORTED, "more than 65535 index parts in one context");   // (DevIndex::gslot, AlnWork::idx_slot)
  const uint32_t index_num = pt.d.index_num;
  ctx->parts.push_back(std::move(pt));
  ctx->n_index_files = std::max(ctx->n_index_files, index_num + 1);
  ++ctx->parts_gen;
  if (ctx->ib.budget) apply_budget(ctx);
}

// device scratch of one call: n items of T (at least one) in a new buffer of `pool`, freed with it
template <class T>
T* scratch(std::vector<DevBuf>& pool, size_t n) {
  pool.emplace_back();
  CK(pool.back().alloc(std::max<size_t>(n, 1) * sizeof(T)));
  return (T*)pool.back().p;
}

// one cub device call, run twice: with no scratch to size it, then in `tmp` (grown as needed).  call(void* tmp, size_t& bytes).
template <class F>
void cub_run(DevBuf& tmp, F&& call) {
  size_t bytes = 0;
  CK(call(nullptr, bytes));
  ensure(tmp, bytes);
  CK(call(tmp.p, bytes));
}

// ---------------------------------------------------------------------------------------------------------------------
// index build on the device (smr_build_dev.cuh): orchestration of one part
// ---------------------------------------------------------------------------------------------------------------------

Part build_part_device(smr_ctx* ctx, const std::vector<RefRecord>& recs, const std::vector<size_t>& members, const BuildOptions& opt,
                       uint32_t index_num, uint32_t part) {
  BuildGeom g{};
  g.L = opt.lnwin; g.half = g.L / 2; g.pread = g.L + 1; g.interval = opt.interval; g.max_pos = opt.max_pos; g.burst_depth = g.pread - g.half - 3;
  g.nseq = (uint32_t)members.size();
  const uint32_t list_bits = 2 * g.half + 1, key_bits = list_bits + 2 * g.burst_depth;
  if (key_bits > 64 || 2 * g.pread > 62 || 2 * (g.half + 1) > 32) fail(SMR_ERR_UNSUPPORTED, "seed length too large for the device builder");
  // host: concatenated builder codes + 0..4 codes, offsets, first window of every sequence
  std::vector<uint64_t> soff(g.nseq + 1, 0);
  std::vector<uint32_t> wstart(g.nseq + 1, 0);
  uint64_t total_win = 0;
  for (uint32_t k = 0; k < g.nseq; ++k) {
    const size_t len = recs[members[k]].seq.size();
    soff[k + 1] = soff[k] + len;
    total_win += (len - g.pread + g.interval) / g.interval;
    if (total_win >= (1ull << 31)) fail(SMR_ERR_UNSUPPORTED, "more than 2^31 windows in one index part");
    wstart[k + 1] = (uint32_t)total_win;
  }
  if (soff[g.nseq] >= 0xFFFFFFFFull) fail(SMR_ERR_UNSUPPORTED, "reference part larger than 4 GB");
  g.nwin = (uint32_t)total_win;
  std::vector<uint8_t> codes(soff[g.nseq]), c04(soff[g.nseq] + 64, 4);
  for (uint32_t k = 0; k < g.nseq; ++k) {
    const RefRecord& r = recs[members[k]];
    memcpy(codes.data() + soff[k], r.seq.data(), r.seq.size());
    memcpy(c04.data() + soff[k], r.seq04.data(), r.seq04.size());
  }
  std::vector<uint32_t> roff(g.nseq + 1);
  for (uint32_t k = 0; k <= g.nseq; ++k) roff[k] = (uint32_t)soff[k];
  std::vector<DevBuf> tmp;   // scratch of this build, freed on return
  cudaStream_t st = ctx->stream;
  const uint32_t n = g.nwin;
  const unsigned tb = 256, gw = (n + tb - 1) / tb;
  uint8_t* d_codes = scratch<uint8_t>(tmp, codes.size() + 64);
  uint64_t* d_soff = scratch<uint64_t>(tmp, soff.size());
  uint32_t* d_wstart = scratch<uint32_t>(tmp, wstart.size());
  CK(cudaMemcpyAsync(d_codes, codes.data(), codes.size(), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_soff, soff.data(), soff.size() * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_wstart, wstart.data(), wstart.size() * 4, cudaMemcpyHostToDevice, st));
  uint64_t *keyA = scratch<uint64_t>(tmp, n), *keyB = scratch<uint64_t>(tmp, n);
  uint32_t *valA = scratch<uint32_t>(tmp, n), *valB = scratch<uint32_t>(tmp, n), *u0 = scratch<uint32_t>(tmp, n), *u1 = scratch<uint32_t>(tmp, n),
           *u2 = scratch<uint32_t>(tmp, n), *u3 = scratch<uint32_t>(tmp, n), *win_id = scratch<uint32_t>(tmp, n);
  // cub scratch, sized exactly for the largest call (entries: at most 2n), so that cub_run never grows it
  size_t cub_bytes = 0, need = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, need, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, 2 * (size_t)n, 0, 64, st); cub_bytes = std::max(cub_bytes, need);
  cub::DeviceScan::InclusiveSum(nullptr, need, (uint32_t*)nullptr, (uint32_t*)nullptr, 2 * (size_t)n, st); cub_bytes = std::max(cub_bytes, need);
  cub::DeviceScan::InclusiveScan(nullptr, need, (uint32_t*)nullptr, (uint32_t*)nullptr, cuda::maximum<uint32_t>{}, 2 * (size_t)n, st); cub_bytes = std::max(cub_bytes, need);
  DevBuf d_cub;
  CK(d_cub.alloc(cub_bytes + 256));
  // 1. windows sorted by value (stable: equal values keep scan order)
  bld_windows_kernel<<<gw, tb, 0, st>>>(d_codes, d_soff, d_wstart, g, keyA, valA);
  CK(cudaGetLastError());
  cub_run(d_cub, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, keyA, keyB, valA, valB, (size_t)n, 0, (int)(2 * g.pread), st); });
  // 2. distinct (L+1)-mers, ids of the L-mers
  bld_heads_kernel<<<gw, tb, 0, st>>>(keyB, n, u0, u1);
  CK(cudaGetLastError());
  cub_run(d_cub, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, u0, u2, (size_t)n, st); });
  cub_run(d_cub, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, u1, u3, (size_t)n, st); });
  uint32_t nent = 0, nids = 0;
  CK(cudaMemcpyAsync(&nent, u2 + (n - 1), 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&nids, u3 + (n - 1), 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint32_t E = 2 * nent;
  uint32_t *e_list = scratch<uint32_t>(tmp, E), *e_pref = scratch<uint32_t>(tmp, E), *e_text = scratch<uint32_t>(tmp, E), *e_id = scratch<uint32_t>(tmp, E),
           *e_arr = scratch<uint32_t>(tmp, E), *e_tpar = scratch<uint32_t>(tmp, E);
  uint8_t* e_leaf = scratch<uint8_t>(tmp, E);
  CK(cudaMemsetAsync(e_tpar, 0, (size_t)E * 4, st)); CK(cudaMemsetAsync(e_leaf, 0, E, st));
  bld_entries_kernel<<<gw, tb, 0, st>>>(keyB, valB, u0, u2, u3, g, nent, win_id, e_list, e_pref, e_text, e_id, e_arr);
  CK(cudaGetLastError());
  // 3. positions (persistent arrays)
  bld_poskeys_kernel<<<gw, tb, 0, st>>>(win_id, n, keyA);
  CK(cudaGetLastError());
  cub_run(d_cub, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, keyA, keyB, (size_t)n, 0, 64, st); });
  bld_posflag_kernel<<<gw, tb, 0, st>>>(keyB, n, u0);
  CK(cudaGetLastError());
  cub_run(d_cub, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveScan(t, b, u0, u1, cuda::maximum<uint32_t>{}, (size_t)n, st); });
  bld_poskeep_kernel<<<gw, tb, 0, st>>>(u1, n, g.max_pos, u2);
  CK(cudaGetLastError());
  cub_run(d_cub, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, u2, u3, (size_t)n, st); });
  uint32_t npos = 0;
  CK(cudaMemcpyAsync(&npos, u3 + (n - 1), 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  Part pt;
  pt.d.index_num = index_num; pt.d.part = part;
  const size_t nk = (size_t)1 << (2 * g.half);
  const size_t len[kSearchArrays] = {nk * 16, ftext_words(E) * 4, (size_t)E * 4, ((size_t)nids + 1) * 4, (size_t)npos * 8};
  alloc_search(ctx, pt, len);
  uint4* p_flookup = (uint4*)pt.d.flookup; uint32_t* p_ftext = (uint32_t*)pt.d.ftext; uint32_t* p_fid = (uint32_t*)pt.d.fid;
  uint32_t* p_posoff = (uint32_t*)pt.d.pos_off; uint2* p_pos = (uint2*)pt.d.pos;
  bld_poswrite_kernel<<<gw, tb, 0, st>>>(keyB, u1, u2, u3, d_wstart, g, nids, p_posoff, p_pos);
  CK(cudaGetLastError());
  // 4. burst-trie order of the entries: first occurrence order, then one stable sort + one decision pass per level
  const unsigned ge = (E + tb - 1) / tb;
  uint64_t *ekA = scratch<uint64_t>(tmp, E), *ekB = scratch<uint64_t>(tmp, E);
  uint32_t *pA = scratch<uint32_t>(tmp, E), *pB = scratch<uint32_t>(tmp, E);
  bld_arrkey_kernel<<<ge, tb, 0, st>>>(e_arr, E, ekA, pA);
  CK(cudaGetLastError());
  cub_run(d_cub, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, ekA, ekB, pA, pB, (size_t)E, 0, 32, st); });
  for (uint32_t d = 1; d <= g.burst_depth; ++d) {
    bld_levelkey_kernel<<<ge, tb, 0, st>>>(pB, e_list, e_pref, e_leaf, E, d, g.burst_depth, ekA, pA);
    CK(cudaGetLastError());
    cub_run(d_cub, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, ekA, ekB, pA, pB, (size_t)E, 0, (int)key_bits, st); });
    if (d < g.burst_depth) { bld_level_kernel<<<ge, tb, 0, st>>>(ekB, pB, E, d, e_arr, e_tpar, e_leaf); CK(cudaGetLastError()); }
  }
  // 5. the lists and their lookup rows
  bld_flist_kernel<<<ge, tb, 0, st>>>(pB, e_list, e_text, e_id, E, p_ftext, p_fid, (uint32_t*)p_flookup, 0);
  bld_flist_kernel<<<ge, tb, 0, st>>>(pB, e_list, e_text, e_id, E, p_ftext, p_fid, (uint32_t*)p_flookup, 1);
  CK(cudaGetLastError());
  // 6. references for the Smith-Waterman side
  uint8_t* p_ref = part_array<uint8_t>(ctx, pt, c04.size(), c04.data());
  uint32_t* p_roff = part_array<uint32_t>(ctx, pt, roff.size(), roff.data());
  CK(cudaStreamSynchronize(st));
  pt.d.lnwin = g.L; pt.d.partialwin = g.half; pt.d.nref = g.nseq; pt.d.nids = nids;
  pt.d.refseq = p_ref; pt.d.ref_off = p_roff;
  pt.n_entries = E; pt.n_ids = nids; pt.n_pos = npos; pt.n_refseq = c04.size();
  return pt;
}

DevParams to_dev(const smr_params& p) {
  DevParams d;
  d.match = p.match; d.mismatch = p.mismatch; d.score_N = p.score_N; d.gap_open = p.gap_open; d.gap_ext = p.gap_ext;
  d.num_seeds = p.num_seeds; d.min_lis = p.min_lis; d.edges = p.edges; d.edges_is_percent = p.edges_is_percent;
  d.num_alignments = p.num_alignments; d.is_best = p.is_best; d.is_forward = p.is_forward; d.is_reverse = p.is_reverse;
  d.is_full_search = p.is_full_search;
  d.one = 1;
  return d;
}

uint32_t pow2_ge(uint32_t v) { uint32_t p = 1; while (p < v) p <<= 1; return p; }

// scalars block layout (u32): [0]=work_n [1]=lis work_next [2]=final work_next [3]=lis work_next of the second cursor ; cigar_used (u64) at byte 16 ;
// finalize job count (u32) at byte 24 ; task queue cursors at 128..
struct Scalars { uint32_t* work_n; uint32_t* lis_next; uint32_t* fin_next; uint32_t* lis_next_b; unsigned long long* cigar_used; uint32_t* fin_jobs; uint32_t* q_head; uint32_t* q_tail; uint32_t* planners_done; };
Scalars scalars_of(const Batch& b) {
  uint8_t* p = (uint8_t*)b.scalars.p;
  return Scalars{(uint32_t*)p, (uint32_t*)(p + 4), (uint32_t*)(p + 8), (uint32_t*)(p + 12), (unsigned long long*)(p + 16), (uint32_t*)(p + 24), (uint32_t*)(p + 128), (uint32_t*)(p + 256), (uint32_t*)(p + 384)};
}

// the arenas of a run as the kernels see them: the chunk-independent parts of LisGlobals and FinalGlobals, and the launch sizes
struct RunGeom {
  LisGlobals lg{};
  FinalGlobals fg{};
  uint32_t lis_ctas = 0, lis_warps = 0, final_warps = 0, tb_threads = 0, seed_ctas = 0, lane_hits_cap = 0;
};

RunGeom setup_arenas(smr_ctx* ctx, uint32_t scale, uint32_t max_len) {
  auto& A = ctx->run;
  RunGeom g;
  LisGlobals& lg = g.lg; FinalGlobals& fg = g.fg;
  uint32_t max_nref = 1;
  for (auto& pt : ctx->parts) max_nref = std::max(max_nref, pt.d.nref);
  lg.hist_cap = max_nref;
  lg.cand_cap = std::max(64u, max_nref);
  lg.pair_cap = pow2_ge(4096u * scale);
  lg.task_cap = 2 * lg.pair_cap;
  // SW windows are at most read length + 2 * edges columns (alignment.cpp:272-357; edges may be a percentage of the read)
  const uint32_t edges = ctx->prm.edges_is_percent ? (uint32_t)((ctx->prm.edges / 100.0) * (double)max_len) : (uint32_t)std::max(0, ctx->prm.edges);
  lg.row_cap = max_len + 2 * edges + 2 * 64 + 64;
  // planner and scorer warps wait for each other: EVERY CTA of the grid must be resident at once
  int occ = 0;
  for (auto k : {lis_kernel<false, false>, lis_kernel<true, false>, lis_kernel<false, true>, lis_kernel<true, true>})
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kLisSmemBytes));
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, lis_kernel<true, false>, kLisWarpsPerCta * 32, kLisSmemBytes));   // (same launch bounds and shared memory for all)
  if (occ < 1) fail(SMR_ERR_CUDA, "lis_kernel does not fit on an SM");
  g.lis_ctas = (uint32_t)ctx->sm_count * std::min<uint32_t>(ctx->lis_ctas_per_sm, (uint32_t)occ);
  g.lis_warps = g.lis_ctas * kPlannerWarps;   // planner warps (each owns an arena)
  lg.pall_cap = 32768u * scale;
  lg.arena_stride = lis_arena_bytes(lg.hist_cap, lg.cand_cap, lg.pair_cap, lg.task_cap, lg.pall_cap);
  // keep the arena total under ~16 GB (of the 80 GB of an H100): fewer persistent CTAs for huge reference sets
  const size_t budget = (size_t)16 << 30;
  while (g.lis_ctas > 16 && lg.arena_stride * g.lis_warps > budget) { g.lis_ctas /= 2; g.lis_warps = g.lis_ctas * kPlannerWarps; }
  lg.arena_base = ensure<uint8_t>(A.lis, lg.arena_stride * g.lis_warps);
  lg.epochs = ensure<uint32_t>(A.lis_epochs, (size_t)g.lis_warps * 4);
  lg.ring = ensure<QSlot>(A.lis_queue, (size_t)2 * kQueueCap * sizeof(QSlot) + 64);
  lg.done = ensure<uint32_t>(A.lis_done, (size_t)g.lis_warps * 4 + 64);
  const size_t dbg_bytes = (size_t)(kTlBase + kTlRows * kTlBuckets) * 8;
  ensure(A.lis_dbg, dbg_bytes);
  CK(cudaMemsetAsync(A.lis_dbg.p, 0, dbg_bytes, ctx->stream));
  // (the timeline costs the instrumented kernel an atomic per scored pair)
  lg.dbg = (getenv("SMR_TIMELINE") || getenv("SMR_VERBOSE")) ? (unsigned long long*)A.lis_dbg.p : nullptr;
  lg.score_rows = ensure<int32_t>(A.lis_rows, (size_t)g.lis_ctas * kScorerWarps * 2 * lg.row_cap * 4);
  // histogram epochs start at 0 over a zeroed histogram (every run: the arena layout depends on the scale of the run)
  CK(cudaMemset2DAsync(A.lis.p, lg.arena_stride, 0, lis_arena_zero_bytes(lg.hist_cap), g.lis_warps, ctx->stream));   // votes + bitmaps only
  CK(cudaMemsetAsync(A.lis_epochs.p, 0, (size_t)g.lis_warps * 4, ctx->stream));
  fg.cap_w = 2 * 256 * scale + 8;          // band widths up to 256*scale
  fg.cap_cig = 2 * (max_len + 64) + 16;
  fg.row_cap = lg.row_cap;
  fg.cap_dir = (size_t)65536 * scale + (size_t)max_len * 9 * 3 + 64;
  g.final_warps = (uint32_t)ctx->sm_count * kFinalCtasPerSm * kFinalWarpsPerCta;
  fg.arena_stride = final_arena_bytes(fg.cap_w, fg.cap_cig, fg.row_cap, fg.cap_dir);
  while (g.final_warps > 64 && fg.arena_stride * g.final_warps > budget) g.final_warps /= 2;
  fg.arena_base = ensure<uint8_t>(A.fin, fg.arena_stride * g.final_warps);
  // traceback stage: one thread per alignment, 1024 threads per SM
  g.tb_threads = (uint32_t)ctx->sm_count * 1024u;
  fg.tb_cap_w = 2 * 32 * scale + 8;                       // band widths up to 32*scale
  fg.tb_cap_cig = 128 * scale;
  fg.tb_cap_dir = (size_t)32768 * scale;                  // (2*band+1) * readLen * 3 bytes: band 32 at 150 nt
  fg.tb_stride = ((size_t)fg.tb_cap_w * 12 + (size_t)fg.tb_cap_cig * 4 + fg.tb_cap_dir + 255) & ~(size_t)255;
  while (g.tb_threads > 4096 && fg.tb_stride * g.tb_threads > budget) g.tb_threads /= 2;
  fg.tb_arena = ensure<uint8_t>(A.tb, fg.tb_stride * g.tb_threads);
  g.lane_hits_cap = kLaneHitCap * scale;
  const uint32_t lane_hits_warps = scale == 1 ? (uint32_t)ctx->sm_count * kSeedCtasPerSm * kSeedWarpsPerCta : 1024u;
  g.seed_ctas = lane_hits_warps / kSeedWarpsPerCta;
  ensure(A.lane_hits, (size_t)lane_hits_warps * g.lane_hits_cap * 32 * 4);
  return g;
}

// the reads c0 .. c0 + n of a batch as the kernels see them
DevBatch make_batch(const Batch& s, uint32_t c0, uint32_t n) {
  DevBatch b{};
  b.nreads = n; b.r0 = c0; b.seq_base0 = s.off32[c0];
  b.seq04 = (const uint8_t*)s.seq04.p; b.seq_off = (const uint32_t*)s.seq_off.p;
  b.pk03 = (const uint32_t*)s.pk03.p; b.pk03alt = (const uint32_t*)s.pk03alt.p; b.pk_off = (const uint32_t*)s.pk_off.p;
  b.has_n = (const uint8_t*)s.has_n.p; b.hit_scale = s.scale; b.hits = (uint2*)s.hits.p;
  b.hit_cnt = (uint32_t*)s.hit_cnt.p; b.flags = (uint32_t*)s.flags.p; b.state = (ReadState*)s.state.p;
  b.hit_db = (uint16_t*)s.hit_db.p; b.counters = (unsigned long long*)s.counters.p;
  b.hits_stride = s.hits_stride; b.cnt_stride = s.cnt_stride; b.cost = (uint32_t*)s.cost.p;
  b.bins = (uint32_t*)s.bins.p; b.bin_count = (uint32_t*)s.bins.p + (size_t)s.cnt_stride * kCostBins;
  return b;
}

// The layout of n reads of lengths len(r) in b: read offsets (b.off32, b.seq_off), packed-word offsets (b.pk_off: (len + 15) / 16 + 2
// words per read, the layout of pack_reads_kernel), nreads, total_nt and max_len.  Returns the packed-word total.  The device copies
// are staged in the context's pinned buffers: the caller synchronizes before the next layout.
template <class Len>
uint64_t read_layout(smr_ctx* ctx, Batch& b, uint32_t n, Len len) {
  uint32_t* pkoff = ensure<uint32_t>(ctx->h.pkoff, (size_t)(n + 1) * 4);
  uint32_t* off32 = ensure<uint32_t>(ctx->h.off32, (size_t)(n + 1) * 4);
  uint64_t total = 0, w = 0; uint32_t max_len = 0;
  for (uint32_t r = 0; r <= n; ++r) {
    off32[r] = (uint32_t)total;
    pkoff[r] = (uint32_t)w;
    if (r < n) {
      const uint64_t l = len(r);
      max_len = std::max<uint32_t>(max_len, (uint32_t)l);
      total += l;
      w += (l + 15) / 16 + 2;     // +2 padding words: window_fwd reads three consecutive words
    }
  }
  if (total >= 0xF0000000ull) fail(SMR_ERR_ARG, "batch larger than 2^32 nucleotides: split it");
  if (w >= 0xFFFFFFFFull) fail(SMR_ERR_ARG, "batch too large");
  upload_async(ctx, b.seq_off, off32, n + 1);
  upload_async(ctx, b.pk_off, pkoff, n + 1);
  b.off32.assign(off32, off32 + n + 1);
  b.nreads = n; b.total_nt = total; b.max_len = max_len;
  return w;
}

// the hit regions of a batch for groups of `nparts` parts
void ensure_hit_regions(Batch& b, uint32_t nparts) {
  ensure(b.hits, b.hits_stride * nparts * 8);
  ensure(b.hit_cnt, (size_t)b.cnt_stride * nparts * 4);
}

// The part of an upload that does not depend on where the reads came from: b's reads and offsets are on the device and b.off32 on the
// host; sizes the batch's other buffers for its scale and 2-bit packs the reads.
void finish_upload(smr_ctx* ctx, Batch& b, uint64_t w) {
  const uint32_t nreads = b.nreads;
  ensure(b.pk03, (size_t)(w + 4) * 4);
  ensure(b.pk03alt, (size_t)(w + 4) * 4);
  ensure(b.has_n, nreads);
  ensure(b.flags, (size_t)nreads * 4);
  ensure(b.state, (size_t)nreads * sizeof(ReadState));
  ensure(b.hit_db, (size_t)nreads * 2);
  const uint64_t nslots = batch_slots(ctx, b, 0, nreads);
  ensure(b.aln_work, (size_t)nslots * sizeof(AlnWork));
  ensure(b.out_aln, (size_t)nslots * sizeof(OutAln));
  if (!b.base.empty()) upload_async(ctx, b.aln_base, b.base.data(), b.base.size());
  ensure(b.scalars, 512);
  ensure(b.counters, (size_t)(dcCount + 64) * 8);
  CK(cudaMemsetAsync(b.pk03.p, 0, (size_t)(w + 4) * 4, ctx->stream));
  CK(cudaMemsetAsync(b.pk03alt.p, 0, (size_t)(w + 4) * 4, ctx->stream));
  // hit regions are per chunk
  uint64_t max_chunk_nt = 0;
  for (uint32_t c0 = 0; c0 < nreads; c0 += ctx->chunk_reads) {
    const uint32_t c1 = std::min(nreads, c0 + ctx->chunk_reads);
    max_chunk_nt = std::max<uint64_t>(max_chunk_nt, b.off32[c1] - b.off32[c0]);
  }
  // one hit-region set per (index,part) of a resident group: the group's parts are seeded before the candidate kernel runs read-major
  // (run_impl grows them if the groups have changed since)
  b.cnt_stride = std::min(nreads, ctx->chunk_reads);
  b.hits_stride = (size_t)((uint64_t)b.scale * (2 * max_chunk_nt + 32ull * b.cnt_stride) + 64);
  ensure_hit_regions(b, max_group_parts(ctx));
  ensure(b.cost, (size_t)b.cnt_stride * 4);
  ensure(b.bins, (size_t)b.cnt_stride * kCostBins * 4 + (size_t)kCostBins * 4);
  // 2-bit packing + N detection
  pack_reads_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(make_batch(b, 0, nreads), (uint32_t*)b.pk03.p, (uint32_t*)b.pk03alt.p, (uint8_t*)b.has_n.p);
  CK(cudaGetLastError());
}

// an empty resident batch with no text behind it
void clear_resident(smr_ctx* ctx) {
  auto& R = ctx->res;
  R.b.nreads = 0; R.b.from_text = false; R.text_bytes = 0; R.mates = false; R.b.run_id = 0;
}

// host reads -> the resident batch (no text behind it)
void upload_batch_impl(smr_ctx* ctx, const uint8_t* seq_cat, const uint64_t* seq_off, uint32_t nreads) {
  clear_resident(ctx);
  if (nreads == 0) return;
  Batch& b = ctx->res.b;
  cudaEvent_t* e = events(ctx, 2);
  CK(cudaEventRecord(e[0], ctx->stream));
  const uint64_t w = read_layout(ctx, b, nreads, [&](uint32_t r) { return seq_off[r + 1] - seq_off[r]; });
  ensure(b.seq04, b.total_nt + 64);
  CK(cudaMemcpyAsync(b.seq04.p, seq_cat + seq_off[0], b.total_nt, cudaMemcpyHostToDevice, ctx->stream));
  finish_upload(ctx, b, w);
  CK(cudaEventRecord(e[1], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->t_h2d = elapsed_ms(e[0], e[1]);
}

// exclusive sum of n u32 (out may equal in) in the context's cub scratch
void exclusive_sum(smr_ctx* ctx, const uint32_t* in, uint32_t* out, uint32_t n) {
  cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, in, out, n, ctx->stream); });
}

// Newline positions of a text (smr_decode.cuh (1)-(3)) in tx.nl: count per 32-byte chunk, scan (the total lands at [nchunks]),
// positions.  A text that does not end in '\n' gets a virtual one at nbytes.  Returns their number.
uint32_t newline_index(smr_ctx* ctx, const uint8_t* text, uint64_t nbytes) {
  auto& X = ctx->tx;
  const int grid = ctx->sm_count * 8;
  const uint64_t nchunks = nbytes / 32 + 1;
  uint32_t* cnt = ensure<uint32_t>(X.cnt, (nchunks + 1) * 4);
  count_newlines_kernel<<<grid, 256, 0, ctx->stream>>>(text, nbytes, cnt, nchunks);
  CK(cudaMemsetAsync(cnt + nchunks, 0, 4, ctx->stream));
  exclusive_sum(ctx, cnt, cnt, (uint32_t)nchunks + 1);
  uint32_t n = 0;
  CK(cudaMemcpyAsync(&n, cnt + nchunks, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ensure(X.nl, ((size_t)n + 1) * 8);
  if (n) write_newlines_kernel<<<grid, 256, 0, ctx->stream>>>(text, nbytes, cnt, nchunks, (uint64_t*)X.nl.p);
  CK(cudaGetLastError());
  return n;
}

TextWords* text_words(smr_ctx* ctx) { return ensure<TextWords>(ctx->tx.words, 64); }

struct TextLayout { uint32_t nlines = 0, nrec = 0, total_nt = 0; uint32_t fmt = kFmtFasta; };

// The line layout of a FASTA / FASTQ text on the device (the line passes of smr_decode.cuh), for the decode and the report writer.
// first_byte is text[0] and names the format.  Leaves in ctx->tx, for each of the nlines lines, its newline position (nl), header
// flag (hdr), sequence bytes (sb), record index (rec) and the offset of its sequence bytes (spos); the arrays hold nlines + 1 items,
// rec and spos the totals at [nlines].
TextLayout text_layout(smr_ctx* ctx, const uint8_t* text, uint64_t nbytes, char first_byte) {
  auto& X = ctx->tx;
  TextLayout L;
  if (nbytes >= 0xF0000000ull) fail(SMR_ERR_ARG, "text batch of 2^32 bytes or more: split it (line counts and sequence offsets are 32-bit on the device)");
  if (nbytes && first_byte != '@' && first_byte != '>') fail(SMR_ERR_ARG, "reads text must start with '@' (FASTQ) or '>' (FASTA)");
  L.fmt = first_byte == '@' ? kFmtFastq : kFmtFasta;
  TextWords* tw = text_words(ctx);
  CK(cudaMemsetAsync(tw, 0, offsetof(TextWords, pk_words), ctx->stream));   // nrec, seq_bytes, err
  const int grid = ctx->sm_count * 8;
  L.nlines = newline_index(ctx, text, nbytes);
  const uint32_t n = L.nlines;
  uint32_t* hdr = ensure<uint32_t>(X.hdr, ((size_t)n + 1) * 4);
  uint32_t* sb = ensure<uint32_t>(X.sb, ((size_t)n + 1) * 4);
  uint32_t* rec = ensure<uint32_t>(X.rec, ((size_t)n + 1) * 4);
  uint32_t* spos = ensure<uint32_t>(X.spos, ((size_t)n + 1) * 4);
  if (n == 0) return L;
  // per line: header flag and sequence bytes; their scans give the record of every line and the offset of its bytes
  line_info_kernel<<<grid, 256, 0, ctx->stream>>>(text, (const uint64_t*)X.nl.p, n, L.fmt, hdr, sb, &tw->err);
  CK(cudaMemsetAsync(hdr + n, 0, 4, ctx->stream));
  CK(cudaMemsetAsync(sb + n, 0, 4, ctx->stream));
  exclusive_sum(ctx, hdr, rec, n + 1);
  exclusive_sum(ctx, sb, spos, n + 1);
  CK(cudaMemcpyAsync(&tw->nrec, rec + n, 4, cudaMemcpyDeviceToDevice, ctx->stream));
  CK(cudaMemcpyAsync(&tw->seq_bytes, spos + n, 4, cudaMemcpyDeviceToDevice, ctx->stream));
  TextWords h;
  CK(cudaMemcpyAsync(&h, tw, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (h.err) fail(SMR_ERR_ARG, h.err & kDecBadHeader ? "reads text: a record does not start with its header character" : "reads text: FASTQ separator line '+' missing");
  L.nrec = h.nrec; L.total_nt = h.seq_bytes;
  return L;
}

// FASTA / FASTQ text -> resident batch (smr_decode.cuh)
// text == nullptr: the text is already in ctx->res.text (inflated on the device), first byte given.  Returns the number of reads.
uint32_t upload_fastx_impl(smr_ctx* ctx, const char* text, uint64_t nbytes, char first_byte = 0) {
  clear_resident(ctx);
  auto& R = ctx->res;
  Batch& b = R.b;
  const auto& X = ctx->tx;
  b.from_text = true; R.text_bytes = nbytes;
  if (nbytes == 0) return 0;
  cudaEvent_t* e = events(ctx, 3);
  CK(cudaEventRecord(e[0], ctx->stream));
  if (text) {
    ensure(R.text, nbytes + 64);
    CK(cudaMemcpyAsync(R.text.p, text, nbytes, cudaMemcpyHostToDevice, ctx->stream));
  }
  CK(cudaEventRecord(e[1], ctx->stream));
  const uint8_t* dt = (const uint8_t*)R.text.p;
  const TextLayout L = text_layout(ctx, dt, nbytes, text ? text[0] : first_byte);
  const uint32_t nreads = L.nrec, total = L.total_nt;
  if (total >= 0xF0000000u) fail(SMR_ERR_ARG, "batch larger than 2^32 nucleotides: split it");
  if (nreads == 0) return 0;
  const int grid = ctx->sm_count * 8;
  TextWords* tw = text_words(ctx);
  ensure(b.seq04, (size_t)total + 64);
  ensure(b.seq_off, (size_t)(nreads + 1) * 4);
  ensure(b.pk_off, (size_t)(nreads + 1) * 4);
  ensure(R.hdroff, (size_t)nreads * 8);
  scatter_lines_kernel<<<grid, 256, 0, ctx->stream>>>(dt, (const uint64_t*)X.nl.p, L.nlines, (const uint32_t*)X.hdr.p, (const uint32_t*)X.rec.p,
                                                       (const uint32_t*)X.sb.p, (const uint32_t*)X.spos.p, (uint8_t*)b.seq04.p,
                                                       (uint32_t*)b.seq_off.p, (uint64_t*)R.hdroff.p);
  CK(cudaMemcpyAsync((uint32_t*)b.seq_off.p + nreads, &tw->seq_bytes, 4, cudaMemcpyDeviceToDevice, ctx->stream));
  // packed-word offsets and the longest read (what read_layout computes on the host); words[nreads] = 0, so pk_off[nreads] is the total
  uint32_t* words = ensure<uint32_t>(ctx->tx.cnt, (size_t)(nreads + 1) * 4);
  uint32_t* pk_off = (uint32_t*)b.pk_off.p;
  CK(cudaMemsetAsync(&tw->max_len, 0, 4, ctx->stream));
  record_words_kernel<<<grid, 256, 0, ctx->stream>>>((const uint32_t*)b.seq_off.p, nreads, words, &tw->max_len);
  exclusive_sum(ctx, words, pk_off, nreads + 1);
  CK(cudaMemcpyAsync(&tw->pk_words, pk_off + nreads, 4, cudaMemcpyDeviceToDevice, ctx->stream));
  ensure(ctx->h.off32, (size_t)(nreads + 1) * 4);
  CK(cudaMemcpyAsync(ctx->h.off32.p, b.seq_off.p, (size_t)(nreads + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream));
  TextWords h;
  CK(cudaMemcpyAsync(&h, tw, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(e[2], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  const uint32_t* off32 = (const uint32_t*)ctx->h.off32.p;
  b.off32.assign(off32, off32 + nreads + 1);
  b.nreads = nreads; b.total_nt = total; b.max_len = h.max_len;
  finish_upload(ctx, b, h.pk_words);
  CK(cudaStreamSynchronize(ctx->stream));
  if (text) ctx->t_h2d = elapsed_ms(e[0], e[1]);
  ctx->t_decode = elapsed_ms(e[1], e[2]);
  return nreads;
}

const char* inf_status_text(uint32_t st) {
  switch (st) {
    case kInfErrCode: return "invalid Huffman code";
    case kInfErrHeader: return "invalid block header";
    case kInfErrOverrun: return "compressed data ends inside a block (truncated file)";
    case kInfErrDistance: return "invalid distance too far back";
    case kInfErrStored: return "invalid stored block lengths";
    case kInfErrMember: return "not a gzip member";
    case kInfErrCrc: return "CRC-32 of a member disagrees with its data";
    case kInfErrSize: return "size field (ISIZE) of a member disagrees with its data";
    default: return "internal error";
  }
}

// distance of the speculative block searches for nbytes of gzip input: 64 KB for large files, down to 8 KB so that a small file
// still makes thousands of spans
uint64_t inflate_chunk(uint64_t nbytes) { return std::min<uint64_t>(65536, std::max<uint64_t>(8192, nbytes / 8192)); }

// One round of the inflate (the five steps of smr_inflate.h) over the compressed bytes gz[0 .. nbytes) (host), from st.at on: the
// output goes to out + at (grown as needed, its first `at` bytes kept).  eof: these bytes end the file; otherwise the round keeps
// what it inflated up to the last block boundary it could reach and st says where the next round resumes.  Returns the bytes
// kept.  The host only walks the list of spans (a few thousand entries) between the COUNT and the WRITE pass.
uint64_t inflate_round(smr_ctx* ctx, const void* gz, uint64_t nbytes, uint64_t chunk_bytes, bool eof, InfStream& st, DevBuf& out, uint64_t at) {
  auto& I = ctx->inf;
  I.spans = I.candidates = 0;
  if (chunk_bytes < 1024) chunk_bytes = 1024;
  cudaEvent_t* e = events(ctx, 3);
  CK(cudaEventRecord(e[0], ctx->stream));
  const size_t padded = (nbytes + 3) / 4 * 4 + 128;
  ensure(I.gz, padded);
  CK(cudaMemsetAsync((uint8_t*)I.gz.p + nbytes / 4 * 4, 0, padded - nbytes / 4 * 4, ctx->stream));
  CK(cudaMemcpyAsync(I.gz.p, gz, nbytes, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaEventRecord(e[1], ctx->stream));
  const uint32_t* w = (const uint32_t*)I.gz.p;
  // FIND
  const uint64_t nchunks = (nbytes + chunk_bytes - 1) / chunk_bytes;
  if (nchunks > (1u << 24)) fail(SMR_ERR_ARG, "gz input: too many chunks");
  std::vector<uint64_t> cand;
  if (nchunks > 1) {
    ensure(I.cand, nchunks * 8);
    inf_find_kernel<<<(unsigned)(nchunks - 1), 256, 0, ctx->stream>>>(w, nbytes, chunk_bytes, (uint64_t*)I.cand.p);
    CK(cudaGetLastError());
    std::vector<uint64_t> raw(nchunks - 1);
    CK(cudaMemcpyAsync(raw.data(), I.cand.p, (nchunks - 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (uint64_t p : raw) if (p != kInfNone && p > st.at.bit) cand.push_back(p);   // chunk order = position order
    if (!cand.empty()) CK(cudaMemcpyAsync(I.cand.p, cand.data(), cand.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  } else ensure(I.cand, 8);
  const uint32_t ncand = (uint32_t)cand.size(), ns = ncand + 1;
  // COUNT
  CK(cudaFuncSetAttribute(inf_span_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kInfSpanSmem));   // per device
  CK(cudaFuncSetAttribute(inf_span_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kInfSpanSmem));
  ensure(I.res, (size_t)ns * sizeof(SpanResult));
  const unsigned ctas = (ns + kInfSpanThreads - 1) / kInfSpanThreads;
  const uint64_t start = st.at.bit, prior = st.carry.len;
  const bool at_member = st.at.at_member;
  inf_span_kernel<false><<<ctas, kInfSpanThreads, kInfSpanSmem, ctx->stream>>>(w, nbytes, start, at_member, prior, (const uint64_t*)I.cand.p, ncand, nullptr, nullptr,
                                                                               nullptr, nullptr, nullptr, ns, nullptr, (SpanResult*)I.res.p);
  CK(cudaGetLastError());
  std::vector<SpanResult> res(ns);
  CK(cudaMemcpyAsync(res.data(), I.res.p, (size_t)ns * sizeof(SpanResult), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  std::vector<uint32_t> real(ns); std::vector<uint64_t> off(ns), cnt(ns), keep(ns);
  uint32_t nreal = 0, why = 0;
  InfResume next;
  const uint64_t total = inf_chain(cand.data(), ncand, res.data(), real.data(), off.data(), nreal, &why, eof, nbytes * 8, at_member, &next);
  if (total == kInfNone) {
    // bytes after the last member that are no member are ignored, as gzip does (a round that resumed at a member's end sees them alone)
    if (at_member && st.members && res[0].status == kInfErrMember) { st.at.eos = true; return 0; }
    fail(SMR_ERR_ARG, std::string("gz input: ") + inf_status_text(why));
  }
  std::vector<uint32_t> moff(nreal + 1, 0);
  for (uint32_t k = 0; k < nreal; ++k) { cnt[k] = res[real[k]].out_n; keep[k] = cnt[k]; moff[k + 1] = moff[k] + res[real[k]].members; }
  keep[nreal - 1] = next.keep_last;
  const uint32_t nmembers = moff[nreal];
  I.spans = nreal; I.candidates = ncand;
  ensure_keep(ctx, out, at + total + 64, at);
  uint8_t* dst = (uint8_t*)out.p + at;
  if (total || (nmembers && st.carry.len)) {
    // WRITE
    uint64_t nsym = 0;
    for (uint32_t k = 0; k < nreal; ++k) nsym = std::max(nsym, off[k] + cnt[k]);
    ensure(I.sym, (nsym + 8) * 2);
    ensure(I.win, (size_t)(nreal + 1) * kInfWindow);
    upload_async(ctx, I.ids, real.data(), nreal);
    upload_async(ctx, I.off, off.data(), nreal);
    upload_async(ctx, I.cnt, cnt.data(), nreal);
    upload_async(ctx, I.moff, moff.data(), nreal + 1);
    ensure(I.mem, (size_t)(nmembers + 1) * sizeof(MemberEnd));
    const uint64_t* d_off = (const uint64_t*)I.off.p;
    const uint64_t* d_cnt = (const uint64_t*)I.cnt.p;
    inf_span_kernel<true><<<(nreal + kInfSpanThreads - 1) / kInfSpanThreads, kInfSpanThreads, kInfSpanSmem, ctx->stream>>>(
        w, nbytes, start, at_member, prior, (const uint64_t*)I.cand.p, ncand, (const uint32_t*)I.ids.p, d_off, d_cnt, (const uint32_t*)I.moff.p,
        (MemberEnd*)I.mem.p, nreal, (uint16_t*)I.sym.p, (SpanResult*)I.res.p);
    CK(cudaGetLastError());
    // WINDOW (seeded with the last 32 KB of the previous round), RESOLVE of the bytes kept
    if (st.have_window) CK(cudaMemcpyAsync(I.win.p, st.win.p, kInfWindow, cudaMemcpyDeviceToDevice, ctx->stream));
    else CK(cudaMemsetAsync(I.win.p, 0, kInfWindow, ctx->stream));
    inf_window_kernel<<<1, 1024, 0, ctx->stream>>>((const uint16_t*)I.sym.p, d_off, d_cnt, nreal, (uint8_t*)I.win.p);
    CK(cudaGetLastError());
    upload_async(ctx, I.cnt, keep.data(), nreal);
    const uint64_t avg = total / nreal + 1;
    const unsigned pieces = (unsigned)std::min<uint64_t>(64, std::max<uint64_t>(1, avg / 8192));
    inf_resolve_kernel<<<dim3(pieces, nreal), 256, 0, ctx->stream>>>((const uint16_t*)I.sym.p, d_off, d_cnt, (const uint8_t*)I.win.p, dst);
    CK(cudaGetLastError());
    std::vector<SpanResult> res2(nreal);
    std::vector<MemberEnd> ends(nmembers);
    CK(cudaMemcpyAsync(res2.data(), I.res.p, (size_t)nreal * sizeof(SpanResult), cudaMemcpyDeviceToHost, ctx->stream));
    if (nmembers) CK(cudaMemcpyAsync(ends.data(), I.mem.p, (size_t)nmembers * sizeof(MemberEnd), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (uint32_t k = 0; k < nreal; ++k) {
      if (res2[k].status != res[real[k]].status || res2[k].out_n != cnt[k] || res2[k].end_bit != res[real[k]].end_bit || res2[k].members != res[real[k]].members)
        fail(SMR_ERR_CUDA, "gz inflate: the write pass disagrees with the count pass");
      for (uint32_t m = moff[k]; m < moff[k + 1]; ++m) ends[m].out_end += off[k];
    }
    // CRC-32 + ISIZE of every member (RFC 1952 2.3.1): pieces on the device, joined here; the open member's part is carried
    std::vector<uint64_t> poff; std::vector<uint32_t> plen, first;
    inf_crc_plan(ends, 32768, poff, plen, first, total);
    const uint32_t npieces = (uint32_t)poff.size();
    std::vector<uint32_t> crcs(npieces);
    if (npieces) {
      upload_async(ctx, I.poff, poff.data(), npieces);
      upload_async(ctx, I.plen, plen.data(), npieces);
      ensure(I.pcrc, (size_t)npieces * 4);
      inf_crc_kernel<<<(npieces + 127) / 128, 128, 0, ctx->stream>>>(dst, (const uint64_t*)I.poff.p, (const uint32_t*)I.plen.p, npieces, (uint32_t*)I.pcrc.p);
      CK(cudaGetLastError());
      CK(cudaMemcpyAsync(crcs.data(), I.pcrc.p, (size_t)npieces * 4, cudaMemcpyDeviceToHost, ctx->stream));
    }
    // the window the next round starts from: the last 32 KB of (previous window, this round's output)
    if (!next.eos) {
      ensure(st.win, kInfWindow);
      ensure(st.win2, kInfWindow);
      if (total >= kInfWindow) CK(cudaMemcpyAsync(st.win.p, dst + total - kInfWindow, kInfWindow, cudaMemcpyDeviceToDevice, ctx->stream));
      else if (total) {
        CK(cudaMemcpyAsync(st.win2.p, (uint8_t*)I.win.p + total, kInfWindow - total, cudaMemcpyDeviceToDevice, ctx->stream));
        CK(cudaMemcpyAsync((uint8_t*)st.win2.p + kInfWindow - total, dst, total, cudaMemcpyDeviceToDevice, ctx->stream));
        std::swap(st.win, st.win2);
      }
      if (total) st.have_window = true;
    }
    CK(cudaEventRecord(e[2], ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (const uint32_t bad = inf_crc_verify(ends, plen, first, crcs.data(), &st.carry)) fail(SMR_ERR_ARG, std::string("gz input: ") + inf_status_text(bad));
  } else {
    CK(cudaEventRecord(e[2], ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  st.members += nmembers;
  st.at = next;
  ctx->t_h2d = elapsed_ms(e[0], e[1]);
  ctx->t_inflate = elapsed_ms(e[1], e[2]);
  return total;
}

// gzip file (host bytes) -> inflated bytes in the resident text, which no batch is decoded from yet; returns their number.  The
// whole file is one round.
uint64_t inflate_impl(smr_ctx* ctx, const void* gz, uint64_t nbytes, uint64_t chunk_bytes) {
  clear_resident(ctx);
  if (nbytes < 18) fail(SMR_ERR_ARG, "gz input: shorter than a gzip header and trailer");
  InfStream st;
  return inflate_round(ctx, gz, nbytes, chunk_bytes, true, st, ctx->res.text, 0);
}

// ---------------------------------------------------------------------------------------------------------------------
// read stream (smr_stream_*): a file pushed piece by piece, counted as the reference counts it and cut into record-aligned batches
// ---------------------------------------------------------------------------------------------------------------------

// the count pass (smr_stream.h) over n bytes of new text at t (device)
void count_text(smr_ctx* ctx, ReadStream& rs, const uint8_t* t, uint64_t n) {
  if (n == 0) return;
  const uint32_t nlines = newline_index(ctx, t, n);
  const uint32_t parts = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)ctx->sm_count * 8, (nlines + 255) / 256));
  const uint32_t per = (uint32_t)(((uint64_t)nlines + parts - 1) / parts + 255) / 256 * 256;
  uint8_t* rc = ensure<uint8_t>(rs.scr.rc, (size_t)(parts + 1) * sizeof(ReadCounts) + 16);
  ReadCounts* part = (ReadCounts*)rc;
  uint64_t* info = (uint64_t*)(rc + (size_t)(parts + 1) * sizeof(ReadCounts));
  count_lines_kernel<<<parts, 256, 0, ctx->stream>>>((const uint64_t*)ctx->tx.nl.p, nlines, n, rs.counts, per, part);
  CK(cudaGetLastError());
  count_fold_kernel<<<1, 1, 0, ctx->stream>>>(part, parts, (const uint64_t*)ctx->tx.nl.p, nlines, n, part + parts, info);
  CK(cudaGetLastError());
  struct { ReadCounts r; uint64_t nl[2]; } h;
  CK(cudaMemcpyAsync(&h.r, part + parts, sizeof(ReadCounts), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(h.nl, info, 16, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  rc_fold(rs.counts, h.r);
  rc_advance(rs.counts, n, h.nl[0], h.nl[1]);
}

// the pending text from [off, n) on, with room for `extra` more bytes after n
void compact_pending(smr_ctx* ctx, StreamSide& sd, uint64_t extra) {
  const uint64_t live = sd.n - sd.off;
  if (sd.off == 0 && sd.text.p && sd.text.cap >= sd.n + extra + 64) return;
  DevBuf nb;
  const uint64_t want = live + extra + 64;
  CK(nb.alloc(want + want / 8 + 256));
  if (live) CK(cudaMemcpyAsync(nb.p, (uint8_t*)sd.text.p + sd.off, live, cudaMemcpyDeviceToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  sd.text = std::move(nb);
  sd.off = 0; sd.n = live;
}

// new text at [from, sd.n): the file's first byte, the count pass; a count-only stream keeps none of it.  A mate stream counts
// nothing (the reference counts the mate files one after another: SMR_STREAM_NEXT_FILE) and checks that both mates are one format.
void took_text(smr_ctx* ctx, ReadStream& rs, StreamSide& sd, uint64_t from) {
  const uint8_t* t = (const uint8_t*)sd.text.p;
  if (sd.n > from && !sd.have_first) {
    CK(cudaMemcpyAsync(&sd.first, t + from, 1, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    sd.have_first = true;
    if (!rs.counts.period) rs.counts.period = sd.first == '@' ? 4 : 2;   // the line cycle of a run's first file holds for all
  }
  if (rs.mates) {
    const StreamSide& m1 = rs.side[0];
    const StreamSide& m2 = rs.side[1];
    if (m1.have_first && m2.have_first && (m1.first == '@') != (m2.first == '@'))
      fail(SMR_ERR_ARG, std::string("mate stream: mate 1 is ") + (m1.first == '@' ? "FASTQ" : "FASTA") + " and mate 2 is " + (m2.first == '@' ? "FASTQ" : "FASTA"));
    return;
  }
  count_text(ctx, rs, t + from, sd.n - from);
  if (rs.count_only) sd.off = sd.n = 0;
}

// the next piece of file `mate` (0 for a single stream, 0 / 1 for mates 1 / 2)
void stream_push_impl(smr_ctx* ctx, uint32_t mate, const uint8_t* bytes, uint64_t n, bool eof) {
  ReadStream& rs = ctx->rs;
  if (!rs.open) fail(SMR_ERR_ARG, "no open read stream: call smr_stream_begin");
  StreamSide& sd = rs.side[mate];
  if (sd.eof) fail(SMR_ERR_ARG, rs.mates ? "mate stream: mate " + std::to_string(mate + 1) + " has ended (eof was pushed)" : "read stream: the file has ended (eof was pushed)");
  sd.eof = eof;
  if (!rs.gz) {
    compact_pending(ctx, sd, n);
    if (n) CK(cudaMemcpyAsync((uint8_t*)sd.text.p + sd.n, bytes, n, cudaMemcpyHostToDevice, ctx->stream));
    const uint64_t from = sd.n;
    sd.n += n;
    took_text(ctx, rs, sd, from);
    return;
  }
  sd.tail.insert(sd.tail.end(), bytes, bytes + n);
  if (sd.inf.at.eos) { sd.tail.clear(); return; }   // bytes after the gzip stream are ignored
  sd.pushed += n;
  const std::string who = rs.mates ? "mate " + std::to_string(mate + 1) + ": " : "";
  if (eof && sd.pushed < 18) fail(SMR_ERR_ARG, who + "gz input: shorter than a gzip header and trailer");
  if (sd.tail.empty() && !eof) return;
  compact_pending(ctx, sd, 0);
  const uint64_t nb = sd.tail.size();
  const uint64_t from = sd.n;
  try {
    sd.n += inflate_round(ctx, sd.tail.data(), nb, inflate_chunk(nb), eof, sd.inf, sd.text, sd.n);
  } catch (Failure& f) {
    f.msg = who + f.msg;
    throw;
  }
  if (sd.inf.at.eos) sd.tail.clear();
  else {
    const uint64_t drop = sd.inf.at.bit / 8;
    sd.tail.erase(sd.tail.begin(), sd.tail.begin() + drop);
    sd.inf.at.bit -= drop * 8;
  }
  took_text(ctx, rs, sd, from);
}

// where the next batch ends in the pending text (bytes from sd.off), or 0 when more text must be pushed first
uint64_t stream_cut(smr_ctx* ctx, ReadStream& rs) {
  StreamSide& sd = rs.side[0];
  const uint64_t avail = sd.n - sd.off, limit = rs.batch_bytes;
  if (avail == 0) return 0;
  if (avail <= limit) return sd.eof ? avail : 0;   // a batch takes whole records up to batch_bytes: wait for more text
  const uint8_t* t = (const uint8_t*)sd.text.p + sd.off;
  unsigned long long* cut = ensure<unsigned long long>(rs.scr.cut, 16);
  uint64_t w = std::min(avail, limit + 1);   // a record end at <= limit is a '\n' before it or a header line starting at it
  for (;;) {
    const uint32_t nl = newline_index(ctx, t, w);
    const unsigned long long init[2] = {0ull, ~0ull};
    CK(cudaMemcpyAsync(cut, init, 16, cudaMemcpyHostToDevice, ctx->stream));
    stream_cut_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(t, (const uint64_t*)ctx->tx.nl.p, nl, w, limit, sd.first == '@' ? kFmtFastq : kFmtFasta, cut);
    CK(cudaGetLastError());
    unsigned long long h[2];
    CK(cudaMemcpyAsync(h, cut, 16, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (h[0]) return h[0];
    if (h[1] != ~0ull) return h[1];   // the first record is longer than a batch: it is the batch
    if (w == avail) return sd.eof ? avail : 0;
    w = std::min(avail, 2 * w);
  }
}

// The record ends of mate m's pending text in its first w bytes, in bytes from its off, to rs.scr.mend[m]; returns their number.
// Once the file has ended and w covers its text, its last record ends at the end of the text, one byte further when the text
// does not end in '\n' (the interleave appends one).
uint32_t mate_ends(smr_ctx* ctx, ReadStream& rs, uint32_t m, uint64_t w) {
  const StreamSide& sd = rs.side[m];
  const uint64_t avail = sd.n - sd.off;
  if (avail == 0) return 0;
  const uint8_t* t = (const uint8_t*)sd.text.p + sd.off;
  const uint32_t fmt = sd.first == '@' ? kFmtFastq : kFmtFasta;
  const uint32_t nl = newline_index(ctx, t, w);
  uint32_t* flag = ensure<uint32_t>(rs.scr.mflag, ((size_t)nl + 1) * 4);
  uint64_t* ends = ensure<uint64_t>(rs.scr.mend[m], ((size_t)nl + 2) * 8);
  const int grid = ctx->sm_count * 8;
  const uint64_t* d_nl = (const uint64_t*)ctx->tx.nl.p;
  if (nl) record_end_flags_kernel<<<grid, 256, 0, ctx->stream>>>(t, d_nl, nl, w, fmt, flag);
  CK(cudaMemsetAsync(flag + nl, 0, 4, ctx->stream));
  exclusive_sum(ctx, flag, flag, nl + 1);
  uint32_t cnt = 0;
  CK(cudaMemcpyAsync(&cnt, flag + nl, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (cnt) record_end_list_kernel<<<grid, 256, 0, ctx->stream>>>(t, d_nl, nl, w, fmt, flag, ends);
  CK(cudaGetLastError());
  if (sd.eof && w == avail) {
    uint64_t last = 0;
    uint8_t c = 0;
    if (cnt) CK(cudaMemcpyAsync(&last, ends + cnt - 1, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(&c, t + avail - 1, 1, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (last < avail) {
      const uint64_t e = avail + (c != '\n');
      CK(cudaMemcpyAsync(ends + cnt, &e, 8, cudaMemcpyHostToDevice, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
      ++cnt;
    }
  }
  return cnt;
}

// The next batch of a mate stream: the k whole pairs whose interleaved text fits in batch_bytes (or the first pair alone when it
// does not fit), interleaved into the resident text.  Returns k; 0 = push more, or (*done) both files are exhausted.  Before both
// files have ended, pairs that fit wait for more text, so that every batch but the last is full.
uint32_t mate_cut(smr_ctx* ctx, ReadStream& rs, uint64_t* nbytes, int* done) {
  StreamSide* sd = rs.side;
  const uint64_t limit = rs.batch_bytes;
  const uint64_t avail[2] = {sd[0].n - sd[0].off, sd[1].n - sd[1].off};
  uint64_t w[2] = {std::min(avail[0], limit + 1), std::min(avail[1], limit + 1)};
  unsigned long long* dk = ensure<unsigned long long>(rs.scr.cut, 16);
  for (;;) {
    uint32_t n[2];
    bool closed[2];   // no more record ends can join the listed ones within batch_bytes: beyond the window, or the file ended
    for (uint32_t m = 0; m < 2; ++m) { n[m] = mate_ends(ctx, rs, m, w[m]); closed[m] = w[m] < avail[m] || sd[m].eof; }
    const uint64_t* ea = (const uint64_t*)rs.scr.mend[0].p;
    const uint64_t* eb = (const uint64_t*)rs.scr.mend[1].p;
    const uint32_t both = std::min(n[0], n[1]);
    if (both) {
      CK(cudaMemsetAsync(dk, 0, 8, ctx->stream));
      mate_fit_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(ea, eb, both, limit, dk);
      CK(cudaGetLastError());
      unsigned long long fit = 0;
      CK(cudaMemcpyAsync(&fit, dk, 8, cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
      uint32_t k = (uint32_t)fit;
      if (k == 0) k = 1;   // the first pair is longer than a batch: it is the batch
      else if (k == both && !(n[0] == k && closed[0]) && !(n[1] == k && closed[1])) return 0;   // pair k + 1 may still fit
      uint64_t end[2];
      CK(cudaMemcpyAsync(&end[0], ea + k - 1, 8, cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaMemcpyAsync(&end[1], eb + k - 1, 8, cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
      *nbytes = end[0] + end[1];
      if (*nbytes >= 0xF0000000ull) fail(SMR_ERR_ARG, "mate stream: one pair of 2^32 bytes or more");
      ensure(ctx->res.text, *nbytes + 64);
      mate_interleave_kernel<<<std::max(1u, std::min<uint32_t>(ctx->sm_count * 16, (k + 7) / 8)), 256, 0, ctx->stream>>>(
          (const uint8_t*)sd[0].text.p + sd[0].off, avail[0], ea, (const uint8_t*)sd[1].text.p + sd[1].off, avail[1], eb, k, (uint8_t*)ctx->res.text.p);
      CK(cudaGetLastError());
      for (uint32_t m = 0; m < 2; ++m) sd[m].off += std::min(end[m], avail[m]);
      return k;
    }
    // a mate without a whole record in its window: it has ended, waits for more text, or its first record is longer than the window
    const bool gone[2] = {sd[0].eof && avail[0] == 0, sd[1].eof && avail[1] == 0};
    if (gone[0] && gone[1]) { *done = 1; return 0; }
    for (uint32_t m = 0; m < 2; ++m)
      if (gone[m] && avail[m ^ 1])
        fail(SMR_ERR_ARG, "mate stream: mate " + std::to_string(m + 1) + " has ended while mate " + std::to_string(2 - m) +
                              " holds more records (the mate files differ in record count)");
    bool grow = false, wait = false;
    for (uint32_t m = 0; m < 2; ++m) {
      if (n[m]) continue;
      if (w[m] < avail[m]) { w[m] = std::min(avail[m], 2 * w[m]); grow = true; }
      else wait = true;
    }
    if (wait || !grow) return 0;
  }
}

uint32_t stream_next_impl(smr_ctx* ctx, int* done) {
  ReadStream& rs = ctx->rs;
  if (!rs.open) fail(SMR_ERR_ARG, "no open read stream: call smr_stream_begin");
  if (rs.count_only) fail(SMR_ERR_ARG, "read stream opened with SMR_STREAM_COUNT_ONLY: it makes no batches");
  if (rs.mates) {
    uint64_t nbytes = 0;
    const uint32_t k = mate_cut(ctx, rs, &nbytes, done);
    if (k == 0) return 0;
    const uint32_t nreads = upload_fastx_impl(ctx, nullptr, nbytes, rs.side[0].first);
    if (nreads != 2 * k) fail(SMR_ERR_ARG, "mate stream: " + std::to_string(k) + " pairs decoded to " + std::to_string(nreads) + " records");
    ctx->res.mates = true;
    return nreads;
  }
  StreamSide& sd = rs.side[0];
  for (;;) {
    *done = sd.eof && sd.n == sd.off;
    const uint64_t cut = stream_cut(ctx, rs);
    if (cut == 0) return 0;
    if (cut >= 0xF0000000ull) fail(SMR_ERR_ARG, "read stream: one record of 2^32 bytes or more");
    ensure(ctx->res.text, cut + 64);
    CK(cudaMemcpyAsync(ctx->res.text.p, (const uint8_t*)sd.text.p + sd.off, cut, cudaMemcpyDeviceToDevice, ctx->stream));
    char c0 = 0;
    CK(cudaMemcpyAsync(&c0, (const uint8_t*)sd.text.p + sd.off, 1, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    sd.off += cut;
    const uint32_t nreads = upload_fastx_impl(ctx, nullptr, cut, c0);
    if (nreads) { *done = 0; return nreads; }
  }
}

// closes the read stream; its scratch stays for the next one
void close_stream(ReadStream& rs) {
  ReadStream::Scratch scr = std::move(rs.scr);
  rs = ReadStream{};
  rs.scr = std::move(scr);
}

// runs f, one call on the open read stream: a stream that fails is closed
template <class F>
void stream_call(smr_ctx* ctx, F&& f) {
  try { f(); } catch (...) { close_stream(ctx->rs); throw; }
}

// Several contexts may share a device (two per GPU let the copies and the host-side result packing of one batch run under the
// kernels of the other).  Their KERNEL sections are serialised: the candidate kernel is persistent and needs every one of its CTAs
// resident at once (planner and scorer warps wait for each other), which two such kernels sharing the SMs could not guarantee.
std::mutex& device_kernel_mutex(int device) {
  static std::mutex m[64];
  return m[device & 63];
}

// All kernels of one pass over a batch; its results and times stay in the batch.  With one group of parts (no index budget, or every
// part within it) each chunk is seeded, searched and finalized in turn.  With several, the run is group-major: each group is uploaded
// into the index arena once, every chunk is seeded and searched over its parts, and every chunk is finalized after the last group.
// The read state carries from group to group as it does from part to part.  Retries and packed re-runs come through here too, and
// upload the groups again.
void run_impl(smr_ctx* ctx, Batch& bt) {
  if (!ctx->have_params) fail(SMR_ERR_ARG, "smr_set_params not called");
  if (ctx->parts.empty()) fail(SMR_ERR_ARG, "no index loaded");
  if (ctx->prm.num_alignments < 0) fail(SMR_ERR_ARG, "num_alignments < 0");
  if (ctx->prm.minoccur != 0) fail(SMR_ERR_UNSUPPORTED, "minoccur != 0 is not supported");
  RunTimes& t = bt.run;
  t = RunTimes{};
  if (&bt == &ctx->res.b) ctx->ib.t_upload = 0;   // a new run of the resident batch; the retries of its download add theirs
  const uint32_t nreads = bt.nreads;
  if (nreads == 0) return;
  const uint32_t slots = slots_of(ctx);
  const uint64_t nslots = batch_slots(ctx, bt, 0, nreads);
  const uint32_t* aln_base = bt.base.empty() ? nullptr : (const uint32_t*)bt.aln_base.p;
  bt.run_slots = slots; bt.run_stats = ctx->host_stats || packed(ctx) || ctx->place_stats; bt.run_id = ++ctx->runs_made;
  std::lock_guard<std::mutex> dev_lock(device_kernel_mutex(ctx->device));   // held until the stream has drained
  auto& A = ctx->run;
  const std::vector<IndexGroup> groups = apply_budget(ctx);
  const uint32_t np = (uint32_t)ctx->parts.size(), ng = (uint32_t)groups.size();
  uint64_t arena_bytes = 0;
  for (const IndexGroup& gr : groups) arena_bytes = std::max(arena_bytes, gr.bytes);
  if (ng > 1 && (ctx->ib.arena.cap < arena_bytes || ctx->ib.arena.cap > ctx->ib.budget)) CK(ctx->ib.arena.alloc(arena_bytes));
  ensure_hit_regions(bt, max_group_parts(ctx));
  // the stride may have grown since the upload sized these (smr_set_aln_slots, then smr_run_resident of the same batch)
  ensure(bt.aln_work, (size_t)nslots * sizeof(AlnWork));
  ensure(bt.out_aln, (size_t)nslots * sizeof(OutAln));
  RunGeom g = setup_arenas(ctx, bt.scale, bt.max_len);
  LisGlobals& lg = g.lg; FinalGlobals& fg = g.fg;
  // device copy of the part tables: [0, np) every part by its ordinal in the context (finalize looks parts up by gslot); with several
  // groups, group k's parts follow from np + first(k), with their ordinals in the group and their search arrays in the arena
  std::vector<DevIndex> hp;
  for (uint32_t i = 0; i < np; ++i) {
    DevIndex d = ctx->parts[i].d; d.slot = d.gslot = (uint16_t)i; d.is_last = (i + 1 == np) ? 1u : 0u;
    hp.push_back(d);
  }
  if (ng > 1)
    for (const IndexGroup& gr : groups)
      for (uint32_t i = gr.first; i < gr.first + gr.n; ++i) {
        DevIndex d = hp[i]; d.slot = (uint16_t)(i - gr.first);
        set_search_ptrs(d, ctx->parts[i], (const uint8_t*)ctx->ib.arena.p + arena_at(ctx, gr, i));
        hp.push_back(d);
      }
  ensure(A.parts, hp.size() * sizeof(DevIndex));
  CK(cudaMemcpyAsync(A.parts.p, hp.data(), hp.size() * sizeof(DevIndex), cudaMemcpyHostToDevice, ctx->stream));
  // cigar pool on the device: generous fixed share per alignment slot
  bt.cigar_cap_dev = nslots * 24 * bt.scale + 4096;
  if (bt.cigar_cap_dev >= 0xFFFFFFFFull) fail(SMR_ERR_CAPACITY, "CIGAR pool of this batch would pass 2^32 words (smr_aln.cigar_off is 32-bit): use smaller batches");
  ensure(bt.cigar_pool, bt.cigar_cap_dev * 4);
  const Scalars sc = scalars_of(bt);
  CK(cudaMemsetAsync(bt.scalars.p, 0, 512, ctx->stream));
  CK(cudaMemsetAsync(bt.counters.p, 0, (size_t)(dcCount + 64) * 8, ctx->stream));
  CK(cudaMemsetAsync(bt.state.p, 0, (size_t)nreads * sizeof(ReadState), ctx->stream));
  CK(cudaMemsetAsync(bt.flags.p, 0, (size_t)nreads * 4, ctx->stream));
  CK(cudaMemsetAsync(bt.hit_db.p, 0xFF, (size_t)nreads * 2, ctx->stream));
  if (ng > 1) CK(cudaMemsetAsync(ensure(A.kept, (size_t)nreads * 4), 0, (size_t)nreads * 4, ctx->stream));
  const DevParams dp = to_dev(ctx->prm);
  lg.aln_work = (AlnWork*)bt.aln_work.p; lg.work_next = sc.lis_next; lg.work_next_b = sc.lis_next_b;
  if (aln_base) lg.aln_base = aln_base; else lg.slots = slots;
  lg.q_head = sc.q_head; lg.q_tail = sc.q_tail; lg.planners_done = sc.planners_done;
  fg.parts = (const DevIndex*)A.parts.p; fg.aln_work = (const AlnWork*)bt.aln_work.p; fg.out = (OutAln*)bt.out_aln.p;
  if (aln_base) fg.aln_base = aln_base; else fg.slots = slots;
  fg.cigar_pool = (uint32_t*)bt.cigar_pool.p; fg.cigar_cap = bt.cigar_cap_dev; fg.cigar_used = sc.cigar_used;
  fg.work_next = sc.fin_next; fg.job_count = sc.fin_jobs;
  // events: [0] start, [1] end; per group k and chunk c from 2 + 5 (k nchunks + c) on: seed, candidate kernel, end of it, and (group 0
  // only) finalize, end of it; then two per group around its upload
  const uint32_t nchunks = (nreads + ctx->chunk_reads - 1) / ctx->chunk_reads;
  cudaEvent_t* e = events(ctx, 2 + 5 * (size_t)nchunks * ng + 2 * (size_t)ng);
  cudaEvent_t* eu = e + 2 + 5 * (size_t)nchunks * ng;
  // seed kernels, bins and the candidate kernel of the parts hp[t0, t0 + tn) over the chunk at c0
  auto candidates = [&](uint32_t t0, uint32_t tn, uint32_t c0, cudaEvent_t* ek) {
    const uint32_t n = std::min(ctx->chunk_reads, nreads - c0);
    DevBatch b = make_batch(bt, c0, n);
    CK(cudaMemsetAsync(sc.work_n, 0, 16, ctx->stream));  // (unused word), the two cursors of the candidate kernel's read schedule, finalize's cursor (zeroed again before it runs)
    CK(cudaMemsetAsync(b.cost, 0, (size_t)n * 4, ctx->stream));
    CK(cudaMemsetAsync(b.bin_count, 0, (size_t)kCostBins * 4, ctx->stream));
    CK(cudaEventRecord(ek[0], ctx->stream));
    ensure(A.seed_ctr, (size_t)tn * 4);
    CK(cudaMemsetAsync(A.seed_ctr.p, 0, (size_t)tn * 4, ctx->stream));   // one work counter per seed launch
    for (uint32_t pi = 0; pi < tn; ++pi) {
      uint32_t* next_read = (uint32_t*)A.seed_ctr.p + pi;
      if (ctx->instr) seed_kernel<true><<<g.seed_ctas, kSeedWarpsPerCta * 32, 0, ctx->stream>>>(hp[t0 + pi], b, dp, (uint32_t*)A.lane_hits.p, g.lane_hits_cap, next_read);
      else seed_kernel<false><<<g.seed_ctas, kSeedWarpsPerCta * 32, 0, ctx->stream>>>(hp[t0 + pi], b, dp, (uint32_t*)A.lane_hits.p, g.lane_hits_cap, next_read);
      CK(cudaGetLastError());
      t.launches += 1;
    }
    bin_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(b);
    CK(cudaGetLastError());
    CK(cudaEventRecord(ek[1], ctx->stream));
    lg.parts = (const DevIndex*)A.parts.p + t0; lg.nparts = tn;
    lis_reset_kernel<<<kQueueCap / 256, 256, 0, ctx->stream>>>(lg, g.lis_warps);
    CK(cudaGetLastError());
    (ctx->instr ? (aln_base ? lis_kernel<true, true> : lis_kernel<true, false>) : (aln_base ? lis_kernel<false, true> : lis_kernel<false, false>))
        <<<g.lis_ctas, kLisWarpsPerCta * 32, kLisSmemBytes, ctx->stream>>>(b, dp, lg);
    CK(cudaGetLastError());
    CK(cudaEventRecord(ek[2], ctx->stream));
    t.launches += 2;
  };
  // finalize the chunk at c0
  auto finalize = [&](uint32_t c0, cudaEvent_t* ek) {
    const uint32_t n = std::min(ctx->chunk_reads, nreads - c0);
    DevBatch b = make_batch(bt, c0, n);
    CK(cudaMemsetAsync(sc.fin_next, 0, 4, ctx->stream));
    CK(cudaMemsetAsync(sc.fin_jobs, 0, 4, ctx->stream));
    CK(cudaEventRecord(ek[3], ctx->stream));
    const uint64_t chunk_slots = batch_slots(ctx, bt, c0, c0 + n);
    fg.jobs = ensure<TraceJob>(A.tb_jobs, (size_t)chunk_slots * sizeof(TraceJob));
    fg.job_list = ensure<uint32_t>(A.fin_list, (size_t)chunk_slots * 4);
    // the packed layout always computes the stats: the caller's pointer only decides whether they are copied
    fg.stats = bt.run_stats ? ensure<AlnStats>(bt.aln_stats, (size_t)nslots * sizeof(AlnStats)) : nullptr;
    const uint32_t jobs_grid = (uint32_t)std::min<uint64_t>((std::max<uint64_t>(chunk_slots, 1) + 255) / 256, (uint64_t)ctx->sm_count * 8);
    (aln_base ? final_jobs_kernel<true> : final_jobs_kernel<false>)<<<jobs_grid, 256, 0, ctx->stream>>>(b, fg);
    CK(cudaGetLastError());
    (aln_base ? finalize_kernel<true> : finalize_kernel<false>)<<<g.final_warps / kFinalWarpsPerCta, kFinalWarpsPerCta * 32, 0, ctx->stream>>>(b, dp, fg);
    CK(cudaGetLastError());
    (aln_base ? traceback_kernel<true> : traceback_kernel<false>)<<<g.tb_threads / 128, 128, 0, ctx->stream>>>(b, dp, fg);
    CK(cudaGetLastError());
    CK(cudaEventRecord(ek[4], ctx->stream));
    t.launches += 3;
  };
  const uint32_t flag_grid = std::min<uint32_t>((nreads + 255) / 256, (uint32_t)ctx->sm_count * 8);
  CK(cudaEventRecord(e[0], ctx->stream));
  if (ng == 1) {
    for (uint32_t c0 = 0, k = 0; c0 < nreads; c0 += ctx->chunk_reads, ++k) {
      candidates(0, np, c0, e + 2 + 5 * k);
      finalize(c0, e + 2 + 5 * k);
    }
  } else {
    for (uint32_t gi = 0; gi < ng; ++gi) {
      const IndexGroup& gr = groups[gi];
      CK(cudaEventRecord(eu[2 * gi], ctx->stream));
      for (uint32_t i = gr.first; i < gr.first + gr.n; ++i) {
        const Part& pt = ctx->parts[i];
        CK(cudaMemcpyAsync((uint8_t*)ctx->ib.arena.p + arena_at(ctx, gr, i), pt.host.p, search_bytes(pt), cudaMemcpyHostToDevice, ctx->stream));
      }
      CK(cudaEventRecord(eu[2 * gi + 1], ctx->stream));
      ctx->ib.uploads += 1; ctx->ib.upload_bytes += gr.bytes;
      for (uint32_t c0 = 0, k = 0; c0 < nreads; c0 += ctx->chunk_reads, ++k) candidates(np + gr.first, gr.n, c0, e + 2 + 5 * ((size_t)gi * nchunks + k));
      group_flags_kernel<<<flag_grid, 256, 0, ctx->stream>>>((uint32_t*)bt.flags.p, (uint32_t*)A.kept.p, nreads, gi + 1 == ng ? 1 : 0);
      CK(cudaGetLastError());
      t.launches += 1;
    }
    for (uint32_t c0 = 0, k = 0; c0 < nreads; c0 += ctx->chunk_reads, ++k) finalize(c0, e + 2 + 5 * k);
  }
  CK(cudaEventRecord(e[1], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  t.total = elapsed_ms(e[0], e[1]);
  for (uint32_t k = 0; k < nchunks * ng; ++k) {
    const cudaEvent_t* ek = e + 2 + 5 * k;
    t.seed += elapsed_ms(ek[0], ek[1]);
    t.lis += elapsed_ms(ek[1], ek[2]);
    if (k < nchunks) t.final += elapsed_ms(ek[3], ek[4]);
  }
  if (ng > 1)
    for (uint32_t gi = 0; gi < ng; ++gi) ctx->ib.t_upload += elapsed_ms(eu[2 * gi], eu[2 * gi + 1]);
  if (getenv("SMR_VERBOSE")) {
    unsigned long long d[16]; cudaMemcpy(d, A.lis_dbg.p, 128, cudaMemcpyDeviceToHost);
    fprintf(stderr, "[smr] slowest read %llu: %.2f ms; cycles vote %llu order %llu group %llu plan %llu wait %llu replay %llu; sw calls %llu, tasks scored %llu, rounds %llu\n", d[10], d[0] / 1.965e6, d[1], d[2], d[3], d[4], d[5], d[6], d[7], d[8], d[9]);
  }
  if (ctx->instr && getenv("SMR_TIMELINE")) {   // ns per role and state in 1 ms buckets since the kernel's start (this run's candidate launches summed)
    std::vector<unsigned long long> tl((size_t)kTlRows * kTlBuckets);
    cudaMemcpy(tl.data(), (const unsigned long long*)A.lis_dbg.p + kTlBase, tl.size() * 8, cudaMemcpyDeviceToHost);
    static const char* names[kTlRows] = {"scorer_wait_ns", "scorer_busy_ns", "planner_wait_ns", "planner_vote_group_ns", "reads_done", "planner_alive_ns"};
    for (int r = 0; r < kTlRows; ++r) {
      int last = 0; for (int k = 0; k < kTlBuckets; ++k) if (tl[(size_t)r * kTlBuckets + k]) last = k + 1;
      fprintf(stderr, "[smr timeline] %s", names[r]);
      for (int k = 0; k < last; ++k) fprintf(stderr, " %llu", tl[(size_t)r * kTlBuckets + k]);
      fprintf(stderr, "\n");
    }
  }
}

// the device counters 1 .. dcCount - 1 are copied to the caller's counters of the same index (download_impl)
static_assert(+dcNumShort == +SMR_CNT_NUM_SHORT && +dcSwCalls == +SMR_CNT_SW_CALLS && +dcSwCells == +SMR_CNT_SW_CELLS &&
                  +dcWindows == +SMR_CNT_WINDOWS && +dcNodes == +SMR_CNT_TRIE_NODES && +dcBuckets == +SMR_CNT_BUCKETS &&
                  +dcEntries == +SMR_CNT_BUCKET_ENTRIES && +dcPosEntries == +SMR_CNT_POS_ENTRIES && +dcLisCalls == +SMR_CNT_LIS_CALLS,
              "DevCnt and the SMR_CNT_* indices disagree");
static_assert(+dcCount <= +SMR_CNT_FIXED, "device counters overlap reads_matched_per_db");

struct HostOut {
  smr_read_result* results; smr_aln* alns; uint32_t* cigar_pool; uint64_t cigar_cap; uint64_t cigar_used;
  uint64_t* counters; uint32_t n_counters;
  bool pool_short = false;   // cigar_cap was exceeded: nothing more is written, cigar_used goes on counting the words the batch needs
};

// a read stored more alignments than the stride (kOvfSlots): the batch needs smr_set_aln_slots(need) (smr_aln_slots_needed)
[[noreturn]] void fail_need_slots(smr_ctx* ctx, uint32_t need, uint32_t slots) {
  ctx->need_slots = need;
  fail(SMR_ERR_CAPACITY, "all-alignments mode: a read stored " + std::to_string(need) + " alignments, the result stride is " +
                             std::to_string(slots) + " (smr_set_aln_slots(" + std::to_string(need) + ") or more, then call again)");
}
const char* const kCigarOffsetMsg = "CIGAR pool offset passes 2^32 words (smr_aln.cigar_off is 32-bit): use smaller batches";
const char* const kTraceErrorMsg = "trace back error (ssw.c:707 is fatal in the reference too)";

// copies the results of a batch's run to the host; returns the reads whose scratch overflowed (rerun_flagged runs them again)
std::vector<PackFlag> download_impl(smr_ctx* ctx, const Batch& b, HostOut& out, const uint32_t* map /*local->caller index or null*/) {
  const uint32_t n = b.nreads;
  std::vector<PackFlag> flagged;
  if (n == 0) return flagged;
  const uint32_t slots = slots_of(ctx);
  cudaEvent_t* e = events(ctx, 2);
  CK(cudaEventRecord(e[0], ctx->stream));
  const ReadState* st = ensure<ReadState>(ctx->h.state, (size_t)n * sizeof(ReadState));
  const uint32_t* fl = ensure<uint32_t>(ctx->h.flags, (size_t)n * 4);
  const uint16_t* hdb = ensure<uint16_t>(ctx->h.hitdb, (size_t)n * 2);
  const OutAln* oa = ensure<OutAln>(ctx->h.outaln, (size_t)n * slots * sizeof(OutAln));
  const AlnStats* ast = nullptr;
  if (ctx->host_stats) {
    ast = ensure<AlnStats>(ctx->h.stats, (size_t)n * slots * sizeof(AlnStats));
    CK(cudaMemcpyAsync(ctx->h.stats.p, b.aln_stats.p, (size_t)n * slots * sizeof(AlnStats), cudaMemcpyDeviceToHost, ctx->stream));
  }
  unsigned long long used = 0;
  std::vector<unsigned long long> cnt(dcCount + 64);
  CK(cudaMemcpyAsync(ctx->h.state.p, b.state.p, (size_t)n * sizeof(ReadState), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(ctx->h.flags.p, b.flags.p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(ctx->h.hitdb.p, b.hit_db.p, (size_t)n * 2, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(ctx->h.outaln.p, b.out_aln.p, (size_t)n * slots * sizeof(OutAln), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(&used, scalars_of(b).cigar_used, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(cnt.data(), b.counters.p, cnt.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  used = std::min<unsigned long long>(used, b.cigar_cap_dev);
  const uint32_t* cig = ensure<uint32_t>(ctx->h.cigar, (size_t)used * 4 + 16);
  if (used) CK(cudaMemcpyAsync(ctx->h.cigar.p, b.cigar_pool.p, used * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(e[1], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->t_d2h += elapsed_ms(e[0], e[1]);
  // a trace back error fails the call after what it can still write; the capacity errors below take precedence
  bool trace_error = false;
  auto fail_on_trace_error = [&] { if (trace_error) fail(SMR_ERR_INDEX, "trace back error (ssw.c:707 is fatal in the reference too)"); };
  // pass 1 (sequential, cheap): flagged reads, cigar offsets in the caller's pool (running sum in read order), counters
  std::vector<uint64_t>& coff = ctx->h.coff; coff.resize((size_t)n + 1);
  uint64_t run = out.cigar_used;
  uint32_t need_slots = 0;
  for (uint32_t r = 0; r < n; ++r) {
    coff[r] = run;
    if (fl[r] & kErrTrace) trace_error = true;
    if (fl[r] & kOvfSlots) { need_slots = std::max(need_slots, st[r].n_align); continue; }   // not retried: the stride is the caller's
    if (fl[r]) { flagged.push_back(PackFlag{r, fl[r], st[r].n_align}); continue; }
    const ReadState& s = st[r];
    for (uint32_t k = 0; k < slots && k < s.n_align; ++k) run += oa[(size_t)r * slots + k].cigar_len;
    if (s.is_hit && out.counters) {
      if (out.n_counters > SMR_CNT_NUM_ALIGNED) out.counters[SMR_CNT_NUM_ALIGNED]++;
      const uint32_t ci = SMR_CNT_FIXED + hdb[r];
      if (hdb[r] != 0xFFFF && ci < out.n_counters) out.counters[ci]++;
    }
  }
  coff[n] = run;
  if (need_slots) fail_need_slots(ctx, need_slots, slots);
  if (run >= 0xFFFFFFFFull) fail(SMR_ERR_CAPACITY, kCigarOffsetMsg);
  out.cigar_used = run;
  // a pool too small fails the call only at its end (download_resident): the flagged reads are still retried, so that
  // cigar_used names every word the batch needs and one larger pool is enough
  if (run > out.cigar_cap) out.pool_short = true;
  if (out.pool_short) { fail_on_trace_error(); return flagged; }
  // pass 2: results, alignments and cigars of disjoint read ranges, by a few host threads for large batches
  auto pack = [&](uint32_t lo, uint32_t hi) {
    for (uint32_t r = lo; r < hi; ++r) {
      if (fl[r]) continue;
      const uint32_t dst = map ? map[r] : r;
      smr_read_result& o = out.results[dst];
      const ReadState& s = st[r];
      o.lastIndex = s.lastIndex; o.lastPart = s.lastPart; o.hit_seeds = s.hit_seeds; o.min_index = s.min_index; o.max_index = s.max_index;
      o.n_align = s.n_align; o.max_SW_count = s.max_SW_count; o.is_done = s.is_done; o.is_hit = s.is_hit;
      uint64_t at = coff[r];
      for (uint32_t k = 0; k < slots; ++k) {
        smr_aln& a = out.alns[(size_t)dst * slots + k];
        memset(&a, 0, sizeof(a));
        if (k >= s.n_align) continue;
        const OutAln& d = oa[(size_t)r * slots + k];
        memcpy(out.cigar_pool + at, cig + d.cigar_off, (size_t)d.cigar_len * 4);
        a.cigar_off = (uint32_t)at; a.cigar_len = d.cigar_len; at += d.cigar_len;
        a.ref_num = d.ref_num; a.ref_begin1 = d.ref_begin1; a.ref_end1 = d.ref_end1; a.read_begin1 = d.read_begin1; a.read_end1 = d.read_end1;
        a.readlen = d.readlen; a.score1 = d.score1; a.part = d.part; a.index_num = d.index_num; a.strand = d.strand;
        if (ctx->host_stats) { const AlnStats& st2 = ast[(size_t)r * slots + k]; ctx->host_stats[(size_t)dst * slots + k] = smr_aln_stats{st2.n_miss, st2.n_gap, st2.n_match, st2.n_match_denovo}; }
      }
    }
  };
  const uint32_t nthr = n >= (1u << 16) ? std::min<uint32_t>(8, std::max<uint32_t>(1, std::thread::hardware_concurrency() / 2)) : 1;
  if (nthr <= 1) pack(0, n);
  else {
    std::vector<std::thread> pool;
    for (uint32_t t = 0; t < nthr; ++t) pool.emplace_back(pack, (uint32_t)((uint64_t)n * t / nthr), (uint32_t)((uint64_t)n * (t + 1) / nthr));
    for (auto& th : pool) th.join();
  }
  // device counter k is the caller's counter k (pinned by the static_asserts at HostOut); dcNumAligned is counted in pass 1
  if (out.counters)
    for (uint32_t k = dcNumShort; k < dcCount && k < out.n_counters; ++k) out.counters[k] += cnt[k];
  fail_on_trace_error();
  return flagged;
}

// The re-run planner.  The reads `fl` that a run of batch `from` flagged (map[k]: the resident batch's index of its read k; null: k)
// run again as batches of their own, gathered from `from` on the device.  Each is handed to consume(batch, its map, exact) once it
// has run, which takes its results and returns the reads it flagged; those are planned the same way.  Reads flagged kOvfSlots alone
// stored more alignments than their room: they run again at their exact count (exact) and the same scale.  Every other flagged read
// overflowed its scratch: it runs again at 8x the scale with room for max(stride, the count it reached), for 3 scales at most.  The
// reads are cut into sub-batches of at most ctx->retry_slots slots (a larger read alone), each run with its own re-runs before the
// next: the order in which the host download writes them and the strided placement scans their CIGARs.  A sub-batch whose reads
// all have room for the stride runs on the strided arenas.  The batch frees itself after its re-runs, but for what consume moves out.
template <class Consume>
void rerun_flagged(smr_ctx* ctx, const Batch& from, const std::vector<PackFlag>& fl, const uint32_t* map, int depth, Consume& consume) {
  const uint32_t S = slots_of(ctx);
  std::vector<uint32_t> idx[2], cap[2];   // [0]: run again for their count, [1]: for their scratch
  for (const PackFlag& f : fl) {
    const int x = f.flags != kOvfSlots;
    idx[x].push_back(f.read); cap[x].push_back(x ? std::max(S, f.n_align) : f.n_align);
    if (x) for (int bit = 0; bit < 6; ++bit) if (f.flags & (1u << bit)) ctx->flag_hist[bit]++;
  }
  if (depth >= 3 && !idx[1].empty()) fail(SMR_ERR_CAPACITY, "scratch overflow persists after 3 retries (" + std::to_string(idx[1].size()) + " reads)");
  for (int x = 0; x < 2; ++x) {
    const std::vector<uint32_t>& I = idx[x];
    const std::vector<uint32_t>& C = cap[x];
    const uint32_t scale = x ? from.scale * 8 : from.scale;
    for (size_t a = 0; a < I.size();) {
      size_t e = a;
      uint64_t total = 0;
      bool strided = true;
      while (e < I.size() && (e == a || total + C[e] <= ctx->retry_slots)) { strided &= C[e] == S; total += C[e++]; }
      if (total >= (1ull << 31)) fail(SMR_ERR_CAPACITY, "a batch run again for its alignment count would hold 2^31 slots or more (a read that stores that many, or SMR_RETRY_SLOTS too large)");
      const uint32_t n = (uint32_t)(e - a);
      if (x && getenv("SMR_VERBOSE")) fprintf(stderr, "[smr] %u reads overflowed their scratch at scale %u: retrying with scale %u (causes so far: lane %llu region %llu pairs %llu trace %llu cigar %llu err %llu)\n", n, from.scale, scale,
          (unsigned long long)ctx->flag_hist[0], (unsigned long long)ctx->flag_hist[1], (unsigned long long)ctx->flag_hist[2], (unsigned long long)ctx->flag_hist[3], (unsigned long long)ctx->flag_hist[4], (unsigned long long)ctx->flag_hist[5]);
      std::vector<uint32_t> src(n), bmap(n);
      for (uint32_t k = 0; k < n; ++k) { src[k] = from.off32[I[a + k]]; bmap[k] = map ? map[I[a + k]] : I[a + k]; }
      Batch b;
      b.scale = scale;
      if (!strided) {
        b.base.resize((size_t)n + 1, 0);
        for (uint32_t k = 0; k < n; ++k) b.base[k + 1] = b.base[k] + C[a + k];
      }
      const uint64_t w = read_layout(ctx, b, n, [&](uint32_t k) { return from.off32[I[a + k] + 1] - src[k]; });
      DevBuf d_src;
      upload_async(ctx, d_src, src.data(), n);
      ensure(b.seq04, b.total_nt + 64);
      gather_reads_kernel<<<std::min<uint32_t>((n + 7) / 8, (uint32_t)ctx->sm_count * 8), 256, 0, ctx->stream>>>(
          (const uint8_t*)from.seq04.p, (const uint32_t*)d_src.p, n, (const uint32_t*)b.seq_off.p, (uint8_t*)b.seq04.p);
      CK(cudaGetLastError());
      finish_upload(ctx, b, w);
      run_impl(ctx, b);
      ctx->t_run += b.run;
      const std::vector<PackFlag> again = consume(b, bmap.data(), x == 0);
      rerun_flagged(ctx, b, again, bmap.data(), depth + x, consume);
      a = e;
    }
  }
}

// the arenas grow with a retry's scale (after 64x, tens of GB): the next run allocates them again at its own, whether the retry
// succeeds or not
void release_retry_arenas(smr_ctx* ctx) { for (DevBuf* s : {&ctx->run.lis, &ctx->run.fin, &ctx->run.tb, &ctx->run.lane_hits}) s->reset(); }

// the results of the resident batch's last run into the caller's arrays, its flagged reads retried; the resident batch and its
// device results stay as they are
void download_resident(smr_ctx* ctx, HostOut& out) {
  ctx->t_run = ctx->res.b.run; ctx->t_d2h = 0;
  const std::vector<PackFlag> flagged = download_impl(ctx, ctx->res.b, out, nullptr);
  if (!flagged.empty()) {
    const auto release = on_exit([ctx] { release_retry_arenas(ctx); });
    auto consume = [&](const Batch& b, const uint32_t* map, bool) { return download_impl(ctx, b, out, map); };
    rerun_flagged(ctx, ctx->res.b, flagged, nullptr, 0, consume);
  }
  // the caller's CIGAR pool was too small: *cigar_used names the words the batch needs
  if (out.pool_short)
    fail(SMR_ERR_CAPACITY, "cigar pool too small: the batch needs " + std::to_string(out.cigar_used) + " words, cigar_cap is " + std::to_string(out.cigar_cap));
}

// ---------------------------------------------------------------------------------------------------------------------
// device placement (smr_place_results, smr_place_results_packed, smr_place.cuh): the final results of the resident batch's last
// run kept on the device, in the bytes the host download of its layout writes (smr_download_results,
// smr_download_results_packed)
// ---------------------------------------------------------------------------------------------------------------------
// the counters a placement keeps: SMR_CNT_FIXED + one reads_matched_per_db entry per index
uint32_t place_counters(const smr_ctx* ctx) { return SMR_CNT_FIXED + std::max(1u, ctx->n_index_files); }

// the placed arrays, as the report-side calls take them
struct PlacedArrays {
  const smr_read_result* res; const smr_aln* aln; const uint32_t* cig; uint64_t cig_words; const smr_aln_stats* st; uint32_t n;
  uint64_t nslots;   // the alignment rows: n * stride, or packed the sum of n_align
};

// The placed results of the resident batch's last run for the _placed call `call`; need_stats: the call reads the stats.
PlacedArrays placed_of(const smr_ctx* ctx, const char* call, bool need_stats) {
  const auto& P = ctx->pl;
  if (P.run_id == 0 || P.run_id != ctx->res.b.run_id || P.packed != packed(ctx)) {
    if (packed(ctx))
      fail(SMR_ERR_UNSUPPORTED, std::string(call) + ": no placed results of the resident batch's last run in the packed layout "
                                "(smr_place_results places the strided layout only): call smr_place_results_packed after smr_run_resident, "
                                "or download them (smr_download_results_packed) and pass them to the call that takes result arrays");
    fail(SMR_ERR_ARG, std::string(call) + ": no placed results of the resident batch's last run: call smr_place_results after smr_run_resident");
  }
  if (P.trace) fail(SMR_ERR_INDEX, kTraceErrorMsg);
  if (!P.packed && P.slots != slots_of(ctx)) fail(SMR_ERR_ARG, std::string(call) + ": the results were placed at another stride");
  if (need_stats && !P.stats)
    fail(SMR_ERR_ARG, std::string(call) + ": the placed run computed no smr_aln_stats: call smr_set_place_stats(ctx, 1) before smr_run_resident");
  return PlacedArrays{(const smr_read_result*)P.res.p, (const smr_aln*)P.aln.p, (const uint32_t*)P.cig.p, P.cig_words,
                      P.stats ? (const smr_aln_stats*)P.st.p : nullptr, P.nreads, P.n_alns};
}

// The result buffers of a re-run sub-batch, kept on the device until the scatter; the rest of its batch (reads, seed scratch,
// candidate work) frees itself when its re-runs are done, and the context's arenas are released after the last one.
struct KeptRun { DevBuf state, hit_db, out_aln, aln_stats, cigar_pool, counters, aln_base; };

// The runs of a placement: runs[0] is the resident batch's first run, runs[k] the re-run whose buffers are kept[k - 1].
// ctx->pl.src names, per read of the resident batch, the run and the read in it that hold its final results.
struct PlaceRuns {
  std::deque<KeptRun> kept;
  std::vector<PackRun> runs;
  uint32_t reads = 0;          // the reads of all runs (the run-order CIGAR scan has one entry per read of each run)
  bool trace_error = false;
  uint64_t slot_reads = 0, slot_batches = 0; uint32_t slot_max = 0;   // re-runs for the alignment count (SMR_VERBOSE)
};

// a run as the placement reads it (its buffers stay where the run left them); first: its read 0's entry in the run-order scan
PackRun pack_run_of(const Batch& b, uint32_t first) {
  return PackRun{(const ReadState*)b.state.p, (const uint16_t*)b.hit_db.p, (const OutAln*)b.out_aln.p, (const AlnStats*)b.aln_stats.p,
                 (const uint32_t*)b.cigar_pool.p, b.base.empty() ? nullptr : (const uint32_t*)b.aln_base.p,
                 (const unsigned long long*)b.counters.p, b.run_slots, first};
}

// the reads of a run that carry a flag, in read order: a compaction of its flags on the device (a scan of one bit per read), of
// which only the read index, the flags and n_align come to the host
std::vector<PackFlag> flagged_reads(smr_ctx* ctx, const Batch& b) {
  auto& P = ctx->pl;
  const uint32_t n = b.nreads;
  const uint32_t* flags = (const uint32_t*)b.flags.p;
  uint32_t* bit = ensure<uint32_t>(P.fsel, ((size_t)n + 1) * 4);
  uint32_t* pos = ensure<uint32_t>(P.scal, ((size_t)n + 1) * 4);
  PackFlag* out = ensure<PackFlag>(P.fout, (size_t)n * sizeof(PackFlag) + 16);
  const uint32_t grid = std::min<uint32_t>((n + 256) / 256, (uint32_t)ctx->sm_count * 8);
  pack_flag_bits_kernel<<<grid, 256, 0, ctx->stream>>>(flags, n, bit);
  CK(cudaGetLastError());
  exclusive_sum(ctx, bit, pos, n + 1);
  pack_flagged_kernel<<<grid, 256, 0, ctx->stream>>>(flags, (const ReadState*)b.state.p, n, pos, out);
  CK(cudaGetLastError());
  uint32_t m = 0;
  CK(cudaMemcpyAsync(&m, pos + n, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  std::vector<PackFlag> h(m);
  if (m) {
    CK(cudaMemcpyAsync(h.data(), out, (size_t)m * sizeof(PackFlag), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  return h;
}

// The results of the resident batch's last run, placed on the device in ctx->pl: the first run's results, and the flagged reads
// run again by rerun_flagged, whose result buffers stay on the device; then every read placed from the run that completed it
// (smr_place.cuh: a count pass over each read's source run, two scans, a group of lanes per read to scatter).  In the strided layout, as the
// host download: a read flagged kOvfSlots fails the call with SMR_ERR_CAPACITY (smr_aln_slots_needed) and a trace back error with
// SMR_ERR_INDEX, before anything is placed; in the packed layout a trace back error fails each call that reads the placement.  The
// re-runs compute the stats when the first run did, whatever smr_set_place_stats says now.  The resident batch and its device
// results stay as they are.
void place(smr_ctx* ctx) {
  auto& P = ctx->pl;
  const Batch& R = ctx->res.b;
  const bool pk = packed(ctx);
  const uint32_t n = R.nreads, S = slots_of(ctx), ncnt = place_counters(ctx), stride = pk ? 0 : S;
  P.run_id = 0;
  P.nreads = n; P.slots = S; P.stats = R.run_stats; P.packed = pk; P.trace = false; P.cig_words = 0; P.n_alns = 0; P.t_place = 0;
  P.cnt_host.assign(ncnt, 0);
  ctx->t_run = R.run; ctx->t_d2h = 0;
  if (n == 0) { P.t_run = ctx->t_run; P.run_id = R.run_id; return; }
  const bool keep = ctx->place_stats;
  const auto restore = on_exit([ctx, keep] { ctx->place_stats = keep; });
  ctx->place_stats = P.stats;
  const uint32_t grid = std::min<uint32_t>((n + 255) / 256, (uint32_t)ctx->sm_count * 8);
  uint2* src = ensure<uint2>(P.src, (size_t)n * sizeof(uint2) + 16);
  pack_src_init_kernel<<<grid, 256, 0, ctx->stream>>>(src, n);
  CK(cudaGetLastError());
  PlaceRuns K;
  auto take = [&](const Batch& b, const std::vector<PackFlag>& fl) {   // b is run K.runs.size()
    uint32_t need = 0;
    for (const PackFlag& f : fl) {
      if (f.flags & kErrTrace) K.trace_error = true;
      if (!pk && (f.flags & kOvfSlots)) need = std::max(need, f.n_align);
    }
    if (need) fail_need_slots(ctx, need, S);
    if (!pk && K.trace_error) fail(SMR_ERR_INDEX, kTraceErrorMsg);
    K.runs.push_back(pack_run_of(b, K.reads));
    K.reads += b.nreads;
  };
  const std::vector<PackFlag> flagged = flagged_reads(ctx, R);
  take(R, flagged);
  auto consume = [&](Batch& b, const uint32_t* map, bool exact) {
    const uint32_t m = b.nreads;
    DevBuf d_map;
    upload_async(ctx, d_map, map, m);
    pack_src_kernel<<<std::min<uint32_t>((m + 255) / 256, (uint32_t)ctx->sm_count * 8), 256, 0, ctx->stream>>>(
        (const uint32_t*)b.flags.p, (const uint32_t*)d_map.p, m, (uint32_t)K.runs.size(), src);
    CK(cudaGetLastError());
    std::vector<PackFlag> fl = flagged_reads(ctx, b);   // synchronises: d_map may free
    take(b, fl);
    if (exact) {
      K.slot_reads += m; K.slot_batches += 1;
      for (uint32_t k = 0; k < m; ++k) K.slot_max = std::max(K.slot_max, b.base[k + 1] - b.base[k]);
    }
    KeptRun& k = K.kept.emplace_back();
    k.state = std::move(b.state); k.hit_db = std::move(b.hit_db); k.out_aln = std::move(b.out_aln); k.aln_stats = std::move(b.aln_stats);
    k.cigar_pool = std::move(b.cigar_pool); k.counters = std::move(b.counters); k.aln_base = std::move(b.aln_base);
    return fl;
  };
  if (!flagged.empty()) {
    const auto release = on_exit([ctx] { release_retry_arenas(ctx); });
    rerun_flagged(ctx, R, flagged, nullptr, 0, consume);
  }
  if (K.slot_reads && getenv("SMR_VERBOSE"))
    fprintf(stderr, "[smr] packed results: %llu reads stored more than %u alignments and were run again at their own count in %llu sub-batches (largest count %u)\n",
            (unsigned long long)K.slot_reads, S, (unsigned long long)K.slot_batches, K.slot_max);
  // count, scan, scatter; the CIGAR words in read order (packed) or in run order (strided: one entry per read of each run)
  const uint32_t nruns = (uint32_t)K.runs.size(), nw = pk ? n : K.reads;
  upload_async(ctx, P.runs, K.runs.data(), nruns);
  uint64_t* nal = ensure<uint64_t>(P.nal, ((size_t)n + 1) * 8);
  uint64_t* words = ensure<uint64_t>(P.words, ((size_t)nw + 1) * 8);
  uint64_t* aoff = ensure<uint64_t>(P.aoff, ((size_t)n + 1) * 8);
  uint64_t* off = ensure<uint64_t>(P.off, ((size_t)nw + 1) * 8);
  ensure(P.cnt, (size_t)ncnt * 8);
  cudaEvent_t* e = events(ctx, 2);
  CK(cudaEventRecord(e[0], ctx->stream));
  CK(cudaMemsetAsync(P.cnt.p, 0, (size_t)ncnt * 8, ctx->stream));
  if (!pk) CK(cudaMemsetAsync(words, 0, ((size_t)nw + 1) * 8, ctx->stream));
  pack_count_kernel<<<grid, 256, (size_t)ncnt * 8, ctx->stream>>>((const PackRun*)P.runs.p, nruns, src, n, stride, nal, words, (unsigned long long*)P.cnt.p, ncnt);
  CK(cudaGetLastError());
  cub_run(ctx->cub_tmp, [&](void* t, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(t, bytes, nal, aoff, (int)(n + 1), ctx->stream); });
  cub_run(ctx->cub_tmp, [&](void* t, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(t, bytes, words, off, (int)(nw + 1), ctx->stream); });
  uint64_t tot[2] = {0, 0};
  CK(cudaMemcpyAsync(&tot[0], aoff + n, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(&tot[1], off + nw, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (tot[1] >= 0xFFFFFFFFull) fail(SMR_ERR_CAPACITY, kCigarOffsetMsg);
  ensure(P.res, (size_t)n * sizeof(smr_read_result) + 16);
  ensure(P.aln, tot[0] * sizeof(smr_aln) + 16);
  if (P.stats) ensure(P.st, tot[0] * sizeof(smr_aln_stats) + 16);
  ensure(P.cig, tot[1] * 4 + 16);
  const PackOut o{(smr_read_result*)P.res.p, (smr_aln*)P.aln.p, P.stats ? (smr_aln_stats*)P.st.p : nullptr, (uint32_t*)P.cig.p, aoff, off};
  uint32_t lg = 5;   // 2^lg lanes per read: a warp when packed, the stride rounded up to a power of two when strided
  if (stride) for (lg = 0; (1u << lg) < stride && lg < 5; ++lg) {}
  const uint32_t per_block = 8u << (5 - lg);
  pack_scatter_kernel<<<std::min<uint32_t>((n + per_block - 1) / per_block, (uint32_t)ctx->sm_count * 16), 256, 0, ctx->stream>>>(
      (const PackRun*)P.runs.p, src, n, stride, lg, o);
  CK(cudaGetLastError());
  CK(cudaEventRecord(e[1], ctx->stream));
  CK(cudaMemcpyAsync(P.cnt_host.data(), P.cnt.p, (size_t)ncnt * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));   // before the kept runs free themselves
  P.t_place = elapsed_ms(e[0], e[1]);
  P.n_alns = tot[0]; P.cig_words = tot[1]; P.trace = K.trace_error; P.t_run = ctx->t_run;
  P.run_id = R.run_id;
}

// The placement of the resident batch's last run in the context's layout (once per run: a later call finds it placed).  `call`
// names the entry point in its refusals.
void place_once(smr_ctx* ctx, const char* call) {
  const Batch& R = ctx->res.b;
  if (R.run_id == 0) fail(SMR_ERR_ARG, std::string(call) + ": the resident batch has not been run (smr_run_resident)");
  if (packed(ctx) && (!R.run_stats || R.run_slots != slots_of(ctx)))
    fail(SMR_ERR_ARG, "the resident batch was not run in the packed layout at this stride: call smr_run_resident again");
  if (R.run_slots != slots_of(ctx)) fail(SMR_ERR_ARG, std::string(call) + ": the resident batch was run at another stride: call smr_run_resident again");
  const auto& P = ctx->pl;
  if (P.run_id == R.run_id && P.packed == packed(ctx)) { ctx->t_run = P.t_run; return; }
  place(ctx);
}

struct PackedOut {
  smr_read_result* results; smr_aln* alns; uint64_t aln_cap; smr_aln_stats* stats; uint32_t* cigar_pool; uint64_t cigar_cap;
  uint64_t* counters; uint32_t n_counters;
  uint64_t aln_used = 0, cigar_used = 0;
};

// The packed download of the resident batch's last run: placed on the device once per run (place_once), then copied.  Both sizes
// are set before a capacity check can fail, and a call with arrays that large writes the same bytes.
void download_packed(smr_ctx* ctx, PackedOut& out) {
  const Batch& R = ctx->res.b;
  ctx->t_run = R.run;
  if (R.nreads == 0) return;
  place_once(ctx, "smr_download_results_packed");
  const auto& P = ctx->pl;
  out.aln_used = P.n_alns; out.cigar_used = P.cig_words;
  if (out.aln_used > out.aln_cap)
    fail(SMR_ERR_CAPACITY, "alignment array too small: the batch stores " + std::to_string(out.aln_used) + " alignments, aln_cap is " + std::to_string(out.aln_cap));
  if (out.cigar_used > out.cigar_cap)
    fail(SMR_ERR_CAPACITY, "cigar pool too small: the batch needs " + std::to_string(out.cigar_used) + " words, cigar_cap is " + std::to_string(out.cigar_cap));
  cudaEvent_t* e = events(ctx, 2);
  CK(cudaEventRecord(e[0], ctx->stream));
  CK(cudaMemcpyAsync(out.results, P.res.p, (size_t)P.nreads * sizeof(smr_read_result), cudaMemcpyDeviceToHost, ctx->stream));
  if (P.n_alns) CK(cudaMemcpyAsync(out.alns, P.aln.p, P.n_alns * sizeof(smr_aln), cudaMemcpyDeviceToHost, ctx->stream));
  if (out.stats && P.n_alns) CK(cudaMemcpyAsync(out.stats, P.st.p, P.n_alns * sizeof(smr_aln_stats), cudaMemcpyDeviceToHost, ctx->stream));
  if (P.cig_words) CK(cudaMemcpyAsync(out.cigar_pool, P.cig.p, P.cig_words * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(e[1], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->t_d2h = elapsed_ms(e[0], e[1]);
  if (out.counters)
    for (uint32_t k = 0; k < out.n_counters && k < P.cnt_host.size(); ++k) out.counters[k] += P.cnt_host[k];
  if (P.trace) fail(SMR_ERR_INDEX, kTraceErrorMsg);
}

// ---------------------------------------------------------------------------------------------------------------------
// report writer (smr_report.cuh)
// ---------------------------------------------------------------------------------------------------------------------
// fails with the text of the report error bits e (RptArgs::err), if any
void rpt_check(uint32_t e) {
  if (!e) return;
  fail(SMR_ERR_ARG, e & kRptErrLen ? "an alignment's readlen or read_end1 disagrees with the length of its read in the text"
                    : e & kRptErrGroup ? "an alignment names an (index, part) that is not loaded"
                    : e & kRptErrRef ? "an alignment's ref_num is beyond the reference names of its part"
                    : e & kRptErrQual ? "reads text: a FASTQ record without its quality line"
                    : e & kRptErrCigar ? "an alignment's CIGAR lies outside cigar_words" : "an alignment's CIGAR runs past its read or its reference");
}

// fails with the text of the BAM error bits of e, naming the batch's read `bad`, if any
void rpt_check_bam(uint32_t e, uint32_t bad) {
  const uint32_t b = e & (kRptErrBamName | kRptErrBamQualLen | kRptErrBamQualByte);
  if (b)
    fail(SMR_ERR_ARG, "BAM: read " + std::to_string(bad) + " of the batch " +
                      (b & kRptErrBamName ? "has a QNAME longer than 254 bytes"
                       : b & kRptErrBamQualLen ? "has a quality line whose length differs from its sequence's"
                                               : "has a quality byte outside '!'..'~'"));
}

// A report-side call's checks of its batch: the arrays (stats_msg: stats are read, the text if missing; arrays_msg: the text of
// missing results or alns, stats_msg if null), an even read count when paired (mates 2k, 2k+1), fewer than 2^31 result slots.
void rpt_check_batch(const smr_ctx* ctx, const char* what, const smr_read_result* results, const smr_aln* alns, const smr_aln_stats* stats,
                     uint32_t nreads, bool paired, const char* stats_msg, const char* arrays_msg = nullptr, bool dev = false) {
  if (nreads && stats_msg && !stats) fail(SMR_ERR_ARG, stats_msg);
  if (nreads && (!results || !alns)) fail(SMR_ERR_ARG, arrays_msg ? arrays_msg : stats_msg);
  if (paired && (nreads & 1u)) fail(SMR_ERR_ARG, "a paired batch holds mates 2k and 2k+1: the number of reads must be even");
  if (result_slots(ctx, results, nreads, dev) >= (1ull << 31)) fail(SMR_ERR_ARG, std::string("batch too large for ") + what + ": split it");
}

// the loaded (index, part)s in the reference's report order (index, then part)
std::vector<const Part*> report_groups(const smr_ctx* ctx) {
  std::vector<const Part*> gp;
  for (const Part& pt : ctx->parts) gp.push_back(&pt);
  std::sort(gp.begin(), gp.end(), [](const Part* a, const Part* b) { return a->d.index_num != b->d.index_num ? a->d.index_num < b->d.index_num : a->d.part < b->d.part; });
  return gp;
}

// The RptGroup table of the loaded (index, part)s in report order.  names / scoring: the caller prints reference ids
// (smr_set_report_refs) / E-values and bit scores (smr_set_report_scoring), which every group must then have.
std::vector<RptGroup> rpt_groups(const smr_ctx* ctx, bool names, bool scoring) {
  std::vector<RptGroup> hg;
  uint32_t ref_base = 0;   // the refIDs of BAM: the references of every group in this order, one after another (smr_bam_header)
  for (const Part* pt : report_groups(ctx)) {
    const uint32_t ix = pt->d.index_num;
    if (names && !pt->has_rnames)
      fail(SMR_ERR_ARG, "smr_set_report_refs was not called for index " + std::to_string(ix) + " part " + std::to_string(pt->d.part));
    const smr_ctx::RptScore* sc = ix < ctx->rpt_score.size() && ctx->rpt_score[ix].set ? &ctx->rpt_score[ix] : nullptr;
    if (scoring && !sc) fail(SMR_ERR_ARG, "smr_set_report_scoring was not called for index " + std::to_string(ix));
    hg.push_back(RptGroup{pt->rnames, pt->rname_off, sc ? (const double*)sc->ev.p : nullptr, sc ? (const uint32_t*)sc->bits.p : nullptr, pt->n_rnames,
                          ix, pt->d.part, ref_base, pt->d.refseq, pt->d.ref_off});
    ref_base += pt->d.nref;
  }
  return hg;
}

// The first half of a report-side call, after rpt_check_batch: text, results and groups on the device (e[0] recorded before the
// copies, e[1] after them), the record layout of the text (text_layout, then rpt_records_kernel); returns the report arguments.
// Their error word (err) is zeroed here; the caller reads it back with its results and passes it to rpt_check.  dev: results,
// alns, cigar and stats are the placed device arrays (placed_of), read where they are instead of uploaded.
RptArgs rpt_prologue(smr_ctx* ctx, const char* text, uint64_t nbytes, const smr_read_result* results, const smr_aln* alns, const uint32_t* cigar,
                     uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads, const std::vector<RptGroup>& hg, const cudaEvent_t* e,
                     bool dev = false) {
  auto& S = ctx->r;
  CK(cudaEventRecord(e[0], ctx->stream));
  const uint32_t slots = slots_of(ctx), G = (uint32_t)hg.size();
  const uint64_t N = result_slots(ctx, results, nreads, dev);
  // the text
  const uint8_t* dt;
  if (text) {
    upload_async(ctx, S.text, (const uint8_t*)text, nbytes);
    dt = (const uint8_t*)S.text.p;
  } else {
    if (!ctx->res.text_bytes) fail(SMR_ERR_ARG, "no resident text: smr_upload_fastx[_gz] was not called, or pass the text");
    nbytes = ctx->res.text_bytes;
    dt = (const uint8_t*)ctx->res.text.p;
  }
  char c0 = 0;
  if (nbytes) { if (text) c0 = text[0]; else CK(cudaMemcpy(&c0, dt, 1, cudaMemcpyDeviceToHost)); }
  // results
  if (!dev) {
    upload_async(ctx, S.res, results, nreads);
    upload_async(ctx, S.aln, alns, N);
    upload_async(ctx, S.cig, cigar, cigar ? cigar_words : 0);
    upload_async(ctx, S.st, stats, stats ? N : 0);
  }
  upload_async(ctx, S.grp, hg.data(), G);
  CK(cudaEventRecord(e[1], ctx->stream));
  const TextLayout L = text_layout(ctx, dt, nbytes, c0);
  if (L.nrec != nreads) fail(SMR_ERR_ARG, "the text holds " + std::to_string(L.nrec) + " records, the results " + std::to_string(nreads) + " reads");
  // per record
  const uint64_t fstride = (uint64_t)nreads + 1;
  ensure(S.line, fstride * 4);
  ensure(S.recs, fstride * sizeof(RptRec));
  const auto& X = ctx->tx;
  RptArgs a{};
  a.text = dt; a.nbytes = nbytes; a.nl = (const uint64_t*)X.nl.p; a.spos = (const uint32_t*)X.spos.p; a.nlines = L.nlines; a.fastq = L.fmt == kFmtFastq;
  a.rec = (const RptRec*)S.recs.p; a.nreads = nreads; a.slots = slots; a.nslots = N;
  a.res = (const smr_read_result*)S.res.p; a.aln = (const smr_aln*)S.aln.p; a.cigar = (const uint32_t*)S.cig.p;
  a.cigar_words = cigar ? cigar_words : 0; a.st = (const smr_aln_stats*)S.st.p;
  if (dev) {   // a call without stats still gets a readable array, as an upload of none leaves one
    a.res = results; a.aln = alns; a.cigar = cigar;
    a.st = stats ? stats : ensure<smr_aln_stats>(S.st, 16);
  }
  a.grp = (const RptGroup*)S.grp.p; a.ngroups = G; a.err = &text_words(ctx)->rpt_err;
  CK(cudaMemsetAsync(a.err, 0, 4, ctx->stream));
  if (nreads) {
    const int grid = ctx->sm_count * 8;
    rpt_header_lines_kernel<<<grid, 256, 0, ctx->stream>>>((const uint32_t*)X.hdr.p, (const uint32_t*)X.rec.p, L.nlines, (uint32_t*)S.line.p);
    rpt_records_kernel<<<grid, 256, 0, ctx->stream>>>(a, (const uint32_t*)S.line.p, (RptRec*)S.recs.p);
    if (packed(ctx)) {   // where each read's alignments start, and the read of each slot
      uint32_t* aoff = ensure<uint32_t>(S.aoff, fstride * 4);
      rpt_counts_kernel<<<grid, 256, 0, ctx->stream>>>(a.res, nreads, aoff);
      exclusive_sum(ctx, aoff, aoff, nreads + 1);
      a.aln_off = aoff;
      a.slot_read = ensure<uint32_t>(S.sread, (N + 1) * 4);
      rpt_slot_read_kernel<<<grid, 256, 0, ctx->stream>>>(a.res, nreads, aoff, (uint32_t*)a.slot_read);
    }
    CK(cudaGetLastError());
  }
  return a;
}

// the report timings (smr_last_report_timings) from the four events of a call: the upload, the device work, the download
void set_rpt_times(smr_ctx* ctx, const cudaEvent_t* e) { for (int k = 0; k < 3; ++k) ctx->t_rpt[k] = elapsed_ms(e[k], e[k + 1]); }

// ---------------------------------------------------------------------------------------------------------------------
// gzip deflate (smr_deflate.cuh)
// ---------------------------------------------------------------------------------------------------------------------
// The streams [sb[k], se[k]) of the device bytes `in` (padded by >= 8 readable bytes), each non-empty one compressed to one gzip
// member, into the host buffer `out` one after another; so[0 .. ns] = their offsets.  If the members do not fit in cap, fails with
// SMR_ERR_CAPACITY with so filled (a retry gives the same bytes).  e_dev is recorded before the D2H, e_end after it.  hlen:
// kGzHeader, zlib's gzip header; kBgzfHeader, the BGZF header with each member's BSIZE (the caller cuts the BGZF blocks).
void gzip_streams(smr_ctx* ctx, const uint8_t* in, const std::vector<uint64_t>& sb, const std::vector<uint64_t>& se, char* out, uint64_t cap,
                  uint64_t* so, cudaEvent_t e_dev, cudaEvent_t e_end, uint32_t hlen = kGzHeader) {
  auto& Z = ctx->z;
  const uint32_t ns = (uint32_t)sb.size();
  std::vector<DefChunk> ch;
  def_plan(sb.data(), se.data(), ns, ch);
  const uint32_t nch = (uint32_t)ch.size();
  std::vector<DefInfo> info(nch);
  std::vector<uint32_t> crcs(nch);
  if (nch) {
    const uint64_t end = se[ns - 1];
    std::vector<uint64_t> poff(nch); std::vector<uint32_t> plen(nch);
    for (uint32_t c = 0; c < nch; ++c) { poff[c] = ch[c].b; plen[c] = (uint32_t)(ch[c].e - ch[c].b); }
    upload_async(ctx, Z.chunk, ch.data(), nch);
    upload_async(ctx, Z.poff, poff.data(), nch);
    upload_async(ctx, Z.plen, plen.data(), nch);
    ensure(Z.m, (end + 1) * 4);
    ensure(Z.freq, (size_t)nch * kDefFreqStride * 4);
    ensure(Z.codes, (size_t)nch * sizeof(DefCodes));
    ensure(Z.hdr, (size_t)nch * kDefHdrWords * 4);
    ensure(Z.info, (size_t)nch * sizeof(DefInfo));
    ensure(Z.scratch, (size_t)nch * kDefScratch);
    ensure(Z.crc, (size_t)nch * 4);
    CK(cudaMemsetAsync(Z.freq.p, 0, (size_t)nch * kDefFreqStride * 4, ctx->stream));
    CK(cudaMemsetAsync(Z.hdr.p, 0, (size_t)nch * kDefHdrWords * 4, ctx->stream));
    CK(cudaMemsetAsync(Z.scratch.p, 0, (size_t)nch * kDefScratch, ctx->stream));
    const DefChunk* dch = (const DefChunk*)Z.chunk.p;
    uint32_t* m = (uint32_t*)Z.m.p;
    DefInfo* dinfo = (DefInfo*)Z.info.p;
    def_match_kernel<<<nch, 32, 0, ctx->stream>>>(in, dch, m);
    def_parse_kernel<<<(nch + 127) / 128, 128, 0, ctx->stream>>>(in, dch, nch, m, (uint32_t*)Z.freq.p, dinfo);
    def_code_kernel<<<(nch + 1) / 2, 64, 0, ctx->stream>>>(dch, nch, (const uint32_t*)Z.freq.p, (DefCodes*)Z.codes.p, (uint32_t*)Z.hdr.p, dinfo);
    def_write_kernel<<<(nch + 3) / 4, 128, 0, ctx->stream>>>(in, dch, nch, m, (const DefCodes*)Z.codes.p, (const uint32_t*)Z.hdr.p, dinfo,
                                                             (uint8_t*)Z.scratch.p);
    inf_crc_kernel<<<(nch + 127) / 128, 128, 0, ctx->stream>>>(in, (const uint64_t*)Z.poff.p, (const uint32_t*)Z.plen.p, nch, (uint32_t*)Z.crc.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(info.data(), Z.info.p, (size_t)nch * sizeof(DefInfo), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(crcs.data(), Z.crc.p, (size_t)nch * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  // the byte-size scan: chunk c goes to dst[c]; every member is header, its chunks, trailer
  std::vector<uint64_t> dst(nch);
  std::vector<uint32_t> trl(2 * (size_t)ns + 2, 0);
  std::vector<uint8_t> hdr((size_t)ns * hlen + 1);
  uint64_t at = 0;
  uint32_t c = 0;
  for (uint32_t k = 0; k < ns; ++k) {
    so[k] = at;
    if (se[k] == sb[k]) continue;
    at += hlen;
    uint32_t crc = 0;
    for (; c < nch && ch[c].stream == k; ++c) { dst[c] = at; at += info[c].bytes; crc = crc_concat(crc, crcs[c], ch[c].e - ch[c].b); }
    trl[2 * k] = crc; trl[2 * k + 1] = (uint32_t)(se[k] - sb[k]);
    at += 8;
    if (hlen == kBgzfHeader) bgzf_header(&hdr[(size_t)k * hlen], (uint32_t)(at - so[k]));
    else for (uint32_t i = 0; i < hlen; ++i) hdr[(size_t)k * hlen + i] = gz_header_byte(i);
  }
  so[ns] = at;
  if (at && (!out || cap < at)) fail(SMR_ERR_CAPACITY, "output buffer too small: stream_off holds the compressed sizes");
  if (nch) {
    upload_async(ctx, Z.dst, dst.data(), nch);
    upload_async(ctx, Z.trl, trl.data(), trl.size());
    upload_async(ctx, Z.ghdr, hdr.data(), hdr.size());
    ensure(Z.out, at);
    def_place_kernel<<<nch, 256, 0, ctx->stream>>>((const DefChunk*)Z.chunk.p, (const DefInfo*)Z.info.p, (const uint8_t*)Z.scratch.p,
                                                   (const uint64_t*)Z.dst.p, (const uint32_t*)Z.trl.p, (const uint8_t*)Z.ghdr.p, hlen, (uint8_t*)Z.out.p);
    CK(cudaGetLastError());
  }
  CK(cudaEventRecord(e_dev, ctx->stream));
  if (at) CK(cudaMemcpyAsync(out, Z.out.p, at, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(e_end, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
}

// The rows of a report-side format call written uncompressed into ctx->r.out (the first half of format_reports_impl): checks,
// prologue, routing (the skip of empty reads), row order, the size passes, scans and write passes, and the BAM refusals.  Returns the
// stream offsets (nso = 2 * groups + read files + 1 of them); e[0], e[1] are recorded by the prologue.  Without gz or bam, so_out gets
// the offsets and a buffer smaller than the rows fails with SMR_ERR_CAPACITY before the writes.
std::vector<uint64_t> rpt_write_rows(smr_ctx* ctx, const smr_report_opts* o, const char* text, uint64_t nbytes, const smr_read_result* results,
                                     const smr_aln* alns, const uint32_t* cigar, uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads,
                                     char* out, uint64_t cap, uint64_t* so_out, bool gz, bool pairwise, bool dev, bool bam, cudaEvent_t* e) {
  const bool mates = o->mates || (!text && ctx->res.mates);   // the resident batch of a mate stream is mates
  const bool paired = o->paired_in || o->paired_out || mates;
  if (pairwise) {   // -blast '0 cigar' is refused by the reference too (options.cpp:584-588)
    if (!o->blast || o->blast_format != 0 || o->blast_cols[0] || o->sam || o->fastx || o->other || o->denovo)
      fail(SMR_ERR_ARG, "pairwise BLAST: opts must ask for -blast 0 alone (blast = 1, blast_format = 0, no BLAST columns, no SAM or read files)");
  } else if (bam) {
    if (!o->sam || o->blast || o->fastx || o->other || o->denovo)
      fail(SMR_ERR_ARG, "BAM: opts must ask for SAM alone (sam = 1, no BLAST, no read files)");
  } else {
    if ((o->out2 || o->sout) && !paired) fail(SMR_ERR_UNSUPPORTED, "-out2 / -sout: only a paired batch (mates, paired_in or paired_out) has mates to split");
    if (o->blast && o->blast_format != 1)
      fail(SMR_ERR_UNSUPPORTED, "smr_format_reports writes tabular BLAST (-blast 1) only: pairwise BLAST (-blast 0) is smr_format_blast_pairwise");
  }
  if (o->paired_in && o->paired_out) fail(SMR_ERR_ARG, "paired_in and paired_out are exclusive");
  if (!pairwise && o->sout && (o->paired_in || o->paired_out)) fail(SMR_ERR_ARG, "-sout cannot be used with paired_in or paired_out");
  const uint32_t num_out = pairwise || bam ? 1 : o->out2 && o->sout ? 4 : o->out2 || o->sout ? 2 : 1;   // ReportFxBase::set_num_out
  const uint32_t nfx = pairwise || bam ? 0 : 3 * num_out;                                                // aligned, other, denovo: num_out files each
  // a null results or alns array: no text of its own, the last one stays
  rpt_check_batch(ctx, "the report writer", results, alns, stats, nreads, paired,
                  o->sam || (o->blast && !pairwise) || o->denovo ? "SAM, BLAST and denovo need the smr_aln_stats of the batch" : nullptr, ctx->err.c_str(), dev);
  uint32_t ncols = 0, cols[4] = {0, 0, 0, 0};
  if (o->blast)
    for (; ncols < 4 && o->blast_cols[ncols]; ++ncols) {
      if (o->blast_cols[ncols] < SMR_BLAST_COL_CIGAR || o->blast_cols[ncols] > SMR_BLAST_COL_QSTRAND) fail(SMR_ERR_ARG, "unknown BLAST column");
      cols[ncols] = (uint32_t)o->blast_cols[ncols];
    }
  const std::vector<RptGroup> hg = rpt_groups(ctx, o->sam || o->blast, o->blast);
  const uint32_t G = (uint32_t)hg.size(), nso = 2 * G + nfx + 1;
  RptArgs a = rpt_prologue(ctx, text, nbytes, results, alns, cigar, cigar_words, stats, nreads, hg, e, dev);
  const uint64_t N = a.nslots;
  const int grid = ctx->sm_count * 8;
  auto& S = ctx->r;
  // per record, routing, row order
  const uint64_t fstride = (uint64_t)nreads + 1;
  uint32_t* flags = ensure<uint32_t>(S.flags, fstride * 4);
  const uint32_t* keys = ensure<uint32_t>(S.keys, (N + 1) * 4);
  uint32_t* keys2 = ensure<uint32_t>(S.keys2, (N + 1) * 4);
  const uint32_t* vals = ensure<uint32_t>(S.vals, (N + 1) * 4);
  uint32_t* rows = ensure<uint32_t>(S.rows, (N + 1) * 4);
  uint64_t* first = ensure<uint64_t>(S.first, ((size_t)G + 1) * 8);
  uint64_t* sz = ensure<uint64_t>(S.sz, (N + 1) * 8);
  uint64_t* off = ensure<uint64_t>(S.off, (N + 1) * 8);
  uint64_t* bsz = ensure<uint64_t>(S.bsz, (N + 1) * 8);
  uint64_t* boff = ensure<uint64_t>(S.boff, (N + 1) * 8);
  uint64_t* fxsz = ensure<uint64_t>(S.fxsz, nfx * fstride * 8);
  uint64_t* fxoff = ensure<uint64_t>(S.fxoff, nfx * fstride * 8);
  uint64_t* so = ensure<uint64_t>(S.so, (size_t)nso * 8);
  uint32_t* bad = &text_words(ctx)->rpt_bad;
  if (bam) CK(cudaMemsetAsync(bad, 0xFF, 4, ctx->stream));
  for (int k = 0; k < 4; ++k) a.cols[k] = cols[k];
  a.ncols = ncols; a.min_id = o->min_id; a.min_cov = o->min_cov;
  a.paired_in = o->paired_in != 0; a.paired_out = o->paired_out != 0; a.mates = mates; a.denovo = o->denovo != 0;
  a.out2 = o->out2 != 0; a.num_out = num_out;
  a.fx_mask = (o->fastx ? kRptAligned : 0u) | (o->other ? kRptOther : 0u) | (o->denovo ? kRptDenovo : 0u);
  CK(cudaMemsetAsync(sz, 0, (N + 1) * 8, ctx->stream));
  CK(cudaMemsetAsync(bsz, 0, (N + 1) * 8, ctx->stream));
  CK(cudaMemsetAsync(fxsz, 0, nfx * fstride * 8, ctx->stream));
  CK(cudaMemsetAsync(first, 0, ((size_t)G + 1) * 8, ctx->stream));
  if (nreads) {
    rpt_route_kernel<<<grid, 256, 0, ctx->stream>>>(a, flags);
    rpt_row_keys_kernel<<<grid, 256, 0, ctx->stream>>>(a, flags, (uint32_t*)keys, (uint32_t*)vals);
    int nbits = 1;
    while ((1u << nbits) <= G) ++nbits;
    cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, keys, keys2, vals, rows, (int)N, 0, nbits, ctx->stream); });
    rpt_group_first_kernel<<<(G + 128) / 128, 128, 0, ctx->stream>>>(keys2, N, G, first);
    if (bam) rpt_bam_size_kernel<<<grid, 256, 0, ctx->stream>>>(a, rows, first, sz, bad);
    else if (o->sam) rpt_sam_size_kernel<<<grid, 256, 0, ctx->stream>>>(a, rows, first, sz);
    if (o->blast && pairwise) rpt_pw_size_kernel<<<grid, 256, 0, ctx->stream>>>(a, rows, first, bsz);
    else if (o->blast) rpt_blast_kernel<<<grid, 256, 0, ctx->stream>>>(a, rows, first, bsz, nullptr, nullptr);
    if (o->fastx || o->other || o->denovo) {
      rpt_fx_size_kernel<<<grid, 256, 0, ctx->stream>>>(a, flags, fxsz, fstride);
    }
    cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, sz, off, (int)(N + 1), ctx->stream); });
    cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, bsz, boff, (int)(N + 1), ctx->stream); });
    if (nfx) cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, fxsz, fxoff, (int)(nfx * fstride), ctx->stream); });
  } else {
    CK(cudaMemsetAsync(off, 0, 8, ctx->stream));
    CK(cudaMemsetAsync(boff, 0, 8, ctx->stream));
    CK(cudaMemsetAsync(fxoff, 0, nfx * fstride * 8, ctx->stream));
  }
  rpt_stream_off_kernel<<<1, 32, 0, ctx->stream>>>(first, G, off, boff, fxoff, nreads, fstride, nfx, so);
  CK(cudaGetLastError());
  std::vector<uint64_t> hso(nso);
  uint32_t err = 0, hbad = 0;
  CK(cudaMemcpyAsync(hso.data(), so, (size_t)nso * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(&err, a.err, 4, cudaMemcpyDeviceToHost, ctx->stream));
  if (bam) CK(cudaMemcpyAsync(&hbad, bad, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (bam) rpt_check_bam(err, hbad);
  rpt_check(err);
  const uint32_t s0 = pairwise ? G : 0;   // the first stream handed out: pairwise, the BLAST streams alone (the SAM ones are empty)
  if (!gz && !bam) memcpy(so_out, hso.data() + s0, (size_t)(nso - s0) * 8);
  const uint64_t total = hso[nso - 1];
  if (!gz && !bam && total && (!out || cap < total)) fail(SMR_ERR_CAPACITY, "output buffer too small: stream_off holds the sizes");
  // the encoder reads up to 8 bytes past a stream's end (def_load32): the padding is part of the one allocation before the writes,
  // since ensure() does not keep what a buffer held
  if (total || gz || bam) ensure(S.out, total + (gz || bam ? 8 : 0));
  if (total) {
    char* dout = (char*)S.out.p;
    if (bam) rpt_bam_write_kernel<<<grid, 256, 0, ctx->stream>>>(a, rows, first, off, dout, bad);
    else if (o->sam) rpt_sam_write_kernel<<<grid, 256, 0, ctx->stream>>>(a, rows, first, off, dout);
    if (o->blast && pairwise) rpt_pw_write_kernel<<<grid, 256, 0, ctx->stream>>>(a, rows, first, boff, dout + hso[G]);
    else if (o->blast) rpt_blast_kernel<<<grid, 256, 0, ctx->stream>>>(a, rows, first, nullptr, boff, dout + hso[G]);
    if (o->fastx || o->other || o->denovo) rpt_fx_write_kernel<<<grid, 256, 0, ctx->stream>>>(a, flags, fxoff, fstride, so + 2 * G, dout);
    CK(cudaGetLastError());
  }
  if (bam) {   // the quality bytes the write pass checked, then each group's records cut into BGZF blocks
    CK(cudaMemcpyAsync(&err, a.err, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(&hbad, bad, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    rpt_check_bam(err, hbad);
  }
  return hso;
}

// pairwise: smr_format_blast_pairwise[_gz], the pairwise BLAST rows alone (-blast 0), one stream per group; bam:
// smr_format_bam_placed, the SAM rows as BAM records in BGZF blocks, one stream per group; otherwise the streams of
// smr_format_reports[_gz].  All share the routing (the skip of empty reads), the row order and the scans (rpt_write_rows).
void format_reports_impl(smr_ctx* ctx, const smr_report_opts* o, const char* text, uint64_t nbytes, const smr_read_result* results,
                         const smr_aln* alns, const uint32_t* cigar, uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads,
                         char* out, uint64_t cap, uint64_t* so_out, bool gz, bool pairwise, bool dev = false, bool bam = false) {
  cudaEvent_t* e = events(ctx, 4);
  const std::vector<uint64_t> hso = rpt_write_rows(ctx, o, text, nbytes, results, alns, cigar, cigar_words, stats, nreads, out, cap, so_out, gz,
                                                   pairwise, dev, bam, e);
  auto& S = ctx->r;
  const uint32_t nso = (uint32_t)hso.size(), G = bam || pairwise ? (nso - 1) / 2 : 0;
  const uint32_t s0 = pairwise ? G : 0;
  const uint64_t total = hso[nso - 1];
  if (bam) {   // each group's records cut into BGZF blocks
    std::vector<uint64_t> sb, se;
    std::vector<size_t> gb(G + 1);   // the first block of each group
    for (uint32_t g = 0; g < G; ++g) { gb[g] = sb.size(); bgzf_blocks(hso[g], hso[g + 1], sb, se); }
    gb[G] = sb.size();
    std::vector<uint64_t> bso(sb.size() + 1, 0);
    const auto put_offsets = on_exit([&] { for (uint32_t g = 0; g <= G; ++g) so_out[g] = bso[gb[g]]; });   // a buffer too small names the sizes
    gzip_streams(ctx, (const uint8_t*)S.out.p, sb, se, out, cap, bso.data(), e[2], e[3], kBgzfHeader);
  } else if (gz) {   // every non-empty stream to one gzip member, before the D2H
    std::vector<uint64_t> sb(hso.begin() + s0, hso.end() - 1), se(hso.begin() + s0 + 1, hso.end());
    gzip_streams(ctx, (const uint8_t*)S.out.p, sb, se, out, cap, so_out, e[2], e[3]);
  } else {
    CK(cudaEventRecord(e[2], ctx->stream));
    if (total) CK(cudaMemcpyAsync(out, S.out.p, total, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaEventRecord(e[3], ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  set_rpt_times(ctx, e);
}

// ---------------------------------------------------------------------------------------------------------------------
// Coordinate-sorted BAM and its BAI index (smr_bamsort.cuh)
// ---------------------------------------------------------------------------------------------------------------------
void bam_sort_open(smr_ctx* ctx) {
  if (!ctx->bs.active) fail(SMR_ERR_ARG, "no open sorted BAM: call smr_bam_sort_begin first");
  if (ctx->bs.gen != ctx->parts_gen)
    fail(SMR_ERR_ARG, "an index part was loaded or its report ids were set after smr_bam_sort_begin: begin the sorted BAM again");
}

// the bits of a sort key: pos + 1 and the strand in the low 32, the refID above
int bam_sort_bits(const smr_ctx* ctx) {
  int b = 32;
  while ((1ull << (b - 32)) < ctx->bs.lin_off.size()) ++b;
  return b;
}

void bam_sort_begin_impl(smr_ctx* ctx) {
  auto& B = ctx->bs;
  B.active = false;
  const std::vector<RptGroup> hg = rpt_groups(ctx, true, false);
  const std::vector<const Part*> gp = report_groups(ctx);
  B.lin_off.assign(1, 0);
  for (size_t g = 0; g < gp.size(); ++g) {
    std::vector<uint32_t> roff((size_t)hg[g].nref + 1);
    CK(cudaMemcpy(roff.data(), hg[g].ref_off, roff.size() * 4, cudaMemcpyDeviceToHost));
    for (uint32_t k = 0; k < hg[g].nref; ++k) {
      const uint64_t len = roff[k + 1] - roff[k];
      if (len >= (1ull << 29))
        fail(SMR_ERR_UNSUPPORTED, "sorted BAM: reference " + gp[g]->h_rnames[k] + " (refID " + std::to_string(hg[g].ref_base + k) + ") has " +
                                      std::to_string(len) + " bases, and a BAI index addresses fewer than 2^29");
      B.lin_off.push_back(B.lin_off.back() + (len + 16383) / 16384);
    }
  }
  B.run_rec.assign(1, 0);
  B.run_bytes.assign(1, 0);
  B.planned = false;
  B.pieces.clear();
  B.gen = ctx->parts_gen;
  B.active = true;
}

// the placed batch's BAM records sorted into a run, into out; the run's keys and sizes appended to the accumulator
void bam_sort_add_impl(smr_ctx* ctx, const smr_report_opts* o, char* out, uint64_t cap, uint64_t* nbytes) {
  auto& B = ctx->bs;
  bam_sort_open(ctx);
  const PlacedArrays p = placed_of(ctx, "smr_bam_sort_add_placed", true);
  cudaEvent_t* e = events(ctx, 4);
  const std::vector<uint64_t> hso = rpt_write_rows(ctx, o, nullptr, 0, p.res, p.aln, p.cig, p.cig_words, p.st, p.n, nullptr, 0, nullptr, false,
                                                   false, true, true, e);
  const uint64_t total = hso.back();
  const uint32_t G = (uint32_t)(hso.size() - 1) / 2;
  *nbytes = total;
  if (total && (!out || cap < total)) fail(SMR_ERR_CAPACITY, "output buffer too small: *nbytes holds the size of the run");
  uint64_t n = 0;
  CK(cudaMemcpy(&n, (const uint64_t*)ctx->r.first.p + G, 8, cudaMemcpyDeviceToHost));
  const uint64_t at = B.run_rec.back();
  if (at + n >= (1ull << 31)) fail(SMR_ERR_CAPACITY, "sorted BAM of 2^31 records or more");
  ensure_keep(ctx, B.key, (at + n) * 8, at * 8);
  ensure_keep(ctx, B.size, (at + n) * 4, at * 4);
  const int grid = ctx->sm_count * 8;
  if (n) {
    const uint8_t* rec = (const uint8_t*)ctx->r.out.p;
    const uint64_t* off = (const uint64_t*)ctx->r.off.p;
    uint64_t* bkey = ensure<uint64_t>(B.bkey, n * 8);
    uint64_t* sbkey = ensure<uint64_t>(B.sbkey, n * 8);
    uint32_t* ord = ensure<uint32_t>(B.ord, n * 4);
    uint32_t* perm = ensure<uint32_t>(B.bperm, n * 4);
    uint64_t* ssz = ensure<uint64_t>(B.ssz, (n + 1) * 8);
    uint64_t* soff = ensure<uint64_t>(B.soff, n * 8);
    uint64_t* doff = ensure<uint64_t>(B.doff, (n + 1) * 8);
    uint8_t* gat = ensure<uint8_t>(B.gat, total);
    bsort_key_kernel<<<grid, 256, 0, ctx->stream>>>(rec, off, n, bkey, ord);
    const int bits = bam_sort_bits(ctx);
    cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, (const uint64_t*)bkey, sbkey, (const uint32_t*)ord, perm, (int)n, 0, bits, ctx->stream); });
    bsort_run_order_kernel<<<grid, 256, 0, ctx->stream>>>(perm, sbkey, off, n, ssz, soff, (uint64_t*)B.key.p, (uint32_t*)B.size.p, at);
    cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, (const uint64_t*)ssz, doff, (int)(n + 1), ctx->stream); });
    bsort_gather_kernel<<<grid, 256, 0, ctx->stream>>>(rec, total, soff, doff, n, gat, false, nullptr);
    CK(cudaGetLastError());
  }
  CK(cudaEventRecord(e[2], ctx->stream));
  if (total) CK(cudaMemcpyAsync(out, B.gat.p, total, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(e[3], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  B.run_rec.push_back(at + n);
  B.run_bytes.push_back(B.run_bytes.back() + total);
  B.planned = false;
  set_rpt_times(ctx, e);
}

// one stable sort of every run's records, the windows cut from it and each window's byte range of each run
void bam_sort_plan_impl(smr_ctx* ctx, uint64_t window_bytes, uint64_t header_bytes, uint64_t* ranges, uint64_t cap, uint64_t* n_windows) {
  auto& B = ctx->bs;
  bam_sort_open(ctx);
  if (!window_bytes) fail(SMR_ERR_ARG, "sorted BAM: window_bytes must be at least 1");
  B.planned = false;
  const uint64_t M = B.run_rec.back();
  const uint32_t R = (uint32_t)B.run_rec.size() - 1;
  const int grid = ctx->sm_count * 8;
  B.pdoff_h.assign(M + 1, 0);
  std::vector<uint32_t> perm(M);
  std::vector<uint64_t> coff(M + 1, 0);
  if (M) {
    uint32_t* ord = ensure<uint32_t>(B.ord, M * 4);
    uint32_t* pperm = ensure<uint32_t>(B.pperm, M * 4);
    uint64_t* pkey = ensure<uint64_t>(B.pkey, M * 8);
    uint64_t* psz = ensure<uint64_t>(B.psz, (M + 1) * 8);
    uint64_t* csz = ensure<uint64_t>(B.csz, (M + 1) * 8);
    uint64_t* pdoff = ensure<uint64_t>(B.pdoff, (M + 1) * 8);
    uint64_t* dcoff = ensure<uint64_t>(B.coff, (M + 1) * 8);
    bsort_iota_kernel<<<grid, 256, 0, ctx->stream>>>(ord, M);
    const int bits = bam_sort_bits(ctx);
    cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, (const uint64_t*)B.key.p, pkey, (const uint32_t*)ord, pperm, (int)M, 0, bits, ctx->stream); });
    bsort_plan_sizes_kernel<<<grid, 256, 0, ctx->stream>>>(pperm, (const uint32_t*)B.size.p, M, psz, csz);
    cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, (const uint64_t*)psz, pdoff, (int)(M + 1), ctx->stream); });
    cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, (const uint64_t*)csz, dcoff, (int)(M + 1), ctx->stream); });
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(B.pdoff_h.data(), pdoff, (M + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(perm.data(), pperm, M * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(coff.data(), dcoff, (M + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  // greedy windows of whole records, each at most window_bytes unless one record is larger
  B.win_rec.assign(1, 0);
  for (uint64_t t = 0; t < M;) {
    uint64_t t1 = (uint64_t)(std::upper_bound(B.pdoff_h.begin() + t + 1, B.pdoff_h.end(), B.pdoff_h[t] + window_bytes) - B.pdoff_h.begin()) - 1;
    if (t1 <= t) t1 = t + 1;
    B.win_rec.push_back(t1);
    t = t1;
  }
  const uint64_t nw = B.win_rec.size() - 1;
  *n_windows = nw;
  const uint64_t need = nw * R * 2;
  if (need && (!ranges || cap < need)) fail(SMR_ERR_CAPACITY, "ranges too small: it takes n_windows * runs * 2 entries (*n_windows is set)");
  // a run's records in a window are one range of it, since the run is sorted and the sort stable
  std::vector<uint32_t> run_of(M);
  for (uint32_t r = 0; r < R; ++r) std::fill(run_of.begin() + B.run_rec[r], run_of.begin() + B.run_rec[r + 1], r);
  for (uint64_t w = 0; w < nw; ++w) {
    uint64_t* rg = ranges + w * R * 2;
    for (uint32_t r = 0; r < R; ++r) { rg[2 * r] = ~0ull; rg[2 * r + 1] = 0; }
    for (uint64_t t = B.win_rec[w]; t < B.win_rec[w + 1]; ++t) {
      const uint32_t o = perm[t], r = run_of[o];
      const uint64_t b = coff[o] - B.run_bytes[r];
      rg[2 * r] = std::min(rg[2 * r], b);
      rg[2 * r + 1] = std::max(rg[2 * r + 1], b + coff[o + 1] - coff[o]);
    }
    for (uint32_t r = 0; r < R; ++r) if (rg[2 * r] == ~0ull) rg[2 * r] = 0;
  }
  B.ranges_h.assign(ranges, ranges + need);
  // the window pass's tables: the run starts, the linear index minima (all ones: no record yet)
  upload_async(ctx, B.runs, B.run_rec.data(), B.run_rec.size());
  upload_async(ctx, B.linoff, B.lin_off.data(), B.lin_off.size());
  ensure(B.lin, B.lin_off.back() * 8 + 8);
  CK(cudaMemsetAsync(B.lin.p, 0xFF, B.lin_off.back() * 8 + 8, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  B.header_bytes = header_bytes;
  B.coffset = header_bytes;
  B.next = 0;
  B.pieces.clear();
  B.planned = true;
}

void bam_sort_planned(smr_ctx* ctx) {
  bam_sort_open(ctx);
  if (!ctx->bs.planned) fail(SMR_ERR_ARG, "sorted BAM: no plan of the runs added: call smr_bam_sort_plan first");
}

// window w: the staged ranges gathered into sorted order, compressed into BGZF blocks, and its index pieces and minima
void bam_sort_window_impl(smr_ctx* ctx, uint64_t w, const void* staged, uint64_t nbytes, char* out, uint64_t cap, uint64_t* out_bytes) {
  auto& B = ctx->bs;
  bam_sort_planned(ctx);
  const uint64_t nw = B.win_rec.size() - 1;
  if (w != B.next || w >= nw)
    fail(SMR_ERR_ARG, "sorted BAM: window " + std::to_string(w) + " out of order: the windows come in order, and the next is " + std::to_string(B.next) +
                          " of " + std::to_string(nw));
  const uint64_t t0 = B.win_rec[w], n = B.win_rec[w + 1] - t0;
  const uint64_t wbytes = B.pdoff_h[t0 + n] - B.pdoff_h[t0];
  if (nbytes != wbytes)
    fail(SMR_ERR_ARG, "sorted BAM: window " + std::to_string(w) + " is " + std::to_string(wbytes) + " bytes, and " + std::to_string(nbytes) + " were staged");
  if (!staged) fail(SMR_ERR_ARG, "sorted BAM: no staged bytes");
  const uint32_t R = (uint32_t)B.run_rec.size() - 1;
  std::vector<int64_t> adj(R);
  for (uint64_t r = 0, base = 0; r < R; ++r) {   // run r's range sits at `base` in the staged bytes
    const uint64_t lo = B.ranges_h[(w * R + r) * 2], hi = B.ranges_h[(w * R + r) * 2 + 1];
    adj[r] = (int64_t)base - (int64_t)B.run_bytes[r] - (int64_t)lo;
    base += hi - lo;
  }
  cudaEvent_t* e = events(ctx, 5);
  CK(cudaEventRecord(e[0], ctx->stream));
  upload_async(ctx, B.stage, (const uint8_t*)staged, nbytes);
  upload_async(ctx, B.adj, adj.data(), R);
  CK(cudaEventRecord(e[1], ctx->stream));
  const int grid = ctx->sm_count * 8;
  const uint64_t* doff = (const uint64_t*)B.pdoff.p + t0;
  uint64_t* soff = ensure<uint64_t>(B.wsoff, n * 8);
  uint8_t* win = ensure<uint8_t>(B.win, wbytes + 8);
  uint32_t* err = ensure<uint32_t>(B.err, 4);
  CK(cudaMemsetAsync(err, 0, 4, ctx->stream));
  CK(cudaMemsetAsync(win + wbytes, 0, 8, ctx->stream));
  bsort_window_src_kernel<<<grid, 256, 0, ctx->stream>>>((const uint32_t*)B.pperm.p, (const uint64_t*)B.coff.p, (const uint64_t*)B.runs.p, R,
                                                         (const int64_t*)B.adj.p, t0, n, soff);
  bsort_gather_kernel<<<grid, 256, 0, ctx->stream>>>((const uint8_t*)B.stage.p, nbytes, soff, doff, n, win, true, err);
  CK(cudaGetLastError());
  uint32_t herr = 0;
  CK(cudaMemcpyAsync(&herr, err, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (herr) fail(SMR_ERR_ARG, "sorted BAM: a staged record's block_size disagrees with the runs added (stage window " + std::to_string(w) + "'s ranges of the runs, in run order)");
  std::vector<uint64_t> sb, se;
  bgzf_blocks(0, wbytes, sb, se);
  const uint32_t ns = (uint32_t)sb.size();
  std::vector<uint64_t> so(ns + 1, 0);
  {
    const auto put_size = on_exit([&] { *out_bytes = so.back(); });   // a buffer too small fails, and names the size needed
    gzip_streams(ctx, win, sb, se, out, cap, so.data(), e[2], e[3], kBgzfHeader);
  }
  // the index pass over the compressed window
  upload_async(ctx, B.bso, so.data(), so.size());
  uint64_t* vb = ensure<uint64_t>(B.vb, n * 8);
  uint64_t* ve = ensure<uint64_t>(B.ve, n * 8);
  uint64_t* rb = ensure<uint64_t>(B.rb, n * 8);
  uint32_t* head = ensure<uint32_t>(B.head, (n + 1) * 4);
  uint32_t* pid = ensure<uint32_t>(B.pid, (n + 1) * 4);
  bsort_index_kernel<kBgzfBlock><<<grid, 256, 0, ctx->stream>>>(win, doff, n, (const uint64_t*)B.bso.p, ns, B.coffset, (const uint64_t*)B.linoff.p,
                                                                (unsigned long long*)B.lin.p, vb, ve, rb, head);
  cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, (const uint32_t*)head, pid, (int)(n + 1), ctx->stream); });
  uint32_t np = 0;
  CK(cudaMemcpyAsync(&np, pid + n, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  BamPiece* pc = ensure<BamPiece>(B.piece, (size_t)np * sizeof(BamPiece));
  bsort_pieces_kernel<<<grid, 256, 0, ctx->stream>>>(vb, ve, rb, head, pid, n, pc);
  CK(cudaGetLastError());
  const size_t at = B.pieces.size();
  B.pieces.resize(at + np);
  CK(cudaMemcpyAsync(B.pieces.data() + at, pc, (size_t)np * sizeof(BamPiece), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(e[4], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  B.coffset += so[ns];
  ++B.next;
  ctx->t_rpt[0] = elapsed_ms(e[0], e[1]);
  ctx->t_rpt[1] = elapsed_ms(e[1], e[2]) + elapsed_ms(e[3], e[4]);
  ctx->t_rpt[2] = elapsed_ms(e[2], e[3]);
}

// the BAI bytes (SAMv1 5.2) from the pieces and the linear minima of every window; closes the sorted BAM
void bam_sort_index_impl(smr_ctx* ctx, char* out, uint64_t cap, uint64_t* nbytes) {
  auto& B = ctx->bs;
  bam_sort_planned(ctx);
  const uint64_t nw = B.win_rec.size() - 1;
  if (B.next != nw)
    fail(SMR_ERR_ARG, "sorted BAM: the index comes after the last window: " + std::to_string(B.next) + " of " + std::to_string(nw) + " windows done");
  const uint32_t nref = (uint32_t)B.lin_off.size() - 1;
  std::vector<uint64_t> lin(B.lin_off.back());
  if (!lin.empty()) CK(cudaMemcpy(lin.data(), B.lin.p, lin.size() * 8, cudaMemcpyDeviceToHost));
  std::vector<uint8_t> h;
  auto le32 = [&](uint32_t v) { for (int k = 0; k < 4; ++k) h.push_back((uint8_t)(v >> (8 * k))); };
  auto le64 = [&](uint64_t v) { for (int k = 0; k < 8; ++k) h.push_back((uint8_t)(v >> (8 * k))); };
  h.insert(h.end(), {'B', 'A', 'I', 1});
  le32(nref);
  size_t p = 0;   // the pieces are in file order, so in refID order
  for (uint32_t k = 0; k < nref; ++k) {
    std::vector<std::pair<uint32_t, std::vector<std::pair<uint64_t, uint64_t>>>> bins;   // bin -> merged chunks in ascending vbeg
    std::vector<std::pair<uint32_t, size_t>> order;
    uint64_t n_mapped = 0, first = ~0ull, last = 0;
    const size_t p0 = p;
    for (; p < B.pieces.size() && (B.pieces[p].refbin >> 32) == k; ++p) {
      const BamPiece& pc = B.pieces[p];
      order.emplace_back((uint32_t)pc.refbin, p);
      n_mapped += pc.last - pc.first + 1;
      first = std::min(first, pc.vbeg);
      last = std::max(last, pc.vend);
    }
    std::stable_sort(order.begin(), order.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    for (const auto& [bin, i] : order) {
      const BamPiece& pc = B.pieces[i];
      if (bins.empty() || bins.back().first != bin) bins.push_back({bin, {}});
      auto& ch = bins.back().second;
      if (!ch.empty() && fmt::bam_chunks_merge(ch.back().second, pc.vbeg)) ch.back().second = pc.vend;
      else ch.emplace_back(pc.vbeg, pc.vend);
    }
    const bool any = p > p0;
    le32((uint32_t)bins.size() + (any ? 1 : 0));
    for (const auto& [bin, ch] : bins) {
      le32(bin);
      le32((uint32_t)ch.size());
      for (const auto& c : ch) { le64(c.first); le64(c.second); }
    }
    if (any) { le32(37450); le32(2); le64(first); le64(last); le64(n_mapped); le64(0); }
    // the linear index: the last window a record overlaps bounds it; an empty window takes the one before, or the first that is set
    const uint64_t l0 = B.lin_off[k], l1 = B.lin_off[k + 1];
    uint64_t n_intv = 0, lead = ~0ull;
    for (uint64_t i = l0; i < l1; ++i) if (lin[i] != ~0ull) { n_intv = i - l0 + 1; if (lead == ~0ull) lead = lin[i]; }
    le32((uint32_t)n_intv);
    for (uint64_t i = 0, cur = lead; i < n_intv; ++i) {
      if (lin[l0 + i] != ~0ull) cur = lin[l0 + i];
      le64(cur);
    }
  }
  le64(0);   // n_no_coor
  *nbytes = h.size();
  if (!out || cap < h.size()) fail(SMR_ERR_CAPACITY, "output buffer too small: *nbytes holds the size of the index");
  memcpy(out, h.data(), h.size());
  B.active = false;
}

// ---------------------------------------------------------------------------------------------------------------------
// OTU map (smr_otu.cuh)
// ---------------------------------------------------------------------------------------------------------------------
void otu_open(smr_ctx* ctx) {
  if (!ctx->otu.active) fail(SMR_ERR_ARG, "no open OTU map: call smr_otu_begin first");
  if (ctx->otu.gen != ctx->parts_gen)
    fail(SMR_ERR_ARG, "an index part was loaded or its report ids were set after smr_otu_begin: begin the OTU map again");
}

void otu_begin_impl(smr_ctx* ctx, const smr_otu_opts* o) {
  auto& U = ctx->otu;
  U.active = false;
  if (!ctx->have_params || !ctx->prm.is_best)
    fail(SMR_ERR_ARG, "the OTU map is made from the best alignments: params.is_best must be 1 (-otu_map cannot be set with -no-best)");
  if (o->paired_in && o->paired_out) fail(SMR_ERR_ARG, "paired_in and paired_out are exclusive");
  if (o->feed != SMR_OTU_SINGLE && o->feed != SMR_OTU_ONE_FILE && o->feed != SMR_OTU_TWO_FILES) fail(SMR_ERR_ARG, "unknown OTU feed");
  if (o->feed == SMR_OTU_SINGLE && (o->paired_in || o->paired_out))
    fail(SMR_ERR_UNSUPPORTED, "paired reads: the reference's OTU pass reads only the first mate file of two, but every record of one interleaved file: "
                              "say which with feed SMR_OTU_ONE_FILE or SMR_OTU_TWO_FILES");
  U.groups = rpt_groups(ctx, true, false);
  const std::vector<const Part*> gp = report_groups(ctx);
  const uint32_t G = (uint32_t)gp.size();
  // ranks of the reference ids in unsigned byte order (std::string compares as unsigned char)
  std::vector<const std::string*> ids;
  for (const Part* pt : gp) for (const std::string& s : pt->h_rnames) ids.push_back(&s);
  std::sort(ids.begin(), ids.end(), [](const std::string* a, const std::string* b) { return *a < *b; });
  ids.erase(std::unique(ids.begin(), ids.end(), [](const std::string* a, const std::string* b) { return *a == *b; }), ids.end());
  std::vector<uint32_t> rank, rank_off(std::max(G, 1u), 0);
  for (uint32_t g = 0; g < G; ++g) {
    rank_off[g] = (uint32_t)rank.size();
    for (const std::string& s : gp[g]->h_rnames)
      rank.push_back((uint32_t)(std::lower_bound(ids.begin(), ids.end(), &s, [](const std::string* a, const std::string* b) { return *a < *b; }) - ids.begin()));
  }
  uint32_t gbits = 1, rbits = 1;
  while ((1ull << gbits) <= G) ++gbits;
  while ((1ull << rbits) <= ids.size()) ++rbits;
  upload_async(ctx, U.rank, rank.data(), rank.size());
  upload_async(ctx, U.rank_off, rank_off.data(), rank_off.size());
  upload_async(ctx, U.grp, U.groups.data(), G);
  CK(cudaStreamSynchronize(ctx->stream));
  U.gbits = gbits; U.kbits = gbits + rbits;
  U.min_id = o->min_id; U.min_cov = o->min_cov; U.feed = (uint32_t)o->feed;
  U.n = 0; U.pool_bytes = 0;
  for (double& t : U.t) t = 0;
  U.gen = ctx->parts_gen;
  U.active = true;
}

// returns the number of entries added
uint64_t otu_add_impl(smr_ctx* ctx, const char* text, uint64_t nbytes, const smr_read_result* results, const smr_aln* alns, const smr_aln_stats* stats,
                      uint32_t nreads, bool dev = false) {
  auto& U = ctx->otu;
  otu_open(ctx);
  if (!text && ctx->res.mates && U.feed != SMR_OTU_TWO_FILES)
    fail(SMR_ERR_UNSUPPORTED, "a mate stream's batch is two mate files: open the OTU map with feed SMR_OTU_TWO_FILES");
  rpt_check_batch(ctx, "the OTU map", results, alns, stats, nreads, U.feed != SMR_OTU_SINGLE,
                  "the OTU map needs the results, alignments and smr_aln_stats of the batch", nullptr, dev);
  cudaEvent_t* e = events(ctx, 3);
  const RptArgs a = rpt_prologue(ctx, text, nbytes, results, alns, nullptr, 0, stats, nreads, U.groups, e, dev);
  const uint64_t N = a.nslots;
  const OtuArgs oa{(const uint32_t*)U.rank.p, (const uint32_t*)U.rank_off.p, U.gbits, U.min_id, U.min_cov, U.feed};
  uint32_t* flag = ensure<uint32_t>(U.flag, (N + 1) * 4);
  uint32_t* pos = ensure<uint32_t>(U.pos, (N + 1) * 4);
  uint64_t* nsz = ensure<uint64_t>(U.nsz, (N + 1) * 8);
  uint64_t* noff = ensure<uint64_t>(U.noff, (N + 1) * 8);
  const int grid = ctx->sm_count * 8;
  CK(cudaMemsetAsync(flag + N, 0, 4, ctx->stream));
  CK(cudaMemsetAsync(nsz + N, 0, 8, ctx->stream));
  otu_flag_kernel<<<grid, 256, 0, ctx->stream>>>(a, oa, flag, nsz);
  cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, flag, pos, (int)(N + 1), ctx->stream); });
  cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, nsz, noff, (int)(N + 1), ctx->stream); });
  CK(cudaGetLastError());
  uint32_t m = 0, err = 0; uint64_t bytes = 0;
  CK(cudaMemcpyAsync(&m, pos + N, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(&bytes, noff + N, 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(&err, a.err, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  rpt_check(err);
  if (U.n + m >= (1ull << 31)) fail(SMR_ERR_CAPACITY, "OTU map of 2^31 entries or more");
  ensure_keep(ctx, U.key, (U.n + m) * 8, U.n * 8);
  ensure_keep(ctx, U.ent, (U.n + m) * sizeof(OtuEnt), U.n * sizeof(OtuEnt));
  ensure_keep(ctx, U.pool, U.pool_bytes + bytes, U.pool_bytes);
  if (m) otu_append_kernel<<<grid, 256, 0, ctx->stream>>>(a, oa, flag, pos, noff, U.n, U.pool_bytes, (uint64_t*)U.key.p, (OtuEnt*)U.ent.p, (char*)U.pool.p);
  CK(cudaGetLastError());
  CK(cudaEventRecord(e[2], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  U.n += m; U.pool_bytes += bytes;
  U.t[0] += elapsed_ms(e[0], e[1]);
  U.t[1] += elapsed_ms(e[1], e[2]);
  return m;
}

void otu_finish_impl(smr_ctx* ctx, char* out, uint64_t cap, uint64_t counts[3]) {
  auto& U = ctx->otu;
  otu_open(ctx);
  const uint64_t m = U.n;
  cudaEvent_t* e = events(ctx, 2);
  CK(cudaEventRecord(e[0], ctx->stream));
  uint64_t bytes = 0; uint32_t runs = 0;
  const int grid = ctx->sm_count * 8;
  if (m) {
    uint32_t* vals = ensure<uint32_t>(U.vals, m * 4);
    uint32_t* sidx = ensure<uint32_t>(U.sidx, m * 4);
    uint64_t* skey = ensure<uint64_t>(U.skey, m * 8);
    uint64_t* size = ensure<uint64_t>(U.size, (m + 1) * 8);
    uint64_t* off = ensure<uint64_t>(U.off, (m + 1) * 8);
    uint32_t* scal = ensure<uint32_t>(U.scal, 16);
    otu_iota_kernel<<<grid, 256, 0, ctx->stream>>>(vals, m);
    cub_run(ctx->cub_tmp, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortPairs(t, b, (const uint64_t*)U.key.p, skey, (const uint32_t*)vals, sidx, (int)m, 0, (int)U.kbits, ctx->stream);
    });
    CK(cudaMemsetAsync(scal, 0, 16, ctx->stream));
    CK(cudaMemsetAsync(size + m, 0, 8, ctx->stream));
    otu_size_kernel<<<grid, 256, 0, ctx->stream>>>(skey, sidx, (const OtuEnt*)U.ent.p, m, U.gbits, (const RptGroup*)U.grp.p, size, scal);
    cub_run(ctx->cub_tmp, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, size, off, (int)(m + 1), ctx->stream); });
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(&bytes, off + m, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(&runs, scal, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  counts[0] = bytes; counts[1] = runs; counts[2] = m;
  if (bytes && (!out || cap < bytes)) fail(SMR_ERR_CAPACITY, "output buffer too small: counts[0] holds the size");
  if (bytes) {
    ensure(U.out, bytes);
    otu_write_kernel<<<grid, 256, 0, ctx->stream>>>((const uint64_t*)U.skey.p, (const uint32_t*)U.sidx.p, (const OtuEnt*)U.ent.p, m, U.gbits,
                                                    (const RptGroup*)U.grp.p, (const char*)U.pool.p, (const uint64_t*)U.off.p, (char*)U.out.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, U.out.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CK(cudaEventRecord(e[1], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  U.t[2] = elapsed_ms(e[0], e[1]);
  U.active = false;
}

// ---------------------------------------------------------------------------------------------------------------------
// De novo statistics (smr_otu.cuh, denovo_stats_kernel)
// ---------------------------------------------------------------------------------------------------------------------
void denovo_stats_impl(smr_ctx* ctx, const smr_denovo_opts* o, const char* text, uint64_t nbytes, const smr_read_result* results,
                       const smr_aln* alns, const smr_aln_stats* stats, uint32_t nreads, uint32_t* per_read, uint64_t totals[4], bool dev = false) {
  rpt_check_batch(ctx, "the denovo statistics", results, alns, stats, nreads, false,
                  "the denovo statistics need the results, alignments and smr_aln_stats of the batch", nullptr, dev);
  const bool paired = o->paired || (!text && ctx->res.mates);   // the resident batch of a mate stream is mates
  cudaEvent_t* e = events(ctx, 4);
  // the loaded (index, part)s: an alignment of any other is refused
  const RptArgs a = rpt_prologue(ctx, text, nbytes, results, alns, nullptr, 0, stats, nreads, rpt_groups(ctx, false, false), e, dev);
  uint32_t* dread = ensure<uint32_t>(ctx->dn.read, ((size_t)nreads + 1) * 16);
  unsigned long long* dtot = ensure<unsigned long long>(ctx->dn.tot, 32);
  CK(cudaMemsetAsync(dread, 0, (size_t)nreads * 16, ctx->stream));
  CK(cudaMemsetAsync(dtot, 0, 32, ctx->stream));
  if (nreads) denovo_stats_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(a, o->min_id, o->min_cov, paired, dread, dtot);
  CK(cudaGetLastError());
  uint64_t tot[4] = {0, 0, 0, 0}; uint32_t err = 0;
  CK(cudaMemcpyAsync(&err, a.err, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(e[2], ctx->stream));
  CK(cudaMemcpyAsync(tot, dtot, 32, cudaMemcpyDeviceToHost, ctx->stream));
  if (per_read && nreads) CK(cudaMemcpyAsync(per_read, dread, (size_t)nreads * 16, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(e[3], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  rpt_check(err);
  for (int k = 0; k < 4; ++k) totals[k] += tot[k];
  set_rpt_times(ctx, e);
}

}  // namespace

extern "C" {

// Internal code throws; every entry point that can fail is a function-try-block that turns the failure into a status and an error text here.
#define SMR_CATCH(ctx) \
  catch (const Failure& f) { (ctx)->err = f.msg; return f.code; } \
  catch (const std::bad_alloc&) { if (ctx) (ctx)->err = "out of host memory"; return SMR_ERR_CAPACITY; } \
  catch (const std::exception& ex) { if (ctx) (ctx)->err = std::string("internal error: ") + ex.what(); return SMR_ERR_CUDA; }

int smr_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

int smr_init(int device, smr_ctx** out) try {
  if (!out) return SMR_ERR_ARG;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0 || device < 0 || device >= n) return SMR_ERR_NO_DEVICE;
  smr_ctx* ctx = new smr_ctx();
  ctx->device = device;
  if (cudaSetDevice(device) != cudaSuccess) { delete ctx; return SMR_ERR_NO_DEVICE; }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete ctx; return SMR_ERR_NO_DEVICE; }
  ctx->sm_count = prop.multiProcessorCount;
  if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return SMR_ERR_CUDA; }
  if (const char* e = getenv("SMR_CHUNK_READS")) { const long v = atol(e); if (v >= 32 && v <= (1l << 22)) ctx->chunk_reads = (uint32_t)v; }   // tests: several chunks per batch
  if (const char* e = getenv("SMR_INSTR")) ctx->instr = atoi(e) != 0;   // instrumented instantiations of the seed and candidate kernels (smr_set_instrumentation)
  if (const char* e = getenv("SMR_RETRY_SLOTS")) { const long long v = atoll(e); if (v >= 1) ctx->retry_slots = (uint64_t)v; }   // tests: many sub-batches
  if (const char* e = getenv("SMR_LIS_CTAS_PER_SM")) { const int v = atoi(e); if (v >= 1 && v <= 16) ctx->lis_ctas_per_sm = (uint32_t)v; }
  *out = ctx;
  return SMR_OK;
} catch (const std::bad_alloc&) { return SMR_ERR_CAPACITY; } catch (const std::exception&) { return SMR_ERR_CUDA; }

void smr_destroy(smr_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  for (cudaEvent_t e : ctx->ev) cudaEventDestroy(e);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;   // the buffers free themselves
}

const char* smr_last_error(const smr_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int smr_load_index_part(smr_ctx* ctx, uint32_t index_num, uint32_t part, const void* kmer_file, size_t kmer_bytes,
                        const void* bursttrie_file, size_t bursttrie_bytes, const void* pos_file, size_t pos_bytes,
                        const uint8_t* refseq_cat, const uint64_t* ref_off, uint32_t nref, uint32_t lnwin, uint32_t minimal_score,
                        const uint32_t skiplengths[3]) try {
  if (!ctx || !kmer_file || !bursttrie_file || !pos_file || !refseq_cat || !ref_off || !skiplengths) return SMR_ERR_ARG;
  if (skiplengths[0] == 0 || skiplengths[1] == 0 || skiplengths[2] == 0) { ctx->err = "skiplengths must be positive"; return SMR_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  FlatIndex fx;
  std::string e;
  try {
    e = flatten_index(kmer_file, kmer_bytes, bursttrie_file, bursttrie_bytes, pos_file, pos_bytes, lnwin, fx);
  } catch (const std::exception& ex) { e = std::string("index files could not be read: ") + ex.what(); }   // bad_alloc / length_error on a malformed file
  if (!e.empty()) { ctx->err = e; return SMR_ERR_INDEX; }
  const uint64_t ref_total = ref_off[nref] - ref_off[0];
  if (ref_total >= 0xFFFFFFFFull) { ctx->err = "reference part larger than 4 GB"; return SMR_ERR_UNSUPPORTED; }
  for (const auto& sp : fx.pos) if (sp.seq >= nref) { ctx->err = "position table names a sequence beyond the references"; return SMR_ERR_INDEX; }
  Part pt;
  pt.d.index_num = index_num; pt.d.part = part; pt.d.lnwin = lnwin; pt.d.partialwin = lnwin / 2; pt.d.minimal_score = minimal_score;
  for (int i = 0; i < 3; ++i) pt.d.skip[i] = skiplengths[i];
  pt.d.nref = nref; pt.d.nids = (uint32_t)(fx.pos_off.size() - 1);
  std::vector<uint32_t> roff(nref + 1);
  for (uint32_t i = 0; i <= nref; ++i) roff[i] = (uint32_t)(ref_off[i] - ref_off[0]);
  std::vector<uint8_t> rseq(refseq_cat + ref_off[0], refseq_cat + ref_off[nref]);
  rseq.resize(rseq.size() + 64, 4);
  std::vector<uint32_t> ftext(ftext_words(fx.flist.size()), 0), fid(fx.flist.size());
  for (size_t i = 0; i < fx.flist.size(); ++i) { ftext[i] = fx.flist[i].tail; fid[i] = fx.flist[i].id; }   // an flist item's tail holds the full text
  const size_t len[kSearchArrays] = {fx.flookup.size() * 4, ftext.size() * 4, fid.size() * 4, fx.pos_off.size() * 4, fx.pos.size() * sizeof(SeqPos)};
  const void* src[kSearchArrays] = {fx.flookup.data(), ftext.data(), fid.data(), fx.pos_off.data(), fx.pos.data()};
  pt.d.index_num = index_num; pt.d.part = part;
  uint8_t* sb = alloc_search(ctx, pt, len);
  for (int k = 0; k < kSearchArrays; ++k)
    if (len[k]) CK(cudaMemcpyAsync(sb + search_at(pt, k), src[k], len[k], cudaMemcpyHostToDevice, ctx->stream));
  pt.d.refseq = part_array<uint8_t>(ctx, pt, rseq.size(), rseq.data());
  pt.d.ref_off = part_array<uint32_t>(ctx, pt, roff.size(), roff.data());
  CK(cudaStreamSynchronize(ctx->stream));
  pt.n_refseq = rseq.size();
  pt.n_nodes = fx.nodes.size(); pt.n_entries = fx.entries.size(); pt.n_ids = pt.d.nids; pt.n_pos = fx.pos.size();
  add_part(ctx, std::move(pt));
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_build_index_device(smr_ctx* ctx, uint32_t index_num, const char* fasta_path, uint32_t lnwin, uint32_t interval, uint32_t max_pos, double max_mb,
                           const uint32_t skiplengths[3], uint32_t minimal_score, uint32_t* nparts, uint64_t report6[6]) try {
  if (!ctx || !fasta_path || !skiplengths) return SMR_ERR_ARG;
  if (skiplengths[0] == 0 || skiplengths[1] == 0 || skiplengths[2] == 0) { ctx->err = "skiplengths must be positive"; return SMR_ERR_ARG; }
  if (lnwin < 8 || lnwin > 26 || (lnwin & 1)) { ctx->err = "unsupported seed length"; return SMR_ERR_ARG; }
  if (interval == 0) { ctx->err = "interval must be >= 1"; return SMR_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  BuildOptions opt; opt.lnwin = lnwin; opt.interval = interval; opt.max_pos = max_pos; opt.max_mb = max_mb;
  std::vector<RefRecord> recs;
  double freq[4] = {0, 0, 0, 0};
  uint64_t full_len = 0; size_t fsize = 0;
  std::string e;
  try {
    e = parse_reference_fasta(fasta_path, lnwin + 1, true, recs, freq, full_len, fsize);
  } catch (const std::exception& ex) { e = std::string("index build failed: ") + ex.what(); }
  if (!e.empty()) { ctx->err = e; return SMR_ERR_INDEX; }
  uint32_t part = 0;
  uint64_t rep[6] = {0, recs.size(), 0, 0, 0, 0};
  size_t first = 0;
  while (first < recs.size()) {
    std::vector<size_t> members; size_t next = first; uint64_t start_part = 0, seq_part_size = 0;
    e = next_index_part(recs, first, lnwin + 1, max_mb, members, next, start_part, seq_part_size);
    if (!e.empty()) { ctx->err = e; return SMR_ERR_INDEX; }
    if (members.empty()) break;
    Part pt = build_part_device(ctx, recs, members, opt, index_num, part);
    pt.d.minimal_score = minimal_score;
    for (int i = 0; i < 3; ++i) pt.d.skip[i] = skiplengths[i];
    rep[3] += pt.n_ids; rep[5] += pt.bytes;
    add_part(ctx, std::move(pt));
    ++part; first = next;
  }
  if (part == 0) { ctx->err = "no index was created"; return SMR_ERR_INDEX; }
  rep[0] = part;
  if (nparts) *nparts = part;
  if (report6) memcpy(report6, rep, sizeof(rep));
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_debug_index_array(smr_ctx* ctx, uint32_t slot, uint32_t which, void* out, uint64_t cap_bytes, uint64_t* nbytes) try {
  if (!ctx || !nbytes || slot >= ctx->parts.size()) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const Part& pt = ctx->parts[slot];
  const void* src = nullptr; uint64_t n = 0;
  // the search arrays of a part whose device copy an index budget has freed are read from its host copy
  auto copy = [&](void* dst, const void* dev, int k, uint64_t bytes) {
    if (pt.search.p) CK(cudaMemcpy(dst, dev, bytes, cudaMemcpyDeviceToHost));
    else memcpy(dst, (const uint8_t*)pt.host.p + search_at(pt, k), bytes);
  };
  switch (which) {
    case 0: src = pt.d.flookup; n = ((uint64_t)16) << (2 * pt.d.partialwin); break;
    case 1: n = (uint64_t)pt.n_entries * 8; break;   // {text, id} pairs, interleaved below
    case 2: src = pt.d.pos_off; n = ((uint64_t)pt.n_ids + 1) * 4; break;
    case 3: src = pt.d.pos; n = (uint64_t)pt.n_pos * 8; break;
    case 4: src = pt.d.refseq; n = pt.n_refseq; break;
    case 5: src = pt.d.ref_off; n = ((uint64_t)pt.d.nref + 1) * 4; break;
    default: ctx->err = "no such array"; return SMR_ERR_ARG;
  }
  *nbytes = n;
  if (!out) return SMR_OK;
  if (cap_bytes < n) { ctx->err = "buffer too small"; return SMR_ERR_CAPACITY; }
  if (which == 1) {
    std::vector<uint32_t> text(pt.n_entries), id(pt.n_entries), pairs(2 * pt.n_entries);
    if (n) copy(text.data(), pt.d.ftext, 1, n / 2);
    if (n) copy(id.data(), pt.d.fid, 2, n / 2);
    for (size_t i = 0; i < pt.n_entries; ++i) { pairs[2 * i] = text[i]; pairs[2 * i + 1] = id[i]; }
    if (n) memcpy(out, pairs.data(), n);
    return SMR_OK;
  }
  if (n && which < 4) copy(out, src, which == 0 ? 0 : which + 1, n);   // flookup, pos_off, pos: search arrays 0, 3, 4
  else if (n) CK(cudaMemcpy(out, src, n, cudaMemcpyDeviceToHost));
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_set_minimal_score(smr_ctx* ctx, uint32_t index_num, uint32_t minimal_score) {
  if (!ctx) return SMR_ERR_ARG;
  bool any = false;
  for (auto& pt : ctx->parts) if (pt.d.index_num == index_num) { pt.d.minimal_score = minimal_score; any = true; }
  if (!any) { ctx->err = "no such index"; return SMR_ERR_ARG; }
  return SMR_OK;
}

int smr_set_params(smr_ctx* ctx, const smr_params* p) {
  if (!ctx || !p) return SMR_ERR_ARG;
  if (p->match < -128 || p->match > 127 || p->gap_open < 0 || p->gap_ext < 0) { ctx->err = "scores out of range"; return SMR_ERR_ARG; }
  ctx->prm = *p; ctx->have_params = true;
  return SMR_OK;
}

int smr_set_aln_slots(smr_ctx* ctx, uint32_t slots) {
  if (!ctx || slots == 0 || slots > (1u << 20)) return SMR_ERR_ARG;
  ctx->all_slots = slots;
  return SMR_OK;
}

uint32_t smr_aln_slots(const smr_ctx* ctx) { return ctx ? slots_of(ctx) : 0; }
uint32_t smr_aln_slots_needed(const smr_ctx* ctx) { return ctx ? ctx->need_slots : 0; }

int smr_index_info(const smr_ctx* ctx, uint64_t out[6]) {
  if (!ctx || !out) return SMR_ERR_ARG;
  memset(out, 0, 6 * sizeof(uint64_t));
  out[0] = ctx->parts.size();
  for (auto& pt : ctx->parts) {
    out[1] += pt.bytes; out[2] += pt.n_nodes; out[3] += pt.n_entries; out[4] += pt.n_ids; out[5] += pt.n_pos;
    if (!pt.search.p) for (size_t b : pt.search_len) out[1] -= b;   // its search arrays are held on the host
  }
  out[1] += ctx->ib.arena.cap;
  return SMR_OK;
}

int smr_set_index_budget(smr_ctx* ctx, uint64_t bytes) try {
  if (!ctx) return SMR_ERR_ARG;
  for (const Part& pt : ctx->parts) check_budget(ctx, pt, bytes);
  ctx->ib.budget = bytes;
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_index_residency(const smr_ctx* ctx, uint64_t out[7]) {
  if (!ctx || !out) return SMR_ERR_ARG;
  memset(out, 0, 7 * sizeof(uint64_t));
  const std::vector<IndexGroup> gs = index_groups(ctx);
  out[0] = gs.size();
  for (const IndexGroup& g : gs) out[1] = std::max<uint64_t>(out[1], g.bytes);
  for (const Part& pt : ctx->parts) { out[2] += pt.search.cap; out[3] += pt.host.cap; }
  out[2] += ctx->ib.arena.cap;
  out[4] = ctx->ib.uploads; out[5] = ctx->ib.upload_bytes;
  out[6] = (uint64_t)std::llround(ctx->ib.t_upload * 1000.0);
  return SMR_OK;
}

int smr_set_aln_layout(smr_ctx* ctx, uint32_t layout) {
  if (!ctx) return SMR_ERR_ARG;
  if (layout != SMR_ALNS_STRIDED && layout != SMR_ALNS_PACKED) { ctx->err = "smr_set_aln_layout: unknown layout " + std::to_string(layout); return SMR_ERR_ARG; }
  ctx->layout = layout;
  return SMR_OK;
}

// the strided entry points have no alignment capacity to size a packed result by
#define SMR_REFUSE_PACKED(ctx, call, instead)                                                                      \
  if (packed(ctx)) { (ctx)->err = call " writes the strided layout: in the packed layout call " instead; return SMR_ERR_ARG; }

int smr_align_batch(smr_ctx* ctx, const uint8_t* seq_cat, const uint64_t* seq_off, uint32_t nreads, smr_read_result* results, smr_aln* alns,
                    uint32_t* cigar_pool, uint64_t cigar_cap, uint64_t* cigar_used, uint64_t* counters, uint32_t n_counters) try {
  if (!ctx || !seq_cat || !seq_off || !results || !alns || (!cigar_pool && cigar_cap)) return SMR_ERR_ARG;
  SMR_REFUSE_PACKED(ctx, "smr_align_batch", "smr_align_batch_packed")
  CK(cudaSetDevice(ctx->device));
  const uint32_t slots = slots_of(ctx);
  memset(results, 0, (size_t)nreads * sizeof(smr_read_result));
  memset(alns, 0, (size_t)nreads * slots * sizeof(smr_aln));
  HostOut out{results, alns, cigar_pool, cigar_cap, 0, counters, n_counters};
  const auto put_used = on_exit([&] { if (cigar_used) *cigar_used = out.cigar_used; });   // a pool too small fails, and names the words needed
  upload_batch_impl(ctx, seq_cat, seq_off, nreads);
  run_impl(ctx, ctx->res.b);
  download_resident(ctx, out);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_set_instrumentation(smr_ctx* ctx, int on) {
  if (!ctx) return SMR_ERR_ARG;
  ctx->instr = on != 0;
  return SMR_OK;
}

int smr_set_stats_buffer(smr_ctx* ctx, smr_aln_stats* stats) {
  if (!ctx) return SMR_ERR_ARG;
  if (stats) SMR_REFUSE_PACKED(ctx, "smr_set_stats_buffer", "smr_align_batch_packed / smr_download_results_packed with their stats argument")
  ctx->host_stats = stats;
  return SMR_OK;
}

int smr_upload_batch(smr_ctx* ctx, const uint8_t* seq_cat, const uint64_t* seq_off, uint32_t nreads) try {
  if (!ctx || !seq_cat || !seq_off) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  upload_batch_impl(ctx, seq_cat, seq_off, nreads);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_upload_fastx(smr_ctx* ctx, const char* text, uint64_t nbytes, uint32_t* nreads) try {
  if (!ctx || (!text && nbytes) || !nreads) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  *nreads = 0;   // as it stays if the upload fails
  *nreads = upload_fastx_impl(ctx, text, nbytes);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_upload_fastx_gz(smr_ctx* ctx, const void* gz, uint64_t nbytes, uint32_t* nreads) try {
  if (!ctx || !gz || !nreads) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  *nreads = 0;
  const char* e = getenv("SMR_INFLATE_CHUNK");
  const uint64_t total = inflate_impl(ctx, gz, nbytes, e ? strtoull(e, nullptr, 10) : inflate_chunk(nbytes));
  if (total == 0) return SMR_OK;
  char c0 = 0;
  CK(cudaMemcpy(&c0, ctx->res.text.p, 1, cudaMemcpyDeviceToHost));
  *nreads = upload_fastx_impl(ctx, nullptr, total, c0);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_resident_text(smr_ctx* ctx, char* text, uint64_t cap, uint64_t* nbytes) try {
  if (!ctx || !nbytes) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const auto& R = ctx->res;
  *nbytes = R.text_bytes;
  if (!text || R.text_bytes == 0) return SMR_OK;
  if (cap < R.text_bytes) { ctx->err = "text buffer too small"; return SMR_ERR_CAPACITY; }
  CK(cudaMemcpy(text, R.text.p, R.text_bytes, cudaMemcpyDeviceToHost));
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_debug_inflate(smr_ctx* ctx, const void* gz, uint64_t nbytes, uint64_t chunk_bytes, uint8_t* out, uint64_t out_cap, uint64_t* out_bytes, uint32_t info[4]) try {
  if (!ctx || !gz || !out_bytes) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  if (chunk_bytes == 0) chunk_bytes = inflate_chunk(nbytes);
  *out_bytes = 0;   // as it stays if the inflate fails
  *out_bytes = inflate_impl(ctx, gz, nbytes, chunk_bytes);
  if (info) { info[0] = ctx->inf.spans; info[1] = ctx->inf.candidates; info[2] = (uint32_t)(ctx->t_inflate * 1000.0); info[3] = (uint32_t)(ctx->t_h2d * 1000.0); }
  if (out && *out_bytes) {
    if (out_cap < *out_bytes) { ctx->err = "output buffer too small"; return SMR_ERR_CAPACITY; }
    CK(cudaMemcpy(out, ctx->res.text.p, *out_bytes, cudaMemcpyDeviceToHost));
  }
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_stream_begin(smr_ctx* ctx, uint32_t flags, uint64_t batch_bytes) try {
  if (!ctx) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const CountState before = ctx->rs.counts;
  close_stream(ctx->rs);
  if (flags & ~(uint32_t)(SMR_STREAM_GZ | SMR_STREAM_COUNT_ONLY | SMR_STREAM_NEXT_FILE | SMR_STREAM_MATES)) fail(SMR_ERR_ARG, "smr_stream_begin: unknown flags");
  if ((flags & SMR_STREAM_MATES) && (flags & (SMR_STREAM_COUNT_ONLY | SMR_STREAM_NEXT_FILE)))
    fail(SMR_ERR_ARG, "smr_stream_begin: a mate stream makes batches and counts nothing: count mate files one after another (SMR_STREAM_NEXT_FILE)");
  if (flags & SMR_STREAM_NEXT_FILE) ctx->rs.counts = rc_next_file(before, flags & SMR_STREAM_GZ);
  if (!(flags & SMR_STREAM_COUNT_ONLY) && (batch_bytes == 0 || batch_bytes >= 0xF0000000ull)) fail(SMR_ERR_ARG, "smr_stream_begin: batch_bytes must be in [1, 0xF0000000)");
  ReadStream& rs = ctx->rs;
  rs.gz = flags & SMR_STREAM_GZ; rs.count_only = flags & SMR_STREAM_COUNT_ONLY; rs.mates = flags & SMR_STREAM_MATES; rs.batch_bytes = batch_bytes;
  rs.open = true;
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_stream_push(smr_ctx* ctx, const void* bytes, uint64_t n, int eof) try {
  if (!ctx || (!bytes && n)) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  stream_call(ctx, [&] {
    if (ctx->rs.mates) fail(SMR_ERR_ARG, "smr_stream_push on a mate stream: push each mate with smr_stream_push_mate");
    stream_push_impl(ctx, 0, (const uint8_t*)bytes, n, eof != 0);
  });
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_stream_push_mate(smr_ctx* ctx, uint32_t mate, const void* bytes, uint64_t n, int eof) try {
  if (!ctx || (!bytes && n)) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  stream_call(ctx, [&] {
    if (!ctx->rs.mates) fail(SMR_ERR_ARG, "smr_stream_push_mate on a stream not opened with SMR_STREAM_MATES");
    if (mate != 1 && mate != 2) fail(SMR_ERR_ARG, "smr_stream_push_mate: mate must be 1 or 2");
    stream_push_impl(ctx, mate - 1, (const uint8_t*)bytes, n, eof != 0);
  });
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_stream_next(smr_ctx* ctx, uint32_t* nreads, int* done) try {
  if (!ctx || !nreads || !done) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  *nreads = 0; *done = 0;
  stream_call(ctx, [&] { *nreads = stream_next_impl(ctx, done); });
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_stream_counts(smr_ctx* ctx, uint64_t out[4]) {
  if (!ctx || !out) return SMR_ERR_ARG;
  const CountState& c = ctx->rs.counts;
  out[0] = c.reads; out[1] = c.length; out[2] = rc_min(c); out[3] = c.max_len;
  return SMR_OK;
}

int smr_resident_layout(smr_ctx* ctx, uint64_t* header_text_off, uint64_t* read_off, uint8_t* seq04, uint64_t seq_cap) try {
  if (!ctx) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const Batch& b = ctx->res.b;
  const uint32_t n = b.nreads;
  if (read_off) for (uint32_t r = 0; r <= n; ++r) read_off[r] = n ? b.off32[r] : 0;
  if (header_text_off && n) {
    if (!b.from_text) { ctx->err = "the resident batch was not uploaded as text"; return SMR_ERR_ARG; }
    CK(cudaMemcpy(header_text_off, ctx->res.hdroff.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
  }
  if (seq04 && n) {
    if (seq_cap < b.total_nt) { ctx->err = "sequence buffer too small"; return SMR_ERR_CAPACITY; }
    CK(cudaMemcpy(seq04, b.seq04.p, b.total_nt, cudaMemcpyDeviceToHost));
  }
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_run_resident(smr_ctx* ctx) try {
  if (!ctx) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  run_impl(ctx, ctx->res.b);
  ctx->t_run = ctx->res.b.run;
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_download_results(smr_ctx* ctx, smr_read_result* results, smr_aln* alns, uint32_t* cigar_pool, uint64_t cigar_cap, uint64_t* cigar_used,
                         uint64_t* counters, uint32_t n_counters) try {
  if (!ctx || !results || !alns) return SMR_ERR_ARG;
  SMR_REFUSE_PACKED(ctx, "smr_download_results", "smr_download_results_packed")
  CK(cudaSetDevice(ctx->device));
  const uint32_t slots = slots_of(ctx);
  const uint32_t n = ctx->res.b.nreads;
  memset(results, 0, (size_t)n * sizeof(smr_read_result));
  memset(alns, 0, (size_t)n * slots * sizeof(smr_aln));
  HostOut out{results, alns, cigar_pool, cigar_cap, 0, counters, n_counters};
  const auto put_used = on_exit([&] { if (cigar_used) *cigar_used = out.cigar_used; });   // a pool too small fails, and names the words needed
  download_resident(ctx, out);
  return SMR_OK;
} SMR_CATCH(ctx)

// the packed calls' shared part: the results of the resident batch's last run, written as download_packed places them
static int packed_call(smr_ctx* ctx, smr_read_result* results, smr_aln* alns, uint64_t aln_cap, uint64_t* aln_used, smr_aln_stats* stats,
                uint32_t* cigar_pool, uint64_t cigar_cap, uint64_t* cigar_used, uint64_t* counters, uint32_t n_counters,
                const uint8_t* seq_cat, const uint64_t* seq_off, uint32_t nreads, bool align) try {
  if (!ctx) return SMR_ERR_ARG;
  if (!results || (!alns && aln_cap) || (!cigar_pool && cigar_cap) || (align && (!seq_cat || !seq_off))) { ctx->err = "null result array"; return SMR_ERR_ARG; }
  if (!packed(ctx)) { ctx->err = "the packed calls need smr_set_aln_layout(ctx, SMR_ALNS_PACKED)"; return SMR_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  PackedOut out{results, alns, aln_cap, stats, cigar_pool, cigar_cap, counters, n_counters};
  const auto put_used = on_exit([&] { if (aln_used) *aln_used = out.aln_used; if (cigar_used) *cigar_used = out.cigar_used; });
  if (align) {
    upload_batch_impl(ctx, seq_cat, seq_off, nreads);
    run_impl(ctx, ctx->res.b);
  }
  memset(results, 0, (size_t)ctx->res.b.nreads * sizeof(smr_read_result));
  download_packed(ctx, out);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_align_batch_packed(smr_ctx* ctx, const uint8_t* seq_cat, const uint64_t* seq_off, uint32_t nreads, smr_read_result* results,
                           smr_aln* alns, uint64_t aln_cap, uint64_t* aln_used, smr_aln_stats* stats, uint32_t* cigar_pool, uint64_t cigar_cap,
                           uint64_t* cigar_used, uint64_t* counters, uint32_t n_counters) {
  return packed_call(ctx, results, alns, aln_cap, aln_used, stats, cigar_pool, cigar_cap, cigar_used, counters, n_counters, seq_cat, seq_off, nreads, true);
}

int smr_download_results_packed(smr_ctx* ctx, smr_read_result* results, smr_aln* alns, uint64_t aln_cap, uint64_t* aln_used,
                                smr_aln_stats* stats, uint32_t* cigar_pool, uint64_t cigar_cap, uint64_t* cigar_used, uint64_t* counters,
                                uint32_t n_counters) {
  return packed_call(ctx, results, alns, aln_cap, aln_used, stats, cigar_pool, cigar_cap, cigar_used, counters, n_counters, nullptr, nullptr, 0, false);
}

int smr_set_report_refs(smr_ctx* ctx, uint32_t index_num, uint32_t part, const char* names_cat, const uint64_t* name_off, uint32_t nref) try {
  if (!ctx || !name_off || (!names_cat && name_off[nref])) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  for (Part& pt : ctx->parts) {
    if (pt.d.index_num != index_num || pt.d.part != part) continue;
    if (nref != pt.d.nref) { ctx->err = "smr_set_report_refs: " + std::to_string(nref) + " names for a part of " + std::to_string(pt.d.nref) + " references"; return SMR_ERR_ARG; }
    std::vector<char> names(names_cat, names_cat + name_off[nref]);
    std::vector<uint64_t> off(name_off, name_off + nref + 1);
    pt.rnames = part_array<char>(ctx, pt, names.size(), names.data());
    pt.rname_off = part_array<uint64_t>(ctx, pt, off.size(), off.data());
    CK(cudaStreamSynchronize(ctx->stream));
    pt.n_rnames = nref; pt.has_rnames = true;
    pt.h_rnames.resize(nref);
    for (uint32_t k = 0; k < nref; ++k) if (name_off[k + 1] > name_off[k]) pt.h_rnames[k].assign(names_cat + name_off[k], name_off[k + 1] - name_off[k]);
    ++ctx->parts_gen;
    return SMR_OK;
  }
  ctx->err = "smr_set_report_refs: index " + std::to_string(index_num) + " part " + std::to_string(part) + " is not loaded";
  return SMR_ERR_ARG;
} SMR_CATCH(ctx)

int smr_set_report_scoring(smr_ctx* ctx, uint32_t index_num, double lambda, double K, uint64_t full_ref, uint64_t full_read) try {
  if (!ctx || !(K > 0)) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  if (ctx->rpt_score.size() <= index_num) ctx->rpt_score.resize(index_num + 1);
  auto& sc = ctx->rpt_score[index_num];
  std::vector<double> ev(65536);
  std::vector<uint32_t> bits(65536);
  for (uint32_t s = 0; s < 65536; ++s) {   // report_blast.cpp:117-126, operand order kept
    const float b = (float)(lambda * s - std::log(K)) / (float)std::log(2);
    bits[s] = b > 0 ? (uint32_t)b : 0u;
    ev[s] = (double)K * full_ref * full_read * std::exp(-lambda * s);
  }
  ensure(sc.ev, ev.size() * 8);
  ensure(sc.bits, bits.size() * 4);
  CK(cudaMemcpy(sc.ev.p, ev.data(), ev.size() * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(sc.bits.p, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice));
  sc.set = true;
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_format_reports(smr_ctx* ctx, const smr_report_opts* opts, const char* text, uint64_t nbytes, const smr_read_result* results,
                       const smr_aln* alns, const uint32_t* cigar_pool, uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads,
                       char* out, uint64_t cap, uint64_t* stream_off) try {
  if (!ctx || !opts || !stream_off || (!text && nbytes)) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  format_reports_impl(ctx, opts, text, nbytes, results, alns, cigar_pool, cigar_words, stats, nreads, out, cap, stream_off, false, false);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_format_reports_gz(smr_ctx* ctx, const smr_report_opts* opts, const char* text, uint64_t nbytes, const smr_read_result* results,
                          const smr_aln* alns, const uint32_t* cigar_pool, uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads,
                          char* out, uint64_t cap, uint64_t* stream_off) try {
  if (!ctx || !opts || !stream_off || (!text && nbytes)) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  format_reports_impl(ctx, opts, text, nbytes, results, alns, cigar_pool, cigar_words, stats, nreads, out, cap, stream_off, true, false);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_format_blast_pairwise(smr_ctx* ctx, const smr_report_opts* opts, const char* text, uint64_t nbytes, const smr_read_result* results,
                              const smr_aln* alns, const uint32_t* cigar_pool, uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads,
                              char* out, uint64_t cap, uint64_t* stream_off) try {
  if (!ctx || !opts || !stream_off || (!text && nbytes)) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  format_reports_impl(ctx, opts, text, nbytes, results, alns, cigar_pool, cigar_words, stats, nreads, out, cap, stream_off, false, true);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_format_blast_pairwise_gz(smr_ctx* ctx, const smr_report_opts* opts, const char* text, uint64_t nbytes, const smr_read_result* results,
                                 const smr_aln* alns, const uint32_t* cigar_pool, uint64_t cigar_words, const smr_aln_stats* stats, uint32_t nreads,
                                 char* out, uint64_t cap, uint64_t* stream_off) try {
  if (!ctx || !opts || !stream_off || (!text && nbytes)) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  format_reports_impl(ctx, opts, text, nbytes, results, alns, cigar_pool, cigar_words, stats, nreads, out, cap, stream_off, true, true);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_gzip(smr_ctx* ctx, const void* in, uint64_t n, void* out, uint64_t cap, uint64_t* out_bytes) try {
  if (!ctx || !out_bytes || (!in && n)) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  *out_bytes = 0;
  cudaEvent_t* e = events(ctx, 4);
  CK(cudaEventRecord(e[0], ctx->stream));
  if (n == 0) {   // one empty member
    *out_bytes = sizeof kGzEmpty;
    if (!out || cap < sizeof kGzEmpty) { ctx->err = "output buffer too small: out_bytes holds the size"; return SMR_ERR_CAPACITY; }
    memcpy(out, kGzEmpty, sizeof kGzEmpty);
    ctx->t_rpt[0] = ctx->t_rpt[1] = ctx->t_rpt[2] = 0;
    return SMR_OK;
  }
  ensure(ctx->z.in, n + 64);
  CK(cudaMemsetAsync((uint8_t*)ctx->z.in.p + n, 0, 64, ctx->stream));
  CK(cudaMemcpyAsync(ctx->z.in.p, in, n, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaEventRecord(e[1], ctx->stream));
  uint64_t so[2] = {0, 0};
  {
    const auto put_size = on_exit([&] { *out_bytes = so[1]; });   // a buffer too small fails, and names the size needed
    gzip_streams(ctx, (const uint8_t*)ctx->z.in.p, {0}, {n}, (char*)out, cap, so, e[2], e[3]);
  }
  set_rpt_times(ctx, e);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_last_report_timings(const smr_ctx* ctx, double out[3]) {
  if (!ctx || !out) return SMR_ERR_ARG;
  for (int k = 0; k < 3; ++k) out[k] = ctx->t_rpt[k];
  return SMR_OK;
}

int smr_last_timings(const smr_ctx* ctx, double out[8]) {
  if (!ctx || !out) return SMR_ERR_ARG;
  out[0] = ctx->t_run.total; out[1] = ctx->t_run.seed; out[2] = ctx->t_run.lis; out[3] = ctx->t_run.final; out[4] = ctx->t_h2d; out[5] = ctx->t_d2h;
  out[6] = (double)ctx->t_run.launches; out[7] = ctx->t_decode;
  return SMR_OK;
}

int smr_debug_dpx_peak(smr_ctx* ctx, double* giga_ops_per_s) try {
  if (!ctx || !giga_ops_per_s) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  DevBuf d;
  CK(d.alloc(64));
  const int iters = 1 << 14, ctas = ctx->sm_count * 8, thr = 256;
  cudaEvent_t* e = events(ctx, 2);
  double best = 0;
  for (int rep = 0; rep < 4; ++rep) {
    CK(cudaEventRecord(e[0], ctx->stream));
    dpx_peak_kernel<<<ctas, thr, 0, ctx->stream>>>((int32_t*)d.p, iters, -2, -1000000);
    CK(cudaGetLastError());
    CK(cudaEventRecord(e[1], ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const double ms = elapsed_ms(e[0], e[1]);
    const double ops = (double)ctas * thr * iters * 8.0;
    if (rep > 0) best = std::max(best, ops / (ms * 1e-3) / 1e9);
  }
  *giga_ops_per_s = best;
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_debug_seed_windows(smr_ctx* ctx, uint32_t part_slot, const uint8_t* seq_cat, const uint64_t* seq_off, uint32_t nreads,
                           const uint32_t* win_read, const uint32_t* win_pos, uint32_t nwin, uint32_t* ids, uint32_t cap, uint32_t* counts,
                           uint8_t* zero) try {
  if (!ctx || part_slot >= ctx->parts.size() || !seq_cat || !seq_off || !win_read || !win_pos || !ids || !counts || !zero) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const uint32_t cap_arg = cap;
  cap &= 0x7FFFFFFFu;
  const uint64_t total = seq_off[nreads] - seq_off[0];
  std::vector<uint32_t> off32(nreads + 1);
  for (uint32_t r = 0; r <= nreads; ++r) off32[r] = (uint32_t)(seq_off[r] - seq_off[0]);
  std::vector<DevBuf> tmp;
  uint8_t* d_seq = scratch<uint8_t>(tmp, total + 64);
  uint32_t *d_off = scratch<uint32_t>(tmp, (size_t)nreads + 1), *d_wr = scratch<uint32_t>(tmp, (size_t)nwin + 1), *d_wp = scratch<uint32_t>(tmp, (size_t)nwin + 1),
           *d_ids = scratch<uint32_t>(tmp, (size_t)nwin * cap + 1), *d_cnt = scratch<uint32_t>(tmp, (size_t)nwin + 1);
  uint8_t* d_zero = scratch<uint8_t>(tmp, (size_t)nwin + 4);
  CK(cudaMemcpy(d_seq, seq_cat + seq_off[0], total, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_off, off32.data(), (size_t)(nreads + 1) * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_wr, win_read, (size_t)nwin * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_wp, win_pos, (size_t)nwin * 4, cudaMemcpyHostToDevice));
  CK(cudaMemset(d_ids, 0, (size_t)nwin * cap * 4));
  const Part& pt = ctx->parts[part_slot];
  DevIndex d = pt.d;
  if (!pt.search.p) {   // an index budget holds the part's search arrays on the host: a device copy for this call
    uint8_t* sb = scratch<uint8_t>(tmp, search_bytes(pt));
    CK(cudaMemcpy(sb, pt.host.p, search_bytes(pt), cudaMemcpyHostToDevice));
    set_search_ptrs(d, pt, sb);
  }
  const int mode = cap_arg >= 0x80000000u ? 1 : 0;   // high bit of cap selects the per-lane fallback path (tests exercise both)
  seed_debug_kernel<<<(nwin + kSeedWarpsPerCta * 32 - 1) / (kSeedWarpsPerCta * 32), kSeedWarpsPerCta * 32, 0, ctx->stream>>>(
      d, d_seq, d_off, d_wr, d_wp, nwin, d_ids, cap, d_cnt, d_zero, ctx->have_params ? ctx->prm.is_full_search : 0, mode);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaMemcpy(ids, d_ids, (size_t)nwin * cap * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(counts, d_cnt, (size_t)nwin * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(zero, d_zero, nwin, cudaMemcpyDeviceToHost));
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_debug_ssw(smr_ctx* ctx, const uint8_t* q_cat, const uint64_t* q_off, const uint8_t* t_cat, const uint64_t* t_off, uint32_t npairs,
                  uint32_t filters, int32_t* out, uint32_t* cigars, uint32_t cigar_cap) try {
  if (!ctx || !q_cat || !q_off || !t_cat || !t_off || !out || !cigars || !ctx->have_params) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const uint64_t qt = q_off[npairs] - q_off[0], tt = t_off[npairs] - t_off[0];
  std::vector<uint32_t> qo(npairs + 1), to(npairs + 1);
  uint32_t maxlen = 0;
  for (uint32_t i = 0; i <= npairs; ++i) { qo[i] = (uint32_t)(q_off[i] - q_off[0]); to[i] = (uint32_t)(t_off[i] - t_off[0]); }
  for (uint32_t i = 0; i < npairs; ++i) maxlen = std::max(maxlen, std::max(qo[i + 1] - qo[i], to[i + 1] - to[i]));
  std::vector<DevBuf> tmp;
  FinalGlobals g{};
  g.cap_w = 2 * 2048 + 8; g.cap_cig = 2 * (maxlen + 64) + 16; g.row_cap = maxlen + 128; g.cap_dir = (size_t)(2 * 64 + 1) * (maxlen + 8) * 3 + 65536;
  const uint32_t nwarps = 512;
  g.arena_stride = final_arena_bytes(g.cap_w, g.cap_cig, g.row_cap, g.cap_dir);
  g.arena_base = scratch<uint8_t>(tmp, g.arena_stride * nwarps);
  uint8_t *dq = scratch<uint8_t>(tmp, qt + 64), *dt = scratch<uint8_t>(tmp, tt + 64);
  uint32_t *dqo = scratch<uint32_t>(tmp, (size_t)npairs + 1), *dto = scratch<uint32_t>(tmp, (size_t)npairs + 1), *dc = scratch<uint32_t>(tmp, (size_t)npairs * cigar_cap + 1);
  int32_t* dout = scratch<int32_t>(tmp, (size_t)npairs * 6 + 1);
  CK(cudaMemcpy(dq, q_cat + q_off[0], qt, cudaMemcpyHostToDevice)); CK(cudaMemcpy(dt, t_cat + t_off[0], tt, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dqo, qo.data(), (size_t)(npairs + 1) * 4, cudaMemcpyHostToDevice)); CK(cudaMemcpy(dto, to.data(), (size_t)(npairs + 1) * 4, cudaMemcpyHostToDevice));
  CK(cudaMemset(dc, 0, (size_t)npairs * cigar_cap * 4));
  ssw_debug_kernel<<<nwarps / kFinalWarpsPerCta, kFinalWarpsPerCta * 32, 0, ctx->stream>>>(dq, dqo, dt, dto, npairs, filters, to_dev(ctx->prm), dout, dc,
                                                                                           cigar_cap, g);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaMemcpy(out, dout, (size_t)npairs * 6 * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(cigars, dc, (size_t)npairs * cigar_cap * 4, cudaMemcpyDeviceToHost));
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_otu_begin(smr_ctx* ctx, const smr_otu_opts* opts) try {
  if (!ctx || !opts) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  otu_begin_impl(ctx, opts);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_otu_add(smr_ctx* ctx, const char* text, uint64_t nbytes, const smr_read_result* results, const smr_aln* alns, const smr_aln_stats* stats,
                uint32_t nreads, uint64_t* n_added) try {
  if (!ctx || (!text && nbytes)) return SMR_ERR_ARG;
  if (n_added) *n_added = 0;
  CK(cudaSetDevice(ctx->device));
  const uint64_t m = otu_add_impl(ctx, text, nbytes, results, alns, stats, nreads);
  if (n_added) *n_added = m;
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_otu_finish(smr_ctx* ctx, char* out, uint64_t cap, uint64_t counts[3]) try {
  if (!ctx || !counts) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  otu_finish_impl(ctx, out, cap, counts);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_last_otu_timings(const smr_ctx* ctx, double out[3]) {
  if (!ctx || !out) return SMR_ERR_ARG;
  for (int k = 0; k < 3; ++k) out[k] = ctx->otu.t[k];
  return SMR_OK;
}

int smr_denovo_stats(smr_ctx* ctx, const smr_denovo_opts* opts, const char* text, uint64_t nbytes, const smr_read_result* results,
                     const smr_aln* alns, const smr_aln_stats* stats, uint32_t nreads, uint32_t* per_read, uint64_t totals[4]) try {
  if (!ctx || !opts || !totals || (!text && nbytes)) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  denovo_stats_impl(ctx, opts, text, nbytes, results, alns, stats, nreads, per_read, totals);
  return SMR_OK;
} SMR_CATCH(ctx)

// -- results placed on the device (smr_place.cuh) --
int smr_set_place_stats(smr_ctx* ctx, int on) {
  if (!ctx) return SMR_ERR_ARG;
  ctx->place_stats = on != 0;
  return SMR_OK;
}

// smr_place_results[_packed] past their layout refusals
static void place_results_impl(smr_ctx* ctx, const char* call, uint64_t* counters, uint32_t n_counters, uint64_t* n_alns, uint64_t* cigar_words) {
  CK(cudaSetDevice(ctx->device));
  place_once(ctx, call);
  const auto& P = ctx->pl;
  if (n_alns) *n_alns = P.n_alns;
  if (cigar_words) *cigar_words = P.cig_words;
  if (counters)
    for (uint32_t k = 0; k < n_counters && k < P.cnt_host.size(); ++k) counters[k] += P.cnt_host[k];
  if (P.trace) fail(SMR_ERR_INDEX, kTraceErrorMsg);
}

int smr_place_results(smr_ctx* ctx, uint64_t* counters, uint32_t n_counters, uint64_t* n_alns, uint64_t* cigar_words) try {
  if (!ctx) return SMR_ERR_ARG;
  if (n_alns) *n_alns = 0;
  if (cigar_words) *cigar_words = 0;
  if (packed(ctx)) {
    ctx->err = "smr_place_results places the strided layout only: in the packed layout call smr_download_results_packed";
    return SMR_ERR_UNSUPPORTED;
  }
  place_results_impl(ctx, "smr_place_results", counters, n_counters, n_alns, cigar_words);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_place_results_packed(smr_ctx* ctx, uint64_t* counters, uint32_t n_counters, uint64_t* n_alns, uint64_t* cigar_words) try {
  if (!ctx) return SMR_ERR_ARG;
  if (n_alns) *n_alns = 0;
  if (cigar_words) *cigar_words = 0;
  if (!packed(ctx)) {
    ctx->err = "smr_place_results_packed places the packed layout only: in the strided layout call smr_place_results";
    return SMR_ERR_ARG;
  }
  place_results_impl(ctx, "smr_place_results_packed", counters, n_counters, n_alns, cigar_words);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_download_placed(smr_ctx* ctx, smr_read_result* results, smr_aln* alns, smr_aln_stats* stats, uint32_t* cigar_pool, uint64_t cigar_cap) try {
  if (!ctx) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const PlacedArrays p = placed_of(ctx, "smr_download_placed", stats != nullptr);
  const uint64_t N = p.nslots;
  if (p.n && (!results || !alns)) fail(SMR_ERR_ARG, "smr_download_placed: null result array");
  if (p.cig_words > cigar_cap || (p.cig_words && !cigar_pool))
    fail(SMR_ERR_CAPACITY, "cigar pool too small: the batch needs " + std::to_string(p.cig_words) + " words, cigar_cap is " + std::to_string(cigar_cap));
  if (p.n) {
    CK(cudaMemcpyAsync(results, p.res, (size_t)p.n * sizeof(smr_read_result), cudaMemcpyDeviceToHost, ctx->stream));
    if (N) CK(cudaMemcpyAsync(alns, p.aln, N * sizeof(smr_aln), cudaMemcpyDeviceToHost, ctx->stream));
    if (stats && N) CK(cudaMemcpyAsync(stats, p.st, N * sizeof(smr_aln_stats), cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (p.cig_words) CK(cudaMemcpyAsync(cigar_pool, p.cig, p.cig_words * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_last_place_timing(const smr_ctx* ctx, double* ms) {
  if (!ctx || !ms) return SMR_ERR_ARG;
  *ms = ctx->pl.t_place;
  return SMR_OK;
}

// the report-side calls on the placed results: format_reports_impl and the rest with dev = true
static int format_placed(smr_ctx* ctx, const char* call, const smr_report_opts* o, char* out, uint64_t cap, uint64_t* stream_off, bool gz,
                         bool pairwise) try {
  if (!ctx || !o || !stream_off) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const PlacedArrays p = placed_of(ctx, call, o->sam || (o->blast && !pairwise) || o->denovo);
  format_reports_impl(ctx, o, nullptr, 0, p.res, p.aln, p.cig, p.cig_words, p.st, p.n, out, cap, stream_off, gz, pairwise, true);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_format_reports_placed(smr_ctx* ctx, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* stream_off) {
  return format_placed(ctx, "smr_format_reports_placed", opts, out, cap, stream_off, false, false);
}
int smr_format_reports_placed_gz(smr_ctx* ctx, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* stream_off) {
  return format_placed(ctx, "smr_format_reports_placed_gz", opts, out, cap, stream_off, true, false);
}
int smr_format_blast_pairwise_placed(smr_ctx* ctx, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* stream_off) {
  return format_placed(ctx, "smr_format_blast_pairwise_placed", opts, out, cap, stream_off, false, true);
}
int smr_format_blast_pairwise_placed_gz(smr_ctx* ctx, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* stream_off) {
  return format_placed(ctx, "smr_format_blast_pairwise_placed_gz", opts, out, cap, stream_off, true, true);
}

int smr_format_bam_placed(smr_ctx* ctx, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* stream_off) try {
  if (!ctx || !opts || !stream_off) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const PlacedArrays p = placed_of(ctx, "smr_format_bam_placed", true);
  format_reports_impl(ctx, opts, nullptr, 0, p.res, p.aln, p.cig, p.cig_words, p.st, p.n, out, cap, stream_off, false, false, true, true);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_bam_header(smr_ctx* ctx, const char* text, uint64_t nbytes, char* out, uint64_t cap, uint64_t* out_bytes) try {
  if (!ctx || !out_bytes || (!text && nbytes)) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  *out_bytes = 0;
  if (nbytes > 0x7FFFFFFFull) fail(SMR_ERR_ARG, "BAM header: a text of 2^31 bytes or more");
  cudaEvent_t* e = events(ctx, 4);
  CK(cudaEventRecord(e[0], ctx->stream));
  // magic, l_text, text, n_ref, then (l_name, name NUL, l_ref) of every reference in the refID order of rpt_groups
  std::vector<uint8_t> h;
  auto le32 = [&](uint32_t v) { for (int k = 0; k < 4; ++k) h.push_back((uint8_t)(v >> (8 * k))); };
  h.insert(h.end(), {'B', 'A', 'M', 1});
  le32((uint32_t)nbytes);
  h.insert(h.end(), text, text + nbytes);
  const std::vector<RptGroup> hg = rpt_groups(ctx, true, false);
  const std::vector<const Part*> gp = report_groups(ctx);
  le32(hg.empty() ? 0 : hg.back().ref_base + hg.back().nref);
  for (size_t g = 0; g < gp.size(); ++g) {
    std::vector<uint32_t> roff((size_t)hg[g].nref + 1);
    CK(cudaMemcpy(roff.data(), hg[g].ref_off, roff.size() * 4, cudaMemcpyDeviceToHost));
    for (uint32_t k = 0; k < hg[g].nref; ++k) {
      const std::string& name = gp[g]->h_rnames[k];
      le32((uint32_t)name.size() + 1);
      h.insert(h.end(), name.begin(), name.end());
      h.push_back(0);
      le32(roff[k + 1] - roff[k]);
    }
  }
  const uint64_t n = h.size();
  ensure(ctx->z.in, n + 64);
  CK(cudaMemsetAsync((uint8_t*)ctx->z.in.p + n, 0, 64, ctx->stream));
  CK(cudaMemcpyAsync(ctx->z.in.p, h.data(), n, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaEventRecord(e[1], ctx->stream));
  std::vector<uint64_t> sb, se;
  bgzf_blocks(0, n, sb, se);
  std::vector<uint64_t> so(sb.size() + 1, 0);
  {
    const auto put_size = on_exit([&] { *out_bytes = so.back(); });   // a buffer too small fails, and names the size needed
    gzip_streams(ctx, (const uint8_t*)ctx->z.in.p, sb, se, out, cap, so.data(), e[2], e[3], kBgzfHeader);
  }
  set_rpt_times(ctx, e);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_bam_sort_begin(smr_ctx* ctx) try {
  if (!ctx) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  bam_sort_begin_impl(ctx);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_bam_sort_add_placed(smr_ctx* ctx, const smr_report_opts* opts, char* out, uint64_t cap, uint64_t* nbytes) try {
  if (!ctx || !opts || !nbytes) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  *nbytes = 0;
  bam_sort_add_impl(ctx, opts, out, cap, nbytes);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_bam_sort_plan(smr_ctx* ctx, uint64_t window_bytes, uint64_t header_bytes, uint64_t* ranges, uint64_t cap, uint64_t* n_windows) try {
  if (!ctx || !n_windows) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  *n_windows = 0;
  bam_sort_plan_impl(ctx, window_bytes, header_bytes, ranges, cap, n_windows);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_bam_sort_window(smr_ctx* ctx, uint64_t w, const void* staged, uint64_t nbytes, char* out, uint64_t cap, uint64_t* out_bytes) try {
  if (!ctx || !out_bytes) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  *out_bytes = 0;
  bam_sort_window_impl(ctx, w, staged, nbytes, out, cap, out_bytes);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_bam_sort_index(smr_ctx* ctx, char* out, uint64_t cap, uint64_t* nbytes) try {
  if (!ctx || !nbytes) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  *nbytes = 0;
  bam_sort_index_impl(ctx, out, cap, nbytes);
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_otu_add_placed(smr_ctx* ctx, uint64_t* n_added) try {
  if (!ctx) return SMR_ERR_ARG;
  if (n_added) *n_added = 0;
  CK(cudaSetDevice(ctx->device));
  const PlacedArrays p = placed_of(ctx, "smr_otu_add_placed", true);
  const uint64_t m = otu_add_impl(ctx, nullptr, 0, p.res, p.aln, p.st, p.n, true);
  if (n_added) *n_added = m;
  return SMR_OK;
} SMR_CATCH(ctx)

int smr_denovo_stats_placed(smr_ctx* ctx, const smr_denovo_opts* opts, uint32_t* per_read, uint64_t totals[4]) try {
  if (!ctx || !opts || !totals) return SMR_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  const PlacedArrays p = placed_of(ctx, "smr_denovo_stats_placed", true);
  denovo_stats_impl(ctx, opts, nullptr, 0, p.res, p.aln, p.st, p.n, per_read, totals, true);
  return SMR_OK;
} SMR_CATCH(ctx)

}  // extern "C"
