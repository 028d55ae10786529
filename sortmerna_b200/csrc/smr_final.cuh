// Finalize: for every STORED alignment, the reverse Smith-Waterman pass (begin coordinates,
// src/sortmerna/ssw.c:899-915) and the banded traceback (CIGAR, ssw.c:917-935 -> banded_sw :577-773),
// then the coordinate shift of compute_lis_alignment (src/sortmerna/alignment.cpp:394-405).
// The reference computes both for every ssw_align call that reaches the score filter (on average
// 7-14 calls per read); they are pure functions of (query segment, reference window, score), so
// computing them once per alignment that survives is equivalent.
#pragma once
#include "smr_lis.cuh"

namespace smr {

// layout-compatible with smr_aln (include/smr_b200.h)
struct OutAln {
  uint32_t cigar_off, cigar_len, ref_num;
  int32_t ref_begin1, ref_end1, read_begin1, read_end1;
  uint32_t readlen;
  uint16_t score1, part, index_num;
  uint8_t strand, pad;
};

// what the traceback stage needs for one stored alignment (filled by finalize_kernel, indexed like the job list)
struct TraceJob {
  uint32_t valid;          // 0: a locate pass failed (kErrTrace is set on the read), no traceback
  uint32_t idx_slot, ref_num, ref_off;   // reference window start = refseq[ref_off[ref_num] + ref_off]
  int32_t q_start, q_step;               // query view start / step into seq04 of the read (step -1 + complement for the minus strand)
  int32_t rl, ql, score, band;
};

struct AlnStats { uint32_t n_miss, n_gap, n_match, n_match_denovo; };   // layout of smr_aln_stats

struct FinalGlobals {
  uint8_t* arena_base; size_t arena_stride;
  uint32_t cap_w, cap_cig, row_cap; size_t cap_dir;
  const DevIndex* parts;             // [nparts] device copy of every loaded part, by DevIndex::gslot (refseq / ref_off only are read)
  const AlnWork* aln_work; OutAln* out;
  union {                            // one or the other, as in LisGlobals (a larger FinalGlobals changes the strided kernels' code)
    uint32_t slots;                  // <kPacked = false> kernels: read r's alignments at r * slots
    const uint32_t* aln_base;        // <kPacked = true> kernels: [nreads + 1] packed arenas (LisGlobals::aln_base)
  };
  uint32_t* cigar_pool; unsigned long long cigar_cap; unsigned long long* cigar_used;
  uint32_t* work_next;
  // the stored alignments of the chunk: job_list[0 .. *job_count) = slots of the chunk from its first one (final_slot)
  uint32_t* job_list; uint32_t* job_count;
  // traceback stage (one THREAD per alignment)
  struct TraceJob* jobs;             // [slots of the chunk], indexed like job_list
  uint8_t* tb_arena; size_t tb_stride; uint32_t tb_cap_w, tb_cap_cig; size_t tb_cap_dir;
  AlnStats* stats;                   // indexed like out, or nullptr
};

// Slot wi of the chunk (counted from the chunk's first slot): its read r, its index k among r's alignments, and (packed) `at`, its
// index in aln_work / out / stats (final_at).  Strided: wi = (read in chunk) * slots + k.  Packed: r is the last read whose first
// slot is at or before at.
struct FinalSlot { uint32_t r, k; size_t at; };
__device__ __noinline__ FinalSlot final_slot_packed(const uint32_t* __restrict__ base, const uint32_t r0, const uint32_t n, const uint32_t wi) {
  const uint32_t at = base[r0] + wi;
  uint32_t lo = r0, hi = r0 + n - 1;
  while (lo < hi) { const uint32_t m = (lo + hi + 1) / 2; if (base[m] <= at) lo = m; else hi = m - 1; }
  return FinalSlot{lo, at - base[lo], at};
}
__device__ __forceinline__ FinalSlot final_slot_strided(const DevBatch& b, const FinalGlobals& g, const uint32_t wi) {
  return FinalSlot{b.r0 + wi / g.slots, wi % g.slots, 0};
}
template <bool kPacked>
__device__ __forceinline__ FinalSlot final_slot(const DevBatch& b, const FinalGlobals& g, const uint32_t wi) {
  return kPacked ? final_slot_packed(g.aln_base, b.r0, b.nreads, wi) : final_slot_strided(b, g, wi);
}
// the index of slot s in aln_work / out / stats (strided: computed where it is used, so that the strided kernels keep their code)
template <bool kPacked>
__device__ __forceinline__ size_t final_at(const FinalGlobals& g, const FinalSlot& s) { return kPacked ? s.at : (size_t)s.r * g.slots + s.k; }
__host__ __device__ inline size_t final_arena_bytes(uint32_t cap_w, uint32_t cap_cig, uint32_t row_cap, size_t cap_dir) {
  size_t b = (size_t)cap_w * 12 + (size_t)cap_cig * 4 + (size_t)row_cap * 8 + cap_dir;
  return (b + 255) & ~(size_t)255;
}

constexpr int kFinalWarpsPerCta = 4;
#ifndef SMR_FINAL_MIN_CTAS
#define SMR_FINAL_MIN_CTAS 6     // resident CTAs per SM the register budget is set for (3: 167 registers, 4: 128, 5: 96, 6: 80; more CTAs were faster)
#endif
constexpr int kFinalCtasPerSm = SMR_FINAL_MIN_CTAS;

// the dense job list: every live (read, slot) of the chunk -- slot k < n_align of a read without flags -- in any order.  A read
// flagged kOvfSlots is not traced back: its alignments are stored again by a run at its own size, or the call fails.
template <bool kPacked>
__global__ void __launch_bounds__(256)
final_jobs_kernel(DevBatch b, FinalGlobals g) {
  const uint32_t total = kPacked ? g.aln_base[b.r0 + b.nreads] - g.aln_base[b.r0] : b.nreads * g.slots;
  const unsigned lane = lane_id();
  for (uint32_t w0 = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; w0 < total; w0 += gridDim.x * blockDim.x) {
    const uint32_t wi = w0 + lane;
    bool live = false;
    if (wi < total) {
      const FinalSlot s = final_slot<kPacked>(b, g, wi);
      live = s.k < b.state[s.r].n_align && !b.flags[s.r];
    }
    const unsigned m = __ballot_sync(kFull, live);
    if (!m) continue;
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(g.job_count, (uint32_t)__popc(m));
    base = __shfl_sync(kFull, base, 0);
    if (live) g.job_list[base + __popc(m & ((1u << lane) - 1u))] = wi;
  }
}

// Per warp shared memory of the finalize kernels: the packed passes' two query profiles and two windows.
struct FinalSmem {
  uint32_t prof[2 * kPairProfWords];
  __align__(16) uint8_t win[2][kPairWinBytes];
};

__device__ __forceinline__ TraceArena final_arena(const FinalGlobals& g, const uint32_t warp, int32_t*& rowH, int32_t*& rowF) {
  uint8_t* p = g.arena_base + (size_t)warp * g.arena_stride;
  TraceArena A;
  A.cap_w = g.cap_w; A.cap_cig = g.cap_cig; A.cap_dir = g.cap_dir; A.stride = 1;
  A.hb = (int32_t*)p; p += (size_t)g.cap_w * 4;
  A.eb = (int32_t*)p; p += (size_t)g.cap_w * 4;
  A.hc = (int32_t*)p; p += (size_t)g.cap_w * 4;
  A.cig = (uint32_t*)p; p += (size_t)g.cap_cig * 4;
  rowH = (int32_t*)p; p += (size_t)g.row_cap * 4;
  rowF = (int32_t*)p; p += (size_t)g.row_cap * 4;
  A.dir = (int8_t*)p;
  return A;
}

// the locate problem of stored alignment wi (final_slot): query segment, window, score
template <bool kPacked>
__device__ __forceinline__ PairLoc final_loc(const DevBatch& b, const FinalGlobals& g, const uint32_t wi) {
  const FinalSlot s = final_slot<kPacked>(b, g, wi);
  const uint32_t r = s.r;
  const AlnWork a = g.aln_work[final_at<kPacked>(g, s)];
  const DevIndex& ix = g.parts[a.idx_slot];
  const uint32_t seq_base = b.seq_off[r], len = b.seq_off[r + 1] - seq_base;
  PairLoc L;
  L.q = a.strand ? SeqView{b.seq04 + seq_base, (int32_t)a.q_start, 1, false} : SeqView{b.seq04 + seq_base, (int32_t)(len - 1 - a.q_start), -1, true};
  L.t = SeqView{ix.refseq + ix.ref_off[a.ref_num], (int32_t)a.win_ref_start, 1, false};
  L.m = (int32_t)a.q_len; L.n = (int32_t)a.win_len; L.target = (int32_t)a.score1;
  return L;
}
__device__ __forceinline__ bool final_packed(const PairLoc& L, const SwScore sc) { return L.target > 0 && L.m > 0 && sw_pair_ok(L.m, L.n, sc); }
__device__ __forceinline__ PairLoc no_loc() { return PairLoc{SeqView{nullptr, 0, 1, false}, 0, SeqView{nullptr, 0, 1, false}, 0, 0}; }
// the reverse problem: the prefixes that end at the forward end point (column<<16 | row), reversed (ssw.c:899-915)
__device__ __forceinline__ PairLoc reverse_loc(const PairLoc& L, const uint32_t e) {
  const int32_t ref = (int32_t)(e >> 16), read = (int32_t)(e & 0xFFFFu);
  return PairLoc{L.q.reversed_prefix(read), read + 1, L.t.reversed_prefix(ref), ref + 1, L.target};
}

// The rest of one job after the packed passes: packed = both end points came from them (kPairNoHit: no cell held the score);
// otherwise sw_forward runs here, forward and on the reversed prefixes ending at its end point.  Then the output row and the
// traceback job.
template <bool kPacked>
__device__ __noinline__ void final_finish(const DevBatch& b, const SwScore sc, const FinalGlobals& g, int32_t* rowH, int32_t* rowF,
                                          const uint32_t ji, const uint32_t wi, const bool packed, const uint32_t ef, const uint32_t er) {
  const unsigned lane = lane_id();
  const PairLoc L = final_loc<kPacked>(b, g, wi);
  SwEnd fwd{0, -1, 0}, rev{0, -1, 0};
  if (packed) {
    if (ef != kPairNoHit) fwd = SwEnd{L.target, (int32_t)(ef >> 16), (int32_t)(ef & 0xFFFFu)};
    if (er != kPairNoHit) rev = SwEnd{L.target, (int32_t)(er >> 16), (int32_t)(er & 0xFFFFu)};
  } else {
    fwd = sw_forward(L.q, L.m, L.t, L.n, sc, rowH, rowF);
    if ((fwd.score & 0xFFFF) == L.target) rev = sw_forward(L.q.reversed_prefix(fwd.read), fwd.read + 1, L.t.reversed_prefix(fwd.ref), fwd.ref + 1, sc, rowH, rowF);
  }
  if (lane != 0) return;
  const FinalSlot s = final_slot<kPacked>(b, g, wi);
  const uint32_t r = s.r;
  TraceJob j;
  if ((fwd.score & 0xFFFF) != L.target || rev.score != L.target) {
    atomicOr(&b.flags[r], kErrTrace);
    j.valid = 0;
    g.jobs[ji] = j;
    return;
  }
  const AlnWork a = g.aln_work[final_at<kPacked>(g, s)];
  const int32_t a_ref_end = fwd.ref, a_read_end = fwd.read;
  const int32_t ref_begin = a_ref_end - rev.ref, read_begin = a_read_end - rev.read;
  const int32_t rl = a_ref_end - ref_begin + 1, ql = a_read_end - read_begin + 1;
  const int32_t band = (rl > ql ? rl - ql : ql - rl) + 1;                                  // ssw.c:924
  OutAln o;
  o.cigar_off = 0; o.cigar_len = 0; o.ref_num = a.ref_num;
  o.ref_begin1 = ref_begin + (int32_t)a.win_ref_start; o.ref_end1 = a_ref_end + (int32_t)a.win_ref_start;   // alignment.cpp:396-399
  o.read_begin1 = read_begin + (int32_t)a.q_start; o.read_end1 = a_read_end + (int32_t)a.q_start;
  o.readlen = b.seq_off[r + 1] - b.seq_off[r]; o.score1 = a.score1; o.part = a.part; o.index_num = a.index_num; o.strand = a.strand; o.pad = 0;
  g.out[final_at<kPacked>(g, s)] = o;
  const SeqView qs = L.q.sub(read_begin);
  j.valid = 1; j.idx_slot = a.idx_slot; j.ref_num = a.ref_num; j.ref_off = a.win_ref_start + (uint32_t)ref_begin;
  j.q_start = qs.start; j.q_step = qs.step; j.rl = rl; j.ql = ql; j.score = (int32_t)a.score1; j.band = band;
  g.jobs[ji] = j;
}

// Forward pass again, now with the end-point tie-breaks (ssw.c:310-336), then the reverse pass over the prefixes that end at the
// forward optimum, for the jobs job_list[2i], job_list[2i + 1] of a warp: both in one packed pass (sw_pair_run) where their
// shapes and the scores allow it (sw_pair_ok), sw_forward otherwise; a lone last job runs with an empty second half.  kPacked: as
// traceback_kernel.
template <bool kPacked>
__global__ void __launch_bounds__(kFinalWarpsPerCta * 32, kFinalCtasPerSm)
finalize_kernel(DevBatch b, DevParams prm, FinalGlobals g) {
  __shared__ FinalSmem s_fin[kFinalWarpsPerCta];
  const unsigned lane = lane_id();
  const uint32_t warp = blockIdx.x * kFinalWarpsPerCta + (threadIdx.x >> 5);
  int32_t *rowH, *rowF;
  final_arena(g, warp, rowH, rowF);
  FinalSmem& S = s_fin[threadIdx.x >> 5];
  const SwScore sc{prm.match, prm.mismatch, prm.score_N, prm.gap_open, prm.gap_ext, prm.one};
  const uint32_t njobs = *g.job_count;
  for (;;) {
    uint32_t j0 = 0;
    if (lane == 0) j0 = atomicAdd(g.work_next, 2u);
    j0 = __shfl_sync(kFull, j0, 0);
    if (j0 >= njobs) break;
    const bool two = j0 + 1 < njobs;
    const uint32_t w0 = g.job_list[j0], w1 = two ? g.job_list[j0 + 1] : 0u;
    uint2 ef = make_uint2(kPairNoHit, kPairNoHit), er = ef;
    bool p0, p1;
    {
      const PairLoc L0 = final_loc<kPacked>(b, g, w0), L1 = two ? final_loc<kPacked>(b, g, w1) : no_loc();
      p0 = final_packed(L0, sc); p1 = two && final_packed(L1, sc);
      if (p0 || p1) ef = sw_pair_run<true>(p0 ? L0 : no_loc(), p1 ? L1 : no_loc(), sc, S.prof, S.win[0], S.win[1]);
    }
    const bool r0 = p0 && ef.x != kPairNoHit, r1 = p1 && ef.y != kPairNoHit;
    if (r0 || r1) {
      const PairLoc R0 = r0 ? reverse_loc(final_loc<kPacked>(b, g, w0), ef.x) : no_loc(), R1 = r1 ? reverse_loc(final_loc<kPacked>(b, g, w1), ef.y) : no_loc();
      er = sw_pair_run<true>(R0, R1, sc, S.prof, S.win[0], S.win[1]);
    }
    final_finish<kPacked>(b, sc, g, rowH, rowF, j0, w0, p0, ef.x, er.x);
    if (two) final_finish<kPacked>(b, sc, g, rowH, rowF, j0 + 1, w1, p1, ef.y, er.y);
    __syncwarp();
  }
}

// banded_sw (ssw.c:577-773) for every stored alignment, one THREAD per alignment (the DP rows are a serial chain of
// 3..2*band+1 cells; 32 alignments per warp keep the lanes busy where one-lane-per-warp left 31 idle).  kPacked: the run's arenas
// are packed (g.aln_base); the strided instantiation is the code it was before packed arenas existed.
template <bool kPacked>
__global__ void __launch_bounds__(128)
traceback_kernel(DevBatch b, DevParams prm, FinalGlobals g) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nthreads = gridDim.x * blockDim.x;
  const uint32_t lane = threadIdx.x & 31;
  // the 32 arenas of a warp are interleaved element-wise: lanes walking their own band in step touch consecutive addresses
  uint8_t* p = g.tb_arena + (size_t)(tid >> 5) * g.tb_stride * 32;
  TraceArena A;
  A.cap_w = g.tb_cap_w; A.cap_cig = g.tb_cap_cig; A.cap_dir = g.tb_cap_dir; A.stride = 32;
  A.hb = (int32_t*)p + lane; p += (size_t)g.tb_cap_w * 4 * 32;
  A.eb = (int32_t*)p + lane; p += (size_t)g.tb_cap_w * 4 * 32;
  A.hc = (int32_t*)p + lane; p += (size_t)g.tb_cap_w * 4 * 32;
  A.cig = (uint32_t*)p + lane; p += (size_t)g.tb_cap_cig * 4 * 32;
  A.dir = (int8_t*)p + lane;
  const SwScore sc{prm.match, prm.mismatch, prm.score_N, prm.gap_open, prm.gap_ext, prm.one};
  const uint32_t njobs = *g.job_count;
  for (uint32_t ji = tid; ji < njobs; ji += nthreads) {
    const TraceJob j = g.jobs[ji];
    if (!j.valid) continue;
    const uint32_t wi = g.job_list[ji];
    const FinalSlot s = final_slot<kPacked>(b, g, wi);
    const uint32_t r = s.r;
    const DevIndex& ix = g.parts[j.idx_slot];
    const SeqView t{ix.refseq + ix.ref_off[j.ref_num], (int32_t)j.ref_off, 1, false};
    const SeqView q{b.seq04 + b.seq_off[r], j.q_start, j.q_step, j.q_step < 0};
    for (uint32_t i = 0; i < g.tb_cap_w; ++i) { A.hb[i * 32] = 0; A.eb[i * 32] = 0; A.hc[i * 32] = 0; }
    const int32_t nc = banded_traceback_lane(t, q, j.rl, j.ql, j.score, sc, j.band, A);
    if (nc < 0) { atomicOr(&b.flags[r], nc == -1 ? kOvfTrace : kErrTrace); continue; }
    const unsigned long long off = atomicAdd(g.cigar_used, (unsigned long long)nc);
    if (off + (unsigned long long)nc > g.cigar_cap) { atomicOr(&b.flags[r], kOvfCigar); continue; }
    for (int32_t i = 0; i < nc; ++i) g.cigar_pool[off + i] = A.cig[(size_t)(nc - 1 - i) * 32];        // ssw.c:750-758 (reverse)
    const size_t at = final_at<kPacked>(g, s);
    OutAln* o = g.out + at;
    o->cigar_off = (uint32_t)off; o->cigar_len = (uint32_t)nc;
    if (g.stats) {   // Read::calc_miss_gap_match (read.cpp:547-589): walk the CIGAR over the 0-4 codes of reference and read
      // qd: the read as denovo_stats_run sees it (processor.cpp:329-333: 0-4 codes, never reverse-complemented)
      const SeqView qd{b.seq04 + b.seq_off[r], o->read_begin1, 1, false};
      uint32_t miss = 0, gap = 0, match = 0, match_d = 0;
      int32_t x = 0, y = 0;
      for (int32_t i = nc - 1; i >= 0; --i) {
        const uint32_t c = A.cig[(size_t)i * 32], op = c & 0xFu, ln = c >> 4;
        if (op == 0) {
          for (uint32_t u = 0; u < ln; ++u, ++x, ++y) {
            const uint32_t tc = t.at(x);
            if (tc != q.at(y)) ++miss; else ++match;
            match_d += tc == qd.at(y);
          }
        }
        else if (op == 1) { y += (int32_t)ln; gap += ln; }
        else { x += (int32_t)ln; gap += ln; }
      }
      g.stats[at] = AlnStats{miss, gap, match, match_d};
    }
  }
}

// unit-test kernel: full ssw_align(flag=2) equivalent on explicit pairs, one warp per pair (smr_debug_ssw).  The packed kernel is
// checked against the s32 arg-max kernel sw_forward, the pairs (2i, 2i + 1) in one pass as the candidate and finalize kernels run
// them; a pair outside sw_pair_ok is left out.  A disagreement replaces the score with a marker: -12345 the packed score pass (the
// candidate kernel's), -12347 the packed locate (the finalize kernel's), forward and on the reversed prefixes.
__global__ void __launch_bounds__(kFinalWarpsPerCta * 32)
ssw_debug_kernel(const uint8_t* qcat, const uint32_t* qoff, const uint8_t* tcat, const uint32_t* toff, uint32_t npairs, uint32_t filters,
                 DevParams prm, int32_t* out, uint32_t* cigars, uint32_t cigar_cap, FinalGlobals g) {
  __shared__ FinalSmem s_fin[kFinalWarpsPerCta];
  const unsigned lane = lane_id();
  const uint32_t warp = blockIdx.x * kFinalWarpsPerCta + (threadIdx.x >> 5), nwarps = gridDim.x * kFinalWarpsPerCta;
  int32_t *rowH, *rowF;
  TraceArena A = final_arena(g, warp, rowH, rowF);
  FinalSmem& S = s_fin[threadIdx.x >> 5];
  const SwScore sc{prm.match, prm.mismatch, prm.score_N, prm.gap_open, prm.gap_ext, prm.one};
  for (uint32_t k0 = 2 * warp; k0 < npairs; k0 += 2 * nwarps) {
    PairLoc P[2], L[2], RL[2];
    SwEnd fe[2], re[2];
#pragma unroll 1
    for (uint32_t h = 0; h < 2; ++h) {
      P[h] = no_loc(); L[h] = no_loc(); RL[h] = no_loc();
      const uint32_t k = k0 + h;
      if (k >= npairs) break;
      const int32_t m = (int32_t)(qoff[k + 1] - qoff[k]), n = (int32_t)(toff[k + 1] - toff[k]);
      const SeqView q{qcat + qoff[k], 0, 1, false}, t{tcat + toff[k], 0, 1, false};
      int32_t* o = out + (size_t)k * 6;
      const SwEnd f = sw_forward(q, m, t, n, sc, rowH, rowF);
      if (m > 0 && sw_pair_ok(m, n, sc)) {
        P[h] = PairLoc{q, m, t, n, f.score};
        if (f.score > 0) {
          L[h] = P[h];
          fe[h] = f;
          RL[h] = PairLoc{q.reversed_prefix(f.read), f.read + 1, t.reversed_prefix(f.ref), f.ref + 1, f.score};
          re[h] = sw_forward(RL[h].q, RL[h].m, RL[h].t, RL[h].n, sc, rowH, rowF);
        }
      }
      int32_t rb = -1, qb = -1, nc = 0;
      if ((uint32_t)(f.score & 0xFFFF) >= filters && f.score > 0) {
        const SwEnd rev = sw_forward(q.reversed_prefix(f.read), f.read + 1, t.reversed_prefix(f.ref), f.ref + 1, sc, rowH, rowF);
        rb = f.ref - rev.ref; qb = f.read - rev.read;
        const int32_t rl = f.ref - rb + 1, ql = f.read - qb + 1;
        for (uint32_t i = lane; i < g.cap_w; i += 32) { A.hb[i] = 0; A.eb[i] = 0; A.hc[i] = 0; }
        __syncwarp();
        if (lane == 0) nc = banded_traceback_lane(t.sub(rb), q.sub(qb), rl, ql, f.score, sc, (rl > ql ? rl - ql : ql - rl) + 1, A);
        nc = __shfl_sync(kFull, nc, 0);
        __syncwarp();
        for (int32_t i = lane; i < nc && i < (int32_t)cigar_cap; i += 32) cigars[(size_t)k * cigar_cap + i] = A.cig[nc - 1 - i];
      }
      if (lane == 0) { o[0] = f.score; o[1] = rb; o[2] = f.ref; o[3] = qb; o[4] = f.read; o[5] = nc; }
      __syncwarp();
    }
    // the packed score pass of both pairs at once, best scores of 0 included
    if (P[0].m || P[1].m) {
      const uint32_t s2 = sw_pair_run<false>(P[0], P[1], sc, S.prof, S.win[0], S.win[1]);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (P[h].m && (h ? s2 >> 16 : s2 & 0xFFFFu) != (uint32_t)P[h].target && lane == 0) out[(size_t)(k0 + h) * 6] = -12345;
      __syncwarp();
    }
    // the packed locate of both pairs at once, forward and on the reversed prefixes ending at each pair's own end point
    if (L[0].m || L[1].m) {
      const uint2 ef = sw_pair_run<true>(L[0], L[1], sc, S.prof, S.win[0], S.win[1]);
      const uint2 er = sw_pair_run<true>(RL[0], RL[1], sc, S.prof, S.win[0], S.win[1]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!L[h].m) continue;
        const uint32_t wf = ((uint32_t)fe[h].ref << 16) | (uint32_t)fe[h].read, wr = ((uint32_t)re[h].ref << 16) | (uint32_t)re[h].read;
        const bool bad = (h ? ef.y : ef.x) != wf || re[h].score != L[h].target || (h ? er.y : er.x) != wr;
        if (bad && lane == 0) out[(size_t)(k0 + h) * 6] = -12347;
      }
      __syncwarp();
    }
  }
}

// DPX issue-rate micro-benchmark: 8 independent VIADDMNMX chains per thread (the dependent-free peak SURVEY 8(d)
// asks to measure on the box instead of quoting a datasheet).  out[0] receives a value so nothing is optimised away.
__global__ void dpx_peak_kernel(int32_t* out, int iters, int32_t a, int32_t b) {
  int32_t x0 = threadIdx.x, x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3, x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
  for (int i = 0; i < iters; ++i) {
    x0 = __viaddmax_s32(x0, a, b); x1 = __viaddmax_s32(x1, a, b); x2 = __viaddmax_s32(x2, a, b); x3 = __viaddmax_s32(x3, a, b);
    x4 = __viaddmax_s32(x4, a, b); x5 = __viaddmax_s32(x5, a, b); x6 = __viaddmax_s32(x6, a, b); x7 = __viaddmax_s32(x7, a, b);
  }
  if ((x0 ^ x1 ^ x2 ^ x3 ^ x4 ^ x5 ^ x6 ^ x7) == 0x7fffffff) out[0] = x0;
}

}  // namespace smr
