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

// what the traceback stage needs for one stored alignment (filled by finalize_kernel)
struct TraceJob {
  uint32_t valid;          // 1 = traceback wanted
  uint32_t idx_slot, ref_num, ref_off;   // reference window start = refseq[ref_off[ref_num] + ref_off]
  int32_t q_start, q_step;               // query view start / step into seq04 of the read (step -1 + complement for the minus strand)
  int32_t rl, ql, score, band;
};

struct AlnStats { uint32_t n_miss, n_gap, n_match, n_match_denovo; };   // layout of smr_aln_stats

struct FinalGlobals {
  uint8_t* arena_base; size_t arena_stride;
  uint32_t cap_w, cap_cig, row_cap; size_t cap_dir;
  const DevIndex* parts;             // [nparts] device copy
  const AlnWork* aln_work; OutAln* out; uint32_t slots;
  uint32_t* cigar_pool; unsigned long long cigar_cap; unsigned long long* cigar_used;
  uint32_t* work_next;
  // traceback stage (one THREAD per alignment)
  struct TraceJob* jobs;             // [nreads_chunk * slots]
  uint8_t* tb_arena; size_t tb_stride; uint32_t tb_cap_w, tb_cap_cig; size_t tb_cap_dir;
  AlnStats* stats;                   // [nreads * slots] or nullptr
};
__host__ __device__ inline size_t final_arena_bytes(uint32_t cap_w, uint32_t cap_cig, uint32_t row_cap, size_t cap_dir) {
  size_t b = (size_t)cap_w * 12 + (size_t)cap_cig * 4 + (size_t)row_cap * 8 + cap_dir;
  return (b + 255) & ~(size_t)255;
}

constexpr int kFinalWarpsPerCta = 4;
#ifndef SMR_FINAL_MIN_CTAS
#define SMR_FINAL_MIN_CTAS 6     // resident CTAs per SM the register budget is set for (3: 167 registers, 4: 128, 5: 96, 6: 80; more CTAs were faster)
#endif
constexpr int kFinalCtasPerSm = SMR_FINAL_MIN_CTAS;

__global__ void __launch_bounds__(kFinalWarpsPerCta * 32, kFinalCtasPerSm)
finalize_kernel(DevBatch b, DevParams prm, FinalGlobals g) {
  __shared__ __align__(16) uint8_t s_ref[kFinalWarpsPerCta][kRefStage + 64];
  __shared__ int32_t s_prof[kFinalWarpsPerCta][kProfWords];
  const unsigned lane = lane_id();
  const uint32_t warp = blockIdx.x * kFinalWarpsPerCta + (threadIdx.x >> 5);
  uint8_t* p = g.arena_base + (size_t)warp * g.arena_stride;
  TraceArena A;
  A.cap_w = g.cap_w; A.cap_cig = g.cap_cig; A.cap_dir = g.cap_dir; A.stride = 1;
  A.hb = (int32_t*)p; p += (size_t)g.cap_w * 4;
  A.eb = (int32_t*)p; p += (size_t)g.cap_w * 4;
  A.hc = (int32_t*)p; p += (size_t)g.cap_w * 4;
  A.cig = (uint32_t*)p; p += (size_t)g.cap_cig * 4;
  int32_t* rowH = (int32_t*)p; p += (size_t)g.row_cap * 4;
  int32_t* rowF = (int32_t*)p; p += (size_t)g.row_cap * 4;
  A.dir = (int8_t*)p;
  const SwScore sc{prm.match, prm.mismatch, prm.score_N, prm.gap_open, prm.gap_ext, prm.one};
  const uint32_t total = b.nreads * g.slots;
  for (;;) {
    uint32_t wi = 0;
    if (lane == 0) wi = atomicAdd(g.work_next, 1u);
    wi = __shfl_sync(kFull, wi, 0);
    if (wi >= total) break;
    const uint32_t r = b.r0 + wi / g.slots, k = wi % g.slots;
    if (k >= b.state[r].n_align || b.flags[r]) { if (lane == 0) g.jobs[(size_t)wi].valid = 0; continue; }
    const AlnWork a = g.aln_work[(size_t)r * g.slots + k];
    const DevIndex& ix = g.parts[a.idx_slot];
    const uint32_t seq_base = b.seq_off[r], len = b.seq_off[r + 1] - seq_base;
    SeqView q = a.strand ? SeqView{b.seq04 + seq_base, (int32_t)a.q_start, 1, false}
                         : SeqView{b.seq04 + seq_base, (int32_t)(len - 1 - a.q_start), -1, true};
    const SeqView t{ix.refseq + ix.ref_off[a.ref_num], (int32_t)a.win_ref_start, 1, false};
    // forward pass again, now with the end-point tie-breaks (ssw.c:310-336), then the reverse pass over
    // the prefixes that end at the forward optimum (ssw.c:899-915)
    uint8_t* sr = s_ref[threadIdx.x >> 5]; int32_t* sp = s_prof[threadIdx.x >> 5];
    const SwEnd fwd = sw_locate(q, (int32_t)a.q_len, t, (int32_t)a.win_len, sc, (int32_t)a.score1, sr, sp, rowH, rowF);
    if ((uint32_t)(fwd.score & 0xFFFF) != a.score1) { if (lane == 0) { atomicOr(&b.flags[r], kErrTrace); g.jobs[(size_t)wi].valid = 0; } continue; }
    const int32_t a_ref_end = fwd.ref, a_read_end = fwd.read;
    const SwEnd rev = sw_locate(q.reversed_prefix(a_read_end), a_read_end + 1, t.reversed_prefix(a_ref_end), a_ref_end + 1, sc, (int32_t)a.score1, sr, sp, rowH, rowF);
    if (rev.score != (int32_t)a.score1) { if (lane == 0) { atomicOr(&b.flags[r], kErrTrace); g.jobs[(size_t)wi].valid = 0; } continue; }
    const int32_t ref_begin = a_ref_end - rev.ref, read_begin = a_read_end - rev.read;
    const int32_t rl = a_ref_end - ref_begin + 1, ql = a_read_end - read_begin + 1;
    const int32_t band = (rl > ql ? rl - ql : ql - rl) + 1;                                  // ssw.c:924
    if (lane == 0) {
      OutAln o;
      o.cigar_off = 0; o.cigar_len = 0; o.ref_num = a.ref_num;
      o.ref_begin1 = ref_begin + (int32_t)a.win_ref_start; o.ref_end1 = a_ref_end + (int32_t)a.win_ref_start;   // alignment.cpp:396-399
      o.read_begin1 = read_begin + (int32_t)a.q_start; o.read_end1 = a_read_end + (int32_t)a.q_start;
      o.readlen = len; o.score1 = a.score1; o.part = a.part; o.index_num = a.index_num; o.strand = a.strand; o.pad = 0;
      g.out[(size_t)r * g.slots + k] = o;
      TraceJob j;
      const SeqView qs = q.sub(read_begin);
      j.valid = 1; j.idx_slot = a.idx_slot; j.ref_num = a.ref_num; j.ref_off = a.win_ref_start + (uint32_t)ref_begin;
      j.q_start = qs.start; j.q_step = qs.step; j.rl = rl; j.ql = ql; j.score = (int32_t)a.score1; j.band = band;
      g.jobs[(size_t)wi] = j;
    }
    __syncwarp();
  }
}

// banded_sw (ssw.c:577-773) for every stored alignment, one THREAD per alignment (the DP rows are a serial chain of
// 3..2*band+1 cells; 32 alignments per warp keep the lanes busy where one-lane-per-warp left 31 idle)
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
  const uint32_t total = b.nreads * g.slots;
  for (uint32_t wi = tid; wi < total; wi += nthreads) {
    const TraceJob j = g.jobs[wi];
    if (!j.valid) continue;
    const uint32_t r = b.r0 + wi / g.slots, k = wi % g.slots;
    const DevIndex& ix = g.parts[j.idx_slot];
    const SeqView t{ix.refseq + ix.ref_off[j.ref_num], (int32_t)j.ref_off, 1, false};
    const SeqView q{b.seq04 + b.seq_off[r], j.q_start, j.q_step, j.q_step < 0};
    for (uint32_t i = 0; i < g.tb_cap_w; ++i) { A.hb[i * 32] = 0; A.eb[i * 32] = 0; A.hc[i * 32] = 0; }
    const int32_t nc = banded_traceback_lane(t, q, j.rl, j.ql, j.score, sc, j.band, A);
    if (nc < 0) { atomicOr(&b.flags[r], nc == -1 ? kOvfTrace : kErrTrace); continue; }
    const unsigned long long off = atomicAdd(g.cigar_used, (unsigned long long)nc);
    if (off + (unsigned long long)nc > g.cigar_cap) { atomicOr(&b.flags[r], kOvfCigar); continue; }
    for (int32_t i = 0; i < nc; ++i) g.cigar_pool[off + i] = A.cig[(size_t)(nc - 1 - i) * 32];        // ssw.c:750-758 (reverse)
    OutAln* o = g.out + (size_t)r * g.slots + k;
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
      g.stats[(size_t)r * g.slots + k] = AlnStats{miss, gap, match, match_d};
    }
  }
}

// unit-test kernel: full ssw_align(flag=2) equivalent on explicit pairs, one warp per pair (smr_debug_ssw)
__global__ void __launch_bounds__(kFinalWarpsPerCta * 32)
ssw_debug_kernel(const uint8_t* qcat, const uint32_t* qoff, const uint8_t* tcat, const uint32_t* toff, uint32_t npairs, uint32_t filters,
                 DevParams prm, int32_t* out, uint32_t* cigars, uint32_t cigar_cap, FinalGlobals g) {
  __shared__ __align__(16) uint8_t s_ref[kFinalWarpsPerCta][kRefStage + 64];
  __shared__ int32_t s_prof[kFinalWarpsPerCta][kProfWords];
  const unsigned lane = lane_id();
  const uint32_t warp = blockIdx.x * kFinalWarpsPerCta + (threadIdx.x >> 5), nwarps = gridDim.x * kFinalWarpsPerCta;
  uint8_t* p = g.arena_base + (size_t)warp * g.arena_stride;
  TraceArena A;
  A.cap_w = g.cap_w; A.cap_cig = g.cap_cig; A.cap_dir = g.cap_dir; A.stride = 1;
  A.hb = (int32_t*)p; p += (size_t)g.cap_w * 4;
  A.eb = (int32_t*)p; p += (size_t)g.cap_w * 4;
  A.hc = (int32_t*)p; p += (size_t)g.cap_w * 4;
  A.cig = (uint32_t*)p; p += (size_t)g.cap_cig * 4;
  int32_t* rowH = (int32_t*)p; p += (size_t)g.row_cap * 4;
  int32_t* rowF = (int32_t*)p; p += (size_t)g.row_cap * 4;
  A.dir = (int8_t*)p;
  const SwScore sc{prm.match, prm.mismatch, prm.score_N, prm.gap_open, prm.gap_ext, prm.one};
  for (uint32_t k = warp; k < npairs; k += nwarps) {
    const int32_t m = (int32_t)(qoff[k + 1] - qoff[k]), n = (int32_t)(toff[k + 1] - toff[k]);
    const SeqView q{qcat + qoff[k], 0, 1, false}, t{tcat + toff[k], 0, 1, false};
    int32_t* o = out + (size_t)k * 6;
    SwEnd f = sw_forward(q, m, t, n, sc, rowH, rowF);
    // the score-only kernel of the candidate loop must agree with the arg-max kernel
    if (sw_score(q, m, t, n, sc, s_ref[threadIdx.x >> 5], s_prof[threadIdx.x >> 5], rowH, rowF) != f.score) f.score = -12345;
    if (f.score > 0) {   // the score-known locate kernel (finalize) must agree with the arg-max kernel on the end point
      const SwEnd l = sw_locate(q, m, t, n, sc, f.score, s_ref[threadIdx.x >> 5], s_prof[threadIdx.x >> 5], rowH, rowF);
      if (l.ref != f.ref || l.read != f.read) f.score = -12346;
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
