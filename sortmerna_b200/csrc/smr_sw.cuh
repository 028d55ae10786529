// Smith-Waterman for (query segment, reference window) pairs, cooperatively by one warp.
//
// Stands in for ssw_init / ssw_align (src/sortmerna/ssw.c:788-941): the striped SSE2 kernels
// sw_sse2_byte / sw_sse2_word (:150-575) become a warp-wide anti-diagonal wavefront -- lane l owns R
// consecutive query rows, reference columns stream through the lanes one column per step, the
// H/F values of a lane's last row travel to the next lane by shuffle -- in two kernels:
//   sw_pair_warp  two problems per pass in the 16-bit halves of every register (DPX 16x2), for the
//                 shapes and scores sw_pair_ok accepts: the score pass of the candidate kernel and,
//                 with the score known, the end-point search of the finalize kernel;
//   sw_warp       one problem in s32 with its arg-max, any shape: every other problem, and the
//                 reference the debug kernel checks the packed kernel against.
// banded_sw (:577-773) keeps its scalar band arithmetic (CIGARs must match bit for bit, so the band
// coordinates, direction codes and band doubling are the reference's).
//
// Cell arithmetic uses the DPX instructions (__viaddmax_s16x2, __vimax3_s32_relu, ...); the problem is
// an integer recurrence, not a contraction, so tensor cores do not apply.  Outputs are defined by true
// affine-gap local scores plus the reference's tie-breaks (SURVEY Appendix A.6):
//   end   = among cells holding the global maximum: smallest reference column, then smallest read row
//   begin = same rule on the reversed prefixes (ssw.c:899-915).
#pragma once
#include "smr_dev.cuh"

namespace smr {

// strided byte view: element i = f(base[start + i*step]); comp => 3-x for x<4 (complement[], common.hpp:93)
struct SeqView {
  const uint8_t* base; int32_t start, step; bool comp;
  __device__ __forceinline__ uint32_t at(int32_t i) const {
    const uint32_t c = __ldg(base + start + (int64_t)i * step);
    return (comp && c < 4u) ? 3u - c : c;
  }
  __device__ __forceinline__ SeqView sub(int32_t off) const { return SeqView{base, start + off * step, step, comp}; }
  // the prefix [0..end] reversed (seq_reverse, ssw.c:775-786)
  __device__ __forceinline__ SeqView reversed_prefix(int32_t end) const { return SeqView{base, start + end * step, -step, comp}; }
};

struct SwScore { int32_t match, mismatch, sN, go, ge, one; };  // one == 1 at run time (keeps IMADs on the fma pipe)
struct SwEnd { int32_t score, ref, read; };

// Forward score pass.  q: query (m rows), t: target (n columns).  rowH/rowF: scratch of >= n ints each,
// used only when m > 32*R (the query is then processed in row blocks of 32*R rows).
template <int R>
__device__ SwEnd sw_warp(const SeqView q, const int32_t m, const SeqView t, const int32_t n, const SwScore sc,
                         int32_t* __restrict__ rowH, int32_t* __restrict__ rowF) {
  const int lane = (int)lane_id();
  int32_t best = 0, best_j = 0x7FFFFFFF, best_i = 0x7FFFFFFF;
  const bool multi = m > 32 * R;
  for (int32_t blk0 = 0; blk0 < m; blk0 += 32 * R) {
    const int32_t i0 = blk0 + lane * R;
    int32_t qc[R], qmis[R], Hp[R], E[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int32_t i = i0 + r;
      uint32_t c = i < m ? q.at(i) : 7u;
      qmis[r] = c == 7u ? -(1 << 20) : (c >= 4u ? sc.sN : sc.mismatch);  // mat[ref*5+read] (read.cpp:274-288)
      qc[r] = c >= 4u ? (c == 7u ? 7 : 5) : (int32_t)c;                   // N never compares equal
      Hp[r] = 0; E[r] = 0;
    }
    int32_t diagH = 0, outH = 0, outF = 0;
    uint32_t chunk_cur = lane < n ? t.at(lane) : 0u, chunk_prev = 0u;
    const int32_t nsteps = n + 31;
    for (int32_t ts = 0; ts < nsteps; ++ts) {
      if ((ts & 31) == 0 && ts > 0) { chunk_prev = chunk_cur; chunk_cur = (ts + lane) < n ? t.at(ts + lane) : 0u; }
      // reference character of column j = ts - lane: source lane s supplies position ts - ((ts - s) & 31)
      const int32_t pos_s = ts - ((ts - lane) & 31);
      const uint32_t supply = pos_s >= (ts & ~31) ? chunk_cur : chunk_prev;
      const int32_t rc = (int32_t)__shfl_sync(kFull, supply, (ts - lane) & 31);
      int32_t upH = __shfl_up_sync(kFull, outH, 1), upF = __shfl_up_sync(kFull, outF, 1);
      const int32_t j = ts - lane;
      const bool active = (j >= 0) && (j < n);
      if (lane == 0) {
        if (multi && blk0 > 0 && active) { upH = rowH[j]; upF = rowF[j]; } else { upH = 0; upF = 0; }
      }
      if (active) {
        int32_t diag = diagH, F = upF, colmax = 0;
        diagH = upH;
        const int32_t misN = rc == 4 ? 1 : 0;
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int32_t miss = misN ? sc.sN : qmis[r];
          const int32_t s = (rc == qc[r]) ? sc.match : miss;
          const int32_t h = __vimax3_s32_relu(diag + s, E[r], F);
          diag = Hp[r]; Hp[r] = h;
          const int32_t open = h - sc.go;
          E[r] = __viaddmax_s32(E[r], -sc.ge, open);
          F = __viaddmax_s32(F, -sc.ge, open);
          colmax = max(colmax, h);
        }
        outH = Hp[R - 1]; outF = max(F, 0);
        if (multi && lane == 31) { rowH[j] = outH; rowF[j] = outF; }
        if (colmax > best || (colmax == best && colmax > 0 && j < best_j)) {
          best = colmax; best_j = j;
          int rr = 0;
#pragma unroll
          for (int r = R - 1; r >= 0; --r) if (Hp[r] == colmax) rr = r;
          best_i = i0 + rr;
        }
      }
    }
    if (multi) __syncwarp();
  }
  // warp arg-max: score desc, column asc, row asc
  unsigned long long key = ((unsigned long long)(uint32_t)best << 42) | ((unsigned long long)(0x1FFFFF - min(best_j, 0x1FFFFF)) << 21) |
                           (unsigned long long)(0x1FFFFF - min(best_i, 0x1FFFFF));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const unsigned long long k2 = __shfl_xor_sync(kFull, key, o); key = k2 > key ? k2 : key; }
  SwEnd e;
  e.score = (int32_t)(key >> 42);
  e.ref = 0x1FFFFF - (int32_t)((key >> 21) & 0x1FFFFF);
  e.read = 0x1FFFFF - (int32_t)(key & 0x1FFFFF);
  if (e.score == 0) { e.ref = -1; e.read = 0; }  // ssw.c:179 (byte kernel, no overflow): end_ref stays -1
  return e;
}

// one instantiation for any shape (row blocks of 256 rows): the rarely taken fallback of the candidate kernel
__device__ __noinline__ SwEnd sw_forward_any(const SeqView q, const int32_t m, const SeqView t, const int32_t n, const SwScore sc,
                                             int32_t* rowH, int32_t* rowF) {
  return sw_warp<8>(q, m, t, n, sc, rowH, rowF);
}

// rows per lane for a query of m rows: the smallest R with 32*R >= m (R = 8 and row blocks beyond 256 rows in sw_warp)
__device__ __forceinline__ int pair_rows(const int32_t m) { return m <= 32 ? 1 : m <= 64 ? 2 : m <= 96 ? 3 : m <= 128 ? 4 : m <= 160 ? 5 : m <= 192 ? 6 : 8; }

__device__ __noinline__ SwEnd sw_forward(const SeqView q, const int32_t m, const SeqView t, const int32_t n, const SwScore sc,
                                         int32_t* rowH, int32_t* rowF) {
  switch (pair_rows(m)) {
    case 1: return sw_warp<1>(q, m, t, n, sc, rowH, rowF);
    case 2: return sw_warp<2>(q, m, t, n, sc, rowH, rowF);
    case 3: return sw_warp<3>(q, m, t, n, sc, rowH, rowF);
    case 4: return sw_warp<4>(q, m, t, n, sc, rowH, rowF);
    case 5: return sw_warp<5>(q, m, t, n, sc, rowH, rowF);
    case 6: return sw_warp<6>(q, m, t, n, sc, rowH, rowF);
    default: return sw_warp<8>(q, m, t, n, sc, rowH, rowF);
  }
}

// ---------------------------------------------------------------------------------------------
// Packed pass: TWO independent (query, window) problems per warp pass, problem A in the low and
// problem B in the high 16 bits of every register (the exact 16-bit path of the reference is the word
// kernel sw_sse2_word, ssw.c:399-575; packing two ALIGNMENTS rather than two cells of one alignment keeps
// the vertical F chain of a lane's rows intact).  It is the hot loop of the candidate kernel.  Accept / replace /
// stop decisions of compute_lis_alignment only consume score1 (alignment.cpp:388-469), so the arg-max bookkeeping
// of sw_warp is left to the finalize kernel, which re-runs the pass with the score known (FIND) for the few
// alignments that end up stored.
//
// Each window is staged in shared memory with 32 sentinel columns on both sides, so lanes need no "column in range"
// predicate: columns outside [0,n) only ever produce values strictly below the running maximum (every step away from
// a real cell costs a mismatch or a gap), and real cells never read them.  Rows past the query end score kPairDead in
// every column, which keeps them below it too.
//
// The query profile turns the per-cell "compare + select" of the substitution score into a shared load (LSU pipe), so
// the ALU pipe, which bounds the loop, issues only the max-type DPX instructions of the cell update.  With
// X = max(0, diag + s, E), which does not depend on F, we have H = max(X, F) and, because gap_ext <= gap_open,
//   F(r+1) = max(F(r) - ge, H(r) - go) = max(F(r) - ge, X(r) - go),
// so the loop-carried chain down a lane's R rows is ONE instruction per row.  F is carried as G = F + go:
//   X = max(diag + s, E, 0)         VIADDMNMX.S16x2.RELU
//   G' = max(G - ge, X)             VIADDMNMX.S16x2      (= F' + go)
//   H = max(G - go, X)              VIADDMNMX.S16x2
//   E' = max(E - ge, H - go)        VIADD.16x2 + VIADDMNMX.S16x2
//   best = max(best, H, H')         VIMNMX3.S16x2 per two rows
// = 5.5 ALU-pipe instructions per PAIR of cells.  The boundary G = 0 (row -1) stands for F = -go, which like every
// negative F can never win against X >= 0.
// Valid while every score fits 15 bits: m * match <= kPairMaxScore (checked by sw_pair_ok).
// Query profile per problem: prof[tb][rp][lane] = s(row 2rp, tb) | s(row 2rp+1, tb) << 16 (rows of the lane's strip), so
// one LDS per problem serves two rows and a PRMT per row merges the two problems' scores into one register.
// ---------------------------------------------------------------------------------------------
constexpr int kRefStage = 448;    // staged window bytes per warp; longer windows use sw_warp
constexpr int kProfTables = 6;    // reference letter A,C,G,T,N + the out-of-window sentinel
constexpr int kPairProfWords = kProfTables * 4 * 32;   // per problem: 6 tables x 4 row pairs (R <= 8) x 32 lanes
constexpr int32_t kPairMaxScore = 32000;
constexpr int32_t kPairDead = -32000;                  // substitution score of rows past the query end

__device__ __forceinline__ bool sw_pair_ok(const int32_t m, const int32_t n, const SwScore sc) {
  return m <= 256 && n <= kRefStage && sc.mismatch < 0 && sc.mismatch > -1024 && sc.go > 0 && sc.go < 1024 && sc.sN < 0 && sc.sN > -1024 &&
         sc.ge <= sc.go && sc.ge >= 0 && sc.match >= 0 && m * sc.match <= kPairMaxScore;
}

__device__ __forceinline__ uint32_t pack16(const int32_t lo, const int32_t hi) { return ((uint32_t)lo & 0xFFFFu) | ((uint32_t)hi << 16); }

constexpr int kPairRP = 4;   // row pairs per lane in the profile layout (fixed: one layout for every R <= 8)
constexpr uint32_t kPairNoHit = 0x7FFFFFFFu;
constexpr uint32_t kPairNoTarget = 0x7FFFu;          // a target no 15-bit score reaches: the half is not searched

// FIND = false: returns the packed best scores (A low, B high).
// FIND = true: `tgt2` packs the (known) best score of each problem; returns, per problem, the first cell holding it in the reference's
// order (smallest column, then smallest row: ssw.c:310-336) as column<<16 | row, or kPairNoHit.  Every cell is <= its problem's
// maximum, so "a cell of this column holds the target" is "the lane's running maximum reached the target in this step": the
// running maximum of the score pass is compared with the target once per step, and a lane's rows are only searched in the
// step where one of its halves first reaches it -- that column is the lane's first hit column, and the smallest row holding the
// target there is its hit.  Sentinel columns and dead rows stay strictly below any positive target (see above).
template <int R, bool FIND = false>
__device__ __noinline__ auto sw_pair_warp(const uint32_t* __restrict__ profA, const uint32_t* __restrict__ profB, const uint8_t* __restrict__ refA,
                                          const uint8_t* __restrict__ refB, const int32_t nmax, const SwScore sc, const uint32_t tgt2 = 0) {
  constexpr int RP = (R + 1) / 2;
  const int lane = (int)lane_id();
  uint32_t Hp[R], E[R];
#pragma unroll
  for (int r = 0; r < R; ++r) { Hp[r] = 0; E[r] = 0; }
  uint32_t diagH = 0, upH = 0, upF = 0, best = 0;
  // FIND: need1 = target - 1 per half still searched (0x7FFE once found): the sign bit of need1 - best is set where best >= target
  uint32_t need1 = __vsub2(tgt2, 0x00010001u), foundA = kPairNoHit, foundB = kPairNoHit;
  (void)need1; (void)foundA; (void)foundB;
  const uint8_t* cpA = refA + 32 - lane;
  const uint8_t* cpB = refB + 32 - lane;
  const uint32_t* pA = profA + lane;
  const uint32_t* pB = profB + lane;
  const int32_t nsteps = nmax + 31;
  const uint32_t nge2 = pack16(-sc.ge, -sc.ge), ngo2 = pack16(-sc.go, -sc.go);
  const uint32_t nz = lane ? (uint32_t)sc.one : 0u;
  // software pipeline, two deep: the column letters are fetched two steps ahead, the substitution scores one step ahead
  uint32_t sc_cur[R];
  {
    const uint32_t* ta = pA + (int32_t)cpA[0] * (kPairRP * 32);
    const uint32_t* tb = pB + (int32_t)cpB[0] * (kPairRP * 32);
#pragma unroll
    for (int rp = 0; rp < RP; ++rp) {
      const uint32_t wa = ta[rp * 32], wb = tb[rp * 32];
      sc_cur[2 * rp] = __byte_perm(wa, wb, 0x5410);
      if (2 * rp + 1 < R) sc_cur[2 * rp + 1] = __byte_perm(wa, wb, 0x7632);
    }
  }
  int32_t ia = (int32_t)cpA[1] * (kPairRP * 32), ib = (int32_t)cpB[1] * (kPairRP * 32);
#pragma unroll 2
  for (int32_t ts = 0; ts < nsteps; ++ts) {
    uint32_t sc_next[R];
    {
      const uint32_t* ta = pA + ia;
      const uint32_t* tb = pB + ib;
      ia = (int32_t)cpA[ts + 2] * (kPairRP * 32); ib = (int32_t)cpB[ts + 2] * (kPairRP * 32);   // [nsteps + 1] is still inside the trailing sentinels
#pragma unroll
      for (int rp = 0; rp < RP; ++rp) {
        const uint32_t wa = ta[rp * 32], wb = tb[rp * 32];
        sc_next[2 * rp] = __byte_perm(wa, wb, 0x5410);
        if (2 * rp + 1 < R) sc_next[2 * rp + 1] = __byte_perm(wa, wb, 0x7632);
      }
    }
    // the boundary values of this step were requested (shuffled) right after the F chain of the previous step, so that the
    // shuffle latency (30 cycles) runs under the H / E updates of the other rows instead of heading the step's critical path:
    // a dependent VIADDMNMX.S16x2 issues every 8.4 cycles, the loop-carried chain is IMAD + R of them
    uint32_t X[R], F[R + 1];
#pragma unroll
    for (int r = 0; r < R; ++r) X[r] = __viaddmax_s16x2_relu(r == 0 ? diagH : Hp[r - 1], sc_cur[r], E[r]);
    diagH = upH;
    F[0] = upF;
    // vertical chain F[r+1] = max(F[r] - ge, X[r]): R dependent instructions (8.4 cycles each).  With four scorer warps per SM
    // sub-partition the pipe is full anyway (tools/ubench/dp.cu: 2 warps saturate it), so no ALU work is spent on shortening it
    // (measured: a two-row look-ahead, F[r+2] = max(F[r] - 2 ge, max(X[r] - ge, X[r+1])), 2 more instructions per step: slower;
    //  one-row-per-word profiles merged by IMAD instead of PRMT, 4 more shared loads per step: slower still -- the LSU pipe, not the ALU)
#pragma unroll
    for (int r = 0; r < R; ++r) F[r + 1] = __viaddmax_s16x2(F[r], nge2, X[r]);
    const uint32_t hl = __viaddmax_s16x2(F[R - 1], ngo2, X[R - 1]);
    const uint32_t rawH = __shfl_up_sync(kFull, hl, 1), rawF = __shfl_up_sync(kFull, F[R], 1);
#pragma unroll
    for (int r = 0; r < R - 1; ++r) {
      const uint32_t h = __viaddmax_s16x2(F[r], ngo2, X[r]);
      E[r] = __viaddmax_s16x2(E[r], nge2, __vadd2(h, ngo2));
      Hp[r] = h;
    }
    E[R - 1] = __viaddmax_s16x2(E[R - 1], nge2, __vadd2(hl, ngo2));
    Hp[R - 1] = hl;
    upH = rawH * nz; upF = rawF * nz;   // row -1 is all zeros (consumed at the top of the next step); a multiply (fma pipe), not a select (alu pipe)
#pragma unroll
    for (int r = 0; r + 1 < R; r += 2) best = __vimax3_s16x2(best, Hp[r], Hp[r + 1]);
    if (R & 1) best = __vmaxs2(best, Hp[R - 1]);
    if constexpr (FIND) {
      const uint32_t reached = __vsub2(need1, best) & 0x80008000u;
      if (reached) {   // once per half and lane at most
        const uint32_t col = (uint32_t)(ts - lane) << 16;
        if (reached & 0x8000u) {
          int rr = R;
#pragma unroll
          for (int r = R - 1; r >= 0; --r) if (((Hp[r] ^ tgt2) & 0xFFFFu) == 0u) rr = r;
          if (rr < R) foundA = col | (uint32_t)(lane * R + rr);
          need1 = (need1 & 0xFFFF0000u) | (kPairNoTarget - 1u);
        }
        if (reached & 0x80000000u) {
          int rr = R;
#pragma unroll
          for (int r = R - 1; r >= 0; --r) if (((Hp[r] ^ tgt2) >> 16) == 0u) rr = r;
          if (rr < R) foundB = col | (uint32_t)(lane * R + rr);
          need1 = (need1 & 0xFFFFu) | ((kPairNoTarget - 1u) << 16);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) sc_cur[r] = sc_next[r];
  }
  if constexpr (FIND) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { foundA = min(foundA, __shfl_xor_sync(kFull, foundA, o)); foundB = min(foundB, __shfl_xor_sync(kFull, foundB, o)); }
    return make_uint2(foundA, foundB);
  } else {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = __vmaxs2(best, __shfl_xor_sync(kFull, best, o));
    return best;
  }
}

// query profile of one problem for the packed pass: R rows per lane (run-time), m real rows; one copy of this code serves every R.
// qb: the query bytes (0..4) staged in shared memory by the bulk copy; element i = qb[i * step], complemented on the minus strand.
__device__ __noinline__ void pair_profile(const uint8_t* __restrict__ qb, const int32_t step, const bool comp, const int32_t m, const int R, const SwScore sc,
                                          uint32_t* __restrict__ prof) {
  const int lane = (int)lane_id();
#pragma unroll 1
  for (int rp = 0; rp < kPairRP; ++rp) {
    const int32_t r0 = 2 * rp, i0 = lane * R + r0;
    uint32_t c0 = (r0 < R && i0 < m) ? (uint32_t)qb[i0 * step] : 7u, c1 = (r0 + 1 < R && i0 + 1 < m) ? (uint32_t)qb[(i0 + 1) * step] : 7u;
    if (comp) { if (c0 < 4u) c0 = 3u - c0; if (c1 < 4u) c1 = 3u - c1; }
    const int32_t mis0 = c0 == 7u ? kPairDead : (c0 >= 4u ? sc.sN : sc.mismatch), mis1 = c1 == 7u ? kPairDead : (c1 >= 4u ? sc.sN : sc.mismatch);
#pragma unroll
    for (int tb = 0; tb < 4; ++tb) prof[(tb * kPairRP + rp) * 32 + lane] = pack16(c0 == (uint32_t)tb ? sc.match : mis0, c1 == (uint32_t)tb ? sc.match : mis1);
    prof[(4 * kPairRP + rp) * 32 + lane] = pack16(c0 == 7u ? kPairDead : sc.sN, c1 == 7u ? kPairDead : sc.sN);   // reference N
    prof[(5 * kPairRP + rp) * 32 + lane] = pack16(mis0, mis1);                                                   // outside the window: never a match
  }
}

// A window of n columns lies in shared memory at w[0 .. n) (bulk copy of the reference bytes, 0..4): write the sentinel
// letter (table 5) into the 32 columns before it and from column n up to column nstage + 32.
__device__ __forceinline__ void pair_sentinels(uint8_t* __restrict__ w, const int32_t n, const int32_t nstage) {
  const int lane = (int)lane_id();
  w[lane - 32] = 5;
  for (int32_t j = n + lane; j < nstage + 33; j += 32) w[j] = 5;
}

// the packed pass for R rows per lane: profiles and windows (column 0 at ra[32] / rb[32], sentinels in place) are in shared memory
template <bool FIND>
__device__ __forceinline__ auto sw_pair_dispatch(const int R, const uint32_t* pa, const uint32_t* pb, const uint8_t* ra, const uint8_t* rb, const int32_t nmax,
                                                 const SwScore sc, const uint32_t tgt2 = 0) {
  switch (R) {
    case 1: return sw_pair_warp<1, FIND>(pa, pb, ra, rb, nmax, sc, tgt2);
    case 2: return sw_pair_warp<2, FIND>(pa, pb, ra, rb, nmax, sc, tgt2);
    case 3: return sw_pair_warp<3, FIND>(pa, pb, ra, rb, nmax, sc, tgt2);
    case 4: return sw_pair_warp<4, FIND>(pa, pb, ra, rb, nmax, sc, tgt2);
    case 5: return sw_pair_warp<5, FIND>(pa, pb, ra, rb, nmax, sc, tgt2);
    case 6: return sw_pair_warp<6, FIND>(pa, pb, ra, rb, nmax, sc, tgt2);
    default: return sw_pair_warp<8, FIND>(pa, pb, ra, rb, nmax, sc, tgt2);
  }
}

// Packed pass: the window of one problem, staged from global memory at w[0 .. n) (letters 0..4) with the sentinel letter in the
// 32 columns before it and from column n up to column nstage + 32 (w has kRefStage + 33 bytes after it and 32 before it).  All loads
// of a lane are issued before its first store.
constexpr int kPairWinBytes = kRefStage + 72;   // per window: 32 leading sentinels, kRefStage columns, 33 trailing, padding
__device__ __forceinline__ void pair_stage(const SeqView t, const int32_t n, const int32_t nstage, uint8_t* __restrict__ w) {
  constexpr int K = (kRefStage + 65 + 31) / 32;
  const int lane = (int)lane_id();
  uint32_t v[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const int32_t j = lane + 32 * k - 32;
    v[k] = (j >= 0 && j < n) ? min(t.at(j), 4u) : 5u;
  }
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const int32_t j = lane + 32 * k - 32;
    if (j <= nstage + 32) w[j] = (uint8_t)v[k];
  }
}

// One half of a packed pass: query q (m rows), window t (n columns) and, for a locate, its known best score target > 0.
// m == 0: no problem.
struct PairLoc { SeqView q; int32_t m; SeqView t; int32_t n, target; };

// Both problems in one packed pass.  FIND = false: the packed best scores (A low, B high; the targets are ignored).  FIND = true:
// the end points (column<<16 | row, or kPairNoHit) of both problems' first cells holding their targets.
// prof: 2 * kPairProfWords words, wa / wb: kPairWinBytes bytes each, all shared memory owned by this warp.  Both halves must pass
// sw_pair_ok (or be empty).
template <bool FIND>
__device__ __noinline__ auto sw_pair_run(const PairLoc A, const PairLoc B, const SwScore sc, uint32_t* prof, uint8_t* wa, uint8_t* wb) {
  const int R = pair_rows(max(A.m, B.m));
  const int32_t nmax = max(A.m ? A.n : 0, B.m ? B.n : 0);   // (an empty half's window is not looked at)
  __syncwarp();
  pair_stage(A.t, A.m ? A.n : 0, nmax, wa + 32);
  pair_stage(B.t, B.m ? B.n : 0, nmax, wb + 32);
  pair_profile(A.q.base + A.q.start, A.q.step, A.q.comp, A.m, R, sc, prof);
  const uint32_t* pb = prof;
  if (B.m) { pair_profile(B.q.base + B.q.start, B.q.step, B.q.comp, B.m, R, sc, prof + kPairProfWords); pb = prof + kPairProfWords; }
  __syncwarp();
  const uint32_t tgt2 = pack16(A.m ? A.target : (int32_t)kPairNoTarget, B.m ? B.target : (int32_t)kPairNoTarget);
  return sw_pair_dispatch<FIND>(R, prof, pb, wa, wb, nmax, sc, tgt2);
}

// ---- TMA bulk copy + mbarrier (cp.async.bulk; SASS: UBLKCP / SYNCS) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// global -> shared bulk copy (16-byte aligned source, destination and size); completion is counted on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---------------------------------------------------------------------------------------------
// banded_sw (ssw.c:577-773) -- executed by ONE lane; band coordinates as set_u / set_d (:70,:73)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int32_t band_u(int32_t w, int32_t i, int32_t j) { int32_t x = i - w; x = x > 0 ? x : 0; return j - x + 1; }
__device__ __forceinline__ int32_t band_d(int32_t w, int32_t i, int32_t j, int32_t p) { int32_t x = i - w; x = x > 0 ? x : 0; return (j - x) * 3 + p; }

struct TraceArena {
  int32_t* hb; int32_t* eb; int32_t* hc;  // band rows, cap_w ints each
  int8_t* dir; size_t cap_dir;            // direction matrix
  uint32_t* cig; uint32_t cap_cig;        // cigar scratch (reverse order)
  uint32_t cap_w;
  uint32_t stride;                        // element k of every array lives at [k * stride]: 1 = private contiguous arena,
                                          // 32 = arenas of the 32 lanes of a warp interleaved (coalesced when lanes run in step)
};

// returns: >=0 cigar length (cig holds the ops in REVERSE order), -1 arena too small, -2 trace back error
__device__ int32_t banded_traceback_lane(const SeqView t, const SeqView q, const int32_t refLen, const int32_t readLen, const int32_t score,
                                         const SwScore sc, int32_t band_width, TraceArena& A) {
  // the caller zeroes hb/eb/hc[0..cap_w) (the reference's band rows keep their contents across the
  // band-doubling iterations, ssw.c:601-606; only the cells named below are reset per iteration)
  const size_t S = A.stride;
  int32_t maxv = 0, width = 0, width_d = 0;
  do {
    width = band_width * 2 + 3; width_d = band_width * 2 + 1;
    if ((uint32_t)(width + 1) > A.cap_w) return -1;
    if ((size_t)width_d * readLen * 3 + 8 > A.cap_dir) return -1;
    for (int32_t j = 1; j < width - 1; ++j) A.hb[j * S] = 0;
    for (int32_t i = 0; i < readLen; ++i) {
      const int32_t beg = max(0, i - band_width), end = min(refLen - 1, i + band_width);
      const int32_t edge = end + 1 < width - 1 ? end + 1 : width - 1;
      int32_t f = 0, u = 0, hleft = 0;   // hleft: H of the left neighbour, hc[u - 1] (hc[0] = 0 at the row's first cell)
      A.hb[0] = 0; A.eb[0] = 0; A.hb[edge * S] = 0; A.eb[edge * S] = 0; A.hc[0] = 0;
      int8_t* dl = A.dir + (size_t)width_d * i * 3 * S;
      const uint32_t qi = q.at(i);
      for (int32_t j = beg; j <= end; ++j) {
        u = band_u(band_width, i, j);
        const int32_t up = band_u(band_width, i - 1, j), dg = band_u(band_width, i - 1, j - 1);
        const int32_t de = band_d(band_width, i, j, 0), df = de + 1, dh = de + 2;
        int32_t t1 = i == 0 ? -sc.go : A.hb[up * S] - sc.go;
        int32_t t2 = i == 0 ? -sc.ge : A.eb[up * S] - sc.ge;
        const int32_t ev = t1 > t2 ? t1 : t2;
        A.eb[u * S] = ev;
        const int8_t cde = t1 > t2 ? 3 : 2;
        dl[de * S] = cde;
        t1 = hleft - sc.go; t2 = f - sc.ge;
        f = t1 > t2 ? t1 : t2;
        const int8_t cdf = t1 > t2 ? 5 : 4;
        dl[df * S] = cdf;
        const int32_t e1 = ev > 0 ? ev : 0, f1 = f > 0 ? f : 0;
        t1 = e1 > f1 ? e1 : f1;
        const uint32_t tj = t.at(j);
        const int32_t s = (tj >= 4u || qi >= 4u) ? sc.sN : (tj == qi ? sc.match : sc.mismatch);
        t2 = A.hb[dg * S] + s;
        const int32_t hv = t1 > t2 ? t1 : t2;
        A.hc[u * S] = hv; hleft = hv;
        if (hv > maxv) maxv = hv;
        dl[dh * S] = (t1 <= t2) ? (int8_t)1 : (e1 > f1 ? cde : cdf);
      }
      for (int32_t j = 1; j <= u; ++j) A.hb[j * S] = A.hc[j * S];
    }
    band_width *= 2;
  } while (maxv < score);
  band_width /= 2;
  // trace back (ssw.c:674-747)
  int32_t i = readLen - 1, j = refLen - 1, run = 0, cur_op = 0, op = 0, which = 2;
  uint32_t l = 0;
  int64_t row_off = (int64_t)width_d * (readLen - 1) * 3;     // element offset of the current row in the direction matrix
  while (i > 0) {
    const int32_t tt = band_d(band_width, i, j, which);
    const int64_t abs_off = row_off + tt;        // same linear layout as the reference's direction array
    if (abs_off < 0 || abs_off >= (int64_t)width_d * readLen * 3) return -2;
    switch (A.dir[abs_off * S]) {
      case 1: --i; --j; which = 2; row_off -= width_d * 3; op = 0; break;
      case 2: --i; which = 0; row_off -= width_d * 3; op = 1; break;
      case 3: --i; which = 2; row_off -= width_d * 3; op = 1; break;
      case 4: --j; which = 1; op = 2; break;
      case 5: --j; which = 2; op = 2; break;
      default: return -2;
    }
    if (op == cur_op) ++run;
    else {
      if (l >= A.cap_cig) return -1;
      A.cig[(l++) * S] = (uint32_t)run << 4 | (uint32_t)cur_op; cur_op = op; run = 1;
    }
  }
  if (l + 2 > A.cap_cig) return -1;
  if (op == 0) A.cig[(l++) * S] = (uint32_t)(run + 1) << 4;
  else { A.cig[(l++) * S] = (uint32_t)run << 4 | (uint32_t)op; A.cig[(l++) * S] = 16u; }
  return (int32_t)l;
}

}  // namespace smr
