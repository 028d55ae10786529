// Device placement of a run's results (smr_place_results, smr_place_results_packed, smr_download_results_packed): every read's
// final results, from the resident batch's first run or from the re-run that completed it, placed on the device in the bytes the
// caller's layout holds, for the report-side calls to read in place.  src[r] names the run and the read in it that hold read r's
// results; the runs stay on the device until the scatter.  One count pass (rows and CIGAR words per read, the counters), two
// exclusive scans (alignment offsets, CIGAR offsets), one scatter pass with a group of lanes per read (a warp when packed).
// - packed layout (stride 0): read r's n_align alignments at sum_{j<r} n_align(j), the CIGARs compacted in read order.
// - strided layout (stride S): read r's S rows at r * S, zeroed past n_align (stats alike), the CIGARs compacted in run order --
//   the first run's reads, then each re-run's in the order they were made -- which is the order the host download writes them.
#pragma once
#include "smr_final.cuh"
#include "../../include/smr_b200.h"

namespace smr {

// one run of a placement, as the run left it on the device
struct PackRun {
  const ReadState* st; const uint16_t* hit_db; const OutAln* oa; const AlnStats* ast; const uint32_t* cigar;
  const uint32_t* base;        // read k's first slot (a re-run's packed arenas); null: k * slots
  const unsigned long long* cnt;   // the run's device counters
  uint32_t slots;
  uint32_t first;              // strided layout: the entry of its read 0 in the run-order CIGAR scan
};

// a read flagged by a run, as the host forms the re-runs from it
struct PackFlag { uint32_t read, flags, n_align; };

// the reads of a run that carry a flag, in read order: bit[r] = 1 for each (then an exclusive scan, pos), then out[pos[r]]
__global__ void __launch_bounds__(256) pack_flag_bits_kernel(const uint32_t* __restrict__ flags, uint32_t n, uint32_t* __restrict__ bit) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r <= n; r += gridDim.x * blockDim.x) bit[r] = r < n && flags[r] ? 1u : 0u;
}

// out[pos[r]] = (r, its flags, its n_align) for each flagged read r
__global__ void __launch_bounds__(256) pack_flagged_kernel(const uint32_t* __restrict__ flags, const ReadState* __restrict__ st, uint32_t n,
                                                           const uint32_t* __restrict__ pos, PackFlag* __restrict__ out) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    const uint32_t f = flags[r];
    if (f) out[pos[r]] = PackFlag{r, f, st[r].n_align};
  }
}

// src[r] = (0, r): every read from the first run until a re-run stores it
__global__ void __launch_bounds__(256) pack_src_init_kernel(uint2* __restrict__ src, uint32_t n) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) src[r] = make_uint2(0u, r);
}

// a re-run (ordinal run) of n reads: its unflagged read k holds the results of read map[k] of the resident batch
__global__ void __launch_bounds__(256) pack_src_kernel(const uint32_t* __restrict__ flags, const uint32_t* __restrict__ map, uint32_t n,
                                                       uint32_t run, uint2* __restrict__ src) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    if (!flags[k]) src[map[k]] = make_uint2(run, k);
}

// nal[r] = the rows of read r (stride 0: its n_align; else the stride), nal[n] = 0; the CIGAR words of read r from its source run
// into words[r] (stride 0; words[n] = 0) or words[first + read in its run] (strided: words is zeroed, of sum of run sizes + 1
// entries); counters into cnt[0 .. ncnt): SMR_CNT_NUM_ALIGNED and reads_matched_per_db once per read, and the device counters
// 1 .. dcCount - 1 of every run (block 0).  Dynamic shared memory: ncnt u64.
__global__ void __launch_bounds__(256) pack_count_kernel(const PackRun* __restrict__ runs, uint32_t nruns, const uint2* __restrict__ src,
                                                         uint32_t n, uint32_t stride, uint64_t* __restrict__ nal, uint64_t* __restrict__ words,
                                                         unsigned long long* __restrict__ cnt, uint32_t ncnt) {
  extern __shared__ unsigned long long s_cnt[];
  for (uint32_t k = threadIdx.x; k < ncnt; k += blockDim.x) s_cnt[k] = 0;
  __syncthreads();
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    const uint2 s = src[r];
    const PackRun& d = runs[s.x];
    const ReadState st = d.st[s.y];
    const size_t b = d.base ? (size_t)d.base[s.y] : (size_t)s.y * d.slots;
    const uint32_t na = stride ? min(st.n_align, stride) : st.n_align;
    uint64_t sum = 0;
    for (uint32_t j = 0; j < na; ++j) sum += d.oa[b + j].cigar_len;
    nal[r] = stride ? stride : st.n_align;
    words[stride ? (size_t)d.first + s.y : r] = sum;
    if (st.is_hit) {
      atomicAdd(&s_cnt[SMR_CNT_NUM_ALIGNED], 1ull);
      const uint16_t db = d.hit_db[s.y];
      if (db != 0xFFFF && SMR_CNT_FIXED + (uint32_t)db < ncnt) atomicAdd(&s_cnt[SMR_CNT_FIXED + db], 1ull);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { nal[n] = 0; if (!stride) words[n] = 0; }
  __syncthreads();
  if (blockIdx.x == 0) {
    constexpr uint32_t kw = dcCount - dcNumShort;
    for (uint32_t i = threadIdx.x; i < nruns * kw; i += blockDim.x) {
      const uint32_t k = dcNumShort + i % kw;
      if (k < ncnt) atomicAdd(&s_cnt[k], runs[i / kw].cnt[k]);
    }
    __syncthreads();
  }
  for (uint32_t k = threadIdx.x; k < ncnt; k += blockDim.x)
    if (s_cnt[k]) atomicAdd(&cnt[k], s_cnt[k]);
}

// where the placed results go
struct PackOut {
  smr_read_result* res; smr_aln* aln; smr_aln_stats* st; uint32_t* cigar;   // st: null = no stats
  const uint64_t* aln_off;   // read r's first row (the scan of nal)
  const uint64_t* cig_off;   // read r's first CIGAR word (the scan of words, indexed as pack_count_kernel wrote it)
};

// A group of G = 2^lg lanes per read (32 in the packed layout, where a read may hold thousands of alignments; in the
// strided layout the smallest power of two >= the stride, up to 32), 32 / G reads per warp pass.  The group's first lane writes
// its result; the lanes take its rows G at a time, each placing one alignment, its stats and its CIGAR words after those of the
// lanes before it (a scan of cigar_len over the group), or zeros past n_align (strided).  stride: as pack_count_kernel.
__global__ void __launch_bounds__(256) pack_scatter_kernel(const PackRun* __restrict__ runs, const uint2* __restrict__ src, uint32_t n,
                                                           uint32_t stride, uint32_t lg, PackOut o) {
  const uint32_t G = 1u << lg, lane = threadIdx.x & 31, q = lane & (G - 1), per = 32u >> lg;
  const uint32_t warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t r0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * per; r0 < n; r0 += warps * per) {   // warp-uniform
    const bool live = r0 + (lane >> lg) < n;   // a group past the last read takes part in the shuffles with no rows to write
    const uint32_t r = min(r0 + (lane >> lg), n - 1);
    const uint2 s = src[r];
    const PackRun& d = runs[s.x];
    const ReadState st = d.st[s.y];
    if (live && q == 0) {
      smr_read_result x;
      x.lastIndex = st.lastIndex; x.lastPart = st.lastPart; x.hit_seeds = st.hit_seeds; x.min_index = st.min_index; x.max_index = st.max_index;
      x.n_align = st.n_align; x.max_SW_count = st.max_SW_count; x.is_done = st.is_done; x.is_hit = st.is_hit;
      o.res[r] = x;
    }
    const size_t b = d.base ? (size_t)d.base[s.y] : (size_t)s.y * d.slots;
    const uint32_t na = !live ? 0 : stride ? min(st.n_align, stride) : st.n_align, rows = stride ? stride : st.n_align;   // rows: uniform over the warp
    const uint64_t to = o.aln_off[r];
    uint64_t at = o.cig_off[stride ? (size_t)d.first + s.y : r];
    for (uint32_t j0 = 0; j0 < rows; j0 += G) {
      const uint32_t j = j0 + q;
      const uint32_t len = j < na ? d.oa[b + j].cigar_len : 0;
      uint32_t incl = len;
      for (uint32_t k = 1; k < G; k <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, k, G);
        if (q >= k) incl += v;
      }
      if (j < na) {
        const OutAln a = d.oa[b + j];
        const uint64_t c = at + incl - len;
        for (uint32_t w = 0; w < a.cigar_len; ++w) o.cigar[c + w] = d.cigar[a.cigar_off + w];
        smr_aln x = {};
        x.cigar_off = (uint32_t)c; x.cigar_len = a.cigar_len;
        x.ref_num = a.ref_num; x.ref_begin1 = a.ref_begin1; x.ref_end1 = a.ref_end1; x.read_begin1 = a.read_begin1; x.read_end1 = a.read_end1;
        x.readlen = a.readlen; x.score1 = a.score1; x.part = a.part; x.index_num = a.index_num; x.strand = a.strand;
        o.aln[to + j] = x;
        if (o.st) { const AlnStats q2 = d.ast[b + j]; o.st[to + j] = smr_aln_stats{q2.n_miss, q2.n_gap, q2.n_match, q2.n_match_denovo}; }
      } else if (live && j < rows) {
        o.aln[to + j] = smr_aln{};
        if (o.st) o.st[to + j] = smr_aln_stats{};
      }
      at += __shfl_sync(0xffffffffu, incl, G - 1, G);
    }
  }
}

}  // namespace smr
