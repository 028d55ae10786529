// Device placement of a run's results (smr_place_results): the strided run of a batch -> the caller's strided layout of
// smr_download_results, written into device arrays the report-side calls read in place.  The bytes are those the host download
// writes: smr_read_result[n], smr_aln[n * slots] zeroed past n_align, smr_aln_stats alike, and the CIGARs compacted in read order
// from `base` (a scratch-overflow retry appends after the reads placed before it).  One count pass (CIGAR words per read and the
// counters), one exclusive scan of the words, one scatter pass.  Reads flagged by the run (scratch overflow, kOvfSlots, trace
// error) are skipped: their rows are written by the retry that runs them, or the placement fails.
#pragma once
#include "smr_final.cuh"
#include "../../include/smr_b200.h"

namespace smr {

// what the count pass hands to the host
struct PlaceWords {
  uint32_t trace;       // a read carries kErrTrace
  uint32_t need_slots;  // the largest n_align of a read flagged kOvfSlots (0: none)
  uint32_t flagged;     // reads flagged for a retry
  uint32_t pad;
};

// one run of a batch, as the run left it on the device
struct PlaceIn {
  const ReadState* st; const uint32_t* flags; const uint16_t* hit_db; const OutAln* oa; const AlnStats* ast;   // ast: null = no stats
  const uint32_t* cigar;   // the run's device CIGAR pool (OutAln::cigar_off indexes it)
  uint32_t n, slots;
};

// words[r] = CIGAR words of read r (0 for a flagged read), words[n] = 0; counters into cnt[0 .. ncnt): SMR_CNT_NUM_ALIGNED and
// reads_matched_per_db per read placed, and the run's device counters 1 .. dcCount - 1 (block 0).  Dynamic shared memory: ncnt u64.
__global__ void __launch_bounds__(256) place_count_kernel(PlaceIn in, const unsigned long long* __restrict__ dev_cnt, uint64_t* __restrict__ words,
                                                          unsigned long long* __restrict__ cnt, uint32_t ncnt, PlaceWords* __restrict__ w) {
  extern __shared__ unsigned long long s_cnt[];
  for (uint32_t k = threadIdx.x; k < ncnt; k += blockDim.x) s_cnt[k] = 0;
  __syncthreads();
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < in.n; r += gridDim.x * blockDim.x) {
    const uint32_t f = in.flags[r];
    uint64_t sum = 0;
    if (f) {
      if (f & kErrTrace) atomicOr(&w->trace, 1u);
      if (f & kOvfSlots) atomicMax(&w->need_slots, in.st[r].n_align);
      else atomicAdd(&w->flagged, 1u);
    } else {
      const ReadState s = in.st[r];
      const uint32_t na = min(s.n_align, in.slots);
      for (uint32_t k = 0; k < na; ++k) sum += in.oa[(size_t)r * in.slots + k].cigar_len;
      if (s.is_hit) {
        atomicAdd(&s_cnt[SMR_CNT_NUM_ALIGNED], 1ull);
        const uint16_t db = in.hit_db[r];
        if (db != 0xFFFF && SMR_CNT_FIXED + (uint32_t)db < ncnt) atomicAdd(&s_cnt[SMR_CNT_FIXED + db], 1ull);
      }
    }
    words[r] = sum;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) words[in.n] = 0;
  __syncthreads();
  for (uint32_t k = threadIdx.x; k < ncnt; k += blockDim.x) {
    unsigned long long v = s_cnt[k];
    if (blockIdx.x == 0 && k >= dcNumShort && k < dcCount) v += dev_cnt[k];
    if (v) atomicAdd(&cnt[k], v);
  }
}

// where the placed results go
struct PlaceOut {
  smr_read_result* res; smr_aln* aln; smr_aln_stats* st;   // st: null = no stats
  uint32_t* cigar;
  const uint32_t* map;     // read r of the run -> its row (null: r)
  uint64_t base;           // the CIGAR words placed before this run
};

// one thread per read: its result, its `slots` alignment rows and its CIGARs at base + off[r]
__global__ void __launch_bounds__(256) place_scatter_kernel(PlaceIn in, const uint64_t* __restrict__ off, PlaceOut o) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < in.n; r += gridDim.x * blockDim.x) {
    if (in.flags[r]) continue;
    const uint32_t dst = o.map ? o.map[r] : r;
    const ReadState s = in.st[r];
    smr_read_result x;
    x.lastIndex = s.lastIndex; x.lastPart = s.lastPart; x.hit_seeds = s.hit_seeds; x.min_index = s.min_index; x.max_index = s.max_index;
    x.n_align = s.n_align; x.max_SW_count = s.max_SW_count; x.is_done = s.is_done; x.is_hit = s.is_hit;
    o.res[dst] = x;
    uint64_t at = o.base + off[r];
    for (uint32_t k = 0; k < in.slots; ++k) {
      const size_t src = (size_t)r * in.slots + k, to = (size_t)dst * in.slots + k;
      smr_aln a = {};
      smr_aln_stats t = {};
      if (k < s.n_align) {
        const OutAln d = in.oa[src];
        for (uint32_t j = 0; j < d.cigar_len; ++j) o.cigar[at + j] = in.cigar[d.cigar_off + j];
        a.cigar_off = (uint32_t)at; a.cigar_len = d.cigar_len; at += d.cigar_len;
        a.ref_num = d.ref_num; a.ref_begin1 = d.ref_begin1; a.ref_end1 = d.ref_end1; a.read_begin1 = d.read_begin1; a.read_end1 = d.read_end1;
        a.readlen = d.readlen; a.score1 = d.score1; a.part = d.part; a.index_num = d.index_num; a.strand = d.strand;
        if (o.st) { const AlnStats q = in.ast[src]; t = smr_aln_stats{q.n_miss, q.n_gap, q.n_match, q.n_match_denovo}; }
      }
      o.aln[to] = a;
      if (o.st) o.st[to] = t;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Packed placement (smr_place_results_packed, smr_download_results_packed): every read's final results, from the first run
// (strided at the first stride) or from the re-run that stored it at its own count, placed in read order with no stride:
// smr_aln[sum n_align] and smr_aln_stats alike, aln_off[n + 1], the CIGARs compacted in read order.  The runs stay on the device
// until the scatter; src[r] names the run and the read in it that hold read r's results.
// ---------------------------------------------------------------------------------------------------------------------
// one run of a packed placement, as the run left it on the device
struct PackRun {
  const ReadState* st; const uint16_t* hit_db; const OutAln* oa; const AlnStats* ast; const uint32_t* cigar;
  const uint32_t* base;        // read k's first slot (a re-run's packed arenas); null: k * slots
  const unsigned long long* cnt;   // the run's device counters
  uint32_t slots, pad;
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

// nal[r] = n_align and words[r] = CIGAR words of read r from its source run, nal[n] = words[n] = 0; counters into cnt[0 .. ncnt):
// SMR_CNT_NUM_ALIGNED and reads_matched_per_db once per read, and the device counters 1 .. dcCount - 1 of every run (block 0).
// Dynamic shared memory: ncnt u64.
__global__ void __launch_bounds__(256) pack_count_kernel(const PackRun* __restrict__ runs, uint32_t nruns, const uint2* __restrict__ src,
                                                         uint32_t n, uint64_t* __restrict__ nal, uint64_t* __restrict__ words,
                                                         unsigned long long* __restrict__ cnt, uint32_t ncnt) {
  extern __shared__ unsigned long long s_cnt[];
  for (uint32_t k = threadIdx.x; k < ncnt; k += blockDim.x) s_cnt[k] = 0;
  __syncthreads();
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    const uint2 s = src[r];
    const PackRun& d = runs[s.x];
    const ReadState st = d.st[s.y];
    const size_t b = d.base ? (size_t)d.base[s.y] : (size_t)s.y * d.slots;
    uint64_t sum = 0;
    for (uint32_t j = 0; j < st.n_align; ++j) sum += d.oa[b + j].cigar_len;
    nal[r] = st.n_align;
    words[r] = sum;
    if (st.is_hit) {
      atomicAdd(&s_cnt[SMR_CNT_NUM_ALIGNED], 1ull);
      const uint16_t db = d.hit_db[s.y];
      if (db != 0xFFFF && SMR_CNT_FIXED + (uint32_t)db < ncnt) atomicAdd(&s_cnt[SMR_CNT_FIXED + db], 1ull);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { nal[n] = 0; words[n] = 0; }
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

// where the packed results go
struct PackOut {
  smr_read_result* res; smr_aln* aln; smr_aln_stats* st; uint32_t* cigar;
  const uint64_t* aln_off;   // read r's first alignment (the scan of n_align)
  const uint64_t* cig_off;   // read r's first CIGAR word (the scan of its words)
};

// One warp per read: lane 0 writes its result; the lanes take its alignments 32 at a time, each placing one alignment, its stats
// and its CIGAR words after those of the lanes before it (a warp scan of cigar_len).  A read may hold thousands of alignments.
__global__ void __launch_bounds__(256) pack_scatter_kernel(const PackRun* __restrict__ runs, const uint2* __restrict__ src, uint32_t n,
                                                           PackOut o) {
  const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += warps) {
    const uint2 s = src[r];
    const PackRun& d = runs[s.x];
    const ReadState st = d.st[s.y];
    if (lane == 0) {
      smr_read_result x;
      x.lastIndex = st.lastIndex; x.lastPart = st.lastPart; x.hit_seeds = st.hit_seeds; x.min_index = st.min_index; x.max_index = st.max_index;
      x.n_align = st.n_align; x.max_SW_count = st.max_SW_count; x.is_done = st.is_done; x.is_hit = st.is_hit;
      o.res[r] = x;
    }
    const size_t b = d.base ? (size_t)d.base[s.y] : (size_t)s.y * d.slots;
    const uint64_t to = o.aln_off[r];
    uint64_t at = o.cig_off[r];
    for (uint32_t j0 = 0; j0 < st.n_align; j0 += 32) {
      const uint32_t j = j0 + lane;
      const uint32_t len = j < st.n_align ? d.oa[b + j].cigar_len : 0;
      uint32_t incl = len;
      for (uint32_t k = 1; k < 32; k <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, k);
        if (lane >= k) incl += v;
      }
      if (j < st.n_align) {
        const OutAln a = d.oa[b + j];
        const uint64_t c = at + incl - len;
        for (uint32_t w = 0; w < a.cigar_len; ++w) o.cigar[c + w] = d.cigar[a.cigar_off + w];
        smr_aln x = {};
        x.cigar_off = (uint32_t)c; x.cigar_len = a.cigar_len;
        x.ref_num = a.ref_num; x.ref_begin1 = a.ref_begin1; x.ref_end1 = a.ref_end1; x.read_begin1 = a.read_begin1; x.read_end1 = a.read_end1;
        x.readlen = a.readlen; x.score1 = a.score1; x.part = a.part; x.index_num = a.index_num; x.strand = a.strand;
        o.aln[to + j] = x;
        if (o.st) { const AlnStats q = d.ast[b + j]; o.st[to + j] = smr_aln_stats{q.n_miss, q.n_gap, q.n_match, q.n_match_denovo}; }
      }
      at += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
}

}  // namespace smr
