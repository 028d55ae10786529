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

}  // namespace smr
