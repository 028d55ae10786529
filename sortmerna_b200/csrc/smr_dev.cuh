// Device-side data layout shared by all kernels (sm_90a).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace smr {

constexpr int kWarp = 32;
constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr uint32_t kNoneDev = 0xFFFFFFFFu;

// One loaded (index, part); every pointer is HBM-resident (see smr_index.h for the layout).  The search arrays (flookup .. pos) are
// those of the part's resident group (an index budget runs a batch over groups of parts, smr_set_index_budget); refseq and ref_off
// are always resident.
struct DevIndex {
  uint32_t index_num, part, lnwin, partialwin;
  uint32_t minimal_score;
  uint32_t skip[3];
  uint32_t nref, nids;
  uint32_t is_last;          // last (index,part) in --ref order (paralleltraversal.cpp:294)
  uint16_t slot;             // ordinal of this part in its resident group: its hit regions and the group's part table (LisGlobals::parts)
  uint16_t gslot;            // ordinal of this part in the context: AlnWork::idx_slot, the full part table (FinalGlobals::parts)
  const uint4* flookup;      // [4^partialwin] {offF, cntF, offR, cntR}: entry indices into ftext and fid
  const uint32_t* ftext;     // entry texts (path + tail, partialwin+1 chars, first char lowest), DFS order per (9-mer, direction);
                             // zero-padded to a multiple of 8 entries (the seed kernel reads whole aligned 32-byte chunks)
  const uint32_t* fid;       // entry ids, same order
  const uint32_t* pos_off;   // [nids+1]
  const uint2* pos;          // {pos, seq}, each id's list sorted by (seq,pos)
  const uint8_t* refseq;     // 0..4
  const uint32_t* ref_off;   // [nref+1]
};
// words allocated for the texts of n entries
__host__ __device__ inline size_t ftext_words(size_t n) { return (n + 7) & ~(size_t)7; }

struct DevParams {
  int32_t match, mismatch, score_N, gap_open, gap_ext;
  int32_t num_seeds, min_lis, edges, edges_is_percent;
  int32_t num_alignments, is_best;
  int32_t is_forward, is_reverse, is_full_search;
  int32_t one;   // 1 (run-time constant, see SwScore::one)
};

// Per-read carried state = the KVDB blob of the reference (read.cpp:429-462) + pass-local flags.
struct ReadState {
  uint32_t lastIndex, lastPart;
  uint32_t hit_seeds;
  uint32_t min_index, max_index;
  uint32_t n_align;
  uint16_t max_SW_count;
  uint8_t is_done, is_hit;
};

// A stored alignment while the batch is in flight.  Begin coordinates and the CIGAR are produced
// by the finalize kernel (reverse pass + banded traceback are pure functions of these fields).
struct AlnWork {
  uint32_t ref_num;
  uint32_t win_ref_start;   // align_ref_start - head (alignment.cpp:373)
  uint32_t win_len;         // align_length
  uint32_t q_start, q_len;  // align_que_start, align_length - head - tail (alignment.cpp:365-366)
  uint16_t score1, part, index_num;
  uint16_t idx_slot;        // ordinal of the loaded (index,part) in the context
  uint8_t strand, pad0;
};

// hit record produced by the seed kernel: id + (window position | variant << 24)
constexpr uint32_t kVarFwd = 0, kVarRevT = 1, kVarRevA = 2;  // reverse strand with N->T / N->A (SURVEY A.10)
constexpr uint32_t kWinMask = 0x00FFFFFFu;   // hit.y = window position | variant << 24 | pass class << 28 (the first pass whose grid holds the position)

// overflow / status flags per read (cleared by a retry with larger scratch)
constexpr uint32_t kOvfSeedLane = 1u;   // more hits in one window than the per-lane buffer
constexpr uint32_t kOvfSeedRegion = 2u; // more hits for the read than its region
constexpr uint32_t kOvfPairs = 4u;      // candidate with more (refpos,readpos) pairs than the pair buffer
constexpr uint32_t kOvfTrace = 8u;      // traceback direction matrix larger than the arena
constexpr uint32_t kOvfCigar = 16u;     // cigar pool exhausted
constexpr uint32_t kErrTrace = 32u;     // "Trace back error" (ssw.c:707) -- fatal in the reference
constexpr uint32_t kOvfSlots = 64u;     // num_alignments == 0: more accepted alignments than the caller's stride (not retried: SMR_ERR_CAPACITY)

// instrumentation counters (device side, u64), same order as SMR_CNT_* after the first two
enum DevCnt { dcNumAligned = 0, dcNumShort, dcSwCalls, dcSwCells, dcWindows, dcNodes, dcBuckets, dcEntries, dcPosEntries,
              dcLisCalls, dcMaxReadCycles, dcSumReadCycles, dcLisKernelCycles,
              dcCycVote, dcCycOrder, dcCycGroup, dcCycPlan, dcCycWait, dcCycReplay, dcSpecCalls, dcSpecCells, dcSpecPairs, dcSlowPairs,
              dcScWait, dcScLoad, dcScSw, dcScPub, dcRoundsA, dcRoundsB, dcW1Cyc, dcW1Cnt, dcMaxReadBusy, dcCount = 32 };

__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}
__device__ __forceinline__ uint32_t warp_sum_u32(uint32_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}
__device__ __forceinline__ uint32_t warp_incl_scan_u32(uint32_t v) {
  const unsigned l = lane_id();
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(kFull, v, o); if ((int)l >= o) v += t; }
  return v;
}

}  // namespace smr
