// Seed search: one warp per read, one lane per 18-mer window, both strands, all three passes.
//
// Stands in for the window loop of traverse() (src/sortmerna/paralleltraversal.cpp:124-250), the
// bit-vector construction init_win_f/init_win_r (src/sortmerna/bitvector.cpp:56-132), Read::hashKmer
// (src/sortmerna/read.cpp:601-611) and the trie x Levenshtein-automaton DFS traversetrie_align
// (src/sortmerna/traverse_bursttrie.cpp:100-298).
//
// GPU mapping: the index is a set of flat HBM arrays (smr_index.h); a window search is a chain of
// dependent 8/32-byte sector reads (lookup -> root node -> child nodes -> bucket entries), so the
// kernel is HBM/L2-latency bound and is parallelised over (read, strand, window) -- 90 windows per
// 150-nt read -- with warp ballot/shuffle compaction of the hits into a per-read region.
// All windows of all passes are searched up front (a window's hits depend only on (read, strand,
// position, index)); the candidate kernel later replays the reference's pass order on them.
#pragma once
#include "smr_dev.cuh"
#include "smr_levbits.h"

namespace smr {

// ---------------------------------------------------------------------------------------------
// How a window is searched here.
//
// The reference walks the mini burst trie of the window's exact 9-mer half in lock step with a table-driven
// universal Levenshtein automaton for d=1 (traverse_bursttrie.cpp:68-298, bit-vectors bitvector.cpp:56-132),
// pruning sub-tries the automaton rejects.  That automaton accepts at depth d exactly when the d+1 text
// characters read so far are within one edit of the 9-nt other half, and reaches state 9 at depth 8 exactly
// on an exact match (proved against the table and against dynamic-programming edit distance on millions of
// cases: tests/test_lev_equivalence.py; the oracle keeps the table).  Pointer chasing and per-window DFS
// stacks are the wrong shape for a GPU (the first version of this kernel ran with 2 of 32 lanes active), so:
//   * at load time every mini trie is flattened into ONE contiguous list of its entries in the DFS order of
//     the reference, each entry carrying its full text = trie path letters + bucket tail (smr_index.h);
//   * a window search tests EVERY entry of the list of its 9-mer with bit-parallel predicates (smr_levbits.h) --
//     entries in sub-tries the reference would have pruned simply classify as "no match", so the outcome is the
//     same, and the ~2.4x more entries cost less than the pruning did;
//   * the 32 windows of a round are searched together: their lists form one entry stream, eight entry texts per
//     lane per step (one aligned 32-byte sector, no divergence), each screened with four masked compares
//     (half_screen); the few survivors are compacted with ballot/popc into a shared list, classified exactly there
//     (classify_bits, which drops the survivors that do not match), and each lane then replays the reference's
//     order-dependent rules (0-error exit, per-window de-duplication, traverse_bursttrie.cpp:249-281) over its own
//     matches.
// ---------------------------------------------------------------------------------------------
// reverse the order of the pw 2-bit characters of v
__device__ __forceinline__ uint32_t rev_chars(uint32_t v, uint32_t pw) {
  uint32_t x = __brev(v) >> (32 - 2 * pw);
  return ((x & 0x55555555u) << 1) | ((x >> 1) & 0x55555555u);
}

// 2-bit packed reads, first base most significant: base i of a read lives in word i>>4 at bit 30-2*(i&15).
// Returns the L-mer starting at forward position p as a 2L-bit integer (first base most significant).
__device__ __forceinline__ uint64_t window_fwd(const uint32_t* __restrict__ pk, uint32_t p, uint32_t L) {
  const uint32_t wi = p >> 4, s = 2 * (p & 15);
  const uint64_t hi = ((uint64_t)__ldg(pk + wi) << 32) | __ldg(pk + wi + 1);
  const uint64_t lo = (uint64_t)__ldg(pk + wi + 2) << 32;
  const uint64_t v = s ? ((hi << s) | (lo >> (64 - s))) : hi;
  return v >> (64 - 2 * L);
}
// reverse complement of a 2L-bit L-mer (Read::revIntStr, read.cpp:350-357, on the 0..3 alphabet)
__device__ __forceinline__ uint64_t revcomp_bits(uint64_t v, uint32_t L) {
  uint64_t x = __brevll(v) >> (64 - 2 * L);
  x = ((x & 0x5555555555555555ull) << 1) | ((x >> 1) & 0x5555555555555555ull);
  return ~x & ((1ull << (2 * L)) - 1);
}

// Per-lane hit buffer (ids of one window, needed for the per-window de-duplication,
// traverse_bursttrie.cpp:265-279).  The first kLaneSmemIds slots live in shared memory (slot k at sbuf[k*32]), the rest in
// an HBM scratch (slot k at buf[k*stride]); a window rarely has more than three ids.
constexpr uint32_t kLaneSmemIds = 8;
struct LaneHits {
  uint32_t* sbuf; uint32_t* buf; uint32_t stride, cap, n; bool overflow;
};
__device__ __forceinline__ uint32_t lh_get(const LaneHits& lh, uint32_t k) { return k < kLaneSmemIds ? lh.sbuf[k * 32] : lh.buf[k * lh.stride]; }
__device__ __forceinline__ void lh_set(LaneHits& lh, uint32_t k, uint32_t id) { if (k < kLaneSmemIds) lh.sbuf[k * 32] = id; else lh.buf[k * lh.stride] = id; }

struct SeedStats { uint32_t entries, lists; };   // list entries classified; non-empty flat lists scanned (the "buckets" of SURVEY 8(d): one per sub-search)

// the reference's per-entry side effects (traverse_bursttrie.cpp:249-281) applied to a classification code;
// returns true when the window search ends on a 0-error match
__device__ __forceinline__ bool apply_entry(uint32_t code, uint32_t id, bool full_search, LaneHits& lh) {
  const uint32_t d1 = code & 3u;
  if (d1 == 0) return false;
  const bool z = (code & 4u) && !full_search;
  if (d1 == 2 && z) { lh.n = 1; lh_set(lh, 0, id); lh.overflow = false; return true; }                // :256-262
  for (uint32_t f = 0; f < lh.n && f < lh.cap; ++f) if (lh_get(lh, f) == id) return false;             // duplicate: :265-277
  if (lh.n < lh.cap) lh_set(lh, lh.n, id); else lh.overflow = true;
  lh.n++;
  if (d1 == 1 && z) { lh.n = 1; lh_set(lh, 0, id); lh.overflow = false; return true; }                // 0-error one step after the push
  return false;
}

// class of a window position = the first pass whose grid contains it (paralleltraversal.cpp:118-131)
__device__ __forceinline__ uint32_t pass_class(uint32_t p, uint32_t s0, uint32_t s1, uint32_t s2) {
  if (p % s0 == 0) return 0;
  if (p % s1 == 0) return 1;
  if (p % s2 == 0) return 2;
  return 3;
}

constexpr int kAccStep = 256;  // survivors one step can add (32 lanes x 8 entries)
constexpr int kAccCap = 384;   // entries buffered: a step that leaves more than kAccCap - kAccStep classifies them, and flushes when more
                               // than that many are matches, so the next step fits

struct CoopSmem {              // per warp
  uint4 tab[64];               // the non-empty lists of a round in stream order: {first chunk - first stream chunk, pattern, first entry, end entry}
  uint32_t id[kAccCap];        // buffered entries in stream order: entry index (its id once the flush has loaded it), text (its
  uint32_t text[kAccCap];      // classification code once classified), owner
  uint8_t meta[kAccCap];       // owner lane | 32 for a mirror list
  uint8_t own[64];             // the same for list k
  uint16_t run[2][2][32];      // [forward / mirror][begin / end][lane]: the lane's matches of the current flush
  uint32_t ids[kLaneSmemIds][32];   // LaneHits::sbuf
};

// The two sub-searches of the 32 windows of a round as ONE entry stream:
//   (a) forward: trie_F list of the first half, pattern = second half (paralleltraversal.cpp:161-186);
//   (b) mirror: trie_R list of the second half, pattern = first half (:188-240) -- the reference runs (b) only without a
//       0-error hit in (a); here every (a) list precedes every (b) list in the stream and a lane stops replaying its matches
//       at its 0-error hit, so streaming (b) regardless changes nothing but the entries read (~5 % of the windows).
// The unit of work is a CHUNK = the texts of one aligned group of eight entries (one 32-byte sector of ix.ftext, two 16-byte
// loads): a lane finds the list of its chunk once (REDUX.OR of the lists that start in this step + popc, one shared-memory row)
// and screens eight texts with half_screen(), which passes every text within one edit and ~1 % of the others.  The ids are not
// streamed: survivors (text, entry index, owner) are compacted in stream order; when the buffer fills, the lanes classify the
// new survivors 32 at a time with their owner's pattern (classify_bits) and keep only the matches, in place and in order.  At a
// flush the lanes load the ids of all buffered matches from ix.fid, then every lane finds the (at most two) runs of its own
// matches and replays them -- the reference's order-dependent rules (0-error exit, per-window de-duplication,
// traverse_bursttrie.cpp:249-281) -- all lanes in parallel.
// offF/cntF/PF, offR/cntR/PR: the lane's two lists, entry indices into ix.ftext / ix.fid (cnt == 0: none).  Appends to lh; sets zero.
template <bool INSTR>
__device__ void coop_stream(const DevIndex& ix, CoopSmem& sm, const uint32_t offF, const uint32_t cntF, const uint32_t PF,
                            const uint32_t offR, const uint32_t cntR, const uint32_t PR, const bool full_search,
                            LaneHits& lh, bool& zero, SeedStats& st) {
  const unsigned lane = lane_id();
  const uint32_t pw = ix.partialwin;
  const HalfMasks km = half_masks(pw);
  const uint4* __restrict__ ft4 = reinterpret_cast<const uint4*>(ix.ftext);   // chunk g = ft4[2g], ft4[2g+1]
  const uint32_t gF = offF >> 3, nF = cntF ? ((offF + cntF + 7u) >> 3) - gF : 0u;
  const uint32_t gR = offR >> 3, nR = cntR ? ((offR + cntR + 7u) >> 3) - gR : 0u;
  const uint32_t inF = warp_incl_scan_u32(nF), inR = warp_incl_scan_u32(nR);
  const uint32_t totF = __shfl_sync(kFull, inF, 31), E = totF + __shfl_sync(kFull, inR, 31);
  const uint32_t exF = nF ? inF - nF : kNoneDev, exR = nR ? totF + inR - nR : kNoneDev;   // first stream chunk of each list (none: never starts)
  if (INSTR) { st.entries += cntF + cntR; st.lists += (cntF ? 1u : 0u) + (cntR ? 1u : 0u); }
  if (E == 0) return;
  const uint32_t lt = (1u << lane) - 1u, le = lt | (1u << lane);
  {
    const unsigned mF = __ballot_sync(kFull, nF != 0), mR = __ballot_sync(kFull, nR != 0);
    if (nF) { const uint32_t k = __popc(mF & lt); sm.tab[k] = make_uint4(gF - exF, PF, offF, offF + cntF); sm.own[k] = (uint8_t)lane; }
    if (nR) { const uint32_t k = __popc(mF) + __popc(mR & lt); sm.tab[k] = make_uint4(gR - exR, PR, offR, offR + cntR); sm.own[k] = (uint8_t)(lane | 32u); }
  }
  __syncwarp();
  uint32_t cum = 0, nacc = 0, ncls = 0;   // buffered entries; the first ncls of them are classified matches
  // the chunk of a lane in step e0: its list (row k of the table), its chunk g, the list's pattern and its two 16-byte loads --
  // issued one step ahead of their use (the list's bounds are read from the table only when the chunk has a match)
  uint32_t kn, gn, Pn; uint4 q0n, q1n;
  auto fetch = [&](const uint32_t e0) {
    const uint32_t dF = exF - e0, dR = exR - e0;   // a list that began in an earlier step wraps to a huge value
    const uint32_t bit = (dF < 32u ? (1u << dF) : 0u) | (dR < 32u ? (1u << dR) : 0u);
    const uint32_t starts = __reduce_or_sync(kFull, bit);
    const uint32_t e = e0 + lane;
    kn = cum + __popc(starts & le) - 1u;      // the list of chunk e (step 0 always has a list starting at chunk 0)
    cum += __popc(starts);
    const uint2 t = *reinterpret_cast<const uint2*>(&sm.tab[kn]);
    gn = t.x + e; Pn = t.y;
    q0n = make_uint4(0, 0, 0, 0); q1n = q0n;
    if (e < E) { q0n = __ldg(ft4 + 2 * (size_t)gn); q1n = __ldg(ft4 + 2 * (size_t)gn + 1); }
  };
  fetch(0);
  for (uint32_t e0 = 0; e0 < E; e0 += 32) {
    const uint32_t k = kn, g = gn, P = Pn; const uint4 q0 = q0n, q1 = q1n;
    if (e0 + 32 < E) fetch(e0 + 32);
    const uint32_t Pd = P >> 2, Pi = P << 2;
    const uint32_t hit8 = (half_screen(P, Pd, Pi, q0.x, km) ? 1u : 0u) | (half_screen(P, Pd, Pi, q0.y, km) ? 2u : 0u) |
                          (half_screen(P, Pd, Pi, q0.z, km) ? 4u : 0u) | (half_screen(P, Pd, Pi, q0.w, km) ? 8u : 0u) |
                          (half_screen(P, Pd, Pi, q1.x, km) ? 16u : 0u) | (half_screen(P, Pd, Pi, q1.y, km) ? 32u : 0u) |
                          (half_screen(P, Pd, Pi, q1.z, km) ? 64u : 0u) | (half_screen(P, Pd, Pi, q1.w, km) ? 128u : 0u);
    const bool any = e0 + lane < E && hit8;
    const unsigned am = __ballot_sync(kFull, any);
    if (am) {   // entries outside [first, end) of the list dropped, survivors compacted in stream order (lane-major, then entry)
      uint32_t mk = 0;
      const uint32_t i0 = 8u * g;
      if (any) {
        const uint2 t = *reinterpret_cast<const uint2*>(&sm.tab[k].z);
        const uint32_t lo = t.x > i0 ? min(t.x - i0, 8u) : 0u, hi = min(t.y - i0, 8u);
        mk = hit8 & ((1u << hi) - 1u) & ~((1u << lo) - 1u);
      }
      const uint32_t nm = __popc(mk);
      const unsigned b0 = __ballot_sync(kFull, nm & 1u), b1 = __ballot_sync(kFull, nm & 2u), b2 = __ballot_sync(kFull, nm & 4u),
                     b3 = __ballot_sync(kFull, nm & 8u);
      uint32_t slot = nacc + __popc(b0 & lt) + 2u * __popc(b1 & lt) + 4u * __popc(b2 & lt) + 8u * __popc(b3 & lt);
      const uint8_t own = sm.own[k];
      while (mk) {
        const uint32_t j = (uint32_t)__ffs((int)mk) - 1u;
        mk &= mk - 1u;
        const uint4 q = j < 4 ? q0 : q1;
        const uint32_t jj = j & 3u;
        sm.text[slot] = jj == 0 ? q.x : (jj == 1 ? q.y : (jj == 2 ? q.z : q.w));
        sm.id[slot] = i0 + j;
        sm.meta[slot] = own;
        ++slot;
      }
      nacc += __popc(b0) + 2u * __popc(b1) + 4u * __popc(b2) + 8u * __popc(b3);
    }
    const bool last = e0 + 32 >= E;
    if (nacc > ncls && (nacc > (uint32_t)(kAccCap - kAccStep) || last)) {
      // classify the survivors not classified yet with their owner's pattern and keep the matches in place, in stream order
      // (the text slot then holds the classification code); the buffer is replayed once it holds enough matches
      __syncwarp();   // the survivors the lanes compacted above are visible to every lane
      uint32_t nm = ncls;
      for (uint32_t b = ncls; b < nacc; b += 32) {
        const uint32_t i = b + lane;
        const bool in = i < nacc;
        const uint32_t m = in ? sm.meta[i] : 0u, x = in ? sm.id[i] : 0u;
        const uint32_t Pf = __shfl_sync(kFull, PF, m & 31u), Pr = __shfl_sync(kFull, PR, m & 31u);
        const uint32_t code = in ? classify_bits((m & 32u) ? Pr : Pf, sm.text[i], pw) : 0u;
        const unsigned keep = __ballot_sync(kFull, (code & 3u) != 0u);
        __syncwarp();   // every lane has read its slot before any is overwritten
        if ((code & 3u) != 0u) {
          const uint32_t o = nm + __popc(keep & lt);
          sm.text[o] = code; sm.id[o] = x; sm.meta[o] = (uint8_t)m;
        }
        nm += __popc(keep);
        __syncwarp();
      }
      nacc = ncls = nm;
    }
    if (nacc && (nacc > (uint32_t)(kAccCap - kAccStep) || last)) {   // flush the matches: load their ids and replay them
      sm.run[0][0][lane] = 0; sm.run[0][1][lane] = 0; sm.run[1][0][lane] = 0; sm.run[1][1][lane] = 0;
      __syncwarp();
      for (uint32_t i = lane; i < nacc; i += 32) {   // a list's matches are contiguous: mark where each (owner, direction) run begins and ends
        sm.id[i] = __ldg(ix.fid + sm.id[i]);
        const uint32_t m = sm.meta[i];
        const uint32_t prev = i ? sm.meta[i - 1] : 0xFFu, next = i + 1 < nacc ? sm.meta[i + 1] : 0xFFu;
        if (m != prev) sm.run[m >> 5][0][m & 31u] = (uint16_t)i;
        if (m != next) sm.run[m >> 5][1][m & 31u] = (uint16_t)(i + 1);
      }
      __syncwarp();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t end = sm.run[h][1][lane];
        for (uint32_t i = sm.run[h][0][lane]; i < end && !zero; ++i) zero = apply_entry(sm.text[i], sm.id[i], full_search, lh);
      }
      nacc = ncls = 0;
      __syncwarp();
    }
  }
  __syncwarp();   // the table is rewritten by the next round
}

// ---------------------------------------------------------------------------------------------
// batch layout on the device
// ---------------------------------------------------------------------------------------------
struct DevBatch {
  uint32_t nreads;
  const uint8_t* seq04;      // 0..4, concatenated
  const uint32_t* seq_off;   // [nreads+1]
  const uint32_t* pk03;      // 2-bit packed, N->A(0) (seqToIntStr, read.cpp:334-347)
  const uint32_t* pk03alt;   // 2-bit packed, N->T(3): its reverse complement is the "N->A" reverse strand (SURVEY A.10)
  const uint32_t* pk_off;    // [nreads+1] word offsets
  const uint8_t* has_n;      // [nreads]
  uint32_t hit_scale;        // read r owns hits[hit_base(r) .. +hit_cap(r)): see hit_base()/hit_cap()
  uint32_t seq_base0;        // seq_off of the first read of the chunk, r0 = first read of the chunk
  uint32_t r0;
  uint2* hits;               // {id, win_pos | variant<<24}; one region set per (index,part): part p starts at p*hits_stride
  size_t hits_stride;        // entries per part
  uint32_t cnt_stride;       // hit_cnt of (part p, read r) lives at hit_cnt[p*cnt_stride + (r - r0)]
  uint32_t* cost;            // [chunk] estimated candidate work of a read (sum of position-list lengths of its hits, all parts)
  uint32_t* bins;            // [kCostBins * cnt_stride] reads of this chunk binned by log2(cost): heaviest-first schedule
  uint32_t* bin_count;       // [kCostBins]
  uint16_t* hit_db;          // [nreads] index_num of the first accepted alignment (reads_matched_per_db)
  uint32_t* hit_cnt;         // [nreads]
  uint32_t* flags;           // [nreads] overflow flags
  ReadState* state;          // [nreads]
  unsigned long long* counters;  // [dcCount + n_index_files]
};

// per-read hit region: capacity proportional to the read length (2 hits per nucleotide covers the
// ~1 window per 3 nt x 2-3 strand variants with ~2-3 ids per window), scaled up on a retry
__device__ __forceinline__ uint32_t hit_cap(const DevBatch& b, uint32_t r) { return b.hit_scale * (2u * (b.seq_off[r + 1] - b.seq_off[r]) + 32u); }
__device__ __forceinline__ size_t hit_base(const DevBatch& b, uint32_t part, uint32_t r) {
  return (size_t)part * b.hits_stride + (size_t)b.hit_scale * (2ull * (b.seq_off[r] - b.seq_base0) + 32ull * (r - b.r0));
}
constexpr int kCostBins = 24;

// 2-bit packing of a batch: one warp per read
__global__ void pack_reads_kernel(DevBatch b, uint32_t* pk03, uint32_t* pk03alt, uint8_t* has_n) {
  // grid-stride over reads; each warp packs one read
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const unsigned lane = lane_id();
  for (uint32_t r = b.r0 + warp; r < b.r0 + b.nreads; r += nwarps) {
    const uint32_t o = b.seq_off[r], len = b.seq_off[r + 1] - o;
    const uint32_t wo = b.pk_off[r], nw = b.pk_off[r + 1] - wo;
    bool anyn = false;
    for (uint32_t w = lane; w < nw; w += 32) {
      uint32_t a = 0, t = 0;
      for (uint32_t k = 0; k < 16; ++k) {
        const uint32_t i = w * 16 + k;
        uint32_t c = i < len ? b.seq04[o + i] : 0u;
        uint32_t ca = c, ct = c;
        if (c > 3) { ca = 0; ct = 3; anyn = anyn || (i < len); }
        a |= ca << (30 - 2 * k); t |= ct << (30 - 2 * k);
      }
      pk03[wo + w] = a;
      if (pk03alt) pk03alt[wo + w] = t;
    }
    anyn = __any_sync(kFull, anyn);
    if (lane == 0) has_n[r] = anyn ? 1 : 0;
  }
}

// one window of a read: position, strand variant, the two 9-mer keys and their lookup rows
struct SeedWin { uint4 lf, lr; uint32_t keyf, keyr, p, var; bool active; };
__device__ __forceinline__ SeedWin seed_window(const DevIndex& ix, const uint32_t* __restrict__ pk, const uint32_t* __restrict__ pka, uint32_t len,
                                               uint32_t L, uint32_t pw, uint32_t npos, uint32_t step, uint32_t s0, uint32_t s1, uint32_t s2,
                                               uint32_t v_lo, uint32_t nq, uint32_t qq) {
  SeedWin w;
  const uint32_t vr = (qq >= npos ? 1u : 0u) + (qq >= 2 * npos ? 1u : 0u);   // windows are variant-major; at most three variants
  w.var = v_lo + vr; w.p = (qq - vr * npos) * step;
  w.active = qq < nq;
  if (w.active && step == 1) w.active = (w.p % s0 == 0) || (w.p % s1 == 0) || (w.p % s2 == 0);
  w.keyf = w.keyr = 0;
  w.lf = w.lr = make_uint4(0, 0, 0, 0);
  if (w.active) {
    uint64_t V;
    if (w.var == kVarFwd) V = window_fwd(pk, w.p, L);
    else V = revcomp_bits(window_fwd(w.var == kVarRevT ? pk : pka, len - w.p - L, L), L);
    w.keyf = (uint32_t)(V >> (2 * pw)); w.keyr = (uint32_t)(V & ((1ull << (2 * pw)) - 1));
    w.lf = __ldg(&ix.flookup[w.keyf]);
    w.lr = __ldg(&ix.flookup[w.keyr]);
  }
  return w;
}

constexpr int kSeedWarpsPerCta = 4;
#ifndef SMR_SEED_MIN_CTAS
#define SMR_SEED_MIN_CTAS 8
#endif
constexpr int kSeedCtasPerSm = SMR_SEED_MIN_CTAS;   // resident CTAs per SM the register budget is set for (8: 64 registers)
constexpr int kSeedGrab = 4;      // reads a warp draws from the work counter at a time
constexpr int kLaneHitCap = 128;  // ids per window in the per-warp HBM scratch (x scale on a retry)

// The seed kernel.  grid-stride over reads, one warp per read.
//   lane_hits_g: per-lane id buffers [total warps][cap_g][32]
template <bool INSTR>
__global__ void __launch_bounds__(kSeedWarpsPerCta * 32, kSeedCtasPerSm)
seed_kernel(DevIndex ix, DevBatch b, DevParams prm, uint32_t* lane_hits_g, uint32_t cap_g, uint32_t* next_read) {
  __shared__ CoopSmem s_coop[kSeedWarpsPerCta];
  const unsigned lane = lane_id();
  const uint32_t wic = threadIdx.x >> 5;
  const uint32_t warp = blockIdx.x * kSeedWarpsPerCta + wic;
  const uint32_t L = ix.lnwin, pw = ix.partialwin;
  const bool full = prm.is_full_search != 0;
  CoopSmem& sm = s_coop[wic];
  LaneHits lh;
  lh.sbuf = &sm.ids[0][lane]; lh.buf = lane_hits_g + (size_t)warp * cap_g * 32 + lane; lh.stride = 32; lh.cap = cap_g;   // per-window ids live in a per-warp HBM scratch
  SeedStats st{0, 0};
  uint32_t n_windows = 0, n_short = 0;
  const bool single = (prm.is_forward != 0) != (prm.is_reverse != 0);
  const bool do_fwd = !(single && prm.is_reverse), do_rev = !(single && prm.is_forward);
  // window positions: union of the three pass grids (paralleltraversal.cpp:118-124,262-277).  With the
  // default 18/9/3 every pass position is a multiple of the last shift.
  const uint32_t s0 = ix.skip[0], s1 = ix.skip[1], s2 = ix.skip[2];
  const uint32_t step = (s0 % s2 == 0 && s1 % s2 == 0) ? s2 : 1u;

  // reads are handed out kSeedGrab at a time from a counter: a warp that drew cheap reads (no hit in this database) takes more
  for (uint32_t g0 = 0;;) {
    if (lane == 0) g0 = atomicAdd(next_read, (uint32_t)kSeedGrab);
    g0 = __shfl_sync(kFull, g0, 0);
    if (g0 >= b.nreads) break;
  for (uint32_t r = b.r0 + g0; r < b.r0 + min(g0 + (uint32_t)kSeedGrab, b.nreads); ++r) {
    const uint32_t len = b.seq_off[r + 1] - b.seq_off[r];
    const uint32_t cnt_idx = ix.slot * b.cnt_stride + (r - b.r0);
    if (lane == 0) b.hit_cnt[cnt_idx] = 0;
    if (len < L) { n_short += (lane == 0 && ix.is_last); continue; }           // processor.cpp:109-114 (reset per pass, :228)
    // (reads that become is_done in an earlier part are still searched here: parts are seeded before the
    //  candidate kernel replays them read-major; the candidate kernel skips them, processor.cpp:120-126)
    if (b.flags[r]) continue;                                                   // scratch overflow earlier: the read is redone by the retry
    const bool hasn = b.has_n[r] != 0;
    const uint32_t* pk = b.pk03 + b.pk_off[r];
    const uint32_t* pka = hasn ? b.pk03alt + b.pk_off[r] : pk;
    const uint32_t npos = (len - L) / step + 1;          // positions q*step, q < npos
    const size_t region = hit_base(b, ix.slot, r); const uint32_t region_cap = hit_cap(b, r);
    uint32_t total = 0, flags = 0, cost = 0;
    // the windows of all strand variants form one sequence (variant-major), 32 per round
    const uint32_t nvar = hasn ? 3u : 2u;
    const uint32_t v_lo = do_fwd ? 0u : 1u, v_hi = do_rev ? nvar : 1u;      // variants searched: [v_lo, v_hi)
    const uint32_t nq = (v_hi - v_lo) * npos;
    // the lane's window of round q0: keys + both lookups (paralleltraversal.cpp:161,215), fetched one round ahead
    SeedWin nx = seed_window(ix, pk, pka, len, L, pw, npos, step, s0, s1, s2, v_lo, nq, lane);
    for (uint32_t q0 = 0; q0 < nq; q0 += 32) {
      const SeedWin w = nx;
      if (q0 + 32 < nq) nx = seed_window(ix, pk, pka, len, L, pw, npos, step, s0, s1, s2, v_lo, nq, q0 + 32 + lane);
      lh.n = 0; lh.overflow = false;
      n_windows += w.active ? 1u : 0u;
      bool zero = false;
      // (a) exact first half, <= 1 error in the second half (P = w[9..18) ascending); (b) exact second half, <= 1 error in the reversed first half
      coop_stream<INSTR>(ix, sm, w.lf.x, w.lf.y, rev_chars(w.keyr, pw), w.lr.z, w.lr.w, w.keyf, full, lh, zero, st);
      if (lh.overflow) flags |= kOvfSeedLane;
      const uint32_t n = lh.overflow ? 0u : lh.n;
      const unsigned hm = __ballot_sync(kFull, n != 0);
      if (hm) {
        const uint32_t incl = warp_incl_scan_u32(n), tot = __shfl_sync(kFull, incl, 31);
        if (total + tot > region_cap) { flags |= kOvfSeedRegion; }
        else if (n) {
          const size_t base = region + total + incl - n;
          const uint32_t tag = w.p | (w.var << 24) | (pass_class(w.p, s0, s1, s2) << 28);
          for (uint32_t k = 0; k < n; ++k) {
            const uint32_t id = lh_get(lh, k);
            b.hits[base + k] = make_uint2(id, tag);
            cost += __ldg(ix.pos_off + id + 1) - __ldg(ix.pos_off + id);
          }
        }
        total += tot;
      }
      __syncwarp();
    }
    flags = __reduce_or_sync(kFull, flags);
    cost = warp_sum_u32(min(cost, 1u << 24));
    if (lane == 0) {
      b.hit_cnt[cnt_idx] = (flags & kOvfSeedRegion) ? 0u : total;
      if (flags) atomicOr(&b.flags[r], flags);
      if (total) atomicAdd(&b.cost[r - b.r0], max(cost, 1u));
    }
  }
  }
  // instrumentation + num_short (processor.cpp:113)
  const uint32_t ns = warp_sum_u32(n_short);
  if (lane == 0 && ns) atomicAdd(&b.counters[dcNumShort], (unsigned long long)ns);
  if (INSTR) {
    const uint64_t w = warp_sum_u64(n_windows), ne = warp_sum_u64(st.entries), nl = warp_sum_u64(st.lists);
    if (lane == 0) { atomicAdd(&b.counters[dcWindows], (unsigned long long)w); atomicAdd(&b.counters[dcEntries], (unsigned long long)ne); atomicAdd(&b.counters[dcBuckets], (unsigned long long)nl); }
  }
}

// heaviest-first schedule for the candidate kernel: a few reads carry thousands of Smith-Waterman calls
// (16S/23S conserved regions vote for thousands of references), so reads are binned by log2 of their
// estimated work and the persistent warps drain the bins from the heaviest down.
__global__ void bin_kernel(DevBatch b) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b.nreads) return;
  const uint32_t c = b.cost[i];
  if (c == 0 || b.flags[b.r0 + i]) return;
  const uint32_t bin = min((uint32_t)(kCostBins - 1), 31u - (uint32_t)__clz(c));
  const uint32_t slot = atomicAdd(&b.bin_count[bin], 1u);
  b.bins[(size_t)bin * b.cnt_stride + slot] = b.r0 + i;
}

// A batch run over several resident groups of parts (index budget): kOvfSlots only says that a read stored more alignments than its
// room, and the read goes on searching, as it does through the parts of one group.  The seed kernel and bin_kernel skip every flagged
// read, so between groups the bit is moved to `kept` (restore = 0) and put back before finalize (restore = 1).  Scratch-overflow
// flags stay, and stop the read as they do within a group.
__global__ void group_flags_kernel(uint32_t* flags, uint32_t* kept, uint32_t n, int restore) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (restore) { flags[i] |= kept[i]; continue; }
    const uint32_t f = flags[i];
    if (f & kOvfSlots) { kept[i] = kOvfSlots; flags[i] = f & ~kOvfSlots; }
  }
}

// unit-test kernel: explicit windows through the SAME cooperative path as seed_kernel (mode 0), or by one
// lane scanning its own list sequentially (mode 1) (smr_debug_seed_windows)
__global__ void __launch_bounds__(kSeedWarpsPerCta * 32)
seed_debug_kernel(DevIndex ix, const uint8_t* seq03, const uint32_t* seq_off, const uint32_t* win_read, const uint32_t* win_pos, uint32_t nwin,
                  uint32_t* ids, uint32_t cap, uint32_t* counts, uint8_t* zero, int full_search, int mode) {
  __shared__ CoopSmem s_coop[kSeedWarpsPerCta];
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;   // whole warps stay together: nwin is padded by the launch
  const bool active = k < nwin;
  const uint32_t pw = ix.partialwin;
  uint64_t V = 0;
  if (active) {
    const uint8_t* sq = seq03 + seq_off[win_read[k]] + win_pos[k];
    for (uint32_t i = 0; i < ix.lnwin; ++i) V = (V << 2) | (sq[i] & 3u);
  }
  CoopSmem& sm = s_coop[threadIdx.x >> 5];
  LaneHits lh; lh.sbuf = &sm.ids[0][threadIdx.x & 31]; lh.buf = ids + (size_t)(active ? k : 0) * cap; lh.stride = 1; lh.cap = active ? cap : 0; lh.n = 0; lh.overflow = false;
  SeedStats st{0, 0};
  bool z = false;
  const bool full = full_search != 0;
  const uint32_t keyf = (uint32_t)(V >> (2 * pw)), keyr = (uint32_t)(V & ((1ull << (2 * pw)) - 1));
  const uint32_t Pf = rev_chars(keyr, pw), Pr = keyf;
  if (mode == 0) {
    const uint4 lf = active ? __ldg(&ix.flookup[keyf]) : make_uint4(0, 0, 0, 0);
    const uint4 lr = active ? __ldg(&ix.flookup[keyr]) : make_uint4(0, 0, 0, 0);
    coop_stream<false>(ix, sm, lf.x, lf.y, Pf, lr.z, lr.w, Pr, full, lh, z, st);
  } else if (active) {
    const uint4 lf = __ldg(&ix.flookup[keyf]);
    for (uint32_t i = lf.x; i < lf.x + lf.y && !z; ++i) z = apply_entry(classify_bits(Pf, __ldg(ix.ftext + i), pw), __ldg(ix.fid + i), full, lh);
    if (!z) {
      const uint4 lr = __ldg(&ix.flookup[keyr]);
      for (uint32_t i = lr.z; i < lr.z + lr.w && !z; ++i) z = apply_entry(classify_bits(Pr, __ldg(ix.ftext + i), pw), __ldg(ix.fid + i), full, lh);
    }
  }
  if (active) {
    counts[k] = lh.n; zero[k] = z ? 1 : 0;
    for (uint32_t f = 0; f < lh.n && f < lh.cap && f < kLaneSmemIds; ++f) lh.buf[f] = lh.sbuf[f * 32];   // the ids kept in shared memory
  }
}

}  // namespace smr
