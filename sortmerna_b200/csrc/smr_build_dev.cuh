// Index builder on the device: reference sequences (2-bit codes) -> the resident arrays the kernels read (DevIndex: flookup,
// ftext, fid, pos_off, pos), without the on-disk files in between.  Stands in for build_index + Index::load
// (src/sortmerna/indexdb.cpp:1119-2095, src/sortmerna/index.cpp:143-357) (SURVEY 8(f)(3)); the host builder smr_build.cpp writes
// the files, this one makes the same index content where it is used.
//
// The reference inserts every (L+1)-mer window into two pointer tries, one at a time (insert_prefix, indexdb.cpp:147-304).
// What that sequential process leaves behind is a function of the SET of distinct (L+1)-mers and of the order in which they first
// occur, so it can be computed with sorts:
//   * distinct (L+1)-mers and their first window: sort the windows by value (stable) and keep the run heads; the id of an L-mer is
//     its rank among the distinct L-mers (the reference's CMPH numbering is an arbitrary bijection as well, indexdb.cpp:1571-1590);
//   * position lists (add_kmer_to_table, :318-348): windows sorted by (id, window), the first max_pos of every id;
//   * mini burst tries (one per 9-mer and direction): a bucket with prefix P (d characters, d < burst depth) turns into a node when
//     a NEW entry is inserted into it while it already holds 16 -- entries handed down by the burst of its parent do not trigger
//     (:221-299).  With the entries of a list ordered by first occurrence: bucket P bursts at its j-th entry, j = max(17, 1 + entries
//     of P that existed when the parent burst), if it has that many.  One stable sort by (list, prefix of d characters) per level
//     puts every candidate bucket into one contiguous run in order of first occurrence; one thread per run decides.  The final
//     order -- by (list, path of the leaf bucket, first occurrence) -- is the order of the reference's depth-first traversal
//     (traverse_bursttrie.cpp:117-295), i.e. exactly what flatten_index (smr_index.cpp) produces from the files.
// Sorting uses cub::DeviceRadixSort (CUDA toolkit); everything else is the kernels below.
#pragma once
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cuda/functional>
#include "smr_dev.cuh"

namespace smr {

struct BuildGeom {
  uint32_t L, half, pread;      // seed length, L/2, L+1
  uint32_t interval, max_pos;
  uint32_t burst_depth;         // pread - half - 3 (indexdb.cpp:221): buckets below this depth may burst
  uint32_t nseq, nwin;
};
constexpr uint32_t kBurstEntries = 16;   // THRESHOLD / ENTRYSIZE (include/indexdb.hpp:57-60): a bucket bursts at its 17th entry

// sequence of window w: the last s with win_start[s] <= w
__device__ __forceinline__ uint32_t bld_win_seq(const uint32_t* __restrict__ win_start, uint32_t nseq, uint32_t w) {
  uint32_t lo = 0, hi = nseq;
  while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (win_start[mid] <= w) lo = mid; else hi = mid; }
  return lo;
}

// the (L+1)-mer of every window, first character most significant (indexdb.cpp:1437-1475)
__global__ void bld_windows_kernel(const uint8_t* __restrict__ codes, const uint64_t* __restrict__ seq_off, const uint32_t* __restrict__ win_start,
                                   BuildGeom g, uint64_t* key, uint32_t* val) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= g.nwin) return;
  const uint32_t s = bld_win_seq(win_start, g.nseq, w);
  const uint8_t* p = codes + seq_off[s] + (size_t)(w - win_start[s]) * g.interval;
  uint64_t v = 0;
  for (uint32_t i = 0; i < g.pread; ++i) v = (v << 2) | p[i];
  key[w] = v; val[w] = w;
}

// run heads of the sorted windows: distinct (L+1)-mers (entries) and distinct L-mers (ids)
__global__ void bld_heads_kernel(const uint64_t* __restrict__ key, uint32_t n, uint32_t* head_e, uint32_t* head_id) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = key[i], kp = i ? key[i - 1] : ~0ull;
  head_e[i] = (i == 0 || k != kp) ? 1u : 0u;
  head_id[i] = (i == 0 || (k >> 2) != (kp >> 2)) ? 1u : 0u;
}

// Entry arrays (2 per distinct (L+1)-mer: forward list of the first half, mirror list of the last half) + the id of every window.
//   e_list: kmer * 2 + direction;  e_pref: the first burst_depth tail characters, first character most significant;
//   e_text: the half+1 tail characters, first character in the lowest bits (Entry::tail with the trie path, smr_index.h)
__global__ void bld_entries_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ val, const uint32_t* __restrict__ head_e,
                                   const uint32_t* __restrict__ scan_e, const uint32_t* __restrict__ scan_id, BuildGeom g, uint32_t nent,
                                   uint32_t* win_id, uint32_t* e_list, uint32_t* e_pref, uint32_t* e_text, uint32_t* e_id, uint32_t* e_arr) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.nwin) return;
  const uint32_t id = scan_id[i] - 1;
  win_id[val[i]] = id;
  if (!head_e[i]) return;
  const uint32_t u = scan_e[i] - 1;
  const uint64_t v = key[i];
  const uint32_t half = g.half, tl = half + 1;
  // character k of the window: (v >> 2*(pread-1-k)) & 3
  auto ch = [&](uint32_t k) -> uint32_t { return (uint32_t)(v >> (2 * (g.pread - 1 - k))) & 3u; };
  const uint32_t kf = (uint32_t)(v >> (2 * tl)), kr = (uint32_t)(v & ((1ull << (2 * half)) - 1));
  uint32_t tf = 0, tr = 0, pf = 0, pr = 0;
  for (uint32_t k = 0; k < tl; ++k) {
    const uint32_t cf = ch(half + k), cr = ch(half - k);   // forward tail s[half + k], mirror tail s[half - k] (indexdb.cpp:1466-1500)
    tf |= cf << (2 * k); tr |= cr << (2 * k);
    if (k < g.burst_depth) { pf = (pf << 2) | cf; pr = (pr << 2) | cr; }
  }
  e_list[u] = kf * 2; e_pref[u] = pf; e_text[u] = tf; e_id[u] = id; e_arr[u] = val[i];
  e_list[nent + u] = kr * 2 + 1; e_pref[nent + u] = pr; e_text[nent + u] = tr; e_id[nent + u] = id; e_arr[nent + u] = val[i];
}

// positions: windows sorted by (id, window); rank within the id decides what max_pos keeps
__global__ void bld_poskeys_kernel(const uint32_t* __restrict__ win_id, uint32_t n, uint64_t* key) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w < n) key[w] = ((uint64_t)win_id[w] << 32) | w;
}
__global__ void bld_posflag_kernel(const uint64_t* __restrict__ key, uint32_t n, uint32_t* start) {   // index of the run head, for a max-scan
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) start[i] = (i == 0 || (key[i] >> 32) != (key[i - 1] >> 32)) ? i : 0u;
}
__global__ void bld_poskeep_kernel(const uint32_t* __restrict__ start, uint32_t n, uint32_t max_pos, uint32_t* keep) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keep[i] = (max_pos == 0 || i - start[i] < max_pos) ? 1u : 0u;
}
__global__ void bld_poswrite_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ start, const uint32_t* __restrict__ keep,
                                    const uint32_t* __restrict__ kscan /*inclusive*/, const uint32_t* __restrict__ win_start, BuildGeom g, uint32_t nids,
                                    uint32_t* pos_off, uint2* pos) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.nwin) return;
  const uint32_t id = (uint32_t)(key[i] >> 32), w = (uint32_t)key[i];
  const uint32_t at = kscan[i] - keep[i];
  if (start[i] == i || i == 0) pos_off[id] = at;
  if (i == g.nwin - 1) pos_off[nids] = kscan[i];
  if (keep[i]) {
    const uint32_t s = bld_win_seq(win_start, g.nseq, w);
    pos[at] = make_uint2((w - win_start[s]) * g.interval, s);
  }
}

// level keys: list, then the path the entry is known to follow so far (decided: the path of its leaf; undecided: d characters)
// (computed per POSITION of the current order, which is the order of first occurrence within equal keys: the sorts are stable)
__global__ void bld_levelkey_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ e_list, const uint32_t* __restrict__ e_pref,
                                    const uint8_t* __restrict__ e_leaf, uint32_t n, uint32_t d, uint32_t burst_depth, uint64_t* key, uint32_t* val) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t e = perm[i];
  const uint32_t depth = e_leaf[e] ? e_leaf[e] : d;
  const uint32_t drop = 2 * (burst_depth - depth);
  key[i] = ((uint64_t)e_list[e] << (2 * burst_depth)) | ((e_pref[e] >> drop) << drop);
  val[i] = e;
}
__global__ void bld_arrkey_kernel(const uint32_t* __restrict__ e_arr, uint32_t n, uint64_t* key, uint32_t* val) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) { key[e] = e_arr[e]; val[e] = e; }
}

// One thread per run of undecided entries with equal (list, d-character prefix), in order of first occurrence: does this bucket burst?
//   e_tpar: 1 + first-occurrence window of the entry whose insertion burst the parent (0: no parent burst, depth 1)
__global__ void bld_level_kernel(const uint64_t* __restrict__ key, const uint32_t* __restrict__ perm, uint32_t n, uint32_t d,
                                 const uint32_t* __restrict__ e_arr, uint32_t* e_tpar, uint8_t* e_leaf) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t e0 = perm[i];
  if (e_leaf[e0]) return;
  const uint64_t k = key[i];
  if (i && key[i - 1] == k) return;                  // not the head of its run
  const uint32_t tpar = e_tpar[e0];
  uint32_t cnt = 0, m0 = 0;
  for (uint32_t j = i; j < n && key[j] == k; ++j) { ++cnt; if (e_arr[perm[j]] < tpar) ++m0; }
  const uint32_t jb = max(kBurstEntries + 1, m0 + 1);
  if (cnt >= jb) {
    const uint32_t t = e_arr[perm[i + jb - 1]] + 1;
    for (uint32_t j = i; j < i + cnt; ++j) e_tpar[perm[j]] = t;
  } else {
    for (uint32_t j = i; j < i + cnt; ++j) e_leaf[perm[j]] = (uint8_t)d;
  }
}

// the entry texts and ids in final order + the lookup rows
__global__ void bld_flist_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ e_list, const uint32_t* __restrict__ e_text,
                                 const uint32_t* __restrict__ e_id, uint32_t n, uint32_t* ftext, uint32_t* fid, uint32_t* flookup /*4 words per kmer*/, int pass) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t e = perm[i], l = e_list[e];
  if (pass == 0) {
    ftext[i] = e_text[e];
    fid[i] = e_id[e];
    if (i == 0 || e_list[perm[i - 1]] != l) flookup[(size_t)(l >> 1) * 4 + 2 * (l & 1u)] = i;
  } else if (i == n - 1 || e_list[perm[i + 1]] != l) {
    const size_t at = (size_t)(l >> 1) * 4 + 2 * (l & 1u);
    flookup[at + 1] = i + 1 - flookup[at];
  }
}

}  // namespace smr
