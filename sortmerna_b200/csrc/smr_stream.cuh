// Read stream on the device (smr_stream_begin / push / next / counts): the count pass of smr_stream.h over a piece of text, the
// record-aligned cut of the pending text into batches, and a mate stream's pair cut and interleave of its two texts.  All run over
// the newline index of smr_decode.cuh (count_newlines_kernel, write_newlines_kernel and the scan between them); only a few scalars
// go to the host.
#pragma once
#include <cstdint>
#include <cub/block/block_scan.cuh>

#include "smr_decode.cuh"
#include "smr_stream.h"

namespace smr {

struct RcJoin { __device__ ReadCounts operator()(const ReadCounts& a, const ReadCounts& b) const { return rc_join(a, b); } };

// count pass, step 1: CTA b takes lines [b * per, (b + 1) * per) in file order, 256 at a time, and leaves their ReadCounts in part[b]
__global__ void __launch_bounds__(256) count_lines_kernel(const uint64_t* __restrict__ nl, uint32_t nlines, uint64_t n, CountState s, uint32_t per,
                                                          ReadCounts* __restrict__ part) {
  using Scan = cub::BlockScan<ReadCounts, 256>;
  __shared__ typename Scan::TempStorage tmp;
  const uint64_t l0 = (uint64_t)blockIdx.x * per, l1 = l0 + per < nlines ? l0 + per : (uint64_t)nlines;
  ReadCounts acc = rc_none();
  for (uint64_t base = l0; base < l1; base += 256) {
    const uint64_t i = base + threadIdx.x;
    ReadCounts x = rc_none(), y, agg;
    if (i < l1) rc_line(nl, i, n, s, x);
    Scan(tmp).InclusiveScan(x, y, RcJoin(), agg);
    __syncthreads();
    acc = rc_join(acc, agg);
  }
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

// count pass, step 2: the CTA results joined in order; out = {ReadCounts, real newlines, position of the last one}
__global__ void count_fold_kernel(const ReadCounts* __restrict__ part, uint32_t nparts, const uint64_t* __restrict__ nl, uint32_t nlines, uint64_t n,
                                  ReadCounts* out, uint64_t* nl_info) {
  ReadCounts acc = rc_none();
  for (uint32_t k = 0; k < nparts; ++k) acc = rc_join(acc, part[k]);
  *out = acc;
  const uint64_t nreal = nlines - (nlines && nl[nlines - 1] >= n ? 1 : 0);   // the last entry may be the virtual newline at n
  nl_info[0] = nreal; nl_info[1] = nreal ? nl[nreal - 1] : 0;
}

// The end of a record at line i of a pending text (which starts at a record start), for a window of its first w bytes; 0: none.
// The decode's own records:  FASTQ: after the '\n' of every line 4r + 3;   FASTA: at the start of every header line ('>' after a
// '\n') but the first.
__device__ __forceinline__ uint64_t stream_record_end(const uint8_t* text, const uint64_t* nl, uint32_t i, uint64_t w, uint32_t fmt) {
  if (fmt == kFmtFastq) return (i & 3u) == 3u && nl[i] < w ? nl[i] + 1 : 0;
  return i > 0 && nl[i - 1] + 1 < w && text[nl[i - 1] + 1] == '>' ? nl[i - 1] + 1 : 0;
}

// Record ends in the first w bytes of the pending text, for a batch of at most `limit` bytes:
// cut[0] = the last record end <= limit (0: none), cut[1] = the first record end (~0: none).
__global__ void stream_cut_kernel(const uint8_t* __restrict__ text, const uint64_t* __restrict__ nl, uint32_t nlines, uint64_t w, uint64_t limit,
                                  uint32_t fmt, unsigned long long* cut) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nlines; i += gridDim.x * blockDim.x) {
    const uint64_t e = stream_record_end(text, nl, i, w, fmt);
    if (!e) continue;
    if (e <= limit) atomicMax(cut, (unsigned long long)e);
    atomicMin(cut + 1, (unsigned long long)e);
  }
}

// ---- mate stream: the record ends of each mate's pending text, the number of pairs that fit, the interleave ----
// line i ends a record: flag[i] = 1 (an exclusive scan of the flags numbers the records)
__global__ void record_end_flags_kernel(const uint8_t* __restrict__ text, const uint64_t* __restrict__ nl, uint32_t nlines, uint64_t w, uint32_t fmt,
                                        uint32_t* __restrict__ flag) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nlines; i += gridDim.x * blockDim.x)
    flag[i] = stream_record_end(text, nl, i, w, fmt) != 0;
}

// ends[k] = the end of record k (pos: the exclusive scan of record_end_flags_kernel's flags)
__global__ void record_end_list_kernel(const uint8_t* __restrict__ text, const uint64_t* __restrict__ nl, uint32_t nlines, uint64_t w, uint32_t fmt,
                                       const uint32_t* __restrict__ pos, uint64_t* __restrict__ ends) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nlines; i += gridDim.x * blockDim.x) {
    const uint64_t e = stream_record_end(text, nl, i, w, fmt);
    if (e) ends[pos[i]] = e;
  }
}

// *k = the largest number of pairs whose interleaved text fits in limit bytes: pair i ends at ea[i] + eb[i] (both increase with i)
__global__ void mate_fit_kernel(const uint64_t* __restrict__ ea, const uint64_t* __restrict__ eb, uint32_t m, uint64_t limit, unsigned long long* k) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x)
    if (ea[i] + eb[i] <= limit) atomicMax(k, (unsigned long long)i + 1);
}

// bytes [b, e) of a mate's text t of n bytes to dst by the lanes of a warp; e == n + 1 is a last line without '\n', which gets one
// (Readfeed::split).  16-byte copies when source and destination share their alignment.
__device__ __forceinline__ void mate_record_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ t, uint64_t b, uint64_t e, uint64_t n, unsigned lane) {
  const uint8_t* src = t + b;
  const uint64_t len = (e < n ? e : n) - b;
  uint64_t head = len, nv = 0;
  if (((reinterpret_cast<uintptr_t>(dst) ^ reinterpret_cast<uintptr_t>(src)) & 15u) == 0) {
    head = (16u - (reinterpret_cast<uintptr_t>(dst) & 15u)) & 15u;
    if (head > len) head = len;
    nv = (len - head) / 16;
  }
  for (uint64_t k = lane; k < head; k += 32) dst[k] = src[k];
  const uint4* s4 = reinterpret_cast<const uint4*>(src + head);
  uint4* d4 = reinterpret_cast<uint4*>(dst + head);
  for (uint64_t k = lane; k < nv; k += 32) d4[k] = s4[k];
  for (uint64_t k = head + nv * 16 + lane; k < len; k += 32) dst[k] = src[k];
  if (e > n && lane == 0) dst[len] = '\n';
}

// pair p = record p of mate 1, then record p of mate 2, at ea[p - 1] + eb[p - 1]: one warp per pair
__global__ void __launch_bounds__(256) mate_interleave_kernel(const uint8_t* __restrict__ ta, uint64_t na, const uint64_t* __restrict__ ea,
                                                              const uint8_t* __restrict__ tb, uint64_t nb, const uint64_t* __restrict__ eb,
                                                              uint32_t k, uint8_t* __restrict__ out) {
  const unsigned lane = threadIdx.x & 31u;
  for (uint32_t p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < k; p += (gridDim.x * blockDim.x) >> 5) {
    const uint64_t a0 = p ? ea[p - 1] : 0, a1 = ea[p], b0 = p ? eb[p - 1] : 0;
    uint8_t* dst = out + a0 + b0;
    mate_record_copy(dst, ta, a0, a1, na, lane);
    mate_record_copy(dst + (a1 - a0), tb, b0, eb[p], nb, lane);
  }
}

}  // namespace smr
