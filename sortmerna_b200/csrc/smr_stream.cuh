// Read stream on the device (smr_stream_begin / push / next / counts): the count pass of smr_stream.h over a piece of text, and
// the record-aligned cut of the pending text into batches.  Both run over the newline index of smr_decode.cuh (count_newlines_kernel,
// write_newlines_kernel and the scan between them); only a few scalars go to the host.
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

// Record ends in the first w bytes of the pending text (which starts at a record start), for a batch of at most `limit` bytes:
// cut[0] = the last record end <= limit (0: none), cut[1] = the first record end (~0: none).  The decode's own records:
//   FASTQ: after the '\n' of every line 4r + 3;   FASTA: at the start of every header line ('>' after a '\n') but the first.
__global__ void stream_cut_kernel(const uint8_t* __restrict__ text, const uint64_t* __restrict__ nl, uint32_t nlines, uint64_t w, uint64_t limit,
                                  uint32_t fmt, unsigned long long* cut) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nlines; i += gridDim.x * blockDim.x) {
    uint64_t e = 0;
    if (fmt == kFmtFastq) {
      if ((i & 3u) == 3u && nl[i] < w) e = nl[i] + 1;
    } else if (i > 0 && nl[i - 1] + 1 < w && text[nl[i - 1] + 1] == '>') e = nl[i - 1] + 1;
    if (!e) continue;
    if (e <= limit) atomicMax(cut, (unsigned long long)e);
    atomicMin(cut + 1, (unsigned long long)e);
  }
}

}  // namespace smr
