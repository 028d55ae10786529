// Input decode on the device (SURVEY 8(f)(2)): raw FASTA / FASTQ text -> the resident read batch the alignment kernels use
// (0-4 codes + offsets), without a host-side record parser.  Stands in for what the reference does per read on the host:
// the record split of Readfeed (src/sortmerna/readfeed.cpp:683-770: 4 lines per FASTQ record; FASTA header '>' + sequence
// lines up to the next header), Read::Read(readstr) (read.cpp:141-176) and the alphabet of Read::init / seqToIntStr via
// nt_table (include/common.hpp:68-77: ACGTU in either case -> 0..3, everything else 4).
//
// All passes are streaming and HBM-bound: (1) newline count per 32-byte chunk, (3) newline positions, (4) per line: header flag +
// sequence bytes, (6) one warp per sequence line encodes its bytes.  The host (text_layout in smr_capi.cu) runs the scans between
// them with cub: (2) over the chunk counts, (5) over the lines, giving the record index of every line and the offset of every
// sequence line in the concatenated read buffer.
#pragma once
#include <cstdint>

#include "smr_dev.cuh"

namespace smr {

// ---- (1) newlines per 32-byte chunk; a text that does not end in '\n' gets a virtual one at position n ----
// A text that does not start on a 16-byte boundary (a piece of a read stream) is read byte by byte.
__global__ void count_newlines_kernel(const uint8_t* __restrict__ text, uint64_t n, uint32_t* __restrict__ counts, uint64_t nchunks) {
  const bool aligned = ((uintptr_t)text & 15u) == 0;
  for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t b0 = c * 32;
    uint32_t k = 0;
    if (b0 + 32 <= n && aligned) {
      const uint4 a = __ldg((const uint4*)(text + b0)), b = __ldg((const uint4*)(text + b0 + 16));
      const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t x = w[i] ^ 0x0A0A0A0Au;                      // zero bytes where '\n'
        const uint32_t t = (x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu;         // exact per-byte zero test (no borrow between bytes)
        k += __popc(~(t | x | 0x7F7F7F7Fu));
      }
    } else {
      for (uint64_t i = b0; i < n && i < b0 + 32; ++i) k += text[i] == '\n';
      if (n > 0 && text[n - 1] != '\n' && b0 + 32 > n && b0 <= n) k += 1;   // the virtual final newline lives in the last chunk
    }
    counts[c] = k;
  }
}
// (3) positions of the newlines, in order
__global__ void write_newlines_kernel(const uint8_t* __restrict__ text, uint64_t n, const uint32_t* __restrict__ first, uint64_t nchunks,
                                      uint64_t* __restrict__ nl_pos) {
  const bool aligned = ((uintptr_t)text & 15u) == 0;
  for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t b0 = c * 32;
    uint32_t k = first[c];
    if (b0 + 32 <= n && aligned) {
      const uint4 a = __ldg((const uint4*)(text + b0)), b = __ldg((const uint4*)(text + b0 + 16));
      const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t x = w[i] ^ 0x0A0A0A0Au;
        uint32_t z = ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x | 0x7F7F7F7Fu);   // 0x80 in every byte that is '\n'
        while (z) { const uint32_t bit = __ffs(z) - 1; z &= z - 1; nl_pos[k++] = b0 + 4 * i + (bit >> 3); }
      }
    } else {
      for (uint64_t i = b0; i < n && i < b0 + 32; ++i) if (text[i] == '\n') nl_pos[k++] = i;
      if (n > 0 && text[n - 1] != '\n' && b0 + 32 > n) nl_pos[k] = n;
    }
  }
}

enum : uint32_t { kFmtFasta = 0, kFmtFastq = 1 };
enum : uint32_t { kDecBadHeader = 1, kDecBadPlus = 2, kDecTruncated = 4 };

// (4) per line: is it a record header; how many sequence bytes does it contribute.  Lines end before '\n' and an optional '\r'.
//     FASTQ: line 4r is the header ('@'), 4r+1 the sequence, 4r+2 starts with '+', 4r+3 the quality string.
//     FASTA: a line starting with '>' is a header, every other line is sequence (blank lines contribute nothing).
//     nlines_eff = lines up to the last non-empty one.
__global__ void line_info_kernel(const uint8_t* __restrict__ text, const uint64_t* __restrict__ nl_pos, uint32_t nlines, uint32_t fmt,
                                 uint32_t* __restrict__ is_hdr, uint32_t* __restrict__ seq_bytes, uint32_t* __restrict__ err) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nlines; i += gridDim.x * blockDim.x) {
    const uint64_t s = i ? nl_pos[i - 1] + 1 : 0;
    uint64_t e = nl_pos[i];
    if (e > s && text[e - 1] == '\r') --e;
    const uint32_t len = (uint32_t)(e - s);
    uint32_t h = 0, sb = 0;
    if (fmt == kFmtFastq) {
      const uint32_t k = i & 3u;
      if (k == 0) { if (len) { h = 1; if (text[s] != '@') atomicOr(err, kDecBadHeader); } }
      else if (k == 1) sb = len;
      else if (k == 2) {   // the separator line of a record that has a header
        const uint64_t s2 = i >= 3 ? nl_pos[i - 3] + 1 : 0, e2 = nl_pos[i - 2];
        if (e2 > s2 && text[s2] != '\r' && (len == 0 || text[s] != '+')) atomicOr(err, kDecBadPlus);
      }
    } else {
      if (len && text[s] == '>') h = 1; else sb = len;
      if (i == 0 && !h) atomicOr(err, kDecBadHeader);
    }
    is_hdr[i] = h; seq_bytes[i] = sb;
  }
}

// (6) one warp per line: headers publish the start of their record; sequence lines are encoded into the read buffer
__global__ void __launch_bounds__(256) scatter_lines_kernel(const uint8_t* __restrict__ text, const uint64_t* __restrict__ nl_pos, uint32_t nlines,
                                                            const uint32_t* __restrict__ is_hdr, const uint32_t* __restrict__ rec_idx,
                                                            const uint32_t* __restrict__ seq_bytes, const uint32_t* __restrict__ seq_pos,
                                                            uint8_t* __restrict__ seq04, uint32_t* __restrict__ seq_off,
                                                            uint64_t* __restrict__ hdr_text_off) {
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const unsigned lane = lane_id();
  for (uint32_t i = warp; i < nlines; i += nwarps) {
    const uint64_t s = i ? nl_pos[i - 1] + 1 : 0;
    if (is_hdr[i]) {
      if (lane == 0) { seq_off[rec_idx[i]] = seq_pos[i]; hdr_text_off[rec_idx[i]] = s; }
      continue;
    }
    const uint32_t nb = seq_bytes[i], o = seq_pos[i];
    for (uint32_t k = lane; k < nb; k += 32) {
      const uint32_t c = text[s + k] & 0xDFu;   // upper case
      seq04[o + k] = c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : (c == 'T' || c == 'U') ? 3 : 4;
    }
  }
}

// per record: packed-word count ((len + 15) / 16 + 2, the layout of pack_reads_kernel) and the longest read
__global__ void record_words_kernel(const uint32_t* __restrict__ seq_off, uint32_t nreads, uint32_t* __restrict__ words, uint32_t* __restrict__ max_len) {
  uint32_t m = 0;
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r <= nreads; r += gridDim.x * blockDim.x) {
    uint32_t w = 0;
    if (r < nreads) { const uint32_t len = seq_off[r + 1] - seq_off[r]; w = (len + 15) / 16 + 2; m = max(m, len); }
    words[r] = w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(kFull, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(max_len, m);
}

// one warp per read: n reads of the 0-4 codes `src`, read k starting at src_off[k], copied to dst at dst_off[k] (dst_off[k + 1] -
// dst_off[k] codes each); gathers the flagged reads of a batch into the batch of their scratch-overflow retry
__global__ void __launch_bounds__(256) gather_reads_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ src_off, uint32_t n,
                                                           const uint32_t* __restrict__ dst_off, uint8_t* __restrict__ dst) {
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t k = warp; k < n; k += nwarps) {
    const uint32_t s = src_off[k], o = dst_off[k], len = dst_off[k + 1] - o;
    for (uint32_t i = lane_id(); i < len; i += 32) dst[o + i] = src[s + i];
  }
}

}  // namespace smr
