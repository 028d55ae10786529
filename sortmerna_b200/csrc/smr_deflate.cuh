// gzip deflate on the device: the kernels around smr_deflate.h (MATCH / PARSE / CODE / WRITE / PLACE, described there), for gzip
// members and for the BGZF blocks of BAM, which differ in the header PLACE writes and in how the caller cuts the streams.  The CRC-32
// of every chunk is inf_crc_kernel of smr_inflate.cuh (a chunk is at most one 32 KB piece); the host joins them with crc_concat.
//
// GPU mapping: MATCH is one warp per chunk with the chunk's hash table (16 KB) in shared memory, 32 positions per step; PARSE is
// one thread per chunk (the greedy walk); CODE is one warp per chunk, two lanes building the two Huffman codes; WRITE is one warp
// per chunk, each lane writing a 1/32 share of the symbols; PLACE is one CTA per chunk.
#pragma once
#include <cuda_runtime.h>
#include "smr_deflate.h"
#include "smr_inflate.cuh"

namespace smr {

// MATCH: CTA (one warp) c fills m[b .. e) of chunk c.  A tile is 32 consecutive positions of [h, e); a position looks up its hash
// slot as left by the tiles before, plus the nearest lower lane of the same hash; then the highest lane of every hash pushes the
// group's newest kDefWays positions into the slot.  tests/deflate_check.cpp does the same tile by tile.
__global__ void __launch_bounds__(32) def_match_kernel(const uint8_t* __restrict__ t, const DefChunk* __restrict__ ch, uint32_t* __restrict__ m) {
  __shared__ uint16_t tab[(1u << kDefHashBits) * kDefWays];
  const DefChunk c = ch[blockIdx.x];
  const uint32_t lane = threadIdx.x;
  for (uint32_t i = lane; i < (1u << kDefHashBits) * kDefWays; i += 32) tab[i] = (uint16_t)kDefNoPos;
  __syncwarp();
  for (uint64_t base = c.h; base < c.e; base += kDefTile) {
    const uint64_t p = base + lane;
    const bool ok = p + 4 <= c.e;
    const uint32_t h = ok ? def_hash(t, p) : (1u << kDefHashBits) + lane;   // lanes without a hash form groups of their own
    const uint32_t grp = __match_any_sync(0xFFFFFFFFu, h);
    uint16_t* slot = tab + (h & ((1u << kDefHashBits) - 1)) * kDefWays;
    if (p >= c.b && p < c.e) {
      uint32_t r = 0;
      if (ok) {
        const uint32_t lower = grp & ((1u << lane) - 1);
        r = def_match_at(t, c, p, lower ? base + (31 - __clz(lower)) : kInfNone, slot);
      }
      m[p] = r;
    }
    __syncwarp();
    if (ok && lane == 31u - __clz(grp)) {
      uint16_t v[kDefWays];
      uint32_t k = 0, g = grp;
      while (k < kDefWays && g) { const uint32_t l = 31 - __clz(g); v[k++] = (uint16_t)(base + l - c.h); g &= ~(1u << l); }
      for (uint32_t j = 0; k < kDefWays; ++j) v[k++] = slot[j];
      for (uint32_t j = 0; j < kDefWays; ++j) slot[j] = v[j];
    }
    __syncwarp();
  }
}

// PARSE: thread c walks chunk c (symbols in place of its matches, counts into freq, zeroed)
__global__ void __launch_bounds__(128) def_parse_kernel(const uint8_t* __restrict__ t, const DefChunk* __restrict__ ch, uint32_t nch, uint32_t* m,
                                                         uint32_t* freq, DefInfo* info) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nch) return;
  info[c].nsym = def_parse(m, ch[c].b, ch[c].e, t, freq + (size_t)c * kDefFreqStride);
}

// CODE: warp per chunk (hdr zeroed).  Lanes 0 and 1 build the litlen and the distance code at once; lane 0 then builds the
// code-length code, the header and the chunk's size.  The Huffman builds are serial over <= 286 symbols; the other lanes idle.
__global__ void __launch_bounds__(64) def_code_kernel(const DefChunk* __restrict__ ch, uint32_t nch, const uint32_t* __restrict__ freq, DefCodes* codes,
                                                       uint32_t* hdr, DefInfo* info) {
  const uint32_t c = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31u;
  if (c >= nch) return;
  const uint32_t* f = freq + (size_t)c * kDefFreqStride;
  if (lane < 2) def_code_tree(f, lane, codes[c]);
  __syncwarp();
  if (lane == 0) {
    DefInfo in = info[c];
    def_code_block(f, ch[c].e - ch[c].b, (ch[c].flags & kDefLast) != 0, codes[c], hdr + (size_t)c * kDefHdrWords, in);
    info[c] = in;
  }
}

// WRITE: warp per chunk into its kDefScratch bytes of `out` (zeroed): header words, then lane l's symbols [l*n/32, (l+1)*n/32) at
// the bit offset the warp's scan of the lanes' sizes gives, then the byte-wise tail.
__global__ void __launch_bounds__(128) def_write_kernel(const uint8_t* __restrict__ t, const DefChunk* __restrict__ ch, uint32_t nch, const uint32_t* __restrict__ sym,
                                                         const DefCodes* __restrict__ codes, const uint32_t* __restrict__ hdr, const DefInfo* __restrict__ info,
                                                         uint8_t* out) {
  const uint32_t c = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31u;
  if (c >= nch) return;
  const DefChunk k = ch[c];
  const DefInfo in = info[c];
  const bool fin = (k.flags & kDefLast) != 0;
  uint8_t* o = out + (size_t)c * kDefScratch;
  if (!in.stored) {
    const uint32_t* hw = hdr + (size_t)c * kDefHdrWords;
    for (uint32_t w = lane; w < (in.hdr_bits + 31) / 32; w += 32) bo_or(reinterpret_cast<uint32_t*>(o) + w, hw[w]);
    const DefCodes& C = codes[c];
    const uint32_t lo = (uint32_t)((uint64_t)lane * in.nsym / 32), hi = (uint32_t)((uint64_t)(lane + 1) * in.nsym / 32);
    const uint64_t bits = def_range_bits(sym + k.b, lo, hi, C);
    uint64_t pre = bits;
    for (uint32_t d = 1; d < 32; d <<= 1) { const uint64_t v = __shfl_up_sync(0xFFFFFFFFu, pre, d); if (lane >= d) pre += v; }
    def_write_range(reinterpret_cast<uint32_t*>(o), in.hdr_bits + pre - bits, sym + k.b, lo, hi, C, lane == 31);
  }
  __syncwarp();
  def_write_tail(o, t + k.b, k.e - k.b, in, fin, lane, 32);
}

// PLACE: CTA c copies chunk c to out + dst[c]; the stream's first chunk writes the member's header (hlen bytes at hdr[stream *
// hlen], gzip or BGZF) before it, its last the trailer (trl[2 * stream], trl[2 * stream + 1] = CRC-32, ISIZE) after it.
__global__ void __launch_bounds__(256) def_place_kernel(const DefChunk* __restrict__ ch, const DefInfo* __restrict__ info, const uint8_t* __restrict__ scratch,
                                                         const uint64_t* __restrict__ dst, const uint32_t* __restrict__ trl, const uint8_t* __restrict__ hdr,
                                                         uint32_t hlen, uint8_t* out) {
  const uint32_t c = blockIdx.x;
  const uint64_t d = dst[c];
  const uint32_t n = info[c].bytes;
  const uint8_t* s = scratch + (size_t)c * kDefScratch;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) out[d + i] = s[i];
  const DefChunk k = ch[c];
  if ((k.flags & kDefFirst) && threadIdx.x < hlen) out[d - hlen + threadIdx.x] = hdr[(size_t)k.stream * hlen + threadIdx.x];
  if ((k.flags & kDefLast) && threadIdx.x < 8) out[d + n + threadIdx.x] = (uint8_t)(trl[2 * k.stream + threadIdx.x / 4] >> (8 * (threadIdx.x & 3)));
}

}  // namespace smr
