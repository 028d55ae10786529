// gzip inflate on the device: the five kernels around smr_inflate.h (FIND / COUNT / WRITE / WINDOW / RESOLVE, described there).
// Replaces the host-side inflate of the reference's read feed (src/sortmerna/readfeed.cpp:683-770 via izlib / rapidgzip) for
// smr_upload_fastx_gz (SURVEY 8(f)(2)).
//
// GPU mapping: Huffman decoding is a serial bit chain, so the parallelism is ACROSS spans: one thread per span, the
// thread's 2.5 KB of decode tables in shared memory (32 decoders per CTA, 82 KB; two CTAs per SM -> 9.4 k spans in flight), the
// 16-bit symbols and the final bytes streamed through HBM.  A 1 GB .gz at 64 KB chunks is 16 k spans: two waves.
#pragma once
#include <cuda_runtime.h>
#include "smr_inflate.h"

namespace smr {

constexpr int kInfSpanThreads = 32;
struct InfTabsPadded { HuffTabs t; uint32_t pad; };   // 641 words: the decoders of a warp fall into different banks for equal table indices
constexpr size_t kInfSpanSmem = sizeof(InfTabsPadded) * kInfSpanThreads;

// FIND: CTA j searches chunk j+1 of the compressed file, blockDim bit offsets per round, and keeps the first that parses.
__global__ void __launch_bounds__(256) inf_find_kernel(const uint32_t* __restrict__ w, uint64_t nbytes, uint64_t chunk_bytes, uint64_t* cand) {
  __shared__ unsigned long long best;
  const uint64_t j = (uint64_t)blockIdx.x + 1, nbits = nbytes * 8;
  const uint64_t p0 = j * chunk_bytes * 8, p1 = min(nbits, (j + 1) * chunk_bytes * 8);
  if (threadIdx.x == 0) best = kInfNone;
  __syncthreads();
  for (uint64_t base = p0; base < p1; base += blockDim.x) {
    const uint64_t p = base + threadIdx.x;
    const int hit = p < p1 && inf_probe_block(w, nbits, p);
    if (hit) atomicMin(&best, (unsigned long long)p);
    if (__syncthreads_or(hit)) break;
  }
  __syncthreads();
  if (threadIdx.x == 0) cand[blockIdx.x] = best;
}

// COUNT / WRITE: thread t decodes span ids[t] (COUNT: ids == nullptr, span t).  Span 0 starts at bit start0 (a gzip header when
// at_member0; else a block of a member of which prior0 bytes came before), span i at cand[i-1].
template <bool WRITE>
__global__ void __launch_bounds__(kInfSpanThreads) inf_span_kernel(const uint32_t* __restrict__ w, uint64_t nbytes, uint64_t start0, bool at_member0, uint64_t prior0,
                                                                    const uint64_t* __restrict__ cand, uint32_t ncand,
                                                                    const uint32_t* __restrict__ ids, const uint64_t* __restrict__ off, const uint64_t* __restrict__ cap,
                                                                    const uint32_t* __restrict__ mem_off, MemberEnd* mem, uint32_t nspans, uint16_t* sym, SpanResult* res) {
  extern __shared__ __align__(16) unsigned char inf_smem[];
  InfTabsPadded* tabs = reinterpret_cast<InfTabsPadded*>(inf_smem);
  const uint32_t t = blockIdx.x * kInfSpanThreads + threadIdx.x;
  if (t >= nspans) return;
  const uint32_t i = WRITE ? ids[t] : t;
  SpanResult r;
  inflate_span<WRITE>(w, nbytes, i ? cand[i - 1] : start0, i == 0 && at_member0, cand, ncand, i, tabs[threadIdx.x].t, WRITE ? sym + off[t] : nullptr, WRITE ? cap[t] : 0ull,
                      WRITE ? mem + mem_off[t] : nullptr, r, i == 0 && !at_member0 ? prior0 : kInfNone);
  res[t] = r;
}

// WINDOW: the 32 KB every real span leaves behind, resolved front to back by ONE CTA (span k needs only window k); window 0 is the
// caller's: zeros at the start of a file, the last 32 KB of the previous round's output when a round resumes.
__global__ void __launch_bounds__(1024) inf_window_kernel(const uint16_t* __restrict__ sym, const uint64_t* __restrict__ off, const uint64_t* __restrict__ cnt,
                                                           uint32_t nreal, uint8_t* win) {
  __shared__ uint8_t prev[kInfWindow];
  for (uint32_t j = threadIdx.x; j < kInfWindow; j += blockDim.x) prev[j] = win[j];
  __syncthreads();
  for (uint32_t k = 0; k < nreal; ++k) {
    const uint16_t* s = sym + off[k];
    const uint64_t n = cnt[k];
    uint8_t v[kInfWindow / 1024];
#pragma unroll
    for (uint32_t i = 0; i < kInfWindow / 1024; ++i) v[i] = inf_window_byte(s, n, prev, threadIdx.x + i * 1024);
    __syncthreads();
    uint8_t* g = win + (size_t)(k + 1) * kInfWindow;
#pragma unroll
    for (uint32_t i = 0; i < kInfWindow / 1024; ++i) { prev[threadIdx.x + i * 1024] = v[i]; g[threadIdx.x + i * 1024] = v[i]; }
    __syncthreads();
  }
}

// RESOLVE: every symbol becomes a byte.  grid = (pieces, real spans).
__global__ void __launch_bounds__(256) inf_resolve_kernel(const uint16_t* __restrict__ sym, const uint64_t* __restrict__ off, const uint64_t* __restrict__ cnt,
                                                           const uint8_t* __restrict__ win, uint8_t* out) {
  const uint32_t k = blockIdx.y;
  const uint64_t o = off[k], n = cnt[k];
  const uint8_t* pw = win + (size_t)k * kInfWindow;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) out[o + j] = inf_resolve(sym[o + j], pw);
}

// CRC: one thread per piece of the inflated text (the host cuts the members into pieces of <= 32 KB and joins the values).
__global__ void __launch_bounds__(128) inf_crc_kernel(const uint8_t* __restrict__ text, const uint64_t* __restrict__ piece_off, const uint32_t* __restrict__ piece_len,
                                                       uint32_t npieces, uint32_t* crc) {
  __shared__ uint32_t tab[256];
  for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) tab[i] = crc_table_entry(i);
  __syncthreads();
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < npieces) crc[t] = crc_piece(text + piece_off[t], piece_len[t], tab);
}

}  // namespace smr
