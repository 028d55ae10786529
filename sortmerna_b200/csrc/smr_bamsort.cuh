// Coordinate-sorted aligned.bam and its BAI index on the device (smr_bam_sort_*; DESIGN 5i).
//   add     the BAM writer's records of one batch (smr_report.cuh) get samtools' coordinate key (bsort_key_kernel); a stable radix
//           sort of the batch on it gives the batch's sorted run, gathered one warp per record (bsort_gather_kernel) and handed to
//           the caller uncompressed; the keys and sizes of the run are appended to the accumulator (12 B per record).
//   plan    one stable radix sort of (key, record ordinal) over every run, so equal keys keep run order, then the order inside a run
//           (which kept the writer's row order); the host cuts the sorted records into windows of whole records.
//   window  the caller stages the window's byte range of each run; the records are gathered into sorted order, cut into BGZF
//           blocks and compressed (gzip_streams), and one thread per record (bsort_index_kernel) computes its virtual offsets, the
//           linear index minima (atomicMin per reference and 16 kb window) and the heads of its runs of equal (refID, bin), which
//           bsort_pieces_kernel turns into the window's chunk pieces.
//   index   the host merges the pieces per (reference, bin) by htslib's rule (fmt::bam_chunks_merge) and writes the BAI bytes.
#pragma once
#include <cstdint>

#include "smr_fmt.h"

namespace smr {

// a maximal run of consecutive records (in file order) of one (refID, bin): [vbeg of its first, vend of its last)
struct BamPiece {
  uint64_t refbin;        // refID << 32 | bin
  uint64_t vbeg, vend;
  uint32_t first, last;   // its records, as indexes into the window
};

__device__ __forceinline__ uint32_t bsort_u32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
__device__ __forceinline__ uint32_t bsort_u16(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8; }

// record j of the batch at rec + off[j]: its key, its size, and j as the sort's value
__global__ void bsort_key_kernel(const uint8_t* __restrict__ rec, const uint64_t* __restrict__ off, uint64_t n, uint64_t* __restrict__ key,
                                 uint32_t* __restrict__ ord) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* p = rec + off[j];
    key[j] = fmt::bam_sort_key((int32_t)bsort_u32(p + 4), (int32_t)bsort_u32(p + 8), bsort_u16(p + 18));
    ord[j] = (uint32_t)j;
  }
}

// the batch in sorted order: record t is record perm[t] of the writer, at off[perm[t]]; its size (for the scan of the run's offsets),
// its source offset, and its key and size appended to the accumulator at acc_at + t
__global__ void bsort_run_order_kernel(const uint32_t* __restrict__ perm, const uint64_t* __restrict__ skey, const uint64_t* __restrict__ off,
                                       uint64_t n, uint64_t* __restrict__ ssz, uint64_t* __restrict__ soff, uint64_t* __restrict__ acc_key,
                                       uint32_t* __restrict__ acc_size, uint64_t acc_at) {
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t j = perm[t];
    const uint64_t s = off[j + 1] - off[j];
    ssz[t] = s; soff[t] = off[j];
    acc_key[acc_at + t] = skey[t];
    acc_size[acc_at + t] = (uint32_t)s;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) ssz[n] = 0;
}

// plan: psz[t] = the size of the t-th record in sorted order (perm), csz[o] = the size of record o in accumulator order; both with a
// zero at n for the exclusive scans
__global__ void bsort_plan_sizes_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ size, uint64_t n, uint64_t* __restrict__ psz,
                                        uint64_t* __restrict__ csz) {
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (uint64_t)gridDim.x * blockDim.x) {
    psz[t] = size[perm[t]];
    csz[t] = size[t];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { psz[n] = 0; csz[n] = 0; }
}

// window: the staged offset of the window's i-th record (sorted record t0 + i): its byte offset in the run file's concatenation
// (coff) moved by the staging of its run (adj[r]; run r holds the accumulator's records [run_rec[r], run_rec[r + 1]))
__global__ void bsort_window_src_kernel(const uint32_t* __restrict__ perm, const uint64_t* __restrict__ coff, const uint64_t* __restrict__ run_rec,
                                        uint32_t nruns, const int64_t* __restrict__ adj, uint64_t t0, uint64_t n, uint64_t* __restrict__ soff) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t o = perm[t0 + i];
    uint32_t lo = 0, hi = nruns;   // the last run whose first record is <= o
    while (hi - lo > 1) { const uint32_t m = (lo + hi) / 2; if (run_rec[m] <= o) lo = m; else hi = m; }
    soff[i] = (uint64_t)((int64_t)coff[o] + adj[lo]);
  }
}

// one warp per record: record i (src + soff[i]) to dst + doff[i] - doff[0], its size doff[i + 1] - doff[i].  check: the source must
// lie in [0, src_bytes) and hold block_size = size - 4, or *err is set and the record is not copied.
__global__ void __launch_bounds__(256) bsort_gather_kernel(const uint8_t* __restrict__ src, uint64_t src_bytes, const uint64_t* __restrict__ soff,
                                                           const uint64_t* __restrict__ doff, uint64_t n, uint8_t* __restrict__ dst,
                                                           bool check, uint32_t* err) {
  const unsigned lane = threadIdx.x & 31;
  for (uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
    const uint64_t s = soff[i], d = doff[i] - doff[0], len = doff[i + 1] - doff[i];
    if (check) {
      const bool ok = len >= 4 && s + len <= src_bytes && bsort_u32(src + s) == len - 4;
      if (!ok) { if (lane == 0) atomicOr(err, 1u); continue; }
    }
    for (uint64_t k = lane; k < len; k += 32) dst[d + k] = src[s + k];
  }
}

// one thread per record of a compressed window (win, its records at doff[i] - doff[0]; the window's BGZF blocks of kBlock input
// bytes start at coffset + bso[k], bso[nblocks] = the next block): vbeg / vend, the key of (refID, bin) and whether the record opens a
// piece (head); the linear index minima lin[lin_off[refID] + w] for every 16 kb window w the record overlaps.
template <uint32_t kBlock>
__global__ void bsort_index_kernel(const uint8_t* __restrict__ win, const uint64_t* __restrict__ doff, uint64_t n, const uint64_t* __restrict__ bso,
                                   uint32_t nblocks, uint64_t coffset, const uint64_t* __restrict__ lin_off, unsigned long long* __restrict__ lin,
                                   uint64_t* __restrict__ vb, uint64_t* __restrict__ ve, uint64_t* __restrict__ rb, uint32_t* __restrict__ head) {
  const uint64_t wbytes = doff[n] - doff[0];
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t d = doff[i] - doff[0], e = doff[i + 1] - doff[0];
    const uint8_t* p = win + d;
    const uint32_t ref = bsort_u32(p + 4), pos = bsort_u32(p + 8), bin = bsort_u16(p + 14), ncig = bsort_u16(p + 16);
    const uint8_t* cig = p + 36 + p[12];
    uint64_t span = 0;   // reference bases: M, D, N, =, X
    for (uint32_t c = 0; c < ncig; ++c) {
      const uint32_t w = bsort_u32(cig + 4 * c), op = w & 15;
      if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) span += w >> 4;
    }
    const uint64_t end = pos + (span ? span : 1);
    const uint64_t kb = d / kBlock;
    const uint64_t vbeg = fmt::bam_voffset(coffset + bso[kb], (uint32_t)(d - kb * kBlock));
    uint64_t vend;
    if (e == wbytes) vend = fmt::bam_voffset(coffset + bso[nblocks], 0);
    else { const uint64_t ke = e / kBlock; vend = fmt::bam_voffset(coffset + bso[ke], (uint32_t)(e - ke * kBlock)); }
    vb[i] = vbeg; ve[i] = vend;
    const uint64_t key = (uint64_t)ref << 32 | bin;
    rb[i] = key;
    uint32_t h = 1;
    if (i) { const uint8_t* q = win + (doff[i - 1] - doff[0]); h = ((uint64_t)bsort_u32(q + 4) << 32 | bsort_u16(q + 14)) != key; }
    head[i] = h;
    const uint64_t l0 = lin_off[ref], l1 = lin_off[ref + 1];
    for (uint64_t w = pos >> 14; w <= (end - 1) >> 14 && l0 + w < l1; ++w) atomicMin(lin + l0 + w, (unsigned long long)vbeg);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) head[n] = 0;
}

// the window's pieces: pid = the exclusive scan of head, so record i is in piece pid[i] + head[i] - 1; a head opens its piece, the
// record before the next head closes it
__global__ void bsort_pieces_kernel(const uint64_t* __restrict__ vb, const uint64_t* __restrict__ ve, const uint64_t* __restrict__ rb,
                                    const uint32_t* __restrict__ head, const uint32_t* __restrict__ pid, uint64_t n, BamPiece* __restrict__ pc) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    BamPiece& p = pc[pid[i] + head[i] - 1];
    if (head[i]) { p.refbin = rb[i]; p.vbeg = vb[i]; p.first = (uint32_t)i; }
    if (i + 1 == n || head[i + 1]) { p.vend = ve[i]; p.last = (uint32_t)i; }
  }
}

__global__ void bsort_iota_kernel(uint32_t* __restrict__ v, uint64_t n) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) v[i] = (uint32_t)i;
}

}  // namespace smr
