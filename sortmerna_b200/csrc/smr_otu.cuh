// OTU map on the device: the reference's otu_map.txt (fill_otu_map / fill_otu_map2 / OtuMap::write, src/sortmerna/otumap.cpp:84-281)
// accumulated over the batches of one read file.
//   add     one thread per (read, slot) applies the OTU rule to every stored alignment; the passing ones are compacted in (read, slot)
//           order and appended to the accumulator: a sort key (rank of the reference id, (index, part) group), the group and ref_num of
//           the alignment, and a copy of the read's QNAME in a name pool (one warp per entry).
//   finish  one stable radix sort of all entries on the key, then a size pass, a scan and a write pass: one line per reference id, its
//           reads in (batch, read, slot) order within each group and group 0's before group 1's -- the order of the std::map the
//           reference fills at -threads 1, walking (index, part) groups in load order and reads in file order.
// The rank of a reference id is its position among all distinct ids of the loaded groups in unsigned byte order (std::map<std::string>);
// equal ids share a rank, so an id that occurs in two groups is one line.
// Paired reads (OtuArgs::feed): one interleaved file gives every record to the map, two mate files only records 2k (the first file's).
// De novo statistics: denovo_stats_kernel, the reference's denovo_stats pass (processor.cpp:287-438) at -threads 1; its per-read
// counters are the gate of the OTU map and the denovo4 of the KVDB blobs, its sums the figures of aligned.log.
#pragma once
#include <cstdint>

#include "smr_report.cuh"

namespace smr {

struct OtuEnt {
  uint64_t name_off;   // into the name pool
  uint32_t name_len, grp, ref_num, pad;
};

struct OtuArgs {
  const uint32_t* rank;       // rank of (group g, ref_num k) at rank[rank_off[g] + k]
  const uint32_t* rank_off;   // [ngroups]
  uint32_t gbits;             // key = rank << gbits | group
  double min_id, min_cov;
  uint32_t feed;              // SMR_OTU_ONE_FILE / SMR_OTU_TWO_FILES: records 2k and 2k+1 are mates; 0 single-end
};

// denovo_stats_run (processor.cpp:329-345): the read's c_yid_ycov > 0 -- one of its alignments passes both thresholds with
// floor(x * 1000 + 0.5) / 1000.0 (fill_otu_map2 looks at a read only then, otumap.cpp:160).  A pair whose second mate is empty was
// skipped by denovo_stats_run (processor.cpp:323-327), so neither mate counts.
__device__ bool otu_read_counts(const RptArgs& a, const OtuArgs& o, uint32_t r) {
  if (o.feed && a.rec[r | 1u].seq_len == 0) return false;
  const uint32_t n = a.res[r].n_align;
  for (uint32_t k = 0; k < n; ++k)
    if (denovo_class(a.aln[rpt_slot(a, r, k)], a.st[rpt_slot(a, r, k)], o.min_id, o.min_cov) == kDnYidYcov) return true;
  return false;
}

// fill_otu_map2 (otumap.cpp:157-163): the same rounding, but scaled back with * 0.001, which is one ulp above / 1000.0 for 144 of the
// k in 0..1000 and never below -- written out separately, no FMA, operands in the reference's order
__device__ __forceinline__ bool otu_passes(const smr_aln& al, const smr_aln_stats& st, const OtuArgs& o) {
  const double id = (double)st.n_match_denovo / (double)(st.n_miss + st.n_gap + st.n_match);
  const int32_t span = al.read_end1 - al.read_begin1 + 1;
  const double cov = (double)(span < 0 ? -span : span) / (double)al.readlen;
  const double idr = __dmul_rn(floor(__dadd_rn(__dmul_rn(id, 1000.0), 0.5)), 0.001);
  const double covr = __dmul_rn(floor(__dadd_rn(__dmul_rn(cov, 1000.0), 0.5)), 0.001);
  return idr >= o.min_id && covr >= o.min_cov;
}

// per (read, slot): flag = 1 for an entry of the map; nsz = length of its QNAME (0 otherwise)
__global__ void otu_flag_kernel(RptArgs a, OtuArgs o, uint32_t* __restrict__ flag, uint64_t* __restrict__ nsz) {
  const uint64_t n = a.nslots;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = rpt_read_of(a, i), k = (uint32_t)(i - rpt_slot(a, r, 0));
    bool pass = false;
    if (k < a.res[r].n_align) {
      const smr_aln& al = a.aln[i];
      const uint32_t g = rpt_group_of(a, al);
      if (g == a.ngroups) atomicOr(a.err, kRptErrGroup);
      else if (al.ref_num >= a.grp[g].nref) atomicOr(a.err, kRptErrRef);
      if (al.readlen != a.rec[r].seq_len || al.read_end1 >= (int32_t)a.rec[r].seq_len) atomicOr(a.err, kRptErrLen);
      // two mate files: the OTU pass reads the first file alone (readfeed slot 0 at -threads 1, otumap.cpp:144)
      pass = !(o.feed == SMR_OTU_TWO_FILES && (r & 1u)) && otu_passes(al, a.st[i], o) && otu_read_counts(a, o, r);
    }
    flag[i] = pass;
    nsz[i] = pass ? a.rec[r].name_len : 0;
  }
}

// passing (read, slot)s -> entries base + pos[i]: key, group, ref_num, QNAME copied by a warp into the pool at pool_base + noff[i]
__global__ void __launch_bounds__(256) otu_append_kernel(RptArgs a, OtuArgs o, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos,
                                                         const uint64_t* __restrict__ noff, uint64_t base, uint64_t pool_base, uint64_t* __restrict__ key,
                                                         OtuEnt* __restrict__ ent, char* __restrict__ pool) {
  const uint64_t n = a.nslots;
  const unsigned lane = lane_id();
  for (uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
    if (!flag[i]) continue;
    const uint32_t r = rpt_read_of(a, i);
    const RptRec& rc = a.rec[r];
    const uint64_t dst = pool_base + noff[i];
    for (uint32_t k = lane; k < rc.name_len; k += 32) pool[dst + k] = (char)a.text[rc.hdr + rc.name_beg + k];
    if (lane == 0) {
      const smr_aln& al = a.aln[i];
      const uint32_t g = rpt_group_of(a, al);
      const uint64_t e = base + pos[i];
      key[e] = (uint64_t)o.rank[o.rank_off[g] + al.ref_num] << o.gbits | g;
      ent[e] = OtuEnt{dst, rc.name_len, g, al.ref_num, 0};
    }
  }
}

// ---- finish: skey / sidx = the entries sorted on their key ----
__global__ void otu_iota_kernel(uint32_t* __restrict__ v, uint64_t m) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (uint64_t)gridDim.x * blockDim.x) v[j] = (uint32_t)j;
}

__device__ __forceinline__ bool otu_head(const uint64_t* skey, uint32_t gbits, uint64_t j) { return j == 0 || (skey[j] >> gbits) != (skey[j - 1] >> gbits); }

__global__ void otu_size_kernel(const uint64_t* __restrict__ skey, const uint32_t* __restrict__ sidx, const OtuEnt* __restrict__ ent, uint64_t m,
                                uint32_t gbits, const RptGroup* __restrict__ grp, uint64_t* __restrict__ size, uint32_t* __restrict__ runs) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (uint64_t)gridDim.x * blockDim.x) {
    const OtuEnt e = ent[sidx[j]];
    uint64_t s = e.name_len + 1;   // QNAME + '\t' or '\n'
    if (otu_head(skey, gbits, j)) {
      const RptGroup& G = grp[e.grp];
      s += G.name_off[e.ref_num + 1] - G.name_off[e.ref_num] + 1;   // ref_id + '\t'
      atomicAdd(runs, 1u);
    }
    size[j] = s;
  }
}

__global__ void __launch_bounds__(256) otu_write_kernel(const uint64_t* __restrict__ skey, const uint32_t* __restrict__ sidx, const OtuEnt* __restrict__ ent,
                                                        uint64_t m, uint32_t gbits, const RptGroup* __restrict__ grp, const char* __restrict__ pool,
                                                        const uint64_t* __restrict__ off, char* __restrict__ out) {
  const unsigned lane = lane_id();
  for (uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < m; j += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
    const OtuEnt e = ent[sidx[j]];
    char* dst = out + off[j];
    if (otu_head(skey, gbits, j)) {
      const RptGroup& G = grp[e.grp];
      const uint64_t b = G.name_off[e.ref_num], len = G.name_off[e.ref_num + 1] - b;
      for (uint64_t k = lane; k < len; k += 32) dst[k] = G.names[b + k];
      if (lane == 0) dst[len] = '\t';
      dst += len + 1;
    }
    for (uint32_t k = lane; k < e.name_len; k += 32) dst[k] = pool[e.name_off + k];
    if (lane == 0) dst[e.name_len] = j + 1 == m || otu_head(skey, gbits, j + 1) ? '\n' : '\t';
  }
}

// ---- denovo_stats (smr_denovo_stats): the four counters of every read and their column sums ----
// One thread per (read, slot); a warp takes 32 consecutive (read, slot)s, so the slots of one read mostly share a warp: lanes with the
// same (read, class) add to per_read once, through their leader (__match_any_sync).  Totals are summed per thread, then per block
// in shared memory, then one 64-bit atomic per counter per block: integers, so the sums do not depend on the grid.
__global__ void __launch_bounds__(256) denovo_stats_kernel(RptArgs a, double min_id, double min_cov, uint32_t paired, uint32_t* __restrict__ per_read,
                                                           unsigned long long* __restrict__ totals) {
  __shared__ unsigned long long s_tot[4];
  if (threadIdx.x < 4) s_tot[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t n = a.nslots;
  const unsigned lane = lane_id();
  uint32_t t[4] = {0, 0, 0, 0};
  // warp-uniform loop: every lane takes part in the match of every round
  for (uint64_t base = (((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~31ull); base < n; base += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = base + lane;
    uint64_t key = ~0ull;
    if (i < n) {
      const uint32_t r = rpt_read_of(a, i), k = (uint32_t)(i - rpt_slot(a, r, 0));
      if (k < a.res[r].n_align) {
        const smr_aln& al = a.aln[i];
        if (rpt_group_of(a, al) == a.ngroups) atomicOr(a.err, kRptErrGroup);
        if (al.readlen != a.rec[r].seq_len || al.read_end1 >= (int32_t)a.rec[r].seq_len) atomicOr(a.err, kRptErrLen);
        // a pair whose second mate is empty is skipped (processor.cpp:323-327); so is a last record without its mate, as the
        // reference skips the last record of an odd interleaved file
        else if (!(paired && ((r | 1u) >= a.nreads || a.rec[r | 1u].seq_len == 0))) {
          const uint32_t c = denovo_class(al, a.st[i], min_id, min_cov);
#pragma unroll
          for (uint32_t j = 0; j < 4; ++j) t[j] += c == j;   // no dynamic index: t stays in registers
          key = (uint64_t)r * 4 + c;
        }
      }
    }
    const unsigned same = __match_any_sync(0xffffffffu, key);
    if (key != ~0ull && lane == (unsigned)(__ffs(same) - 1)) atomicAdd(per_read + key, (uint32_t)__popc(same));
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    uint32_t v = t[c];
    for (int d = 16; d; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
    if (lane == 0 && v) atomicAdd(&s_tot[c], (unsigned long long)v);
  }
  __syncthreads();
  if (threadIdx.x < 4 && s_tot[threadIdx.x]) atomicAdd(totals + threadIdx.x, s_tot[threadIdx.x]);
}

}  // namespace smr
