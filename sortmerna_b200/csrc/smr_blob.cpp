// KVDB blob writer (SURVEY 8(f)(4)): the byte string Read::toBinString() stores under the read id
// (src/sortmerna/read.cpp:429-462 -> alignment_struct2::toString, read.cpp:79-101 -> s_align2::toString, include/ssw.hpp:106-140),
// produced for a whole batch straight from the result buffers of smr_align_batch / smr_download_results, so the unchanged
// report stage (Read::load_db, read.cpp:467-539) and -task 1/2 resume read exactly what the CPU path would have stored.
//
// Layout per read with at least one stored alignment (reads without alignments get an empty blob, read.cpp:431-432):
//   u32 lastIndex, lastPart, c_yid_ycov, n_yid_ncov, n_nid_ycov, n_denovo; u8 is_done, is_hit, null_align_output;
//   u16 max_SW_count; i32 num_alignments; u32 hit_seeds; u64 alignment_bytes;
//   alignment = u32 min_index, max_index; u64 n; n x ( u64 bytes; u64 ncigar; u32 cigar[ncigar]; u32 ref_num;
//               i32 ref_begin1, ref_end1, read_begin1, read_end1; u32 readlen; u16 score1, part, index_num; u8 strand )
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "../../include/smr_b200.h"

namespace {

inline uint64_t aln_bytes(uint32_t ncigar) { return 8 + 4ull * ncigar + 4 + 16 + 4 + 6 + 1; }
inline uint64_t blob_bytes(const smr_read_result& r, const smr_aln* a) {
  if (r.n_align == 0) return 0;
  uint64_t b = 24 + 3 + 2 + 4 + 4 + 8 + 8 + 8;
  for (uint32_t k = 0; k < r.n_align; ++k) b += 8 + aln_bytes(a[k].cigar_len);
  return b;
}
template <class T> inline void put(uint8_t*& p, T v) { memcpy(p, &v, sizeof(T)); p += sizeof(T); }

// the blobs of reads 0 .. nreads, read r's alignments at alns + first(r)
template <class First>
int pack_blobs(const smr_read_result* results, const smr_aln* alns, const uint32_t* cigar_pool, uint32_t nreads, First first,
               int32_t num_alignments, const uint32_t* denovo4, uint8_t* out, uint64_t out_cap, uint64_t* blob_off) {
  blob_off[0] = 0;
  for (uint32_t r = 0; r < nreads; ++r) blob_off[r + 1] = blob_off[r] + blob_bytes(results[r], alns + first(r));
  if (!out) return SMR_OK;                       // sizing call
  if (blob_off[nreads] > out_cap) return SMR_ERR_CAPACITY;
  if (blob_off[nreads] && !cigar_pool) return SMR_ERR_ARG;
  auto pack = [&](uint32_t lo, uint32_t hi) {
    for (uint32_t r = lo; r < hi; ++r) {
      const smr_read_result& rr = results[r];
      if (rr.n_align == 0) continue;
      const smr_aln* a = alns + first(r);
      uint8_t* p = out + blob_off[r];
      put<uint32_t>(p, rr.lastIndex); put<uint32_t>(p, rr.lastPart);
      for (int k = 0; k < 4; ++k) put<uint32_t>(p, denovo4 ? denovo4[(size_t)r * 4 + k] : 0u);   // c_yid_ycov, n_yid_ncov, n_nid_ycov, n_denovo
      put<uint8_t>(p, rr.is_done); put<uint8_t>(p, rr.is_hit); put<uint8_t>(p, 0);                 // null_align_output
      put<uint16_t>(p, rr.max_SW_count);
      put<int32_t>(p, num_alignments > 0 ? num_alignments : 0);                                    // Read::init (read.cpp:266)
      put<uint32_t>(p, rr.hit_seeds);
      uint64_t abytes = 4 + 4 + 8;
      for (uint32_t k = 0; k < rr.n_align; ++k) abytes += 8 + aln_bytes(a[k].cigar_len);
      put<uint64_t>(p, abytes);
      put<uint32_t>(p, rr.min_index); put<uint32_t>(p, rr.max_index);
      put<uint64_t>(p, (uint64_t)rr.n_align);
      for (uint32_t k = 0; k < rr.n_align; ++k) {
        const smr_aln& x = a[k];
        put<uint64_t>(p, aln_bytes(x.cigar_len));
        put<uint64_t>(p, (uint64_t)x.cigar_len);
        memcpy(p, cigar_pool + x.cigar_off, 4ull * x.cigar_len); p += 4ull * x.cigar_len;
        put<uint32_t>(p, x.ref_num);
        put<int32_t>(p, x.ref_begin1); put<int32_t>(p, x.ref_end1); put<int32_t>(p, x.read_begin1); put<int32_t>(p, x.read_end1);
        put<uint32_t>(p, x.readlen);
        put<uint16_t>(p, x.score1); put<uint16_t>(p, x.part); put<uint16_t>(p, x.index_num);
        put<uint8_t>(p, x.strand);
      }
    }
  };
  const uint32_t nthr = nreads >= (1u << 16) ? std::min<uint32_t>(8, std::max<uint32_t>(1, std::thread::hardware_concurrency() / 2)) : 1;
  if (nthr <= 1) pack(0, nreads);
  else {
    std::vector<std::thread> pool;
    for (uint32_t t = 0; t < nthr; ++t) pool.emplace_back(pack, (uint32_t)((uint64_t)nreads * t / nthr), (uint32_t)((uint64_t)nreads * (t + 1) / nthr));
    for (auto& th : pool) th.join();
  }
  return SMR_OK;
}

}  // namespace

extern "C" int smr_pack_kvdb_blobs(const smr_read_result* results, const smr_aln* alns, const uint32_t* cigar_pool, uint32_t nreads,
                                   uint32_t slots, int32_t num_alignments, const uint32_t* denovo4, uint8_t* out, uint64_t out_cap,
                                   uint64_t* blob_off) {
  if (!results || !alns || !blob_off || slots == 0) return SMR_ERR_ARG;
  return pack_blobs(results, alns, cigar_pool, nreads, [slots](uint32_t r) { return (size_t)r * slots; }, num_alignments, denovo4, out, out_cap, blob_off);
}

extern "C" int smr_pack_kvdb_blobs_packed(const smr_read_result* results, const smr_aln* alns, const uint32_t* cigar_pool, uint32_t nreads,
                                          int32_t num_alignments, const uint32_t* denovo4, uint8_t* out, uint64_t out_cap, uint64_t* blob_off) {
  if (!results || !blob_off) return SMR_ERR_ARG;
  std::vector<size_t> first((size_t)nreads + 1, 0);
  for (uint32_t r = 0; r < nreads; ++r) first[r + 1] = first[r] + results[r].n_align;
  if (first[nreads] && !alns) return SMR_ERR_ARG;
  static const smr_aln none{};
  return pack_blobs(results, first[nreads] ? alns : &none, cigar_pool, nreads, [&first](uint32_t r) { return first[r]; }, num_alignments, denovo4, out,
                    out_cap, blob_off);
}
