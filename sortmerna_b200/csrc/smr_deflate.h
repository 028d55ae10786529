// gzip / DEFLATE encoding (RFC 1952 / RFC 1951) as plain functions shared by the CUDA kernels (smr_deflate.cuh) and by the
// host-side check tests/deflate_check.cpp, which runs the same steps serially and so gives the device's exact bytes.
//
// The counterpart of smr_inflate.h for the report writer's -zip-out output (the reference compresses every report file through
// zlib's gzip wrapper at Z_DEFAULT_COMPRESSION, izlib.cpp:79-93).  The bytes are not zlib's -- its match finder is a serial
// hash-chain walk -- but every file is valid RFC 1952 and decompresses to the reference's content.
//
// How one stream becomes parallel work.  The stream is cut into chunks of kDefChunk bytes; everything below is per chunk:
//   1. MATCH  per position, the longest match among a few earlier occurrences of its 4-byte hash.  A chunk may match into the
//             32 KB before it in the same stream (the whole input is resident, so history is no serial dependency) but never
//             before the stream's start, and no match runs past the chunk's end.  Candidates come from a table of the last
//             kDefWays positions per hash, updated after every tile of 32 positions, plus the nearest same-hash position in the
//             tile itself (def_match_at).
//   2. PARSE  one thread walks the chunk's match array greedily with a one-step lazy check, writes the symbols and counts them.
//   3. CODE   litlen / distance code lengths (limited to 15 bits), the code-length code (7 bits), the dynamic block header, and
//             the chunk's byte size, or the stored form when that is smaller.
//   4. WRITE  the block: lanes write disjoint symbol ranges at bit offsets from a scan of their sizes.  A non-final chunk ends
//             with an empty stored block (Z_SYNC_FLUSH), so it ends on a byte boundary; the stream's last chunk sets BFINAL.
//   5. PLACE  a scan of the chunk byte sizes places the chunks after the gzip header; the trailer's CRC-32 is joined from the
//             per-chunk CRCs of smr_inflate.h (crc_piece / crc_concat).
// There is one fixed algorithm: no level option.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>
#include "smr_inflate.h"   // bitrev, inf_len_sym, inf_dist_sym, crc_*

namespace smr {

constexpr uint32_t kDefChunk = 32768;        // input bytes per chunk (<= 65535: the stored fallback is one block)
constexpr uint32_t kDefWindow = 32768;       // DEFLATE's largest distance
constexpr uint32_t kDefHashBits = 12, kDefWays = 2, kDefTile = 32;
constexpr uint32_t kDefMinMatch = 4, kDefMaxMatch = 258, kDefNice = 64;   // candidates stop being tried once one reaches kDefNice
constexpr uint32_t kDefNoPos = 0xFFFFu;      // empty hash slot (positions are 16-bit offsets into the chunk's window)
constexpr uint32_t kDefFreqStride = 320;     // 286 litlen + 30 distance counts per chunk
constexpr uint32_t kDefHdrWords = 160;       // dynamic header: at most 17 + 19 * 3 + 316 * 14 bits
constexpr uint32_t kDefScratch = kDefChunk + 64;   // output bytes per chunk before placement (the stored form bounds it)
// one member holding nothing (a final fixed-Huffman block with only end-of-block), as zlib writes it
constexpr uint8_t kGzEmpty[20] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};

// one chunk of the input: bytes [b, e), history from h = max(stream start, b - 32768)
enum : uint32_t { kDefFirst = 1, kDefLast = 2 };
struct DefChunk { uint64_t b, e, h; uint32_t flags, stream; };
// what CODE decides for a chunk
struct DefInfo { uint32_t nsym, stored, hdr_bits, bytes; };
// canonical codes of a dynamic block, bit-reversed for the LSB-first writer; lengths 0 = unused
struct DefCodes { uint16_t code[316]; uint8_t len[316]; };

// byte i of zlib's gzip header: no name, mtime 0, XFL 0, OS 3 (1f 8b 08 00 00000000 00 03)
SMR_HD uint8_t gz_header_byte(uint32_t i) { return i == 0 ? 0x1f : i == 1 ? 0x8b : i == 2 ? 8 : i == 9 ? 3 : 0; }
constexpr uint32_t kGzHeader = 10;

// BGZF (SAMv1 4.1): gzip members of at most 64 KiB, each a stream of its own (no history before its first byte), whose header
// carries FLG.FEXTRA and the subfield BC with BSIZE = member bytes - 1.  A block takes kBgzfBlock input bytes, two chunks; with
// both chunks stored (5 + kDefChunk + 5, then 5 + the rest, final) a member is at most kBgzfMaxMember bytes.
constexpr uint32_t kBgzfBlock = 65280;
constexpr uint32_t kBgzfHeader = 18;
constexpr uint32_t kBgzfMaxMember = kBgzfHeader + (5 + kDefChunk + 5) + (5 + kBgzfBlock - kDefChunk) + 8;
static_assert(kBgzfBlock > kDefChunk && kBgzfBlock <= 2 * kDefChunk && kBgzfMaxMember <= 65536, "a BGZF member must fit in 64 KiB");
// the 18 header bytes of a member of `bytes` bytes: 1f 8b 08 04, MTIME 0, XFL 0, OS 255, XLEN 6, 'B' 'C', SLEN 2, BSIZE
inline void bgzf_header(uint8_t* p, uint32_t bytes) {
  static const uint8_t h[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
  memcpy(p, h, 16);
  p[16] = (uint8_t)(bytes - 1); p[17] = (uint8_t)((bytes - 1) >> 8);
}
// [b, e) cut into BGZF blocks of kBgzfBlock bytes, the last holding the rest (none when empty), appended to sb / se
inline void bgzf_blocks(uint64_t b, uint64_t e, std::vector<uint64_t>& sb, std::vector<uint64_t>& se) {
  for (; b < e; b += kBgzfBlock) { sb.push_back(b); se.push_back(std::min<uint64_t>(e, b + kBgzfBlock)); }
}

SMR_HD uint32_t def_load32(const uint8_t* t, uint64_t p) {   // 4 bytes at p, little-endian (the buffer is padded)
#if defined(__CUDA_ARCH__)
  const uint32_t* w = reinterpret_cast<const uint32_t*>(t);
  const uint64_t i = p >> 2;
  return __funnelshift_r(__ldg(w + i), __ldg(w + i + 1), (uint32_t)(p & 3) * 8);
#else
  uint32_t v; memcpy(&v, t + p, 4); return v;
#endif
}
SMR_HD uint32_t def_hash(const uint8_t* t, uint64_t p) { return (def_load32(t, p) * 2654435761u) >> (32 - kDefHashBits); }

// length of the common prefix of t[p..) and t[q..), q < p, at most maxlen
SMR_HD uint32_t def_match_len(const uint8_t* t, uint64_t p, uint64_t q, uint32_t maxlen) {
  uint32_t k = 0;
  while (k < maxlen) {
    const uint32_t x = def_load32(t, p + k) ^ def_load32(t, q + k);
    if (x) { k += (uint32_t)lb_ctz(x) >> 3; break; }
    k += 4;
  }
  return k < maxlen ? k : maxlen;
}

// The match of position p (packed len << 16 | dist, 0 = none) from its candidates, nearest first: the first one of the greatest
// length wins; a match shorter than kDefMinMatch is none.
// Candidates: q_tile (the nearest earlier position of the same hash in p's tile, or kInfNone), then the hash slot's positions
// (offsets from c.h, newest first).  Candidates more than 32 KB back are skipped.
SMR_HD uint32_t def_match_at(const uint8_t* t, const DefChunk& c, uint64_t p, uint64_t q_tile, const uint16_t* slot) {
  const uint32_t maxlen = c.e - p < kDefMaxMatch ? (uint32_t)(c.e - p) : kDefMaxMatch;
  uint32_t best = 0, bl = kDefMinMatch - 1;
  for (uint32_t k = 0; k <= kDefWays && bl < kDefNice; ++k) {
    uint64_t q;
    if (k == 0) { if (q_tile == kInfNone) continue; q = q_tile; }
    else { if (slot[k - 1] == kDefNoPos) break; q = c.h + slot[k - 1]; }
    if (p - q > kDefWindow) continue;
    const uint32_t l = def_match_len(t, p, q, maxlen);
    if (l > bl) { bl = l; best = (l << 16) | (uint32_t)(p - q); }
  }
  return best;
}

// DEFLATE symbols of a length (3..258) and a distance (1..32768); inf_len_sym / inf_dist_sym give back base and extra bits
SMR_HD uint32_t def_len_sym(uint32_t len) {
  if (len == 258) return 285;
  const uint32_t v = len - 3;
  if (v < 8) return 257 + v;
  const uint32_t t = 31 - (uint32_t)lb_clz(v);
  return 257 + 4 * (t - 1) + ((v >> (t - 2)) & 3u);
}
SMR_HD uint32_t def_dist_sym(uint32_t dist) {
  const uint32_t v = dist - 1;
  if (v < 4) return v;
  const uint32_t t = 31 - (uint32_t)lb_clz(v);
  return 2 * t + ((v >> (t - 1)) & 1u);
}
SMR_HD uint32_t def_len_extra(uint32_t s) { uint32_t b, e; inf_len_sym(s, b, e); return e; }
SMR_HD uint32_t def_dist_extra(uint32_t s) { uint32_t b, e; inf_dist_sym(s, b, e); return e; }

// PARSE of one chunk.  m[b .. e) holds the matches of MATCH on entry and the symbols on return, in place: symbol i of the chunk
// goes to m[b + i], and i <= (position consumed) - b, so no match is overwritten before it is read.  A symbol is a byte (< 256) or
// len << 16 | dist.  freq: 286 litlen + 30 distance counts, zero on entry.  Returns the number of symbols (end-of-block excluded).
SMR_HD uint32_t def_parse(uint32_t* m, uint64_t b, uint64_t e, const uint8_t* t, uint32_t* freq) {
  uint32_t n = 0;
  uint64_t p = b;
  while (p < e) {
    const uint32_t cur = m[p], len = cur >> 16;
    if (len && !(p + 1 < e && (m[p + 1] >> 16) > len)) {   // lazy: a longer match one byte on takes the byte as a literal
      m[b + n++] = cur;
      ++freq[def_len_sym(len)];
      ++freq[286 + def_dist_sym(cur & 0xFFFFu)];
      p += len;
    } else {
      const uint32_t c = t[p];
      m[b + n++] = c;
      ++freq[c];
      ++p;
    }
  }
  ++freq[256];
  return n;
}

// Code lengths of a Huffman code over freq[0 .. n) limited to maxbits (n <= 286).  Fewer than two used symbols are topped up with
// the lowest unused ones at weight 1, as zlib does, so every code is complete.  Huffman by two queues over the leaves sorted by
// (weight, symbol); lengths over maxbits are folded back by the count adjustment of miniz (tdefl_huffman_enforce_max_code_size),
// and the lengths are handed out longest first in that same sorted order.
SMR_HD void def_huff_lengths(const uint32_t* freq, uint32_t n, uint32_t maxbits, uint8_t* lens) {
  uint32_t key[286], w[286], iw[286];
  uint16_t lpar[286], ipar[286];
  uint8_t idep[286];
  uint32_t m = 0, extra = 0;
  for (uint32_t s = 0; s < n; ++s) { lens[s] = 0; if (freq[s]) ++m; }
  for (uint32_t s = 0; s < n && m + extra < 2; ++s) if (!freq[s]) { key[extra++] = (1u << 9) | s; }   // weight 1
  uint32_t k = 0;
  for (uint32_t s = 0; s < n; ++s) if (freq[s]) key[extra + k++] = (freq[s] << 9) | s;
  m += extra;
  for (uint32_t i = 1; i < m; ++i) {   // insertion sort by (weight, symbol)
    const uint32_t v = key[i];
    uint32_t j = i;
    while (j > 0 && key[j - 1] > v) { key[j] = key[j - 1]; --j; }
    key[j] = v;
  }
  for (uint32_t i = 0; i < m; ++i) w[i] = key[i] >> 9;
  uint32_t li = 0, ii = 0, ni = 0;
  auto take = [&](bool& leaf, uint32_t& idx) {
    if (li < m && (ii >= ni || w[li] <= iw[ii])) { leaf = true; idx = li++; } else { leaf = false; idx = ii++; }
  };
  for (uint32_t r = 0; r + 1 < m; ++r) {
    bool l1, l2; uint32_t a, c;
    take(l1, a); take(l2, c);
    iw[ni] = (l1 ? w[a] : iw[a]) + (l2 ? w[c] : iw[c]);
    if (l1) lpar[a] = (uint16_t)ni; else ipar[a] = (uint16_t)ni;
    if (l2) lpar[c] = (uint16_t)ni; else ipar[c] = (uint16_t)ni;
    ++ni;
  }
  idep[ni - 1] = 0;
  for (int32_t j = (int32_t)ni - 2; j >= 0; --j) idep[j] = (uint8_t)(idep[ipar[j]] + 1);
  uint32_t cnt[32];
  for (uint32_t l = 0; l < 32; ++l) cnt[l] = 0;
  for (uint32_t i = 0; i < m; ++i) { const uint32_t d = idep[lpar[i]] + 1u; ++cnt[d < maxbits ? d : maxbits]; }
  uint32_t total = 0;
  for (uint32_t l = 1; l <= maxbits; ++l) total += cnt[l] << (maxbits - l);
  while (total != (1u << maxbits)) {
    --cnt[maxbits];
    for (uint32_t l = maxbits - 1; l > 0; --l) if (cnt[l]) { --cnt[l]; cnt[l + 1] += 2; break; }
    --total;
  }
  uint32_t i = 0;
  for (uint32_t l = maxbits; l > 0; --l)
    for (uint32_t c = 0; c < cnt[l]; ++c) lens[key[i++] & 511u] = (uint8_t)l;
}

// canonical codes (RFC 1951 3.2.2) of n lengths, bit-reversed for the LSB-first writer
SMR_HD void def_canon(const uint8_t* lens, uint32_t n, uint16_t* code) {
  uint32_t cnt[16], next[16];
  for (uint32_t l = 0; l < 16; ++l) cnt[l] = 0;
  for (uint32_t s = 0; s < n; ++s) ++cnt[lens[s]];
  cnt[0] = 0;
  uint32_t c = 0;
  for (uint32_t l = 1; l < 16; ++l) { c = (c + cnt[l - 1]) << 1; next[l] = c; }
  for (uint32_t s = 0; s < n; ++s) if (lens[s]) code[s] = (uint16_t)bitrev(next[lens[s]]++, lens[s]);
}

// LSB-first bit writer that ORs whole 32-bit words into a zeroed buffer: writers of adjacent bit ranges may share a boundary word
struct BitOut { uint32_t* w; uint64_t word; uint64_t acc; uint32_t n; };
SMR_HD void bo_or(uint32_t* a, uint32_t v) {
#if defined(__CUDA_ARCH__)
  if (v) atomicOr(a, v);
#else
  *a |= v;
#endif
}
SMR_HD void bo_start(BitOut& o, uint32_t* w, uint64_t bitpos) { o.w = w; o.word = bitpos >> 5; o.n = (uint32_t)(bitpos & 31); o.acc = 0; }
SMR_HD void bo_put(BitOut& o, uint32_t v, uint32_t nb) {   // nb <= 32
  o.acc |= (uint64_t)v << o.n; o.n += nb;
  if (o.n >= 32) { bo_or(o.w + o.word++, (uint32_t)o.acc); o.acc >>= 32; o.n -= 32; }
}
SMR_HD void bo_flush(BitOut& o) { if (o.n) bo_or(o.w + o.word, (uint32_t)o.acc); }

// bits of one symbol (codes given)
SMR_HD uint32_t def_sym_bits(uint32_t s, const DefCodes& C) {
  if (s < 256) return C.len[s];
  const uint32_t ls = def_len_sym(s >> 16), ds = def_dist_sym(s & 0xFFFFu);
  return C.len[ls] + def_len_extra(ls) + C.len[286 + ds] + def_dist_extra(ds);
}
SMR_HD void def_put_sym(BitOut& o, uint32_t s, const DefCodes& C) {
  if (s < 256) { bo_put(o, C.code[s], C.len[s]); return; }
  const uint32_t len = s >> 16, dist = s & 0xFFFFu, ls = def_len_sym(len), ds = def_dist_sym(dist);
  uint32_t lb, le, db, de;
  inf_len_sym(ls, lb, le); inf_dist_sym(ds, db, de);
  bo_put(o, C.code[ls], C.len[ls]);
  if (le) bo_put(o, len - lb, le);
  bo_put(o, C.code[286 + ds], C.len[286 + ds]);
  if (de) bo_put(o, dist - db, de);
}

// CODE of one chunk: the codes, the header bits (hdr, zeroed, kDefHdrWords words) and the chunk's form and byte size.
// In two parts: def_code_tree builds the litlen (tree 0) or the distance code (tree 1) -- on the device two lanes build them at once --
// and def_code_block, given both, the rest.
SMR_HD void def_code_tree(const uint32_t* freq, uint32_t tree, DefCodes& C) {
  const uint32_t at = tree ? 286 : 0, n = tree ? 30 : 286;
  def_huff_lengths(freq + at, n, 15, C.len + at);
  def_canon(C.len + at, n, C.code + at);
}
SMR_HD void def_code_block(const uint32_t* freq, uint64_t nbytes, bool final_chunk, DefCodes& C, uint32_t* hdr, DefInfo& info) {
  uint32_t hlit = 286, hdist = 30;
  while (hlit > 257 && !C.len[hlit - 1]) --hlit;
  while (hdist > 1 && !C.len[286 + hdist - 1]) --hdist;
  // the code lengths of both codes, run-length coded (3.2.7): symbol | extra value << 5
  uint8_t all[316];
  for (uint32_t i = 0; i < hlit; ++i) all[i] = C.len[i];
  for (uint32_t i = 0; i < hdist; ++i) all[hlit + i] = C.len[286 + i];
  const uint32_t n = hlit + hdist;
  uint16_t rle[316];
  uint32_t nr = 0, clf[19];
  for (uint32_t i = 0; i < 19; ++i) clf[i] = 0;
  for (uint32_t i = 0; i < n;) {
    const uint32_t v = all[i];
    uint32_t run = 1;
    while (i + run < n && all[i + run] == v) ++run;
    i += run;
    if (v == 0) {
      while (run >= 11) { const uint32_t r = run < 138 ? run : 138; rle[nr++] = (uint16_t)(18 | (r - 11) << 5); ++clf[18]; run -= r; }
      if (run >= 3) { rle[nr++] = (uint16_t)(17 | (run - 3) << 5); ++clf[17]; run = 0; }
    } else {
      rle[nr++] = (uint16_t)v; ++clf[v]; --run;
      while (run >= 3) { const uint32_t r = run < 6 ? run : 6; rle[nr++] = (uint16_t)(16 | (r - 3) << 5); ++clf[16]; run -= r; }
    }
    for (; run; --run) { rle[nr++] = (uint16_t)v; ++clf[v]; }
  }
  uint8_t cll[19];
  uint16_t clc[19];
  def_huff_lengths(clf, 19, 7, cll);
  def_canon(cll, 19, clc);
  uint32_t hclen = 19;
  while (hclen > 4 && !cll[inf_cl_order(hclen - 1)]) --hclen;
  uint64_t bits = 3 + 14 + 3 * hclen;
  for (uint32_t i = 0; i < nr; ++i) { const uint32_t s = rle[i] & 31u; bits += cll[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0); }
  const uint32_t hdr_bits = (uint32_t)bits;
  for (uint32_t s = 0; s < 286; ++s) if (freq[s]) bits += (uint64_t)freq[s] * (C.len[s] + (s > 256 ? def_len_extra(s) : 0));
  for (uint32_t s = 0; s < 30; ++s) if (freq[286 + s]) bits += (uint64_t)freq[286 + s] * (C.len[286 + s] + def_dist_extra(s));
  const uint64_t dyn = final_chunk ? (bits + 7) / 8 : (bits + 3 + 7) / 8 + 4;
  const uint64_t stored = 5 + nbytes + (final_chunk ? 0 : 5);
  info.stored = dyn >= stored;
  info.bytes = (uint32_t)(info.stored ? stored : dyn);
  info.hdr_bits = hdr_bits;
  if (info.stored) return;
  BitOut o; bo_start(o, hdr, 0);
  bo_put(o, final_chunk ? 1u : 0u, 1); bo_put(o, 2, 2);
  bo_put(o, hlit - 257, 5); bo_put(o, hdist - 1, 5); bo_put(o, hclen - 4, 4);
  for (uint32_t i = 0; i < hclen; ++i) bo_put(o, cll[inf_cl_order(i)], 3);
  for (uint32_t i = 0; i < nr; ++i) {
    const uint32_t s = rle[i] & 31u, x = rle[i] >> 5;
    bo_put(o, clc[s], cll[s]);
    if (s >= 16) bo_put(o, x, s == 16 ? 2 : s == 17 ? 3 : 7);
  }
  bo_flush(o);
}

SMR_HD void def_code(const uint32_t* freq, uint64_t nbytes, bool final_chunk, DefCodes& C, uint32_t* hdr, DefInfo& info) {
  def_code_tree(freq, 0, C);
  def_code_tree(freq, 1, C);
  def_code_block(freq, nbytes, final_chunk, C, hdr, info);
}

// WRITE, the part of lane `lane` of `lanes`: symbols [lo, hi) of the chunk at bit `start` of its scratch; the lane that holds the
// last symbol also writes end-of-block and the chunk's end (sync-flush block or final padding).  Byte-wise parts (stored form, the
// end's LEN / NLEN) are written by def_write_tail.
SMR_HD uint64_t def_range_bits(const uint32_t* sym, uint32_t lo, uint32_t hi, const DefCodes& C) {
  uint64_t b = 0;
  for (uint32_t i = lo; i < hi; ++i) b += def_sym_bits(sym[i], C);
  return b;
}
SMR_HD void def_write_range(uint32_t* out, uint64_t start, const uint32_t* sym, uint32_t lo, uint32_t hi, const DefCodes& C, bool end) {
  BitOut o; bo_start(o, out, start);
  for (uint32_t i = lo; i < hi; ++i) def_put_sym(o, sym[i], C);
  if (end) bo_put(o, C.code[256], C.len[256]);   // then 3 zero bits of the empty stored block's header, already zero
  bo_flush(o);
}
// bytes of the stored form, or the 00 00 FF FF that ends a dynamic non-final chunk (out: the chunk's scratch as bytes)
SMR_HD void def_write_tail(uint8_t* out, const uint8_t* in, uint64_t n, const DefInfo& info, bool final_chunk, uint32_t lane, uint32_t lanes) {
  if (info.stored) {
    if (lane == 0) {
      out[0] = final_chunk ? 1 : 0;
      out[1] = (uint8_t)n; out[2] = (uint8_t)(n >> 8); out[3] = (uint8_t)~n; out[4] = (uint8_t)(~n >> 8);
    }
    for (uint64_t i = lane; i < n; i += lanes) out[5 + i] = in[i];
    if (!final_chunk && lane == 0) { uint8_t* z = out + 5 + n; z[0] = 0; z[1] = 0; z[2] = 0; z[3] = 0xFF; z[4] = 0xFF; }
  } else if (!final_chunk && lane == 0) {
    uint8_t* z = out + info.bytes - 4; z[0] = 0; z[1] = 0; z[2] = 0xFF; z[3] = 0xFF;
  }
}

// the chunks of streams [sb[k], se[k]) (empty streams have none)
inline void def_plan(const uint64_t* sb, const uint64_t* se, uint32_t nstreams, std::vector<DefChunk>& ch) {
  ch.clear();
  for (uint32_t s = 0; s < nstreams; ++s)
    for (uint64_t b = sb[s]; b < se[s]; b += kDefChunk) {
      const uint64_t e = std::min<uint64_t>(se[s], b + kDefChunk);
      ch.push_back(DefChunk{b, e, b - sb[s] > kDefWindow ? b - kDefWindow : sb[s], (b == sb[s] ? kDefFirst : 0u) | (e == se[s] ? kDefLast : 0u), s});
    }
}
inline void def_put32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }

}  // namespace smr
