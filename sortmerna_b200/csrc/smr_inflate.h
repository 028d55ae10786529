// gzip / DEFLATE (RFC 1952 / RFC 1951) decoding as plain functions shared by the CUDA kernels (smr_inflate.cuh) and by the
// host-side check tests/inflate_check.cpp, which runs the very same span logic on the CPU against zlib.
//
// Stands in for the gz half of the reference's read feed: Readfeed::next_gz / izlib::getline inflate a reads file through
// zlib / rapidgzip on the host (src/sortmerna/readfeed.cpp:683-770, izlib.cpp); here the compressed bytes go to the device
// and are inflated there (SURVEY 8(f)(2)).
//
// How one DEFLATE stream becomes parallel work (the two-stage scheme of pugz / rapidgzip, re-laid for a GPU):
//   1. FIND   every chunk of the compressed file (64 KB by default) is searched, one bit offset per thread, for the first
//             position that parses as a non-final dynamic-Huffman block header (strict: complete code-length code, litlen /
//             distance code lengths that form complete prefix codes, end-of-block symbol present).  A hit is a CANDIDATE.
//   2. COUNT  one thread per candidate decodes from its position -- without the 32 KB of history a back-reference may need
//             -- until it lands exactly on a later candidate or the stream ends, and reports where it stopped and how many
//             bytes it produced.  The walk from the true start of the stream over "lands on" links picks the spans that are
//             real; anything else (a false candidate) is dropped.  Correctness never depends on step 1: a block start that was
//             not found only makes a span longer.
//   3. WRITE  the same decode again for the real spans, now storing 16-bit symbols at the span's offset in the output: a
//             byte, or 256 + k for "byte k of the 32 KB that precede this span" (a MARKER).
//   4. WINDOW the last 32 KB of every span are resolved front to back (each needs only the previous span's window);
//   5. RESOLVE every symbol becomes a byte, all spans in parallel.
//
// The five steps run in ROUNDS over whatever part of the file is held, so a file can be inflated as it arrives (the read stream
// of smr_stream_push).  A round that is not the file's last lets its last span decode until the input runs out and resumes the
// next round at the last block boundary that span crossed (InfResume): the output up to there is kept, the 32 KB before it seed
// the window of the next round's first span, and the CRC-32 / length of the member still open carry over (InfCarry).  A whole
// file in memory is the one-round case.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>
#include "smr_levbits.h"   // SMR_HD

namespace smr {

constexpr uint32_t kInfWindow = 32768;
constexpr uint32_t kInfLutBitsL = 9, kInfLutBitsD = 8;
constexpr uint64_t kInfNone = ~0ull;

// status of a decoded span
enum InfStatus : uint32_t { kInfLanded = 0, kInfEos = 1, kInfErrCode = 2, kInfErrHeader = 3, kInfErrOverrun = 4, kInfErrDistance = 5,
                            kInfErrStored = 6, kInfErrMember = 7, kInfErrCapacity = 8, kInfErrCrc = 9, kInfErrSize = 10 };

// ---------------------------------------------------------------------------------------------------------------------
// bit reader over the stream as 32-bit little-endian words (the buffer is padded with >= 64 zero bytes)
// ---------------------------------------------------------------------------------------------------------------------
struct BitIn {
  const uint32_t* w;
  uint64_t buf;
  uint64_t next;   // next word to load into `ahead`
  uint32_t cnt;    // valid bits in buf
  uint32_t ahead;  // w[next - 1], loaded one refill early so that its latency is off the decode chain
};
SMR_HD void bi_seek(BitIn& b, uint64_t bitpos) {
  b.next = bitpos >> 5;
  const uint32_t s = (uint32_t)(bitpos & 31);
  b.buf = (uint64_t)b.w[b.next++] >> s;
  b.cnt = 32 - s;
  b.ahead = b.w[b.next++];
}
SMR_HD void bi_fill(BitIn& b) {   // afterwards cnt >= 33
  if (b.cnt <= 32) { b.buf |= (uint64_t)b.ahead << b.cnt; b.cnt += 32; b.ahead = b.w[b.next++]; }
}
SMR_HD uint64_t bi_pos(const BitIn& b) { return (b.next - 1) * 32 - b.cnt; }
SMR_HD uint32_t bi_peek(const BitIn& b, uint32_t n) { return (uint32_t)(b.buf & ((1ull << n) - 1)); }   // n <= 32 <= cnt
SMR_HD void bi_skip(BitIn& b, uint32_t n) { b.buf >>= n; b.cnt -= n; }
SMR_HD uint32_t bi_get(BitIn& b, uint32_t n) { const uint32_t v = bi_peek(b, n); bi_skip(b, n); return v; }

// ---------------------------------------------------------------------------------------------------------------------
// Huffman tables of one decoder (2.6 KB; in shared memory on the device)
// ---------------------------------------------------------------------------------------------------------------------
struct HuffTabs {
  uint16_t llut[1 << kInfLutBitsL];   // (symbol << 4) | code length for litlen codes of <= 9 bits; 0 = longer code (or none)
  uint16_t dlut[1 << kInfLutBitsD];   // same for distance codes of <= 8 bits
  uint16_t lcount[16], dcount[16];    // codes per length (canonical decode of the long codes)
  uint16_t lsym[288], dsym[32];       // symbols ordered by (length, symbol)
  uint8_t lens[320];                  // code lengths of the block being set up
};

SMR_HD uint32_t bitrev(uint32_t v, uint32_t n) {   // reverse the low n bits
  uint32_t r = 0;
  for (uint32_t i = 0; i < n; ++i) { r = (r << 1) | (v & 1u); v >>= 1; }
  return r;
}

// canonical code from n lengths: count[], sym[] and the first-level table.  Returns 0 complete, 1 incomplete (allowed only for a
// single code of length 1, as zlib's inflate_table does), 2 over-subscribed / incomplete otherwise.  n == 0 codes used: 1 with an empty table.
SMR_HD uint32_t huff_build(const uint8_t* lens, uint32_t n, uint16_t* count, uint16_t* sym, uint16_t* lut, uint32_t lutbits) {
  for (uint32_t l = 0; l < 16; ++l) count[l] = 0;
  for (uint32_t s = 0; s < n; ++s) count[lens[s]]++;
  const uint32_t used = n - count[0];
  int32_t left = 1;
  uint32_t maxlen = 0;
  for (uint32_t l = 1; l < 16; ++l) {
    left <<= 1; left -= (int32_t)count[l];
    if (left < 0) return 2;
    if (count[l]) maxlen = l;
  }
  uint16_t offs[16];
  offs[1] = 0;
  for (uint32_t l = 1; l < 15; ++l) offs[l + 1] = (uint16_t)(offs[l] + count[l]);
  for (uint32_t s = 0; s < n; ++s) if (lens[s]) sym[offs[lens[s]]++] = (uint16_t)s;
  for (uint32_t i = 0; i < (1u << lutbits); ++i) lut[i] = 0;
  uint32_t code = 0, idx = 0;
  for (uint32_t l = 1; l <= lutbits; ++l) {
    for (uint32_t k = 0; k < count[l]; ++k, ++idx, ++code) {
      const uint16_t e = (uint16_t)((sym[idx] << 4) | l);
      for (uint32_t i = bitrev(code, l); i < (1u << lutbits); i += (1u << l)) lut[i] = e;
    }
    code <<= 1;
  }
  count[0] = 0;   // the canonical walk must not count unused symbols
  if (left > 0) return (used == 1 && maxlen == 1) || used == 0 ? 1u : 2u;
  return 0;
}

// one symbol: first-level table, else bit by bit over the canonical code (puff.c's decode()).  Returns the symbol or 0xFFFF.
SMR_HD uint32_t huff_decode(BitIn& b, const uint16_t* lut, uint32_t lutbits, const uint16_t* count, const uint16_t* sym) {
  const uint32_t e = lut[bi_peek(b, lutbits)];
  if (e) { bi_skip(b, e & 15u); return e >> 4; }
  uint32_t code = 0, first = 0, index = 0;
  uint64_t bits = b.buf;
  for (uint32_t l = 1; l < 16; ++l) {
    code |= (uint32_t)(bits & 1u); bits >>= 1;
    const uint32_t c = count[l];
    if (code < first + c) { bi_skip(b, l); return sym[index + (code - first)]; }
    index += c; first += c; first <<= 1; code <<= 1;
  }
  return 0xFFFFu;
}

// order of the code-length code lengths (RFC 1951 3.2.7): 16 17 18 0 8 7 9 6 10 5 11 4 | 12 3 13 2 14 1 15, five bits each
SMR_HD uint32_t inf_cl_order(uint32_t i) {
  const uint64_t a = 16ull | 17ull << 5 | 18ull << 10 | 0ull << 15 | 8ull << 20 | 7ull << 25 | 9ull << 30 | 6ull << 35 | 10ull << 40 | 5ull << 45 | 11ull << 50 | 4ull << 55;
  const uint64_t c = 12ull | 3ull << 5 | 13ull << 10 | 2ull << 15 | 14ull << 20 | 1ull << 25 | 15ull << 30;
  return (uint32_t)((i < 12 ? a >> (5 * i) : c >> (5 * (i - 12))) & 31u);
}

// base values / extra bits of the length and distance symbols (RFC 1951 3.2.5), computed instead of tabulated
SMR_HD void inf_len_sym(uint32_t s /*257..285*/, uint32_t& base, uint32_t& extra) {
  const uint32_t k = s - 257;
  if (k < 8) { base = 3 + k; extra = 0; return; }
  if (k == 28) { base = 258; extra = 0; return; }
  extra = (k >> 2) - 1;
  base = 3 + ((4 + (k & 3)) << extra);
}
SMR_HD void inf_dist_sym(uint32_t s /*0..29*/, uint32_t& base, uint32_t& extra) {
  if (s < 4) { base = 1 + s; extra = 0; return; }
  extra = (s >> 1) - 1;
  base = 1 + ((2 + (s & 1)) << extra);
}

// Dynamic block header after BFINAL/BTYPE (RFC 1951 3.2.7): code lengths into lens[0 .. hlit+hdist).  Returns false when the
// header is not one a compliant encoder writes (the same rules serve the candidate search and the real decode).
// `cnt`/`sy`: scratch for the code-length code (16 + 19 entries), `lut7`: 128 entries.
SMR_HD bool inf_dynamic_header(BitIn& b, uint8_t* lens, uint32_t& hlit, uint32_t& hdist, uint16_t* cnt, uint16_t* sy, uint16_t* lut7) {
  bi_fill(b);
  hlit = bi_get(b, 5) + 257; hdist = bi_get(b, 5) + 1;
  const uint32_t hclen = bi_get(b, 4) + 4;
  if (hlit > 286 || hdist > 30) return false;
  uint8_t cl[19];
  for (uint32_t i = 0; i < 19; ++i) cl[i] = 0;
  for (uint32_t i = 0; i < hclen; ++i) { bi_fill(b); cl[inf_cl_order(i)] = (uint8_t)bi_get(b, 3); }
  if (huff_build(cl, 19, cnt, sy, lut7, 7) != 0) return false;   // zlib: the code-length code must be complete
  uint32_t i = 0;
  const uint32_t n = hlit + hdist;
  while (i < n) {
    bi_fill(b);
    const uint32_t s = huff_decode(b, lut7, 7, cnt, sy);
    if (s < 16) { lens[i++] = (uint8_t)s; continue; }
    if (s > 18) return false;
    uint32_t rep, val = 0;
    if (s == 16) { if (i == 0) return false; val = lens[i - 1]; rep = 3 + bi_get(b, 2); }
    else if (s == 17) rep = 3 + bi_get(b, 3);
    else rep = 11 + bi_get(b, 7);
    if (i + rep > n) return false;
    for (uint32_t k = 0; k < rep; ++k) lens[i++] = (uint8_t)val;
  }
  return lens[256] != 0;   // zlib: "invalid code -- missing end-of-block"
}

// Does a non-final dynamic block start at bit p?  (candidate test of the FIND step; thread-local scratch)
SMR_HD bool inf_probe_block(const uint32_t* w, uint64_t nbits, uint64_t p) {
  if (p + 17 + 8 * 8 > nbits) return false;
  BitIn b; b.w = w; bi_seek(b, p); bi_fill(b);
  const uint32_t h = bi_peek(b, 13);
  if ((h & 7u) != 4u) return false;                       // BFINAL = 0, BTYPE = 2 (bits: final, then type LSB first)
  if (((h >> 3) & 31u) > 29u || ((h >> 8) & 31u) > 29u) return false;
  bi_skip(b, 3);
  // cheap pre-check of the code-length code before anything is built: Kraft sum of the 3-bit lengths must be exactly 1
  {
    BitIn c = b; bi_fill(c); bi_skip(c, 10);
    const uint32_t hclen = bi_get(c, 4) + 4;
    uint32_t kraft = 0;
    for (uint32_t i = 0; i < hclen; ++i) { bi_fill(c); const uint32_t l = bi_get(c, 3); if (l) kraft += 128u >> l; }
    if (kraft != 128u) return false;
  }
  uint8_t lens[320];
  uint16_t cnt[16], sy[19], lut7[128];
  uint32_t hlit, hdist;
  if (!inf_dynamic_header(b, lens, hlit, hdist, cnt, sy, lut7)) return false;
  if (bi_pos(b) > nbits) return false;
  // both codes must be usable: Kraft sums (a single length-1 distance code or no distance code at all is legal)
  uint32_t kl = 0, kd = 0, nd = 0, maxd = 0;
  for (uint32_t i = 0; i < hlit; ++i) if (lens[i]) kl += 32768u >> lens[i];
  for (uint32_t i = 0; i < hdist; ++i) if (lens[hlit + i]) { kd += 32768u >> lens[hlit + i]; ++nd; if (lens[hlit + i] > maxd) maxd = lens[hlit + i]; }
  if (kl != 32768u) return false;
  if (kd != 32768u && !(nd == 0 || (nd == 1 && maxd == 1))) return false;
  return true;
}

// ---------------------------------------------------------------------------------------------------------------------
// gzip member header (RFC 1952 2.3) at byte `at`; returns the byte after it or kInfNone
// ---------------------------------------------------------------------------------------------------------------------
SMR_HD uint64_t gz_member_header(const uint8_t* p, uint64_t nbytes, uint64_t at) {
  if (at + 18 > nbytes) return kInfNone;
  if (p[at] != 0x1f || p[at + 1] != 0x8b || p[at + 2] != 8) return kInfNone;
  const uint32_t flg = p[at + 3];
  if (flg & 0xE0u) return kInfNone;
  uint64_t q = at + 10;
  if (flg & 4u) { if (q + 2 > nbytes) return kInfNone; q += 2 + (uint64_t)(p[q] | (p[q + 1] << 8)); }
  if (flg & 8u) { while (q < nbytes && p[q]) ++q; ++q; }
  if (flg & 16u) { while (q < nbytes && p[q]) ++q; ++q; }
  if (flg & 2u) q += 2;
  return q + 8 <= nbytes ? q : kInfNone;
}

// Could the bytes at `at` still become a gzip member header once more bytes arrive?  (what is there matches ID1 ID2 CM FLG)
SMR_HD bool gz_member_short(const uint8_t* p, uint64_t nbytes, uint64_t at) {
  const uint8_t id[3] = {0x1f, 0x8b, 8};
  for (uint64_t k = 0; k < 3; ++k) if (at + k < nbytes && p[at + k] != id[k]) return false;
  return !(at + 3 < nbytes && (p[at + 3] & 0xE0u));
}

struct SpanResult {
  uint64_t end_bit;     // landed: the candidate position; eos: first bit after the last trailer
  uint64_t out_n;       // bytes produced
  uint32_t status;      // InfStatus
  uint32_t isize_sum;   // sum of the ISIZE fields of the members that ended in this span (mod 2^32)
  uint32_t members;     // gzip members that ended in this span
  uint32_t pad;
  uint64_t blk_bit;     // start of the last block the span began to decode (a round that ran out of input resumes there)
  uint64_t blk_out;     // bytes produced before that block
  uint64_t stop_bit;    // how far the decoder had read when it stopped (an error this close to the end of a partial input may be the cut);
                        // a member header that failed: nbits if more bytes may still complete it, else its start
};
struct MemberEnd { uint64_t out_end; uint32_t crc, isize; };   // trailer of a member (RFC 1952 2.3.1); out_end counts from the span's first byte

// One span: decode from `start_bit` (a block start; or a member header when `at_member` is set) until a block boundary that is one of
// the sorted candidate positions cand[first_cand ..ncand) or the end of the gzip stream.  WRITE: 16-bit symbols to out[0 .. out_cap).
// member_prior: bytes of the open member produced before start_bit, when they are known (the first span of a resumed round);
// kInfNone otherwise.
template <bool WRITE>
SMR_HD void inflate_span(const uint32_t* w, uint64_t nbytes, uint64_t start_bit, bool at_member, const uint64_t* cand, uint32_t ncand,
                         uint32_t first_cand, HuffTabs& T, uint16_t* out, uint64_t out_cap, MemberEnd* mem, SpanResult& res,
                         uint64_t member_prior = kInfNone) {
  const uint8_t* bytes = reinterpret_cast<const uint8_t*>(w);
  const uint64_t nbits = nbytes * 8, wlimit = (nbits >> 5) + 3;   // a decoder that has loaded this many words ran past the end
  bool member_known = member_prior != kInfNone;
  uint64_t n = 0, member_base = 0 - member_prior, blk_bit = start_bit, blk_out = 0;   // member_base wraps: n - member_base = bytes of the member
  uint32_t nextc = first_cand, isize_sum = 0, members = 0;
  BitIn b; b.w = w;
  bool seeked = false;
  auto finish = [&](uint32_t st, uint64_t endb) {
    res.end_bit = endb; res.out_n = n; res.status = st; res.isize_sum = isize_sum; res.members = members; res.pad = 0;
    res.blk_bit = blk_bit; res.blk_out = blk_out; res.stop_bit = seeked ? bi_pos(b) : endb;
  };
  uint64_t pos = start_bit;
  if (at_member) {
    const uint64_t q = gz_member_header(bytes, nbytes, pos >> 3);
    if (q == kInfNone) { finish(kInfErrMember, pos); if (gz_member_short(bytes, nbytes, pos >> 3)) res.stop_bit = nbits; return; }
    pos = q * 8; member_base = 0; member_known = true;
  }
  bi_seek(b, pos); seeked = true;
  bool first_block = true;
  for (;;) {
    pos = bi_pos(b);
    blk_bit = pos; blk_out = n;
    if (pos + 3 > nbits) { finish(kInfErrOverrun, pos); return; }
    if (!first_block || at_member) {   // a block boundary reached by decoding: is it another span's start?
      while (nextc < ncand && cand[nextc] < pos) ++nextc;
      if (nextc < ncand && cand[nextc] == pos && pos != start_bit) { finish(kInfLanded, pos); return; }
    }
    first_block = false;
    bi_fill(b);
    const uint32_t bfinal = bi_get(b, 1), btype = bi_get(b, 2);
    if (btype == 3) { finish(kInfErrHeader, pos); return; }
    if (btype == 0) {   // stored (RFC 1951 3.2.4)
      uint64_t q = (bi_pos(b) + 7) >> 3;
      if (q + 4 > nbytes) { finish(kInfErrOverrun, pos); return; }
      const uint32_t len = bytes[q] | (bytes[q + 1] << 8), nlen = bytes[q + 2] | (bytes[q + 3] << 8);
      if ((len ^ nlen) != 0xFFFFu) { finish(kInfErrStored, pos); return; }
      q += 4;
      if (q + len > nbytes) { finish(kInfErrOverrun, pos); return; }
      if (WRITE) { if (n + len > out_cap) { finish(kInfErrCapacity, pos); return; } for (uint32_t i = 0; i < len; ++i) out[n + i] = bytes[q + i]; }
      n += len;
      bi_seek(b, (q + len) * 8);
    } else {
      if (btype == 1) {   // fixed codes (3.2.6)
        for (uint32_t i = 0; i < 144; ++i) T.lens[i] = 8;
        for (uint32_t i = 144; i < 256; ++i) T.lens[i] = 9;
        for (uint32_t i = 256; i < 280; ++i) T.lens[i] = 7;
        for (uint32_t i = 280; i < 288; ++i) T.lens[i] = 8;
        huff_build(T.lens, 288, T.lcount, T.lsym, T.llut, kInfLutBitsL);
        for (uint32_t i = 0; i < 30; ++i) T.lens[i] = 5;
        huff_build(T.lens, 30, T.dcount, T.dsym, T.dlut, kInfLutBitsD);
      } else {
        uint32_t hlit, hdist;
        // the code-length code borrows the distance arrays, which are built afterwards
        if (!inf_dynamic_header(b, T.lens, hlit, hdist, T.dcount, T.dsym, T.dlut)) { finish(kInfErrHeader, pos); return; }
        if (huff_build(T.lens, hlit, T.lcount, T.lsym, T.llut, kInfLutBitsL) == 2) { finish(kInfErrHeader, pos); return; }
        if (huff_build(T.lens + hlit, hdist, T.dcount, T.dsym, T.dlut, kInfLutBitsD) == 2) { finish(kInfErrHeader, pos); return; }
      }
      for (;;) {   // symbols of the block (3.2.3)
        bi_fill(b);
        uint32_t s = huff_decode(b, T.llut, kInfLutBitsL, T.lcount, T.lsym);
        if (b.next > wlimit) { finish(kInfErrOverrun, pos); return; }
        if (s < 256) {
          if (WRITE) { if (n >= out_cap) { finish(kInfErrCapacity, pos); return; } out[n] = (uint16_t)s; }
          ++n;
          continue;
        }
        if (s == 256) break;
        if (s > 285) { finish(kInfErrCode, bi_pos(b)); return; }
        uint32_t lbase, lextra, dbase, dextra;
        inf_len_sym(s, lbase, lextra);
        const uint32_t len = lbase + bi_get(b, lextra);     // <= 5 bits; at least 33 - 15 were left
        bi_fill(b);
        const uint32_t ds = huff_decode(b, T.dlut, kInfLutBitsD, T.dcount, T.dsym);
        if (ds > 29) { finish(kInfErrCode, bi_pos(b)); return; }
        inf_dist_sym(ds, dbase, dextra);
        const uint32_t dist = dbase + bi_get(b, dextra);    // <= 13 bits after <= 15 of the code
        if (member_known && dist > n - member_base) { finish(kInfErrDistance, bi_pos(b)); return; }   // zlib: "invalid distance too far back"
        if (WRITE) {
          if (n + len > out_cap) { finish(kInfErrCapacity, pos); return; }
          // the copy (3.2.3): up to `dist` symbols never overlap what they produce, so they are loaded together before they are
          // stored -- one memory latency per group instead of one per symbol
          const uint32_t grp = dist < 8u ? dist : 8u;
          for (uint32_t i = 0; i < len; i += grp) {
            uint16_t tmp[8];
            const uint32_t m = len - i < grp ? len - i : grp;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
            for (uint32_t j = 0; j < 8; ++j) if (j < m) {
              const int64_t v = (int64_t)(n + i + j) - (int64_t)dist;
              tmp[j] = v >= 0 ? out[v] : (uint16_t)(256 + kInfWindow + v);
            }
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
            for (uint32_t j = 0; j < 8; ++j) if (j < m) out[n + i + j] = tmp[j];
          }
        }
        n += len;
        if (bi_pos(b) > nbits) { finish(kInfErrOverrun, pos); return; }
      }
      if (bi_pos(b) > nbits) { finish(kInfErrOverrun, pos); return; }
    }
    if (bfinal) {   // member trailer (RFC 1952: CRC32, ISIZE), then another member or the end
      uint64_t q = (bi_pos(b) + 7) >> 3;
      if (q + 8 > nbytes) { finish(kInfErrOverrun, pos); return; }
      const uint32_t crc = (uint32_t)bytes[q] | ((uint32_t)bytes[q + 1] << 8) | ((uint32_t)bytes[q + 2] << 16) | ((uint32_t)bytes[q + 3] << 24);
      const uint32_t isz = (uint32_t)bytes[q + 4] | ((uint32_t)bytes[q + 5] << 8) | ((uint32_t)bytes[q + 6] << 16) | ((uint32_t)bytes[q + 7] << 24);
      if (WRITE && mem) { mem[members].out_end = n; mem[members].crc = crc; mem[members].isize = isz; }
      ++members; isize_sum += isz;
      q += 8;
      const uint64_t h = gz_member_header(bytes, nbytes, q);
      if (h == kInfNone) { finish(kInfEos, q * 8); return; }   // gzip: trailing bytes that are no member are ignored
      member_base = n; member_known = true;
      bi_seek(b, h * 8);
    }
  }
}

// CRC-32 (RFC 1952 8): per piece on the device, pieces joined on the host.  Polynomials are kept reflected (bit 31 = x^0).
constexpr uint32_t kCrcPoly = 0xEDB88320u;
SMR_HD uint32_t crc_table_entry(uint32_t i) {
  uint32_t c = i;
  for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ kCrcPoly : c >> 1;
  return c;
}
SMR_HD uint32_t crc_piece(const uint8_t* p, uint64_t n, const uint32_t* tab) {
  uint32_t c = 0xFFFFFFFFu;
  for (uint64_t i = 0; i < n; ++i) c = tab[(c ^ p[i]) & 255u] ^ (c >> 8);
  return ~c;
}
inline uint32_t crc_mulmod(uint32_t a, uint32_t b) {   // a * b mod P
  uint32_t prod = 0;
  for (int i = 0; i < 32; ++i) {
    if (a & (0x80000000u >> i)) prod ^= b;
    b = (b & 1u) ? (b >> 1) ^ kCrcPoly : b >> 1;
  }
  return prod;
}
inline uint32_t crc_concat(uint32_t crc_a, uint32_t crc_b, uint64_t len_b) {   // CRC of A||B from the CRCs of A and B
  uint32_t r = 0x80000000u, base = 0x00800000u;   // 1, x^8
  for (uint64_t n = len_b; n; n >>= 1) { if (n & 1u) r = crc_mulmod(r, base); base = crc_mulmod(base, base); }
  return crc_mulmod(r, crc_a) ^ crc_b;
}

// Host side of the CRC / ISIZE check: the members (trailers in stream order, out_end = offset in the whole output) are cut into
// pieces that end at multiples of `piece` bytes; `first[m]` = first piece of member m.  Output past the last trailer, up to
// `total`, belongs to the member still open at the end of a round: its pieces follow, from first[ends.size()] to first[ends.size() + 1].
inline void inf_crc_plan(const std::vector<MemberEnd>& ends, uint32_t piece, std::vector<uint64_t>& poff, std::vector<uint32_t>& plen, std::vector<uint32_t>& first,
                         uint64_t total = 0) {
  poff.clear(); plen.clear(); first.clear();
  uint64_t a = 0;
  for (const MemberEnd& m : ends) {
    first.push_back((uint32_t)poff.size());
    while (a < m.out_end) {
      const uint64_t stop = std::min<uint64_t>(m.out_end, (a / piece + 1) * piece);
      poff.push_back(a); plen.push_back((uint32_t)(stop - a));
      a = stop;
    }
  }
  first.push_back((uint32_t)poff.size());
  while (a < total) {
    const uint64_t stop = std::min<uint64_t>(total, (a / piece + 1) * piece);
    poff.push_back(a); plen.push_back((uint32_t)(stop - a));
    a = stop;
  }
  first.push_back((uint32_t)poff.size());
}
// CRC-32 and length of the member that is open where a round ends; the next round's first member starts with them
struct InfCarry { uint32_t crc = 0; uint64_t len = 0; };   // 0 = CRC of the empty string
inline uint32_t inf_crc_verify(const std::vector<MemberEnd>& ends, const std::vector<uint32_t>& plen, const std::vector<uint32_t>& first, const uint32_t* crcs,
                               InfCarry* carry = nullptr) {
  InfCarry c0;
  InfCarry& cy = carry ? *carry : c0;
  uint64_t a = 0 - cy.len;   // wraps: out_end - a = the member's whole length
  for (size_t m = 0; m < ends.size(); ++m) {
    if ((uint32_t)(ends[m].out_end - a) != ends[m].isize) return kInfErrSize;
    uint32_t c = m ? 0u : cy.crc;
    for (uint32_t k = first[m]; k < first[m + 1]; ++k) c = crc_concat(c, crcs[k], plen[k]);
    if (c != ends[m].crc) return kInfErrCrc;
    a = ends[m].out_end;
  }
  if (!ends.empty()) cy = InfCarry{};
  if (first.size() > ends.size() + 1)
    for (uint32_t k = first[ends.size()]; k < first[ends.size() + 1]; ++k) { cy.crc = crc_concat(cy.crc, crcs[k], plen[k]); cy.len += plen[k]; }
  return 0;
}

// a resolved byte: the symbol itself, or the byte of the previous span's window a marker names
SMR_HD uint8_t inf_resolve(uint16_t sym, const uint8_t* prev_window) { return sym < 256 ? (uint8_t)sym : prev_window[sym - 256]; }
// byte k of the window a span of n symbols (at `syms`) leaves behind: its own tail, preceded by the tail of the previous window
SMR_HD uint8_t inf_window_byte(const uint16_t* syms, uint64_t n, const uint8_t* prev_window, uint32_t k) {
  const int64_t v = (int64_t)n - (int64_t)kInfWindow + (int64_t)k;
  return v >= 0 ? inf_resolve(syms[v], prev_window) : prev_window[kInfWindow + v];
}

// Where a round of the inflate ends.  bit: where the next round starts (in the round's input); at_member: a gzip member header is
// due there; keep_last: the bytes of the chain's last span that are kept (its output up to `bit`); eos: the stream ended.
struct InfResume { uint64_t bit = 0; bool at_member = true; bool eos = false; uint64_t keep_last = 0; };

// The walk over the COUNT results (host side): span 0 is the start of the round, span i >= 1 starts at cand[i - 1].  Fills
// `real` with the spans that are reached and `off` with their output offsets; returns the bytes the round keeps or kInfNone
// with *why set.  A round over the whole rest of the file (eof) must end in the end of the gzip stream.  Otherwise (next != null,
// eof false) the chain may end in a span that ran out of input: the round keeps the output up to that span's last block boundary
// and *next says where to resume.  The sum of the ISIZE fields is checked here when the round covers whole members (isize_check);
// every member is checked again, with its CRC, after the write pass.
inline uint64_t inf_chain(const uint64_t* cand, uint32_t ncand, const SpanResult* res, uint32_t* real, uint64_t* off, uint32_t& nreal, uint32_t* why,
                          bool eof = true, uint64_t nbits = 0, bool isize_check = true, InfResume* next = nullptr) {
  uint64_t total = 0;
  uint32_t isize = 0;
  nreal = 0;
  uint32_t i = 0;
  for (;;) {
    real[nreal] = i; off[nreal] = total; ++nreal;
    total += res[i].out_n; isize += res[i].isize_sum;
    if (next) next->keep_last = res[i].out_n;
    if (res[i].status == kInfEos) {
      if (next) { next->bit = res[i].end_bit; next->at_member = true; next->eos = eof; }
      break;
    }
    if (res[i].status != kInfLanded) {
      // before the end of the file: the last span stopped because the input ran out -- or it met an error close enough to the end
      // that the missing bytes may be the cause (a decode error reads at most 64 bits past what it consumed), or a member header
      // that has not fully arrived
      const bool cut = res[i].status == kInfErrMember ? res[i].stop_bit >= nbits : (res[i].status == kInfErrOverrun || res[i].stop_bit + 128 > nbits);
      if (!eof && next && cut) {
        total -= res[i].out_n - res[i].blk_out;
        next->keep_last = res[i].blk_out;
        if (res[i].status == kInfErrMember) next->bit = res[i].end_bit;
        else { next->bit = res[i].blk_bit; next->at_member = false; }
        next->eos = false;
        return total;
      }
      *why = res[i].status; return kInfNone;
    }
    uint32_t lo = i, hi = ncand;   // the candidate it landed on: cand[] is sorted, and it lies after span i's own start
    while (lo < hi) { const uint32_t mid = (lo + hi) / 2; if (cand[mid] < res[i].end_bit) lo = mid + 1; else hi = mid; }
    if (lo >= ncand || cand[lo] != res[i].end_bit) { *why = kInfErrMember; return kInfNone; }
    i = lo + 1;
  }
  if (isize_check && (uint32_t)total != isize) { *why = kInfErrSize; return kInfNone; }   // RFC 1952 ISIZE: sizes mod 2^32 (per member again after the write pass)
  return total;
}

}  // namespace smr
