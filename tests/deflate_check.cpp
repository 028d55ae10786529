// Host-side run of sortmerna_b200/csrc/smr_deflate.h: the MATCH / PARSE / CODE / WRITE / PLACE steps the CUDA kernels perform
// (smr_deflate.cuh), serially on the CPU, giving the bytes the device writes.  tests/test_deflate_host.py checks them with zlib.
//   deflate_check in.bin out.gz   -> one gzip member; prints "ok bytes N chunks C stored S"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../sortmerna_b200/csrc/smr_deflate.h"
using namespace smr;

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<uint8_t> raw;
  { uint8_t buf[65536]; size_t k; while ((k = fread(buf, 1, sizeof buf, f)) > 0) raw.insert(raw.end(), buf, buf + k); fclose(f); }
  const uint64_t n = raw.size();
  std::vector<uint8_t> out;
  uint32_t nstored = 0;
  std::vector<DefChunk> ch;
  const uint64_t sb = 0, se = n;
  def_plan(&sb, &se, 1, ch);
  if (ch.empty()) {
    out.assign(kGzEmpty, kGzEmpty + 20);
  } else {
    std::vector<uint8_t> t(n + 64, 0);
    memcpy(t.data(), raw.data(), n);
    std::vector<uint32_t> m(n + 1, 0);
    const uint32_t nch = (uint32_t)ch.size();
    std::vector<uint32_t> freq((size_t)nch * kDefFreqStride, 0), hdr((size_t)nch * kDefHdrWords, 0);
    std::vector<DefCodes> codes(nch);
    std::vector<DefInfo> info(nch);
    std::vector<uint8_t> scratch((size_t)nch * kDefScratch, 0);
    std::vector<uint16_t> tab((1u << kDefHashBits) * kDefWays);
    for (uint32_t c = 0; c < nch; ++c) {
      const DefChunk& k = ch[c];
      // MATCH, tile by tile as def_match_kernel
      std::fill(tab.begin(), tab.end(), (uint16_t)kDefNoPos);
      for (uint64_t base = k.h; base < k.e; base += kDefTile) {
        uint32_t h[kDefTile];
        bool ok[kDefTile];
        for (uint32_t l = 0; l < kDefTile; ++l) { const uint64_t p = base + l; ok[l] = p + 4 <= k.e; h[l] = ok[l] ? def_hash(t.data(), p) : 0; }
        for (uint32_t l = 0; l < kDefTile; ++l) {
          const uint64_t p = base + l;
          if (p < k.b || p >= k.e) continue;
          uint32_t r = 0;
          if (ok[l]) {
            uint64_t q = kInfNone;
            for (uint32_t j = l; j-- > 0;) if (ok[j] && h[j] == h[l]) { q = base + j; break; }
            r = def_match_at(t.data(), k, p, q, tab.data() + h[l] * kDefWays);
          }
          m[p] = r;
        }
        for (uint32_t l = 0; l < kDefTile; ++l) {
          if (!ok[l]) continue;
          uint16_t* s = tab.data() + h[l] * kDefWays;
          for (uint32_t j = kDefWays - 1; j > 0; --j) s[j] = s[j - 1];
          s[0] = (uint16_t)(base + l - k.h);
        }
      }
    }
    for (uint32_t c = 0; c < nch; ++c) info[c].nsym = def_parse(m.data(), ch[c].b, ch[c].e, t.data(), freq.data() + (size_t)c * kDefFreqStride);   // PARSE
    for (uint32_t c = 0; c < nch; ++c)   // CODE
      def_code(freq.data() + (size_t)c * kDefFreqStride, ch[c].e - ch[c].b, (ch[c].flags & kDefLast) != 0, codes[c], hdr.data() + (size_t)c * kDefHdrWords, info[c]);
    for (uint32_t c = 0; c < nch; ++c) {   // WRITE, lane by lane as def_write_kernel
      const DefChunk& k = ch[c];
      const DefInfo& in = info[c];
      uint8_t* o = scratch.data() + (size_t)c * kDefScratch;
      uint32_t* ow = reinterpret_cast<uint32_t*>(o);
      nstored += in.stored;
      if (!in.stored) {
        for (uint32_t w = 0; w < (in.hdr_bits + 31) / 32; ++w) bo_or(ow + w, hdr[(size_t)c * kDefHdrWords + w]);
        uint64_t pre = 0;
        for (uint32_t lane = 0; lane < 32; ++lane) {
          const uint32_t lo = (uint32_t)((uint64_t)lane * in.nsym / 32), hi = (uint32_t)((uint64_t)(lane + 1) * in.nsym / 32);
          def_write_range(ow, in.hdr_bits + pre, m.data() + k.b, lo, hi, codes[c], lane == 31);
          pre += def_range_bits(m.data() + k.b, lo, hi, codes[c]);
        }
      }
      for (uint32_t lane = 0; lane < 32; ++lane) def_write_tail(o, t.data() + k.b, k.e - k.b, in, (k.flags & kDefLast) != 0, lane, 32);
    }
    // PLACE: header, chunks, trailer (CRC-32 joined from the chunks' CRCs as on the device)
    std::vector<uint32_t> tabc(256);
    for (uint32_t i = 0; i < 256; ++i) tabc[i] = crc_table_entry(i);
    uint32_t crc = 0;
    for (uint32_t i = 0; i < 10; ++i) out.push_back(gz_header_byte(i));
    for (uint32_t c = 0; c < nch; ++c) {
      const uint8_t* o = scratch.data() + (size_t)c * kDefScratch;
      out.insert(out.end(), o, o + info[c].bytes);
      crc = crc_concat(crc, crc_piece(t.data() + ch[c].b, ch[c].e - ch[c].b, tabc.data()), ch[c].e - ch[c].b);
    }
    uint8_t tr[8];
    def_put32(tr, crc); def_put32(tr + 4, (uint32_t)n);
    out.insert(out.end(), tr, tr + 8);
  }
  f = fopen(argv[2], "wb");
  if (!f) return 2;
  fwrite(out.data(), 1, out.size(), f); fclose(f);
  printf("ok bytes %zu chunks %zu stored %u\n", out.size(), ch.size(), nstored);
  return 0;
}
