// Host-side run of the BGZF framing of BAM (sortmerna_b200/csrc/smr_deflate.h): the input cut into blocks (bgzf_blocks), each block
// compressed by the MATCH / PARSE / CODE / WRITE / PLACE steps the CUDA kernels perform (smr_deflate.cuh), serially as
// tests/deflate_check.cpp runs them, behind the header PLACE writes (bgzf_header).  Also prints BAM's field helpers of smr_fmt.h.
// tests/test_bam_host.py checks both.
//   bgzf_check blocks in.bin out.bgzf   -> the BGZF blocks of the input; prints "ok bytes N blocks B max_member M"
//   bgzf_check fields                   -> one line per case: "bin beg end value", "nt4 letter value", "int value bytes type"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../sortmerna_b200/csrc/smr_deflate.h"
#include "../sortmerna_b200/csrc/smr_fmt.h"
using namespace smr;

static int fields() {
  const int64_t pts[] = {0, 1, 16383, 16384, 16385, 131071, 131072, 1048575, 1048576, 8388607, 8388608, 67108863, 67108864, 536870911};
  for (int64_t b : pts)
    for (int64_t len : {1, 2, 100, 16384, 131072, 1048576, 8388608, 67108864})
      if (b + len <= (1ll << 29)) printf("bin %lld %lld %u\n", (long long)b, (long long)(b + len), fmt::bam_reg2bin(b, b + len));
  for (char c : {'A', 'C', 'G', 'T', 'N'}) printf("nt4 %c %u\n", c, fmt::bam_nt4(c));
  for (uint64_t v : {0ull, 1ull, 255ull, 256ull, 65535ull, 65536ull, 4294967295ull}) {
    const uint32_t n = fmt::bam_int_bytes(v);
    printf("int %llu %u %c\n", (unsigned long long)v, n, fmt::bam_int_type(n));
  }
  return 0;
}

int main(int argc, char** argv) {
  if (argc == 2 && !strcmp(argv[1], "fields")) return fields();
  if (argc < 4 || strcmp(argv[1], "blocks")) return 2;
  FILE* f = fopen(argv[2], "rb");
  if (!f) return 2;
  std::vector<uint8_t> raw;
  { uint8_t buf[65536]; size_t k; while ((k = fread(buf, 1, sizeof buf, f)) > 0) raw.insert(raw.end(), buf, buf + k); fclose(f); }
  const uint64_t n = raw.size();
  std::vector<uint64_t> sb, se;
  bgzf_blocks(0, n, sb, se);
  std::vector<DefChunk> ch;
  def_plan(sb.data(), se.data(), (uint32_t)sb.size(), ch);
  std::vector<uint8_t> t(n + 64, 0);
  memcpy(t.data(), raw.data(), n);
  std::vector<uint32_t> m(n + 1, 0);
  const uint32_t nch = (uint32_t)ch.size();
  std::vector<uint32_t> freq((size_t)nch * kDefFreqStride, 0), hdr((size_t)nch * kDefHdrWords, 0);
  std::vector<DefCodes> codes(nch);
  std::vector<DefInfo> info(nch);
  std::vector<uint8_t> scratch((size_t)nch * kDefScratch, 0);
  std::vector<uint16_t> tab((1u << kDefHashBits) * kDefWays);
  for (uint32_t c = 0; c < nch; ++c) {   // MATCH, tile by tile as def_match_kernel
    const DefChunk& k = ch[c];
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
  // PLACE: per block the BGZF header with its BSIZE, the block's chunks, the trailer (CRC-32 joined from the chunks' CRCs)
  std::vector<uint32_t> tabc(256);
  for (uint32_t i = 0; i < 256; ++i) tabc[i] = crc_table_entry(i);
  std::vector<uint8_t> out;
  uint64_t max_member = 0;
  uint32_t c = 0;
  for (uint32_t b = 0; b < sb.size(); ++b) {
    const size_t at = out.size();
    out.resize(at + kBgzfHeader);
    uint32_t crc = 0;
    for (; c < nch && ch[c].stream == b; ++c) {
      const uint8_t* o = scratch.data() + (size_t)c * kDefScratch;
      out.insert(out.end(), o, o + info[c].bytes);
      crc = crc_concat(crc, crc_piece(t.data() + ch[c].b, ch[c].e - ch[c].b, tabc.data()), ch[c].e - ch[c].b);
    }
    uint8_t tr[8];
    def_put32(tr, crc); def_put32(tr + 4, (uint32_t)(se[b] - sb[b]));
    out.insert(out.end(), tr, tr + 8);
    bgzf_header(&out[at], (uint32_t)(out.size() - at));
    max_member = std::max<uint64_t>(max_member, out.size() - at);
  }
  f = fopen(argv[3], "wb");
  if (!f) return 2;
  fwrite(out.data(), 1, out.size(), f); fclose(f);
  printf("ok bytes %zu blocks %zu max_member %llu bound %u\n", out.size(), sb.size(), (unsigned long long)max_member, kBgzfMaxMember);
  return 0;
}
