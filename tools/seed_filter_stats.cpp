// The seed kernel's entry stream (coop_stream, sortmerna_b200/csrc/smr_seed.cuh) replayed on the host for one flattened
// index part, to count what the streaming screen lets through.  Run by tools/seed_filter_stats.py:
//   seed_filter_stats <flookup.u32> <flist.u32> <reads.u8> <read_len> <lnwin> <step>
// reads.u8: reads of read_len bases in the 0..3 alphabet, back to back.  Windows, rounds, lists and chunks as the kernel walks
// them: positions q*step, forward strand then reverse complement, 32 windows per round, every forward list of a round then
// every mirror list, eight entries per chunk, 32 chunks per step.  Prints one line of counts:
//   windows W rounds R entries E chunk_entries C survivors S matches M classify_passes K flushes F flushes_before B
// E: list entries; C: entries streamed, chunk padding included; K / F: classify passes and flushes of the buffer as coop_stream
// runs them now; B: flushes when only matches were buffered (the stream before the screen).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>
#include "../sortmerna_b200/csrc/smr_levbits.h"

template <class T> static std::vector<T> slurp(const char* p) {
  std::ifstream f(p, std::ios::binary);
  std::vector<char> b((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  std::vector<T> v(b.size() / sizeof(T));
  if (!v.empty()) memcpy(v.data(), b.data(), v.size() * sizeof(T));
  return v;
}

static uint32_t rev_chars(uint32_t v, uint32_t pw) {  // first character most significant -> lowest
  uint32_t x = 0;
  for (uint32_t i = 0; i < pw; ++i) x |= ((v >> (2 * (pw - 1 - i))) & 3u) << (2 * i);
  return x;
}

int main(int argc, char** argv) {
  if (argc < 7) return 2;
  const auto lk = slurp<uint32_t>(argv[1]);
  const auto fl = slurp<uint32_t>(argv[2]);   // (text, id) pairs
  const auto rd = slurp<uint8_t>(argv[3]);
  const uint32_t len = (uint32_t)atoi(argv[4]), L = (uint32_t)atoi(argv[5]), step = (uint32_t)atoi(argv[6]), pw = L / 2;
  const size_t nreads = rd.size() / len;
  const int kCap = 384, kStep = 256;
  const smr::HalfMasks hm = smr::half_masks(pw);
  auto text = [&](size_t i) { return i < fl.size() / 2 ? fl[2 * i] : 0u; };
  unsigned long long windows = 0, rounds = 0, entries = 0, chunk_entries = 0, surv = 0, match = 0, passes = 0, flushes = 0,
                     flushes_before = 0;
  const uint32_t npos = (len - L) / step + 1;
  struct List { uint32_t off, cnt, P; };
  for (size_t r = 0; r < nreads; ++r) {
    const uint8_t* s = rd.data() + r * len;
    const uint32_t nq = 2 * npos;
    for (uint32_t q0 = 0; q0 < nq; q0 += 32) {
      std::vector<List> lists[2];
      for (uint32_t q = q0; q < q0 + 32 && q < nq; ++q) {
        const uint32_t var = q / npos, p = (q % npos) * step;
        uint64_t V = 0;
        for (uint32_t i = 0; i < L; ++i) V = (V << 2) | (var ? 3u - s[len - p - 1 - i] : s[p + i]);
        const uint32_t keyf = (uint32_t)(V >> (2 * pw)), keyr = (uint32_t)(V & ((1ull << (2 * pw)) - 1));
        lists[0].push_back({lk[4 * (size_t)keyf], lk[4 * (size_t)keyf + 1], rev_chars(keyr, pw)});
        lists[1].push_back({lk[4 * (size_t)keyr + 2], lk[4 * (size_t)keyr + 3], keyf});
        ++windows;
      }
      ++rounds;
      // per stream chunk: survivors and matches
      std::vector<uint32_t> cs, cm;
      for (int h = 0; h < 2; ++h)
        for (const List& l : lists[h]) {
          if (!l.cnt) continue;
          entries += l.cnt;
          const uint32_t P = l.P;
          for (uint32_t g = l.off >> 3; g < (l.off + l.cnt + 7) >> 3; ++g) {
            uint32_t ns = 0, nm = 0;
            for (uint32_t i = 8 * g; i < 8 * g + 8; ++i) {
              if (i < l.off || i >= l.off + l.cnt) continue;
              const uint32_t T = text(i);
              if (!smr::half_screen(P, P >> 2, P << 2, T, hm)) continue;
              ++ns;
              nm += (smr::classify_bits(P, T, pw) & 3u) ? 1u : 0u;
            }
            cs.push_back(ns); cm.push_back(nm);
          }
        }
      chunk_entries += 8ull * cs.size();
      uint32_t nacc = 0, ncls = 0, nbuf = 0, nold = 0;
      for (size_t e0 = 0; e0 < cs.size(); e0 += 32) {
        const bool last = e0 + 32 >= cs.size();
        for (size_t e = e0; e < e0 + 32 && e < cs.size(); ++e) { nacc += cs[e]; nbuf += cm[e]; nold += cm[e]; surv += cs[e]; match += cm[e]; }
        if (nacc > ncls && (nacc > (uint32_t)(kCap - kStep) || last)) { ++passes; nacc = ncls = nbuf; }
        if (nacc && (nacc > (uint32_t)(kCap - kStep) || last)) { ++flushes; nacc = ncls = nbuf = 0; }
        if (nold && (nold > (uint32_t)(kCap - kStep) || last)) { ++flushes_before; nold = 0; }
      }
    }
  }
  printf("windows %llu rounds %llu entries %llu chunk_entries %llu survivors %llu matches %llu classify_passes %llu flushes %llu "
         "flushes_before %llu\n", windows, rounds, entries, chunk_entries, surv, match, passes, flushes, flushes_before);
  return 0;
}
