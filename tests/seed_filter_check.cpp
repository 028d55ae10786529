// Host-side proof obligations for the seed kernel's streaming screen (half_screen, sortmerna_b200/csrc/smr_levbits.h), run by
// tests/test_seed_filter.py.  For P of pw characters and T of pw+1 characters:
//   1. half_screen accepts every T that within_one_edit accepts (a screen that drops a match would change results);
//   2. half_screen(T) && (classify_bits(P, T, pw) & 3) != 0 equals within_one_edit(P, T), which is what the kernel decides
//      with (within_one_edit itself is proven against edit distance by tests/lev_bits_check.cpp).
// Cases: pw = 9 exhaustively (every P, every T within one edit of it, enumerated); for pw = 4..15, every (P, T) pair where
// 4^(2pw+1) is small, and above that every one-edit neighbour of random patterns plus random pairs.
// Prints "pw W cases N neighbours M missed A mismatched B screened S" per pw (S: random pairs that pass the screen, per
// million) and exits non-zero when any A or B is not 0.
#include <cstdio>
#include <cstdlib>
#include <random>
#include "../sortmerna_b200/csrc/smr_levbits.h"

struct Tally { long cases = 0, neighbours = 0, missed = 0, mismatched = 0, rnd = 0, screened = 0; };

static bool screen(uint32_t P, uint32_t T, const smr::HalfMasks& m) { return smr::half_screen(P, P >> 2, P << 2, T, m); }

static void check(uint32_t P, uint32_t T, uint32_t pw, const smr::LevMasks& lm, const smr::HalfMasks& hm, Tally& t) {
  const bool s = screen(P, T, hm), w = smr::within_one_edit(P, T, lm);
  t.cases++;
  if (w && !s) t.missed++;
  if ((s && (smr::classify_bits(P, T, pw) & 3u) != 0u) != w) t.mismatched++;
}

// every text of pw+1 characters one of whose prefixes is within one edit of P: a substitution (or none) in the first pw
// characters with any last character, a deletion with any last two characters, an insertion
template <class F> static void neighbours(uint32_t P, uint32_t pw, F&& f) {
  for (uint32_t j = 0; j < pw; ++j)   // c = p_j: the unedited pattern (pw times over)
    for (uint32_t c = 0; c < 4; ++c) {
      const uint32_t S = (P & ~(3u << (2 * j))) | (c << (2 * j));
      for (uint32_t e = 0; e < 4; ++e) f(S | (e << (2 * pw)));
    }
  for (uint32_t j = 0; j < pw; ++j) {   // deletion of p_j
    const uint32_t low = P & (uint32_t)((1ull << (2 * j)) - 1ull), high = (uint32_t)((uint64_t)P >> (2 * (j + 1)));
    const uint32_t D = low | (high << (2 * j));   // pw-1 characters
    for (uint32_t e = 0; e < 16; ++e) f(D | (e << (2 * (pw - 1))));
  }
  for (uint32_t j = 0; j <= pw; ++j)   // insertion of c before p_j
    for (uint32_t c = 0; c < 4; ++c) {
      const uint32_t low = P & (uint32_t)((1ull << (2 * j)) - 1ull), high = (uint32_t)((uint64_t)P >> (2 * j));
      f(low | (c << (2 * j)) | (uint32_t)((uint64_t)high << (2 * (j + 1))));
    }
}

int main(int argc, char** argv) {
  const long nrand = argc > 1 ? atol(argv[1]) : 2000000;
  std::mt19937_64 rng(20261017);
  long bad = 0;
  for (uint32_t pw = 4; pw <= 15; ++pw) {
    const smr::LevMasks lm = smr::lev_masks(pw);
    const smr::HalfMasks hm = smr::half_masks(pw);
    const uint64_t np = 1ull << (2 * pw), nt = 1ull << (2 * (pw + 1));
    Tally t;
    auto nb = [&](uint32_t P) {
      neighbours(P, pw, [&](uint32_t T) {
        t.neighbours++;
        if (!smr::within_one_edit(P, T, lm)) { t.mismatched++; return; }   // the enumeration itself is wrong
        check(P, T, pw, lm, hm, t);
      });
    };
    if (pw <= 6) {
      for (uint64_t P = 0; P < np; ++P)
        for (uint64_t T = 0; T < nt; ++T) check((uint32_t)P, (uint32_t)T, pw, lm, hm, t);
    }
    if (pw == 9) {
      for (uint64_t P = 0; P < np; ++P) nb((uint32_t)P);
    } else if (pw > 6) {
      for (long i = 0; i < nrand / 64; ++i) nb((uint32_t)(rng() & (np - 1)));
    }
    for (long i = 0; i < nrand; ++i) {   // random pairs: how much the screen lets through
      const uint32_t P = (uint32_t)(rng() & (np - 1)), T = (uint32_t)(rng() & (nt - 1));
      check(P, T, pw, lm, hm, t);
      t.rnd++;
      t.screened += screen(P, T, hm) ? 1 : 0;
    }
    printf("pw %u cases %ld neighbours %ld missed %ld mismatched %ld screened %ld\n", pw, t.cases, t.neighbours, t.missed,
           t.mismatched, t.rnd ? (long)(1e6 * (double)t.screened / (double)t.rnd) : 0L);
    bad += t.missed + t.mismatched;
  }
  return bad ? 1 : 0;
}
