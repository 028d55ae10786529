// Bit-parallel "within one edit" predicates on 2-bit packed strings (first character in the lowest two
// bits).  Shared by the CUDA kernels and by the host-side check tests/lev_bits_check.cpp, which proves
// them equal to (a) dynamic-programming edit distance and (b) the reference's table-driven universal
// Levenshtein automaton (traverse_bursttrie.cpp:68-98) on millions of random cases.
#pragma once
#include <cstdint>
#if defined(__CUDACC__)
#define SMR_HD __host__ __device__ __forceinline__
#else
#define SMR_HD inline
#endif

namespace smr {

SMR_HD uint32_t lb_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__popc(x);
#else
  return (uint32_t)__builtin_popcount(x);
#endif
}
SMR_HD int32_t lb_ctz(uint32_t x) {  // x != 0
#if defined(__CUDA_ARCH__)
  return __ffs((int)x) - 1;
#else
  return __builtin_ctz(x);
#endif
}
SMR_HD int32_t lb_clz(uint32_t x) {  // x != 0
#if defined(__CUDA_ARCH__)
  return __clz((int)x);
#else
  return __builtin_clz(x);
#endif
}

SMR_HD uint32_t neq2(uint32_t x) { return (x | (x >> 1)) & 0x55555555u; }        // bit 2i set iff character i differs
SMR_HD uint32_t mk2(uint32_t k) { return ((1u << (2 * k)) - 1u) & 0x55555555u; }  // the first k characters (k < 16)
SMR_HD int32_t firstmis(uint32_t m, int32_t dflt) { return m ? (lb_ctz(m) >> 1) : dflt; }
SMR_HD int32_t lastmis(uint32_t m) { return m ? ((31 - lb_clz(m)) >> 1) : -1; }

// P: pattern of pw characters; T: text of pw+1 characters.
// code bits [1:0]: first text length at which T is within one edit of P: 0 none, 1 -> pw-1 chars (one deletion),
//                  2 -> pw chars (at most one substitution), 3 -> pw+1 chars (one insertion)
// code bit 2:      the first pw characters of T equal P
SMR_HD uint32_t classify_bits(uint32_t P, uint32_t T, uint32_t pw) {
  const uint32_t A = neq2(T ^ P), B = neq2(T ^ (P >> 2)), C = neq2((T >> 2) ^ P);
  const uint32_t A9 = A & mk2(pw), A8 = A & mk2(pw - 1), B8 = B & mk2(pw - 1), C9 = C & mk2(pw);
  const bool acc7 = lastmis(B8) < firstmis(A8, (int32_t)pw - 1);
  const bool acc8 = lb_popc(A9) <= 1;
  const bool acc9 = lastmis(C9) < firstmis(A9, (int32_t)pw);
  return (acc7 ? 1u : (acc8 ? 2u : (acc9 ? 3u : 0u))) | (A9 == 0 ? 4u : 0u);
}
// The streaming test of the seed kernel: (classify_bits(P, T, pw) & 3) != 0 in ~20 integer instructions, no clz / ffs.
// "every mismatch of the shifted alignment lies before the first mismatch of the straight one" is an unsigned
// comparison against the lowest set bit (a sentinel bit stands for "no mismatch").
struct LevMasks { uint32_t m9, m8, s9, s8; };
SMR_HD LevMasks lev_masks(uint32_t pw) { return LevMasks{mk2(pw), mk2(pw - 1), 1u << (2 * pw), 1u << (2 * (pw - 1))}; }
SMR_HD bool within_one_edit(uint32_t P, uint32_t T, const LevMasks& k) {
  const uint32_t x = T ^ P, y = T ^ (P >> 2), z = (T >> 2) ^ P;
  const uint32_t A9 = (x | (x >> 1)) & k.m9, B8 = (y | (y >> 1)) & k.m8, C9 = (z | (z >> 1)) & k.m9;
  const uint32_t a8 = (A9 & k.m8) | k.s8, a9 = A9 | k.s9;
  return ((A9 & (A9 - 1u)) == 0u) | (B8 < (a8 & (0u - a8))) | (C9 < (a9 & (0u - a9)));
}
// The streaming screen of the seed kernel, about half the instructions of within_one_edit.  With h = pw/2, a text within
// one edit of P (an edit at position j, or none) passes at least one of four exact comparisons:
//   lo:  t_i = p_i     for i in [0, h)       no edit, or an edit at j >= h
//   hi:  t_i = p_i     for i in [h, pw)      substitution at j < h
//   del: t_i = p_{i+1} for i in [h, pw-1)    deletion at j < h
//   ins: t_{i+1} = p_i for i in [h, pw)      insertion at j < h
// each one masked XOR tested against zero, with P, P >> 2 and P << 2 (the shifted patterns are computed once per pattern).
// It only screens: some texts that pass are not within one edit, and (classify_bits & 3) != 0 decides
// (tests/seed_filter_check.cpp proves both on every pw the flattener accepts).
struct HalfMasks { uint32_t lo, hi, del, ins; };
SMR_HD uint32_t char_bits(uint32_t a, uint32_t b) {  // the bits of characters [a, b), 0 <= a <= b <= 16 (b = 16: no 32-bit shift)
  return (uint32_t)((1ull << (2 * b)) - 1ull) & ~(uint32_t)((1ull << (2 * a)) - 1ull);
}
SMR_HD HalfMasks half_masks(uint32_t pw) {
  const uint32_t h = pw / 2;
  return HalfMasks{char_bits(0, h), char_bits(h, pw), char_bits(h, pw - 1), char_bits(h + 1, pw + 1)};
}
// Pd = P >> 2, Pi = P << 2
SMR_HD bool half_screen(uint32_t P, uint32_t Pd, uint32_t Pi, uint32_t T, const HalfMasks& m) {
  const uint32_t x = T ^ P;
  return ((x & m.lo) == 0u) | ((x & m.hi) == 0u) | (((T ^ Pd) & m.del) == 0u) | (((T ^ Pi) & m.ins) == 0u);
}
// is the k-character prefix of T within one edit of SOME prefix of P (the automaton is not in its dead state)?  1 <= k <= pw-1
SMR_HD bool viable_bits(uint32_t P, uint32_t T, uint32_t k) {
  const uint32_t Ak = neq2(T ^ P) & mk2(k);
  if (lb_popc(Ak) <= 1) return true;
  const int32_t a = firstmis(Ak, (int32_t)k);
  if (lastmis(neq2(T ^ (P >> 2)) & mk2(k)) < a) return true;
  return lastmis(neq2((T >> 2) ^ P) & mk2(k - 1)) < a;
}

}  // namespace smr
