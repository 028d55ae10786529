// Number formatting of the report writer (smr_report.cuh), shared by the kernels and the host-side checker of the tests
// (tests/report_fmt_check.cpp compiles this header with g++ and compares it with snprintf).
//
// The reference prints its numbers through std::stringstream: integers as %u / %d, and the floating-point BLAST columns (%id, E-value,
// %qcov) after ss.precision(3) in the default float field, which is exactly C's "%.3g" of the double (report_blast.cpp:306-342).
// fmt_g3 reproduces that correctly rounded (round-half-even on the exact binary value, as glibc does):
//   1. the decimal exponent e of x is estimated from its binary exponent and x is scaled to y = x * 10^(2-e) in [100, 1000) with at
//      most 16 correctly rounded double operations (relative error below 2e-15, absolute error on y below 2e-12);
//   2. the three digits are round(y) unless y lies within 1e-9 of a rounding half, where the scaled value cannot decide.  Then x is
//      compared with the half-way point (2N+1)/2 * 10^(e-2) exactly, in integers: x = m*2^q, so both sides are products of m or 2N+1
//      with powers of 2 and 5 (at most ~820 bits for any double, BigInt below).
// No exp, log or pow is evaluated, so host and device give the same bytes.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#endif
#ifndef __device__
#define __device__
#endif
#endif

namespace smr {
namespace fmt {

__host__ __device__ inline int put_u64(char* o, uint64_t v) {
  char t[20];
  int n = 0;
  do { t[n++] = (char)('0' + v % 10); v /= 10; } while (v);
  for (int i = 0; i < n; ++i) o[i] = t[n - 1 - i];
  return n;
}
__host__ __device__ inline int put_i64(char* o, int64_t v) {
  if (v < 0) { o[0] = '-'; return 1 + put_u64(o + 1, 0ull - (uint64_t)v); }
  return put_u64(o, (uint64_t)v);
}

// unsigned big integer, little-endian 32-bit limbs: only what the near-tie comparison needs
struct BigInt {
  static constexpr int kLimbs = 40;   // 1280 bits; the largest operand of fmt_g3 has ~820
  uint32_t w[kLimbs];
  int n;
  __host__ __device__ explicit BigInt(uint64_t v) : n(0) {
    for (int i = 0; i < kLimbs; ++i) w[i] = 0;
    while (v) { w[n++] = (uint32_t)v; v >>= 32; }
  }
  __host__ __device__ void mul(uint32_t f) {
    uint64_t c = 0;
    for (int i = 0; i < n; ++i) { const uint64_t t = (uint64_t)w[i] * f + c; w[i] = (uint32_t)t; c = t >> 32; }
    if (c) w[n++] = (uint32_t)c;
  }
  __host__ __device__ void mul_pow5(int k) {
    for (; k >= 13; k -= 13) mul(1220703125u);   // 5^13
    uint32_t f = 1;
    for (; k > 0; --k) f *= 5;
    if (f > 1) mul(f);
  }
  __host__ __device__ void shl(int bits) {
    if (n == 0 || bits <= 0) return;
    const int limbs = bits / 32, b = bits % 32;
    for (int i = n - 1 + limbs + 1; i >= 0; --i) {
      const int s = i - limbs;
      const uint32_t hi = (s >= 0 && s < n) ? w[s] : 0u, lo = (s - 1 >= 0 && s - 1 < n) ? w[s - 1] : 0u;
      w[i] = b ? (hi << b) | (lo >> (32 - b)) : hi;
    }
    n += limbs + 1;
    while (n > 0 && w[n - 1] == 0) --n;
  }
};
__host__ __device__ inline int cmp(const BigInt& a, const BigInt& b) {
  if (a.n != b.n) return a.n < b.n ? -1 : 1;
  for (int i = a.n - 1; i >= 0; --i)
    if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
  return 0;
}

// sign of m*2^q - (2h+1)/2 * 10^d, exactly
__host__ __device__ inline int cmp_half(uint64_t m, int q, uint32_t h, int d) {
  int a2 = q + 1, a5 = 0, b2 = d, b5 = d;   // 2x = m*2^(q+1);  (2h+1) * 10^d = (2h+1) * 2^d * 5^d
  if (b5 < 0) { a5 = -b5; b5 = 0; }
  const int k = a2 < b2 ? a2 : b2;
  a2 -= k; b2 -= k;
  BigInt A(m), B(2ull * h + 1);
  A.mul_pow5(a5); A.shl(a2);
  B.mul_pow5(b5); B.shl(b2);
  return cmp(A, B);
}

__host__ __device__ inline double scale10(double y, int k) {   // y * 10^k by correctly rounded steps (10^0..10^22 are exact doubles)
  for (; k >= 22; k -= 22) y *= 1e22;
  for (; k <= -22; k += 22) y /= 1e22;
  double p = 1.0;
  for (int i = 0; i < (k < 0 ? -k : k); ++i) p *= 10.0;
  return k < 0 ? y / p : y * p;
}

__host__ __device__ inline uint64_t dbl_bits(double x) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(x);
#else
  uint64_t b;
  memcpy(&b, &x, 8);
  return b;
#endif
}

// printf("%.3g", x) into o (at most 12 bytes: "-1.23e-308" is the longest); returns the length
__host__ __device__ inline int fmt_g3(double x, char* o) {
  uint64_t bits = dbl_bits(x);
  int len = 0;
  if (bits >> 63) { o[len++] = '-'; bits &= ~(1ull << 63); x = -x; }
  const int ef = (int)(bits >> 52) & 0x7FF;
  const uint64_t frac = bits & ((1ull << 52) - 1);
  if (ef == 0x7FF) {
    o[len] = frac ? 'n' : 'i'; o[len + 1] = frac ? 'a' : 'n'; o[len + 2] = frac ? 'n' : 'f';
    return len + 3;
  }
  if (ef == 0 && frac == 0) { o[len++] = '0'; return len; }
  const uint64_t m = ef ? frac | (1ull << 52) : frac;
  const int q = ef ? ef - 1075 : -1074;
  int b2 = q + 63;   // floor(log2 x)
  while (!(m >> (b2 - q))) --b2;
  int e = (int)floor(b2 * 0.30102999566398120);   // within one of floor(log10 x); the loop below settles it
  double y = scale10(x, 2 - e);
  for (int it = 0; it < 3 && (y < 100.0 || y >= 1000.0); ++it) {
    e += y < 100.0 ? -1 : 1;
    y = scale10(x, 2 - e);
  }
  uint32_t n0 = (uint32_t)y;   // y in [~100, ~1000]
  const double f = y - (double)n0;
  uint32_t n;
  if (f - 0.5 < 1e-9 && 0.5 - f < 1e-9) {
    const int c = cmp_half(m, q, n0, e - 2);
    n = c > 0 ? n0 + 1 : c < 0 ? n0 : n0 + (n0 & 1);
  } else {
    n = f > 0.5 ? n0 + 1 : n0;
  }
  if (n >= 1000) { n /= 10; ++e; }   // 999.5 -> 1.00e(e+1)
  if (n < 100) { n *= 10; --e; }     // an estimate just below 100 that did not round up cannot happen; kept for safety
  char dg[3] = {(char)('0' + n / 100), (char)('0' + n / 10 % 10), (char)('0' + n % 10)};
  int nd = 3;
  while (nd > 1 && dg[nd - 1] == '0') --nd;   // %g strips trailing zeros
  if (e < -4 || e >= 3) {
    o[len++] = dg[0];
    if (nd > 1) { o[len++] = '.'; for (int i = 1; i < nd; ++i) o[len++] = dg[i]; }
    o[len++] = 'e';
    o[len++] = e < 0 ? '-' : '+';
    const int ae = e < 0 ? -e : e;
    if (ae < 10) o[len++] = '0';
    len += put_u64(o + len, (uint64_t)ae);
  } else if (e >= 0) {   // integer part = the first e+1 digits
    for (int i = 0; i <= e; ++i) o[len++] = dg[i];
    if (nd > e + 1) { o[len++] = '.'; for (int i = e + 1; i < nd; ++i) o[len++] = dg[i]; }
  } else {
    o[len++] = '0'; o[len++] = '.';
    for (int i = 0; i < -e - 1; ++i) o[len++] = '0';
    for (int i = 0; i < nd; ++i) o[len++] = dg[i];
  }
  return len;
}

// BAM's fields of a SAM row (the BAM writer of smr_report.cuh; tests/bgzf_check.cpp prints them for the host test)
// the BAI bin of the 0-based region [beg, end) (SAMv1 5.3, reg2bin)
__host__ __device__ inline uint32_t bam_reg2bin(int64_t beg, int64_t end) {
  --end;
  if (beg >> 14 == end >> 14) return ((1u << 15) - 1) / 7 + (uint32_t)(beg >> 14);
  if (beg >> 17 == end >> 17) return ((1u << 12) - 1) / 7 + (uint32_t)(beg >> 17);
  if (beg >> 20 == end >> 20) return ((1u << 9) - 1) / 7 + (uint32_t)(beg >> 20);
  if (beg >> 23 == end >> 23) return ((1u << 6) - 1) / 7 + (uint32_t)(beg >> 23);
  if (beg >> 26 == end >> 26) return ((1u << 3) - 1) / 7 + (uint32_t)(beg >> 26);
  return 0;
}
// the 4-bit code ("=ACMGRSVTWYHKDBN") of a letter SAM's SEQ prints (A, C, G, T, N)
__host__ __device__ inline uint32_t bam_nt4(char c) { return c == 'A' ? 1 : c == 'C' ? 2 : c == 'G' ? 4 : c == 'T' ? 8 : 15; }
// the bytes and the type htslib gives a SAM ":i:" value v >= 0: 'C' up to 255, 'S' up to 65535, 'I' above
__host__ __device__ inline uint32_t bam_int_bytes(uint64_t v) { return v <= 0xFF ? 1 : v <= 0xFFFF ? 2 : 4; }
__host__ __device__ inline char bam_int_type(uint32_t bytes) { return bytes == 1 ? 'C' : bytes == 2 ? 'S' : 'I'; }

// The coordinate-sorted BAM (smr_bamsort.cuh; tests/bamsort_check.cpp prints these for the host test)
// samtools' coordinate key of a record: refID, then pos + 1, then the reverse-strand bit
__host__ __device__ inline uint64_t bam_sort_key(int32_t ref_id, int32_t pos, uint32_t flag) {
  return (uint64_t)(uint32_t)ref_id << 32 | (uint64_t)(uint32_t)(pos + 1) << 1 | ((flag & 16) ? 1u : 0u);
}
// BGZF's virtual offset: the compressed offset of a block, and the offset inside its uncompressed bytes
__host__ __device__ inline uint64_t bam_voffset(uint64_t coffset, uint32_t in_block) { return coffset << 16 | in_block; }
// htslib's merge_chunks rule: a chunk that starts in the block where the previous one (in ascending vbeg) ends joins it
__host__ __device__ inline bool bam_chunks_merge(uint64_t prev_vend, uint64_t vbeg) { return prev_vend >> 16 == vbeg >> 16; }

}  // namespace fmt
}  // namespace smr
