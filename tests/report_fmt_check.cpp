// CPU checker of the report writer's number formatting (sortmerna_b200/csrc/smr_fmt.h) against the C library's printf.
//   report_fmt_check ratios      every 100*m/(m+k), m+k <= 4096, and every 100*a/L, L <= 30000 (the %id and %qcov columns)
//   report_fmt_check random N S  N doubles with uniformly random bit patterns (every exponent, subnormals), seed S
//   report_fmt_check bounds      the neighbours of every rounding half d.dd5 * 10^e, e in [-320, 308]
//   report_fmt_check special     0, subnormals, powers of ten and their neighbours, the largest double, inf; and %u / %d
// Prints "ok <values checked>" or the first mismatches; exit status 1 on any mismatch.
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <thread>
#include <vector>

#include "../sortmerna_b200/csrc/smr_fmt.h"

static std::atomic<uint64_t> g_checked{0}, g_bad{0};

static bool check(double x) {
  char a[64], b[64];
  const int n = smr::fmt::fmt_g3(x, a);
  a[n] = 0;
  snprintf(b, sizeof b, "%.3g", x);
  if (strcmp(a, b) != 0) {
    if (g_bad.fetch_add(1) < 20) printf("mismatch %.17g (%a): got %s want %s\n", x, x, a, b);
    return false;
  }
  return true;
}

template <class F>
static void parallel(uint64_t n, F f) {
  const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
  std::vector<std::thread> th;
  for (unsigned t = 0; t < nt; ++t)
    th.emplace_back([&, t] {
      uint64_t c = 0;
      for (uint64_t i = t; i < n; i += nt) c += f(i);
      g_checked += c;
    });
  for (auto& x : th) x.join();
}

int main(int argc, char** argv) {
  const std::string mode = argc > 1 ? argv[1] : "";
  if (mode == "ratios") {
    parallel(4097, [](uint64_t tot) {   // (double)n_match / n_tot * 100 (read.cpp:587, report_blast.cpp:308)
      uint64_t c = 0;
      for (uint64_t m = 0; tot && m <= tot; ++m, ++c) check((double)m / (double)tot * 100);
      return c;
    });
    parallel(30001, [](uint64_t L) {   // (double)abs(aligned length) / readlen * 100 (read.cpp:588, report_blast.cpp:341)
      uint64_t c = 0;
      for (uint64_t a = 0; L && a <= L; ++a, ++c) check((double)a / (double)L * 100);
      return c;
    });
  } else if (mode == "random") {
    const uint64_t n = argc > 2 ? strtoull(argv[2], nullptr, 10) : 10000000, seed = argc > 3 ? strtoull(argv[3], nullptr, 10) : 1;
    parallel(64, [&](uint64_t t) {
      std::mt19937_64 rng(seed * 1000003 + t);
      uint64_t c = 0;
      for (uint64_t i = t; i < n; i += 64, ++c) {
        uint64_t b = rng();
        double x;
        memcpy(&x, &b, 8);
        if (std::isnan(x)) x = std::ldexp((double)(b >> 12), -1074);   // "nan" vs "-nan" is not a value the writer prints
        check(x);
      }
      return c;
    });
  } else if (mode == "bounds") {
    parallel(629, [](uint64_t k) {
      const int e = (int)k - 320;
      uint64_t c = 0;
      for (int d = 100; d <= 999; ++d) {
        char s[48];
        snprintf(s, sizeof s, "%d.%02d5e%d", d / 100, d % 100, e);
        const double h = strtod(s, nullptr);
        double lo = h, hi = h;
        for (int j = 0; j < 3; ++j) { c += 2; check(lo); check(hi); lo = std::nextafter(lo, 0.0); hi = std::nextafter(hi, INFINITY); }
        c += check(-h);
      }
      return c;
    });
  } else if (mode == "special") {
    std::vector<double> v = {0.0, -0.0, INFINITY, -INFINITY, 5e-324, 1e-323, 2.2250738585072009e-308, 2.2250738585072014e-308, 1.7976931348623157e308,
                             0.5, 1.0, 1.125, 1.375, 0.125, 100.0, 999.5, 99.95, 9.995, 0.0001, 0.00001, 1e-5, 123456789.0, 0.1, 0.2, 0.3};
    for (int k = 1; k < 64; ++k) v.push_back(std::ldexp(1.0, -1074 + k * 16));
    for (int e = -324; e <= 308; ++e) {
      char s[32];
      snprintf(s, sizeof s, "1e%d", e);
      const double p = strtod(s, nullptr);
      v.push_back(p); v.push_back(std::nextafter(p, 0.0)); v.push_back(std::nextafter(p, INFINITY));
    }
    for (double x : v) { check(x); ++g_checked; }
    const uint64_t ints[] = {0, 1, 9, 10, 99, 100, 65535, 4294967295ull, 18446744073709551615ull};
    for (uint64_t u : ints) {
      char a[32], b[32];
      a[smr::fmt::put_u64(a, u)] = 0;
      snprintf(b, sizeof b, "%llu", (unsigned long long)u);
      if (strcmp(a, b)) { printf("mismatch %%u %s %s\n", a, b); ++g_bad; }
      const int64_t i = -(int64_t)(u >> 1);
      a[smr::fmt::put_i64(a, i)] = 0;
      snprintf(b, sizeof b, "%lld", (long long)i);
      if (strcmp(a, b)) { printf("mismatch %%d %s %s\n", a, b); ++g_bad; }
      g_checked += 2;
    }
  } else {
    fprintf(stderr, "usage: %s ratios | random N SEED | bounds | special\n", argv[0]);
    return 2;
  }
  if (g_bad) { printf("%llu mismatches in %llu values\n", (unsigned long long)g_bad.load(), (unsigned long long)g_checked.load()); return 1; }
  printf("ok %llu\n", (unsigned long long)g_checked.load());
  return 0;
}
