// Host-side run of the read stream's two passes, with the functions the kernels use:
//   stream_check inflate in.gz out.bin piece_bytes  -> the resumable inflate of smr_inflate.h, one round per pushed piece, as
//                                                     inflate_round in smr_capi.cu runs it; prints "ok bytes N rounds R" or
//                                                     "error <status> piece <k>"
//   stream_check count in.txt piece_bytes           -> the count pass of smr_stream.h over the pieces; prints "reads length min max"
// tests/test_stream_host.py compares them with zlib and with a Python restatement of the reference's count_reads_parallel.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "../sortmerna_b200/csrc/smr_inflate.h"
#include "../sortmerna_b200/csrc/smr_stream.h"
using namespace smr;

static std::vector<uint8_t> slurp(const char* path) {
  std::vector<uint8_t> raw;
  FILE* f = fopen(path, "rb");
  if (!f) exit(2);
  uint8_t buf[65536]; size_t k;
  while ((k = fread(buf, 1, sizeof buf, f)) > 0) raw.insert(raw.end(), buf, buf + k);
  fclose(f);
  return raw;
}

struct HostStream { InfResume at; InfCarry carry; uint32_t members = 0; std::vector<uint8_t> window = std::vector<uint8_t>(kInfWindow, 0); };

// one round over tail (the resume point at st.at.bit); appends the bytes it keeps to out; returns 0 or an InfStatus
static uint32_t round_host(const std::vector<uint8_t>& tail, bool eof, HostStream& st, std::vector<uint8_t>& out) {
  const uint64_t nbytes = tail.size(), nbits = nbytes * 8;
  const uint64_t CH = std::min<uint64_t>(65536, std::max<uint64_t>(8192, nbytes / 8192));
  std::vector<uint32_t> w((nbytes + 64 + 3) / 4 + 1, 0);
  memcpy(w.data(), tail.data(), nbytes);
  std::vector<uint64_t> cand;
  for (uint64_t c = CH; c < nbytes; c += CH) {
    const uint64_t end = std::min(nbits, (c + CH) * 8);
    for (uint64_t p = c * 8; p < end; ++p) if (inf_probe_block(w.data(), nbits, p)) { if (p > st.at.bit) cand.push_back(p); break; }
  }
  const uint32_t ns = (uint32_t)cand.size() + 1;
  std::vector<SpanResult> res(ns);
  HuffTabs T;
  const bool at_member = st.at.at_member;
  const uint64_t start = st.at.bit, prior = at_member ? kInfNone : st.carry.len;
  for (uint32_t i = 0; i < ns; ++i)
    inflate_span<false>(w.data(), nbytes, i ? cand[i - 1] : start, i == 0 && at_member, cand.data(), (uint32_t)cand.size(), i, T, nullptr, 0, nullptr, res[i],
                        i == 0 ? prior : kInfNone);
  std::vector<uint32_t> real(ns); std::vector<uint64_t> off(ns);
  uint32_t nreal = 0, why = 0;
  InfResume next;
  const uint64_t total = inf_chain(cand.data(), (uint32_t)cand.size(), res.data(), real.data(), off.data(), nreal, &why, eof, nbits, at_member, &next);
  if (total == kInfNone) {
    if (at_member && st.members && res[0].status == kInfErrMember) { st.at.eos = true; return 0; }
    return why;
  }
  std::vector<uint64_t> keep(nreal);
  uint64_t nsym = 0;
  for (uint32_t k = 0; k < nreal; ++k) { keep[k] = res[real[k]].out_n; nsym = std::max(nsym, off[k] + keep[k]); }
  keep[nreal - 1] = next.keep_last;
  std::vector<uint16_t> sym(nsym + 1);
  std::vector<MemberEnd> ends;
  for (uint32_t k = 0; k < nreal; ++k) {
    const uint32_t i = real[k];
    SpanResult r;
    std::vector<MemberEnd> mine(res[i].members + 1);
    inflate_span<true>(w.data(), nbytes, i ? cand[i - 1] : start, i == 0 && at_member, cand.data(), (uint32_t)cand.size(), i, T, sym.data() + off[k], res[i].out_n,
                       mine.data(), r, i == 0 ? prior : kInfNone);
    if (r.status != res[i].status || r.out_n != res[i].out_n || r.members != res[i].members) return 100;
    for (uint32_t m = 0; m < r.members; ++m) { mine[m].out_end += off[k]; ends.push_back(mine[m]); }
  }
  std::vector<uint8_t> win((size_t)(nreal + 1) * kInfWindow), got(total);
  memcpy(win.data(), st.window.data(), kInfWindow);
  for (uint32_t k = 0; k < nreal; ++k)
    for (uint32_t j = 0; j < kInfWindow; ++j) win[(size_t)(k + 1) * kInfWindow + j] = inf_window_byte(sym.data() + off[k], res[real[k]].out_n, win.data() + (size_t)k * kInfWindow, j);
  for (uint32_t k = 0; k < nreal; ++k)
    for (uint64_t j = 0; j < keep[k]; ++j) got[off[k] + j] = inf_resolve(sym[off[k] + j], win.data() + (size_t)k * kInfWindow);
  if (total || (!ends.empty() && st.carry.len)) {
    std::vector<uint64_t> poff; std::vector<uint32_t> plen, first, crcs, tab(256);
    for (uint32_t i = 0; i < 256; ++i) tab[i] = crc_table_entry(i);
    inf_crc_plan(ends, 32768, poff, plen, first, total);
    crcs.resize(poff.size());
    for (size_t k = 0; k < poff.size(); ++k) crcs[k] = crc_piece(got.data() + poff[k], plen[k], tab.data());
    if (const uint32_t bad = inf_crc_verify(ends, plen, first, crcs.data(), &st.carry)) return bad;
  }
  // the window of the next round
  std::vector<uint8_t> nw(st.window);
  nw.insert(nw.end(), got.begin(), got.end());
  st.window.assign(nw.end() - kInfWindow, nw.end());
  st.members += (uint32_t)ends.size();
  st.at = next;
  out.insert(out.end(), got.begin(), got.end());
  return 0;
}

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  const std::string mode = argv[1];
  const std::vector<uint8_t> raw = slurp(argv[2]);
  const uint64_t piece = strtoull(argv[argc - 1], nullptr, 10);
  if (mode == "inflate") {
    HostStream st;
    std::vector<uint8_t> tail, out;
    uint32_t rounds = 0, k = 0;
    for (uint64_t p = 0; p < raw.size() || k == 0; p += piece, ++k) {
      const uint64_t e = std::min<uint64_t>(raw.size(), p + piece);
      const bool eof = e == raw.size();
      tail.insert(tail.end(), raw.begin() + p, raw.begin() + e);
      if (st.at.eos) { tail.clear(); if (eof) break; continue; }
      if (eof && raw.size() < 18) { printf("error %u piece %u\n", (unsigned)kInfErrMember, k); return 1; }
      if (tail.empty() && !eof) continue;
      const uint32_t bad = round_host(tail, eof, st, out);
      ++rounds;
      if (bad) { printf("error %u piece %u\n", bad, k); return 1; }
      if (st.at.eos) tail.clear();
      else { const uint64_t drop = st.at.bit / 8; tail.erase(tail.begin(), tail.begin() + drop); st.at.bit -= drop * 8; }
      if (eof) break;
    }
    FILE* f = fopen(argv[3], "wb");
    fwrite(out.data(), 1, out.size(), f); fclose(f);
    printf("ok bytes %zu rounds %u\n", out.size(), rounds);
    return 0;
  }
  if (mode == "count") {
    CountState s;
    if (!raw.empty()) s.period = raw[0] == '@' ? 4 : 2;
    for (uint64_t p = 0; p < raw.size(); p += piece) {
      const uint64_t n = std::min<uint64_t>(raw.size(), p + piece) - p;
      std::vector<uint64_t> nl;
      for (uint64_t i = 0; i < n; ++i) if (raw[p + i] == '\n') nl.push_back(i);
      if (n && raw[p + n - 1] != '\n') nl.push_back(n);   // the virtual final newline of the device's index
      ReadCounts acc = rc_none();
      for (uint64_t i = 0; i < nl.size(); ++i) { ReadCounts x; if (rc_line(nl.data(), i, n, s, x)) acc = rc_join(acc, x); }
      const uint64_t nreal = nl.size() - (!nl.empty() && nl.back() >= n ? 1 : 0);
      rc_fold(s, acc);
      rc_advance(s, n, nreal, nreal ? nl[nreal - 1] : 0);
    }
    printf("%llu %llu %u %u\n", (unsigned long long)s.reads, (unsigned long long)s.length, s.min_len, s.max_len);
    return 0;
  }
  return 2;
}
