// The read-count pass of a read stream (smr_stream_counts) as plain functions, shared by the kernels of smr_stream.cuh and the
// host-side check tests/stream_check.cpp.
//
// It restates Readfeed::count_reads_parallel (src/sortmerna/readfeed.cpp:1486-1663), whose totals the reference computes before
// it aligns anything: Refstats::minimal_score and the read length behind every E-value come from them.  Its rule is a per-byte
// model, not the records the decoder sees:
//   - a fixed line cycle, 4 lines per record if the file's first byte is '@' (FASTQ), else 2 (FASTA), counted over '\n' only;
//   - a line at cycle position 1 that ends in '\n' is one read, of length = every byte before that '\n' (a '\r' counts);
//   - a last sequence line without its '\n' is not counted;
//   - multi-line FASTA is read as 2-line records all the same;
//   - the minimum starts "unset" (0) and an empty sequence line sets it back to 0, so it is the shortest read after the last
//     empty one.
// For a flat multi-line FASTA the reference's result depends on -threads (each split restarts the cycle at a '>' line); this is
// the single-split result, which is what -threads 1 and every gzip file give.
#pragma once
#include <cstdint>
#include "smr_levbits.h"   // SMR_HD

namespace smr {

// the reads of a run of lines, in file order: how many, their total length, the longest, whether one was empty, and the shortest
// after the last empty one (~0u: none)
struct ReadCounts { uint64_t n, sum; uint32_t max, hasz, mafter, pad; };

SMR_HD ReadCounts rc_none() { return ReadCounts{0, 0, 0, 0, 0xFFFFFFFFu, 0}; }
SMR_HD ReadCounts rc_read(uint64_t len) {
  const uint32_t l = (uint32_t)len;   // the reference keeps min / max as uint32_t
  return ReadCounts{1, len, l, l == 0 ? 1u : 0u, l == 0 ? 0xFFFFFFFFu : l, 0};
}
// a, then b (associative, not commutative)
SMR_HD ReadCounts rc_join(const ReadCounts& a, const ReadCounts& b) {
  ReadCounts r;
  r.n = a.n + b.n; r.sum = a.sum + b.sum;
  r.max = a.max > b.max ? a.max : b.max;
  r.hasz = a.hasz | b.hasz;
  r.mafter = b.hasz ? b.mafter : (a.mafter < b.mafter ? a.mafter : b.mafter);
  r.pad = 0;
  return r;
}

// the totals of count_reads_parallel so far and the line cycle where the text pushed so far ends
struct CountState {
  uint64_t reads = 0, length = 0;
  uint32_t min_len = 0, max_len = 0;
  uint32_t period = 0;     // 4 (FASTQ) or 2 (FASTA); 0 until the first byte is seen
  uint32_t cycle = 0;      // position in the cycle of the line in progress
  uint64_t line_len = 0;   // bytes of the line in progress
  bool flat = false;       // a flat file after others: its minimum is merged with prior_min when it ends
  uint32_t prior_min = 0;
};

// min_read_len after the files so far.  Each flat file is counted alone and merged as readfeed.cpp:1651-1652 merges a split:
// "if (min == 0 || (r > 0 && r < min)) min = r"
SMR_HD uint32_t rc_min(const CountState& s) {
  if (!s.flat) return s.min_len;
  return s.prior_min == 0 || (s.min_len > 0 && s.min_len < s.prior_min) ? s.min_len : s.prior_min;
}

// the count of the next -reads file of the same run (readfeed.cpp:1497-1662): totals go on, the line cycle of the first file
// holds, the cycle restarts; a gzip file updates the run's minimum read by read, a flat file has its own, merged at its end
SMR_HD CountState rc_next_file(const CountState& s, bool gz) {
  CountState n = s;
  n.cycle = 0; n.line_len = 0;
  const uint32_t m = rc_min(s);
  n.flat = !gz;
  n.min_len = gz ? m : 0;
  n.prior_min = gz ? 0 : m;
  return n;
}

// min_read_len as the reference updates it read by read: "if (min == 0 || len < min) min = len"
SMR_HD void rc_fold(CountState& s, const ReadCounts& p) {
  if (p.n == 0) return;
  const uint32_t m = p.mafter == 0xFFFFFFFFu ? 0u : p.mafter;
  if (p.hasz) s.min_len = m;
  else s.min_len = s.min_len == 0 ? m : (m < s.min_len ? m : s.min_len);
  s.reads += p.n; s.length += p.sum;
  if (p.max > s.max_len) s.max_len = p.max;
}

// the read a line makes, if any: line i of a piece ends at nl[i] (< n: a real '\n'), starts after nl[i - 1] (or at the piece's
// start, after the line_len bytes the earlier pieces held)
SMR_HD bool rc_line(const uint64_t* nl, uint64_t i, uint64_t n, const CountState& s, ReadCounts& out) {
  if (nl[i] >= n || (s.cycle + i) % s.period != 1) return false;
  const uint64_t start = i ? nl[i - 1] + 1 : 0;
  out = rc_read(nl[i] - start + (i ? 0 : s.line_len));
  return true;
}

// after a piece of n bytes with nreal '\n' (the last at last_nl): the cycle and the line in progress
SMR_HD void rc_advance(CountState& s, uint64_t n, uint64_t nreal, uint64_t last_nl) {
  if (nreal == 0) { s.line_len += n; return; }
  s.cycle = (uint32_t)((s.cycle + nreal) % s.period);
  s.line_len = n - (last_nl + 1);
}

}  // namespace smr
