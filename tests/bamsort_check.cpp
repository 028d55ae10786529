// Prints the sorted BAM's helpers of smr_fmt.h (the coordinate key, the virtual offset, the chunk merge rule) for
// tests/test_bam_sort_host.py, which checks them against tests/bai_spec.py.
//   bamsort_check   -> one line per case: "key ref pos flag value", "voff coffset in_block value", "merge prev_vend vbeg 0|1"
#include <cstdio>
#include <initializer_list>
#include "../sortmerna_b200/csrc/smr_fmt.h"
using namespace smr;

int main() {
  for (int32_t ref : {0, 1, 7, 65535, 2147483647})
    for (int32_t pos : {-1, 0, 1, 16383, 16384, 536870910})
      for (uint32_t flag : {0u, 16u, 4u, 20u})
        printf("key %d %d %u %llu\n", ref, pos, flag, (unsigned long long)fmt::bam_sort_key(ref, pos, flag));
  for (uint64_t c : {0ull, 1ull, 65321ull, 1ull << 40, (1ull << 48) - 1})
    for (uint32_t in : {0u, 1u, 65279u, 65280u})
      printf("voff %llu %u %llu\n", (unsigned long long)c, in, (unsigned long long)fmt::bam_voffset(c, in));
  const uint64_t v[] = {0, 1, 65535, 65536, 65537, 3ull << 16 | 5, 4ull << 16, (123456ull << 16) | 65279};
  for (uint64_t a : v)
    for (uint64_t b : v) printf("merge %llu %llu %d\n", (unsigned long long)a, (unsigned long long)b, fmt::bam_chunks_merge(a, b) ? 1 : 0);
  return 0;
}
