"""Prints the role timeline of the instrumented candidate kernel (SMR_TIMELINE=1, stderr of a bench run): per 4 ms, the share of the
scorer warps busy / waiting, of the planner warps waiting for scores / voting and grouping / doing the rest, and the reads finished.
Usage: python tools/timeline_summary.py <stderr file> [scorers per SM] [planners per SM]"""
import sys


def main():
    f = sys.argv[1]
    ns_, np_ = (int(sys.argv[2]) if len(sys.argv) > 2 else 16) * 132, (int(sys.argv[3]) if len(sys.argv) > 3 else 15) * 132
    lines = [l for l in open(f) if l.startswith("[smr timeline]")]
    rows = {}
    for l in lines[-6:]:          # the last run in the file
        t = l.split(); rows[t[2]] = [int(x) for x in t[3:]]
    n = max(len(v) for v in rows.values())
    g = lambda k, i: rows[k][i] if i < len(rows[k]) else 0
    print(" ms   scorers busy% wait%   planners wait% vote+group% other% alive%   reads done")
    for i in range(0, n, 4):
        s = lambda k: sum(g(k, j) for j in range(i, min(i + 4, n)))
        w = min(4, n - i) * 1e6
        pa, pw, pv = s("planner_alive_ns"), s("planner_wait_ns"), s("planner_vote_group_ns")
        print("%3d   %12.1f %5.1f   %13.1f %11.1f %6.1f %6.1f   %d" % (i, 100 * s("scorer_busy_ns") / (ns_ * w), 100 * s("scorer_wait_ns") / (ns_ * w),
              100 * pw / (np_ * w), 100 * pv / (np_ * w), 100 * (pa - pw - pv) / (np_ * w), 100 * pa / (np_ * w), s("reads_done")))


if __name__ == "__main__":
    main()
