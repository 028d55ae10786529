"""How many streamed list entries survive the seed kernel's screen (half_screen, sortmerna_b200/csrc/smr_levbits.h) on the
bench workload, counted on the host: the 8 seeded stand-in databases indexed as bench.py indexes them, flattened as the
library flattens them (tests/flatten_dump.cpp), and N reads of bench.py's CPU generator walked window by window the way
coop_stream walks them (tools/seed_filter_stats.cpp).  Per database and in total: entries streamed (chunk padding
included), screen survivors, true matches, and buffer flushes per round now and before the screen.
Usage: python tools/seed_filter_stats.py [N]   (default 20000; no GPU needed)"""
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from sortmerna_b200 import hostio  # noqa: E402
from tools import stage_data, synth_databases  # noqa: E402

SKIPS = (18, 9, 3)
STEP = SKIPS[2]   # every pass position is a multiple of the last shift


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
    with tempfile.TemporaryDirectory(prefix="smr_filter_stats_") as d:
        fastas = synth_databases.write(os.path.join(d, "db"))
        idx_dir, _ = stage_data.ensure_indexes(fastas, os.path.join(d, "idx"))
        pre = hostio.find_index_prefixes(idx_dir)
        refs = [hostio.load_references(f) for f in fastas]
        reads = bench._gen_reads_numpy(bench.DbPool(refs), n, bench.GEN_SEED + 99)
        rp = os.path.join(d, "reads.u8")
        reads.tofile(rp)
        exe = {}
        for name, srcs in (("flatten_dump", ["tests/flatten_dump.cpp", "sortmerna_b200/csrc/smr_index.cpp"]),
                           ("seed_filter_stats", ["tools/seed_filter_stats.cpp"])):
            exe[name] = os.path.join(d, name)
            subprocess.check_call(["g++", "-O2", "-std=c++17"] + [os.path.join(ROOT, s) for s in srcs] + ["-o", exe[name]])

        def one(f):
            p = pre[os.path.basename(f)]
            lnwin = hostio.parse_stats(p).lnwin
            out = os.path.join(d, "flat_" + os.path.basename(f))
            os.makedirs(out)
            subprocess.check_call([exe["flatten_dump"], p, "0", str(lnwin), out])
            r = subprocess.run([exe["seed_filter_stats"], os.path.join(out, "flookup.u32"), os.path.join(out, "flist.u32"), rp,
                                str(bench.READ_LEN), str(lnwin), str(STEP)], stdout=subprocess.PIPE, text=True, check=True)
            t = r.stdout.split()
            return {t[i]: int(t[i + 1]) for i in range(0, len(t), 2)}

        with ThreadPoolExecutor(8) as ex:
            rows = list(ex.map(one, fastas))
    tot = {k: sum(r[k] for r in rows) for k in rows[0]}
    print(f"{n} reads of the bench generator, {len(fastas)} databases")
    for f, r in [(os.path.basename(f), r) for f, r in zip(fastas, rows)] + [("total", tot)]:
        ce = max(r["chunk_entries"], 1)
        print(f"{f:34s} streamed {r['chunk_entries']:12d} (list entries {r['entries']:12d})  survivors {r['survivors']:10d} "
              f"({100 * r['survivors'] / ce:.3f} %)  matches {r['matches']:10d} ({100 * r['matches'] / ce:.3f} %)  "
              f"survivors/matches {r['survivors'] / max(r['matches'], 1):.2f}  per round: classify passes "
              f"{r['classify_passes'] / r['rounds']:.3f} flushes {r['flushes'] / r['rounds']:.3f} "
              f"(before the screen {r['flushes_before'] / r['rounds']:.3f})")


if __name__ == "__main__":
    main()
