"""api.run_files against the hand-written stream loop on the benchmark workload: bench.py's seeded reads as one .fastq.gz (a block of
reads deflated once and repeated, as tools/bench_stream.py makes it) aligned against the 8 databases.  The old loop is
bench_stream.py's end-to-end leg: read_counts, minimal scores and E-value parameters, the on-disk index loaded, then stream_fastx
with run_resident / download / ReportWriter.write and close.  The new one is run_files on the same file with the same minimal
scores, its index built on the device.  Both write -sam, then -fastx -other; the legs alternate, --rounds times each.
Reports reads/s of the streamed pass, from the first batch until every report file is complete (ReportWriter.close() for the old
loop, the part files of the groups after the first appended for run_files; the count pass and the index excluded from both), and
run_files' per-stage seconds: batch production, run, placement, formatting (with the OTU map and denovo statistics when asked), the
writer thread's writes and its wait, the caller's wait for a free output buffer, and the part-file appends.  Prints one JSON line with the card's name and power limit.
Run on the GPU:  python tools/bench_run_files.py [--block-reads 200000] [--copies 12] [--rounds 2] [--batch-mb 256]"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from sortmerna_b200 import api, hostio  # noqa: E402
from tools.bench_stream import write_repeated_gz  # noqa: E402

LEGS = {"sam": dict(sam=True), "fastx_other": dict(fastx=True, other=True)}


def old_loop(fq, fastas, prefixes, refs, stats, gum, out_dir, opts, batch, piece):
    """bench_stream.py's end-to-end leg; returns (reads, seconds of the streamed pass, minimal scores)"""
    al = api.Aligner(0)
    try:
        al.set_params(api.default_params())
        c = al.read_counts(fq, piece_bytes=piece)
        ms = [hostio.minimal_score(st, lam, K, c["length"], c["reads"]) for st, (lam, K) in zip(stats, gum)]
        bench.load_resident_index(al, "files", fastas, prefixes, refs, ms, stats)
        for k, (lam, K) in enumerate(gum):
            al.set_report_scoring(k, lam, K, *hostio.evalue_params(stats[k], K, c["length"], c["reads"]))
        w = api.ReportWriter(out_dir, al, **opts)
        t0 = time.perf_counter()
        n = 0
        for k in al.stream_fastx(fq, batch_bytes=batch, piece_bytes=piece):
            al.run_resident(with_stats=bool(opts.get("sam")))
            w.write(al.download())
            n += k
        w.close()
        return n, time.perf_counter() - t0, ms
    finally:
        al.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block-reads", type=int, default=200_000)
    ap.add_argument("--copies", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch-mb", type=int, default=256)
    ap.add_argument("--piece-mb", type=int, default=256)
    args = ap.parse_args()
    batch, piece = args.batch_mb << 20, args.piece_mb << 20
    out = dict(card=bench.card(0), batch_mb=args.batch_mb, piece_mb=args.piece_mb)
    with tempfile.TemporaryDirectory(prefix="smr_bench_runfiles_") as work:
        fastas, _, prefixes, refs, stats, _ = bench.load_databases(work)
        pool = bench.DbPool(refs)
        reads = bench._gen_reads_numpy(pool, args.block_reads, bench.GEN_SEED + 777)
        p = os.path.join(work, "block.fq")
        bench.write_fastq(p, reads)
        block = open(p, "rb").read()
        os.remove(p)
        fq = os.path.join(work, "reads.fastq.gz")
        gz = write_repeated_gz(fq, block, args.copies)
        out.update(reads=args.block_reads * args.copies, gz_gb=gz / 1e9, text_gb=len(block) * args.copies / 1e9)
        g = json.load(open(os.path.join(ROOT, "sortmerna_b200", "gumbel_defaults.json")))["gumbel"]
        gum = [(g[os.path.basename(f)]["lambda_"], g[os.path.basename(f)]["K"]) for f in fastas]
        res = {}
        for leg, opts in LEGS.items():
            r = res[leg] = dict(old_reads_s=[], new_reads_s=[], new_seconds=[])
            for rnd in range(args.rounds):
                d_old, d_new = os.path.join(work, "old"), os.path.join(work, "new")
                n, t, ms = old_loop(fq, fastas, prefixes, refs, stats, gum, d_old, opts, batch, piece)
                r["old_reads_s"].append(n / t)
                q = api.run_files(fastas, [fq], d_new, gumbel=gum, minimal_score=ms, batch_bytes=batch, piece_bytes=piece, zip_out=False, **opts)
                assert q["reads"] == n
                r["new_reads_s"].append(q["reads"] / q["seconds"]["stream"])
                r["new_seconds"].append({k: round(v, 3) for k, v in q["seconds"].items()})
                if rnd == 0:   # the same files, apart from the SAM header and aligned.log (ReportWriter is given neither here)
                    names = sorted(f for f in os.listdir(d_old) if not f.startswith("."))
                    assert sorted(names + ["aligned.log"]) == sorted(os.listdir(d_new)), (names, os.listdir(d_new))
                    for f in names:
                        a, b = open(os.path.join(d_old, f), "rb").read(), open(os.path.join(d_new, f), "rb").read()
                        if f == "aligned.sam":
                            b = b[b.index(b"\n", b.index(b"@PG")) + 1:]
                        assert a == b, f
                    r["files_gb"] = sum(os.path.getsize(os.path.join(d_new, f)) for f in names) / 1e9
                shutil.rmtree(d_old)
                shutil.rmtree(d_new)
        out["legs"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
