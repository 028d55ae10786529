"""Rate of the read stream (smr_stream_*, Aligner.read_counts / stream_fastx) on the benchmark workload: bench.py's seeded reads,
written as one .fastq.gz whose text passes 4 GiB (a block of reads deflated once, ending in a full flush, and repeated: one gzip
member).  Prints one JSON line with the card's name and power limit:
  * count: the count pass (SMR_STREAM_COUNT_ONLY) over the big file: wall time, GB/s of compressed and of inflated bytes;
  * batches: batch production over the big file (push = read from disk + inflate round + count; next = cut + decode), per batch;
  * fits: a smaller file of the same block (text under the 3.75 GB limit of smr_upload_fastx_gz): whole-file upload_fastx_gz
    (read + inflate + decode) next to streaming the same bytes (read + inflate + count + cut + decode), the cost of streaming;
  * end_to_end: the smaller file counted (minimal scores and E-value parameters from read_counts), then streamed with alignment
    (run_resident / download) and SAM through ReportWriter, reads/s of the streamed pass.
With --mates, only the mate leg: the same block split into two mate files (records 2k and 2k+1), each repeated into a .fastq.gz of
--mate-copies blocks, against the one-file .fastq.gz of the interleaved block repeated as often (the same text):
  * batches: batch production of stream_mates (two pushes a round, pair cut, interleave, decode) in pairs/s, and of stream_fastx
    over the interleaved file, alternating, --rounds times each;
  * end_to_end: alignment against the 8 databases (run_resident / download) and the -paired_in -out2 -fastx -other files through
    ReportWriter, over the mate stream and over the interleaved file (-paired_in -out2 as well), one pass each.
Run on the GPU:  python tools/bench_stream.py [--block-reads 200000] [--piece-mb 256] [--batch-mb 256] [--mates]"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from sortmerna_b200 import api, hostio  # noqa: E402


def write_repeated_gz(path, block, copies, level=6):
    """one gzip member: `block` deflated once (a full flush at its end makes it independent of what precedes it), `copies` times"""
    co = zlib.compressobj(level, zlib.DEFLATED, -15)
    body = co.compress(block) + co.flush(zlib.Z_FULL_FLUSH)
    crc = 0
    with open(path, "wb") as f:
        f.write(b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff")
        for _ in range(copies):
            f.write(body)
            crc = zlib.crc32(block, crc)
        f.write(b"\x03\x00")   # final empty fixed-Huffman block
        f.write(crc.to_bytes(4, "little") + ((len(block) * copies) & 0xFFFFFFFF).to_bytes(4, "little"))
    return os.path.getsize(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block-reads", type=int, default=200_000)
    ap.add_argument("--piece-mb", type=int, default=256)
    ap.add_argument("--batch-mb", type=int, default=256)
    ap.add_argument("--fit-copies", type=int, default=12)
    ap.add_argument("--mates", action="store_true")
    ap.add_argument("--mate-copies", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if args.mates:
        return mates(args)
    piece, batch = args.piece_mb << 20, args.batch_mb << 20
    out = dict(card=bench.card(0), piece_mb=args.piece_mb, batch_mb=args.batch_mb)
    with tempfile.TemporaryDirectory(prefix="smr_bench_stream_") as work:
        fastas, idx_dir, prefixes, refs, stats, _ = bench.load_databases(work)
        pool = bench.DbPool(refs)
        reads = bench._gen_reads_numpy(pool, args.block_reads, bench.GEN_SEED + 777)
        fq = os.path.join(work, "block.fq")
        bench.write_fastq(fq, reads)
        block = open(fq, "rb").read()
        os.remove(fq)
        copies = 2**32 // len(block) + 1
        big = os.path.join(work, "big.fastq.gz")
        gz_bytes = write_repeated_gz(big, block, copies)
        text_bytes = len(block) * copies
        out.update(block_reads=args.block_reads, copies=copies, reads=args.block_reads * copies, gz_gb=gz_bytes / 1e9, text_gb=text_bytes / 1e9)

        al = api.Aligner(0)
        al.set_params(api.default_params())
        # count pass
        al.read_counts(big, piece_bytes=piece)   # warm-up: buffers, module load
        t0 = time.perf_counter()
        c = al.read_counts(big, piece_bytes=piece)
        t = time.perf_counter() - t0
        assert c["reads"] == args.block_reads * copies, c
        out["count"] = dict(s=t, gz_gb_s=gz_bytes / 1e9 / t, text_gb_s=text_bytes / 1e9 / t, counts=c)
        # batch production
        per, n_total = [], 0
        t0 = time.perf_counter()
        last = t0
        for n in al.stream_fastx(big, batch_bytes=batch, piece_bytes=piece):
            now = time.perf_counter()
            per.append(now - last)
            last = now
            n_total += n
        t = time.perf_counter() - t0
        assert n_total == args.block_reads * copies
        out["batches"] = dict(s=t, batches=len(per), ms_per_batch=1e3 * t / len(per), max_ms=1e3 * max(per), text_gb_s=text_bytes / 1e9 / t,
                              reads_s=n_total / t)
        os.remove(big)
        # a file that still fits: whole-file upload next to streaming
        fit = os.path.join(work, "fit.fastq.gz")
        fit_gz = write_repeated_gz(fit, block, args.fit_copies)
        fit_text = len(block) * args.fit_copies
        raw = open(fit, "rb").read()
        al.upload_fastx_gz(raw)
        t0 = time.perf_counter()
        raw = open(fit, "rb").read()
        n_whole = al.upload_fastx_gz(raw)
        t_whole = time.perf_counter() - t0
        del raw
        t0 = time.perf_counter()
        n_str = sum(al.stream_fastx(fit, batch_bytes=batch, piece_bytes=piece))
        t_str = time.perf_counter() - t0
        assert n_whole == n_str == args.block_reads * args.fit_copies
        out["fits"] = dict(gz_gb=fit_gz / 1e9, text_gb=fit_text / 1e9, whole_upload_s=t_whole, stream_s=t_str, stream_over_whole=t_str / t_whole)
        # end to end: the count pass, then alignment and SAM over the streamed batches, scored from the counts (as the reference
        # computes minimal_score and the E-values from its own count pass)
        t0 = time.perf_counter()
        c = al.read_counts(fit, piece_bytes=piece)
        g = json.load(open(os.path.join(ROOT, "sortmerna_b200", "gumbel_defaults.json")))["gumbel"]
        gum = [(g[os.path.basename(f)]["lambda_"], g[os.path.basename(f)]["K"]) for f in fastas]
        ms = [hostio.minimal_score(st, lam, K, c["length"], c["reads"]) for st, (lam, K) in zip(stats, gum)]
        bench.load_resident_index(al, "files", fastas, prefixes, refs, ms, stats)
        for k, (lam, K) in enumerate(gum):
            al.set_report_scoring(k, lam, K, *hostio.evalue_params(stats[k], K, c["length"], c["reads"]))
        t_setup = time.perf_counter() - t0
        rdir = os.path.join(work, "reports")
        os.makedirs(rdir)
        w = api.ReportWriter(rdir, al, sam=True)
        t0 = time.perf_counter()
        n_done = 0
        for n in al.stream_fastx(fit, batch_bytes=batch, piece_bytes=piece):
            al.run_resident(with_stats=True)
            w.write(al.download())
            n_done += n
        w.close()
        t = time.perf_counter() - t0
        sam_bytes = sum(os.path.getsize(os.path.join(rdir, f)) for f in os.listdir(rdir))
        out["end_to_end"] = dict(reads=n_done, s=t, reads_s=n_done / t, sam_gb=sam_bytes / 1e9, count_and_index_s=t_setup, minimal_scores=ms)
        al.close()
    print(json.dumps(out))


def mates(args):
    piece, batch = args.piece_mb << 20, args.batch_mb << 20
    out = dict(card=bench.card(0), piece_mb=args.piece_mb, batch_mb=args.batch_mb)
    with tempfile.TemporaryDirectory(prefix="smr_bench_mates_") as work:
        fastas, idx_dir, prefixes, refs, stats, _ = bench.load_databases(work)
        pool = bench.DbPool(refs)
        reads = bench._gen_reads_numpy(pool, args.block_reads, bench.GEN_SEED + 778)
        fq = os.path.join(work, "block.fq")
        bench.write_fastq(fq, reads)
        block = open(fq, "rb").read()
        os.remove(fq)
        rec = len(block) // args.block_reads   # bench.write_fastq writes records of one size
        recs = [block[i:i + rec] for i in range(0, len(block), rec)]
        m1, m2, inter = os.path.join(work, "r1.fastq.gz"), os.path.join(work, "r2.fastq.gz"), os.path.join(work, "inter.fastq.gz")
        gz = write_repeated_gz(m1, b"".join(recs[0::2]), args.mate_copies) + write_repeated_gz(m2, b"".join(recs[1::2]), args.mate_copies)
        gz_inter = write_repeated_gz(inter, block, args.mate_copies)
        pairs = args.block_reads // 2 * args.mate_copies
        out.update(pairs=pairs, text_gb=len(block) * args.mate_copies / 1e9, mates_gz_gb=gz / 1e9, interleaved_gz_gb=gz_inter / 1e9)

        al = api.Aligner(0)
        al.set_params(api.default_params())
        legs = dict(mates=lambda: al.stream_mates(m1, m2, batch_bytes=batch, piece_bytes=piece),
                    single=lambda: al.stream_fastx(inter, batch_bytes=batch, piece_bytes=piece))
        for leg in legs.values():   # warm-up: buffers, module load
            for _ in leg():
                break
        times = {k: [] for k in legs}
        nb = {}
        for _ in range(args.rounds):
            for k, leg in legs.items():
                t0 = time.perf_counter()
                n_total, n_batches = 0, 0
                for n in leg():
                    n_total += n
                    n_batches += 1
                times[k].append(time.perf_counter() - t0)
                assert n_total == 2 * pairs, (k, n_total)
                nb[k] = n_batches
        out["batches"] = {k: dict(s=v, batches=nb[k], pairs_s=[pairs / t for t in v], ms_per_batch=[1e3 * t / nb[k] for t in v]) for k, v in times.items()}
        out["batches"]["mates_over_single"] = min(times["mates"]) / min(times["single"])

        c = al.read_counts([m1, m2], piece_bytes=piece)
        g = json.load(open(os.path.join(ROOT, "sortmerna_b200", "gumbel_defaults.json")))["gumbel"]
        gum = [(g[os.path.basename(f)]["lambda_"], g[os.path.basename(f)]["K"]) for f in fastas]
        ms = [hostio.minimal_score(st, lam, K, c["length"], c["reads"]) for st, (lam, K) in zip(stats, gum)]
        bench.load_resident_index(al, "files", fastas, prefixes, refs, ms, stats)
        e2e = {}
        for k, leg in legs.items():
            rdir = os.path.join(work, "reports_" + k)
            w = api.ReportWriter(rdir, al, fastx=True, other=True, paired_in=True, out2=True)
            t0 = time.perf_counter()
            for _ in leg():
                al.run_resident()
                w.write(al.download())
            paths = w.close()
            t = time.perf_counter() - t0
            e2e[k] = dict(s=t, pairs_s=pairs / t, files={os.path.basename(p): os.path.getsize(p) for p in paths})
            shutil.rmtree(rdir)
        assert e2e["mates"]["files"] == e2e["single"]["files"]
        out["end_to_end"] = e2e
        al.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
