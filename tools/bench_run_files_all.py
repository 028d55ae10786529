"""api.run_files at -num_alignments 0 -sam, on two read files:
- bench: bench.py's seeded reads as one .fastq.gz (a block of --block-reads reads deflated once and repeated --copies times, as
  tools/bench_run_files.py makes it), against the 8 databases;
- near: reads from tools/bench_heavy.py's near-copy database (groups of copies of a 1400 bp ancestor), where a read stores many
  alignments, at --near-batch-mb per batch.
Reports reads/s of the streamed pass (run_files' "stream" seconds), its per-stage seconds, the layout run_files chose ("strided"
when the build predates the packed run driver) and the device bytes of the result arrays of one batch, computed from the struct
sizes (228 B per alignment slot, tools/bench_all_alignments.DEV_SLOT_BYTES) and the n_align of the first batch's reads: strided,
reads x the largest n_align (the stride the placement grows to); packed, reads x the first stride (16) plus the slots of the reads
that run again.  The placement's device time per batch comes from a packed Aligner on the first batch where the build has
place_packed().  Run it in the parent's tree and in this one, alternately, to compare.  Prints one JSON line with the card's name
and power limit.
Run on the GPU:  python tools/bench_run_files_all.py [--block-reads 200000] [--copies 12] [--near-reads 200000]"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from sortmerna_b200 import api, hostio  # noqa: E402
from tools import bench_heavy  # noqa: E402
from tools.bench_stream import write_repeated_gz  # noqa: E402

SLOT_BYTES = 32 + 40 + 40 + 4 + 16 + 24 * 4   # AlnWork, OutAln, TraceJob + job-list entry, AlnStats, CIGAR share (run_impl)
FIRST_STRIDE = 16


def first_batch_counts(fastas, ms, fq, batch, piece, lnwin=18):
    """n_align of the first batch's reads (packed download), and the placement's device ms where the build has place_packed()"""
    al = api.Aligner(0)
    try:
        al.set_params(api.default_params(num_alignments=0))
        for k, f in enumerate(fastas):
            st, _ = hostio.fasta_index_stats(f, lnwin, 3072.0)
            al.build_index_device(k, f, hostio.split_by_parts(hostio.load_references(f), st), int(ms[k]), (lnwin, lnwin // 2, 3), lnwin)
        al.set_aln_layout("packed")
        for _ in al.stream_fastx(fq, batch_bytes=batch, piece_bytes=piece):
            al.run_resident(with_stats=True)
            place_ms = al.place_packed()["place_ms"] if hasattr(al, "place_packed") else None
            cnt = al.download()["res"]["n_align"].astype(np.int64)
            return cnt, place_ms
    finally:
        al.close()


def leg(fastas, gum, fq, work, batch, piece):
    d = os.path.join(work, "out")
    c = api.Aligner(0)
    counts = c.read_counts(fq, piece)
    c.close()
    stats = [hostio.fasta_index_stats(f, 18, 3072.0)[0] for f in fastas]
    ms = [hostio.minimal_score(st, lam, K, counts["length"], counts["reads"]) for st, (lam, K) in zip(stats, gum)]
    r = api.run_files(fastas, [fq], d, api.default_params(num_alignments=0), gumbel=gum, minimal_score=ms, sam=True, batch_bytes=batch,
                      piece_bytes=piece)
    cnt, place_ms = first_batch_counts(fastas, ms, fq, batch, piece)
    n = cnt.size
    strided = n * max(1, int(cnt.max())) * SLOT_BYTES
    packed = (n * FIRST_STRIDE + int(cnt[cnt > FIRST_STRIDE].sum())) * SLOT_BYTES
    sam = os.path.getsize(os.path.join(d, "aligned.sam"))
    for f in os.listdir(d):
        os.remove(os.path.join(d, f))
    return dict(reads=r["reads"], batches=r["batches"], layout=r.get("layout", "strided"), reads_s=r["reads"] / r["seconds"]["stream"],
                seconds={k: round(v, 3) for k, v in r["seconds"].items()}, sam_gb=sam / 1e9, first_batch_reads=n,
                n_align_max=int(cnt.max()), n_align_mean=float(cnt.mean()), dev_result_bytes_strided=strided,
                dev_result_bytes_packed=packed, place_ms_first_batch=place_ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block-reads", type=int, default=200_000)
    ap.add_argument("--copies", type=int, default=12)
    ap.add_argument("--near-reads", type=int, default=200_000)
    ap.add_argument("--batch-mb", type=int, default=256)
    ap.add_argument("--near-batch-mb", type=int, default=16)
    ap.add_argument("--workloads", default="bench,near")
    args = ap.parse_args()
    out = dict(card=bench.card(0), batch_mb=args.batch_mb, near_batch_mb=args.near_batch_mb, slot_bytes=SLOT_BYTES, legs={})
    g = json.load(open(os.path.join(ROOT, "sortmerna_b200", "gumbel_defaults.json")))["gumbel"]
    with tempfile.TemporaryDirectory(prefix="smr_bench_rf_all_") as work:
        for wl in args.workloads.split(","):
            if wl == "bench":
                fastas, _, _, refs, _, _ = bench.load_databases(work)
                reads = bench._gen_reads_numpy(bench.DbPool(refs), args.block_reads, bench.GEN_SEED + 777)
                p = os.path.join(work, "block.fq")
                bench.write_fastq(p, reads)
                block = open(p, "rb").read()
                os.remove(p)
                fq = os.path.join(work, "reads.fastq.gz")
                write_repeated_gz(fq, block, args.copies)
                gum = [(g[os.path.basename(f)]["lambda_"], g[os.path.basename(f)]["K"]) for f in fastas]
                out["legs"][wl] = leg(fastas, gum, fq, work, args.batch_mb << 20, 256 << 20)
            else:
                fasta = os.path.join(work, "heavy.fasta")
                bench_heavy.write_database(fasta, 100, 1400)
                refs = hostio.load_references(fasta)
                reads = bench_heavy.gen_reads(refs, args.near_reads, bench_heavy.SEED + 1)
                fq = os.path.join(work, "near.fq")
                bench.write_fastq(fq, reads)
                gk = g[bench_heavy.GUMBEL_OF]
                out["legs"][wl] = leg([fasta], [(gk["lambda_"], gk["K"])], fq, work, args.near_batch_mb << 20, 64 << 20)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
