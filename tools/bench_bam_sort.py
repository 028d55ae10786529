"""The coordinate-sorted aligned.bam (-bam_sorted) next to the unsorted one (-bam), on the workload of tools/bench_bam.py: bench.py's
seeded reads as one .fastq.gz aligned against the 8 databases through api.run_files in 256 MB batches.  The two legs alternate in
one process, --rounds times each.  Reports per leg the reads/s of the streamed pass (run_files' "stream" seconds, which hold the
sorted leg's finish) and the size of aligned.bam; for -bam_sorted also the finish (seconds["bam_sort"]) split into plan, reading
the run file, upload, the device time of the window calls (gather, compression, index pass), their D2H, the writes and the index,
the sizes of aligned.bam.bai and of the run file, the records (from the index's pseudo-bins), and the device bytes the records take
(computed, not measured): the accumulator's 12 B per record and the finish's sort and offsets, 48 B per record.  Prints one JSON line
with the card's name and power limit.
Run on the GPU:  python tools/bench_bam_sort.py [--block-reads 200000] [--copies 12] [--rounds 2] [--batch-mb 256]"""
import argparse
import json
import os
import shutil
import struct
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from sortmerna_b200 import api, hostio  # noqa: E402
from tools.bench_stream import write_repeated_gz  # noqa: E402

LEGS = {"bam": dict(bam=True), "bam_sorted": dict(bam_sorted=True)}
ACC_B, FINISH_B = 12, 48   # per record: key + size; the finish's ordinals, sorted keys and ordinals, sizes and offsets of both orders


def mapped_records(bai: bytes) -> int:
    """the n_mapped of every reference's pseudo-bin"""
    n_ref, at, total = struct.unpack_from("<i", bai, 4)[0], 8, 0
    for _ in range(n_ref):
        n_bin = struct.unpack_from("<i", bai, at)[0]
        at += 4
        for _ in range(n_bin):
            b, n = struct.unpack_from("<Ii", bai, at)
            if b == 37450:
                total += struct.unpack_from("<Q", bai, at + 8 + 16)[0]
            at += 8 + 16 * n
        at += 4 + 8 * struct.unpack_from("<i", bai, at)[0]
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block-reads", type=int, default=200_000)
    ap.add_argument("--copies", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch-mb", type=int, default=256)
    ap.add_argument("--piece-mb", type=int, default=256)
    args = ap.parse_args()
    batch, piece = args.batch_mb << 20, args.piece_mb << 20
    out = dict(card=bench.card(0), batch_mb=args.batch_mb, piece_mb=args.piece_mb, window_mb=api.BAM_SORT_WINDOW >> 20)
    run_bytes, finish = [0], []
    add, fin = api.Aligner.bam_sort_add, api.Aligner.bam_sort_finish

    def timed_add(self, *a, **kw):
        buf, nb = add(self, *a, **kw)
        run_bytes[0] += nb
        return buf, nb

    def timed_finish(self, *a, **kw):
        bai = fin(self, *a, **kw)
        finish.append(dict(self.bam_sort_seconds))
        return bai
    api.Aligner.bam_sort_add, api.Aligner.bam_sort_finish = timed_add, timed_finish
    with tempfile.TemporaryDirectory(prefix="smr_bench_bam_sort_") as work:
        fastas, _, _, refs, stats, _ = bench.load_databases(work)
        reads = bench._gen_reads_numpy(bench.DbPool(refs), args.block_reads, bench.GEN_SEED + 777)
        p = os.path.join(work, "block.fq")
        bench.write_fastq(p, reads)
        block = open(p, "rb").read()
        os.remove(p)
        fq = os.path.join(work, "reads.fastq.gz")
        gz = write_repeated_gz(fq, block, args.copies)
        out.update(reads=args.block_reads * args.copies, gz_gb=gz / 1e9, text_gb=len(block) * args.copies / 1e9)
        g = json.load(open(os.path.join(ROOT, "sortmerna_b200", "gumbel_defaults.json")))["gumbel"]
        gum = [(g[os.path.basename(f)]["lambda_"], g[os.path.basename(f)]["K"]) for f in fastas]
        al = api.Aligner(0)   # the minimal scores of the file, computed once for every leg
        c = al.read_counts(fq, piece_bytes=piece)
        al.close()
        ms = [hostio.minimal_score(st, lam, K, c["length"], c["reads"]) for st, (lam, K) in zip(stats, gum)]
        res = {leg: dict(reads_s=[], bam_gb=None, seconds=[]) for leg in LEGS}
        for rnd in range(args.rounds):
            for leg, opts in LEGS.items():
                d = os.path.join(work, leg)
                run_bytes[0] = 0
                del finish[:]
                q = api.run_files(fastas, [fq], d, gumbel=gum, minimal_score=ms, batch_bytes=batch, piece_bytes=piece, cmd="bench_bam_sort ",
                                  **opts)
                r = res[leg]
                r["reads_s"].append(round(q["reads"] / q["seconds"]["stream"]))
                r["seconds"].append({k: round(v, 3) for k, v in q["seconds"].items()})
                r["bam_gb"] = os.path.getsize(os.path.join(d, "aligned.bam")) / 1e9
                r["batches"] = q["batches"]
                if leg == "bam_sorted":
                    bai = open(os.path.join(d, "aligned.bam.bai"), "rb").read()
                    n = mapped_records(bai)
                    r.setdefault("finish", []).append({k: round(v, 3) for k, v in finish[0].items()})
                    r.update(bai_mb=len(bai) / 1e6, run_file_gb=run_bytes[0] / 1e9, records=n, accumulator_mb=n * ACC_B / 1e6,
                             finish_scratch_mb=n * FINISH_B / 1e6)
                shutil.rmtree(d)
        out["legs"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
