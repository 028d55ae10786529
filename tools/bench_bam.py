"""aligned.bam next to aligned.sam on the workload of tools/bench_run_files.py: bench.py's seeded reads as one .fastq.gz aligned against
the 8 databases through api.run_files.  Three legs alternate in one process, --rounds times each: -sam, -bam, and -sam -zip-out.
Reports per leg the reads/s of the streamed pass (run_files' "stream" seconds: from the first batch until every report file is
complete), the size of the report file, and for -bam the device time of each batch's smr_format_bam_placed call
(smr_last_report_timings: upload, device work with the BGZF compression, download).  Prints one JSON line with the card's name and
power limit.
Run on the GPU:  python tools/bench_bam.py [--block-reads 200000] [--copies 12] [--rounds 2] [--batch-mb 256]"""
import argparse
import json
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from sortmerna_b200 import api, hostio  # noqa: E402
from tools.bench_stream import write_repeated_gz  # noqa: E402

LEGS = {"sam": dict(sam=True), "bam": dict(bam=True), "sam_zip": dict(sam=True, zip_out=True)}
FILES = {"sam": "aligned.sam", "bam": "aligned.bam", "sam_zip": "aligned.sam.gz"}


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
    # the device times of every BAM call run_files makes
    bam_ms = []
    fmt = api.Aligner.format_placed_into

    def timed(self, *a, **kw):
        r = fmt(self, *a, **kw)
        if kw.get("bam"):
            bam_ms.append(self.report_timings())
        return r
    api.Aligner.format_placed_into = timed
    with tempfile.TemporaryDirectory(prefix="smr_bench_bam_") as work:
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
        res = {leg: dict(reads_s=[], file_gb=None, seconds=[]) for leg in LEGS}
        for rnd in range(args.rounds):
            for leg, opts in LEGS.items():
                d = os.path.join(work, leg)
                del bam_ms[:]
                q = api.run_files(fastas, [fq], d, gumbel=gum, minimal_score=ms, batch_bytes=batch, piece_bytes=piece, cmd="bench_bam ", **opts)
                r = res[leg]
                r["reads_s"].append(round(q["reads"] / q["seconds"]["stream"]))
                r["seconds"].append({k: round(v, 3) for k, v in q["seconds"].items()})
                r["file_gb"] = os.path.getsize(os.path.join(d, FILES[leg])) / 1e9
                if leg == "bam":
                    r.setdefault("bam_call_ms", []).append([[round(v, 2) for v in t.values()] for t in bam_ms])
                    r["batches"] = q["batches"]
                shutil.rmtree(d)
        out["legs"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
