"""All alignments (-num_alignments 0) in the two result layouts, on two workloads:
- heavy: tools/bench_heavy.py's near-copy database (groups of 30-50 copies of a 1400 bp ancestor at 0.2-1 %), where a read stores
  tens of alignments at N = 0;
- bench: bench.py's workload (the 8 seeded stand-in databases, synthetic 150 bp reads).
For each workload and for N = 0 and N = 1 it runs, alternating in one process, the packed layout (first-pass stride 16, reads that
store more run again at their own count; N when N > 0) and the strided layout at the stride the batch needs (grown by Aligner.align from the
stride the library names).  Per leg: the kernel time (CUDA events inside the C ABI, re-runs included) and the end-to-end rate (upload,
run, download, host clock), the bytes of the result arrays on the device (computed from the struct sizes, see DEV_SLOT_BYTES; for
packed, the first run's plus the largest re-run sub-batch's, which are allocated at the same time) and on
the host (the arrays the call returns; the library keeps the packed placement, of the same size, on the device for repeated
downloads), the host staging of the download (computed, HOST_STAGE_SLOT_BYTES; the packed download no longer stages since its
placement moved to the device), the n_align distribution, and the reads run again and their sub-batches (from the
library's SMR_VERBOSE line, in one untimed extra run).  Every leg also checks that both layouts return the same alignments.
Prints one JSON line with the card name and power limit.
Run on the GPU:  python tools/bench_all_alignments.py --reads 200000 --steps 3"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from sortmerna_b200 import api, hostio  # noqa: E402
from tools import bench_heavy, stage_data  # noqa: E402

# device bytes per alignment slot of a run: AlnWork 32, OutAln 40, TraceJob 40 + its job-list entry 4, AlnStats 16, and the CIGAR
# pool's share of 24 words (smr_capi.cu run_impl)
DEV_SLOT_BYTES = 32 + 40 + 40 + 4 + 16 + 24 * 4
# host bytes per slot a download stages from the device before it places anything: OutAln 40 + AlnStats 16 (the CIGAR words and the
# per-read state come on top); the strided download stages in the context's page-locked buffers, which it keeps, the packed one in
# per-run buffers it frees once the reads are placed
HOST_STAGE_SLOT_BYTES = 40 + 16
FIRST_STRIDE = 16
RETRY_SLOTS = 1 << 24   # the library's default slot budget of one re-run sub-batch (SMR_RETRY_SLOTS)
RERUN = re.compile(rb"packed results: (\d+) reads stored more than \d+ alignments and were run again at their own count in (\d+) sub-batches")


def _databases(work, which, nreads):
    """(aligner factory, reads per step generator)"""
    if which == "heavy":
        fasta = os.path.join(work, "heavy.fasta")
        bench_heavy.write_database(fasta, 100, 1400)
        idx_dir, _ = stage_data.ensure_indexes([fasta], os.path.join(work, "idx_heavy"))
        prefix = hostio.find_index_prefixes(idx_dir)[os.path.basename(fasta)]
        refs, st = hostio.load_references(fasta), hostio.parse_stats(prefix)
        g = json.load(open(os.path.join(ROOT, "sortmerna_b200", "gumbel_defaults.json")))["gumbel"][bench_heavy.GUMBEL_OF]
        ms = [hostio.minimal_score(st, g["lambda_"], g["K"], nreads * bench.READ_LEN, nreads)]

        def load(al):
            al.build_index_device(0, fasta, refs, ms[0], (18, 9, 3), st.lnwin)

        return load, lambda s: bench_heavy.gen_reads(refs, nreads, bench_heavy.SEED + 1 + s).reshape(-1)
    fastas, _, prefixes, refs, stats, _ = bench.load_databases(work)
    ms = bench.minimal_scores(stats, fastas, nreads)
    pool = bench.DbPool(refs)

    def load(al):
        bench.load_resident_index(al, "device", fastas, prefixes, refs, ms, stats)

    return load, lambda s: bench.gen_reads(pool, nreads, bench.GEN_SEED + s).reshape(-1)


def _verbose_download(al):
    """one run and download with SMR_VERBOSE on, stderr captured: (reads run again, sub-batches).  (The run is needed: the library
    places a run's packed results once, and a later download of the same run only copies them.)"""
    with tempfile.TemporaryFile() as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        os.environ["SMR_VERBOSE"] = "1"
        try:
            al.run_resident(with_stats=True)
            al.download()
        finally:
            del os.environ["SMR_VERBOSE"]
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        m = RERUN.findall(f.read())
    return (int(m[-1][0]), int(m[-1][1])) if m else (0, 0)


def _largest_rerun(cnt, stride):
    """slots of the largest sub-batch the packed download runs again (reads that overflow only the stride; the library's split)"""
    best = cur = 0
    for c in (int(x) for x in cnt if x > stride):
        if cur and cur + c > RETRY_SLOTS:
            best, cur = max(best, cur), 0
        cur += c
    return max(best, cur)


def _leg(al, layout, cat, off, n, na):
    t0 = time.perf_counter()
    al.upload(cat, off)
    al.run_resident(with_stats=True)
    out = al.download()
    e2e = time.perf_counter() - t0
    kern = al.timings()["total_ms"]
    cnt = out["res"]["n_align"].astype(np.int64)
    if layout == "packed":   # the first run's arenas and the largest re-run sub-batch are allocated at once
        stride = na if na > 0 else FIRST_STRIDE
        dev_slots = n * stride + _largest_rerun(cnt, stride)
        staged = n * stride + int(cnt[cnt > stride].sum())   # the first run's slots, then every re-run's
        host = out["alns"].nbytes + out["stats"].nbytes + out["aln_off"].nbytes
    else:
        dev_slots = n * out["slots"]
        staged = dev_slots
        host = out["alns"].nbytes + out["stats"].nbytes
    host += out["res"].nbytes + out["cigar"].nbytes
    return out, dict(kernel_ms=kern, e2e_s=e2e, dev_slot_bytes=dev_slots * DEV_SLOT_BYTES, host_result_bytes=int(host),
                     host_staging_bytes=staged * HOST_STAGE_SLOT_BYTES,
                     n_align=dict(mean=float(cnt.mean()), p99=float(np.percentile(cnt, 99)), max=int(cnt.max())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=200_000, help="reads per step")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--workloads", default="heavy,bench")
    args = ap.parse_args()
    out = dict(card=bench.card(0), reads_per_step=args.reads, steps=args.steps, first_pass_stride=FIRST_STRIDE, dev_slot_bytes=DEV_SLOT_BYTES,
               legs={})
    with tempfile.TemporaryDirectory(prefix="smr_bench_all_") as work:
        for wl in args.workloads.split(","):
            load, gen = _databases(work, wl, args.reads)
            off = np.arange(args.reads + 1, dtype=np.uint64) * bench.READ_LEN
            batches = [gen(s) for s in range(args.steps)]
            for na in (0, 1):
                als = {}
                for layout in ("packed", "strided"):
                    al = api.Aligner(0)
                    al.set_params(api.default_params(num_alignments=na))
                    load(al)
                    al.set_aln_layout(layout)
                    al.set_aln_slots(FIRST_STRIDE)
                    als[layout] = al
                # the sizes the batches need, kept by each Aligner (strided: the stride; packed: the alignment and CIGAR array sizes),
                # and a warm-up of both
                for b in batches:
                    for al in als.values():
                        al.align(b, off)
                for layout, al in als.items():
                    _leg(al, layout, batches[0], off, args.reads, na)
                rec = {k: [] for k in als}
                for s in range(args.steps):
                    res = {}
                    for layout in (("packed", "strided") if s % 2 == 0 else ("strided", "packed")):
                        res[layout], r = _leg(als[layout], layout, batches[s], off, args.reads, na)
                        rec[layout].append(r)
                    p, q = res["packed"], api.pack_alns(res["strided"])
                    if not (np.array_equal(p["res"], q["res"]) and p["alns"]["score1"].tolist() == q["alns"]["score1"].tolist()):
                        raise SystemExit(f"{wl} N={na} step {s}: the layouts disagree")
                reruns, batches_ = _verbose_download(als["packed"])
                leg = {}
                for layout, rs in rec.items():
                    leg[layout] = dict(kernel_ms=[round(r["kernel_ms"], 2) for r in rs],
                                       e2e_reads_per_s=[round(args.reads / r["e2e_s"]) for r in rs],
                                       kernel_reads_per_s=[round(args.reads / (r["kernel_ms"] / 1e3)) for r in rs],
                                       dev_result_bytes=rs[-1]["dev_slot_bytes"], host_result_bytes=rs[-1]["host_result_bytes"],
                                       host_staging_bytes=rs[-1]["host_staging_bytes"],
                                       n_align=rs[-1]["n_align"])
                leg["strided"]["stride"] = int(als["strided"].L.smr_aln_slots(als["strided"].h))
                leg["packed"]["reads_run_again"], leg["packed"]["sub_batches"] = reruns, batches_
                out["legs"][f"{wl}_N{na}"] = leg
                for al in als.values():
                    al.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
