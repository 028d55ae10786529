"""Parity of whole read sets through the GPU path against what the unmodified reference binary printed for the same inputs: the
pass/fail totals and every SAM row.  The reference's results are stored under tests/golden/ (totals, minimal scores, the number and
SHA-256 of its sorted SAM rows and the first rows themselves, so that a failure names the first row that differs);
`python tests/test_gpu_bundled_sets.py` regenerates them where oracle/_ref/sortmerna_ref is built.

  * bench_workload: 20,000 reads of bench.py's workload against its 8 full-size databases (the seeded stand-ins of
    tools/synth_databases.py) -- BASELINE configs 3/5 in small.
  * set2_amplicon: shaped like BASELINE config 2 / the reference's t3 (amplicon reads, all from the database, against a 16S
    database indexed with -max_pos 250): 3,000 amplicons of 150-250 nt sampled with 1 % substitutions from the golden bacterial
    slice.
  * set4_mates: BASELINE config 4's shape through the library -- the golden mate reads against 8 databases (the two golden slices
    and six stand-ins)."""
import hashlib
import json
import os
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from sortmerna_b200 import api, hostio  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
N_WORKLOAD = 20000
N_AMPLICONS = 3000
HEAD_ROWS = 20


def workload(d):
    """bench_workload: (database FASTA paths, reads FASTQ, index options); the reads come from bench.py's CPU generator"""
    import bench
    from tools import synth_databases
    fastas = synth_databases.write(os.path.join(d, "db"))
    refs = [hostio.load_references(f) for f in fastas]
    reads = bench._gen_reads_numpy(bench.DbPool(refs), N_WORKLOAD, bench.GEN_SEED + 4242)
    fq = os.path.join(d, "wl.fq")
    bench.write_fastq(fq, reads)
    return fastas, fq, {}


def amplicons(d):
    """set2_amplicon: amplicons sampled from tests/golden/db_bac.fasta, forward strand, 1 % substitutions, indexed with -max_pos 250"""
    fasta = os.path.join(GOLDEN, "db_bac.fasta")
    refs = hostio.load_references(fasta)
    rng = np.random.default_rng(550)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    out = []
    for i in range(N_AMPLICONS):
        k = int(rng.integers(0, refs.n))
        a, b = int(refs.off[k]), int(refs.off[k + 1])
        ln = int(rng.integers(150, 251))
        st = a + int(rng.integers(0, b - a - ln + 1))
        s = refs.cat[st:st + ln].copy()
        s[s > 3] = rng.integers(0, 4, int((s > 3).sum()), dtype=np.uint8)
        sub = rng.random(ln) < 0.01
        s[sub] = (s[sub] + rng.integers(1, 4, int(sub.sum()), dtype=np.uint8)) & 3
        out.append(b">amplicon_%d\n%s\n" % (i, acgt[s].tobytes()))
    fa = os.path.join(d, "amplicons.fasta")
    with open(fa, "wb") as f:
        f.write(b"".join(out))
    return [fasta], fa, {"max_pos": 250}


def mates_vs_8(d):
    """set4_mates: both golden mate files (integration_common.golden_mates) as one read file against 8 databases: the two golden
    slices the reads come from, then six of the stand-ins (arc-16s ... rfam-5.8s)"""
    from integration_common import golden_mates
    from tools import synth_databases
    fastas = [os.path.join(GOLDEN, "db_arc.fasta"), os.path.join(GOLDEN, "db_bac.fasta")] + synth_databases.write(os.path.join(d, "db"))[2:]
    fq = os.path.join(d, "mates.fq")
    with open(fq, "wb") as f:
        for m in golden_mates(d):
            f.write(open(m, "rb").read())
    return fastas, fq, {}


CASES = {"bench_workload": workload, "set2_amplicon": amplicons, "set4_mates": mates_vs_8}


def rows_digest(rows):
    return hashlib.sha256("\n".join(sorted(rows)).encode()).hexdigest()


def run_gpu(fastas, reads, minimal_score, d, native_kw):
    from tools import stage_data
    idx_dir, _ = stage_data.ensure_indexes(fastas, os.path.join(d, "idx"), **native_kw)
    pre = hostio.find_index_prefixes(idx_dir)
    refs = [hostio.load_references(f) for f in fastas]
    al = api.Aligner(0)
    al.set_params(api.default_params())
    for k, f in enumerate(fastas):
        p = pre[os.path.basename(f)]
        al.load_index_part(k, 0, p, refs[k], minimal_score[k], (18, 9, 3), hostio.parse_stats(p).lnwin)
    batch = hostio.load_reads(reads)
    got = al.align(batch.cat, batch.off)
    rows = hostio.format_sam_rows(batch, refs, got["res"], got["alns"], got["cigar"], got["slots"])
    al.close()
    return got, rows, batch.n


def check_case(case):
    exp = json.load(open(os.path.join(GOLDEN, case + ".json")))
    with tempfile.TemporaryDirectory(prefix="smr_set_") as d:
        fastas, reads, kw = CASES[case](d)
        got, rows, n = run_gpu(fastas, reads, exp["minimal_score"], d, kw)
    assert exp["passing"] + exp["failing"] == n
    assert int(got["res"]["is_hit"].sum()) == exp["passing"]
    srt = sorted(rows)
    first_diff = next(((i, a, b) for i, (a, b) in enumerate(zip(srt, exp["sam_head"])) if a != b), None)
    assert first_diff is None, f"sorted SAM row {first_diff[0]} differs:\n got  {first_diff[1]}\n want {first_diff[2]}"
    assert len(rows) == exp["sam_rows"]
    assert rows_digest(rows) == exp["sam_sha256"], "SAM rows beyond the stored head differ from the reference's"
    if case == "bench_workload":
        assert 0.5 < exp["passing"] / n < 0.8          # two thirds of the workload derive from the databases
    elif case == "set2_amplicon":
        assert exp["passing"] / n > 0.99               # amplicons of the database: all but a handful align
    else:
        assert exp["passing"] / n > 0.5                # most golden reads derive from the golden slices


@pytest.mark.gpu
def test_bench_workload_sample_vs_reference():
    check_case("bench_workload")


@pytest.mark.gpu
def test_set2_amplicon_vs_bac16s_id85():
    check_case("set2_amplicon")


@pytest.mark.gpu
def test_set4_paired_vs_8_databases():
    check_case("set4_mates")


if __name__ == "__main__":     # regenerate tests/golden/<case>.json with the reference binary (CPU)
    from oracle import ora
    from tools import stage_data
    for case, make in sorted(CASES.items()):
        if sys.argv[1:] and case not in sys.argv[1:]:
            continue
        with tempfile.TemporaryDirectory(prefix="smr_set_") as d:
            fastas, reads, kw = make(d)
            extra = ("-max_pos", str(kw["max_pos"])) if "max_pos" in kw else ()
            ref_idx, _ = stage_data.ensure_indexes(fastas, os.path.join(d, "idx_ref"), extra=extra, builder="reference")
            r = ora.run_reference(fastas, reads, os.path.join(d, "w"), extra=["-sam", "-fastx", "-other"] + list(extra),
                                  threads=os.cpu_count() or 8, idx_dir=ref_idx)
            log = ora.parse_log(r["log"])
            sam = ora.read_sam_rows(os.path.join(r["out_dir"], "aligned.sam"))
        out = dict(reads=log["passing"] + log["failing"], passing=log["passing"], failing=log["failing"], minimal_score=log["minimal_score"],
                   sam_rows=len(sam), sam_sha256=rows_digest(sam), sam_head=sorted(sam)[:HEAD_ROWS])
        with open(os.path.join(GOLDEN, case + ".json"), "w") as f:
            json.dump(out, f, indent=1)
            f.write("\n")
        print(case, {k: v for k, v in out.items() if k != "sam_head"})
