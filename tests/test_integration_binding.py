"""The reference-side binding (integration/align_gpu.cpp): the UNMODIFIED reference host program -- CLI, Readfeed, Refstats,
KVDB, summary, report writers -- linked with the binding in place of its align() must write the files the reference writes:
aligned.sam, aligned.blast, aligned.fq, other.fq byte for byte, aligned.log apart from time stamps.
On a box without a GPU the C ABI behind the binding is the oracle-backed stand-in oracle/capi_oracle_mock.cpp (TEST ONLY), which
checks the binding itself (feed order incl. paired files, KVDB keys / blobs, counters, index and reference hand-over);
tests/test_gpu_integration.py runs the same comparison with the product library on the GPU."""
import os
import shutil
import tempfile

import pytest

from conftest import GOLDEN
from integration_common import REF_DIR, assert_same_outputs, run_host
from sortmerna_b200 import hostio

need = pytest.mark.skipif(not (os.path.exists(os.path.join(REF_DIR, "sortmerna_ref")) and os.path.exists(os.path.join(REF_DIR, "sortmerna_gpu_mock"))),
                          reason="oracle/_ref host binaries not built (oracle/Makefile.ref)")
REPORTS = ["-sam", "-blast", "1 cigar qcov qstrand", "-fastx", "-other"]


@need
@pytest.mark.parametrize("extra", [[], ["-num_alignments", "3"], ["-no-best", "-num_alignments", "2"], ["-F"], ["-otu_map", "-de_novo_otu", "-id", "0.97", "-coverage", "0.97"],
                                   ["-m", "0.5"], ["-match", "2", "-mismatch", "-4", "-gap_open", "6", "-gap_ext", "3", "-N", "-2", "-edges", "10%"],
                                   ["-num_alignments", "0"]],
                         ids=["default", "best3", "nobest2", "fwd", "denovo", "parts", "scores_edges", "all_alignments"])
def test_host_program_with_binding_writes_reference_outputs(extra):
    d = tempfile.mkdtemp(prefix="smr_integ_")
    try:
        reads = [os.path.join(GOLDEN, "reads_mix.fq")]
        ref, _ = run_host("sortmerna_ref", os.path.join(d, "ref"), reads, REPORTS + extra)
        got, log = run_host("sortmerna_gpu_mock", os.path.join(d, "got"), reads, REPORTS + extra)
        assert "Starting alignment (libsmr_b200)" in log
        assert_same_outputs(got, ref)
    finally:
        shutil.rmtree(d, ignore_errors=True)


@need
@pytest.mark.parametrize("threads", [1, 4])
def test_paired_files(threads):
    """Two reads files (paired, -paired_in): the binding follows the reference's alternating feed order (processor.cpp:104-160).
    Inputs avoid the reference's file-switch quirk (see integration/align_gpu.cpp): no read shorter than the seed and
    -num_alignments 3, so that no read is is_done before the second index pass."""
    d = tempfile.mkdtemp(prefix="smr_integ_")
    try:
        h, s, q = hostio.read_fastx(os.path.join(GOLDEN, "reads_mix.fq"))
        keep = [i for i in range(len(h)) if len(s[i]) >= 18][:600]
        paths = []
        for k in (0, 1):
            p = os.path.join(d, f"r{k + 1}.fq")
            with open(p, "w") as f:
                for i in keep[k * 300:k * 300 + 300]:
                    f.write(f"{h[i]}\n{s[i].decode()}\n+\n{q[i].decode()}\n")
            paths.append(p)
        extra = REPORTS + ["-paired_in", "-num_alignments", "3"]
        ref, _ = run_host("sortmerna_ref", os.path.join(d, "ref"), paths, extra, threads=threads)
        got, _ = run_host("sortmerna_gpu_mock", os.path.join(d, "got"), paths, extra, threads=threads)
        assert_same_outputs(got, ref, ref_threads=threads)
    finally:
        shutil.rmtree(d, ignore_errors=True)


@need
def test_paired_feed_deviation_is_pinned():
    """The documented deviation (integration/align_gpu.cpp): for paired files the reference's align2 `continue`s past its file
    switch for a read it skips in the current index pass (shorter than the seed, or is_done from an earlier index:
    processor.cpp:116-124 vs :160) and from then on pairs the wrong mates; the binding searches every read against every index.
    Pinned here: with one too-short read in file 1 the reference aligns FEWER reads than are alignable, the binding aligns
    exactly the reads the reference aligns when the same reads are given as ONE (unpaired) file -- i.e. the binding's paired
    result equals the quirk-free feed, and the difference to the reference's paired run is the quirk, nothing else."""
    d = tempfile.mkdtemp(prefix="smr_integ_")
    try:
        h, s, q = hostio.read_fastx(os.path.join(GOLDEN, "reads_mix.fq"))
        keep = [i for i in range(len(h)) if len(s[i]) >= 18][:400]
        short = next(i for i in range(len(h)) if len(s[i]) < 18)
        f1, f2 = keep[:200], keep[200:400]
        f1[20] = short                                   # one read shorter than the seed early in file 1
        paths = []
        for k, ids in enumerate((f1, f2)):
            p = os.path.join(d, f"r{k + 1}.fq")
            with open(p, "w") as f:
                for i in ids:
                    f.write(f"{h[i]}\n{s[i].decode()}\n+\n{q[i].decode()}\n")
            paths.append(p)
        both = os.path.join(d, "both.fq")                # the same reads, interleaved as the paired feed delivers them, one file
        with open(both, "w") as f:
            for a, b in zip(f1, f2):
                for i in (a, b):
                    f.write(f"{h[i]}\n{s[i].decode()}\n+\n{q[i].decode()}\n")
        extra = ["-sam", "-num_alignments", "3"]
        ref_paired, _ = run_host("sortmerna_ref", os.path.join(d, "refp"), paths, extra + ["-paired_in"], threads=1)
        got_paired, _ = run_host("sortmerna_gpu_mock", os.path.join(d, "gotp"), paths, extra + ["-paired_in"], threads=1)
        ref_single, _ = run_host("sortmerna_ref", os.path.join(d, "refs"), [both], extra, threads=1)
        rows = lambda o: sorted(ln for ln in o["aligned.sam"] if ln and not ln.startswith("@"))
        assert rows(got_paired) == rows(ref_single)      # the binding = the reference on the quirk-free feed of the same reads
        assert len(rows(ref_paired)) < len(rows(ref_single))   # the reference's own paired run loses reads to the quirk
        assert set(rows(ref_paired)) <= set(rows(ref_single))  # ... and aligns nothing differently
    finally:
        shutil.rmtree(d, ignore_errors=True)


@need
def test_two_gpus_small_batches(monkeypatch):
    """SMR_GPUS=2: one context per GPU, batches dispatched concurrently, results stored in batch order, counters summed -- with
    100-read batches so that several rounds of two batches each happen (the stand-in reports two devices)."""
    d = tempfile.mkdtemp(prefix="smr_integ_")
    try:
        reads = [os.path.join(GOLDEN, "reads_mix.fq")]
        extra = REPORTS + ["-num_alignments", "3"]
        ref, _ = run_host("sortmerna_ref", os.path.join(d, "ref"), reads, extra)
        monkeypatch.setenv("SMR_GPUS", "2"); monkeypatch.setenv("SMR_MOCK_DEVICES", "2"); monkeypatch.setenv("SMR_BATCH_READS", "100")
        got, _ = run_host("sortmerna_gpu_mock", os.path.join(d, "got"), reads, extra)
        assert_same_outputs(got, ref)
    finally:
        shutil.rmtree(d, ignore_errors=True)


T9_ROWS = [   # scripts/test.jinja:447-476 (t9 "test_output_all_alignments_f_rc"): the reference's own golden SAM rows
    ["GQ099317.1.1325_157_453_0:0:0_0:0:0_99/1", "0", "GQ099317.1.1325_157_453_0:0:0_0:0:0_99/1", "1", "255", "101M", "*", "0", "0",
     "GCTGGCACGGAGTTAGCCGGGGCTTATAAATGGTACCGTCATTGATTCTTCCCATTCTTTCGAAGTTTACATCCCGAGGGACTTCATCCTTCACGCGGCGT", "*", "AS:i:202", "NM:i:0"],
    ["GQ099317.1.1325_157_453_0:0:0_0:0:0_99/1", "16", "GQ099317.1.1325_157_453_0:0:0_0:0:0_99/1", "102", "255", "101M", "*", "0", "0",
     "ACGCCGCGTGAAGGATGAAGTCCCTCGGGATGTAAACTTCGAAAGAATGGGAAGAATCAATGACGGTACCATTTATAAGCCCCGGCTAACTCCGTGCCAGC", "*", "AS:i:202", "NM:i:0"],
]


def run_t9(binary):
    """the reference's t9 with its original arguments (scripts/test.jinja:425-445): one read against a reference file holding a
    sequence and its reverse complement, `-num_alignments 0` (all alignments)."""
    import subprocess
    d = tempfile.mkdtemp(prefix="smr_t9_")
    try:
        t9 = os.path.join(GOLDEN, "t9")
        cmd = [os.path.join(REF_DIR, binary), "-ref", os.path.join(t9, "ref_GQ099317_forward_and_rc.fasta"), "-reads", os.path.join(t9, "illumina_GQ099317.fasta"),
               "-num_alignments", "0", "-mismatch", "-3", "-sam", "-v", "-workdir", d, "-threads", "1", "-task", "4"]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
        assert p.returncode == 0, p.stdout[-2000:]
        return [ln.rstrip("\n").split("\t") for ln in open(os.path.join(d, "out", "aligned.sam")) if not ln.startswith("@")]
    finally:
        shutil.rmtree(d, ignore_errors=True)


@need
def test_reference_t9_golden_sam_rows():
    assert run_t9("sortmerna_gpu_mock") == T9_ROWS
    assert run_t9("sortmerna_ref") == T9_ROWS


@need
def test_reference_known_answers_t5_t11():
    """Shaped like the reference's t5 (two mate files, paired feed, 5 threads, a 16S database indexed with -max_pos 250) and t11
    (-id 0.97 -coverage 0.97 -otu_map -de_novo_otu -blast, 3 threads), on the golden mates / reads against the golden bacterial
    slice: the host program with the binding writes the totals of the reference binary (t5) and its whole aligned.log (t11,
    incl. 'Total reads for de novo clustering')."""
    import re
    import subprocess
    from integration_common import golden_mates
    d = tempfile.mkdtemp(prefix="smr_kat_")
    fasta = os.path.join(GOLDEN, "db_bac.fasta")

    def run(binary, name, args):
        wd = os.path.join(d, name + binary)
        p = subprocess.run([os.path.join(REF_DIR, binary)] + args + ["-workdir", wd, "-task", "4"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3000)
        assert p.returncode == 0, p.stdout[-2000:]
        return [ln for ln in open(os.path.join(wd, "out", "aligned.log")).read().split("\n") if not re.search(r"Time|time|Command|pid|/tmp/|Date|sec|\d\d:\d\d:\d\d", ln)]
    try:
        m1, m2 = golden_mates(d, gz=True)
        t5 = ["-ref", fasta, "-reads", m1, "-reads", m2, "-max_pos", "250", "-fastx", "-other", "-threads", "5"]
        a, b = run("sortmerna_gpu_mock", "t5", t5), run("sortmerna_ref", "t5", t5)
        totals = lambda log: [ln for ln in log if "E-value threshold" in ln or "Total reads =" in ln]
        assert any("passing E-value threshold" in ln for ln in totals(b)) and totals(a) == totals(b)
        t11 = ["-ref", fasta, "-reads", os.path.join(GOLDEN, "reads_mix.fq"), "-id", "0.97", "-coverage", "0.97",
               "-otu_map", "-de_novo_otu", "-blast", "1 cigar qcov", "-fastx", "-other", "-threads", "3"]
        a, b = run("sortmerna_gpu_mock", "t11", t11), run("sortmerna_ref", "t11", t11)
        assert any("Total reads for de novo clustering" in ln for ln in b)
        assert a == b
    finally:
        shutil.rmtree(d, ignore_errors=True)
