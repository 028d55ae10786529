"""The drop-in, end to end on the GPU: the unmodified reference host program linked with integration/align_gpu.cpp and the
PRODUCT library (oracle/_ref/sortmerna_gpu) writes the files the reference binary writes for the same command line."""
import os
import shutil
import tempfile

import pytest

from conftest import GOLDEN
from integration_common import REF_DIR, assert_same_outputs, golden_mates, run_host

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("extra", [[], ["-num_alignments", "3"]], ids=["default", "best3"])
def test_reference_host_with_gpu_library(extra):
    for b in ("sortmerna_ref", "sortmerna_gpu"):
        if not os.path.exists(os.path.join(REF_DIR, b)):
            pytest.skip(f"oracle/_ref/{b} not built (oracle/Makefile.ref)")
    d = tempfile.mkdtemp(prefix="smr_integ_gpu_")
    try:
        reads = [os.path.join(GOLDEN, "reads_mix.fq")]
        rep = ["-sam", "-blast", "1 cigar qcov qstrand", "-fastx", "-other"]
        ref, _ = run_host("sortmerna_ref", os.path.join(d, "ref"), reads, rep + extra)
        got, log = run_host("sortmerna_gpu", os.path.join(d, "got"), reads, rep + extra)
        assert "Starting alignment (libsmr_b200)" in log
        assert_same_outputs(got, ref)
    finally:
        shutil.rmtree(d, ignore_errors=True)


def test_reference_t9_golden_sam_rows_on_gpu():
    """scripts/test.jinja t9 (exact SAM rows, forward + reverse-complement reference) through the drop-in host program"""
    from test_integration_binding import T9_ROWS, run_t9
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_gpu")):
        pytest.skip("oracle/_ref/sortmerna_gpu not built")
    assert run_t9("sortmerna_gpu") == T9_ROWS


def test_reference_t5_mate_pairs_known_answer():
    """Shaped like the reference's t5 (scripts/test.jinja): two mate files given as two -reads (paired feed, 5 threads) against a
    16S database indexed with -max_pos 250 -- here the golden mates against the golden bacterial slice.  The drop-in host program
    on the GPU writes the totals and the aligned / other read files the reference binary writes."""
    import subprocess
    from tools import stage_data
    for b in ("sortmerna_ref", "sortmerna_gpu"):
        if not os.path.exists(os.path.join(REF_DIR, b)):
            pytest.skip(f"oracle/_ref/{b} not built")
    fasta = os.path.join(GOLDEN, "db_bac.fasta")
    d = tempfile.mkdtemp(prefix="smr_t5_")
    try:
        reads = golden_mates(d)
        idx, _ = stage_data.ensure_indexes([fasta], os.path.join(d, "idx"), extra=("-max_pos", "250"), builder="reference")
        outs = {}
        for b in ("sortmerna_ref", "sortmerna_gpu"):
            wd = os.path.join(d, b)
            cmd = [os.path.join(REF_DIR, b), "-ref", fasta, "-reads", reads[0], "-reads", reads[1], "-max_pos", "250", "-fastx", "-other", "-threads", "5",
                   "-workdir", wd, "-idx-dir", idx, "-task", "4"]
            p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
            assert p.returncode == 0, p.stdout[-2000:]
            log = open(os.path.join(wd, "out", "aligned.log")).read()
            outs[b] = ([ln for ln in log.split("\n") if "E-value threshold" in ln or "Total reads =" in ln],
                       {fn: open(os.path.join(wd, "out", fn)).read() for fn in os.listdir(os.path.join(wd, "out")) if fn.endswith(".fq")})
        assert any("passing E-value threshold" in ln for ln in outs["sortmerna_ref"][0])
        assert outs["sortmerna_gpu"][0] == outs["sortmerna_ref"][0]
        assert outs["sortmerna_gpu"][1] == outs["sortmerna_ref"][1]
    finally:
        shutil.rmtree(d, ignore_errors=True)


def _run_binary(binary, fastas, reads, idx, wd, extra, threads=8, env=None):
    import subprocess
    cmd = [os.path.join(REF_DIR, binary)] + sum((["-ref", f] for f in fastas), []) + sum((["-reads", r] for r in reads), []) + \
          ["-workdir", wd, "-idx-dir", idx, "-threads", str(threads), "-task", "4"] + list(extra)
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800, env=env)
    assert p.returncode == 0, p.stdout[-3000:]
    out = os.path.join(wd, "out")
    files = {}
    import gzip
    for fn in sorted(os.listdir(out)):
        path = os.path.join(out, fn)
        text = gzip.open(path, "rt", errors="replace").read() if fn.endswith(".gz") else open(path, errors="replace").read()   # gz input -> gz reports
        lines = text.split("\n")
        fn = fn[:-3] if fn.endswith(".gz") else fn
        if fn.endswith(".sam"):
            lines = sorted(ln for ln in lines if ln and not ln.startswith("@"))   # several references: row order depends on the slot count (SURVEY 8(c))
        elif fn.endswith(".log"):
            lines = [ln for ln in lines if "E-value threshold" in ln or "Total reads =" in ln]
        files[fn] = lines
    return files, p.stdout


def test_baseline_config4_through_the_binary():
    """BASELINE config 4 in small, through the CLI of the drop-in host program: paired .fastq.gz mates (the golden reads split in
    two and gzipped) against the two golden slices, -sam -fastx -other -paired_in (gz inflate + paired feed + report stage) --
    identical totals, SAM rows and aligned / other reads to the unmodified reference binary; and the same with the index built
    on the GPU from the FASTA file (SMR_INDEX_DEVICE=1) instead of read from the index files.  The two slices are one database
    here: with several, a read the reference marks done in an earlier index makes its paired feed pair the wrong mates in the
    next (the documented deviation, test_paired_feed_deviation_is_pinned), which the binding does not reproduce."""
    from tools import stage_data
    for b in ("sortmerna_ref", "sortmerna_gpu"):
        if not os.path.exists(os.path.join(REF_DIR, b)):
            pytest.skip(f"oracle/_ref/{b} not built")
    d = tempfile.mkdtemp(prefix="smr_cfg4_")
    try:
        fastas = [os.path.join(d, "db_arc_bac.fasta")]
        with open(fastas[0], "wb") as f:
            for n in ("db_arc.fasta", "db_bac.fasta"):
                f.write(open(os.path.join(GOLDEN, n), "rb").read())
        reads = golden_mates(d, gz=True)
        idx, _ = stage_data.ensure_indexes(fastas, os.path.join(d, "idx"), builder="reference")
        extra = ["-sam", "-fastx", "-other", "-paired_in"]
        ref, _ = _run_binary("sortmerna_ref", fastas, reads, idx, os.path.join(d, "ref"), extra)
        got, log = _run_binary("sortmerna_gpu", fastas, reads, idx, os.path.join(d, "got"), extra)
        assert "Starting alignment (libsmr_b200)" in log
        assert any("passing E-value threshold" in ln for ln in ref["aligned.log"])
        assert sorted(got) == sorted(ref)
        for fn in got:
            assert got[fn] == ref[fn], fn
        dev, log = _run_binary("sortmerna_gpu", fastas, reads, idx, os.path.join(d, "dev"), extra, env=dict(os.environ, SMR_INDEX_DEVICE="1"))
        assert "Starting alignment (libsmr_b200)" in log
        for fn in ref:
            assert dev[fn] == ref[fn], "device-built index: " + fn
    finally:
        shutil.rmtree(d, ignore_errors=True)


def test_two_gpus_equal_one_gpu(monkeypatch):
    """SMR_GPUS=2 (one context and one worker thread per GPU, batches in flight concurrently) writes what SMR_GPUS=1 writes:
    the golden reads vs the two golden databases in 64-read batches, so that both GPUs get several.  Needs two devices; skips
    on a machine with one."""
    from sortmerna_b200 import api
    if api.load_library().smr_device_count() < 2:
        pytest.skip("needs two GPUs")
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_gpu")):
        pytest.skip("oracle/_ref/sortmerna_gpu not built")
    d = tempfile.mkdtemp(prefix="smr_2gpu_")
    try:
        reads = [os.path.join(GOLDEN, "reads_mix.fq")]
        extra = ["-sam", "-fastx", "-other"]
        monkeypatch.setenv("SMR_BATCH_READS", "64")
        monkeypatch.setenv("SMR_GPUS", "1")
        one, _ = run_host("sortmerna_gpu", os.path.join(d, "g1"), reads, extra)
        monkeypatch.setenv("SMR_GPUS", "2")
        two, log = run_host("sortmerna_gpu", os.path.join(d, "g2"), reads, extra)
        assert "resident on 2 GPU(s)" in log
        for fn in one:
            assert one[fn] == two[fn], fn
    finally:
        shutil.rmtree(d, ignore_errors=True)
