"""python -m sortmerna_b200 (api.run_files) against the reference binary (oracle/_ref/sortmerna_ref) run with the same options at
-threads 1 on the golden databases and reads, with lambda, K and the minimal scores of the reference's log passed as -gumbel and
-minimal_score.  Every file of out/ must be equal byte for byte, except: BLAST E-values may differ by one unit of their third
digit (the log holds lambda and K to 6 digits, the reference computes with all of them; tests/helpers.py); aligned.log is compared
after summary_common.strip_volatile (command line, pid, time); gzip files are compared inflated (the device encoder's bytes are
not zlib's, DESIGN 5e); and the @PG line of aligned.sam carries each program's own command line.  Several batches write what one
batch writes."""
import gzip
import os
import shutil
import tempfile

import pytest

from conftest import GOLDEN
from integration_common import REF_DIR, golden_mates
from sortmerna_b200 import __main__ as cli
from sortmerna_b200 import api
from summary_common import log_inputs, strip_volatile

pytestmark = pytest.mark.gpu

REFS = [os.path.join(GOLDEN, "db_arc.fasta"), os.path.join(GOLDEN, "db_bac.fasta")]
READS = os.path.join(GOLDEN, "reads_mix.fq")
CASES = {
    "sam_blast_fastx": ["-sam", "-blast", "1 cigar qcov qstrand", "-fastx", "-other"],
    "gz_zip_out": ["-zip-out", "-sam", "-blast", "1 cigar qcov qstrand", "-fastx", "-other"],
    "mates_paired_in_out2": ["-paired_in", "-out2", "-fastx", "-other"],
    "otu_denovo": ["-otu_map", "-de_novo_otu", "-id", "0.9", "-coverage", "0.9", "-fastx"],
    "blast_pairwise": ["-blast", "0"],
    "all_alignments": ["-num_alignments", "0", "-sam", "-blast", "1", "-fastx"],
}


def _need_ref():
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_ref")):
        pytest.skip("oracle/_ref/sortmerna_ref not built (oracle/Makefile.ref)")


def _reads(name, d):
    if name == "gz_zip_out":
        p = os.path.join(d, "reads_mix.fq.gz")
        with open(p, "wb") as f:
            f.write(gzip.compress(open(READS, "rb").read(), 6))
        return [p]
    if name.startswith("mates"):
        return golden_mates(d)
    return [READS]


def _ours(reads, extra, inp, workdir):
    args = [a for r in REFS for a in ("-ref", r)] + [a for r in reads for a in ("-reads", r)] + ["-workdir", workdir, "-threads", "1"]
    for lam, K in inp["gumbel"]:
        args += ["-gumbel", f"{lam},{K}"]
    for m in inp["minimal_score"]:
        args += ["-minimal_score", str(m)]
    return args + list(extra)


def _close_numbers(x: str, y: str) -> bool:
    """x and y alike but for numbers that differ by at most one unit of their third significant digit (BLAST E-values)"""
    fx, fy = x.replace("\t", " ").split(" "), y.replace("\t", " ").split(" ")
    if len(fx) != len(fy):
        return False
    for a, b in zip(fx, fy):
        if a == b:
            continue
        try:
            u, v = float(a), float(b)
        except ValueError:
            return False
        if abs(u - v) > 1.2e-2 * max(abs(v), 1e-300) + 1e-300:
            return False
    return True


def assert_same_out(ours_dir, ref_dir, our_cmd):
    names = sorted(os.listdir(ref_dir))
    assert sorted(os.listdir(ours_dir)) == names
    for fn in names:
        a, b = open(os.path.join(ours_dir, fn), "rb").read(), open(os.path.join(ref_dir, fn), "rb").read()
        if fn.endswith(".gz"):
            a, b = gzip.decompress(a), gzip.decompress(b)
        base = fn[:-3] if fn.endswith(".gz") else fn
        if base == "aligned.log":
            assert strip_volatile(a.decode()) == strip_volatile(b.decode()), fn
        elif base == "aligned.sam":
            la, lb = a.decode().split("\n"), b.decode().split("\n")
            pa, pb = [i for i, ln in enumerate(la) if ln.startswith("@PG")], [i for i, ln in enumerate(lb) if ln.startswith("@PG")]
            assert pa == pb and len(pa) == 1 and la[pa[0]] == "@PG\tID:sortmerna\tVN:1.0\tCL:" + our_cmd, fn
            del la[pa[0]], lb[pb[0]]
            assert la == lb, fn
        elif base == "aligned.blast":
            la, lb = a.decode().split("\n"), b.decode().split("\n")
            assert len(la) == len(lb), fn
            bad = [(x, y) for x, y in zip(la, lb) if x != y and not _close_numbers(x, y)]
            assert not bad, (fn, bad[:3])
        else:
            assert a == b, fn


@pytest.mark.parametrize("name", sorted(CASES))
def test_cli_against_reference_binary(golden_idx_dir, name):
    _need_ref()
    from oracle import ora
    d = tempfile.mkdtemp(prefix="smr_runfiles_")
    try:
        reads = _reads(name, d)
        r = ora.run_reference(REFS, reads, os.path.join(d, "ref"), extra=CASES[name], threads=1, idx_dir=golden_idx_dir)
        inp = log_inputs(r["log"])
        args = _ours(reads, CASES[name], inp, os.path.join(d, "ours"))
        assert cli.main(args) == 0
        cmd = "".join(a + " " for a in ["python -m sortmerna_b200"] + args)
        assert_same_out(os.path.join(d, "ours", "out"), r["out_dir"], cmd)
    finally:
        shutil.rmtree(d, ignore_errors=True)


@pytest.mark.parametrize("name", ["sam_blast_fastx", "mates_paired_in_out2", "otu_denovo"])
def test_three_batches_write_what_one_batch_writes(name, tmp_path):
    reads = _reads(name, str(tmp_path))
    inp = dict(gumbel=[(0.594908, 0.326193), (0.600371, 0.328947)], minimal_score=[37, 36])
    out = {}
    for k, bb in (("one", 1 << 30), ("three", sum(os.path.getsize(p) for p in reads) // 3 + 1)):
        kw = cli.parse_args(_ours(reads, CASES[name], inp, str(tmp_path / k)))
        kw.pop("workdir")
        r = api.run_files(batch_bytes=bb, piece_bytes=4096, cmd="x ", **kw)
        out[k] = {os.path.basename(p): open(p, "rb").read() for p in r["paths"]}
        out[k]["aligned.log"] = strip_volatile(out[k]["aligned.log"].decode())
        out[k]["_reads"] = r["reads"]
        if k == "three":
            assert r["batches"] >= 3
    assert out["three"] == out["one"] and out["one"]["_reads"] > 0
