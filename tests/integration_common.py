"""Run a sortmerna host binary (the reference, or the reference linked with integration/align_gpu.cpp) and normalise its output
files for comparison."""
import os
import re
import subprocess

from conftest import GOLDEN, ROOT

REF_DIR = os.path.join(ROOT, "oracle", "_ref")
_VOLATILE = re.compile(r"Time|time|Command|Process pid|/tmp/|Date|sec|\d\d:\d\d:\d\d")


def run_host(binary, workdir, reads, extra, threads=2):
    cmd = [os.path.join(REF_DIR, binary), "-ref", os.path.join(GOLDEN, "db_arc.fasta"), "-ref", os.path.join(GOLDEN, "db_bac.fasta")]
    for r in reads:
        cmd += ["-reads", r]
    cmd += ["-workdir", workdir, "-threads", str(threads), "-task", "4"] + list(extra)
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:]
    out = {}
    d = os.path.join(workdir, "out")
    for fn in sorted(os.listdir(d)):
        lines = open(os.path.join(d, fn), errors="replace").read().split("\n")
        if fn.endswith(".log"):
            lines = [ln for ln in lines if not _VOLATILE.search(ln)]
        elif fn.endswith(".sam"):
            lines = [ln for ln in lines if not ln.startswith("@PG")]       # carries the command line
        out[fn] = lines
    return out, p.stdout


_PER_DB = re.compile(r"^(\s+\S+\.fasta\t+)([0-9.]+)\s*$")


def assert_same_outputs(a, b, ref_threads=2):
    """a: our run, b: the reference binary's.  With several threads the reference's "Coverage by database" figures come from
    ++readstats.reads_matched_per_db[...] without synchronisation (src/sortmerna/alignment.cpp:415,454-457; SURVEY section 5): now and
    then a run loses an update (66.33 % instead of 66.67 % of 300 reads).  Those lines are compared with a tolerance of one
    percentage point then, and exactly when the reference ran single-threaded (ref_threads=1); everything else is always exact."""
    assert sorted(a) == sorted(b), (sorted(a), sorted(b))
    for fn in a:
        x, y = list(a[fn]), list(b[fn])
        if ref_threads > 1 and fn.endswith(".log") and len(x) == len(y):
            for i, (p, q) in enumerate(zip(x, y)):
                mp, mq = _PER_DB.match(p), _PER_DB.match(q)
                if mp and mq and mp.group(1) == mq.group(1) and abs(float(mp.group(2)) - float(mq.group(2))) <= 1.0:
                    y[i] = p
        assert x == y, f"{fn} differs: first difference {next((p, q) for p, q in zip(x, y) if p != q)}"


def golden_mates(d, gz=False):
    """The reads of tests/golden/reads_mix.fq that are at least one seed (18 nt) long, split into two mate files (alternate records),
    flat or gzip -6: the inputs of the paired-feed tests, shaped like the reference's set4_mate_pairs_metatranscriptomics_{1,2}.fastq(.gz),
    which hold no read shorter than a seed (a shorter one triggers the reference's documented paired-feed quirk,
    test_paired_feed_deviation_is_pinned)."""
    import gzip
    lines = open(os.path.join(GOLDEN, "reads_mix.fq"), "rb").read().split(b"\n")
    recs = [b"\n".join(lines[i:i + 4]) + b"\n" for i in range(0, len(lines) - 3, 4) if lines[i].startswith(b"@") and len(lines[i + 1]) >= 18]
    recs = recs[: len(recs) // 2 * 2]
    paths = []
    for k in (0, 1):
        p = os.path.join(d, f"mates_{k + 1}.fastq" + (".gz" if gz else ""))
        data = b"".join(recs[k::2])
        with (gzip.open(p, "wb", compresslevel=6) if gz else open(p, "wb")) as f:
            f.write(data)
        paths.append(p)
    return paths
