"""Host models of the mate stream and of the paired report routing, without a GPU: the pair cut and the interleave of two mate
texts (smr_stream.cuh, smr_capi.cu mate_cut) restated in numpy, and ReportFastx / ReportFxOther / ReportDenovo::append restated
(as rpt_file_aligned / _other / _denovo of smr_report.cuh) and checked against the reference binary's paired files where it is built."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN
from integration_common import REF_DIR, golden_mates

REF_BIN = os.path.join(REF_DIR, "sortmerna_ref")


def fastq_records(text):
    lines = text.split(b"\n")[:-1]
    return [b"".join(ln + b"\n" for ln in lines[i:i + 4]) for i in range(0, len(lines), 4)]


def record_ends(text):
    """ends of the records of a FASTQ text (after the '\\n' of every line 4r + 3), as the decode's newline index gives them"""
    nl = np.flatnonzero(np.frombuffer(text, np.uint8) == 10)
    return nl[3::4].astype(np.int64) + 1


def pair_cuts(t1, t2, batch_bytes):
    """the batches of the mate stream once both files have ended: k = the most pairs whose interleaved text fits, or 1"""
    ea, eb = record_ends(t1), record_ends(t2)
    assert ea.size == eb.size
    out, a0, b0, k0 = [], 0, 0, 0
    while k0 < ea.size:
        ends = (ea[k0:] - a0) + (eb[k0:] - b0)
        k = max(1, int(np.searchsorted(ends, batch_bytes, side="right")))   # the sums increase: the largest k that fits
        a1, b1 = ea[k0 + k - 1], eb[k0 + k - 1]
        pa, pb = np.concatenate([[a0], ea[k0:k0 + k]]), np.concatenate([[b0], eb[k0:k0 + k]])
        # the interleave: pair p starts at ea[p - 1] + eb[p - 1] of the batch, record of mate 1 first
        buf = np.zeros(int(a1 - a0 + b1 - b0), np.uint8)
        A, B = np.frombuffer(t1, np.uint8), np.frombuffer(t2, np.uint8)
        for p in range(k):
            d = (pa[p] - a0) + (pb[p] - b0)
            la, lb = pa[p + 1] - pa[p], pb[p + 1] - pb[p]
            buf[d:d + la] = A[pa[p]:pa[p + 1]]
            buf[d + la:d + la + lb] = B[pb[p]:pb[p + 1]]
        out.append(buf.tobytes())
        a0, b0, k0 = a1, b1, k0 + k
    return out


def test_pair_cut_and_interleave_model():
    d = tempfile.mkdtemp(prefix="smr_mates_host_")
    try:
        t1, t2 = (open(p, "rb").read() for p in golden_mates(d))
    finally:
        shutil.rmtree(d, ignore_errors=True)
    r1, r2 = fastq_records(t1), fastq_records(t2)
    inter = b"".join(a + b for a, b in zip(r1, r2))
    pair_sizes = [len(a) + len(b) for a, b in zip(r1, r2)]
    for batch in sorted({1, min(pair_sizes) - 1, min(pair_sizes), max(pair_sizes), 1000, 4096, 20000, len(inter) - 1, len(inter), 10 * len(inter)}):
        cuts = pair_cuts(t1, t2, batch)
        assert b"".join(cuts) == inter, batch
        at = 0
        for k, c in enumerate(cuts):
            npairs = len(fastq_records(c)) // 2
            assert len(c) <= batch or npairs == 1, (batch, k)
            at += len(c)
            if k + 1 < len(cuts):   # full: the next pair would not have fit
                nxt = len(fastq_records(cuts[k + 1])[0]) + len(fastq_records(cuts[k + 1])[1])
                assert len(c) + nxt > batch, (batch, k)


# ---- routing: the three append routines at -threads 1, per pair (h0, h1, d0, d1) -> the file index of each mate, or None ----
def route(kind, i, h, hm, d, dm, num_out, out2, paired_in, paired_out):
    if kind == "aligned":   # ReportFastx::append
        both = h and hm
        if not (h or hm):
            return None
        if num_out == 1:
            ok = both if paired_out else (paired_in or h)
            return 0 if ok else None
        if num_out == 2 and out2:
            ok = both if paired_out else (paired_in or h)
            return i if ok else None
        if num_out == 2:
            return 0 if both else 1 if h else None
        return i if both else i + 2 if h else None
    if kind == "other":     # ReportFxOther::append
        anyh = h or hm
        if h and hm:
            return None
        if num_out == 1:
            ok = (not anyh) if paired_in else (paired_out or not h)
            return 0 if ok else None
        if num_out == 2 and out2:
            ok = (not anyh) if paired_in else (paired_out or not h)
            return i if ok else None
        if num_out == 2:
            return 0 if not anyh else 1 if not h else None
        return i if not anyh else i + 2 if not h else None
    # ReportDenovo::append, called when d or dm; idx is carried from the previous mate under -out2 (0 for both mates)
    if not (d or dm):
        return None
    both = d and dm
    if num_out == 1:
        return 0 if (paired_in or d) else None
    if num_out == 2 and out2:
        if paired_out and not both:
            return None
        return i if (paired_in or d) else 0
    if num_out == 2:
        return 0 if both else 1 if d else None
    return i if both else i + 2 if d else None


SUFFIX = {1: [""], 4: ["_paired_fwd", "_paired_rev", "_singleton_fwd", "_singleton_rev"]}


def _run(reads, workdir, extra):
    cmd = [REF_BIN, "-ref", os.path.join(GOLDEN, "db_bac.fasta")]
    for r in reads:
        cmd += ["-reads", r]
    cmd += ["-workdir", workdir, "-threads", "1", "-fastx", "-other", "-otu_map", "-de_novo_otu", "-id", "0.9", "-coverage", "0.9"] + extra
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:]
    return os.path.join(workdir, "out")


@pytest.mark.skipif(not os.path.exists(REF_BIN), reason="oracle/_ref/sortmerna_ref not built (oracle/Makefile.ref)")
def test_routing_model_against_reference_binary():
    """The per-read hit and denovo classes come from the reference's own run of the interleaved file as one unpaired file
    (aligned.fq / aligned_denovo.fq: alignment is per read); the model then predicts every file of its paired runs."""
    d = tempfile.mkdtemp(prefix="smr_mates_route_")
    try:
        mates = golden_mates(d)
        t1, t2 = (open(p, "rb").read() for p in mates)
        r1, r2 = fastq_records(t1), fastq_records(t2)
        inter = os.path.join(d, "inter.fq")
        open(inter, "wb").write(b"".join(a + b for a, b in zip(r1, r2)))
        o = _run([inter], os.path.join(d, "single"), [])
        hit = set(fastq_records(open(os.path.join(o, "aligned.fq"), "rb").read()))
        dn = set(fastq_records(open(os.path.join(o, "aligned_denovo.fq"), "rb").read()))
        assert 0 < len(hit) < 2 * len(r1) and 0 < len(dn)
        for extra in (["-out2"], ["-sout"], ["-out2", "-sout"], ["-paired_in", "-out2"], ["-paired_out", "-out2"], [], ["-paired_in"], ["-paired_out"]):
            out2, sout = "-out2" in extra, "-sout" in extra
            num_out = 4 if out2 and sout else 2 if out2 or sout else 1
            sfx = SUFFIX.get(num_out) or (["_fwd", "_rev"] if out2 else ["_paired", "_singleton"])
            o = _run(mates, os.path.join(d, "_".join(extra) or "plain"), extra)
            for kind, name in (("aligned", "aligned"), ("other", "other"), ("denovo", "aligned_denovo")):
                want = [[] for _ in range(num_out)]
                for a, b in zip(r1, r2):
                    for i, (x, y) in enumerate(((a, b), (b, a))):
                        f = route(kind, i, x in hit, y in hit, x in dn, y in dn, num_out, out2, "-paired_in" in extra, "-paired_out" in extra)
                        if f is not None:
                            want[f].append(x)
                for j, s in enumerate(sfx):
                    got = open(os.path.join(o, f"{name}{s}.fq"), "rb").read()
                    assert got == b"".join(want[j]), (extra, name + s)
    finally:
        shutil.rmtree(d, ignore_errors=True)
