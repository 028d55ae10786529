#!/usr/bin/env python
"""Regenerates the pairwise BLAST fixtures (-blast 0, report_blast.cpp:136-251) from the reference binary
(oracle/_ref/sortmerna_ref -threads 1 -blast 0 -sam) on the committed golden databases, with the golden index (tests/golden/idx):

  blast_pairwise/<case>.blast.gz   the reference's aligned.blast, gzip-compressed
  blast_pairwise.json              per case: databases, reads file, arguments, and the aligned.log numbers (Gumbel lambda / K, minimal
                                   SW scores) a restatement needs to print the same rows
  blast_pairwise_edges.fasta       the synthetic reads of the "edges" case, cut from db_bac.fasta

Cases:
  default         db_bac.fasta, default options
  best3_both      both databases, -num_alignments 3 (reads up to 1,400 nt: many blocks per row)
  scores_exotic   both databases, the scoring of case_scores_exotic (other bit scores and E-values)
  edges           db_bac.fasta on reads made to hit the block edges: alignments of exactly 60 and 120 columns, an I and a D at
                  columns 58 to 61, a block of I columns only, N in a read, the minus strand, and a read over 2,000 nt.  The
                  script checks in the reference's aligned.sam that each of these shapes is there.

Usage: python tests/golden/make_blast_pairwise_golden.py
"""
import gzip
import json
import os
import re
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ora  # noqa: E402
from sortmerna_b200 import hostio  # noqa: E402

SEED = 20261017
EDGES = "blast_pairwise_edges.fasta"
CASES = {
    "default": dict(dbs=["db_bac.fasta"], reads="reads_mix.fq", args=[]),
    "best3_both": dict(dbs=["db_arc.fasta", "db_bac.fasta"], reads="reads_mix.fq", args=["-num_alignments", "3"]),
    "scores_exotic": dict(dbs=["db_arc.fasta", "db_bac.fasta"], reads="reads_mix.fq",
                          args=["-match", "2", "-mismatch", "-7", "-gap_open", "3", "-gap_ext", "1"]),
    "edges": dict(dbs=["db_bac.fasta"], reads=EDGES, args=[]),
}


def _rc(s):
    return s.translate(str.maketrans("ACGTN", "TGCAN"))[::-1]


def make_edge_reads():
    """(name, sequence) of the edges case, from db_bac.fasta"""
    rng = np.random.default_rng(SEED)
    _, seqs, _ = hostio.read_fastx(os.path.join(HERE, "db_bac.fasta"))
    refs = [s.decode().upper() for s in seqs]
    rand = lambda n: "".join("ACGT"[k] for k in rng.integers(0, 4, n))  # noqa: E731
    out = []
    for k, ln in enumerate((60, 120)):
        out.append((f"exact{ln}_fwd", refs[k][100:100 + ln]))
        out.append((f"exact{ln}_rev", _rc(refs[k + 2][300:300 + ln])))
    for col in (58, 59, 60, 61):
        r = refs[10 + col - 58]
        s = next(s for s in range(50, 900) if r[s + col - 1] != r[s + col] != r[s + col + 1] and r[s + col - 1] != r[s + col + 1])
        x = next(c for c in "ACGT" if c not in (r[s + col - 1], r[s + col]))
        out.append((f"ins_at_{col}", r[s:s + col] + x + r[s + col:s + 200]))
        out.append((f"del_at_{col}", r[s:s + col] + r[s + col + 1:s + 201]))
        out.append((f"del_at_{col}_rev", _rc(r[s:s + col] + r[s + col + 1:s + 201])))
    r = refs[20]
    out.append(("ins_block", r[200:490] + rand(70) + r[490:760]))   # I columns 290..359: block 300..359 holds I columns only
    r = list(refs[21][150:400])
    for p in (0, 37, 119, 120, 200):
        r[p] = "N"
    out.append(("with_n", "".join(r)))
    out.append(("with_n_rev", _rc("".join(r))))
    long_ref = max(range(len(refs)), key=lambda i: len(refs[i]))
    out.append(("long_2150", refs[long_ref][:1500] + rand(650)))
    out.append(("long_2150_rev", _rc(rand(300) + refs[long_ref][20:1560] + rand(400))))
    return out


def _cigar_cols(cig):
    return [(int(n), op) for n, op in re.findall(r"(\d+)([MIDS])", cig) if op != "S"]


def check_edges(sam_rows):
    """every shape the edges case is made for is in the reference's alignments"""
    have = set()
    for row in sam_rows:
        f = row.split("\t")
        ops = _cigar_cols(f[5])
        cols = sum(n for n, _ in ops)
        if cols in (60, 120):
            have.add(f"cols{cols}")
        at = 0
        for n, op in ops:
            if op in "ID":
                for c in range(at, at + n):
                    if 58 <= c <= 61:
                        have.add(f"{op}{c}")
                if op == "I" and any(at <= b and b + 60 <= at + n for b in range(0, at + n, 60)):
                    have.add("I_block")
            at += n
        if "N" in f[9]:
            have.add("N")
        if f[1] == "16":
            have.add("minus")
        if len(f[9]) > 2000:
            have.add("long")
    want = {"cols60", "cols120", "I58", "I59", "I60", "I61", "D58", "D59", "D60", "D61", "I_block", "N", "minus", "long"}
    if want - have:
        sys.exit(f"edges: the reference made no alignment of shape {sorted(want - have)}")


def main():
    if not ora.have_reference_binary():
        sys.exit("oracle/_ref/sortmerna_ref missing: make -C oracle -f Makefile.ref")
    with open(os.path.join(HERE, EDGES), "w") as f:
        f.write("".join(f">{n}\n{s}\n" for n, s in make_edge_reads()))
    tmp = tempfile.mkdtemp(prefix="smr_golden_pw_")
    os.makedirs(os.path.join(HERE, "blast_pairwise"), exist_ok=True)
    out = {}
    try:
        sys.path.insert(0, os.path.dirname(HERE))
        from conftest import unpack_index
        idx = os.path.join(tmp, "idx")
        os.makedirs(idx)
        unpack_index(os.path.join(HERE, "idx"), idx)
        for case, c in CASES.items():
            r = ora.run_reference([os.path.join(HERE, d) for d in c["dbs"]], os.path.join(HERE, c["reads"]), os.path.join(tmp, case),
                                  extra=["-blast", "0", "-sam"] + c["args"], threads=1, idx_dir=idx)
            log = ora.parse_log(r["log"])
            blast = open(os.path.join(r["out_dir"], "aligned.blast"), "rb").read()
            sam = ora.read_sam_rows(os.path.join(r["out_dir"], "aligned.sam"))
            if case == "edges":
                check_edges(sam)
            with gzip.GzipFile(os.path.join(HERE, "blast_pairwise", case + ".blast.gz"), "wb", compresslevel=9, mtime=0) as f:
                f.write(blast)
            out[case] = dict(c, lambda_=log["lambda_"], K=log["K"], minimal_score=log["minimal_score"], rows=len(sam), bytes=len(blast))
            print(case, "rows", len(sam), "bytes", len(blast))
        with open(os.path.join(HERE, "blast_pairwise.json"), "w") as f:
            json.dump(out, f, indent=1)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
