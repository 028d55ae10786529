#!/usr/bin/env python
"""Regenerates tests/golden/stream_counts.json: what the UNMODIFIED reference binary (oracle/_ref/sortmerna_ref, -threads 1) writes
to aligned.log -- "Total reads", and per index the Gumbel lambda / K and the minimal SW score -- for read files whose counts follow
the quirks of Readfeed::count_reads_parallel: the golden FASTQ, its .fastq.gz, the golden mates (two files, flat and gzip), a
multi-line FASTA and a CR LF FASTQ.  tests/test_gpu_stream.py checks Aligner.read_counts against these numbers.

Usage: python tests/golden/make_stream_counts.py
"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def inputs(d):
    """{name: [read file paths]}, written under d; deterministic"""
    import gzip

    from integration_common import golden_mates
    fq = open(os.path.join(HERE, "reads_mix.fq"), "rb").read()
    out = {}

    def put(name, data, gz=False):
        p = os.path.join(d, name)
        with (gzip.open(p, "wb", compresslevel=6) if gz else open(p, "wb")) as f:
            f.write(data)
        return p

    out["golden_fq"] = [put("reads.fq", fq)]
    out["golden_fq_gz"] = [put("reads.fq.gz", fq, gz=True)]
    md, mz = os.path.join(d, "mates"), os.path.join(d, "mates_gz")
    os.makedirs(md, exist_ok=True)
    os.makedirs(mz, exist_ok=True)
    out["mates"] = golden_mates(md)
    out["mates_gz"] = golden_mates(mz, gz=True)
    lines = fq.split(b"\n")
    fa = []
    for i in range(0, len(lines) - 3, 4):
        if not lines[i].startswith(b"@"):
            continue
        seq = lines[i + 1]
        fa.append(b">" + lines[i][1:] + b"\n" + b"".join(seq[k:k + 60] + b"\n" for k in range(0, len(seq), 60)))
    out["multiline_fasta"] = [put("reads_ml.fasta", b"".join(fa))]
    out["crlf"] = [put("reads_crlf.fq", fq.replace(b"\n", b"\r\n"))]
    return out


def main():
    from oracle import ora
    if not ora.have_reference_binary():
        sys.exit("oracle/_ref/sortmerna_ref missing: make -C oracle -f Makefile.ref")
    refs = [os.path.join(HERE, "db_arc.fasta"), os.path.join(HERE, "db_bac.fasta")]
    res = {}
    with tempfile.TemporaryDirectory(prefix="smr_stream_counts_") as d:
        idx = os.path.join(d, "idx")
        for name, paths in inputs(d).items():
            wd = os.path.join(d, "wd_" + name)
            r = ora.run_reference(refs, paths, wd, threads=1, idx_dir=idx)
            log = ora.parse_log(r["log"])
            res[name] = dict(total_reads=log["total_reads"], lambda_=log["lambda_"], K=log["K"], minimal_score=log["minimal_score"])
            print(name, res[name])
    with open(os.path.join(HERE, "stream_counts.json"), "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
