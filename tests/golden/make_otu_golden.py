#!/usr/bin/env python
"""Regenerates tests/golden/otu_map.json from the reference binary (oracle/_ref/sortmerna_ref, -threads 1) on the committed golden
reads and databases: per case the arguments, -id / -coverage, the minimal SW scores, the whole otu_map.txt (null when the reference
wrote none) and the two OTU numbers of aligned.log ("passing %id and %coverage" = n_yid_ycov, "Total OTUs").

Cases:
  default / best3 / rev_only / loose   the option sets of denovo.json (make_golden.DENOVO_CASES)
  none                                  -R -id 1 -coverage 1: no alignment passes, no otu_map.txt
  parts                                 -m 0.5: both databases in 3 index parts
  merged                                db_bac.fasta and a renamed copy of it with -num_alignments 2: the same reference ids in
                                        two indexes, so lines gather reads of both (index, part) groups
  paired_files / paired_interleaved     the golden mates (integration_common.golden_mates) with -paired_in, as two files and as one
                                        interleaved file.  The library refuses paired batches; these record what the binary does.

Usage: python tests/golden/make_otu_golden.py
"""
import json
import os
import re
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ora  # noqa: E402

from make_golden import DENOVO_ARGS, DENOVO_CASES  # noqa: E402

OTU = ["-fastx", "-otu_map", "-de_novo_otu"]


def _run(refs, reads, wd, extra, min_id, min_cov):
    r = ora.run_reference(refs, reads, wd, extra=OTU + ["-id", min_id, "-coverage", min_cov] + extra, threads=1)
    log = ora.parse_log(r["log"])
    p = os.path.join(r["out_dir"], "otu_map.txt")
    text = open(p, "rb").read().decode() if os.path.exists(p) else None
    m = re.search(r"passing %+id and %+coverage thresholds = (\d+)", r["log"])
    t = re.search(r"Total OTUs = (\d+)", r["log"])
    return dict(args=extra, min_id=float(min_id), min_cov=float(min_cov), minimal_score=log["minimal_score"], otu_map=text,
                n_yid_ycov=int(m.group(1)) if m else 0, total_otu=int(t.group(1)) if t else 0)


def main():
    if not ora.have_reference_binary():
        sys.exit("oracle/_ref/sortmerna_ref missing: make -C oracle -f Makefile.ref")
    arc, bac, reads = (os.path.join(HERE, f) for f in ("db_arc.fasta", "db_bac.fasta", "reads_mix.fq"))
    tmp = tempfile.mkdtemp(prefix="smr_golden_otu_")
    out = {}
    try:
        for case, extra in DENOVO_CASES.items():
            out[case] = _run([arc, bac], reads, os.path.join(tmp, case), extra, *DENOVO_ARGS[case])
        out["none"] = _run([arc, bac], reads, os.path.join(tmp, "none"), ["-R"], "1", "1")
        out["parts"] = _run([arc, bac], reads, os.path.join(tmp, "parts"), ["-m", "0.5"], "0.97", "0.97")
        copy = os.path.join(tmp, "db_bac_copy.fasta")
        shutil.copy(bac, copy)
        out["merged"] = _run([bac, copy], reads, os.path.join(tmp, "merged"), ["-num_alignments", "2"], "0.97", "0.97")
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from integration_common import golden_mates
        mates = golden_mates(tmp)
        out["paired_files"] = _run([arc, bac], mates, os.path.join(tmp, "pf"), ["-paired_in"], "0.97", "0.97")
        inter = os.path.join(tmp, "mates_interleaved.fastq")
        recs = [open(p, "rb").read().split(b"\n") for p in mates]
        with open(inter, "wb") as f:
            f.write(b"".join(b"\n".join(recs[j][i:i + 4]) + b"\n" for i in range(0, len(recs[0]) - 3, 4) for j in (0, 1)))
        out["paired_interleaved"] = _run([arc, bac], inter, os.path.join(tmp, "pi"), ["-paired_in"], "0.97", "0.97")
        for k, v in out.items():
            print(k, "n_yid_ycov", v["n_yid_ycov"], "total_otu", v["total_otu"], "bytes", None if v["otu_map"] is None else len(v["otu_map"]))
        with open(os.path.join(HERE, "otu_map.json"), "w") as f:
            json.dump(out, f, indent=0)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
