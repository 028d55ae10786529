#!/usr/bin/env python
"""Regenerates tests/golden/ from the reference (run in the build container, where /root/reference
and oracle/_ref/sortmerna_ref exist):

  db_arc.fasta / db_bac.fasta   small slices of the bundled rRNA databases (inputs, not code)
  reads_mix.fq                  seeded synthetic + real reads exercising the edge cases of the path
  idx/*.dat.gz, idx/*.stats     the reference's own index of the two slices
  case_*/expected.json          what the UNMODIFIED reference binary printed for each option set:
                                SAM rows, aligned.log numbers (minimal scores, totals, coverage)
  denovo.json                   denovo_stats counts + aligned_denovo read ids for -id/-coverage option sets
                                (python tests/golden/make_golden.py denovo regenerates only this file)

Usage: python tests/golden/make_golden.py
"""
import gzip
import json
import lzma
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import ora  # noqa: E402
from sortmerna_b200 import hostio  # noqa: E402

REF_DATA = "/root/reference/data"
SEED = 20260924

CASES = {
    # name: extra reference CLI arguments
    "default": [],
    "best3": ["-num_alignments", "3"],
    "nobest2": ["-no-best", "-num_alignments", "2"],
    "fwd_only": ["-F"],
    "rev_only": ["-R"],
    "full_search": ["-full_search"],
    "scores": ["-match", "2", "-mismatch", "-4", "-gap_open", "6", "-gap_ext", "3", "-N", "-2"],
    # 2*gap_open < |mismatch|: the regime where the striped kernel's "no insertion next to a deletion"
    # rule (ssw.c:267,496) could differ from plain Gotoh (SURVEY A.6)
    "scores_exotic": ["-match", "2", "-mismatch", "-7", "-gap_open", "3", "-gap_ext", "1"],
    "edges_pct": ["-edges", "10%"],
    "seeds3": ["-num_seeds", "3"],
    # "all alignments" (alignment.cpp:420-424; the reference's own t9, scripts/test.jinja:425-476): every accepted alignment is stored
    "all": ["-num_alignments", "0"],
}
# index-build options that change the index LAYOUT (not the alignment parameters): the reference builds its own index for these
EXTRA_INDEX_CASES = {
    # 9.5e-6 "MB" per window (indexdb.cpp:1381): both database slices split into 3 index parts -- the per-part loop of align()
    # (processor.cpp:196-262), part-relative ref_num, Read::best re-initialised per part
    "parts": ["-m", "0.5"],
}


def make_extra_index_cases():
    arc_p, bac_p, reads_p = (os.path.join(HERE, f) for f in ("db_arc.fasta", "db_bac.fasta", "reads_mix.fq"))
    tmp = tempfile.mkdtemp(prefix="smr_golden_x_")
    for case, extra in EXTRA_INDEX_CASES.items():
        r = ora.run_reference([arc_p, bac_p], reads_p, os.path.join(tmp, case), extra=["-sam", "-blast", "1 cigar qcov qstrand", "-fastx", "-other"] + extra, threads=1)
        log = ora.parse_log(r["log"])
        sam = ["\t".join(f[:9] + ["*", "*"] + f[11:]) for f in (ln.split("\t") for ln in ora.read_sam_rows(os.path.join(r["out_dir"], "aligned.sam")))]
        blast = [ln.rstrip("\n") for ln in open(os.path.join(r["out_dir"], "aligned.blast"))]
        nparts = [hostio.parse_stats(p).num_parts for p in hostio.find_index_prefixes(r["idx_dir"]).values()]
        os.makedirs(os.path.join(HERE, "case_" + case), exist_ok=True)
        with open(os.path.join(HERE, "case_" + case, "expected.json"), "w") as f:
            json.dump(dict(args=extra, log=log, sam=sam, blast=blast, num_parts=sorted(nparts)), f, indent=0)
        print(case, "passing", log["passing"], "sam rows", len(sam), "parts", nparts)
    shutil.rmtree(tmp, ignore_errors=True)


def take_fasta(src, dst, nseq, skip=0, min_len=0):
    h, s, _ = hostio.read_fastx(src)
    out = []
    for hh, ss in list(zip(h, s))[skip:]:
        if len(ss) >= min_len:
            out.append((hh, ss))
        if len(out) == nseq:
            break
    with open(dst, "w") as f:
        for hh, ss in out:
            f.write(hh + "\n" + ss.decode() + "\n")
    return out


def mutate(rng, seq, sub, indel):
    out = []
    for c in seq:
        r = rng.random()
        if r < indel / 2:
            continue
        if r < indel:
            out.append("ACGT"[rng.integers(4)])
        if rng.random() < sub:
            c = "ACGT"[rng.integers(4)]
        out.append(c)
    return "".join(out)


def rc(s):
    return s.translate(str.maketrans("ACGTN", "TGCAN"))[::-1]


def make_reads(rng, dbs):
    reads = []

    def sample(db, ln, sub, indel, flank=0):
        _, s = db[rng.integers(len(db))]
        s = s.decode().upper().replace("U", "T")
        if len(s) <= ln:
            frag = s
        else:
            p = rng.integers(0, len(s) - ln + 1)
            frag = s[p:p + ln]
        frag = mutate(rng, frag, sub, indel)
        if flank:
            frag = "".join("ACGT"[i] for i in rng.integers(0, 4, flank)) + frag
        if rng.random() < 0.5:
            frag = rc(frag)
        return frag

    arc, bac = dbs
    for i in range(150):
        reads.append((f"arc1_{i}", sample(arc, int(rng.integers(100, 153)), 0.01, 0.001)))
    for i in range(150):
        reads.append((f"bac1_{i}", sample(bac, int(rng.integers(100, 153)), 0.01, 0.001)))
    for i in range(60):
        reads.append((f"arc10_{i}", sample(arc, 150, 0.08, 0.01)))
    for i in range(60):
        reads.append((f"bac10_{i}", sample(bac, 150, 0.08, 0.01)))
    for i in range(40):
        reads.append((f"exact_{i}", sample(arc if i % 2 else bac, int(rng.integers(60, 151)), 0.0, 0.0)))
    for i in range(60):
        reads.append((f"rand_{i}", "".join("ACGT"[k] for k in rng.integers(0, 4, int(rng.integers(40, 200))))))
    for i in range(50):  # ambiguous bases
        s = list(sample(arc if i % 2 else bac, 150, 0.02, 0.002))
        for _ in range(int(rng.integers(1, 4))):
            s[rng.integers(len(s))] = "N"
        reads.append((f"amb_{i}", "".join(s)))
    for i in range(20):  # overhang at reference ends / reads longer than short references
        db = arc if i % 2 else bac
        _, s = db[rng.integers(len(db))]
        s = s.decode().upper().replace("U", "T")
        frag = s[:int(rng.integers(40, 120))] if i % 4 < 2 else s[-int(rng.integers(40, 120)):]
        frag = "".join("ACGT"[k] for k in rng.integers(0, 4, int(rng.integers(10, 60)))) + frag if i % 4 < 2 else frag + "".join(
            "ACGT"[k] for k in rng.integers(0, 4, int(rng.integers(10, 60))))
        reads.append((f"edge_{i}", rc(frag) if rng.random() < 0.5 else frag))
    for i, ln in enumerate((17, 18, 19, 5, 1, 25, 33)):  # around lnwin
        reads.append((f"short_{i}", sample(arc, ln, 0.0, 0.0)))
    for i, ln in enumerate((300, 520, 900, 1400)):  # long reads: several SW row blocks
        reads.append((f"long_{i}", sample(bac if i % 2 else arc, ln, 0.03, 0.003)))
    for i in range(12):  # low complexity
        reads.append((f"lowc_{i}", ("ACGT"[i % 4] * int(rng.integers(30, 90))) + sample(arc, 60, 0.0, 0.0)))
    # real reads from the bundled metatranscriptome
    h, s, _ = hostio.read_fastx(os.path.join(REF_DATA, "set4_mate_pairs_metatranscriptomics_1.fastq"), 120)
    for hh, ss in zip(h, s):
        reads.append((hostio.seq_id(hh), ss.decode()))
    order = rng.permutation(len(reads))
    return [reads[k] for k in order]


def pack_file(src, dst):
    """dst.gz, or dst.xz where gzip -9 would exceed 1 MB (tests/conftest.py unpack_index reads both)"""
    data = open(src, "rb").read()
    gz = gzip.compress(data, 9)
    if len(gz) <= 1_000_000:
        open(dst + ".gz", "wb").write(gz)
    else:
        open(dst + ".xz", "wb").write(lzma.compress(data, preset=9 | lzma.PRESET_EXTREME))


def gz_index(src_dir, dst_dir):
    os.makedirs(dst_dir, exist_ok=True)
    for fn in sorted(os.listdir(src_dir)):
        src = os.path.join(src_dir, fn)
        if fn.endswith(".stats"):
            shutil.copy(src, os.path.join(dst_dir, fn))
        else:
            pack_file(src, os.path.join(dst_dir, fn))


def make_t0(tmp):
    """BASELINE config 1 (scripts/test.jinja t0/t2): data/test_read.fasta vs data/test_ref.fasta -- a 1.5 kb read against one
    reference: the int16 'word' Smith-Waterman path (score ~2000), multi-row-block SW on the GPU, a 30-op CIGAR.  The bundled
    files are wrapped FASTA without a trailing newline, which the reference's Readfeed mis-counts (SURVEY section 4); the feed is
    out of scope here, so both files are rewritten as single-line records first and the reference is run on THOSE."""
    d = os.path.join(HERE, "t0")
    shutil.rmtree(d, ignore_errors=True)
    os.makedirs(d)
    for src, dst in (("test_ref.fasta", "db_t0.fasta"), ("test_read.fasta", "reads_t0.fasta")):
        h, s, _ = hostio.read_fastx(os.path.join(REF_DATA, src))
        with open(os.path.join(d, dst), "w") as f:
            for hh, ss in zip(h, s):
                f.write(hh + "\n" + ss.decode() + "\n")
    wd = os.path.join(tmp, "t0")
    r = ora.run_reference([os.path.join(d, "db_t0.fasta")], os.path.join(d, "reads_t0.fasta"), wd,
                          extra=["-sam", "-blast", "1 cigar qcov qstrand", "-fastx", "-other"], threads=1)
    log = ora.parse_log(r["log"])
    sam = ora.read_sam_rows(os.path.join(r["out_dir"], "aligned.sam"))
    blast = [ln.rstrip("\n") for ln in open(os.path.join(r["out_dir"], "aligned.blast"))]
    json.dump(dict(args=[], log=log, sam=sam, blast=blast), open(os.path.join(d, "expected.json"), "w"), indent=0)
    gz_index(os.path.join(wd, "idx"), os.path.join(d, "idx"))
    print("t0", log["passing"], log["minimal_score"], [x.split("\t")[5][:60] + " " + x.split("\t")[11] for x in sam])


DENOVO_CASES = {"default": [], "best3": ["-num_alignments", "3"], "rev_only": ["-R"], "loose": ["-num_alignments", "2"]}
DENOVO_ARGS = {"default": ("0.97", "0.97"), "best3": ("0.97", "0.97"), "rev_only": ("0.9", "0.9"), "loose": ("0.85", "0.5")}


def make_denovo():
    """denovo.json: what denovo_stats (processor.cpp:287-438) counted and which reads went to aligned_denovo.fq
    (output.cpp:130-141) for '-otu_map -de_novo_otu -id X -coverage Y' on the golden reads."""
    import re
    arc_p, bac_p, reads_p = (os.path.join(HERE, f) for f in ("db_arc.fasta", "db_bac.fasta", "reads_mix.fq"))
    tmp = tempfile.mkdtemp(prefix="smr_golden_dn_")
    res = {}
    for case, extra in DENOVO_CASES.items():
        mid, mcov = DENOVO_ARGS[case]
        r = ora.run_reference([arc_p, bac_p], reads_p, os.path.join(tmp, case),
                              extra=["-fastx", "-otu_map", "-de_novo_otu", "-id", mid, "-coverage", mcov] + extra, threads=1)
        m = re.search(r"num_yid_ycov: (\d+)\s+num_yid_ncov: (\d+)\s+num_nid_ycov: (\d+)\s+num_denovo: (\d+)", r["stdout"])
        h, _, _ = hostio.read_fastx(os.path.join(r["out_dir"], "aligned_denovo.fq"))
        log = ora.parse_log(r["log"])
        res[case] = dict(args=extra, min_id=float(mid), min_cov=float(mcov), counts=[int(x) for x in m.groups()],
                         denovo_reads=sorted(hostio.seq_id(x) for x in h), minimal_score=log["minimal_score"],
                         total_denovo=int(re.search(r"de novo clustering = (\d+)", r["log"]).group(1)))
        print(case, res[case]["counts"], len(res[case]["denovo_reads"]), res[case]["total_denovo"])
    with open(os.path.join(HERE, "denovo.json"), "w") as f:
        json.dump(res, f, indent=0)
    shutil.rmtree(tmp, ignore_errors=True)


def make_one_case(case):
    """python tests/golden/make_golden.py case NAME: (re)generate one option set on the committed inputs."""
    arc_p, bac_p, reads_p = (os.path.join(HERE, f) for f in ("db_arc.fasta", "db_bac.fasta", "reads_mix.fq"))
    tmp = tempfile.mkdtemp(prefix="smr_golden_1_")
    extra = CASES[case]
    r = ora.run_reference([arc_p, bac_p], reads_p, os.path.join(tmp, case), extra=["-sam", "-blast", "1 cigar qcov qstrand", "-fastx", "-other"] + extra, threads=1)
    log = ora.parse_log(r["log"])
    sam = ["\t".join(f[:9] + ["*", "*"] + f[11:]) for f in (ln.split("\t") for ln in ora.read_sam_rows(os.path.join(r["out_dir"], "aligned.sam")))]
    blast = [ln.rstrip("\n") for ln in open(os.path.join(r["out_dir"], "aligned.blast"))]
    os.makedirs(os.path.join(HERE, "case_" + case), exist_ok=True)
    with open(os.path.join(HERE, "case_" + case, "expected.json"), "w") as f:
        json.dump(dict(args=extra, log=log, sam=sam, blast=blast), f, indent=0)
    print(case, "passing", log["passing"], "failing", log["failing"], "sam rows", len(sam), "minimal", log["minimal_score"])
    shutil.rmtree(tmp, ignore_errors=True)


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "case":
        return make_one_case(sys.argv[2])
    if len(sys.argv) > 1 and sys.argv[1] == "denovo":
        return make_denovo()
    if len(sys.argv) > 1 and sys.argv[1] == "extra":
        return make_extra_index_cases()
    if not ora.have_reference_binary():
        sys.exit("oracle/_ref/sortmerna_ref missing: make -C oracle -f Makefile.ref")
    rng = np.random.default_rng(SEED)
    arc_p, bac_p = os.path.join(HERE, "db_arc.fasta"), os.path.join(HERE, "db_bac.fasta")
    arc = take_fasta(os.path.join(REF_DATA, "rRNA_databases/silva-arc-16s-id95.fasta"), arc_p, 110, skip=5)
    bac = take_fasta(os.path.join(REF_DATA, "rRNA_databases/silva-bac-16s-id90.fasta"), bac_p, 90, skip=40)
    reads = make_reads(rng, (arc, bac))
    reads_p = os.path.join(HERE, "reads_mix.fq")
    with open(reads_p, "w") as f:
        for name, s in reads:
            f.write(f"@{name}\n{s}\n+\n{'I' * len(s)}\n")
    idx_dir = os.path.join(HERE, "idx")
    shutil.rmtree(idx_dir, ignore_errors=True)
    tmp = tempfile.mkdtemp(prefix="smr_golden_")
    first = True
    for case, extra in CASES.items():
        wd = os.path.join(tmp, case)
        r = ora.run_reference([arc_p, bac_p], reads_p, wd, extra=["-sam", "-blast", "1 cigar qcov qstrand", "-fastx", "-other"] + extra,
                              threads=1, idx_dir=None if first else os.path.join(tmp, "idx_keep"))
        if first:
            shutil.copytree(os.path.join(wd, "idx"), os.path.join(tmp, "idx_keep"))
            first = False
        log = ora.parse_log(r["log"])
        sam = ora.read_sam_rows(os.path.join(r["out_dir"], "aligned.sam"))
        if case != "default":  # SEQ / QUAL are inputs echoed back: keep them for one case only
            sam = ["\t".join(f[:9] + ["*", "*"] + f[11:]) for f in (ln.split("\t") for ln in sam)]
        blast = [ln.rstrip("\n") for ln in open(os.path.join(r["out_dir"], "aligned.blast"))]
        os.makedirs(os.path.join(HERE, "case_" + case), exist_ok=True)
        with open(os.path.join(HERE, "case_" + case, "expected.json"), "w") as f:
            json.dump(dict(args=extra, log=log, sam=sam, blast=blast), f, indent=0)
        print(case, "passing", log["passing"], "failing", log["failing"], "sam rows", len(sam), "minimal", log["minimal_score"])
    # keep the reference-built index (gz) so the tests do not depend on the builder
    os.makedirs(idx_dir)
    for fn in sorted(os.listdir(os.path.join(tmp, "idx_keep"))):
        src = os.path.join(tmp, "idx_keep", fn)
        if fn.endswith(".stats"):
            # the .stats file embeds the absolute FASTA path; keep it as is (only lnwin/numseq/freqs are read)
            shutil.copy(src, os.path.join(idx_dir, fn))
        else:
            pack_file(src, os.path.join(idx_dir, fn))
    make_t0(tmp)
    make_denovo()
    make_extra_index_cases()
    shutil.rmtree(tmp, ignore_errors=True)
    print("sizes:", {fn: os.path.getsize(os.path.join(idx_dir, fn)) for fn in os.listdir(idx_dir)})


if __name__ == "__main__":
    main()
