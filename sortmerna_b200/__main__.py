"""python -m sortmerna_b200: the reference's command line (sortmerna, include/options.hpp) for what this library covers, run through
api.run_files: read files in, the reference's out/ directory out.  `python -m sortmerna_b200 -h` lists the options."""
from __future__ import annotations

import json
import os
import sys

HELP = """usage: python -m sortmerna_b200 -ref FASTA [-ref FASTA ...] -reads FILE [-reads MATE2] [options]

Aligns the reads against the references on the GPU and writes the reference's report files under WORKDIR/out/ with its file
names.  The files are those the reference writes at -threads 1, whatever -threads says (it is accepted and only printed in
aligned.log).  Options take the reference's names and meanings; any other option is refused.

  -ref FASTA            reference file (repeatable; each is indexed on the device)
  -reads FILE           reads file, FASTA or FASTQ, plain or gzip; twice for two mate files
  -workdir DIR          output under DIR/out/ (default ~/sortmerna/run)
 reports
  -fastx -other -sam -SQ    aligned.<fq|fa>, other.<fq|fa>, aligned.sam, its @SQ lines
  -blast 'F [cols]'     aligned.blast: 1 (tabular, optional columns cigar qcov qstrand) or 0 (pairwise)
  -zip-out [1|0|-1]     compress the report files (-1, the default: as the first reads file is)
  -bam | -bam_sorted    aligned.bam: the rows of aligned.sam as BAM (BGZF); not a reference option
                        with -bam_sorted: sorted by coordinate, and its index aligned.bam.bai; not a reference option either
 alignment
  -num_alignments N -no-best -min_lis N -num_seeds N -passes L1,L2,L3 -edges N[%] -full_search -F -R -e EVALUE
 scoring
  -match N -mismatch N -gap_open N -gap_ext N -N N
 paired reads
  -paired_in -paired_out -out2 -sout
 OTU and de novo
  -otu_map -de_novo_otu -id X -coverage X
 indexing
  -L N -interval N -max_pos N -m MB
  -threads N            accepted; the output is that of the reference at -threads 1
 statistics the library does not compute
  -gumbel LAMBDA,K      Gumbel parameters of each -ref, in -ref order (once per -ref).  Without it, the reference's file name is
                        looked up in sortmerna_b200/gumbel_defaults.json, which holds the default scoring's values only.
  -minimal_score N      the minimal Smith-Waterman score of each -ref (once per -ref), instead of the one computed from -e
"""

FLAGS = {"fastx", "other", "sam", "bam", "bam_sorted", "SQ", "no-best", "full_search", "F", "R", "paired_in", "paired_out", "out2", "sout", "otu_map",
         "de_novo_otu", "h", "help"}
VALUES = {"ref", "reads", "workdir", "blast", "num_alignments", "min_lis", "num_seeds", "passes", "edges", "e", "match", "mismatch",
          "gap_open", "gap_ext", "N", "id", "coverage", "L", "interval", "max_pos", "m", "threads", "gumbel", "minimal_score"}
OPTIONAL_VALUES = {"zip-out"}
REPEATABLE = {"ref", "reads", "gumbel", "minimal_score"}


class UsageError(ValueError):
    pass


def _int(name, v, lo=None):
    try:
        x = int(v)
    except ValueError:
        raise UsageError(f"'-{name}' needs an integer, not '{v}'") from None
    if lo is not None and x < lo:
        raise UsageError(f"'-{name}' needs an integer of at least {lo}, not {x}")
    return x


def _float(name, v):
    try:
        return float(v)
    except ValueError:
        raise UsageError(f"'-{name}' needs a number, not '{v}'") from None


def tokenize(argv: list) -> dict:
    """argv -> {option name: [values]} (flags get [""]); an unknown option, a missing value or a repeated one-off option raises"""
    opts, i = {}, 0
    while i < len(argv):
        a = argv[i]
        if not a.startswith("-") or len(a) < 2:
            raise UsageError(f"unexpected argument '{a}'")
        name = a.lstrip("-")
        if name not in FLAGS | VALUES | OPTIONAL_VALUES:
            raise UsageError(f"option '{a}' is not supported by this program")
        if name in opts and name not in REPEATABLE:
            raise UsageError(f"option '-{name}' is given twice")
        i += 1
        if name in VALUES:
            if i >= len(argv):
                raise UsageError(f"option '-{name}' needs a value")
            v = argv[i]
            i += 1
        elif name in OPTIONAL_VALUES and i < len(argv) and (not argv[i].startswith("-") or argv[i] == "-1"):
            v = argv[i]   # a value never starts with '-' (but -1): the next option is parsed as one, and refused if unknown
            i += 1
        else:
            v = ""
        opts.setdefault(name, []).append(v)
    return opts


def gumbel_defaults():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "gumbel_defaults.json")) as f:
        return json.load(f)


def parse_args(argv: list) -> dict:
    """The command line -> the arguments of api.run_files (and "workdir", "out_dir"), with Runopts::validate's defaults and refusals
    (src/sortmerna/options.cpp:1566-1758).  Raises UsageError with the reason."""
    from . import api
    o = tokenize(argv)
    one = lambda k, d=None: o[k][0] if k in o else d   # noqa: E731
    has = lambda k: k in o   # noqa: E731
    refs, reads = o.get("ref", []), o.get("reads", [])
    if not refs:
        raise UsageError("'-ref' is required")
    if not reads or len(reads) > 2:
        raise UsageError("'-reads' is required, once or twice (two mate files)")
    p = api.default_params()
    for k in ("match", "mismatch", "gap_open", "gap_ext"):
        if has(k):
            setattr(p, k, _int(k, one(k)))
    p.score_N = _int("N", one("N")) if has("N") else p.mismatch
    if p.gap_ext > p.gap_open:
        raise UsageError("-gap_ext must be less than -gap_open")
    if has("num_alignments"):
        p.num_alignments = _int("num_alignments", one("num_alignments"), 0)
    p.is_best = 0 if has("no-best") else 1
    if has("min_lis"):
        if has("num_alignments"):
            raise UsageError("'-min_lis' and '-num_alignments' cannot be set together")
        if not p.is_best:
            raise UsageError("'-min_lis' must be set together with the best alignment search (not with '-no-best')")
        p.min_lis = _int("min_lis", one("min_lis"), 0)
    if has("num_seeds"):
        p.num_seeds = _int("num_seeds", one("num_seeds"), 1)
    if has("edges"):
        v = one("edges")
        p.edges, p.edges_is_percent = _int("edges", v.rstrip("%")), int(v.endswith("%"))
        if not 1 <= p.edges <= 10:
            raise UsageError("'-edges' needs an integer between 1 and 10 (a percentage with '%')")
    if has("full_search"):
        p.is_full_search = 1
    if has("F") != has("R"):
        p.is_forward, p.is_reverse = int(has("F")), int(has("R"))
    paired_in, paired_out = has("paired_in"), has("paired_out")
    if paired_in and paired_out:
        raise UsageError("options '-paired_in' and '-paired_out' are mutually exclusive")
    paired = len(reads) == 2 or paired_in or paired_out
    if has("sout") and (paired_in or paired_out):
        raise UsageError("option '-sout' cannot be used with '-paired_in' or '-paired_out'")
    otu_map = has("otu_map")
    if otu_map and not p.is_best:
        raise UsageError("'-otu_map' cannot be set together with '-no-best': the OTU map is made from the best alignment")
    min_id = _float("id", one("id")) if has("id") else -1.0
    min_cov = _float("coverage", one("coverage")) if has("coverage") else -1.0
    for k, x in (("id", min_id), ("coverage", min_cov)):
        if has(k) and not 0 <= x <= 1:
            raise UsageError(f"'-{k}' needs a number with 0 <= {k} <= 1, not {x:g}")
    if (min_id > 0 or min_cov > 0) and not otu_map:
        raise UsageError("'-id' and '-coverage' can only be used together with '-otu_map'")
    if min_id < 0:
        min_id = 0.97 if otu_map else 0.0
    if min_cov < 0:
        min_cov = 0.97 if otu_map else 0.0
    fastx, sam, bam, blast = has("fastx") or paired_in or paired_out, has("sam"), has("bam") or has("bam_sorted"), one("blast")
    if not (fastx or blast is not None or sam or bam or otu_map or has("de_novo_otu")):
        blast = "1"   # the reference's default output
    if has("num_alignments") and not (blast is not None or sam or bam or fastx):
        raise UsageError("'-num_alignments' needs an output format (-blast, -sam or -fastx)")
    if blast is not None:
        f = blast.split()
        if not f or f[0] not in ("0", "1") or any(c not in api.BLAST_COLS for c in f[1:]) or (f[0] == "0" and len(f) > 1):
            raise UsageError(f"'-blast' takes 1 with the optional columns cigar qcov qstrand, or 0 alone, not '{blast}'")
    zip_flag = -1
    if has("zip-out"):
        v = one("zip-out").lower()
        if v not in ("", "-1", "1", "y", "yes", "t", "true", "0", "n", "no", "f", "false"):
            raise UsageError(f"'-zip-out' takes 1 / true / t / yes / y, 0 / false / f / no / n or -1, not '{one('zip-out')}'")
        zip_flag = 1 if v in ("1", "y", "yes", "t", "true") else 0 if v in ("0", "n", "no", "f", "false") else -1
    lnwin = _int("L", one("L")) if has("L") else 18
    passes = None
    if has("passes"):
        try:
            sk = tuple(int(x) for x in one("passes").split(","))
        except ValueError:
            raise UsageError("'-passes' takes three positive integers L1,L2,L3") from None
        if len(sk) != 3 or min(sk) <= 0:
            raise UsageError("'-passes' takes three positive integers L1,L2,L3")
        passes = [sk] * len(refs)
    gum = o.get("gumbel", [])
    if gum:
        if len(gum) != len(refs):
            raise UsageError(f"'-gumbel' is given {len(gum)} times for {len(refs)} references: give it once per '-ref'")
        try:
            gumbel = [tuple(float(x) for x in g.split(",")) for g in gum]
        except ValueError:
            raise UsageError("'-gumbel' takes LAMBDA,K") from None
        if any(len(g) != 2 for g in gumbel):
            raise UsageError("'-gumbel' takes LAMBDA,K")
    else:
        d = gumbel_defaults()
        if any(getattr(p, k) != v for k, v in d["scoring"].items()):
            raise UsageError("gumbel_defaults.json holds the Gumbel parameters of the default scoring only: give -gumbel LAMBDA,K per -ref")
        missing = [r for r in refs if os.path.basename(r) not in d["gumbel"]]
        if missing:
            raise UsageError(f"no Gumbel parameters for reference '{missing[0]}' in gumbel_defaults.json: give -gumbel LAMBDA,K per -ref")
        gumbel = [(d["gumbel"][os.path.basename(r)]["lambda_"], d["gumbel"][os.path.basename(r)]["K"]) for r in refs]
    ms = o.get("minimal_score")
    if ms is not None:
        if len(ms) != len(refs):
            raise UsageError(f"'-minimal_score' is given {len(ms)} times for {len(refs)} references: give it once per '-ref'")
        ms = [_int("minimal_score", x, 0) for x in ms]
    evalue = _float("e", one("e")) if has("e") else 1.0
    if evalue < 0:
        evalue = 1.0
    workdir = one("workdir", os.path.join(os.path.expanduser("~"), "sortmerna", "run"))
    return dict(refs=refs, reads=reads, out_dir=os.path.join(workdir, "out"), workdir=workdir, params=p, gumbel=gumbel, minimal_score=ms,
                evalue=evalue, sam=sam, bam=bam, bam_sorted=has("bam_sorted"), sq=has("SQ"), blast=blast, fastx=fastx, other=has("other"),
                denovo=(min_id, min_cov) if has("de_novo_otu") else None, otu_map=(min_id, min_cov) if otu_map else None,
                paired_in=paired_in, paired_out=paired_out, out2=has("out2") and paired, sout=has("sout") and paired,
                zip_out=zip_flag == 1 or (zip_flag == -1 and _is_gz(reads[0])), lnwin=lnwin,
                interval=_int("interval", one("interval"), 1) if has("interval") else 1,
                max_pos=_int("max_pos", one("max_pos"), 0) if has("max_pos") else 10000,
                max_mb=_float("m", one("m")) if has("m") else 3072.0, skiplengths=passes,
                threads=_int("threads", one("threads"), 1) if has("threads") else 1)


def _is_gz(path: str) -> bool:
    try:
        with open(path, "rb") as f:
            return f.read(2) == b"\x1f\x8b"
    except OSError:
        raise UsageError(f"cannot read '{path}'") from None


def main(argv=None) -> int:
    argv = sys.argv[1:] if argv is None else list(argv)
    if not argv or "-h" in argv or "--help" in argv or "-help" in argv:
        print(HELP, end="")
        return 0 if argv else 1
    try:
        kw = parse_args(argv)
    except UsageError as e:
        print(f"sortmerna_b200: {e}", file=sys.stderr)
        return 2
    from . import api
    kw.pop("workdir")
    # the reference records its argv, each followed by a space, in aligned.log and the SAM header (Runopts::cmdline)
    kw["cmd"] = "".join(a + " " for a in ["python -m sortmerna_b200"] + argv)
    r = api.run_files(**kw)
    print(f"{r['reads']} reads, {r['num_aligned']} aligned; files in {kw['out_dir']}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
