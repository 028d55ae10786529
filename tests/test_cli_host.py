"""The command line (python -m sortmerna_b200) without a GPU: option parsing and its mapping onto Params and the report options,
the reference's refusals (Runopts::validate), unknown options refused by name, the Gumbel lookup and its message; and the index
statistics run_files computes from a FASTA against the ones the index builder writes."""
import os
import tempfile

import pytest

from conftest import GOLDEN
from sortmerna_b200 import __main__ as cli
from sortmerna_b200 import api, hostio

ARC, BAC = os.path.join(GOLDEN, "db_arc.fasta"), os.path.join(GOLDEN, "db_bac.fasta")
READS = os.path.join(GOLDEN, "reads_mix.fq")
G = ["-gumbel", "0.59,0.32", "-gumbel", "0.6,0.33"]


def parse(*args, gumbel=True):
    return cli.parse_args(["-ref", ARC, "-ref", BAC, "-reads", READS, "-workdir", "/w"] + (G if gumbel else []) + list(args))


def test_defaults():
    k = parse()
    p = k["params"]
    assert (p.match, p.mismatch, p.gap_open, p.gap_ext, p.score_N) == (2, -3, 5, 2, -3)
    assert (p.num_alignments, p.is_best, p.min_lis, p.num_seeds, p.edges, p.edges_is_percent) == (1, 1, 2, 2, 4, 0)
    assert (p.is_forward, p.is_reverse, p.is_full_search) == (1, 1, 0)
    assert k["blast"] == "1" and not (k["sam"] or k["fastx"] or k["other"])   # the reference's default output
    assert k["out_dir"] == "/w/out" and k["refs"] == [ARC, BAC] and k["reads"] == [READS]
    assert k["gumbel"] == [(0.59, 0.32), (0.6, 0.33)] and k["minimal_score"] is None and k["evalue"] == 1.0
    assert not k["zip_out"] and k["otu_map"] is None and k["denovo"] is None and k["threads"] == 1
    assert (k["lnwin"], k["interval"], k["max_pos"], k["max_mb"], k["skiplengths"]) == (18, 1, 10000, 3072.0, None)


def test_mapping():
    k = parse("-sam", "-SQ", "-fastx", "-other", "-blast", "1 cigar qcov qstrand", "-num_alignments", "0", "-num_seeds", "3",
              "-edges", "10%", "-full_search", "-F", "-match", "3", "-mismatch", "-4", "-gap_open", "6", "-gap_ext", "3",
              "-L", "16", "-interval", "2", "-max_pos", "0", "-m", "0.5", "-passes", "16,8,3", "-threads", "4", "-e", "0.1",
              "-minimal_score", "40", "-minimal_score", "41", "-zip-out", "yes")
    p = k["params"]
    assert (p.num_alignments, p.num_seeds, p.edges, p.edges_is_percent, p.is_full_search, p.is_forward, p.is_reverse) == (0, 3, 10, 1, 1, 1, 0)
    assert (p.match, p.mismatch, p.gap_open, p.gap_ext, p.score_N) == (3, -4, 6, 3, -4)   # -N defaults to -mismatch
    assert k["sam"] and k["sq"] and k["fastx"] and k["other"] and k["blast"] == "1 cigar qcov qstrand"
    assert (k["lnwin"], k["interval"], k["max_pos"], k["max_mb"], k["skiplengths"]) == (16, 2, 0, 0.5, [(16, 8, 3)] * 2)
    assert k["threads"] == 4 and k["evalue"] == 0.1 and k["minimal_score"] == [40, 41] and k["zip_out"]
    assert parse("-N", "-1")["params"].score_N == -1
    assert parse("-no-best", "-num_alignments", "2")["params"].is_best == 0
    assert parse("-min_lis", "5")["params"].min_lis == 5
    k = parse("-otu_map", "-de_novo_otu", "-id", "0.9", "-coverage", "0.8")
    assert k["otu_map"] == (0.9, 0.8) and k["denovo"] == (0.9, 0.8) and k["blast"] is None
    assert parse("-otu_map")["otu_map"] == (0.97, 0.97)
    assert parse("-de_novo_otu")["denovo"] == (0.0, 0.0)
    k = parse("-paired_in", "-out2")
    assert k["paired_in"] and k["fastx"] and k["out2"]           # -paired_in sets -fastx, and makes the reads paired
    assert not parse("-out2", "-fastx")["out2"]                  # one unpaired file: -out2 is ignored, as the reference does
    assert parse("-zip-out", "0")["zip_out"] is False and parse("-zip-out")["zip_out"] is False


def test_zip_out_follows_the_input(tmp_path):
    import gzip
    gz = tmp_path / "r.fq.gz"
    gz.write_bytes(gzip.compress(open(READS, "rb").read()))
    args = ["-ref", ARC, "-ref", BAC, "-reads", str(gz)] + G
    assert cli.parse_args(args)["zip_out"] and cli.parse_args(args + ["-zip-out"])["zip_out"]
    assert not cli.parse_args(args + ["-zip-out", "n"])["zip_out"]


def test_two_mate_files():
    k = cli.parse_args(["-ref", ARC, "-reads", READS, "-reads", READS, "-gumbel", "0.59,0.32", "-out2", "-sout", "-fastx"])
    assert k["reads"] == [READS, READS] and k["out2"] and k["sout"]


@pytest.mark.parametrize("args,msg", [
    (["-paired_in", "-paired_out"], "mutually exclusive"),
    (["-sout", "-paired_in"], "'-sout' cannot be used"),
    (["-otu_map", "-no-best"], "cannot be set together with '-no-best'"),
    (["-min_lis", "2", "-num_alignments", "2"], "cannot be set together"),
    (["-min_lis", "2", "-no-best"], "must be set together"),
    (["-id", "0.9"], "only be used together with '-otu_map'"),
    (["-gap_ext", "6"], "-gap_ext must be less than -gap_open"),
    (["-edges", "11"], "between 1 and 10"),
    (["-blast", "0 cigar"], "'-blast' takes"),
    (["-passes", "18,9"], "three positive integers"),
    (["-num_alignments", "2", "-otu_map"], "needs an output format"),
    (["-otu_map", "-id", "5"], "0 <= id <= 1"),
    (["-otu_map", "-coverage", "-0.1"], "0 <= coverage <= 1"),
    (["-zip-out", "maybe"], "'-zip-out' takes"),
])
def test_reference_refusals(args, msg):
    with pytest.raises(cli.UsageError, match=msg):
        parse(*args)


@pytest.mark.parametrize("opt", ["-task", "-idx-dir", "-kvdb", "-aligned", "--print_all_reads", "-v"])
def test_unknown_options_are_refused_by_name(opt):
    with pytest.raises(cli.UsageError, match=f"option '{opt}' is not supported"):
        parse(opt, "1")


def test_zip_out_never_takes_an_option_as_its_value():
    with pytest.raises(cli.UsageError, match="option '-kvdb' is not supported"):
        parse("-zip-out", "-kvdb")
    k = parse("-zip-out", "-sam")
    assert k["sam"] and not k["zip_out"]
    assert parse("-zip-out", "-1", "-fastx")["fastx"]


def test_usage_errors():
    with pytest.raises(cli.UsageError, match="'-ref' is required"):
        cli.parse_args(["-reads", READS])
    with pytest.raises(cli.UsageError, match="'-reads' is required"):
        cli.parse_args(["-ref", ARC])
    with pytest.raises(cli.UsageError, match="given twice"):
        parse("-sam", "-sam")
    with pytest.raises(cli.UsageError, match="needs a value"):
        parse("-match")
    with pytest.raises(cli.UsageError, match="once per '-ref'"):
        cli.parse_args(["-ref", ARC, "-ref", BAC, "-reads", READS, "-gumbel", "0.5,0.3"])
    with pytest.raises(cli.UsageError, match="once per '-ref'"):
        parse("-minimal_score", "30")


def test_gumbel_lookup(tmp_path):
    d = cli.gumbel_defaults()
    name = sorted(d["gumbel"])[0]
    ref = tmp_path / name
    ref.write_bytes(open(ARC, "rb").read())
    k = cli.parse_args(["-ref", str(ref), "-reads", READS])
    assert k["gumbel"] == [(d["gumbel"][name]["lambda_"], d["gumbel"][name]["K"])]
    with pytest.raises(cli.UsageError, match=f"no Gumbel parameters for reference '{ARC}'"):
        cli.parse_args(["-ref", str(ref), "-ref", ARC, "-reads", READS])
    with pytest.raises(cli.UsageError, match="default scoring only"):
        cli.parse_args(["-ref", str(ref), "-reads", READS, "-match", "3"])


def test_main_prints_usage_and_refuses(capsys):
    assert cli.main(["-h"]) == 0 and "-threads N" in capsys.readouterr().out
    assert cli.main(["-ref", ARC, "-reads", READS, "-bogus"]) == 2
    assert "option '-bogus' is not supported" in capsys.readouterr().err


@pytest.mark.parametrize("max_mb", [3072.0, 0.5])
def test_fasta_index_stats_equal_the_builders(max_mb):
    with tempfile.TemporaryDirectory(prefix="smr_cli_") as d:
        for f in (ARC, BAC):
            prefix = os.path.join(d, os.path.basename(f))
            api.build_index(f, prefix, max_mb=max_mb)
            want = hostio.parse_stats(prefix)
            got, seqs = hostio.fasta_index_stats(f, 18, max_mb)
            for k in ("fasta_size", "fasta_name", "background_freq", "full_ref", "lnwin", "numseq", "num_parts", "parts"):
                assert getattr(got, k) == getattr(want, k), k
            assert hostio.sam_header_of(seqs, "x ", True) == hostio.sam_header([prefix], "x ", True)
