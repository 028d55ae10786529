"""hostio.summary_log (Summary::to_string, summary.cpp:102-175) fed with the oracle's counters against the reference binary's
aligned.log (tests/golden/aligned_log, made by tests/golden/make_summary_golden.py), and the paired OTU rule of hostio.otu_map /
hostio.denovo_classes on the oracle's results against the reference's paired runs (tests/golden/otu_map.json)."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import params_kwargs_from_args
from oracle import ora
from sortmerna_b200 import hostio
from summary_common import log_inputs, strip_volatile

LOGS = os.path.join(GOLDEN, "aligned_log")
with open(os.path.join(LOGS, "cases.json")) as _f:
    CASES = json.load(_f)


def _records():
    lines = open(os.path.join(GOLDEN, "reads_mix.fq"), "rb").read().split(b"\n")
    return [lines[i:i + 4] for i in range(0, len(lines) - 3, 4)]


def _oracle(golden, batch, args, minimal_score):
    keep = []
    for i, a in enumerate(args):   # the alignment options alone
        if a == "-num_alignments":
            keep += args[i:i + 2]
    oix = [ora.OracleIndex(p, 0, s.lnwin) for p, s in zip(golden["prefixes"], golden["stats"])]
    out = ora.align(oix, [0, 1], [0, 0], 2, golden["refs"], minimal_score, [18, 9, 3] * 2, ora.default_params(**params_kwargs_from_args(keep)),
                    batch, nthreads=2)
    return out, hostio.host_aln_stats(batch, golden["refs"], out["res"], out["alns"], out["cigar"], out["slots"])


def _thresholds(args):
    mid = float(args[args.index("-id") + 1]) if "-id" in args else 0.97   # the reference's defaults under -otu_map
    mcov = float(args[args.index("-coverage") + 1]) if "-coverage" in args else 0.97
    return mid, mcov


@pytest.mark.parametrize("case", sorted(CASES))
def test_summary_log_matches_reference(golden, case):
    c = CASES[case]
    want = open(os.path.join(LOGS, case + ".log")).read()
    recs = _records()
    sel = [recs[i] for i in (range(len(recs)) if c["reads"] is None else c["reads"])]
    batch = hostio.pack_reads([r[0].decode() for r in sel], [r[1] for r in sel], [r[3] for r in sel])
    inp = log_inputs(want)
    args = c["args"]
    out, st = _oracle(golden, batch, args, inp["minimal_score"])
    lens = [len(s) for s in batch.seqs]
    denovo = otu = None
    if "-otu_map" in args or "-de_novo_otu" in args:
        mid, mcov = _thresholds(args)
        tot = hostio.denovo_classes(out["res"], out["alns"], out["slots"], st, mid, mcov).sum(axis=0, dtype=np.uint64)
        if "-de_novo_otu" in args:
            denovo = int(tot[3])
        if "-otu_map" in args:
            m = hostio.otu_map(golden["refs"], batch.headers, out["res"], out["alns"], out["slots"], st, mid, mcov)
            otu = (int(tot[0]), m["total_otu"])
    got = hostio.summary_log("", ["db_arc.fasta", "db_bac.fasta"], ["reads.fq"], total_reads=batch.n, num_aligned=out["counters"]["num_aligned"],
                             min_len=min(lens), max_len=max(lens), all_reads_len=sum(lens), reads_matched_per_db=[int(x) for x in out["matched"]],
                             sq="-SQ" in args, denovo=denovo, otu=otu, timestamp="Thu Jan  1 00:00:00 1970", **inp)
    assert got.endswith("\n Thu Jan  1 00:00:00 1970\n\n") and got.startswith(" Command:\n    \n\n Process pid = \n\n")
    assert strip_volatile(got) == want


def test_cases_cover_the_edges():
    """an all-aligned run, a none-aligned one, -SQ, and a ratio whose float32 value prints otherwise than its double would"""
    logs = {c: open(os.path.join(LOGS, c + ".log")).read() for c in CASES}
    assert "failing E-value threshold = 0 (0.00)" in logs["all_aligned"]
    assert "passing E-value threshold = 0 (0.00)" in logs["none_aligned"]
    assert "SQ tags are output" in logs["sq"]
    assert "= 13 (8.13)" in logs["float_edge"] and f"{13 / 160 * 100:.2f}" == "8.12"
    assert "Total reads for de novo clustering" in logs["otu_denovo"] and "Total OTUs" in logs["otu_denovo"]


def _mates_batch():
    """the golden mates (integration_common.golden_mates) interleaved: records 2k, 2k+1 are record k of mate 1 and of mate 2"""
    recs = [r for r in _records() if r[0].startswith(b"@") and len(r[1]) >= 18]
    recs = recs[: len(recs) // 2 * 2]
    return hostio.pack_reads([r[0].decode() for r in recs], [r[1] for r in recs], [r[3] for r in recs])


@pytest.mark.parametrize("case,feed", [("paired_files", "two_files"), ("paired_interleaved", "one_file")])
def test_paired_otu_map_matches_reference(golden, case, feed):
    """otu_map.txt of the reference's -paired_in runs: two mate files (the first file's reads alone) and one interleaved file (every
    record); the log's "passing %id and %coverage" figure is the n_yid_ycov total of the paired denovo_stats pass in both"""
    with open(os.path.join(GOLDEN, "otu_map.json")) as f:
        c = json.load(f)[case]
    batch = _mates_batch()
    out, st = _oracle(golden, batch, [], c["minimal_score"])
    lens = np.array([len(s) for s in batch.seqs])
    m = hostio.otu_map(golden["refs"], batch.headers, out["res"], out["alns"], out["slots"], st, c["min_id"], c["min_cov"], feed=feed, seq_lens=lens)
    assert m["text"].decode() == c["otu_map"] and m["total_otu"] == c["total_otu"]
    cls = hostio.denovo_classes(out["res"], out["alns"], out["slots"], st, c["min_id"], c["min_cov"], paired=True, seq_lens=lens)
    assert int(cls[:, 0].sum()) == c["n_yid_ycov"]
    if feed == "two_files":
        assert m["n_yid_ycov"] < c["n_yid_ycov"]


def test_pair_skip_rule():
    """a pair whose second read is empty counts for neither mate, in denovo_classes and in the OTU gate; an empty first read does not
    skip its pair"""
    from sortmerna_b200 import api
    res = np.zeros(4, api.RESULT_DTYPE)
    alns = np.zeros(4, api.ALN_DTYPE)
    st = np.zeros(4, api.STATS_DTYPE)
    for r in (0, 3):
        res["n_align"][r] = 1
        alns[r] = (0, 0, 0, 0, 99, 0, 99, 100, 200, 0, 0, 1, 0)
        st[r] = (0, 0, 100, 100)
    lens = np.array([100, 0, 0, 100])
    assert hostio.denovo_classes(res, alns, 1, st, 0.97, 0.97, paired=True, seq_lens=lens).tolist() == [[0] * 4, [0] * 4, [0] * 4, [1, 0, 0, 0]]
    assert hostio.denovo_classes(res, alns, 1, st, 0.97, 0.97).tolist() == [[1, 0, 0, 0], [0] * 4, [0] * 4, [1, 0, 0, 0]]
