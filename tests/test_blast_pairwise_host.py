"""The pairwise BLAST restatement (hostio.format_blast_pairwise_rows, -blast 0) on the CPU oracle's alignments of each fixture's
reads prints what the reference binary printed (tests/golden/blast_pairwise/): the header lines, the 60-column blocks, their
positions and the '|' / '*' / ' ' line, byte for byte (E-values to their last printed digit, pairwise_common)."""
import pytest

from oracle import ora
from pairwise_common import CASES, assert_pairwise_equal, expected, inputs
from sortmerna_b200 import hostio


def _oracle_rows(case, golden_idx_dir):
    x = inputs(case, golden_idx_dir)
    n = len(x["prefixes"])
    oix = [ora.OracleIndex(p, 0, st.lnwin) for p, st in zip(x["prefixes"], x["stats"])]
    out = ora.align(oix, list(range(n)), [0] * n, n, x["refs"], x["minimal_score"], [18, 9, 3] * n, ora.default_params(**x["params"]),
                    x["batch"])
    return hostio.format_blast_pairwise_rows(x["batch"], x["refs"], out["res"], out["alns"], out["cigar"], out["slots"], x["gumbel"],
                                             x["ev_params"])


@pytest.mark.parametrize("case", sorted(CASES))
def test_restatement_equals_reference(golden_idx_dir, case):
    rows = _oracle_rows(case, golden_idx_dir)
    want = expected(case)
    assert len(rows) == CASES[case]["rows"] and len(want) == CASES[case]["bytes"]
    assert_pairwise_equal("".join(rows).encode(), want)


def test_block_layout():
    """one alignment by hand: 61 columns, an I at column 59 and a D at column 60, cut into a block of 60 and a block of 1 + 1"""
    import numpy as np
    from sortmerna_b200 import api
    ref = hostio.References("r", ["ref1"], hostio.encode_nt("ACGT" * 20), np.array([0, 80], np.uint64))
    enc = hostio.encode_nt(b"CC" + b"ACGT" * 15 + b"G")
    al = np.zeros(1, api.ALN_DTYPE)[0]
    al["ref_begin1"], al["read_begin1"], al["strand"], al["score1"], al["cigar_len"] = 4, 2, 1, 100, 4
    cig = np.array([(59 << 4) | 0, (1 << 4) | 1, (1 << 4) | 2, (1 << 4) | 0], np.uint32)
    lines = hostio._pairwise_row(">read1 x", enc, al, ref, cig, [(0.6, 0.3)], [(1000, 1000)]).split("\n")
    assert lines[:2] == ["Sequence ID: ref1", "Query ID: read1"] and lines[2].startswith("Score: 100 bits (88)\tExpect: ") and lines[3] == ""
    assert lines[4] == "Target: " + " " * 7 + "5    " + ("ACGT" * 15)[:59] + "-    63"
    assert lines[5] == " " * 20 + "|" * 59 + " "
    assert lines[6] == "Query: " + " " * 8 + "3    " + ("ACGT" * 15)[:60] + "    62"
    assert lines[7] == ""
    assert lines[8] == "Target: " + " " * 6 + "64    TA    65"
    assert lines[9] == " " * 20 + " *"
    assert lines[10] == "Query: " + " " * 7 + "63    -G    63"
    assert lines[11:] == ["", ""]
