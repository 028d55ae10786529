"""The seed kernel screens every streamed entry with half_screen (sortmerna_b200/csrc/smr_levbits.h) and classifies only the
survivors exactly.  This host-side check proves that the screen accepts every text within one edit of the pattern and that
screen + exact classification decides exactly as within_one_edit: pw = 9 exhaustively over one-edit neighbours, every
(pattern, text) pair for pw <= 6, and random patterns, neighbours and pairs up to pw = 15."""
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_half_screen_keeps_every_match_and_decides_with_classify_bits():
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "seed_filter_check")
        subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "seed_filter_check.cpp"), "-o", exe])
        out = subprocess.run([exe, "1000000"], stdout=subprocess.PIPE, text=True)
        assert out.returncode == 0, out.stdout
        rows = [ln.split() for ln in out.stdout.splitlines()]
        assert [int(r[1]) for r in rows] == list(range(4, 16)), out.stdout
        for r in rows:
            assert r[6] == "missed" and r[7] == "0" and r[8] == "mismatched" and r[9] == "0", out.stdout
            assert int(r[3]) > 0, out.stdout
        pw9 = rows[9 - 4]
        assert int(pw9[5]) == 4 ** 9 * (9 * 16 + 9 * 16 + 10 * 4), "every one-edit neighbour of every pattern at pw = 9"
        # the screen is worth streaming with: about 1 % of random pairs pass at pw = 9
        assert int(pw9[11]) < 20000, out.stdout
