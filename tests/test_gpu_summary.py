"""aligned.log and the OTU map of paired reads through the library (ReportWriter(summary=..., otu_map=..., otu_feed=...), stream_fastx /
stream_mates): against the reference binary (-threads 1, the golden databases) where it is built -- aligned.log equal apart from the
Command, pid and timestamp lines, otu_map.txt byte-identical -- and the paired maps against tests/golden/otu_map.json without it."""
import gzip
import json
import os
import shutil
import tempfile

import pytest

from conftest import GOLDEN
from integration_common import REF_DIR, golden_mates
from sortmerna_b200 import api
from summary_common import log_inputs, strip_volatile

pytestmark = pytest.mark.gpu

REFS = [os.path.join(GOLDEN, "db_arc.fasta"), os.path.join(GOLDEN, "db_bac.fasta")]
MATE_SETS = {"out2": ["-out2"], "sout": ["-sout"], "out2_sout": ["-out2", "-sout"], "paired_in_out2": ["-paired_in", "-out2"],
             "paired_out_out2": ["-paired_out", "-out2"]}
OTU = ["-otu_map", "-de_novo_otu", "-id", "0.9", "-coverage", "0.9"]


def _need_ref():
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_ref")):
        pytest.skip("oracle/_ref/sortmerna_ref not built (oracle/Makefile.ref)")


def _thresholds(extra):
    return (float(extra[extra.index("-id") + 1]) if "-id" in extra else 0.97, float(extra[extra.index("-coverage") + 1]) if "-coverage" in extra else 0.97)


def _ours(golden, d, reads, extra, ms, gumbel=None, feed=None, batch_bytes=1 << 30):
    """the files ReportWriter writes for the run; reads: one file (stream_fastx) or two (stream_mates)"""
    al = api.Aligner(0)
    try:
        al.set_params(api.default_params())
        for k in range(2):
            al.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], ms[k], (18, 9, 3), golden["stats"][k].lnwin)
        th = _thresholds(extra)
        summary = dict(cmd="", refs=REFS, reads=reads, gumbel=gumbel, minimal_score=ms) if gumbel is not None else None
        w = api.ReportWriter(d, al, otu_map=th if "-otu_map" in extra else None, otu_feed=feed, summary=summary, fastx=True,
                             denovo=th if "-de_novo_otu" in extra else None, out2="-out2" in extra, sout="-sout" in extra,
                             paired_in="-paired_in" in extra, paired_out="-paired_out" in extra)
        gen = al.stream_mates(reads[0], reads[1], batch_bytes=batch_bytes, piece_bytes=4096) if len(reads) == 2 else \
            al.stream_fastx(reads[0], batch_bytes=batch_bytes)
        for _ in gen:
            al.run_resident(with_stats=True)
            w.write(al.download(), None)
        paths = w.close()
        files = {os.path.basename(p): open(p, "rb").read() for p in paths if os.path.basename(p) in ("aligned.log", "otu_map.txt")}
        return files, w
    finally:
        al.close()


def _check_against_reference(golden, golden_idx_dir, d, reads, extra, feed=None):
    from oracle import ora
    r = ora.run_reference(REFS, reads, os.path.join(d, "ref"), extra=["-fastx"] + extra, threads=1, idx_dir=golden_idx_dir)
    inp = log_inputs(r["log"])
    files, w = _ours(golden, os.path.join(d, "ours"), reads, extra, inp["minimal_score"], inp["gumbel"], feed)
    assert strip_volatile(files["aligned.log"].decode()) == strip_volatile(r["log"])
    want_otu = os.path.join(r["out_dir"], "otu_map.txt")
    if "-otu_map" in extra:
        assert files.get("otu_map.txt") == (open(want_otu, "rb").read() if os.path.exists(want_otu) else None)
        assert f"Total OTUs = {w.total_otu}\n" in r["log"]
        assert f"thresholds = {w.denovo_counts['n_yid_ycov']} (" in r["log"]
    return files, w


@pytest.mark.parametrize("shape", ["fastq", "fastq_gz"])
def test_single_end_against_reference_binary(golden, golden_idx_dir, shape):
    _need_ref()
    d = tempfile.mkdtemp(prefix="smr_sum_")
    try:
        reads = os.path.join(d, "reads.fq" + (".gz" if shape == "fastq_gz" else ""))
        data = open(os.path.join(GOLDEN, "reads_mix.fq"), "rb").read()
        open(reads, "wb").write(gzip.compress(data, 6) if shape == "fastq_gz" else data)
        files, w = _check_against_reference(golden, golden_idx_dir, d, [reads], ["-otu_map", "-de_novo_otu"])
        assert w.n_yid_ycov == w.denovo_counts["n_yid_ycov"] > 0   # single-end: map entries and the log's figure agree
    finally:
        shutil.rmtree(d, ignore_errors=True)


@pytest.mark.parametrize("name", sorted(MATE_SETS))
def test_mates_against_reference_binary(golden, golden_idx_dir, name):
    """two mate files through stream_mates: the OTU map holds the first file's reads, the log counts both files"""
    _need_ref()
    d = tempfile.mkdtemp(prefix="smr_sum_")
    try:
        reads = golden_mates(d)
        files, w = _check_against_reference(golden, golden_idx_dir, d, reads, MATE_SETS[name] + OTU, feed="two_files")
        assert w.n_yid_ycov < w.denovo_counts["n_yid_ycov"]
    finally:
        shutil.rmtree(d, ignore_errors=True)


def _interleaved(d, reads):
    recs = [open(p, "rb").read().split(b"\n") for p in reads]
    p = os.path.join(d, "mates_interleaved.fastq")
    with open(p, "wb") as f:
        f.write(b"".join(b"\n".join(recs[j][i:i + 4]) + b"\n" for i in range(0, len(recs[0]) - 3, 4) for j in (0, 1)))
    return p


def test_interleaved_against_reference_binary(golden, golden_idx_dir):
    """the same reads as one interleaved -paired_in file: every record goes to the map"""
    _need_ref()
    d = tempfile.mkdtemp(prefix="smr_sum_")
    try:
        p = _interleaved(d, golden_mates(d))
        _check_against_reference(golden, golden_idx_dir, d, [p], ["-paired_in", "-out2"] + OTU, feed="one_file")
    finally:
        shutil.rmtree(d, ignore_errors=True)


@pytest.mark.parametrize("case,feed", [("paired_files", "two_files"), ("paired_interleaved", "one_file")])
def test_paired_maps_against_committed(golden, case, feed, tmp_path):
    """the reference's -paired_in maps of otu_map.json, with no reference binary; three batches write what one batch writes"""
    with open(os.path.join(GOLDEN, "otu_map.json")) as f:
        c = json.load(f)[case]
    reads = golden_mates(str(tmp_path))
    if feed == "one_file":
        reads = [_interleaved(str(tmp_path), reads)]
    extra = ["-paired_in", "-otu_map", "-id", str(c["min_id"]), "-coverage", str(c["min_cov"])]
    one, w = _ours(golden, str(tmp_path / "one"), reads, extra, c["minimal_score"], feed=feed)
    assert one["otu_map.txt"].decode() == c["otu_map"] and w.total_otu == c["total_otu"]
    if feed == "two_files":
        t = sum(os.path.getsize(p) for p in reads)
        three, w3 = _ours(golden, str(tmp_path / "three"), reads, extra, c["minimal_score"], feed=feed, batch_bytes=t // 3 + 1)
        assert three == one and (w3.total_otu, w3.n_yid_ycov) == (w.total_otu, w.n_yid_ycov)


def test_summary_three_batches_equal_one(golden, tmp_path):
    """aligned.log of the golden mates in three batches equals that of one batch"""
    reads = golden_mates(str(tmp_path))
    ms, gumbel = [37, 36], [(0.594908, 0.326193), (0.600371, 0.328947)]
    t = sum(os.path.getsize(p) for p in reads)
    one, w1 = _ours(golden, str(tmp_path / "one"), reads, OTU, ms, gumbel, feed="two_files")
    three, w3 = _ours(golden, str(tmp_path / "three"), reads, OTU, ms, gumbel, feed="two_files", batch_bytes=t // 3 + 1)
    strip = lambda f: {k: strip_volatile(v.decode()) for k, v in f.items()}   # noqa: E731
    assert strip(three) == strip(one) and w3.denovo_counts == w1.denovo_counts


def test_refusals(golden, tmp_path):
    """a mate-stream batch added to a single-end accumulator is refused; so are an unknown feed and a paired map without a feed"""
    reads = golden_mates(str(tmp_path))
    al = api.Aligner(0)
    try:
        al.set_params(api.default_params())
        for k in range(2):
            al.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], 37 - k, (18, 9, 3), golden["stats"][k].lnwin)
        for _ in al.stream_mates(reads[0], reads[1]):
            al.run_resident(with_stats=True)
            out = al.download()
            al.otu_begin(0.97, 0.97)
            with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED"):
                al.otu_add(out, None)
            al.otu_begin(0.97, 0.97, feed="one_file")
            with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED"):
                al.otu_add(out, None)
            al.otu_begin(0.97, 0.97, feed="two_files")
            assert al.otu_add(out, None) > 0
            text = al.resident_text()
            with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):   # an odd paired batch
                al.otu_add(dict(out, res=out["res"][:-1], alns=out["alns"][:-out["slots"]], stats=out["stats"][:-out["slots"]]),
                           text[:text.rstrip(b"\n").rfind(b"\n@") + 1])
            break
        with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):
            al.otu_begin(0.97, 0.97, feed=7)
        with pytest.raises(api.SmrError, match="SMR_ERR_UNSUPPORTED"):
            api.ReportWriter(str(tmp_path / "w"), al, otu_map=(0.97, 0.97), paired_out=True)
    finally:
        al.close()
