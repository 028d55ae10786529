"""The read stream on the device (smr_stream_*, Aligner.stream_fastx / read_counts): files pushed piece by piece come back as
record-aligned batches that decode to exactly the reads of the whole file, and are counted as the reference's
count_reads_parallel counts them."""
import gzip
import json
import os
import sys
import zlib

import numpy as np
import pytest

import inflate_cases
from conftest import GOLDEN, load_case
from helpers import assert_same_results
from sortmerna_b200 import api, hostio
from test_gpu_reports import BLAST, _aligner
from test_stream_host import count_inputs, ref_count, ref_count_run

sys.path.insert(0, GOLDEN)
import make_stream_counts  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def aligner(golden):
    al = api.Aligner(0)
    al.set_params(api.default_params())
    exp = load_case("default")
    for k in range(2):
        al.load_index_part(k, 0, golden["prefixes"][k], golden["refs"][k], exp["log"]["minimal_score"][k], (18, 9, 3), golden["stats"][k].lnwin)
    yield al
    al.close()


def fasta_text(n, seed=11, width=0):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        seq = "".join(rng.choice(list("ACGTN"), int(rng.integers(40, 200)), p=[0.24, 0.24, 0.24, 0.24, 0.04]))
        if width:
            seq = "\n".join(seq[k:k + width] for k in range(0, len(seq), width))
        out.append(f">seq{i} sample={i % 13}\n{seq}\n")
    return "".join(out).encode()


def layout(al, text):
    """(read lengths, 0-4 codes, header lines) of the resident batch"""
    hdr, off, seq = al.resident_layout()
    heads = [text[int(h):text.index(b"\n", int(h)) if b"\n" in text[int(h):] else len(text)] for h in hdr]
    return np.diff(off.astype(np.int64)), seq, heads


def whole(al, data, gz):
    n = al.upload_fastx_gz(data) if gz else al.upload_fastx(data)
    text = al.resident_text()
    lens, seq, heads = layout(al, text)
    assert lens.size == n
    return lens, seq, heads


def streamed(al, path, batch, piece):
    lens, seqs, heads, sizes = [], [], [], []
    for n in al.stream_fastx(path, batch_bytes=batch, piece_bytes=piece):
        text = al.resident_text()
        ln, sq, hd = layout(al, text)
        assert ln.size == n
        sizes.append((len(text), n, int(al.resident_layout(with_seq=False)[0][1]) if n > 1 else len(text)))
        lens.append(ln); seqs.append(sq); heads += hd
    return np.concatenate(lens) if lens else np.zeros(0, np.int64), np.concatenate(seqs) if seqs else np.zeros(0, np.uint8), heads, sizes


def stream_inputs():
    fq = open(os.path.join(GOLDEN, "reads_mix.fq"), "rb").read()
    txt = inflate_cases.fastq_text(3000, seed=12)
    third = len(txt) // 3
    co = zlib.compressobj(6, zlib.DEFLATED, 31, 9, zlib.Z_FIXED)
    fixed = co.compress(txt) + co.flush()
    return [
        ("golden_fq", fq, False, fq),
        ("golden_fq_gz", gzip.compress(fq, 6), True, fq),
        ("fasta_100k", fasta_text(100000), False, None),
        ("multiline_fasta", fasta_text(3000, width=60), False, None),
        ("crlf", txt.replace(b"\n", b"\r\n"), False, None),
        ("multi_member", gzip.compress(txt[:third], 1) + gzip.compress(txt[third:], 9), True, txt),
        ("gzip1", gzip.compress(txt, 1), True, txt),
        ("gzip9", gzip.compress(txt, 9), True, txt),
        ("stored", gzip.compress(txt, 0), True, txt),
        ("fixed", fixed, True, txt),
    ]


def test_streamed_batches_equal_whole_file(aligner, tmp_path):
    for name, data, gz, _ in stream_inputs():
        path = tmp_path / name
        path.write_bytes(data)
        want = whole(aligner, data, gz)
        for piece in (4096, 65536, len(data) + 1):
            for batch in ((100,) if len(data) < 300000 else ()) + (20000, 1 << 20, len(data) * 10):
                lens, seq, heads, sizes = streamed(aligner, str(path), batch, piece)
                assert np.array_equal(lens, want[0]), (name, piece, batch)
                assert np.array_equal(seq, want[1]), (name, piece, batch)
                assert heads == want[2], (name, piece, batch)
                for k, (nbytes, n, _) in enumerate(sizes):
                    assert nbytes <= batch or n == 1, (name, piece, batch, nbytes, n)   # within batch_bytes, unless one record alone is longer
                    if k + 1 < len(sizes):   # and full: the next batch's first record would not have fit
                        assert nbytes + sizes[k + 1][2] > batch, (name, piece, batch, k, nbytes, sizes[k + 1][2])


def test_streamed_alignments_equal_one_batch(aligner, golden, tmp_path):
    data = open(os.path.join(GOLDEN, "reads_mix.fq"), "rb").read()
    path = tmp_path / "reads.fq.gz"
    path.write_bytes(gzip.compress(data, 6))
    aligner.upload_fastx(data)
    aligner.run_resident()
    want = aligner.download()
    k = 0
    for n in aligner.stream_fastx(str(path), batch_bytes=30000, piece_bytes=8192):
        aligner.run_resident()
        got = aligner.download()
        sub = {"res": want["res"][k:k + n], "alns": want["alns"][k * want["slots"]:(k + n) * want["slots"]], "cigar": want["cigar"], "slots": want["slots"]}
        assert_same_results(got, sub, f"batch at read {k}")
        k += n
    assert k == want["res"].size


def test_read_counts_equal_count_reads_parallel(aligner, tmp_path):
    fq = open(os.path.join(GOLDEN, "reads_mix.fq"), "rb").read()
    exp = load_case("default")["log"]
    p = tmp_path / "reads.fq"
    p.write_bytes(fq)
    pz = tmp_path / "reads.fq.gz"
    pz.write_bytes(gzip.compress(fq, 6))
    want = ref_count(fq)
    assert want["reads"] == exp["total_reads"]
    for piece in (4096, 1 << 20):
        assert aligner.read_counts(str(p), piece_bytes=piece) == want
        assert aligner.read_counts(str(pz), piece_bytes=piece) == want
    for name, data in count_inputs().items():
        q = tmp_path / name
        q.write_bytes(data)
        assert aligner.read_counts(str(q), piece_bytes=4096) == ref_count(data), name
    # several files of one run (mates), flat, gzip and mixed: the minimum follows the reference's per-format rule
    ins = count_inputs()
    parts = [(ins["empty_seq_lines"], False), (ins["empty_last"], True), (ins["fasta"], False), (ins["empty_seq_lines"], True), (ins["fasta"], True)]
    for combo in ([0, 2], [1, 3], [1, 0], [3, 2], [0, 1, 2, 3, 4], [4, 1]):
        files, paths = [], []
        for j in combo:
            data, gz = parts[j]
            q = tmp_path / f"part{j}{'.gz' if gz else ''}"
            q.write_bytes(gzip.compress(data) if gz else data)
            files.append((data, gz)); paths.append(str(q))
        assert aligner.read_counts(paths, piece_bytes=4096) == ref_count_run(files), combo


def test_read_counts_equal_reference_binary(aligner, golden, tmp_path):
    """"Total reads" and every index's minimal SW score the unmodified reference printed at -threads 1 (tests/golden/stream_counts.json,
    made by tests/golden/make_stream_counts.py) follow from read_counts"""
    want = json.load(open(os.path.join(GOLDEN, "stream_counts.json")))
    ins = make_stream_counts.inputs(str(tmp_path))
    assert sorted(ins) == sorted(want)
    for name, paths in ins.items():
        w = want[name]
        for piece in (4096, 1 << 20):
            c = aligner.read_counts(paths, piece_bytes=piece)
            assert c["reads"] == w["total_reads"], (name, c)
            for k in range(2):
                assert hostio.minimal_score(golden["stats"][k], w["lambda_"][k], w["K"][k], c["length"], c["reads"]) == w["minimal_score"][k], (name, k, c)
        files = [(gzip.decompress(open(p, "rb").read()) if p.endswith(".gz") else open(p, "rb").read(), p.endswith(".gz")) for p in paths]
        assert c == ref_count_run(files), name


def test_report_writer_over_streamed_batches(golden, tmp_path):
    """ReportWriter over the streamed batches writes what it writes over one batch, byte for byte: SAM, BLAST, aligned / other /
    denovo reads and otu_map.txt; with zip_out, the same bytes once inflated"""
    exp = load_case("best3")
    text = open(os.path.join(GOLDEN, "reads_mix.fq"), "rb").read()
    path = tmp_path / "reads.fq.gz"
    path.write_bytes(gzip.compress(text, 6))
    a = _aligner(golden, exp)
    for zip_out in (False, True):
        res = {}
        for name in ("one", "streamed"):
            w = api.ReportWriter(str(tmp_path / f"{name}{int(zip_out)}"), a, sam_header=hostio.sam_header(golden["prefixes"], "sortmerna"), sam=True,
                                 blast=BLAST, fastx=True, other=True, denovo=(0.97, 0.97), otu_map=(0.97, 0.97), zip_out=zip_out)
            batches = 0
            if name == "one":
                a.upload_fastx(text)
                a.run_resident(with_stats=True)
                w.write(a.download())
            else:
                for _ in a.stream_fastx(str(path), batch_bytes=40000, piece_bytes=16384):
                    a.run_resident(with_stats=True)
                    w.write(a.download())
                    batches += 1
                assert batches > 3
            res[name] = {os.path.basename(f): open(f, "rb").read() for f in w.close()}
        assert "otu_map.txt" in res["one"] and len(res["one"]) >= 6, sorted(res["one"])
        assert sorted(res["streamed"]) == sorted(res["one"])
        for fn in res["one"]:   # -zip-out: each batch's output is its own gzip member, so the inflated files must agree
            got, want = res["streamed"][fn], res["one"][fn]
            if zip_out and fn.endswith(".gz"):
                got, want = gzip.decompress(got), gzip.decompress(want)
                assert want == plain[fn[:-3]], fn
            assert got == want, (zip_out, fn)
        plain = res["one"]
    a.close()


def test_corrupt_streams_are_refused(aligner, tmp_path):
    txt = inflate_cases.fastq_text(20000, seed=13)
    good = gzip.compress(txt, 6)
    flipped = bytearray(good)
    flipped[len(good) // 2] ^= 0x55
    bad_crc = bytearray(good)
    bad_crc[-8] ^= 1
    for name, data in (("bit_flip", bytes(flipped)), ("truncated", good[:-3000]), ("crc", bytes(bad_crc))):
        path = tmp_path / name
        path.write_bytes(data)
        with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):
            aligner.read_counts(str(path), piece_bytes=65536)
        with pytest.raises(api.SmrError, match="SMR_ERR_ARG"):
            for _ in aligner.stream_fastx(str(path), batch_bytes=100000, piece_bytes=65536):
                pass
        # the context streams again after the failure
        ok = tmp_path / "ok.gz"
        ok.write_bytes(good)
        assert sum(aligner.stream_fastx(str(ok), batch_bytes=100000, piece_bytes=65536)) == 20000


def test_past_four_gib(aligner, tmp_path):
    """A .fastq.gz of more than 2^32 bytes of text: one member, a 64 MB block of records deflated once and repeated (each copy
    ends in a full flush, so it needs no history)."""
    block = inflate_cases.fastq_text(4000, seed=14)
    block = block * (64 * 2**20 // len(block))
    copies = (2**32 // len(block)) + 2
    co = zlib.compressobj(1, zlib.DEFLATED, -15)
    body = co.compress(block) + co.flush(zlib.Z_FULL_FLUSH)
    crc = 0
    path = tmp_path / "big.fastq.gz"
    with open(path, "wb") as f:
        f.write(b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff")
        for _ in range(copies):
            f.write(body)
            crc = zlib.crc32(block, crc)
        f.write(b"\x03\x00")   # final empty fixed block
        f.write(crc.to_bytes(4, "little") + ((len(block) * copies) & 0xFFFFFFFF).to_bytes(4, "little"))
    one = ref_count(block)
    got = aligner.read_counts(str(path), piece_bytes=256 << 20)
    assert got == {"reads": one["reads"] * copies, "length": one["length"] * copies, "min_len": one["min_len"], "max_len": one["max_len"]}
    per_block = one["reads"]

    def header(text, off):
        return text[int(off):text.index(b"\n", int(off))]

    total, batches, last = 0, 0, None
    for n in aligner.stream_fastx(str(path), batch_bytes=512 << 20, piece_bytes=256 << 20):
        # every read in order: the first and last header of each batch are the records the running count names
        text = aligner.resident_text()
        hdr = aligner.resident_layout(with_seq=False)[0]
        assert header(text, hdr[0]) == b"@read%d/1 sample" % (total % 4000), (batches, total)
        assert header(text, hdr[-1]) == b"@read%d/1 sample" % ((total + n - 1) % 4000), (batches, total)
        if batches == 0:
            aligner.run_resident()
            assert aligner.download()["res"].size == n
        total += n
        batches += 1
        last = n
    assert total == per_block * copies and batches > 8
    assert text.endswith(block[-len(text):] if len(text) <= len(block) else block)   # the last batch ends with the file's last record
    aligner.run_resident()
    assert aligner.download()["res"].size == last
