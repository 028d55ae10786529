"""Paired-end reads end to end: two mate files streamed through the device as pairs (smr_stream_push_mate, Aligner.stream_mates)
come back as batches of whole pairs whose decode equals the host's interleaving of the two files, and the paired report files
(-out2 / -sout, ReportWriter) equal the reference binary's."""
import gzip
import os
import shutil
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, load_case
from helpers import assert_same_results
from integration_common import REF_DIR, golden_mates
from sortmerna_b200 import api
from test_gpu_stream import fasta_text, layout

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


def records(text):
    """the records of a FASTQ (4 lines) or FASTA (a '>' line and the lines up to the next) text, each ending in '\\n'"""
    if not text:
        return []
    if not text.endswith(b"\n"):
        text += b"\n"
    lines = text.split(b"\n")[:-1]
    if text[:1] == b"@":
        return [b"".join(ln + b"\n" for ln in lines[i:i + 4]) for i in range(0, len(lines), 4)]
    out = []
    for ln in lines:
        if ln.startswith(b">") or not out:
            out.append(b"")
        out[-1] += ln + b"\n"
    return out


def interleave(t1, t2):
    r1, r2 = records(t1), records(t2)
    assert len(r1) == len(r2)
    return b"".join(a + b for a, b in zip(r1, r2))


def mate_texts(d):
    p = golden_mates(str(d))
    return open(p[0], "rb").read(), open(p[1], "rb").read()


def streamed(al, p1, p2, batch, piece):
    """(lens, codes, headers) of every batch, and per batch (text bytes, reads, bytes of its first pair)"""
    lens, seqs, heads, sizes = [], [], [], []
    for n in al.stream_mates(p1, p2, batch_bytes=batch, piece_bytes=piece):
        text = al.resident_text()
        ln, sq, hd = layout(al, text)
        assert ln.size == n and n % 2 == 0
        hdr = al.resident_layout(with_seq=False)[0]
        sizes.append((len(text), n, int(hdr[2]) if n > 2 else len(text)))
        lens.append(ln); seqs.append(sq); heads += hd
    return np.concatenate(lens), np.concatenate(seqs), heads, sizes


def check_against_whole(al, tmp_path, name, t1, t2, data1, data2, pieces, batches):
    p1, p2 = tmp_path / f"{name}_1", tmp_path / f"{name}_2"
    p1.write_bytes(data1)
    p2.write_bytes(data2)
    inter = interleave(t1, t2)
    al.upload_fastx(inter)
    want_text = al.resident_text()
    want = layout(al, want_text)
    for piece in pieces:
        for batch in batches:
            lens, seq, heads, sizes = streamed(al, str(p1), str(p2), batch, piece)
            assert np.array_equal(lens, want[0]), (name, piece, batch)
            assert np.array_equal(seq, want[1]), (name, piece, batch)
            assert heads == want[2], (name, piece, batch)
            for k, (nbytes, n, _) in enumerate(sizes):
                assert nbytes <= batch or n == 2, (name, piece, batch, nbytes, n)   # within batch_bytes, unless one pair alone is longer
                if k + 1 < len(sizes):   # and full: the next batch's first pair would not have fit
                    assert nbytes + sizes[k + 1][2] > batch, (name, piece, batch, k, nbytes, sizes[k + 1][2])


def test_mate_stream_equals_host_interleave(aligner, tmp_path):
    t1, t2 = mate_texts(tmp_path)
    pair = len(records(t1)[0]) + len(records(t2)[0])
    batches = (pair // 2, 3 * pair, 20000, len(t1) + len(t2), 10 * (len(t1) + len(t2)))
    check_against_whole(aligner, tmp_path, "flat", t1, t2, t1, t2, (4096, 65536, len(t1) + len(t2)), batches)
    for level in (1, 6, 9):
        check_against_whole(aligner, tmp_path, f"gz{level}", t1, t2, gzip.compress(t1, level), gzip.compress(t2, level), (4096, 1 << 20), batches)
    third = len(t2) // 3   # several members, cut at different places in the two files
    members1 = gzip.compress(t1[:len(t1) // 2], 1) + gzip.compress(t1[len(t1) // 2:], 9)
    members2 = gzip.compress(t2[:third], 6) + gzip.compress(t2[third:2 * third], 1) + gzip.compress(t2[2 * third:], 9)
    check_against_whole(aligner, tmp_path, "members", t1, t2, members1, members2, (4096, 65536), (pair // 2, 20000, 1 << 20))
    # CR LF, and mate 2 without the final newline (one is appended, as Readfeed::split does)
    c1, c2 = t1.replace(b"\n", b"\r\n"), t2[:-1]
    check_against_whole(aligner, tmp_path, "crlf", c1, c2, c1, c2, (4096, 1 << 20), (1000, 20000, 1 << 20))
    # multi-line FASTA
    f = fasta_text(600, seed=5, width=60)
    fr = records(f)
    f1, f2 = b"".join(fr[0::2]), b"".join(fr[1::2])
    check_against_whole(aligner, tmp_path, "fasta", f1, f2, f1, f2, (4096, 1 << 20), (300, 5000, 1 << 20))


def test_mate_alignments_equal_one_batch(aligner, tmp_path):
    t1, t2 = mate_texts(tmp_path)
    p1, p2 = tmp_path / "m1.fq.gz", tmp_path / "m2.fq.gz"
    p1.write_bytes(gzip.compress(t1, 6))
    p2.write_bytes(gzip.compress(t2, 6))
    aligner.upload_fastx(interleave(t1, t2))
    aligner.run_resident()
    want = aligner.download()
    k = 0
    for n in aligner.stream_mates(str(p1), str(p2), batch_bytes=30000, piece_bytes=8192):
        aligner.run_resident()
        got = aligner.download()
        sub = {"res": want["res"][k:k + n], "alns": want["alns"][k * want["slots"]:(k + n) * want["slots"]], "cigar": want["cigar"], "slots": want["slots"]}
        assert_same_results(got, sub, f"batch at read {k}")
        k += n
    assert k == want["res"].size


def _refused(al, fn, match):
    with pytest.raises(api.SmrError, match=match):
        fn()


def test_refusals_leave_the_context_usable(aligner, tmp_path):
    t1, t2 = mate_texts(tmp_path)
    r1, r2 = records(t1), records(t2)
    good1, good2 = tmp_path / "g1.fq", tmp_path / "g2.fq"
    good1.write_bytes(t1)
    good2.write_bytes(t2)

    def clean_run():
        assert sum(aligner.stream_mates(str(good1), str(good2), batch_bytes=20000, piece_bytes=65536)) == len(r1) + len(r2)

    short = tmp_path / "short.fq"
    short.write_bytes(b"".join(r2[:-1]))
    for a, b, who in ((good1, short, "mate 2 has ended while mate 1"), (short, good1, "mate 1 has ended while mate 2")):
        for batch in (1000, 1 << 20):
            _refused(aligner, lambda: sum(aligner.stream_mates(str(a), str(b), batch_bytes=batch, piece_bytes=4096)), who)
        clean_run()
    fa = tmp_path / "m2.fa"
    fa.write_bytes(b"".join(b">" + r.split(b"\n")[0][1:] + b"\n" + r.split(b"\n")[1] + b"\n" for r in r2))
    _refused(aligner, lambda: sum(aligner.stream_mates(str(good1), str(fa))), "mate 1 is FASTQ and mate 2 is FASTA")
    clean_run()
    z1, z2 = tmp_path / "z1.fq.gz", tmp_path / "z2.fq.gz"
    z1.write_bytes(gzip.compress(t1, 6))
    bad = bytearray(gzip.compress(t2[len(t2) // 2:], 6))   # a corrupt second member
    bad[len(bad) // 2] ^= 0x55
    z2.write_bytes(gzip.compress(t2[: len(t2) // 2], 6) + bytes(bad))
    _refused(aligner, lambda: sum(aligner.stream_mates(str(z1), str(z2), piece_bytes=4096)), "SMR_ERR_ARG: mate 2: gz input")
    clean_run()
    L, h = aligner.L, aligner.h
    import ctypes as C
    buf = np.frombuffer(t1[:100], np.uint8)
    assert L.smr_stream_begin(h, C.c_uint32(aligner.STREAM_MATES), C.c_uint64(1 << 20)) == 0
    assert L.smr_stream_push(h, api._ptr(buf), C.c_uint64(buf.size), C.c_int(0)) == 2
    assert b"smr_stream_push_mate" in L.smr_last_error(h)
    assert L.smr_stream_begin(h, C.c_uint32(0), C.c_uint64(1 << 20)) == 0
    assert L.smr_stream_push_mate(h, C.c_uint32(1), api._ptr(buf), C.c_uint64(buf.size), C.c_int(0)) == 2
    assert L.smr_stream_begin(h, C.c_uint32(aligner.STREAM_MATES | aligner.STREAM_COUNT_ONLY), C.c_uint64(0)) == 2
    assert L.smr_stream_begin(h, C.c_uint32(aligner.STREAM_MATES), C.c_uint64(1 << 20)) == 0
    assert L.smr_stream_push_mate(h, C.c_uint32(3), api._ptr(buf), C.c_uint64(buf.size), C.c_int(0)) == 2
    clean_run()
    # -sout with paired_in / paired_out; -out2 / -sout on a batch that is not paired stays unsupported
    aligner.run_resident(with_stats=True)
    out = aligner.download()
    for kw in (dict(paired_in=True), dict(paired_out=True)):
        _refused(aligner, lambda: aligner.format_reports(out, None, fastx=True, sout=True, **kw), "SMR_ERR_ARG")
    text = aligner.resident_text()
    _refused(aligner, lambda: aligner.format_reports(out, text, fastx=True, out2=True), "SMR_ERR_UNSUPPORTED")
    s = aligner.format_reports(out, text, fastx=True, out2=True, mates=True)
    assert s["aligned"] == aligner.format_reports(out, None, fastx=True, out2=True)["aligned"]
    clean_run()


OPTION_SETS = {
    "out2": ["-out2"],
    "sout": ["-sout"],
    "out2_sout": ["-out2", "-sout"],
    "paired_in_out2": ["-paired_in", "-out2"],
    "paired_out_out2": ["-paired_out", "-out2"],
}


def _kw(extra):
    return dict(out2="-out2" in extra, sout="-sout" in extra, paired_in="-paired_in" in extra, paired_out="-paired_out" in extra)


def _need_ref():
    if not os.path.exists(os.path.join(REF_DIR, "sortmerna_ref")):
        pytest.skip("oracle/_ref/sortmerna_ref not built (oracle/Makefile.ref)")


def _ours(golden, d, reads, extra, ref, log, denovo, zip_out, batch_bytes=1 << 30, piece_bytes=1 << 20):
    al = api.Aligner(0)
    try:
        al.set_params(api.default_params())
        al.load_index_part(0, 0, golden["prefixes"][1], golden["refs"][1], log["minimal_score"][0], (18, 9, 3), golden["stats"][1].lnwin)
        head = b"".join(ln + b"\n" for ln in ref["aligned.sam"].split(b"\n") if ln.startswith(b"@")).decode()
        w = api.ReportWriter(d, al, sam_header=head, zip_out=zip_out, sam=True, fastx=True, other=True, denovo=denovo, **_kw(extra))
        for _ in al.stream_mates(reads[0], reads[1], batch_bytes=batch_bytes, piece_bytes=piece_bytes):
            al.run_resident(with_stats=True)
            w.write(al.download(), None)
        paths = w.close()
    finally:
        al.close()
    return {os.path.basename(p): (gzip.open(p, "rb").read() if zip_out else open(p, "rb").read()) for p in paths}


@pytest.mark.parametrize("name", sorted(OPTION_SETS) + ["zip_out"])
def test_against_reference_binary(golden, golden_idx_dir, name):
    """every report file of the reference's paired run at -threads 1 (names and bytes; gzip compared after inflate), through
    stream_mates + ReportWriter.  The denovo sets use -otu_map -de_novo_otu -id -coverage (the reference takes -id / -coverage
    only with -otu_map); its otu_map.txt is not compared (the OTU map of two files is not written on the device)."""
    _need_ref()
    from oracle import ora
    fasta = os.path.join(GOLDEN, "db_bac.fasta")
    d = tempfile.mkdtemp(prefix="smr_mates_ref_")
    try:
        zip_out = name == "zip_out"
        reads = golden_mates(d, gz=zip_out)
        extra = list(OPTION_SETS.get(name, ["-paired_in", "-out2"]))
        denovo = None
        if name != "zip_out":
            denovo = (0.9, 0.9)
            extra += ["-otu_map", "-de_novo_otu", "-id", "0.9", "-coverage", "0.9"]
        if zip_out:
            extra += ["-zip-out", "1"]
        r = ora.run_reference([fasta], reads, os.path.join(d, "ref"), extra=["-sam", "-fastx", "-other"] + extra, threads=1, idx_dir=golden_idx_dir)
        skip = ("aligned.log", "otu_map.txt")
        ref = {fn.replace(".gz", ""): (gzip.open if zip_out else open)(os.path.join(r["out_dir"], fn), "rb").read()
               for fn in os.listdir(r["out_dir"]) if fn not in skip}
        log = ora.parse_log(r["log"])
        ours = _ours(golden, os.path.join(d, "ours"), reads, extra, ref, log, denovo, zip_out)
        assert sorted(ours) == sorted(fn for fn in os.listdir(r["out_dir"]) if fn not in skip)
        ours = {fn.replace(".gz", ""): v for fn, v in ours.items()}
        for fn in ref:
            assert ours[fn] == ref[fn], fn
        assert all(len(ref[fn]) > 1000 for fn in ref if fn.startswith("aligned_") and "denovo" not in fn)
        if name == "out2":
            # a denovo mate's partner that is not denovo goes to _fwd (ReportDenovo::append keeps idx across mates)
            assert len(ref["aligned_denovo_fwd.fq"]) > 2 * len(ref["aligned_denovo_rev.fq"]) > 0
            # three batches write what one batch writes
            t = sum(os.path.getsize(p) for p in reads)
            again = _ours(golden, os.path.join(d, "batches"), reads, extra, ref, log, denovo, False, batch_bytes=t // 3 + 1, piece_bytes=4096)
            assert again == ours
    finally:
        shutil.rmtree(d, ignore_errors=True)
