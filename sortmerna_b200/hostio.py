"""Host-side I/O helpers around the alignment hot path (numpy only; no GPU, no oracle).

They restate the small pieces of the reference that sit immediately on either side of the
drop-in boundary so that tests and bench.py can feed the C-ABI the same bytes the reference's
`align()` sees:

  * `encode_nt`      -- `nt_table` (include/common.hpp:68-77): ACGTU -> 0..3, anything else -> 4
  * `load_references`-- `References::load` + `convert_fix` (src/sortmerna/references.cpp:55-164)
  * `read_fastx`     -- single-line-record FASTA/FASTQ reader (the reference's Readfeed is out of scope)
  * `parse_stats`    -- the `.stats` index file (`Refstats::load`, src/sortmerna/refstats.cpp:103-190)
  * `minimal_score`  -- the E-value -> minimal SW score formula (refstats.cpp:236-265) given lambda, K
  * `format_sam_rows`-- the SAM row layout of `ReportSam::append` (src/sortmerna/report_sam.cpp:64-152)
  * `format_blast_rows` / `format_blast_pairwise_rows` -- tabular and pairwise BLAST rows of `ReportBlast::append`
    (src/sortmerna/report_blast.cpp:99-365)
  * `denovo_classes` / `otu_map` -- the denovo_stats pass and the OTU map (processor.cpp:287-438, otumap.cpp:84-281)
  * `summary_log`    -- aligned.log (`Summary::to_string`, src/sortmerna/summary.cpp:102-175)
"""
from __future__ import annotations

import glob
import gzip
import math
import os
import struct
from dataclasses import dataclass, field

import numpy as np

_NT = np.full(256, 4, dtype=np.uint8)
for _c, _v in (("A", 0), ("C", 1), ("G", 2), ("T", 3), ("U", 3)):
    _NT[ord(_c)] = _v
    _NT[ord(_c.lower())] = _v
NT_MAP = "ACGTN"


def encode_nt(seq: bytes | str) -> np.ndarray:
    """ASCII -> 0..4 (4 = ambiguous), include/common.hpp:68-77."""
    if isinstance(seq, str):
        seq = seq.encode()
    return _NT[np.frombuffer(seq, dtype=np.uint8)]


def _open(path: str):
    return gzip.open(path, "rb") if path.endswith(".gz") else open(path, "rb")


def read_fastx(path: str, limit: int | None = None):
    """Return (headers, seqs, quals) of a FASTA/FASTQ file (multi-line FASTA is concatenated)."""
    headers, seqs, quals = [], [], []
    with _open(path) as fh:
        data = fh.read()
    lines = data.split(b"\n")
    i, n = 0, len(lines)
    while i < n:
        ln = lines[i].rstrip(b"\r")
        if not ln:
            i += 1
            continue
        if ln[:1] == b"@":
            headers.append(ln.decode())
            seqs.append(lines[i + 1].rstrip(b"\r"))
            quals.append(lines[i + 3].rstrip(b"\r"))
            i += 4
        elif ln[:1] == b">":
            headers.append(ln.decode())
            i += 1
            parts = []
            while i < n and lines[i][:1] != b">":
                if lines[i].strip():
                    parts.append(lines[i].strip())
                i += 1
            seqs.append(b"".join(parts))
            quals.append(b"")
        else:
            raise ValueError(f"{path}: unexpected line {i}: {ln[:40]!r}")
        if limit is not None and len(seqs) >= limit:
            break
    return headers, seqs, quals


def seq_id(header: str) -> str:
    """Read::getSeqId (read.cpp:365-371): header up to the first space, leading '>'/'@' removed."""
    h = header.split(" ")[0]
    return h.lstrip(">@")


@dataclass
class ReadBatch:
    headers: list
    seqs: list            # raw bytes
    quals: list
    cat: np.ndarray       # uint8, 0..4
    off: np.ndarray       # uint64, nreads+1

    @property
    def n(self):
        return len(self.seqs)


def pack_reads(headers, seqs, quals=None) -> ReadBatch:
    lens = np.fromiter((len(s) for s in seqs), dtype=np.uint64, count=len(seqs))
    off = np.zeros(len(seqs) + 1, dtype=np.uint64)
    np.cumsum(lens, out=off[1:])
    cat = encode_nt(b"".join(seqs)) if seqs else np.zeros(0, np.uint8)
    return ReadBatch(list(headers), list(seqs), list(quals) if quals else [b""] * len(seqs), cat, off)


def load_reads(path: str, limit: int | None = None) -> ReadBatch:
    h, s, q = read_fastx(path, limit)
    return pack_reads(h, s, q)


@dataclass
class References:
    path: str
    ids: list             # BaseRecord::getId -- header up to first space without '>'
    cat: np.ndarray       # uint8 0..4, all sequences concatenated
    off: np.ndarray       # uint64, nref+1

    @property
    def n(self):
        return len(self.ids)


def load_references(path: str) -> References:
    """References::load for a single-part index (references.cpp:55-154)."""
    h, s, _ = read_fastx(path)
    lens = np.fromiter((len(x) for x in s), dtype=np.uint64, count=len(s))
    off = np.zeros(len(s) + 1, dtype=np.uint64)
    np.cumsum(lens, out=off[1:])
    return References(path, [seq_id(x) for x in h], encode_nt(b"".join(s)), off)


def split_by_parts(refs: "References", stats: "IndexStats") -> list:
    """The references of each index part (References::load reads [start_part, start_part + seq_part_size) of the FASTA,
    references.cpp:55-154): `ref_num` of an alignment is relative to its part."""
    out, first = [], 0
    for (_, _, nseq) in stats.parts:
        off = refs.off[first:first + nseq + 1]
        out.append(References(refs.path, refs.ids[first:first + nseq], refs.cat[int(off[0]):int(off[-1])], (off - off[0]).astype(np.uint64)))
        first += nseq
    return out


def _refs_of(refs_by_index, al):
    """refs_by_index[index_num] is a References (single-part index) or the list split_by_parts returns"""
    refs = refs_by_index[int(al["index_num"])]
    return refs[int(al["part"])] if isinstance(refs, (list, tuple)) else refs


@dataclass
class IndexStats:
    """Contents of <prefix>.stats (refstats.cpp:129-190; writer indexdb.cpp:2020-2080)."""
    prefix: str
    fasta_size: int = 0
    fasta_name: str = ""
    background_freq: tuple = (0.25, 0.25, 0.25, 0.25)
    full_ref: int = 0
    lnwin: int = 18
    numseq: int = 0
    num_parts: int = 1
    parts: list = field(default_factory=list)  # (start_part, seq_part_size, numseq_part)


def parse_stats(prefix: str) -> IndexStats:
    with open(prefix + ".stats", "rb") as fh:
        b = fh.read()
    o = 0
    (fsize,) = struct.unpack_from("<Q", b, o); o += 8
    (nlen,) = struct.unpack_from("<I", b, o); o += 4
    name = b[o:o + nlen].split(b"\0")[0].decode(); o += nlen
    freq = struct.unpack_from("<4d", b, o); o += 32
    (full_ref,) = struct.unpack_from("<Q", b, o); o += 8
    (lnwin,) = struct.unpack_from("<I", b, o); o += 4
    (numseq,) = struct.unpack_from("<Q", b, o); o += 8
    (nparts,) = struct.unpack_from("<H", b, o); o += 2
    parts = []
    for _ in range(nparts):
        sp, sz, ns = struct.unpack_from("<QQI", b, o); o += 24  # struct index_parts_stats, 8+8+4(+4 pad)
        parts.append((sp, sz, ns))
    return IndexStats(prefix, fsize, name, freq, full_ref, lnwin, numseq, nparts, parts)


def sam_header(prefixes: list, cmdline: str, sq: bool = False) -> str:
    """The header of aligned.sam (ReportSam::write_header, report_sam.cpp:154-205): @HD, with sq (-SQ) one @SQ line per reference
    sequence of every index in --ref order (read from the sequence table after the part table of <prefix>.stats), and @PG with the
    command line."""
    seqs = []
    for prefix in prefixes:
        with open(prefix + ".stats", "rb") as fh:
            b = fh.read()
        o = 8
        (nlen,) = struct.unpack_from("<I", b, o); o += 4 + nlen + 32 + 8 + 4 + 8
        (nparts,) = struct.unpack_from("<H", b, o); o += 2 + 24 * nparts
        (num_sq,) = struct.unpack_from("<I", b, o); o += 4
        for _ in range(num_sq):
            (lid,) = struct.unpack_from("<I", b, o); o += 4
            sid = b[o:o + lid].decode(); o += lid
            (lseq,) = struct.unpack_from("<I", b, o); o += 4
            seqs.append((sid, lseq))
    return sam_header_of(seqs, cmdline, sq)


def sam_header_of(seqs: list, cmdline: str, sq: bool = False) -> str:
    """sam_header from the (id, length) of every reference sequence of every index in --ref order"""
    out = ["@HD\tVN:1.0\tSO:unsorted\n"]
    if sq:
        out += [f"@SQ\tSN:{sid}\tLN:{lseq}\n" for sid, lseq in seqs]
    out.append(f"@PG\tID:sortmerna\tVN:1.0\tCL:{cmdline}\n")
    return "".join(out)


# the index builder's 2-bit code of a letter (map_nt, indexdb.cpp:83-109): what the background frequencies count
_BUILD_NT = np.zeros(256, np.uint8)
for _c in b"BCDWYbcwy":
    _BUILD_NT[_c] = 1
for _c in b"GKSXgksx":
    _BUILD_NT[_c] = 2
for _c in b"TUtu":
    _BUILD_NT[_c] = 3


def fasta_index_stats(fasta: str, lnwin: int = 18, max_mb: float = 3072.0):
    """What <prefix>.stats of the index of `fasta` holds (build_index STEP 1 and the part split, indexdb.cpp:1188-1271 and
    1381-1431, as smr_build_index writes it), computed from the FASTA alone: (IndexStats with prefix "", [(id, length) of every
    sequence]).  A caller that builds the index on the device (Aligner.build_index_device) takes the minimal score, the E-value
    sizes, the per-part references (split_by_parts) and the -SQ lines of the SAM header from it."""
    with open(fasta, "rb") as fh:
        b = fh.read()
    if not b:
        raise ValueError(f"{fasta}: empty reference file")
    a = np.frombuffer(b, np.uint8)
    pread = lnwin + 1
    starts = np.flatnonzero(a == ord(">"))
    if starts.size == 0 or starts[0] != 0:
        raise ValueError(f"{fasta}: each header of a database FASTA file must begin with '>'")
    ends = np.append(starts[1:], a.size)
    nl = np.flatnonzero(a == ord("\n"))
    seqs, lens, rec = [], [], []
    body = np.zeros(a.size + 1, np.int64)   # body[i]: sequence letters before byte i
    seq_mask = np.zeros(a.size, bool)
    for s0, e0 in zip(starts.tolist(), ends.tolist()):
        k = np.searchsorted(nl, s0)
        h1 = int(nl[k]) if k < nl.size and nl[k] < e0 else e0
        name = b[s0 + 1:h1]
        cut = min((i for i in (name.find(b" "), name.find(b"\t")) if i >= 0), default=len(name))
        seqs.append(name[:cut].decode(errors="replace"))
        rec.append((s0, e0, min(h1 + 1, e0)))
        seq_mask[min(h1 + 1, e0):e0] = True
    seq_mask &= (a != ord("\n")) & (a != ord(" "))
    np.cumsum(seq_mask, out=body[1:])
    lens = [int(body[e0] - body[q0]) for (_, e0, q0) in rec]
    short = [n for n in lens if n < pread]
    if short:
        raise ValueError(f"{fasta}: at least one sequence is shorter than the seed length {pread}")
    freq = np.bincount(_BUILD_NT[a[seq_mask & (a != ord("N"))]], minlength=4).astype(np.float64)
    tot = float(freq.sum())
    parts, first = [], 0
    while first < len(rec):
        size, members, nxt, part_size = 0.0, 0, first, 0
        while nxt < len(rec):
            est = float(lens[nxt] - pread + 1) * 9.5e-6
            if est > max_mb:
                nxt += 1
                continue
            if size + est > max_mb:
                break
            size += est
            part_size = rec[nxt][1] - rec[first][0]
            members += 1
            nxt += 1
        if members == 0:
            if nxt < len(rec):
                raise ValueError(f"{fasta}: every sequence is too large to be indexed with the current memory limit")
            break
        parts.append((rec[first][0], part_size, members))
        first = nxt
    st = IndexStats("", a.size, fasta, tuple(float(f / tot) for f in freq), int(sum(lens)), lnwin, len(rec), len(parts), parts)
    return st, list(zip(seqs, lens))


def find_index_prefixes(idx_dir: str) -> dict:
    """Map reference FASTA basename -> index prefix for every *.stats in idx_dir."""
    out = {}
    for st in glob.glob(os.path.join(idx_dir, "*.stats")):
        s = parse_stats(st[: -len(".stats")])
        out[os.path.basename(s.fasta_name)] = s.prefix
    return out


def minimal_score(stats: IndexStats, lam: float, K: float, all_reads_len: int, all_reads_count: int,
                  evalue: float = 1.0) -> int:
    """refstats.cpp:236-265 (is_score_split = false)."""
    f = stats.background_freq
    entropy = -sum(p * math.log2(p) for p in f)
    full_ref = stats.full_ref
    full_read = all_reads_len
    expect_L = int(math.log(K * full_ref * full_read) / entropy)
    if full_ref > expect_L * stats.numseq:
        full_ref -= expect_L * stats.numseq
    full_read -= expect_L * all_reads_count
    return int(math.log(evalue / (K * full_ref * full_read)) / -lam) & 0xFFFFFFFF


def evalue_params(stats: IndexStats, K: float, all_reads_len: int, all_reads_count: int) -> tuple:
    """the length-corrected (full_ref, full_read) of refstats.cpp:236-257 that the E-value of a BLAST row uses"""
    entropy = -sum(p * math.log2(p) for p in stats.background_freq)
    full_ref, full_read = stats.full_ref, all_reads_len
    expect_L = int(math.log(K * full_ref * full_read) / entropy)
    if full_ref > expect_L * stats.numseq:
        full_ref -= expect_L * stats.numseq
    full_read -= expect_L * all_reads_count
    return full_ref, full_read


def _g3(x: float) -> str:
    """what `ss.precision(3); ss << x` prints (C++ general format, 3 significant digits)"""
    return f"{x:.3g}"


def format_blast_rows(batch: "ReadBatch", refs_by_index: list, results, alns, cigar_pool, slots: int, stats, gumbel: list,
                      ev_params: list) -> list:
    """Tabular BLAST rows with the optional columns 'cigar qcov qstrand' as ReportBlast::append prints them
    (src/sortmerna/report_blast.cpp:99-365).  stats[i] = (n_miss, n_gap, n_match) of alignment i -- from the GPU
    (smr_aln_stats) or from calc_miss_gap_match; gumbel[index] = (lambda, K); ev_params[index] = (full_ref, full_read)."""
    import numpy as _np
    rows = []
    for r in range(batch.n):
        na = int(results["n_align"][r])
        name = seq_id(batch.headers[r])
        rlen = len(batch.seqs[r])
        for a in range(na):
            al = alns[r * slots + a]
            st = stats[r * slots + a]
            idx = int(al["index_num"])
            lam, K = gumbel[idx]
            full_ref, full_read = ev_params[idx]
            score = int(al["score1"])
            bitscore = int(_np.float32(_np.float32(lam * score - math.log(K)) / _np.float32(math.log(2))))   # report_blast.cpp:117-119
            evalue = K * full_ref * full_read * math.exp(-lam * score)                                      # :121-126
            miss, gap, match = int(st["n_miss"]), int(st["n_gap"]), int(st["n_match"])
            pid = match / (miss + gap + match)
            cov = abs(int(al["read_end1"]) - int(al["read_begin1"]) + 1) / int(al["readlen"])
            cig = cigar_pool[int(al["cigar_off"]):int(al["cigar_off"]) + int(al["cigar_len"])]
            cs = (f"{int(al['read_begin1'])}S" if int(al["read_begin1"]) else "") + cigar_string(cig)
            end_mask = rlen - int(al["read_end1"]) - 1
            if end_mask > 0:
                cs += f"{end_mask}S"
            refs = _refs_of(refs_by_index, al)
            rows.append("\t".join([name, refs.ids[int(al["ref_num"])], _g3(pid * 100), str(int(al["read_end1"]) - int(al["read_begin1"]) + 1),
                                   str(miss), str(gap), str(int(al["read_begin1"]) + 1), str(int(al["read_end1"]) + 1),
                                   str(int(al["ref_begin1"]) + 1), str(int(al["ref_end1"]) + 1), _g3(evalue), str(bitscore), cs,
                                   _g3(cov * 100), "+" if bool(al["strand"]) else "-"]))
    return rows


_NT_BYTES = np.frombuffer(NT_MAP.encode(), np.uint8)
PAIRWISE_COLS = 60


def format_blast_pairwise_rows(batch: "ReadBatch", refs_by_index: list, results, alns, cigar_pool, slots: int, gumbel: list,
                               ev_params: list, paired: bool = False) -> list:
    """Pairwise BLAST rows (-blast 0) as ReportBlast::append prints them (src/sortmerna/report_blast.cpp:136-251), one string per
    stored alignment in the order of aligned.blast: (index, part) group, then read, then alignment slot.  Reads are skipped as the
    report writer skips empty reads (paired: a pair whose second mate is empty).  gumbel / ev_params as for format_blast_rows.
    A row is its header lines, then the CIGAR's columns cut into blocks of 60; the reference's three passes per block with their
    carry-over (left, e) come down to that plain chunking."""
    keyed = []
    for r in range(batch.n):
        if len(batch.seqs[(r | 1) if paired else r]) == 0:
            continue
        enc = batch.cat[int(batch.off[r]):int(batch.off[r + 1])]
        for a in range(int(results["n_align"][r])):
            al = alns[r * slots + a]
            keyed.append(((int(al["index_num"]), int(al["part"])), _pairwise_row(batch.headers[r], enc, al, _refs_of(refs_by_index, al),
                                                                                  cigar_pool, gumbel, ev_params)))
    keyed.sort(key=lambda x: x[0])   # stable: read, then slot within a group
    return [row for _, row in keyed]


def _pairwise_row(header, enc, al, refs, cigar_pool, gumbel, ev_params) -> str:
    idx, score, strand = int(al["index_num"]), int(al["score1"]), bool(al["strand"])
    lam, K = gumbel[idx]
    full_ref, full_read = ev_params[idx]
    bits = max(0, int(np.float32(np.float32(lam * score - math.log(K)) / np.float32(math.log(2)))))   # report_blast.cpp:117-119
    evalue = K * full_ref * full_read * math.exp(-lam * score)                                       # :121-126
    ref_num = int(al["ref_num"])
    ref = refs.cat[int(refs.off[ref_num]):int(refs.off[ref_num + 1])]
    read = enc if strand else np.where(enc < 4, 3 - enc, 4)[::-1]
    out = [f"Sequence ID: {refs.ids[ref_num]}\nQuery ID: {seq_id(header)}\n"
           f"Score: {score} bits ({bits})\tExpect: {_g3(evalue)}\tstrand: {'+' if strand else '-'}\n\n"]
    # every column: reference char, middle char, read char, and whether it consumes the reference / the read
    top, mid, bot, dq, dp = [], [], [], [], []
    q, p = int(al["ref_begin1"]), int(al["read_begin1"])
    for c in cigar_pool[int(al["cigar_off"]):int(al["cigar_off"]) + int(al["cigar_len"])]:
        op, n = int(c) & 0xF, int(c) >> 4
        eq, ep = (q + n if op != 1 else q), (p + n if op <= 1 else p)
        if q < 0 or p < 0 or eq > ref.size or ep > read.size:
            raise ValueError(f"CIGAR runs past the read or the reference of {seq_id(header)}")
        t = _NT_BYTES[ref[q:eq]] if op != 1 else np.full(n, ord("-"), np.uint8)
        b = _NT_BYTES[read[p:ep]] if op <= 1 else np.full(n, ord("-"), np.uint8)
        top.append(t)
        bot.append(b)
        mid.append(np.where(t == b, ord("|"), ord("*")).astype(np.uint8) if op == 0 else np.full(n, ord(" "), np.uint8))
        dq.append(np.full(n, op != 1, np.int64))
        dp.append(np.full(n, op <= 1, np.int64))
        q, p = eq, ep
    if top:
        top, mid, bot = (np.concatenate(x).tobytes().decode() for x in (top, mid, bot))
        cq, cp = np.cumsum(np.concatenate(dq)), np.cumsum(np.concatenate(dp))
        q, p = int(al["ref_begin1"]), int(al["read_begin1"])
        for b in range(0, len(top), PAIRWISE_COLS):
            e = min(b + PAIRWISE_COLS, len(top))
            q1, p1 = int(al["ref_begin1"]) + int(cq[e - 1]), int(al["read_begin1"]) + int(cp[e - 1])
            out.append(f"Target: {q + 1:>8}    {top[b:e]}    {q1}\n{' ' * 20}{mid[b:e]}\nQuery: {p + 1:>9}    {bot[b:e]}    {p1}\n\n")
            q, p = q1, p1
    return "".join(out)


def host_aln_stats(batch: "ReadBatch", refs_by_index: list, results, alns, cigar_pool, slots: int):
    """calc_miss_gap_match on the host (numpy) for every stored alignment: the CPU twin of smr_aln_stats, used by the tests."""
    out = np.zeros(batch.n * slots, dtype=[("n_miss", "<u4"), ("n_gap", "<u4"), ("n_match", "<u4"), ("n_match_denovo", "<u4")])
    for r in range(batch.n):
        enc = batch.cat[int(batch.off[r]):int(batch.off[r + 1])]
        for a in range(int(results["n_align"][r])):
            al = alns[r * slots + a]
            refs = _refs_of(refs_by_index, al)
            e04 = enc if bool(al["strand"]) else np.where(enc < 4, 3 - enc, 4)[::-1]
            rseq = refs.cat[int(refs.off[int(al["ref_num"])]):int(refs.off[int(al["ref_num"]) + 1])]
            cig = cigar_pool[int(al["cigar_off"]):int(al["cigar_off"]) + int(al["cigar_len"])]
            m = calc_miss_gap_match(rseq, e04, al, cig)
            # denovo_stats_run (processor.cpp:329-357) walks the same CIGAR over the read WITHOUT reverse-complementing it
            md = m if bool(al["strand"]) else calc_miss_gap_match(rseq, enc, al, cig)
            out[r * slots + a] = (m[0], m[1], m[2], md[2])
    return out


def _pair_skipped(paired: bool, seq_lens, r: int) -> bool:
    """denovo_stats_run (processor.cpp:323-327): a pair whose second read is empty is skipped, both mates; so is a last read
    without its mate"""
    return paired and ((r | 1) >= len(seq_lens) or seq_lens[r | 1] == 0)


def denovo_classes(results, alns, slots: int, stats, min_id: float, min_cov: float, paired: bool = False, seq_lens=None):
    """denovo_stats_run (processor.cpp:329-357) from smr_aln_stats: per read the four counters
    (c_yid_ycov, n_yid_ncov, n_nid_ycov, n_denovo) over its stored alignments; their column sums are Readstats'
    n_yid_ycov / n_yid_ncov / n_nid_ycov / num_denovo.  Returns an (nreads, 4) uint32 array.
    paired: records 2k and 2k+1 are mates, and seq_lens[r] is the length of read r: a pair whose second read is empty counts for
    neither mate."""
    n = results.shape[0]
    out = np.zeros((n, 4), np.uint32)
    for r in range(n):
        if _pair_skipped(paired, seq_lens, r):
            continue
        for a in range(int(results["n_align"][r])):
            al, st = alns[r * slots + a], stats[r * slots + a]
            tot = int(st["n_miss"]) + int(st["n_gap"]) + int(st["n_match"])
            idv = int(st["n_match_denovo"]) / tot
            cov = abs(int(al["read_end1"]) - int(al["read_begin1"]) + 1) / int(al["readlen"])
            is_id = math.floor(idv * 1000.0 + 0.5) / 1000.0 >= min_id      # :336-339 round to 3 decimals
            is_cov = math.floor(cov * 1000.0 + 0.5) / 1000.0 >= min_cov
            out[r, 0 if (is_id and is_cov) else 1 if is_id else 2 if is_cov else 3] += 1
    return out


def _round3(x: float) -> float:
    """denovo_stats_run's rounding to 3 decimals (processor.cpp:334-335)"""
    return math.floor(x * 1000.0 + 0.5) / 1000.0


def _round3_otu(x: float) -> float:
    """fill_otu_map2's rounding (otumap.cpp:160-161): scaled back with * 0.001, one ulp above / 1000.0 for 144 of the k in 0..1000"""
    return math.floor(x * 1000.0 + 0.5) * 0.001


def otu_map(refs_by_index, headers, results, alns, slots: int, stats, min_id: float, min_cov: float, feed=None, seq_lens=None) -> dict:
    """fill_otu_map / fill_otu_map2 / OtuMap::write (otumap.cpp:84-281) at -threads 1: the bytes of otu_map.txt, the number of its
    lines (Total OTUs) and of its entries (for single-end reads the n_yid_ycov of aligned.log).  A read is looked at when one of its
    alignments passes -id and -coverage under denovo_stats_run's rounding (its c_yid_ycov > 0); each of its alignments that passes
    them under fill_otu_map2's rounding appends the read's QNAME to the line of its reference id.  (index, part) groups are walked in
    order, reads in order, alignments in slot order; lines come out in unsigned byte order of the id.
    feed: None (single-end), "one_file" (one interleaved paired file: every record) or "two_files" (two mate files interleaved as
    records 2k, 2k+1: the OTU pass reads the first file alone, readfeed slot 0).  In both paired feeds a pair whose second read is
    empty (seq_lens[2k+1] == 0) was skipped by denovo_stats_run, so its c_yid_ycov stays 0."""
    n = results.shape[0]
    per_read = []
    for r in range(n):
        rows = []
        if _pair_skipped(feed is not None, seq_lens, r) or (feed == "two_files" and r & 1):
            per_read.append(rows)
            continue
        for a in range(int(results["n_align"][r])):
            al, st = alns[r * slots + a], stats[r * slots + a]
            tot = int(st["n_miss"]) + int(st["n_gap"]) + int(st["n_match"])
            idv = int(st["n_match_denovo"]) / tot
            cov = abs(int(al["read_end1"]) - int(al["read_begin1"]) + 1) / int(al["readlen"])
            rows.append((al, idv, cov))
        counts = any(_round3(i) >= min_id and _round3(c) >= min_cov for _, i, c in rows)
        per_read.append(rows if counts else [])
    groups = sorted({(int(al["index_num"]), int(al["part"])) for rows in per_read for al, _, _ in rows})
    lines = {}
    for g in groups:
        for r, rows in enumerate(per_read):
            for al, idv, cov in rows:
                if (int(al["index_num"]), int(al["part"])) != g or not (_round3_otu(idv) >= min_id and _round3_otu(cov) >= min_cov):
                    continue
                ref = _refs_of(refs_by_index, al).ids[int(al["ref_num"])].encode()
                lines.setdefault(ref, []).append(seq_id(headers[r]).encode())
    text = b"".join(k + b"\t" + b"\t".join(v) + b"\n" for k, v in sorted(lines.items()))
    return dict(text=text, total_otu=len(lines), n_yid_ycov=sum(len(v) for v in lines.values()))


def _pct(part: int, whole: int) -> str:
    """(float)part / whole * 100 in float32, as Summary::to_string computes it, printed with std::fixed precision 2"""
    r = np.float32(np.float32(part) / np.float32(whole))
    return f"{float(np.float32(r * np.float32(100))):.2f}"


def summary_log(cmd: str, refs: list, reads: list, total_reads: int, num_aligned: int, min_len: int, max_len: int, all_reads_len: int,
                reads_matched_per_db: list, gumbel: list, minimal_score: list, lnwin=18, skiplengths=None, params=None, threads: int = 1,
                sq: bool = False, pid: str = "", denovo=None, otu=None, timestamp: str | None = None) -> str:
    """aligned.log as Summary::to_string writes it (src/sortmerna/summary.cpp:102-175), byte for byte.
    cmd: the command line (Runopts::cmdline); refs / reads: the -ref and -reads paths as given; total_reads / all_reads_len /
    min_len / max_len: the read-count pass (Aligner.read_counts); num_aligned / reads_matched_per_db: the alignment counters summed
    over the batches; gumbel[i] = (lambda, K) and minimal_score[i] of index i; lnwin: the seed length, one for all or one per index;
    skiplengths[i]: the three pass lengths (None: Refstats' defaults lnwin, lnwin / 2, 3); params: an api.Params (or anything with
    its attribute names) for the seed and SW lines, None for the reference's defaults; pid: the "Process pid" text (the reference
    leaves it empty); denovo: with -de_novo_otu, the num_denovo total of the denovo_stats pass; otu: with -otu_map, (its n_yid_ycov
    total, the lines of otu_map.txt); timestamp: ctime's text without its newline (None: now).
    The ratios are float32, as the reference computes them; from the results block on the stream is std::fixed, precision 2."""
    import time
    lnw = list(lnwin) if isinstance(lnwin, (list, tuple)) else [lnwin] * len(refs)
    p = {k: getattr(params, k) for k in ("num_seeds", "edges", "match", "mismatch", "gap_open", "gap_ext", "score_N")} if params is not None else \
        dict(num_seeds=2, edges=4, match=2, mismatch=-3, gap_open=5, gap_ext=2, score_N=-3)
    o = [f" Command:\n    {cmd}\n\n", f" Process pid = {pid}\n\n", " Parameters summary: \n"]
    for i, ref in enumerate(refs):
        sk = skiplengths[i] if skiplengths is not None else (lnw[i], lnw[i] // 2, 3)
        o.append(f"    Reference file: {ref}\n        Seed length = {lnw[0]}\n        Pass 1 = {sk[0]}, Pass 2 = {sk[1]}, Pass 3 = {sk[2]}\n"
                 f"        Gumbel lambda = {gumbel[i][0]:g}\n        Gumbel K = {gumbel[i][1]:g}\n"
                 f"        Minimal SW score based on E-value = {minimal_score[i]}\n")
    o.append(f"    Number of seeds = {p['num_seeds']}\n    Edges = {p['edges']}\n    SW match = {p['match']}\n    SW mismatch = {p['mismatch']}\n"
             f"    SW gap open penalty = {p['gap_open']}\n    SW gap extend penalty = {p['gap_ext']}\n    SW ambiguous nucleotide = {p['score_N']}\n"
             f"    SQ tags are {'' if sq else 'not '}output\n    Number of alignment processing threads = {threads}\n")
    o += [f"    Reads file: {r}\n" for r in reads]
    o.append(f"    Total reads = {total_reads}\n\n Results:\n")
    if denovo is not None:
        o.append(f"    Total reads for de novo clustering = {denovo}\n")
    r = np.float32(np.float32(num_aligned) / np.float32(total_reads))
    o.append(f"    Total reads passing E-value threshold = {num_aligned} ({_pct(num_aligned, total_reads)})\n"
             f"    Total reads failing E-value threshold = {total_reads - num_aligned} ({float(np.float32((np.float32(1) - r) * np.float32(100))):.2f})\n")
    if otu is not None:
        o.append(f"    Total reads passing %%id and %%coverage thresholds = {otu[0]} ({_pct(otu[0], total_reads)})\n    Total OTUs = {otu[1]}\n")
    o.append(f"    Minimum read length = {min_len}\n    Maximum read length = {max_len}\n    Mean read length    = {all_reads_len // total_reads}\n\n"
             " Coverage by database:\n")
    o += [f"    {ref}\t\t{_pct(m, total_reads)}\n" for ref, m in zip(refs, reads_matched_per_db)]
    o.append(f"\n {time.ctime() if timestamp is None else timestamp}\n\n")
    return "".join(o)


def is_denovo_read(classes: np.ndarray) -> np.ndarray:
    """output.cpp:130-141 (single-end): the read goes to aligned_denovo.* when n_denovo > 0 and the other three are 0"""
    return (classes[:, 3] > 0) & (classes[:, 0] == 0) & (classes[:, 1] == 0) & (classes[:, 2] == 0)


_OPS = "MID"


def cigar_string(cig) -> str:
    return "".join(f"{int(c) >> 4}{_OPS[int(c) & 0xF] if (int(c) & 0xF) < 3 else 'D'}" for c in cig)


def revcomp_str(s: str) -> str:
    return s.translate(str.maketrans("ACGTN", "TGCAN"))[::-1]


def calc_miss_gap_match(ref: np.ndarray, read04: np.ndarray, aln, cigar) -> tuple:
    """Read::calc_miss_gap_match (read.cpp:547-589): (mismatches, gaps, matches)."""
    qb, pb = int(aln["ref_begin1"]), int(aln["read_begin1"])
    miss = gap = match = 0
    for c in cigar:
        op, ln = int(c) & 0xF, int(c) >> 4
        if op == 0:
            a = ref[qb:qb + ln]
            b = read04[pb:pb + ln]
            eq = int(np.count_nonzero(a == b))
            match += eq
            miss += ln - eq
            qb += ln
            pb += ln
        elif op == 1:
            pb += ln
            gap += ln
        else:
            qb += ln
            gap += ln
    return miss, gap, match


def format_sam_rows(batch: ReadBatch, refs_by_index: list, results, alns, cigar_pool, slots: int,
                    with_seq: bool = True) -> list:
    """SAM alignment rows as `ReportSam::append` prints them (report_sam.cpp:64-152), one list entry
    per stored alignment, in read order.  `results`/`alns` are the structured numpy arrays returned
    by the C-ABI (or the oracle); refs_by_index[index_num] is a `References`."""
    rows = []
    for r in range(batch.n):
        na = int(results["n_align"][r])
        if na == 0:
            continue
        seq = batch.seqs[r].decode().upper()
        enc = batch.cat[int(batch.off[r]):int(batch.off[r + 1])]
        name = seq_id(batch.headers[r])
        for a in range(na):
            al = alns[r * slots + a]
            refs = _refs_of(refs_by_index, al)
            cig = cigar_pool[int(al["cigar_off"]):int(al["cigar_off"]) + int(al["cigar_len"])]
            strand = bool(al["strand"])
            cs = ""
            if int(al["read_begin1"]) != 0:
                cs += f"{int(al['read_begin1'])}S"
            cs += cigar_string(cig)
            end_mask = len(seq) - int(al["read_end1"]) - 1
            if end_mask > 0:
                cs += f"{end_mask}S"
            # the read as aligned (04 alphabet, reverse-complemented for the minus strand)
            s04 = "".join(NT_MAP[v] for v in enc)
            e04 = enc
            if not strand:
                s04 = revcomp_str(s04)
                e04 = np.where(enc < 4, 3 - enc, 4)[::-1]
            rseq = refs.cat[int(refs.off[int(al["ref_num"])]):int(refs.off[int(al["ref_num"]) + 1])]
            miss, gap, _ = calc_miss_gap_match(rseq, e04, al, cig)
            q = batch.quals[r].decode() if batch.quals[r] else "*"
            if batch.quals[r] and not strand:
                q = q[::-1]
            row = [name, "16" if not strand else "0", refs.ids[int(al["ref_num"])], str(int(al["ref_begin1"]) + 1),
                   "255", cs, "*", "0", "0", s04 if with_seq else "*", q if with_seq else "*",
                   f"AS:i:{int(al['score1'])}", f"NM:i:{miss + gap}"]
            rows.append("\t".join(row))
    return rows
