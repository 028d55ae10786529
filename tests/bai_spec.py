"""The BAI index written from the SAM/BAM specification (SAMv1 sections 5.1-5.3) and the sorted aligned.bam's rules, independent of
the library: the coordinate key, the virtual offsets of the records of a BGZF file, a BAI writer, a BAI parser and the region query
a reader runs through bins, chunks and the linear index.  The sorted-BAM tests compare the library's aligned.bam.bai with these."""
import bisect
import struct

from bam_spec import members

PSEUDO_BIN = 37450
LINEAR_SHIFT = 14   # 16 kb windows


def sort_key(ref_id: int, pos: int, flag: int) -> int:
    """samtools' coordinate key: refID, then pos + 1, then the reverse strand"""
    return (ref_id & 0xFFFFFFFF) << 32 | ((pos + 1) & 0xFFFFFFFF) << 1 | (1 if flag & 16 else 0)


def reg2bins(beg: int, end: int) -> list:
    """every bin that may hold a record overlapping [beg, end) (SAMv1 5.3)"""
    end -= 1
    out = [0]
    for shift, first in ((26, 1), (23, 9), (20, 73), (17, 585), (14, 4681)):
        out += range(first + (beg >> shift), first + (end >> shift) + 1)
    return out


def ref_span(rec: bytes) -> int:
    """reference bases of a BAM record's CIGAR (M, D, N, =, X), at least 1"""
    l_name, n_cig = rec[12], struct.unpack_from("<H", rec, 16)[0]
    cig = struct.unpack_from("<%dI" % n_cig, rec, 36 + l_name)
    return max(1, sum(w >> 4 for w in cig if (w & 15) in (0, 2, 3, 7, 8)))


def file_records(data: bytes) -> list:
    """the records of a BAM file with their virtual offsets: [(record bytes, vbeg, vend)].  A record that ends where its block ends
    has vend = the next block's offset << 16 (htslib's convention)."""
    starts, coff, raw, at = [], [], bytearray(), 0   # per block (the EOF block too): its uncompressed and its compressed offset
    for m, body in members(data):
        starts.append(len(raw))
        coff.append(at)
        raw += body
        at += len(m)

    def voff(x):   # the last block starting at or before x: the one holding x, or the one starting at x
        k = bisect.bisect_right(starts, x) - 1
        return coff[k] << 16 | (x - starts[k])

    lt = struct.unpack_from("<i", raw, 4)[0]
    p = 8 + lt
    nref = struct.unpack_from("<i", raw, p)[0]
    p += 4
    for _ in range(nref):
        p += 8 + struct.unpack_from("<i", raw, p)[0]
    out = []
    while p < len(raw):
        n = struct.unpack_from("<i", raw, p)[0] + 4
        out.append((bytes(raw[p:p + n]), voff(p), voff(p + n)))
        p += n
    return out


def fields(rec: bytes):
    """(refID, pos, end, bin, flag) of a BAM record"""
    ref, pos = struct.unpack_from("<ii", rec, 4)
    bin_, flag = struct.unpack_from("<H", rec, 14)[0], struct.unpack_from("<H", rec, 18)[0]
    return ref, pos, pos + ref_span(rec), bin_, flag


def write_bai(n_ref: int, recs: list) -> bytes:
    """recs = [(refID, pos, end, bin, vbeg, vend)] in file order (sorted by coordinate) -> the BAI bytes: per reference its bins in
    ascending order with their chunks (maximal runs of consecutive records of one (refID, bin), merged with the chunk before when it
    ends in the block the next one starts in), the pseudo-bin 37450, the linear index of 16 kb windows; n_no_coor = 0"""
    per = [[] for _ in range(n_ref)]
    for r in recs:
        per[r[0]].append(r)
    out = bytearray(b"BAI\1" + struct.pack("<i", n_ref))
    for rs in per:
        pieces, prev = [], None   # [bin, vbeg, vend]: maximal runs of consecutive records of one bin
        for ref, pos, end, b, vb, ve in rs:
            if b == prev:
                pieces[-1][2] = ve
            else:
                pieces.append([b, vb, ve])
            prev = b
        bins = {}
        for b, vb, ve in pieces:
            ch = bins.setdefault(b, [])
            if ch and ch[-1][1] >> 16 == vb >> 16:
                ch[-1][1] = ve
            else:
                ch.append([vb, ve])
        out += struct.pack("<i", len(bins) + (1 if rs else 0))
        for b in sorted(bins):
            out += struct.pack("<Ii", b, len(bins[b]))
            for vb, ve in bins[b]:
                out += struct.pack("<QQ", vb, ve)
        if rs:
            out += struct.pack("<Ii", PSEUDO_BIN, 2) + struct.pack("<QQQQ", rs[0][4], rs[-1][5], len(rs), 0)
        lin = {}
        for ref, pos, end, b, vb, ve in rs:
            for w in range(pos >> LINEAR_SHIFT, ((end - 1) >> LINEAR_SHIFT) + 1):
                lin[w] = min(lin.get(w, vb), vb)
        n_intv = max(lin) + 1 if lin else 0
        out += struct.pack("<i", n_intv)
        cur = lin[min(lin)] if lin else 0
        for w in range(n_intv):
            cur = lin.get(w, cur)
            out += struct.pack("<Q", cur)
    out += struct.pack("<Q", 0)
    return bytes(out)


def parse_bai(data: bytes) -> list:
    """BAI bytes -> per reference {"bins": {bin: [(vbeg, vend)]}, "intv": [ioffset]}"""
    assert data[:4] == b"BAI\1"
    n_ref = struct.unpack_from("<i", data, 4)[0]
    at, refs = 8, []
    for _ in range(n_ref):
        n_bin = struct.unpack_from("<i", data, at)[0]
        at += 4
        bins = {}
        for _ in range(n_bin):
            b, n = struct.unpack_from("<Ii", data, at)
            at += 8
            bins[b] = [struct.unpack_from("<QQ", data, at + 16 * k) for k in range(n)]
            at += 16 * n
        n_intv = struct.unpack_from("<i", data, at)[0]
        at += 4
        refs.append(dict(bins=bins, intv=list(struct.unpack_from("<%dQ" % n_intv, data, at))))
        at += 8 * n_intv
    assert struct.unpack_from("<Q", data, at)[0] == 0 and at + 8 == len(data)
    return refs


def query(bai: list, recs: list, ref: int, beg: int, end: int) -> list:
    """the records a reader reaches through the index for the region [beg, end) of reference ref and that overlap it: recs =
    [(refID, pos, end, bin, vbeg, vend)] in file order; returns their indexes in recs, ascending"""
    ix = bai[ref]
    intv = ix["intv"]
    min_off = 0 if not intv else intv[min(beg >> LINEAR_SHIFT, len(intv) - 1)]
    vbegs = [r[4] for r in recs]
    hit = set()
    for b in reg2bins(beg, end):
        for cb, ce in ix["bins"].get(b, []):
            if ce <= min_off:
                continue
            for i in range(bisect.bisect_left(vbegs, cb), bisect.bisect_left(vbegs, ce)):
                r = recs[i]
                if r[0] == ref and r[1] < end and r[2] > beg:
                    hit.add(i)
    return sorted(hit)


def brute(recs: list, ref: int, beg: int, end: int) -> list:
    return [i for i, r in enumerate(recs) if r[0] == ref and r[1] < end and r[2] > beg]
