"""BAM and BGZF written from the SAM/BAM format specification (SAMv1 sections 4.1, 4.2 and 5.3), independent of the library: the
framing of a BGZF stream, a decoder of BAM files and records back to SAM text, and an encoder of the SAM rows this project writes
(11 fields, then AS:i and NM:i) into BAM records.  The BAM tests compare the library's aligned.bam with these."""
import struct
import zlib

BLOCK = 65280                    # input bytes of a full BGZF block
EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
NT16 = "=ACMGRSVTWYHKDBN"
CIGAR_OPS = "MIDNSHP=X"


def reg2bin(beg: int, end: int) -> int:
    end -= 1
    for shift, first in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return first + (beg >> shift)
    return 0


def int_tag(tag: str, v: int) -> bytes:
    """an integer tag of a value >= 0 in the smallest unsigned type, as htslib parses a SAM ':i:' value"""
    for t, fmt, top in (("C", "<B", 0xFF), ("S", "<H", 0xFFFF), ("I", "<I", 0xFFFFFFFF)):
        if v <= top:
            return tag.encode() + t.encode() + struct.pack(fmt, v)
    raise ValueError(v)


def members(data: bytes) -> list:
    """the BGZF members of a stream, each checked against the specification: [(member bytes, inflated bytes)]"""
    out, at = [], 0
    while at < len(data):
        h = data[at:at + 18]
        assert h[:4] == b"\x1f\x8b\x08\x04", ("member header", at)
        assert h[4:8] == b"\0\0\0\0" and h[8] == 0 and h[9] == 0xFF, ("MTIME, XFL, OS", at)
        assert struct.unpack("<H", h[10:12])[0] == 6 and h[12:14] == b"BC" and struct.unpack("<H", h[14:16])[0] == 2, ("BC subfield", at)
        size = struct.unpack("<H", h[16:18])[0] + 1
        m = data[at:at + size]
        assert len(m) == size and size <= 65536, ("BSIZE", at)
        body = zlib.decompress(m, 31)   # each member inflates alone
        isize = struct.unpack("<I", m[-4:])[0]
        assert isize == len(body) <= BLOCK and struct.unpack("<I", m[-8:-4])[0] == zlib.crc32(body), ("trailer", at)
        out.append((m, body))
        at += size
    return out


def check_stream(data: bytes) -> bytes:
    """the framing of one stream that the writer cut into blocks: every block but the last holds exactly BLOCK bytes; returns the
    stream's inflated bytes"""
    ms = members(data)
    assert all(len(b) == BLOCK for _, b in ms[:-1]), [len(b) for _, b in ms]
    assert all(len(b) > 0 for _, b in ms)
    return b"".join(b for _, b in ms)


def decode_file(data: bytes):
    """aligned.bam -> (header text, [(name, length)], [record bytes]); the file must end with the EOF block"""
    assert data.endswith(EOF_BLOCK) and not data[:-len(EOF_BLOCK)].endswith(EOF_BLOCK)
    raw = b"".join(b for _, b in members(data))
    assert raw[:4] == b"BAM\1"
    lt = struct.unpack_from("<i", raw, 4)[0]
    text = raw[8:8 + lt].decode()
    at = 8 + lt
    nref = struct.unpack_from("<i", raw, at)[0]
    at += 4
    refs = []
    for _ in range(nref):
        ln = struct.unpack_from("<i", raw, at)[0]
        name = raw[at + 4:at + 4 + ln]
        assert name.endswith(b"\0")
        refs.append((name[:-1].decode(), struct.unpack_from("<i", raw, at + 4 + ln)[0]))
        at += 8 + ln
    return text, refs, split_records(raw[at:])


def split_records(raw: bytes) -> list:
    out, at = [], 0
    while at < len(raw):
        n = struct.unpack_from("<i", raw, at)[0]
        out.append(raw[at:at + 4 + n])
        at += 4 + n
    assert at == len(raw)
    return out


def decode_record(rec: bytes, names: list) -> str:
    """one BAM record -> the SAM row this project prints for it (without its newline)"""
    (_, ref_id, pos, l_name, mapq, bin_, n_cig, flag, l_seq, next_id, next_pos, tlen) = struct.unpack_from("<iiiBBHHHiiii", rec, 0)
    at = 36
    qname = rec[at:at + l_name - 1].decode()
    assert rec[at + l_name - 1] == 0
    at += l_name
    cig = struct.unpack_from("<%dI" % n_cig, rec, at)
    at += 4 * n_cig
    span = sum(w >> 4 for w in cig if (w & 15) in (0, 2, 3, 7, 8))
    assert bin_ == reg2bin(pos, pos + max(span, 1)) and mapq == 255 and (next_id, next_pos, tlen) == (-1, -1, 0)
    seq_b = rec[at:at + (l_seq + 1) // 2]
    seq = "".join(NT16[(seq_b[i // 2] >> (4 if i % 2 == 0 else 0)) & 15] for i in range(l_seq))
    if l_seq % 2:
        assert seq_b[-1] & 15 == 0
    at += (l_seq + 1) // 2
    q = rec[at:at + l_seq]
    qual = "*" if l_seq == 0 or all(x == 0xFF for x in q) else "".join(chr(x + 33) for x in q)
    at += l_seq
    tags = []
    while at < len(rec):
        tag, t = rec[at:at + 2].decode(), chr(rec[at + 2])
        fmt = {"C": "<B", "S": "<H", "I": "<I", "c": "<b", "s": "<h", "i": "<i"}[t]
        v = struct.unpack_from(fmt, rec, at + 3)[0]
        assert int_tag(tag, v) == rec[at:at + 3 + struct.calcsize(fmt)], "the smallest type"
        tags.append(f"{tag}:i:{v}")
        at += 3 + struct.calcsize(fmt)
    cigar = "".join(f"{w >> 4}{CIGAR_OPS[w & 15]}" for w in cig) or "*"
    return "\t".join([qname, str(flag), names[ref_id], str(pos + 1), str(mapq), cigar, "*", str(next_pos + 1), str(tlen), seq, qual] + tags)


def encode_row(row: str, ref_id: int) -> bytes:
    """one SAM row of this project (11 fields, AS:i, NM:i) -> its BAM record, refID given"""
    f = row.rstrip("\n").split("\t")
    qname, flag, pos, mapq, cigar, seq, qual = f[0], int(f[1]), int(f[3]) - 1, int(f[4]), f[5], f[9], f[10]
    cig, num = [], ""
    for ch in cigar:
        if ch.isdigit():
            num += ch
        else:
            cig.append(int(num) << 4 | CIGAR_OPS.index(ch))
            num = ""
    span = sum(w >> 4 for w in cig if (w & 15) in (0, 2))
    lseq = len(seq)
    packed = bytearray((lseq + 1) // 2)
    for i, c in enumerate(seq):
        packed[i // 2] |= NT16.index(c) << (4 if i % 2 == 0 else 0)
    q = bytes([0xFF] * lseq) if qual == "*" else bytes(ord(c) - 33 for c in qual)
    tags = b"".join(int_tag(t[:2], int(t[5:])) for t in f[11:])
    body = struct.pack("<iiBBHHHiiii", ref_id, pos, len(qname) + 1, mapq, reg2bin(pos, pos + span), len(cig), flag, lseq, -1, -1, 0)
    body += qname.encode() + b"\0" + struct.pack("<%dI" % len(cig), *cig) + bytes(packed) + q + tags
    return struct.pack("<i", len(body)) + body
