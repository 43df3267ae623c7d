"""
Test helper for the unaligned BAM input path: a writer of uBAM files (BGZF members with the BC extra field and the
28-byte EOF block, at chosen member sizes and zlib levels) and a decoder that turns a BAM file into the FASTQ text the
device writes (cutadapt_b200.h, CG_FORMAT_BAM): per record "@" + name + "\n" + the sequence decoded with
"=ACMGRSVTWYHKDBN" + "\n+\n" + every quality byte + 33 + "\n"; CIGAR and aux tags skipped.
"""
import gzip
import struct
import zlib

import numpy as np

NIBBLES = "=ACMGRSVTWYHKDBN"
_CODE = {c: i for i, c in enumerate(NIBBLES)}
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def header(text: bytes = b"@HD\tVN:1.6\tSO:unsorted\n", refs=()) -> bytes:
    """The BAM header: magic, text, references as (name, length)."""
    out = [b"BAM\x01", struct.pack("<i", len(text)), text, struct.pack("<i", len(refs))]
    for name, length in refs:
        out += [struct.pack("<i", len(name) + 1), name + b"\0", struct.pack("<i", length)]
    return b"".join(out)


def record(name: bytes, seq: str, qual=None, flag: int = 4, cigar=(), tags: bytes = b"", block_size=None) -> bytes:
    """One record.  qual: a sequence of Phred values, or None for an absent quality array (0xFF bytes); cigar: packed
    uint32 operations; block_size: override the consistent value."""
    l_seq = len(seq)
    codes = [_CODE.get(c, 15) for c in seq.upper()]
    if l_seq & 1:
        codes.append(0)
    packed = bytes((codes[i] << 4) | codes[i + 1] for i in range(0, len(codes), 2))
    q = bytes([0xFF] * l_seq) if qual is None else bytes(qual)
    body = (struct.pack("<iiBBHHHiiii", -1, -1, len(name) + 1, 255, 4680, len(cigar), flag, l_seq, -1, -1, 0)
            + name + b"\0" + b"".join(struct.pack("<I", c) for c in cigar) + packed + q + tags)
    return struct.pack("<i", len(body) if block_size is None else block_size) + body


def bgzf(plain: bytes, member: int = 65280, level: int = 6, eof: bool = True) -> bytes:
    """plain as BGZF: members of at most `member` plain bytes, each with the BC extra field (its total size - 1)."""
    out = []
    for at in range(0, len(plain), member):
        piece = plain[at:at + member]
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        data = c.compress(piece) + c.flush()
        size = 18 + len(data) + 8
        assert size <= 65536, "a BGZF member holds at most 64 KiB"
        out.append(b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\x00BC\x02\x00" + struct.pack("<H", size - 1) + data
                   + struct.pack("<II", zlib.crc32(piece), len(piece)))
    if eof:
        out.append(BGZF_EOF)
    return b"".join(out)


def bam_file(records, member: int = 65280, level: int = 6, hdr: bytes = None) -> bytes:
    return bgzf((header() if hdr is None else hdr) + b"".join(records), member, level)


def _skip_header(b: bytes) -> int:
    assert b[:4] == b"BAM\x01"
    (l_text,) = struct.unpack_from("<i", b, 4)
    p = 8 + l_text
    (n_ref,) = struct.unpack_from("<i", b, p)
    p += 4
    for _ in range(n_ref):
        (l_name,) = struct.unpack_from("<i", b, p)
        p += 4 + l_name + 4
    return p


def records_of(plain: bytes):
    """(offset, bytes) of every record of a plain BAM stream."""
    p = _skip_header(plain)
    out = []
    while p < len(plain):
        (bs,) = struct.unpack_from("<i", plain, p)
        out.append((p, plain[p:p + 4 + bs]))
        p += 4 + bs
    return out


def fastq_of_record(rec: bytes) -> bytes:
    l_read_name = rec[12]
    n_cigar, flag, l_seq = struct.unpack_from("<HHi", rec, 16)
    name = rec[36:36 + l_read_name - 1]
    s = 36 + l_read_name + 4 * n_cigar
    packed = np.frombuffer(rec, dtype=np.uint8, count=(l_seq + 1) // 2, offset=s)
    nib = np.empty(2 * len(packed), dtype=np.uint8)
    nib[0::2], nib[1::2] = packed >> 4, packed & 15
    seq = np.frombuffer(NIBBLES.encode(), dtype=np.uint8)[nib[:l_seq]].tobytes()
    q = np.frombuffer(rec, dtype=np.uint8, count=l_seq, offset=s + (l_seq + 1) // 2)
    return b"@" + name + b"\n" + seq + b"\n+\n" + (q + 33).astype(np.uint8).tobytes() + b"\n"


def fastq_of(bam: bytes) -> bytes:
    """The FASTQ text of a BAM file (BGZF) or of a plain BAM stream."""
    plain = gzip.decompress(bam) if bam[:2] == b"\x1f\x8b" else bam
    return b"".join(fastq_of_record(r) for _, r in records_of(plain))


def random_records(rng, n, min_len=150, max_len=150, name_len=(8, 30), qual=True):
    """n records of random reads (ACGT with some N), names of printable characters."""
    recs = []
    for i in range(n):
        L = int(rng.integers(min_len, max_len + 1))
        seq = "".join(rng.choice(list("ACGTN"), size=L, p=[0.24, 0.24, 0.24, 0.24, 0.04]))
        nl = int(rng.integers(name_len[0], name_len[1] + 1))
        name = (f"r{i}:" + "x" * nl)[:max(nl, len(str(i)) + 2)].encode()
        q = rng.integers(0, 42, size=L).tolist() if qual else None
        recs.append(record(name, seq, q))
    return recs
