"""
The BAM input path without a GPU: the host build of cg_bam_core.cuh (tests/hostsim, hs_bam_*) -- the header at every
truncation point, each refusal, the tile walk and its resolve at tile sizes from 64 B to 64 KiB on records that hide
valid-looking record starts behind tile seams, the FASTQ text against tests/bam_oracle.py -- and the input detection of
tools/trim_fastq.py.
"""
import ctypes as C
import gzip
import os
import struct
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import bam_oracle as B  # noqa: E402

BAM_OK, BAM_SHORT, BAM_BAD = 0, 1, 2
R_FLAG, R_NAME, R_NOQUAL, R_QUAL = 1, 2, 3, 4
H_MAGIC, H_NEGATIVE = 1, 2
I64P = C.POINTER(C.c_int64)


def _lib():
    from util import hostsim_lib

    lib = hostsim_lib()
    lib.hs_bam_tile.restype = C.c_int64
    lib.hs_bam_header.argtypes = [C.c_void_p, C.c_int64, I64P, C.POINTER(C.c_int)]
    lib.hs_bam_header.restype = C.c_int
    lib.hs_bam_starts.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, I64P, C.POINTER(C.c_int), I64P]
    lib.hs_bam_starts.restype = C.c_int64
    lib.hs_bam_fastq.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, I64P]
    lib.hs_bam_fastq.restype = C.c_int64
    return lib


def _buf(b: bytes):
    return np.frombuffer(b + bytes(64), dtype=np.uint8)


def hs_header(b: bytes):
    a, n, why = _buf(b), C.c_int64(), C.c_int()
    st = _lib().hs_bam_header(a.ctypes.data, len(b), C.byref(n), C.byref(why))
    return st, n.value, why.value


def hs_starts(recs: bytes, tile: int):
    """(starts, end, end status, tiles walked again) of the records recs (no header)."""
    a = _buf(recs)
    out = np.zeros(len(recs) // 36 + 2, dtype=np.int64)
    end, st, rew = C.c_int64(), C.c_int(), C.c_int64()
    k = _lib().hs_bam_starts(a.ctypes.data, len(recs), tile, out.ctypes.data, C.byref(end), C.byref(st), C.byref(rew))
    return out[:k].tolist(), end.value, st.value, rew.value


def hs_fastq(recs: bytes, starts):
    a = _buf(recs)
    s = np.array(starts, dtype=np.int64)
    out = np.zeros(2 * len(recs) + 64, dtype=np.uint8)
    err = C.c_int64()
    n = _lib().hs_bam_fastq(a.ctypes.data, s.ctypes.data, len(starts), out.ctypes.data, C.byref(err))
    return out[:n].tobytes(), err.value


def serial_starts(recs: bytes):
    p, out = 0, []
    while p < len(recs):
        out.append(p)
        (bs,) = struct.unpack_from("<i", recs, p)
        p += 4 + bs
    return out


def test_tile_constant():
    t = _lib().hs_bam_tile()
    assert t >= 64 and t % 32 == 0


def test_header_every_truncation():
    h = B.header(b"@HD\tVN:1.6\n@CO\tx\n", refs=[(b"chr1", 1000), (b"chrM", 16569)])
    for cut in range(len(h)):
        st, _, _ = hs_header(h[:cut])
        assert st == BAM_SHORT, cut
    assert hs_header(h) == (BAM_OK, len(h), 0)
    assert hs_header(h + b"rest") == (BAM_OK, len(h), 0)
    assert hs_header(B.header(b"")) == (BAM_OK, 12, 0)


def test_header_refused():
    assert hs_header(b"BAM\x02" + bytes(8))[::2] == (BAM_BAD, H_MAGIC)
    assert hs_header(b"BAX")[::2] == (BAM_BAD, H_MAGIC)
    assert hs_header(b"@r\nACGT\n")[::2] == (BAM_BAD, H_MAGIC)
    assert hs_header(b"BAM\x01" + struct.pack("<ii", -1, 0))[::2] == (BAM_BAD, H_NEGATIVE)
    assert hs_header(b"BAM\x01" + struct.pack("<ii", 0, -2))[::2] == (BAM_BAD, H_NEGATIVE)
    assert hs_header(b"BAM\x01" + struct.pack("<iii", 0, 1, 0) + bytes(4))[::2] == (BAM_BAD, H_NEGATIVE)


def _one(rec: bytes):
    starts, end, st, _ = hs_starts(rec, 64)
    return starts, end, st


@pytest.mark.parametrize("rec,code", [
    (B.record(b"r", "ACGT", [30] * 4, flag=0), R_FLAG),
    (B.record(b"r", "ACGT", [30] * 4, flag=4 | 256), R_FLAG),
    (B.record(b"a b", "ACGT", [30] * 4), R_NAME),
    (B.record(b"a\nb", "ACGT", [30] * 4), R_NAME),
    (B.record(b"\xc3\xa9", "ACGT", [30] * 4), R_NAME),
    (B.record(b"r", "ACGT", None), R_NOQUAL),
    (B.record(b"r", "ACGT", [30, 94, 30, 30]), R_QUAL),
    (B.record(b"r", "ACGT", [30, 30, 30, 254]), R_QUAL),
])
def test_refusals(rec, code):
    starts, end, st = _one(rec)
    assert (starts, end, st) == ([0], len(rec), BAM_OK)
    good = B.record(b"ok", "AC", [1, 2])
    _, err = hs_fastq(good + rec, [0, len(good)])
    assert err == (1 << 3) | code


def test_no_refusal_edges():
    recs = [B.record(b"!~", "", []), B.record(b"q", "N", [93]), B.record(b"x" * 254, "ACGTN=RY", [0] * 8)]
    data = b"".join(recs)
    starts, end, st, _ = hs_starts(data, 64)
    assert (starts, end, st) == (serial_starts(data), len(data), BAM_OK)
    text, err = hs_fastq(data, starts)
    assert err == -1 and text == b"".join(B.fastq_of_record(r) for r in recs)


@pytest.mark.parametrize("rec", [
    B.record(b"r", "ACGT", [30] * 4, block_size=31),           # shorter than the fixed part
    B.record(b"r", "ACGT", [30] * 4, block_size=-5),
    B.record(b"r", "ACGT", [30] * 4, block_size=32 + 2 + 2 + 3),  # does not hold its sequence and qualities
    B.record(b"r", "ACGT", [30] * 4)[:12] + b"\x00" + B.record(b"r", "ACGT", [30] * 4)[13:],   # l_read_name 0
    B.record(b"r", "ACGT", [30] * 4)[:20] + struct.pack("<i", -1) + B.record(b"r", "ACGT", [30] * 4)[24:],  # l_seq < 0
    B.record(b"r", "ACGT", [30] * 4)[:37] + b"X" + B.record(b"r", "ACGT", [30] * 4)[38:],   # the name lacks its NUL
])
def test_structurally_invalid(rec):
    good = B.record(b"ok", "AC", [1, 2])
    starts, end, st, _ = hs_starts(good + rec + good, 64)
    assert (starts, end, st) == ([0], len(good), BAM_BAD)


def test_short_at_end():
    recs = b"".join(B.record(b"r%d" % i, "ACGT" * 10, [20] * 40) for i in range(5))
    whole = serial_starts(recs)
    nexts = whole[1:] + [len(recs)]
    for cut in range(len(recs) + 1):
        starts, end, st, _ = hs_starts(recs[:cut], 64)
        done = [s for s, nx in zip(whole, nexts) if nx <= cut]
        want_end = max([nx for nx in nexts if nx <= cut], default=0)
        assert (starts, end, st) == (done, want_end, BAM_OK if want_end == cut else BAM_SHORT), cut


def _packed_seq(packed: bytes) -> str:
    return "".join(B.NIBBLES[b >> 4] + B.NIBBLES[b & 15] for b in packed)


def planted(tile: int, n: int, rng, name_len=(4, 40)):
    """Records that hide valid-looking records: a chain of two in the 4-bit sequence, and one in the aux tags that
    starts exactly at a tile seam, two bytes in front of the next true record.  That one's block_size reaches 12 bytes
    into the true record, where the bytes read as a record too long for the buffer: the tile's walk starts at it, jumps
    over the true entry and stops, so the true entry is walked again."""
    fakes = B.record(b"fake", "ACGT", [30] * 4) + B.record(b"fake2", "ACGTACGT", [20] * 8)
    fake = B.record(b"f", "", [], block_size=48)
    out, p = [], 0
    for i in range(n):
        name = (b"r%d_" % i) + b"x" * int(rng.integers(*name_len))
        pre = rng.integers(0, 256, size=int(rng.integers(0, 40)), dtype=np.uint8).tobytes()
        seq = _packed_seq(pre + fakes)
        q = rng.integers(0, 94, size=len(seq)).tolist()
        tags_at = p + len(B.record(name, seq, q))
        pad = rng.integers(0, 256, size=(-tags_at) % tile, dtype=np.uint8).tobytes()
        r = B.record(name, seq, q, tags=pad + fake + b"\0\0")
        out.append(r)
        p += len(r)
    return b"".join(out)


@pytest.mark.parametrize("tile", [64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536])
def test_tile_walk_planted(tile):
    rng = np.random.default_rng(tile)
    data = planted(tile, 60 if tile <= 4096 else 12, rng)
    starts, end, st, rew = hs_starts(data, tile)
    assert (starts, end, st) == (serial_starts(data), len(data), BAM_OK)
    assert rew > 0                   # the fake chains are taken up at the seams and walked again
    text, err = hs_fastq(data, starts)
    assert err == -1 and text == B.fastq_of(B.header() + data)


@pytest.mark.parametrize("tile", [64, 256, 4096, 65536])
def test_tile_walk_random(tile):
    rng = np.random.default_rng(7 + tile)
    recs = B.random_records(rng, 300, 0, 400)
    data = b"".join(recs)
    starts, end, st, _ = hs_starts(data, tile)
    assert (starts, end, st) == (serial_starts(data), len(data), BAM_OK)
    # every cut of the buffer: the starts of the whole records, the chain stops at the first partial one
    for cut in rng.integers(0, len(data), size=20):
        s2, end2, st2, _ = hs_starts(data[:cut], tile)
        whole = [s for s, nx in zip(starts, starts[1:] + [len(data)]) if nx <= cut]
        assert s2 == whole and st2 == (BAM_OK if end2 == cut else BAM_SHORT)


def test_cigar_tags_and_long_reads():
    rng = np.random.default_rng(3)
    recs = [B.record(b"c%d" % i, "ACGT" * 30, [35] * 120, cigar=[(120 << 4) | 4, (3 << 4) | 0],
                     tags=b"RGZgrp1\0NMi" + struct.pack("<i", 3)) for i in range(20)]
    recs += B.random_records(rng, 3, 20000, 60000)
    data = b"".join(recs)
    starts, end, st, _ = hs_starts(data, 256)
    assert (starts, end, st) == (serial_starts(data), len(data), BAM_OK)
    text, err = hs_fastq(data, starts)
    assert err == -1 and text == B.fastq_of(B.header() + data)


def test_reference_small_bam():
    import json

    kat = json.loads(gzip.decompress(open(os.path.join(HERE, "golden", "bam_input_kat.json.gz"), "rb").read()))
    bam = kat["files"]["data/small.bam"].encode("latin-1")
    plain = gzip.decompress(bam)
    st, hlen, _ = hs_header(plain)
    assert st == BAM_OK
    starts, end, est, _ = hs_starts(plain[hlen:], 64)
    assert len(starts) == 3 and est == BAM_OK
    text, err = hs_fastq(plain[hlen:], starts)
    assert err == -1 and text == B.fastq_of(bam)


def test_tool_detects_bam(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import trim_fastq

    bam = B.bam_file([B.record(b"r", "ACGT", [30] * 4)])
    for name in ("in.bam", "in.dat", "in.gz"):
        (tmp_path / name).write_bytes(bam)
        assert trim_fastq.detect_format(str(tmp_path / name)) == "bam"
    fq = b"@r\nACGT\n+\nIIII\n"
    (tmp_path / "in.fastq.gz").write_bytes(B.bgzf(fq))
    assert trim_fastq.detect_format(str(tmp_path / "in.fastq.gz")) == "fastq"
    (tmp_path / "in.fastq").write_bytes(fq)
    assert trim_fastq.detect_format(str(tmp_path / "in.fastq")) == "fastq"
    (tmp_path / "in.fasta").write_bytes(b">r\nACGT\n")
    assert trim_fastq.detect_format(str(tmp_path / "in.fasta")) == "fasta"
    (tmp_path / "empty.fastq").write_bytes(b"")
    assert trim_fastq.detect_format(str(tmp_path / "empty.fastq")) == "fastq"
