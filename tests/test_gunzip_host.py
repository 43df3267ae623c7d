"""
The gzip input path without a GPU: the host build of cg_gunzip_core.cuh (tests/hostsim, hs_gunzip) against Python's
gzip module on a seeded corpus -- what it accepts it must inflate to the same bytes, what gzip rejects it must reject --
and the chain's `consumed` and the record cuts against pipeline.py's readers.
"""
import ctypes as C
import gzip
import os
import struct
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GU_OK, GU_INVALID, GU_UNSUPPORTED = 0, 1, 3
LIMIT = 1 << 31


def _lib():
    from util import hostsim_lib

    lib = hostsim_lib()
    lib.hs_gunzip.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_void_p] + [C.POINTER(C.c_int64)] * 3
    lib.hs_gunzip.restype = C.c_int
    lib.hs_gu_records.argtypes = [C.c_void_p, C.c_int64, C.c_int]
    lib.hs_gu_records.restype = C.c_int64
    lib.hs_gu_cut.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int64]
    lib.hs_gu_cut.restype = C.c_int64
    return lib


def hs_gunzip(gz: bytes, final=True, after_member=False, limit=LIMIT):
    """(status, plain bytes, consumed, err_at)"""
    lib = _lib()
    src = np.frombuffer(gz + b"\0", dtype=np.uint8)
    ok = _python(gz)
    cap = len(ok) if isinstance(ok, bytes) else 0
    out = np.zeros(max(cap, 1 << 20) + 64, dtype=np.uint8)
    consumed, plain, err = C.c_int64(), C.c_int64(), C.c_int64()
    st = lib.hs_gunzip(src.ctypes.data, len(gz), int(final), int(after_member), limit, out.ctypes.data, C.byref(consumed),
                       C.byref(plain), C.byref(err))
    return st, out[: plain.value].tobytes(), consumed.value, err.value


def _python(gz: bytes):
    try:
        return gzip.decompress(gz)
    except (OSError, EOFError, zlib.error):
        return None


def check(gz: bytes):
    """The host build accepts exactly what gzip accepts, with the same bytes."""
    want = _python(gz)
    st, got, consumed, _ = hs_gunzip(gz)
    if want is None:
        assert st == GU_INVALID, gz[:40]
    else:
        assert st == GU_OK and got == want and consumed == len(gz)
    return st


def deflate(data: bytes, level=6, wbits=-15, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=()):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
    out, at = [], 0
    for pos, mode in flushes:
        out.append(c.compress(data[at:pos]) + c.flush(mode))
        at = pos
    out.append(c.compress(data[at:]) + c.flush())
    return b"".join(out)


def member(data: bytes, raw: bytes = None, flg=0, extra=b"", name=b"", comment=b"", hcrc=b"\0\0", **kw):
    head = b"\x1f\x8b\x08" + bytes([flg]) + b"\0\0\0\0\0\xff"
    if flg & 4:
        head += struct.pack("<H", len(extra)) + extra
    if flg & 8:
        head += name + b"\0"
    if flg & 16:
        head += comment + b"\0"
    if flg & 2:
        head += hcrc
    body = deflate(data, **kw) if raw is None else raw
    return head + body + struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)


def texts(seed=0):
    rng = np.random.default_rng(seed)
    reads = b"".join(b"@r%d\n" % i + rng.choice(np.frombuffer(b"ACGT", np.uint8), 150).tobytes() + b"\n+\n" +
                     rng.integers(33, 75, 150, dtype=np.uint8).tobytes() + b"\n" for i in range(300))
    return [b"", b"A", reads, rng.integers(0, 256, 70000, dtype=np.uint8).tobytes(), b"AC" * 40000,
            rng.integers(0, 4, 100000, dtype=np.uint8).tobytes()]


@pytest.mark.parametrize("level", range(10))
def test_levels(level):
    for t in texts(level):
        check(member(t, level=level))


@pytest.mark.parametrize("strategy", [zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FILTERED])
def test_strategies(strategy):
    for t in texts(1):
        check(member(t, strategy=strategy))


@pytest.mark.parametrize("wbits", range(9, 16))
def test_windows(wbits):
    for t in texts(2)[2:]:
        check(member(t, wbits=-wbits))


def test_sync_and_full_flushes_give_empty_stored_blocks():
    t = texts(3)[2]
    flushes = [(i, zlib.Z_SYNC_FLUSH if i % 2 else zlib.Z_FULL_FLUSH) for i in range(0, len(t), 997)]
    check(member(t, flushes=flushes))
    check(member(b"", flushes=[(0, zlib.Z_SYNC_FLUSH)] * 3))


def test_header_fields_and_reserved_bits():
    t = texts(4)[2]
    for flg, kw in ((4, dict(extra=b"BC\x02\0\0\0")), (8, dict(name=b"reads.fastq")), (16, dict(comment=b"c")),
                    (2, dict(hcrc=b"\x12\x34")), (4 | 8 | 16 | 2, dict(extra=b"xy", name=b"n", comment=b"")),
                    (0xE0, {}), (0xFF, dict(extra=b"", name=b"a", comment=b"b"))):
        check(member(t, flg=flg, **kw))


def test_bgzf_style_members_and_this_projects_members():
    from test_gzip_host import hs_gzip

    t = texts(5)[2] * 20
    bgzf = b"".join(member(t[i:i + 65280], flg=4, extra=b"BC\x02\0\0\0") for i in range(0, len(t), 65280))
    assert check(bgzf) == GU_OK
    assert check(hs_gzip(t)) == GU_OK
    assert check(hs_gzip(t) + member(b"") + member(b"") + b"\0" * 7 + hs_gzip(b"@x\nA\n+\nI\n") + b"\0\0") == GU_OK
    assert check(b"") == GU_OK


def test_long_matches_far_distances_and_overlaps():
    rng = np.random.default_rng(6)
    head = rng.integers(0, 256, 300, dtype=np.uint8).tobytes()
    check(member(head + b"\0" * (32768 - 300) + head))              # distance 32 768
    check(member(b"Q" * 100000))                                     # length 258
    for d in range(1, 32):                                           # overlapping copies
        pat = rng.integers(0, 256, d, dtype=np.uint8).tobytes()
        check(member(pat * (3000 // d)))


def test_stored_blocks_holding_false_candidates():
    t = (b"\x1f\x8b\x08" + bytes(range(40))) * 500
    m = member(t, level=0)
    assert m.count(b"\x1f\x8b\x08") > 100
    assert check(m + m) == GU_OK


def _stored(data, final=1):
    return bytes([final]) + struct.pack("<HH", len(data), ~len(data) & 0xFFFF) + data


def test_corruptions_are_rejected_as_gzip_rejects_them():
    good = member(texts(7)[2])
    bad = [
        good + b"x",                                                 # trailing garbage
        good + b"\0\0\x1f",                                          # a header's first byte
        good[:2] + b"\x07" + good[3:],                               # method 7
        good[:-8] + struct.pack("<I", zlib.crc32(texts(7)[2]) ^ 1) + good[-4:],    # CRC-32
        good[:-4] + struct.pack("<I", len(texts(7)[2]) + 1),         # ISIZE
        b"\0" + good,                                                # zeros in front of the first member
        member(b"abc", raw=b"\x07\0"),                               # block type 3
        member(b"abc", raw=b"\x01\x03\x00\x00\x00abc"),              # LEN / NLEN
        member(b"A" * 10, raw=bytes([0x03 | (30 << 3) % 256]) + b"\0" * 4),   # distance symbols in a fixed block
    ]
    for gz in bad:
        assert _python(gz) is None
        assert check(gz) == GU_INVALID
    # fixed-code symbol 286 (11000110 as an 8-bit code), distance code 30, distance behind the member's start
    def bits(*fields):
        v, n = 0, 0
        for val, width, rev in fields:
            if rev:
                val = int(format(val, f"0{width}b")[::-1], 2)
            v |= val << n
            n += width
        return v.to_bytes((n + 7) // 8 + 1, "little")
    for body in (bits((1, 1, 0), (1, 2, 0), (0b11000110, 8, 1)),
                 bits((1, 1, 0), (1, 2, 0), (0b0000001, 7, 1), (30, 5, 1)),
                 bits((1, 1, 0), (1, 2, 0), (0b0000001, 7, 1), (0, 5, 1))):
        gz = member(b"AAA", raw=body)
        assert _python(gz) is None and check(gz) == GU_INVALID
    # dynamic blocks: HLIT 287, HDIST 31, an over-subscribed and an incomplete code-length code
    for body in (bits((1, 1, 0), (2, 2, 0), (30, 5, 0), (0, 5, 0), (0, 4, 0)) + b"\0" * 8,
                 bits((1, 1, 0), (2, 2, 0), (0, 5, 0), (30, 5, 0), (0, 4, 0)) + b"\0" * 8,
                 bits((1, 1, 0), (2, 2, 0), (0, 5, 0), (0, 5, 0), (0, 4, 0), (1, 3, 0), (1, 3, 0), (1, 3, 0),
                      (1, 3, 0)) + b"\0" * 8,
                 bits((1, 1, 0), (2, 2, 0), (0, 5, 0), (0, 5, 0), (0, 4, 0), (1, 3, 0), (0, 3, 0), (0, 3, 0),
                      (0, 3, 0)) + b"\0" * 8):
        gz = member(b"AAA", raw=body)
        assert _python(gz) is None and check(gz) == GU_INVALID


def test_truncation_at_every_byte_of_a_small_member():
    m = member(b"@r\nACGT\n+\nIIII\n" * 3, flg=8 | 4, name=b"n", extra=b"e")
    for k in range(1, len(m)):
        assert check(m[:k]) == GU_INVALID
        st, _, consumed, _ = hs_gunzip(m[:k], final=False)
        assert st == GU_OK and consumed == 0                        # needs more input, nothing taken
    st, _, consumed, _ = hs_gunzip(m + m[:k], final=False)
    assert st == GU_OK and consumed == len(m)


def test_random_bit_flips_agree_with_gzip():
    rng = np.random.default_rng(8)
    base = member(texts(8)[2][:3000])
    for _ in range(400):
        gz = bytearray(base)
        gz[int(rng.integers(10, len(gz)))] ^= 1 << int(rng.integers(0, 8))
        check(bytes(gz))


def test_consumed_is_the_whole_members_of_every_prefix():
    from test_gzip_host import hs_gzip, members

    t = texts(9)[2] * 3
    ms = [member(t[:5000]), b"\0\0", member(b"")] + [m for m, _ in members(hs_gzip(t))] + \
        [member(t[5000:9000], flg=8, name=b"x")]
    gz = b"".join(ms)
    ends = [int(e) for e, m in zip(np.cumsum([len(m) for m in ms]), ms) if m[:1] != b"\0"]
    rng = np.random.default_rng(9)
    for k in sorted(set(rng.integers(0, len(gz) + 1, 300).tolist()) | set(ends) | {e + 1 for e in ends}):
        k = min(k, len(gz))
        st, plain, consumed, _ = hs_gunzip(gz[:k], final=False)
        assert st == GU_OK
        whole = max([0] + [e for e in ends if e <= k])
        while whole and whole < k and gz[whole] == 0:               # zeros behind a member are taken with it
            whole += 1
        assert consumed == whole
        assert plain == (gzip.decompress(gz[:whole]) if whole else b"")


def test_the_size_limit_stops_the_chain():
    a, b = member(b"A" * 1000), member(b"C" * 1000)
    st, plain, consumed, _ = hs_gunzip(a + b, limit=1500)
    assert st == GU_OK and consumed == len(a) and plain == b"A" * 1000
    st, _, _, err = hs_gunzip(a + b, limit=900)
    assert st == GU_UNSUPPORTED and err == 0


# ---- record cuts -------------------------------------------------------------------------------------------------------

def _buf(rng, fasta):
    parts = []
    if fasta and rng.random() < 0.3:
        parts.append(b"# comment\n")
    for i in range(int(rng.integers(0, 9))):
        if fasta:
            parts.append(b">r%d\n" % i + b"ACGT\n" * int(rng.integers(0, 3)))
        else:
            parts.append(b"@r%d\nAC\n+\nII\n" % i)
    s = b"".join(parts)
    return s[: int(rng.integers(0, len(s) + 1))]


@pytest.mark.parametrize("fasta", [0, 1])
def test_cuts_equal_the_readers(fasta):
    from cutadapt_b200 import pipeline as P

    lib = _lib()
    rng = np.random.default_rng(10 + fasta)
    for _ in range(1500):
        b = _buf(rng, fasta)
        a = np.frombuffer(b + b"\0", dtype=np.uint8)
        single = P._fasta_head(b, len(b)) if fasta else P._fastq_head(b, len(b))
        pairs = P._fasta_pairs_head(b, len(b)) if fasta else P._fastq_head(b, len(b), 8)
        assert lib.hs_gu_cut(a.ctypes.data, len(b), fasta, 0, 0) == single
        assert lib.hs_gu_cut(a.ctypes.data, len(b), fasta, 1, 0) == pairs
        b2 = _buf(rng, fasta)
        a2 = np.frombuffer(b2 + b"\0", dtype=np.uint8)
        if fasta:
            want_r = min(P._fasta_headers(x, P._fasta_head(x, len(x))) for x in (b, b2))
            want = [P._fasta_cut(x, len(x), want_r) if want_r else 0 for x in (b, b2)]
        else:
            want_r = min(x.count(b"\n", 0, P._fastq_head(x, len(x))) // 4 for x in (b, b2))
            want = [P._cut_records(x, len(x), want_r) for x in (b, b2)]
        r = min(lib.hs_gu_records(x.ctypes.data, len(y), fasta) for x, y in ((a, b), (a2, b2)))
        assert r == want_r
        assert [lib.hs_gu_cut(x.ctypes.data, len(y), fasta, 2, r) for x, y in ((a, b), (a2, b2))] == want


def test_tool_sends_inputs_whose_first_member_ends_within_a_mib_to_the_device(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import trim_fastq as T
    from test_gzip_host import hs_gzip

    rng = np.random.default_rng(11)
    plain = rng.integers(0, 256, 3 << 20, dtype=np.uint8).tobytes()        # stored blocks: no compression
    for name, data, device in (("multi.gz", hs_gzip(plain), True), ("single.gz", gzip.compress(plain, 6), False),
                               ("small.gz", gzip.compress(b"@r\nA\n+\nI\n"), True), ("plain.fastq", plain, False),
                               ("bad.gz", b"not gzip", False),
                               ("edge.gz", member(plain[:(1 << 20) - 200], level=0), True),
                               ("over.gz", member(plain[:(1 << 20) + 100], level=0), False)):
        (tmp_path / name).write_bytes(data)
        assert T.gzip_on_device(str(tmp_path / name)) == device, name
