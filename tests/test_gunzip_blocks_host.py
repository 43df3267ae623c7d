"""
Split gzip input streams (CG_GZIN_SPLIT_MEMBERS) without a GPU: the host build of the block path
(tests/hostsim/hostsim_gunzip_blocks.cpp, on cg_gunzip_core.cuh) against Python's gzip and zlib.  A long member is cut
into chunks at a small stride so that small inputs make many chunks; each test drives a sequence of submissions the way
pipeline.py's reader does (the bytes not consumed are passed again in front of the next ones) and checks the joined
plain bytes, `consumed`, `in_member` and the bit offset kept at every step.
"""
import ctypes as C
import gzip
import os
import random
import struct
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_gunzip_host import hs_gunzip  # noqa: E402

GU_OK, GU_INVALID, GU_UNSUPPORTED = 0, 1, 3
LIMIT = 1 << 31


def _lib():
    from util import hostsim_lib

    lib = hostsim_lib()
    lib.hs_gzb_create.argtypes = [C.c_int, C.c_int64, C.c_int64]
    lib.hs_gzb_create.restype = C.c_void_p
    lib.hs_gzb_destroy.argtypes = [C.c_void_p]
    lib.hs_gzb_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int64,
                                  C.POINTER(C.c_int64)]
    lib.hs_gzb_submit.restype = C.c_int
    return lib


def stream(gz: bytes, sub: int, stride=2048, long_member=1024, split=True, limit=LIMIT, cap=None):
    """Submissions of `sub` new bytes each.  Returns (status, plain, err_at, steps, respeculated); a step is
    (consumed, in_member, bit offset)."""
    lib = _lib()
    s = lib.hs_gzb_create(int(split), stride, long_member)
    want = _python(gz)
    cap = cap or max(len(want) if want is not None else 0, 16 * len(gz), 1 << 16) * 2 + 64
    out = np.zeros(cap, dtype=np.uint8)
    info = (C.c_int64 * 7)()
    plain, steps, respec = [], [], 0
    pos, buf = 0, b""
    try:
        while True:
            take = gz[pos:pos + sub]
            pos += len(take)
            buf += take
            final = pos >= len(gz)
            src = np.frombuffer(buf + b"\0", dtype=np.uint8)
            st = lib.hs_gzb_submit(s, src.ctypes.data, len(buf), int(final), limit, out.ctypes.data, cap, info)
            assert st != -1, "output capacity"
            if st != GU_OK:
                return st, b"".join(plain), info[4], steps, respec
            consumed, n_plain, in_member, rs, _, bitoff, _ = list(info)
            assert 0 <= bitoff < 8 and (in_member or bitoff == 0)
            assert in_member in (0, 1) and (split or not in_member)
            plain.append(out[:n_plain].tobytes())
            steps.append((consumed, in_member, bitoff))
            respec += rs
            buf = buf[consumed:]
            if final and not buf:
                return GU_OK, b"".join(plain), 0, steps, respec
            assert not final or consumed or sub < len(gz), "no progress on the final submission"
            if final and not consumed:
                return GU_INVALID, b"".join(plain), info[4], steps, respec
    finally:
        lib.hs_gzb_destroy(s)


def _python(gz: bytes):
    try:
        return gzip.decompress(gz)
    except (OSError, EOFError, zlib.error):
        return None


def fastq(n_reads: int, seed: int) -> bytes:
    rng = random.Random(seed)
    out = []
    for i in range(n_reads):
        seq = "".join(rng.choice("ACGT") for _ in range(rng.randint(60, 150)))
        if rng.random() < 0.3:
            seq = seq[:40] + "AGATCGGAAGAGC" + seq[53:]
        qual = "".join(chr(33 + min(40, max(2, int(rng.gauss(30, 6))))) for _ in seq)
        out.append(f"@read{i} sample:{seed}\n{seq}\n+\n{qual}\n")
    return "".join(out).encode()


PLAIN = fastq(700, 1)


def gz_member(data: bytes, level=6, wbits=15, memlevel=8, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=(), zdict=None):
    kw = {"zdict": zdict} if zdict is not None else {}
    co = zlib.compressobj(level, zlib.DEFLATED, -wbits, memlevel, strategy, **kw)
    body, at = [], 0
    for p, mode in sorted(flushes):
        body.append(co.compress(data[at:p]))
        body.append(co.flush(mode))
        at = p
    body.append(co.compress(data[at:]))
    body.append(co.flush())
    head = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff"
    return head + b"".join(body) + struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)


def check(gz: bytes, subs=(1 << 30, 9000, 1777), **kw):
    want = _python(gz)
    for sub in subs:
        st, got, err, steps, _ = stream(gz, sub, **kw)
        if want is None:
            assert st == GU_INVALID, (sub, st)
        else:
            assert st == GU_OK and got == want, (sub, st, len(got), len(want))
            assert sum(c for c, _, _ in steps) == len(gz)


@pytest.mark.parametrize("level", range(10))
def test_levels(level):
    check(gz_member(PLAIN, level=level))


@pytest.mark.parametrize("strategy", [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE,
                                      zlib.Z_FIXED])
def test_strategies(strategy):
    check(gz_member(PLAIN, strategy=strategy))


@pytest.mark.parametrize("memlevel", range(1, 10))
def test_memlevels(memlevel):
    check(gz_member(PLAIN, memlevel=memlevel), subs=(1 << 30, 5000))


@pytest.mark.parametrize("wbits", range(9, 16))
def test_window_bits(wbits):
    check(gz_member(PLAIN, wbits=wbits), subs=(1 << 30, 7000))


def test_flush_points():
    flushes = [(1000, zlib.Z_SYNC_FLUSH), (50_000, zlib.Z_FULL_FLUSH), (50_001, zlib.Z_SYNC_FLUSH),
               (120_000, zlib.Z_FULL_FLUSH)]
    check(gz_member(PLAIN, flushes=flushes))


@pytest.mark.parametrize("stride", [1024, 4096])
def test_distance_32768_across_chunks_and_submissions(stride):
    rng = random.Random(5)
    block = bytes(rng.choice(b"ACGT\n") for _ in range(32768))
    data = block + block[:20000] + bytes(rng.choice(b"ACGT") for _ in range(40000)) + block[:3000]
    gz = gz_member(data, level=9)
    check(gz, subs=(1 << 30, 4000, 333), stride=stride)


def test_false_dynamic_header_in_stored_payload():
    # a real dynamic block header (the first block of a flushed stream), byte aligned, copied densely into data that
    # level 0 keeps stored: the start search finds those copies behind the nominal chunk starts
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    raw = co.compress(PLAIN[:20000]) + co.flush(zlib.Z_FULL_FLUSH)
    assert raw[0] & 7 == 4                                  # BFINAL 0, BTYPE 10
    piece = raw[:120] + b"\0" * 8
    data = piece * 1500
    gz = gz_member(data, level=0)
    st, got, _, _, respec = stream(gz, 1 << 30, stride=1024)
    assert st == GU_OK and got == data
    assert respec > 0


def test_distance_behind_the_member_start_in_a_speculative_chunk():
    # a preset dictionary lets zlib write matches in front of the stream's first byte; small blocks (memLevel 1) put
    # them chunks behind the member's start
    zdict = fastq(400, 77)[:32768]
    data = PLAIN[:20000] + zdict[-10000:-7000]
    bad = gz_member(data, level=6, memlevel=1, zdict=zdict)
    assert _python(bad) is None and len(bad) > 4 * 1024
    for sub in (1 << 30, 3000):
        st, _, err, _, _ = stream(bad, sub, stride=1024)
        assert st == GU_INVALID and err == 0


def test_truncation():
    gz = gz_member(PLAIN)
    rng = random.Random(3)
    cuts = sorted(set([11, 12, 13, 100, len(gz) - 8, len(gz) - 1] + [rng.randrange(10, len(gz)) for _ in range(25)]))
    for n in cuts:
        st, _, err, _, _ = stream(gz[:n], 5000)
        assert st == GU_INVALID and err == 0, n


def test_bit_flips():
    gz = gz_member(PLAIN[:60000])
    rng = random.Random(4)
    for _ in range(40):
        b = bytearray(gz)
        i = rng.randrange(10, len(b) - 8)
        b[i] ^= 1 << rng.randrange(8)
        b = bytes(b)
        want = _python(b)
        st, got, err, _, _ = stream(b, 1 << 30)
        if want is None:
            assert st == GU_INVALID and err == 0, i
        else:
            assert st == GU_OK and got == want


@pytest.mark.parametrize("field", ["crc", "isize"])
def test_trailer_errors_of_a_member_over_submissions(field):
    gz = bytearray(gz_member(PLAIN))
    gz[-8 if field == "crc" else -4] ^= 0x40
    lead = gz_member(b"@x\nAC\n+\nII\n", level=6)
    for sub in (3000, 1 << 30):
        st, _, err, steps, _ = stream(lead + bytes(gz), sub)
        assert st == GU_INVALID and err == len(lead)


def test_long_short_long_with_padding():
    a, b, c = gz_member(PLAIN), gz_member(PLAIN[:900]), gz_member(fastq(500, 2), level=9)
    gz = a + b"\0" * 7 + b + c + b"\0" * 3 + a
    assert _python(gz) == PLAIN + PLAIN[:900] + fastq(500, 2) + PLAIN
    check(gz, subs=(1 << 30, 6000, 999))
    st, _, err, _, _ = stream(gz[:len(a) + 7 + len(b) + 9], 1 << 30)
    assert st == GU_INVALID and err == len(a) + 7 + len(b)


def test_submission_sizes_and_the_state_kept():
    gz = gz_member(PLAIN, level=6)
    want = _python(gz)
    for sub in (300, 1000, 4096, 20_000, 100_000, len(gz)):
        st, got, _, steps, _ = stream(gz, sub)
        assert st == GU_OK and got == want
        assert any(m for _, m, _ in steps) == (sub < len(gz))
        assert steps[-1][1] == 0


def test_a_member_streams_under_a_small_limit():
    gz = gz_member(PLAIN * 3, level=6)
    st, got, _, steps, _ = stream(gz, 1 << 30, limit=100_000)
    assert st == GU_OK and got == PLAIN * 3
    assert len(steps) > 3 and all(m for _, m, _ in steps[:-1])


@pytest.mark.parametrize("which", ["levels", "flushes", "multi", "truncated", "flipped"])
def test_default_mode_is_unchanged(which):
    gz = {"levels": gz_member(PLAIN, level=1), "flushes": gz_member(PLAIN, flushes=[(4000, zlib.Z_FULL_FLUSH)]),
          "multi": gz_member(PLAIN[:5000]) + gz_member(PLAIN[5000:9000], level=0),
          "truncated": gz_member(PLAIN)[:-3], "flipped": gz_member(PLAIN)[:500] + b"\x55" + gz_member(PLAIN)[501:]}[which]
    st, got, consumed, err = hs_gunzip(gz)
    lib = _lib()
    s = lib.hs_gzb_create(0, 2048, 1024)
    try:
        out = np.zeros(len(PLAIN) * 2 + 64, dtype=np.uint8)
        info = (C.c_int64 * 7)()
        src = np.frombuffer(gz + b"\0", dtype=np.uint8)
        st2 = lib.hs_gzb_submit(s, src.ctypes.data, len(gz), 1, LIMIT, out.ctypes.data, len(out), info)
    finally:
        lib.hs_gzb_destroy(s)
    assert st2 == st
    if st == GU_OK:
        assert (info[0], out[:info[1]].tobytes(), info[2]) == (consumed, got, 0)
    else:
        assert info[4] == err


def submit_once(gz: bytes, final: bool, stride=2048, long_member=1024):
    """One submission on a fresh split stream: (status, info)."""
    lib = _lib()
    s = lib.hs_gzb_create(1, stride, long_member)
    try:
        out = np.zeros(max(64 * len(gz), 1 << 16), dtype=np.uint8)
        info = (C.c_int64 * 7)()
        src = np.frombuffer(gz + b"\0", dtype=np.uint8)
        st = lib.hs_gzb_submit(s, src.ctypes.data, len(gz), int(final), LIMIT, out.ctypes.data, len(out), info)
        return st, list(info), out[:info[1]].tobytes()
    finally:
        lib.hs_gzb_destroy(s)


def test_truncation_at_every_block_boundary():
    # small blocks (memLevel 1); the boundaries are where a stream fed 150 bytes at a time stopped inside the member
    gz = gz_member(PLAIN[:60000], memlevel=1)
    want = _python(gz)
    st, _, _, steps, _ = stream(gz, 150)
    assert st == GU_OK
    bounds, at = [], 0
    for consumed, in_member, bitoff in steps:
        at += consumed
        if in_member:
            bounds.append(at * 8 + bitoff)
    bounds = sorted(set(bounds))
    assert len(bounds) > 20
    for b in bounds:
        prefix = gz[:(b + 7) // 8]
        # not final: no block completes in the < 8 bits behind b, so the stream stops exactly at b, with the plain
        # bytes of every block in front of it
        st, info, got = submit_once(prefix, False)
        assert st == GU_OK and (info[0], info[5], info[2]) == (b >> 3, b & 7, 1), b
        assert want.startswith(got)
        st, info, _ = submit_once(prefix, True)
        assert st == GU_INVALID and info[4] == 0, b
