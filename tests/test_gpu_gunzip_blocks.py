"""
Single-member gzip input inflated block-parallel on the device (cg_gzin_create_ex with CG_GZIN_SPLIT_MEMBERS,
read_gzip_device_*chunks(split_members=True)): every collect family gives the outputs, counters and statistics vectors
of the plain path at submission sizes from below one block to many MiB; paired files that mix a single member with many;
the device's `consumed` / `in_member` sequence against the host build; a member over 2 GiB streamed over submissions;
the corruption classes; determinism.
"""
import ctypes as C
import gzip
import hashlib
import io
import os
import sys
import zlib

import numpy as np
import pytest

from test_gpu_gunzip import OPTS, ADAPTER, fasta_of, layouts, no_gzip_bytes, stats_equal
from test_gunzip_blocks_host import _lib as _hslib
from test_gzip_host import synthetic_reads

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from cutadapt_b200 import _lib  # noqa: E402
from cutadapt_b200.adapters import BackAdapter, FrontAdapter  # noqa: E402
from cutadapt_b200.pipeline import (DeviceChunk, FastqTrimmer, PairedFastqTrimmer, read_fasta_chunks,  # noqa: E402
                                    read_fastq_chunks,
                                    read_gzip_device_chunks, read_gzip_device_interleaved_chunks,
                                    read_gzip_device_paired_chunks, read_interleaved_fastq_chunks,
                                    read_paired_fastq_chunks)

SIZES = [3000, 40000, 1 << 20, 8 << 20]


def one_member(plain: bytes, level=6, strategy=zlib.Z_DEFAULT_STRATEGY) -> bytes:
    if strategy == zlib.Z_DEFAULT_STRATEGY:
        return gzip.compress(plain, level, mtime=0)
    c = zlib.compressobj(level, zlib.DEFLATED, 31, 8, strategy)
    return c.compress(plain) + c.flush()


def single(make, plain, gz, size, method="process_chunks", fasta=False):
    ref, dev = make(), make()
    reader = read_fasta_chunks if fasta else read_fastq_chunks
    want = list(getattr(ref, method)(reader(io.BytesIO(plain), 1 << 16)))
    got = list(getattr(dev, method)(read_gzip_device_chunks(io.BytesIO(gz), dev, size, split_members=True)))
    join = (lambda xs: b"".join(xs)) if method == "process_chunks" else \
        (lambda xs: {k: b"".join(x[k] for x in xs) for k in (xs[0] if xs else {})})
    assert join(got) == join(want)
    assert no_gzip_bytes(dev.statistics) == no_gzip_bytes(ref.statistics)
    assert dev.statistics["in_bytes_gzip"] == len(gz)
    stats_equal(ref, dev)


@pytest.mark.parametrize("level,strategy", [(1, 0), (6, 0), (9, 0), (6, zlib.Z_FIXED)])
@pytest.mark.parametrize("size", SIZES)
def test_fastq_plain_collect(level, strategy, size):
    plain = synthetic_reads(20000, seed=21)
    gz = one_member(plain, level, strategy)
    single(lambda: FastqTrimmer([BackAdapter(ADAPTER, name="a")], **OPTS, collect_statistics=True), plain, gz, size)


@pytest.mark.parametrize("size", SIZES[:3])
def test_fasta_and_fastq_to_fasta(size):
    plain = synthetic_reads(8000, seed=22)
    fa = fasta_of(plain)
    ads = lambda: [BackAdapter(ADAPTER, name="a")]  # noqa: E731
    single(lambda: FastqTrimmer(ads(), input_format="fasta", minimum_length=60, collect_statistics=True), fa,
           one_member(fa), size, fasta=True)
    single(lambda: FastqTrimmer(ads(), output_format="fasta", minimum_length=60, collect_statistics=True), plain,
           one_member(plain, 9), size)


def test_split_demux_and_info():
    plain = synthetic_reads(8000, seed=23)
    gz = one_member(plain)
    kw = dict(OPTS, redirect=("too_short", "too_long", "untrimmed"), collect_statistics=True)
    single(lambda: FastqTrimmer([BackAdapter(ADAPTER, name="a")], **kw), plain, gz, 20000, "process_chunks_split")
    ads = lambda: [BackAdapter(ADAPTER, name="a"), FrontAdapter("ACGTTGCA", name="b")]  # noqa: E731
    for method in ("process_chunk_demux", "process_chunk_info"):
        ref, dev = FastqTrimmer(ads(), **OPTS), FastqTrimmer(ads(), **OPTS)
        want = [getattr(ref, method)(c) for c in read_fastq_chunks(io.BytesIO(plain), 1 << 16)]
        got = [getattr(dev, method)(c) for c in read_gzip_device_chunks(io.BytesIO(gz), dev, 20000, split_members=True)]

        def joined(xs):
            if isinstance(xs[0], dict):
                return {k: b"".join(x[k] for x in xs) for k in xs[0]}
            return tuple(b"".join(x[i] for x in xs) for i in range(2))
        assert joined(got) == joined(want)
        assert no_gzip_bytes(dev.statistics) == ref.statistics


def test_paired_single_member_with_multi_member_and_interleaved():
    r1, r2 = synthetic_reads(6000, seed=24), synthetic_reads(6000, seed=25)
    g1, g2 = one_member(r1), layouts(r2, 6)["bgzf"]
    for kw, method in ((dict(), "process_chunk"), (dict(redirect=("too_short",)), "process_chunk_split")):
        make = lambda: PairedFastqTrimmer([BackAdapter(ADAPTER, name="a")], [BackAdapter(ADAPTER, name="b")],  # noqa
                                          options1=OPTS, options2=OPTS, collect_statistics=True, **kw)
        ref, dev = make(), make()
        want = [getattr(ref, method)(a, b) for a, b in read_paired_fastq_chunks(io.BytesIO(r1), io.BytesIO(r2), 1 << 16)]
        got = [getattr(dev, method)(a, b) for a, b in
               read_gzip_device_paired_chunks(io.BytesIO(g1), io.BytesIO(g2), dev, 30000, split_members=(True, False))]

        def joined(xs):
            if isinstance(xs[0], dict):
                return {k: (b"".join(x[k][0] for x in xs), b"".join(x[k][1] for x in xs)) for k in xs[0]}
            return b"".join(x[0] for x in xs), b"".join(x[1] for x in xs)
        assert joined(got) == joined(want)
        assert [no_gzip_bytes(s) for s in dev.statistics] == [no_gzip_bytes(s) for s in ref.statistics]
        stats_equal(ref, dev)
    l1, l2 = r1.split(b"\n"), r2.split(b"\n")
    il = b"".join(b"\n".join(l1[i:i + 4]) + b"\n" + b"\n".join(l2[i:i + 4]) + b"\n" for i in range(0, len(l1) - 3, 4))
    for kw in (dict(), dict(interleaved_outputs=("output",))):
        ref = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], options1=OPTS, options2=OPTS, **kw)
        dev = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], options1=OPTS, options2=OPTS, **kw)
        want = [ref.process_chunk(c) for c in read_interleaved_fastq_chunks(io.BytesIO(il), 1 << 15)]
        got = [dev.process_chunk(c) for c in
               read_gzip_device_interleaved_chunks(io.BytesIO(one_member(il)), dev, 50000, split_members=True)]
        assert [b"".join(x[k] for x in got) for k in (0, 1)] == [b"".join(x[k] for x in want) for k in (0, 1)]
        assert no_gzip_bytes(dev.statistics[0]) == ref.statistics[0]


def _create(ctx, split=True):
    h = C.c_int32(0)
    _lib.check(_lib.lib().cg_gzin_create_ex(ctx.handle, _lib.CG_GZIN_SPLIT_MEMBERS if split else 0, C.byref(h)))
    return h.value


def _submit(ctx, h, gz, final):
    slot, res = C.c_int32(-1), _lib.cg_gzin_result()
    rc = _lib.lib().cg_fastq_submit_gzip(ctx.handle, h, gz, len(gz), 0, final, C.byref(slot), C.byref(res))
    return rc, slot.value, res


def test_consumed_and_in_member_match_the_host_build():
    ctx = _lib.default_context()
    plain = synthetic_reads(30000, seed=26)
    gz = one_member(plain) + one_member(synthetic_reads(20, seed=3), 1) + one_member(plain, 9)
    hs = _hslib()
    for sub in (20000, 300000, 3 << 20):
        h = _create(ctx)
        stride = max(32768, int(os.environ.get("CUTADAPT_B200_GZIN_STRIDE", _lib.CG_GZIN_STRIDE)))
        s = hs.hs_gzb_create(1, stride, _lib.CG_GZIN_LONG_MEMBER)
        out = np.zeros(len(plain) * 3, dtype=np.uint8)
        info = (C.c_int64 * 7)()
        pos, buf, dev_seq, hs_seq = 0, b"", [], []
        try:
            while True:
                buf += gz[pos:pos + sub]
                pos = min(pos + sub, len(gz))
                final = int(pos == len(gz))
                rc, slot, res = _submit(ctx, h, buf, final)
                assert rc == 0, _lib.lib().cg_last_error()
                if slot >= 0:                  # collected, so the slot is free again
                    FastqTrimmer([BackAdapter(ADAPTER)]).process_chunk(DeviceChunk(slot, res.chunk_bytes))
                src = np.frombuffer(buf + b"\0", dtype=np.uint8)
                assert hs.hs_gzb_submit(s, src.ctypes.data, len(buf), final, 1 << 31, out.ctypes.data, len(out), info) == 0
                dev_seq.append((res.consumed, res.in_member, res.plain_bytes, res.respeculated))
                hs_seq.append((info[0], info[2], info[1], info[3]))
                buf = buf[res.consumed:]
                if final and not buf:
                    break
        finally:
            hs.hs_gzb_destroy(s)
            _lib.check(_lib.lib().cg_gzin_destroy(ctx.handle, h))
        assert dev_seq == hs_seq, sub


def test_a_member_over_2_gib_streams_over_submissions():
    seq = b"ACGTACGTTTGACCAGATCGGAAGAGCACACGTCTGAACTCCAGTCACACGTACGTACGTACGTACGTAAAAACCCCCGGGGGTTTTTACGT"
    rec = b"@r1 x\n" + seq + b"\n+\n" + b"I" * len(seq) + b"\n"
    per = (1 << 24) // len(rec)
    block = rec * per
    n_blocks = (2 << 30) // len(block) + 2                       # a little over 2 GiB of plain bytes
    c = zlib.compressobj(6, zlib.DEFLATED, 31)
    gz = b"".join(c.compress(block) for _ in range(n_blocks)) + c.flush()
    n = per * n_blocks
    unit = FastqTrimmer([BackAdapter(ADAPTER)]).process_chunk(rec * 4)
    assert len(unit) % 4 == 0
    want = hashlib.sha256()
    one = unit[: len(unit) // 4]
    for _ in range(n_blocks):
        want.update(one * per)
    dev = FastqTrimmer([BackAdapter(ADAPTER)])
    got = hashlib.sha256()
    n_chunks = 0
    for out in dev.process_chunks(read_gzip_device_chunks(io.BytesIO(gz), dev, 1 << 20, split_members=True)):
        got.update(out)
        n_chunks += 1
    assert dev.statistics["n_records"] == n and n_chunks > 1
    assert got.hexdigest() == want.hexdigest()


def test_corruptions_are_einval_and_the_context_stays_usable():
    ctx = _lib.default_context()
    plain = synthetic_reads(20000, seed=27)
    lead = one_member(synthetic_reads(30, seed=3))
    good = one_member(plain)
    bad = {"truncated": good[:-3], "crc": good[:-8] + bytes(4) + good[-4:], "isize": good[:-4] + bytes(4),
           "flip": good[:len(good) // 2] + bytes([good[len(good) // 2] ^ 0x10]) + good[len(good) // 2 + 1:]}
    for name, gz in bad.items():
        assert not _ok(lead + gz), name
        for sub in (1 << 30, 100000):
            h = _create(ctx)
            data, pos, buf, rc = lead + gz, 0, b"", 0
            while True:
                buf += data[pos:pos + sub]
                pos = min(pos + sub, len(data))
                rc, slot, res = _submit(ctx, h, buf, int(pos == len(data)))
                if rc:
                    break
                if slot >= 0:
                    FastqTrimmer([BackAdapter(ADAPTER)]).process_chunk(DeviceChunk(slot, res.chunk_bytes))
                buf = buf[res.consumed:]
            assert rc == _lib.CG_EINVAL, name
            assert "byte %d " % len(lead) in _lib.lib().cg_last_error().decode(), name
            _lib.check(_lib.lib().cg_gzin_destroy(ctx.handle, h))
    dev = FastqTrimmer([BackAdapter(ADAPTER)])
    assert b"".join(dev.process_chunks(read_gzip_device_chunks(io.BytesIO(good), dev, split_members=True))) == \
        FastqTrimmer([BackAdapter(ADAPTER)]).process_chunk(plain)


def _ok(gz):
    try:
        gzip.decompress(gz)
        return True
    except (OSError, EOFError, zlib.error):
        return False


def test_determinism():
    plain = synthetic_reads(20000, seed=28)
    gz = one_member(plain, 6)
    outs = []
    for _ in range(2):
        dev = FastqTrimmer([BackAdapter(ADAPTER)], **OPTS)
        outs.append(b"".join(dev.process_chunks(read_gzip_device_chunks(io.BytesIO(gz), dev, 1 << 20,
                                                                        split_members=True))))
    assert outs[0] == outs[1] == FastqTrimmer([BackAdapter(ADAPTER)], **OPTS).process_chunk(plain)


def test_tool_routes_a_long_single_member_input_to_the_device(tmp_path):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    from test_gpu_gunzip import _tool
    from trim_fastq import DEVICE_GZIP_SPLIT_MIN

    rng = np.random.default_rng(29)
    n = 200_000
    seq = rng.choice(np.frombuffer(b"ACGT", np.uint8), (n, 150))
    qual = rng.choice(np.frombuffer(b"#,:FFFF", np.uint8), (n, 150))
    plain = b"".join(b"@r%d\n%s\n+\n%s\n" % (i, seq[i].tobytes(), qual[i].tobytes()) for i in range(n))
    gz = one_member(plain, 6)
    assert len(gz) >= DEVICE_GZIP_SPLIT_MIN
    (tmp_path / "in.fastq.gz").write_bytes(gz)
    (tmp_path / "in.fastq").write_bytes(plain)
    got, st = _tool(tmp_path, tmp_path / "in.fastq.gz", "a.fastq")
    want, st_plain = _tool(tmp_path, tmp_path / "in.fastq", "b.fastq")
    assert st.get("in_bytes_gzip") == len(gz) and "in_bytes_gzip" not in st_plain
    assert got == want
