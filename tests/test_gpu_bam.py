"""
Unaligned BAM input decoded on the device (cg_fastq_submit_gzip with CG_FORMAT_BAM, read_gzip_device_chunks with
FastqTrimmer(input_format="bam")): the reference's small.bam against its stored answer, the slot text against the
decoder of tests/bam_oracle.py at submission sizes from less than one member to many, every single-end collect against
the same collect on the oracle's FASTQ, valid-looking record starts planted at the kernel's tile seams, each refusal
class (code, message, the stream and context still usable), the submits and collects that refuse CG_FORMAT_BAM,
determinism and a 2-million-record file.
"""
import ctypes as C
import gzip
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import bam_oracle as B
from test_bam_host import _lib as _hostsim, planted

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from cutadapt_b200 import _lib  # noqa: E402
from cutadapt_b200.adapters import BackAdapter, FrontAdapter  # noqa: E402
from cutadapt_b200.pipeline import (DeviceChunk, FastqTrimmer, PairedFastqTrimmer, read_fastq_chunks,  # noqa: E402
                                    read_gzip_device_chunks)

ADAPTER = "AGATCGGAAGAGC"
OPTS = dict(quality_cutoff=(0, 20), minimum_length=20)
SIZES = [3000, 40000, 1 << 20, 64 << 20]


def fixed_records(n, read_len, seed, name_len=12):
    """n records of read_len random bases (ACGTN) with names of name_len characters, built as one array: (BAM records,
    their FASTQ text)."""
    rng = np.random.default_rng(seed)
    lrn = name_len + 1
    body = 32 + lrn + (read_len + 1) // 2 + read_len
    rec = np.zeros((n, 4 + body), dtype=np.uint8)
    head = np.zeros(1, dtype=np.dtype([("bs", "<i4"), ("ref", "<i4"), ("pos", "<i4"), ("lrn", "u1"), ("mapq", "u1"),
                                       ("bin", "<u2"), ("ncig", "<u2"), ("flag", "<u2"), ("lseq", "<i4"),
                                       ("nref", "<i4"), ("npos", "<i4"), ("tlen", "<i4")]))
    head[0] = (body, -1, -1, lrn, 255, 4680, 0, 4, read_len, -1, -1, 0)
    rec[:, :36] = np.frombuffer(head.tobytes(), dtype=np.uint8)
    names = np.char.encode(np.char.add("r", np.char.zfill(np.arange(n).astype(str), name_len - 1)), "ascii")
    rec[:, 36:36 + name_len] = np.frombuffer(names.tobytes(), dtype=np.uint8).reshape(n, name_len)
    codes = rng.choice(np.array([1, 2, 4, 8, 15], dtype=np.uint8), size=(n, read_len + (read_len & 1)),
                       p=[0.24, 0.24, 0.24, 0.24, 0.04])
    if read_len & 1:
        codes[:, -1] = 0
    s = 36 + lrn
    rec[:, s:s + (read_len + 1) // 2] = (codes[:, 0::2] << 4) | codes[:, 1::2]
    qual = rng.integers(0, 42, size=(n, read_len), dtype=np.uint8)
    rec[:, s + (read_len + 1) // 2:] = qual
    fq = np.empty((n, name_len + 2 * read_len + 6), dtype=np.uint8)
    fq[:, 0] = ord("@")
    fq[:, 1:1 + name_len] = rec[:, 36:36 + name_len]
    fq[:, 1 + name_len] = ord("\n")
    fq[:, 2 + name_len:2 + name_len + read_len] = np.frombuffer(B.NIBBLES.encode(), dtype=np.uint8)[codes[:, :read_len]]
    o = 2 + name_len + read_len
    fq[:, o:o + 3] = np.frombuffer(b"\n+\n", dtype=np.uint8)
    fq[:, o + 3:o + 3 + read_len] = qual + 33
    fq[:, -1] = ord("\n")
    return rec.tobytes(), fq.tobytes()


def mixed_records(seed=0):
    """ONT-like long reads spanning many members, empty reads, 254-character names, CIGAR operations and aux tags."""
    rng = np.random.default_rng(seed)
    recs = []
    for i in range(40):
        recs += B.random_records(rng, 1, 1000, 100000)
        recs.append(B.record(b"empty%d" % i, "", []))
        recs.append(B.record((b"n%d_" % i).ljust(254, b"Z"), "ACGTN" * 10, [40] * 50))
        recs.append(B.record(b"c%d" % i, "ACGTTGCA" * 20, rng.integers(0, 94, 160).tolist(),
                             cigar=[(150 << 4) | 0, (10 << 4) | 4], tags=b"RGZgrp1\0NMi\x03\0\0\0XAB" + bytes(7)))
    return b"".join(recs)


def device_text(bam: bytes, size: int):
    """The slot text of every chunk (cg_fastq_slot_read), each chunk then collected without trimming, and that
    output."""
    t = FastqTrimmer(None, input_format="bam")
    texts, outs = [], []
    for chunk in read_gzip_device_chunks(io.BytesIO(bam), t, size):
        buf = np.empty(max(chunk.size, 1), dtype=np.uint8)
        n = C.c_int64()
        _lib.check(_lib.lib().cg_fastq_slot_read(t.ctx.handle, chunk.slot, buf.ctypes.data, buf.size, C.byref(n)))
        assert n.value == chunk.size
        texts.append(buf[:n.value].tobytes())
        outs.append(t.process_chunk(chunk))
    assert t.statistics["in_bytes_gzip"] == len(bam)
    return b"".join(texts), b"".join(outs), t


def _kat():
    return json.load(gzip.open(os.path.join(HERE, "golden", "bam_input_kat.json.gz")))


# ---- 1. the reference's answer ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("size", [64, 1 << 16])
def test_reference_small_bam(size):
    kat = _kat()
    files = {k: v.encode("latin-1") for k, v in kat["files"].items()}
    (case,) = kat["cases"]
    raw = files[case["input"]]
    t = FastqTrimmer([BackAdapter(seq, max_errors=case["error_rate"], min_overlap=case["min_overlap"], name="a0")
                      for _, seq, _ in case["adapters"]], input_format="bam")
    out = b"".join(t.process_chunks(read_gzip_device_chunks(io.BytesIO(raw), t, size)))
    assert out == files[case["expected"]]
    assert t.statistics["n_records"] == 3


def test_reference_small_bam_through_the_tool(tmp_path):
    kat = _kat()
    files = {k: v.encode("latin-1") for k, v in kat["files"].items()}
    for name in ("small.bam", "small.data"):
        inp = tmp_path / name
        inp.write_bytes(files["data/small.bam"])
        out = tmp_path / "out.fastq"
        subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), "-a", "TTAGACATATCTCCGTCG",
                        "-o", str(out), str(inp)], check=True, capture_output=True)
        assert out.read_bytes() == files["cut/small_from_bam.fastq"]
    out = tmp_path / "out.fasta"
    subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), "-a", "TTAGACATATCTCCGTCG",
                    "-o", str(out), str(tmp_path / "small.bam")], check=True, capture_output=True)
    lines = files["cut/small_from_bam.fastq"].split(b"\n")
    assert out.read_bytes() == b"".join(b">" + lines[i][1:] + b"\n" + lines[i + 1] + b"\n" for i in range(0, 12, 4))
    for extra in (["--interleaved"], [str(tmp_path / "small.bam")]):
        p = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), "-a", "ACGT", "-o",
                            str(tmp_path / "o.fastq"), "-p", str(tmp_path / "p.fastq"), str(tmp_path / "small.bam")]
                           + extra, capture_output=True, text=True)
        assert p.returncode != 0 and "single-end" in p.stderr


# ---- 2. the slot text ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("size", SIZES)
def test_slot_text_short_reads(size):
    recs, fq = fixed_records(200_000, 150, seed=1)
    bam = B.bgzf(B.header() + recs, level=1)
    text, out, _ = device_text(bam, size)
    assert text == fq and out == fq


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("level", [0, 6])
def test_slot_text_long_empty_named_and_tagged_reads(size, level):
    recs = mixed_records()
    bam = B.bgzf(B.header(b"@HD\tVN:1.6\n" * 2000, refs=[(b"chr%d" % i, 1000 * i) for i in range(50)]) + recs,
                 member=int(np.random.default_rng(size).integers(20000, 65280)), level=level)
    want = B.fastq_of(bam)
    text, out, _ = device_text(bam, size)
    assert text == want and out == want


# ---- 3. every single-end collect -------------------------------------------------------------------------------------

def _same(make, bam, size, method):
    ref, dev = make("fastq"), make("bam")
    want = [getattr(ref, method)(c) for c in read_fastq_chunks(io.BytesIO(B.fastq_of(bam)), 1 << 16)]
    got = [getattr(dev, method)(c) for c in read_gzip_device_chunks(io.BytesIO(bam), dev, size)]

    def joined(xs):
        if isinstance(xs[0], dict):
            return {k: b"".join(x[k] for x in xs) for k in xs[0]}
        if isinstance(xs[0], tuple):
            return tuple(b"".join(x[i] for x in xs) for i in range(len(xs[0])))
        return b"".join(xs)
    assert joined(got) == joined(want)
    assert {k: v for k, v in dev.statistics.items() if k != "in_bytes_gzip"} == ref.statistics
    if ref._stats is not None:
        a, b = ref.statistics_vector(), dev.statistics_vector()
        assert (a[0] == b[0]).all() and a[1:] == b[1:]


@pytest.mark.parametrize("size", [40000, 1 << 20])
def test_collects_equal_the_oracle_fastq(size):
    recs, _ = fixed_records(20_000, 150, seed=2)
    rng = np.random.default_rng(3)
    # adapters planted in some reads: a BAM record of ACGT..ADAPTER..
    extra = [B.record(b"ad%d" % i, "".join(rng.choice(list("ACGT"), 60)) + ADAPTER + "ACGTACGT" * 5,
                      rng.integers(10, 42, 60 + len(ADAPTER) + 40).tolist()) for i in range(2000)]
    bam = B.bgzf(B.header() + recs + b"".join(extra))
    ads = lambda: [BackAdapter(ADAPTER, name="a"), FrontAdapter("ACGTTGCA", name="b")]  # noqa: E731
    for out_fmt in (None, "fasta"):
        _same(lambda f: FastqTrimmer(ads(), input_format=f, output_format=out_fmt, **OPTS, collect_statistics=True),
              bam, size, "process_chunk")
        _same(lambda f: FastqTrimmer(ads(), input_format=f, output_format=out_fmt, **OPTS,
                                     redirect=("too_short", "untrimmed")), bam, size, "process_chunk_split")
        _same(lambda f: FastqTrimmer(ads(), input_format=f, output_format=out_fmt, **OPTS), bam, size,
              "process_chunk_demux")
    _same(lambda f: FastqTrimmer(ads(), input_format=f, **OPTS), bam, size, "process_chunk_info")
    ref, dev = (FastqTrimmer(ads(), input_format=f, **OPTS, rows=("info", "rest")) for f in ("fastq", "bam"))
    want, got = [], []
    for t, chunks, acc in ((ref, read_fastq_chunks(io.BytesIO(B.fastq_of(bam)), 1 << 16), want),
                           (dev, read_gzip_device_chunks(io.BytesIO(bam), dev, size), got)):
        for c in chunks:
            acc.append((t.process_chunk(c), t.last_rows["info"], t.last_rows["rest"]))
    assert [b"".join(x[i] for x in got) for i in range(3)] == [b"".join(x[i] for x in want) for i in range(3)]


# ---- 4. fake record starts at the kernel's tile seams ---------------------------------------------------------------

def test_planted_record_starts_at_the_tile_seams():
    tile = _hostsim().hs_bam_tile()
    data = planted(tile, 200, np.random.default_rng(11))
    bam = B.bgzf(B.header() + data)
    want = B.fastq_of(bam)
    for size in (1 << 20, 64 << 20):          # the one-submission size puts the planted starts exactly at the seams
        text, out, t = device_text(bam, size)
        assert text == want and out == want
        tiles, rewalked = t.bam_tiles
        assert tiles > 0 and rewalked > 0
    dev, ref = FastqTrimmer([BackAdapter(ADAPTER)], input_format="bam"), FastqTrimmer([BackAdapter(ADAPTER)])
    assert b"".join(dev.process_chunks(read_gzip_device_chunks(io.BytesIO(bam), dev, 64 << 20))) == ref.process_chunk(want)


# ---- 5. refusals -----------------------------------------------------------------------------------------------------

def _submit(ctx, h, gz, final=1, fmt=_lib.CG_FORMAT_BAM):
    slot, res = C.c_int32(-1), _lib.cg_gzin_result()
    rc = _lib.lib().cg_fastq_submit_gzip(ctx.handle, h, gz, len(gz), fmt, final, C.byref(slot), C.byref(res))
    return rc, slot.value, res


def _stream(ctx):
    h = C.c_int32(0)
    _lib.check(_lib.lib().cg_gzin_create(ctx.handle, C.byref(h)))
    return h.value


GOOD = [B.record(b"g%d" % i, "ACGTACGTAC", [30] * 10) for i in range(2)]
BAD = {
    "flag": (B.record(b"x", "ACGT", [30] * 4, flag=16), _lib.CG_EUNSUPPORTED, "flag"),
    "no_quality": (B.record(b"x", "ACGT", None), _lib.CG_EUNSUPPORTED, "no quality"),
    "quality": (B.record(b"x", "ACGT", [30, 30, 94, 30]), _lib.CG_EINVAL, "above 93"),
    "name": (B.record(b"x y", "ACGT", [30] * 4), _lib.CG_EINVAL, "name byte"),
    "block_size": (B.record(b"x", "ACGT", [30] * 4, block_size=33), _lib.CG_EINVAL, "do not fit"),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_refusals_name_the_record_and_leave_the_context_usable(case):
    ctx = _lib.default_context()
    rec, code, what = BAD[case]
    hdr = B.header()
    gz = B.bgzf(hdr + b"".join(GOOD) + rec + GOOD[0])
    h = _stream(ctx)
    rc, slot, _ = _submit(ctx, h, gz)
    msg = _lib.lib().cg_last_error().decode()
    assert rc == code and slot == -1, msg
    assert "record 2 " in msg and "byte %d " % (len(hdr) + len(GOOD[0]) + len(GOOD[1])) in msg and what in msg, msg
    # the stream is unchanged: the same stream takes a good file
    good = B.bam_file(GOOD)
    t = FastqTrimmer(None, input_format="bam")
    rc, slot, res = _submit(ctx, h, good)
    assert rc == 0 and slot >= 0 and res.n_records == 2
    assert t.process_chunk(DeviceChunk(slot, res.chunk_bytes)) == B.fastq_of(good)
    _lib.check(_lib.lib().cg_gzin_destroy(ctx.handle, h))


def test_header_and_truncation_refusals():
    ctx = _lib.default_context()
    plain = B.header() + b"".join(GOOD) + GOOD[0]
    cases = {
        "magic": (B.bgzf(b"BAM\x02" + plain[4:]), "not a BAM file"),
        "negative": (B.bgzf(b"BAM\x01" + (-3).to_bytes(4, "little", signed=True) + plain[8:]), "not a BAM file"),
        "empty": (B.bgzf(b""), "inside the BAM header"),
        "header": (B.bgzf(plain[:len(B.header()) - 2]), "inside the BAM header"),
        "record": (B.bgzf(plain[:-5]), "ends inside record 2"),
        "record_head": (B.bgzf(plain[:-len(GOOD[0]) + 2]), "ends inside record 2"),
    }
    for name, (gz, what) in cases.items():
        h = _stream(ctx)
        rc, slot, _ = _submit(ctx, h, gz)
        msg = _lib.lib().cg_last_error().decode()
        assert rc == _lib.CG_EINVAL and slot == -1 and what in msg, (name, msg)
        rc, slot, res = _submit(ctx, h, B.bam_file(GOOD))
        assert rc == 0 and slot >= 0 and res.n_records == 2, name
        FastqTrimmer(None, input_format="bam").process_chunk(DeviceChunk(slot, res.chunk_bytes))
        _lib.check(_lib.lib().cg_gzin_destroy(ctx.handle, h))
    # a header split over submissions waits in the carry
    h = _stream(ctx)
    full = B.bgzf(plain, member=20)
    rc, slot, res = _submit(ctx, h, full[:28 * 2], final=0)
    assert rc == 0 and slot == -1 and res.consumed > 0
    rc, slot, res = _submit(ctx, h, full[res.consumed:], final=1)
    assert rc == 0 and slot >= 0 and res.n_records == 3 and res.carry_bytes == 0
    assert FastqTrimmer(None, input_format="bam").process_chunk(DeviceChunk(slot, res.chunk_bytes)) == B.fastq_of(full)
    _lib.check(_lib.lib().cg_gzin_destroy(ctx.handle, h))


# ---- 6. where CG_FORMAT_BAM is refused -------------------------------------------------------------------------------

def test_bam_refused_outside_the_single_gzip_submit():
    ctx = _lib.default_context()
    L = _lib.lib()
    bam = B.bam_file(GOOD)
    s1, s2 = C.c_int32(-1), C.c_int32(-1)
    fq = b"@r\nACGT\n+\nIIII\n"
    assert L.cg_fastq_submit_interleaved(ctx.handle, fq, len(fq), _lib.CG_FORMAT_BAM, C.byref(s1), C.byref(s2)) == \
        _lib.CG_EINVAL
    h1, h2 = _stream(ctx), _stream(ctx)
    r1, r2 = _lib.cg_gzin_result(), _lib.cg_gzin_result()
    assert L.cg_fastq_submit_gzip_paired(ctx.handle, h1, h2, bam, len(bam), bam, len(bam), _lib.CG_FORMAT_BAM, 1,
                                         C.byref(s1), C.byref(s2), C.byref(r1), C.byref(r2)) == _lib.CG_EINVAL
    assert L.cg_fastq_submit_gzip_interleaved(ctx.handle, h1, bam, len(bam), _lib.CG_FORMAT_BAM, 1, C.byref(s1),
                                              C.byref(s2), C.byref(r1)) == _lib.CG_EINVAL
    # a collect's params.format
    t = FastqTrimmer(None)
    t.params.format = _lib.CG_FORMAT_BAM
    with pytest.raises(Exception):
        t.process_chunk(fq)
    # a stream keeps its format: BAM after FASTQ, FASTQ after BAM
    fqgz = B.bgzf(fq * 10, eof=False)
    rc, slot, res = _submit(ctx, h1, fqgz, final=0, fmt=_lib.CG_FORMAT_FASTQ)
    assert rc == 0
    if slot >= 0:
        FastqTrimmer(None).process_chunk(DeviceChunk(slot, res.chunk_bytes))
    rc, _, _ = _submit(ctx, h1, bam, final=1)
    assert rc == _lib.CG_EINVAL and "one format" in L.cg_last_error().decode()
    rc, slot, res = _submit(ctx, h2, bam[:-28], final=0)
    assert rc == 0
    if slot >= 0:
        FastqTrimmer(None, input_format="bam").process_chunk(DeviceChunk(slot, res.chunk_bytes))
    rc, _, _ = _submit(ctx, h2, fqgz, final=1, fmt=_lib.CG_FORMAT_FASTQ)
    assert rc == _lib.CG_EINVAL and "one format" in L.cg_last_error().decode()
    for h in (h1, h2):
        _lib.check(L.cg_gzin_destroy(ctx.handle, h))
    # the Python layer
    with pytest.raises(ValueError):
        PairedFastqTrimmer([BackAdapter(ADAPTER)], [], input_format="bam")
    with pytest.raises(ValueError):
        FastqTrimmer([BackAdapter(ADAPTER)], input_format="bam").process_chunk(fq)


# ---- 7. determinism and size -----------------------------------------------------------------------------------------

def test_two_runs_identical_and_two_million_records():
    recs, fq = fixed_records(2_000_000, 50, seed=5)
    bam = B.bgzf(B.header() + recs, level=1)
    runs = []
    for _ in range(2):
        t = FastqTrimmer([BackAdapter(ADAPTER)], input_format="bam", **OPTS)
        runs.append(b"".join(t.process_chunks(read_gzip_device_chunks(io.BytesIO(bam), t, 8 << 20))))
    assert runs[0] == runs[1]
    text, out, _ = device_text(bam, 8 << 20)
    assert text == fq and out == fq
