"""
Row outputs (--info-file, --rest-file, --wildcard-file) from every device collect (cg_fastq_request_rows /
cg_fastq_read_rows): the reference's paired info files, every single-end and paired collect against the oracle with the
outputs, counters and statistics of the same call without requests unchanged, gzip input, FASTA input, rows compressed
on the device, and the argument errors of the two calls.
"""
import ctypes as C
import gzip
import io
import os
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest

import fasta_oracle as FO
import rows_oracle as RW
from oracle import oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ads(which):
    import cutadapt_b200.adapters as PA

    if which == 1:
        return [PA.BackAdapter("AGATCGGAAGAGC", name="ilmn"), PA.BackAdapter("TTAGACATATNNAC", name="wild"),
                PA.FrontAdapter("ACGGTCAT", name="front")]
    return [PA.BackAdapter("CAGTGGAGTA", name="r2a"), PA.BackAdapter("GGCTNNTACG", name="r2wild"),
            PA.FrontAdapter("TTGACCAG", name="r2front")]


def _random_fastq(rng, n, adapters, prefix="r", mate=""):
    recs = []
    for i in range(n):
        seq = "".join(rng.choice("ACGT") for _ in range(rng.randint(0, 70)))
        for _ in range(rng.choice([0, 1, 1, 2])):
            a = rng.choice(adapters).replace("N", rng.choice("ACGT"))
            piece = a if rng.random() < 0.6 else a[: rng.randint(3, len(a))]
            at = rng.randint(0, len(seq))
            seq = seq[:at] + piece + seq[at:]
        qual = "".join(chr(33 + rng.choice([2, 10, 20, 30, 38, 40])) for _ in seq)
        recs.append(f"@{prefix}{i}{mate} x\n{seq}\n+\n{qual}\n")
    return "".join(recs).encode()


def _pair_data(seed, n=400):
    rng = random.Random(seed)
    s1 = [a.sequence for a in _ads(1)]
    s2 = [a.sequence for a in _ads(2)]
    return _random_fastq(rng, n, s1, mate="/1"), _random_fastq(rng, n, s2, mate="/2")


# trimmer keyword arguments and the oracle's of the same options
OPTS = dict(quality_cutoff=(5, 20), cut=(2, -1), times=2, minimum_length=15)
KW = dict(quality_trim=True, cutoff_front=5, cutoff_back=20, cut=(2, -1), times=2, minimum_length=15)


def _stats(t):
    v = t.statistics_vector()
    return [(x[0].tolist(), x[1], x[2]) for x in v] if isinstance(v[0], tuple) else (v[0].tolist(), v[1], v[2])


# ---- the reference's known answer ------------------------------------------------------------------------------------

def test_paired_trimmer_reproduces_the_paired_info_files():
    from cutadapt_b200.pipeline import PairedFastqTrimmer

    kat = RW.paired_rows_kat()
    c = kat["cases"][0]
    o = c["options"]
    data1, data2 = (RW.kat_bytes(kat, k) for k in c["inputs"])
    t = PairedFastqTrimmer(FO.kat_adapters(o, "specs1"), FO.kat_adapters(o, "specs2"), o["options1"], o["options2"],
                           rows=("info",), rows2=("info",))
    out = t.process_chunk(data1, data2)
    assert out == tuple(RW.kat_bytes(kat, k) for k in c["expected"]["output"])
    for got, key in zip(t.last_rows["info"], c["expected"]["info"]):
        assert RW.strip_trailing(got) == RW.strip_trailing(RW.kat_bytes(kat, key))


@pytest.mark.parametrize("gz", [False, True])
def test_trim_fastq_reproduces_the_paired_info_files(gz, tmp_path):
    kat = RW.paired_rows_kat()
    c = kat["cases"][0]
    paths = []
    for k in c["inputs"]:
        p = tmp_path / os.path.basename(k)
        p.write_bytes(RW.kat_bytes(kat, k))
        paths.append(str(p))
    ext = ".txt.gz" if gz else ".txt"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py")] + c["argv"] +
                       ["--info-file", "info1" + ext, "--info-file-paired", "info2" + ext, "-o", "o1.fastq", "-p",
                        "o2.fastq"] + paths, capture_output=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    for name, key in zip(("o1.fastq", "o2.fastq"), c["expected"]["output"]):
        assert (tmp_path / name).read_bytes() == RW.kat_bytes(kat, key)
    for name, key in zip(("info1" + ext, "info2" + ext), c["expected"]["info"]):
        got = (tmp_path / name).read_bytes()
        got = gzip.decompress(got) if gz else got
        assert RW.strip_trailing(got) == RW.strip_trailing(RW.kat_bytes(kat, key))


# ---- single-end collects ---------------------------------------------------------------------------------------------

def _single(method, rows=RW.KINDS, **extra):
    from cutadapt_b200.pipeline import FastqTrimmer

    return FastqTrimmer(_ads(1), **OPTS, collect_statistics=True, rows=rows, **extra)


SINGLE = {
    "plain": (dict(), lambda t, d: t.process_chunk(d)),
    "chunks": (dict(), lambda t, d: list(t.process_chunks([d]))),
    "split": (dict(redirect=("too_short", "untrimmed")), lambda t, d: t.process_chunk_split(d)),
    "demux": (dict(), lambda t, d: t.process_chunk_demux(d)),
}


@pytest.mark.parametrize("variant", sorted(SINGLE))
def test_single_end_collects_against_the_oracle(variant):
    extra, run = SINGLE[variant]
    data, _ = _pair_data(11)
    _, _, want = RW.oracle_rows_single(oracle, data, _ads(1), KW)
    with_rows, without = _single(variant, **extra), _single(variant, rows=(), **extra)
    got = run(with_rows, data)
    assert with_rows.last_rows == want
    assert got == run(without, data)
    assert with_rows.statistics == without.statistics
    assert _stats(with_rows) == _stats(without)
    assert without.last_rows == {}


def test_gzip_device_chunks_against_the_oracle():
    from cutadapt_b200.pipeline import read_gzip_device_chunks

    data, _ = _pair_data(12, 3000)
    # many members, so that the file is cut into several chunks
    gz = b"".join(gzip.compress(data[i:i + 40000]) for i in range(0, len(data), 40000))
    assert gzip.decompress(gz) == data
    t = _single("plain")
    outs, rows = [], {k: b"" for k in RW.KINDS}
    chunks = []
    for chunk in read_gzip_device_chunks(io.BytesIO(gz), t, 1 << 16):
        chunks.append(len(chunk))
        outs.append(t.process_chunk(chunk))
        for k in RW.KINDS:
            rows[k] += t.last_rows[k]
    assert len(chunks) > 1
    want_out, _, want = RW.oracle_rows_single(oracle, data, _ads(1), KW)
    assert rows == want
    assert b"".join(outs) == _single("plain", rows=()).process_chunk(data)


# ---- paired collects ---------------------------------------------------------------------------------------------------

def _interleave(a, b):
    la, lb = a.splitlines(True), b.splitlines(True)
    return b"".join(b"".join(la[i:i + 4] + lb[i:i + 4]) for i in range(0, len(la), 4))


def _paired(rows=True, pair_adapters=False, **extra):
    from cutadapt_b200.pipeline import PairedFastqTrimmer

    opts = dict(OPTS)
    if pair_adapters:
        opts.pop("times")
    r = dict(rows=RW.KINDS, rows2=("info",)) if rows else {}
    return PairedFastqTrimmer(_ads(1), _ads(2), opts, opts, pair_adapters=pair_adapters, collect_statistics=True,
                              **r, **extra)


PAIRED = {
    "plain": (dict(), lambda t, a, b: t.process_chunk(a, b)),
    "split": (dict(redirect=("too_short", "untrimmed")), lambda t, a, b: t.process_chunk_split(a, b)),
    "interleaved_input": (dict(), lambda t, a, b: t.process_chunk(_interleave(a, b))),
    "interleaved_outputs": (dict(redirect=("too_short",), interleaved_outputs=("output", "too_short")),
                            lambda t, a, b: t.process_chunk_split(a, b)),
    "demux": (dict(), lambda t, a, b: t.process_chunk_demux(a, b)),
    "combinatorial": (dict(), lambda t, a, b: t.process_chunk_demux(a, b, combinatorial=True)),
    "chunks_split": (dict(redirect=("too_short",)), lambda t, a, b: list(t.process_chunks_split([(a, b)]))),
    "pair_adapters": (dict(pair_adapters=True), lambda t, a, b: t.process_chunk(a, b)),
}


@pytest.mark.parametrize("variant", sorted(PAIRED))
def test_paired_collects_against_the_oracle(variant):
    extra, run = PAIRED[variant]
    a, b = _pair_data(21)
    pair = extra.get("pair_adapters", False)
    kw = dict(KW)
    if pair:
        kw.pop("times")
    _, _, _, _, want1, want2 = RW.oracle_rows_paired(oracle, a, b, _ads(1), _ads(2), kw, kw, pair_adapters=pair)
    with_rows, without = _paired(**extra), _paired(rows=False, **extra)
    got = run(with_rows, a, b)
    assert set(with_rows.last_rows) == set(RW.KINDS)
    for k in RW.KINDS:
        r1, r2 = with_rows.last_rows[k]
        assert r1 == want1[k], k
        assert r2 == (want2[k] if k == "info" else b""), k
    assert got == run(without, a, b)
    assert with_rows.statistics == without.statistics
    assert _stats(with_rows) == _stats(without)


def test_gzip_device_paired_chunks_against_the_oracle():
    from cutadapt_b200.pipeline import read_gzip_device_paired_chunks

    a, b = _pair_data(22, 1500)
    t = _paired()
    rows1, rows2 = {k: b"" for k in RW.KINDS}, b""
    outs = []
    for c1, c2 in read_gzip_device_paired_chunks(io.BytesIO(gzip.compress(a)), io.BytesIO(gzip.compress(b)), t, 1 << 15):
        outs.append(t.process_chunk(c1, c2))
        for k in RW.KINDS:
            rows1[k] += t.last_rows[k][0]
        rows2 += t.last_rows["info"][1]
    _, _, _, _, want1, want2 = RW.oracle_rows_paired(oracle, a, b, _ads(1), _ads(2), KW, KW)
    assert rows1 == want1 and rows2 == want2["info"]
    assert tuple(b"".join(o[i] for o in outs) for i in (0, 1)) == _paired(rows=False).process_chunk(a, b)


# ---- FASTA input, gzip rows --------------------------------------------------------------------------------------------

def test_fasta_info_rows_have_empty_quality_columns():
    from cutadapt_b200.pipeline import FastqTrimmer

    data, _ = _pair_data(31)
    lines = data.splitlines()
    fasta = b"".join(b">" + lines[i][1:] + b"\n" + lines[i + 1] + b"\n" for i in range(0, len(lines), 4))
    fq = FastqTrimmer(_ads(1), times=2, rows=("info",))
    fa = FastqTrimmer(_ads(1), times=2, rows=("info",), input_format="fasta")
    fq.process_chunk(data)
    fa.process_chunk(fasta)
    want = []
    for row in fq.last_rows["info"].splitlines():
        f = row.split(b"\t")
        if f[1] == b"-1":
            f[3] = b""
        else:
            f[8] = f[9] = f[10] = b""
        want.append(b"\t".join(f) + b"\n")
    assert fa.last_rows["info"] == b"".join(want)


def _members(data):
    """Plain sizes of the gzip members of data, in order."""
    sizes = []
    while data:
        d = zlib.decompressobj(31)
        sizes.append(len(d.decompress(data)))
        assert d.eof
        data = d.unused_data
    return sizes


def _submit(ctx, data):
    from cutadapt_b200 import _lib

    buf = np.frombuffer(data, dtype=np.uint8)
    slot = C.c_int32(-1)
    _lib.check(_lib.lib().cg_fastq_submit(ctx.handle, buf.ctypes.data, buf.size, C.byref(slot)))
    return slot.value, buf


def test_gzip_rows_are_the_plain_rows_in_members():
    from cutadapt_b200 import _lib
    from cutadapt_b200.pipeline import FastqTrimmer, _row_text

    data, _ = _pair_data(41, 4000)
    plain = FastqTrimmer(_ads(1), **OPTS, rows=RW.KINDS)
    packed = FastqTrimmer(_ads(1), **OPTS, rows=RW.KINDS, gzip_rows=RW.KINDS)
    assert plain.process_chunk(data) == packed.process_chunk(data)
    for k in RW.KINDS:
        assert gzip.decompress(packed.last_rows[k]) == plain.last_rows[k], k
    assert len(plain.last_rows["info"]) > 3 * _lib.GZ_MEMBER
    # the sizes the library reports, and the members
    lib, t = _lib.lib(), packed
    slot, keep = _submit(t.ctx, data)
    blob, off = _row_text(t.adapters, "info")
    _lib.check(lib.cg_fastq_request_rows(t.ctx.handle, slot, _lib.CG_ROWS_INFO, blob, off.ctypes.data, off.size - 1, 1))
    out = np.empty(2 * len(data) + 4096, dtype=np.uint8)
    res = _lib.cg_fastq_result()
    _lib.check(lib.cg_fastq_collect(t.ctx.handle, slot, t._set.handle, C.byref(t.params), out.ctypes.data, out.size,
                                    C.byref(res)))
    n, n_plain = C.c_int64(0), C.c_int64(0)
    _lib.check(lib.cg_fastq_read_rows(t.ctx.handle, slot, _lib.CG_ROWS_INFO, None, 0, C.byref(n), C.byref(n_plain)))
    dst = np.empty(n.value, dtype=np.uint8)
    _lib.check(lib.cg_fastq_read_rows(t.ctx.handle, slot, _lib.CG_ROWS_INFO, dst.ctypes.data, dst.size, C.byref(n),
                                      C.byref(n_plain)))
    assert n_plain.value == len(plain.last_rows["info"])
    assert n.value <= n_plain.value + _lib.GZ_OVERHEAD * -(-n_plain.value // _lib.GZ_MEMBER)
    sizes = _members(dst.tobytes())
    assert len(sizes) > 3 and max(sizes) <= _lib.GZ_MEMBER and sum(sizes) == n_plain.value
    assert gzip.decompress(dst.tobytes()) == plain.last_rows["info"]


# ---- argument errors ---------------------------------------------------------------------------------------------------

def _einval(rc, what):
    from cutadapt_b200 import _lib

    assert rc == -1, rc                                  # CG_EINVAL
    assert what in _lib.lib().cg_last_error().decode()


def test_request_and_read_errors_leave_the_context_working():
    from cutadapt_b200 import _lib
    from cutadapt_b200.pipeline import FastqTrimmer, _row_text

    lib = _lib.lib()
    data, _ = _pair_data(51, 200)
    t = FastqTrimmer(_ads(1), **OPTS, rows=("info",))
    before = t.process_chunk(data), t.last_rows
    h = t.ctx.handle
    blob, off = _row_text(t.adapters, "info")
    out = np.empty(2 * len(data) + 4096, dtype=np.uint8)
    # a slot that holds no chunk
    slot, keep = _submit(t.ctx, data)
    idle = (slot + 2) % 4
    _einval(lib.cg_fastq_request_rows(h, idle, 0, blob, off.ctypes.data, off.size - 1, 0), "nothing was submitted")
    # an unknown kind
    _einval(lib.cg_fastq_request_rows(h, slot, 3, blob, off.ctypes.data, off.size - 1, 0), "unknown kind")
    _einval(lib.cg_fastq_read_rows(h, slot, -1, None, 0, None, None), "unknown kind")
    # the same kind twice
    _lib.check(lib.cg_fastq_request_rows(h, slot, 0, blob, off.ctypes.data, off.size - 1, 0))
    _einval(lib.cg_fastq_request_rows(h, slot, 0, blob, off.ctypes.data, off.size - 1, 0), "requested already")
    # a kind that was not requested, and rows before the collect
    _einval(lib.cg_fastq_read_rows(h, slot, 1, None, 0, None, None), "were requested")
    _einval(lib.cg_fastq_read_rows(h, slot, 0, None, 0, None, None), "has not run")
    res = _lib.cg_fastq_result()
    _lib.check(lib.cg_fastq_collect(h, slot, t._set.handle, C.byref(t.params), out.ctypes.data, out.size, C.byref(res)))
    n = C.c_int64(0)
    _lib.check(lib.cg_fastq_read_rows(h, slot, 0, None, 0, C.byref(n), None))
    assert n.value == len(before[1]["info"])
    _einval(lib.cg_fastq_read_rows(h, slot, 0, out.ctypes.data, n.value - 1, C.byref(n), None), "too small")
    # n_entries that do not match the collect's set: the collect fails, and its rows cannot be read
    slot, keep = _submit(t.ctx, data)
    _lib.check(lib.cg_fastq_request_rows(h, slot, 0, blob, off.ctypes.data, off.size - 2, 0))
    _einval(lib.cg_fastq_collect(h, slot, t._set.handle, C.byref(t.params), out.ctypes.data, out.size, C.byref(res)),
            "entries")
    _einval(lib.cg_fastq_read_rows(h, slot, 0, None, 0, None, None), "has not run or has failed")
    # the same with a paired collect, mate 2's text wrong
    tp = _paired()
    a, b = _pair_data(52, 100)
    s1, k1 = _submit(t.ctx, a)
    s2, k2 = _submit(t.ctx, b)
    _lib.check(lib.cg_fastq_request_rows(h, s2, 0, blob, off.ctypes.data, off.size - 2, 0))
    o2 = np.empty(out.size, dtype=np.uint8)
    r2 = _lib.cg_fastq_result()
    _einval(lib.cg_fastq_collect_paired(h, s1, s2, tp._set1.handle, tp._set2.handle, C.byref(tp.params1),
                                        C.byref(tp.params2), 0, out.ctypes.data, out.size, o2.ctypes.data, o2.size,
                                        C.byref(res), C.byref(r2)), "mate 2")
    # the context keeps working
    assert (t.process_chunk(data), t.last_rows) == before
    assert tp.ctx is t.ctx
    tp.process_chunk(a, b)
    assert tp.last_rows["info"][0]


@pytest.mark.parametrize("mode", ["plain", "split", "demux", "gzip_input", "interleaved"])
def test_trim_fastq_writes_row_files_with_every_output_mode(mode, tmp_path):
    """tools/trim_fastq.py: -r, --info-file and --wildcard-file next to each kind of output; the files hold the rows
    the trimmer gives for the same reads (R1's on pairs)."""
    from cutadapt_b200.pipeline import FastqTrimmer

    a, b = _pair_data(61, 300)
    inp = tmp_path / "in.fastq"
    inp.write_bytes(a)
    args = ["-a", "ilmn=AGATCGGAAGAGC", "-a", "wild=TTAGACATATNNAC", "-n", "2", "-q", "20", "-m", "15",
            "--info-file", "info.txt", "-r", "rest.txt.gz", "--wildcard-file", "wild.txt"]
    if mode == "split":
        args += ["--too-short-output", "short.fastq", "-o", "out.fastq", str(inp)]
    elif mode == "demux":
        args += ["-o", "demux-{name}.fastq", str(inp)]
    elif mode == "gzip_input":
        gz = tmp_path / "in.fastq.gz"
        gz.write_bytes(b"".join(gzip.compress(a[i:i + 8000]) for i in range(0, len(a), 8000)))
        args += ["-o", "out.fastq", str(gz)]
    elif mode == "interleaved":
        ilv = tmp_path / "in.interleaved.fastq"
        ilv.write_bytes(_interleave(a, b))
        args += ["--interleaved", "-o", "out.fastq", str(ilv)]
    else:
        args += ["-o", "out.fastq", str(inp)]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py")] + args, capture_output=True,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    import cutadapt_b200.adapters as PA

    ads = [PA.BackAdapter("AGATCGGAAGAGC", name="ilmn"), PA.BackAdapter("TTAGACATATNNAC", name="wild")]
    t = FastqTrimmer(ads, times=2, quality_cutoff=(0, 20), minimum_length=15, rows=RW.KINDS)
    t.process_chunk(a)
    assert (tmp_path / "info.txt").read_bytes() == t.last_rows["info"]
    assert gzip.decompress((tmp_path / "rest.txt.gz").read_bytes()) == t.last_rows["rest"]
    assert (tmp_path / "wild.txt").read_bytes() == t.last_rows["wildcard"]
