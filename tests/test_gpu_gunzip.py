"""
gzip input inflated on the device (cg_fastq_submit_gzip*, read_gzip_device_*chunks): for multi-member inputs of FASTQ,
FASTA and FASTQ -> FASTA, every collect gives the outputs, counters and statistics vectors of gzip.decompress plus the
host readers, at submission sizes down to less than one member; paired files with different member layouts, interleaved
input, this project's gzip output read back, a 2-million-record BGZF-style input, determinism, the FASTA re-run case,
the corruption classes (CG_EINVAL, the context still usable) and CG_EUNSUPPORTED for a member too large to inflate.
"""
import ctypes as C
import gzip
import io
import os
import sys
import zlib

import numpy as np
import pytest

from test_gunzip_host import member
from test_gzip_host import hs_gzip, synthetic_reads

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from cutadapt_b200 import _lib  # noqa: E402
from cutadapt_b200.adapters import BackAdapter, FrontAdapter  # noqa: E402
from cutadapt_b200.pipeline import (FastqTrimmer, PairedFastqTrimmer, read_fasta_chunks,  # noqa: E402
                                    read_fastq_chunks, read_gzip_device_chunks, read_gzip_device_interleaved_chunks,
                                    read_gzip_device_paired_chunks, read_interleaved_fasta_chunks,
                                    read_interleaved_fastq_chunks, read_paired_fasta_chunks, read_paired_fastq_chunks)

ADAPTER = "AGATCGGAAGAGC"
OPTS = dict(quality_cutoff=(0, 20), minimum_length=60, maximum_length=140)
SIZES = [3000, 40000, 1 << 20]          # compressed bytes per read: less than one member, a few, many


def layouts(plain: bytes, seed=0):
    """The same plain bytes as this project's members, BGZF-style zlib members of varying size, and members of
    concatenated files with header fields and zero padding."""
    rng = np.random.default_rng(seed)
    out = {"project": hs_gzip(plain)}
    parts, i = [], 0
    while i < len(plain):
        k = int(rng.integers(1000, 65280))
        parts.append(member(plain[i:i + k], flg=4, extra=b"BC\x02\0\0\0", level=int(rng.integers(1, 10))))
        i += k
    out["bgzf"] = b"".join(parts)
    cut = [0] + sorted(rng.integers(0, len(plain), 6).tolist()) + [len(plain)]
    out["concat"] = b"".join(member(plain[a:b], flg=8 | 16, name=b"f%d" % a, comment=b"c") + b"\0" * int(rng.integers(0, 3))
                             for a, b in zip(cut, cut[1:]))
    return out


def fasta_of(fq: bytes) -> bytes:
    lines = fq.split(b"\n")
    return b"".join(b">" + lines[i][1:] + b"\n" + lines[i + 1] + b"\n" for i in range(0, len(lines) - 3, 4))


def stats_equal(a, b):
    if not a.collect_statistics:
        return
    va, vb = a.statistics_vector(), b.statistics_vector()
    if isinstance(a, PairedFastqTrimmer):
        for (x, lx, kx), (y, ly, ky) in zip(va, vb):
            assert (x == y).all() and (lx, kx) == (ly, ky)
    else:
        assert (va[0] == vb[0]).all() and va[1:] == vb[1:]


def no_gzip_bytes(st, gz_out=False):
    """Counters without in_bytes_gzip (and the compressed sizes of gzip outputs, which depend on the chunking)."""
    return {k: v for k, v in st.items() if k != "in_bytes_gzip" and not (gz_out and k == "out_bytes")}


def single(make, plain, gz, size, method="process_chunks", fasta=False):
    ref, dev = make(), make()
    reader = read_fasta_chunks if fasta else read_fastq_chunks
    want = list(getattr(ref, method)(reader(io.BytesIO(plain), 1 << 16)))
    got = list(getattr(dev, method)(read_gzip_device_chunks(io.BytesIO(gz), dev, size)))
    join = (lambda xs: b"".join(xs)) if method == "process_chunks" else \
        (lambda xs: {k: b"".join(x[k] for x in xs) for k in (xs[0] if xs else {})})
    gz_out = bool(dev.gzip_outputs)
    if gz_out:
        assert gzip.decompress(join(got)) == gzip.decompress(join(want))
    else:
        assert join(got) == join(want)
    assert no_gzip_bytes(dev.statistics, gz_out) == no_gzip_bytes(ref.statistics, gz_out)
    assert dev.statistics["in_bytes_gzip"] == len(gz)
    stats_equal(ref, dev)


@pytest.mark.parametrize("layout", ["project", "bgzf", "concat"])
@pytest.mark.parametrize("size", SIZES)
def test_fastq_plain_collect(layout, size):
    plain = synthetic_reads(4000, seed=1)
    gz = layouts(plain, 1)[layout]
    single(lambda: FastqTrimmer([BackAdapter(ADAPTER, name="a")], **OPTS, collect_statistics=True), plain, gz, size)


@pytest.mark.parametrize("size", SIZES)
def test_fasta_and_fastq_to_fasta(size):
    plain = synthetic_reads(3000, seed=2)
    fa = b"# comment\n" + fasta_of(plain)
    ads = lambda: [BackAdapter(ADAPTER, name="a")]  # noqa: E731
    single(lambda: FastqTrimmer(ads(), input_format="fasta", minimum_length=60, collect_statistics=True), fa,
           layouts(fa, 2)["bgzf"], size, fasta=True)
    single(lambda: FastqTrimmer(ads(), output_format="fasta", minimum_length=60, collect_statistics=True), plain,
           layouts(plain, 3)["concat"], size)


def test_split_demux_info_and_gzip_outputs():
    plain = synthetic_reads(3000, seed=3)
    gz = layouts(plain, 4)["project"]
    kw = dict(OPTS, redirect=("too_short", "too_long", "untrimmed"), collect_statistics=True)
    single(lambda: FastqTrimmer([BackAdapter(ADAPTER, name="a")], **kw), plain, gz, 20000, "process_chunks_split")
    single(lambda: FastqTrimmer([BackAdapter(ADAPTER, name="a")], **OPTS, gzip_outputs=("output",)), plain, gz, 20000)
    ads = lambda: [BackAdapter(ADAPTER, name="a"), FrontAdapter("ACGTTGCA", name="b")]  # noqa: E731
    for method in ("process_chunk_demux", "process_chunk_info"):
        ref, dev = FastqTrimmer(ads(), **OPTS), FastqTrimmer(ads(), **OPTS)
        want = [getattr(ref, method)(c) for c in read_fastq_chunks(io.BytesIO(plain), 1 << 16)]
        got = [getattr(dev, method)(c) for c in read_gzip_device_chunks(io.BytesIO(gz), dev, 20000)]

        def joined(xs):
            if isinstance(xs[0], dict):
                return {k: b"".join(x[k] for x in xs) for k in xs[0]}
            return tuple(b"".join(x[i] for x in xs) for i in range(2))
        assert joined(got) == joined(want)
        assert no_gzip_bytes(dev.statistics) == ref.statistics


def test_paired_files_with_different_member_layouts():
    r1, r2 = synthetic_reads(3000, seed=5), synthetic_reads(3000, seed=6)
    g1, g2 = layouts(r1, 5)["project"], layouts(r2, 6)["bgzf"]
    for kw, method in ((dict(), "process_chunk"), (dict(redirect=("too_short",)), "process_chunk_split"),
                       (dict(pair_adapters=True), "process_chunk"), (dict(gzip_outputs=("output",)), "process_chunk")):
        make = lambda: PairedFastqTrimmer([BackAdapter(ADAPTER, name="a")], [BackAdapter("AGATCGGAAGAGC", name="b")],  # noqa
                                          options1=OPTS, options2=OPTS, collect_statistics=True, **kw)
        ref, dev = make(), make()
        want = [getattr(ref, method)(a, b) for a, b in read_paired_fastq_chunks(io.BytesIO(r1), io.BytesIO(r2), 1 << 16)]
        got = [getattr(dev, method)(a, b) for a, b in
               read_gzip_device_paired_chunks(io.BytesIO(g1), io.BytesIO(g2), dev, 10000)]
        # chunk boundaries differ between the readers: compare the concatenations per output and mate
        def joined(xs):
            if isinstance(xs[0], dict):
                return {k: (b"".join(x[k][0] for x in xs), b"".join(x[k][1] for x in xs)) for k in xs[0]}
            return b"".join(x[0] for x in xs), b"".join(x[1] for x in xs)
        if kw.get("gzip_outputs"):
            assert tuple(gzip.decompress(x) for x in joined(got)) == tuple(gzip.decompress(x) for x in joined(want))
        else:
            assert joined(got) == joined(want)
        gz_out = bool(kw.get("gzip_outputs"))
        assert [no_gzip_bytes(s, gz_out) for s in dev.statistics] == [no_gzip_bytes(s, gz_out) for s in ref.statistics]
        stats_equal(ref, dev)
    # FASTA pairs
    f1, f2 = fasta_of(r1), fasta_of(r2)
    ref = PairedFastqTrimmer([BackAdapter(ADAPTER)], [], input_format="fasta")
    dev = PairedFastqTrimmer([BackAdapter(ADAPTER)], [], input_format="fasta")
    want = [ref.process_chunk(a, b) for a, b in read_paired_fasta_chunks(io.BytesIO(f1), io.BytesIO(f2), 1 << 16)]
    got = [dev.process_chunk(a, b) for a, b in read_gzip_device_paired_chunks(
        io.BytesIO(hs_gzip(f1)), io.BytesIO(layouts(f2, 7)["concat"]), dev, 5000)]
    assert [b"".join(x[k] for x in got) for k in (0, 1)] == [b"".join(x[k] for x in want) for k in (0, 1)]


@pytest.mark.parametrize("fasta", [False, True])
def test_interleaved_input_and_outputs(fasta):
    r1, r2 = synthetic_reads(2000, seed=8), synthetic_reads(2000, seed=9)
    l1, l2 = r1.split(b"\n"), r2.split(b"\n")
    il = b"".join(b"\n".join(l1[i:i + 4]) + b"\n" + b"\n".join(l2[i:i + 4]) + b"\n" for i in range(0, len(l1) - 3, 4))
    if fasta:
        il = fasta_of(il)
    gz = layouts(il, 10)["bgzf"]
    fmt = dict(input_format="fasta") if fasta else dict(options1=OPTS, options2=OPTS)
    for kw in (dict(), dict(interleaved_outputs=("output",))):
        ref = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], **fmt, **kw)
        dev = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], **fmt, **kw)
        reader = read_interleaved_fasta_chunks if fasta else read_interleaved_fastq_chunks
        want = [ref.process_chunk(c) for c in reader(io.BytesIO(il), 1 << 15)]
        got = [dev.process_chunk(c) for c in read_gzip_device_interleaved_chunks(io.BytesIO(gz), dev, 7000)]
        assert [b"".join(x[k] for x in got) for k in (0, 1)] == [b"".join(x[k] for x in want) for k in (0, 1)]
        assert no_gzip_bytes(dev.statistics[0]) == ref.statistics[0]


def test_own_gzip_output_read_back_and_determinism():
    plain = synthetic_reads(5000, seed=11)
    t = FastqTrimmer([BackAdapter(ADAPTER)], **OPTS, gzip_outputs=("output",))
    gz = b"".join(t.process_chunks(read_fastq_chunks(io.BytesIO(plain), 1 << 17)))
    trimmed = gzip.decompress(gz)
    outs = []
    for _ in range(2):
        dev = FastqTrimmer([BackAdapter(ADAPTER)])
        outs.append(b"".join(dev.process_chunks(read_gzip_device_chunks(io.BytesIO(gz), dev, 30000))))
    ref = FastqTrimmer([BackAdapter(ADAPTER)])
    assert outs[0] == outs[1] == ref.process_chunk(trimmed)


def test_two_million_records_bgzf():
    rng = np.random.default_rng(12)
    n = 2_000_000
    seq = rng.choice(np.frombuffer(b"ACGT", np.uint8), (n, 50))
    plain = b"".join(b"@%d\n%s\n+\n%s\n" % (i, seq[i].tobytes(), b"I" * 50) for i in range(n))
    gz = b"".join(member(plain[i:i + 65280], flg=4, extra=b"BC\x02\0\0\0", level=1) for i in range(0, len(plain), 65280))
    ref, dev = FastqTrimmer([BackAdapter(ADAPTER)]), FastqTrimmer([BackAdapter(ADAPTER)])
    want = ref.process_chunk(plain)
    got = b"".join(dev.process_chunks(read_gzip_device_chunks(io.BytesIO(gz), dev, 64 << 20)))
    assert got == want
    assert dev.statistics["n_records"] == n


def test_fasta_output_with_rc_suffixes_needs_no_rerun():
    # FASTA records with empty names and short sequences: " rc" makes the output larger than the plain bound
    fa = b"".join(b">\n%s\n" % (b"GCTCTTCCGATCT" if i % 2 else b"A") for i in range(3000))
    ref = FastqTrimmer([BackAdapter(ADAPTER, max_errors=0)], input_format="fasta", revcomp=True)
    dev = FastqTrimmer([BackAdapter(ADAPTER, max_errors=0)], input_format="fasta", revcomp=True)
    want = b"".join(ref.process_chunks(read_fasta_chunks(io.BytesIO(fa), 1 << 20)))
    got = b"".join(dev.process_chunks(read_gzip_device_chunks(io.BytesIO(hs_gzip(fa)), dev)))
    assert got == want and got.count(b" rc") > 1000


def _submit(ctx, h, gz, final=1):
    slot, res = C.c_int32(-1), _lib.cg_gzin_result()
    rc = _lib.lib().cg_fastq_submit_gzip(ctx.handle, h, gz, len(gz), 0, final, C.byref(slot), C.byref(res))
    return rc, slot.value, res


def test_corruptions_are_einval_and_the_context_stays_usable():
    ctx = _lib.default_context()
    plain = synthetic_reads(500, seed=13)
    good = member(plain)
    bad = {                                   # each behind a good member: the error names byte len(good)
        "garbage": b"x", "method": good[:2] + b"\x07" + good[3:], "truncated": good[:-3],
        "crc": good[:-8] + bytes(4) + good[-4:], "isize": good[:-4] + bytes(4),
        "type3": member(b"abc", raw=b"\x07\0"), "stored": member(b"abc", raw=b"\x01\x03\x00\x00\x00abc"),
    }
    for name, gz in bad.items():
        h = C.c_int32(0)
        _lib.check(_lib.lib().cg_gzin_create(ctx.handle, C.byref(h)))
        rc, slot, _ = _submit(ctx, h.value, good + gz, 1)
        assert rc == _lib.CG_EINVAL and slot == -1, name
        assert "byte %d " % len(good) in _lib.lib().cg_last_error().decode(), name
        _lib.check(_lib.lib().cg_gzin_destroy(ctx.handle, h.value))
    h = C.c_int32(0)                          # zeros in front of the first member
    _lib.check(_lib.lib().cg_gzin_create(ctx.handle, C.byref(h)))
    rc, slot, _ = _submit(ctx, h.value, b"\0" + good, 1)
    assert rc == _lib.CG_EINVAL and slot == -1 and "byte 0 " in _lib.lib().cg_last_error().decode()
    _lib.check(_lib.lib().cg_gzin_destroy(ctx.handle, h.value))
    # the context still trims, and a fresh stream still inflates
    dev = FastqTrimmer([BackAdapter(ADAPTER)])
    assert b"".join(dev.process_chunks(read_gzip_device_chunks(io.BytesIO(good), dev))) == \
        FastqTrimmer([BackAdapter(ADAPTER)]).process_chunk(plain)


def test_error_offset_names_the_bad_member():
    ctx = _lib.default_context()
    a = member(b"@r\nACGT\n+\n")                # no whole record: no slot is taken
    h = C.c_int32(0)
    _lib.check(_lib.lib().cg_gzin_create(ctx.handle, C.byref(h)))
    rc, slot, res = _submit(ctx, h.value, a, 0)
    assert rc == 0 and slot == -1 and res.consumed == len(a) and res.carry_bytes == 10
    rc, _, _ = _submit(ctx, h.value, a[:-8] + bytes(8), 1)
    assert rc == _lib.CG_EINVAL
    assert "byte %d " % len(a) in _lib.lib().cg_last_error().decode()
    _lib.check(_lib.lib().cg_gzin_destroy(ctx.handle, h.value))


def test_a_member_too_large_for_one_submission_is_unsupported():
    ctx = _lib.default_context()
    c = zlib.compressobj(9, zlib.DEFLATED, -15)
    block = bytes(1 << 24)
    body = b"".join(c.compress(block) for _ in range(128)) + c.flush()      # 2 GiB of zeros
    crc = 0
    for _ in range(128):
        crc = zlib.crc32(block, crc)
    gz = b"\x1f\x8b\x08\0\0\0\0\0\0\xff" + body + crc.to_bytes(4, "little") + (1 << 31).to_bytes(4, "little")
    h = C.c_int32(0)
    _lib.check(_lib.lib().cg_gzin_create(ctx.handle, C.byref(h)))
    rc, slot, _ = _submit(ctx, h.value, gz, 1)
    assert rc == _lib.CG_EUNSUPPORTED and slot == -1
    assert "host" in _lib.lib().cg_last_error().decode()
    _lib.check(_lib.lib().cg_gzin_destroy(ctx.handle, h.value))


def test_golden_multiblock_input():
    raw = open(os.path.join(HERE, "golden", "multiblock.fastq.gz"), "rb").read()
    plain = gzip.decompress(raw)
    for size in (20, 100, 1 << 16):
        dev = FastqTrimmer([BackAdapter("TTAGACATATCTCCGTCG")])
        got = b"".join(dev.process_chunks(read_gzip_device_chunks(io.BytesIO(raw), dev, size)))
        assert got == FastqTrimmer([BackAdapter("TTAGACATATCTCCGTCG")]).process_chunk(plain)


# ---- the reference's gzip inputs (tests/golden/gzip_input_kat.json.gz, make_gzip_input_golden.py) -------------------

def _gzip_input_kat():
    import json

    return json.load(gzip.open(os.path.join(HERE, "golden", "gzip_input_kat.json.gz")))


def _kat_adapters(case):
    import cutadapt_b200.adapters as PA

    kinds = {"back": PA.BackAdapter, "front": PA.FrontAdapter, "anywhere": PA.AnywhereAdapter}
    return [kinds[kind](seq, max_errors=case["error_rate"], min_overlap=case["min_overlap"], name=name or f"a{i}")
            for i, (kind, seq, name) in enumerate(case["adapters"])]


@pytest.mark.parametrize("size", [64, 1 << 16])
def test_reference_gzip_inputs_through_the_device_reader(size):
    kat = _gzip_input_kat()
    files = {k: v.encode("latin-1") for k, v in kat["files"].items()}
    assert len(kat["cases"]) == 9
    for case in kat["cases"]:
        raw = files[case["input"]]
        fasta = case["input"].endswith(".fasta.gz")
        t = FastqTrimmer(_kat_adapters(case), input_format="fasta" if fasta else "fastq")
        chunks = read_gzip_device_chunks(io.BytesIO(raw), t, size)
        if case["info"]:
            parts = [t.process_chunk_info(c) for c in chunks]
            out, rows = b"".join(p[0] for p in parts), b"".join(p[1] for p in parts)
            want = [w.rstrip() for w in files[case["info"]].decode("latin-1").split("\n")]
            assert [g.rstrip() for g in rows.decode("latin-1").split("\n")] == want, case["name"]
        else:
            out = b"".join(t.process_chunks(chunks))
        assert out == files[case["expected"]], case["name"]
        assert t.statistics["in_bytes_gzip"] == len(raw), case["name"]


# ---- tools/trim_fastq.py: which inputs the device inflates ---------------------------------------------------------

def _tool(tmp_path, inp, out_name, *extra):
    import json
    import subprocess

    out = tmp_path / out_name
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), "-a", ADAPTER, "-q", "20", "-m", "20",
                        *extra, "-o", str(out), str(inp)], check=True, capture_output=True, text=True)
    return out.read_bytes(), json.loads(p.stderr.strip().splitlines()[-1])


def test_tool_routes_multi_member_inputs_to_the_device(tmp_path):
    plain = synthetic_reads(30000, seed=15)
    (tmp_path / "in.fastq").write_bytes(plain)
    multi = layouts(plain, 15)["bgzf"]
    (tmp_path / "multi.fastq.gz").write_bytes(multi)
    single = gzip.compress(plain, 6)
    assert len(single) > 1 << 20                             # its only member ends past the first MiB
    (tmp_path / "single.fastq.gz").write_bytes(single)
    want, st = _tool(tmp_path, tmp_path / "in.fastq", "plain.fastq")
    assert "in_bytes_gzip" not in st
    got, st_multi = _tool(tmp_path, tmp_path / "multi.fastq.gz", "multi.fastq")
    assert got == want and st_multi["in_bytes_gzip"] == len(multi)
    got, st_single = _tool(tmp_path, tmp_path / "single.fastq.gz", "single.fastq")
    assert got == want and "in_bytes_gzip" not in st_single  # the host path
    assert {k: v for k, v in st_multi.items() if k != "in_bytes_gzip"} == st == st_single
    # paired: two multi-member files on the device, and the same files interleaved
    r2 = synthetic_reads(30000, seed=16)
    (tmp_path / "in2.fastq").write_bytes(r2)
    (tmp_path / "multi2.fastq.gz").write_bytes(hs_gzip(r2))
    import subprocess

    def paired(a, b, o1, o2):
        subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), "-a", ADAPTER, "-A", ADAPTER,
                        "-m", "20", "-o", str(tmp_path / o1), "-p", str(tmp_path / o2), str(a), str(b)],
                       check=True, capture_output=True)
        return (tmp_path / o1).read_bytes(), (tmp_path / o2).read_bytes()
    assert paired(tmp_path / "multi.fastq.gz", tmp_path / "multi2.fastq.gz", "g1.fq", "g2.fq") == \
        paired(tmp_path / "in.fastq", tmp_path / "in2.fastq", "p1.fq", "p2.fq")


def test_rows_larger_than_their_estimate_retry_a_device_chunk():
    # one-base reads with a long adapter name: the info rows outgrow per_read * 2 * n_bytes + 1 MiB
    fq = b"".join(b"@\nA\n+\nI\n" for _ in range(400000))
    name = "N" * 40
    ref = FastqTrimmer([BackAdapter("A", name=name, min_overlap=1)])
    dev = FastqTrimmer([BackAdapter("A", name=name, min_overlap=1)])
    want = ref.process_chunk_info(fq)
    got = [dev.process_chunk_info(c) for c in read_gzip_device_chunks(io.BytesIO(hs_gzip(fq)), dev, 1 << 24)]
    assert len(got) == 1 and got[0] == want
    assert len(want[1]) > 4 * len(fq) + (1 << 20)
