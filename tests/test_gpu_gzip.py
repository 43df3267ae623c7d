"""
gzip outputs of the device FASTQ path (cg_fastq_params.gzip_outputs): every compressed output decompresses to the plain
call's bytes, equals the host build of the encoder (tests/hostsim) byte for byte, and leaves counters and statistics as
they are; the mask errors, the buffer bound, many members per output, determinism, the ratio on the bench reads, and
tools/trim_fastq.py with .gz names.
"""
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gzip_host import hs_gzip, members, synthetic_reads, zlib1

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from cutadapt_b200 import _lib  # noqa: E402
from cutadapt_b200.adapters import BackAdapter, FrontAdapter  # noqa: E402
from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer  # noqa: E402

ADAPTER = "AGATCGGAAGAGC"


def reads(n, seed=0):
    return synthetic_reads(n, seed=seed)


def same_member_bytes(z, plain):
    """z decompresses to plain and is what the host build writes for it."""
    assert gzip.decompress(z) == plain if z else plain == b""
    assert z == hs_gzip(plain)


def counters(st):
    return {k: v for k, v in st.items() if k not in ("out_bytes", "out_bytes_plain")}


OPTS = dict(quality_cutoff=(0, 20), minimum_length=60, maximum_length=140)
SPLIT_NAMES = ("output", "too_short", "too_long", "untrimmed")


@pytest.mark.parametrize("names", [("output",), ("too_short",), ("too_long",), ("untrimmed",), SPLIT_NAMES,
                                   ("output", "too_long")])
def test_single_end_split_each_mask(names):
    data = reads(3000, seed=1)
    kw = dict(OPTS, redirect=("too_short", "too_long", "untrimmed"), redirect_formats={"too_long": "fasta"},
              collect_statistics=True)
    plain = FastqTrimmer([BackAdapter(ADAPTER, name="a")], **kw)
    gz = FastqTrimmer([BackAdapter(ADAPTER, name="a")], **kw, gzip_outputs=names)
    want, got = plain.process_chunk_split(data), gz.process_chunk_split(data)
    assert set(want) == set(got)
    for name in want:
        if name in names:
            same_member_bytes(got[name], want[name])
        else:
            assert got[name] == want[name]
    assert counters(gz.statistics) == counters(plain.statistics)
    assert gz.statistics["out_bytes_plain"] == plain.statistics["out_bytes"]
    assert gz.statistics["out_bytes"] == sum(len(v) for v in got.values())
    v1, v2 = plain.statistics_vector()[0], gz.statistics_vector()[0]
    assert (v1 == v2).all()


def test_plain_collect_trim_chunk_info_and_demux():
    data = reads(2500, seed=2)
    ads = lambda: [BackAdapter(ADAPTER, name="a"), FrontAdapter("ACGTTGCA", name="b")]  # noqa: E731
    plain = FastqTrimmer(ads(), **OPTS)
    gz = FastqTrimmer(ads(), **OPTS, gzip_outputs=("output",))
    same_member_bytes(gz.process_chunk(data), plain.process_chunk(data))
    out_p, rows_p = plain.process_chunk_info(data)
    out_g, rows_g = gz.process_chunk_info(data)
    same_member_bytes(out_g, out_p)
    assert rows_g == rows_p                                  # row outputs stay plain
    out_p, rows_p = plain.process_chunk_rest(data)
    out_g, rows_g = gz.process_chunk_rest(data)
    same_member_bytes(out_g, out_p)
    assert rows_g == rows_p
    want, got = plain.process_chunk_demux(data), gz.process_chunk_demux(data)
    assert set(want) == set(got)
    for name in want:
        same_member_bytes(got[name], want[name])
    assert counters(gz.statistics) == counters(plain.statistics)
    # a chunk that every record leaves: outputs are 0 bytes, not empty members
    none = FastqTrimmer(None, minimum_length=10_000, gzip_outputs=("output",))
    assert none.process_chunk(data) == b""
    assert none.process_chunk(b"") == b""
    assert none.statistics["out_bytes_plain"] == 0


def _pairs(n, seed):
    d1, d2 = reads(n, seed), reads(n, seed + 100)
    recs1, recs2 = d1.split(b"\n"), d2.split(b"\n")
    # mate names must match for interleaving: give R2 R1's names
    for i in range(0, len(recs1) - 1, 4):
        recs2[i] = recs1[i]
    d2 = b"\n".join(recs2)
    il = b"".join(b"\n".join(recs1[i:i + 4]) + b"\n" + b"\n".join(recs2[i:i + 4]) + b"\n"
                  for i in range(0, len(recs1) - 1, 4))
    return d1, d2, il


@pytest.mark.parametrize("g1,g2", [(("output",), ("output",)), (("output",), ()), ((), ("too_short",)),
                                   (SPLIT_NAMES, SPLIT_NAMES)])
def test_paired_split_and_plain(g1, g2):
    d1, d2, _ = _pairs(1500, 3)
    kw = dict(options1=OPTS, options2=OPTS, redirect=("too_short", "untrimmed"), collect_statistics=True)
    plain = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], **kw)
    gz = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], **kw, gzip_outputs=g1, gzip_outputs2=g2)
    want, got = plain.process_chunk_split(d1, d2), gz.process_chunk_split(d1, d2)
    for name in want:
        for k, names in ((0, g1), (1, g2)):
            if name in names:
                same_member_bytes(got[name][k], want[name][k])
            else:
                assert got[name][k] == want[name][k]
    for a, b in zip(plain.statistics, gz.statistics):
        assert counters(a) == counters(b)
    for (v1, _, _), (v2, _, _) in zip(plain.statistics_vector(), gz.statistics_vector()):
        assert (v1 == v2).all()
    plain2 = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], options1=OPTS, options2=OPTS)
    gz2 = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], options1=OPTS, options2=OPTS,
                             gzip_outputs=g1, gzip_outputs2=g2)
    for (w, g, names) in zip(plain2.process_chunk(d1, d2), gz2.process_chunk(d1, d2), (g1, g2)):
        if "output" in names:
            same_member_bytes(g, w)
        else:
            assert g == w


def test_interleaved_outputs_and_pair_demux():
    d1, d2, il = _pairs(1500, 4)
    kw = dict(options1=OPTS, options2=OPTS, redirect=("too_short",), interleaved_outputs=("output",))
    plain = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], **kw)
    gz = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], **kw,
                            gzip_outputs=("output", "too_short"), gzip_outputs2=("output",))
    for args in ((d1, d2), (il,)):
        want, got = plain.process_chunk_split(*args), gz.process_chunk_split(*args)
        same_member_bytes(got["output"][0], want["output"][0])
        assert got["output"][1] == want["output"][1] == b""
        same_member_bytes(got["too_short"][0], want["too_short"][0])
        assert got["too_short"][1] == want["too_short"][1]
    bad = PairedFastqTrimmer([BackAdapter(ADAPTER)], [BackAdapter(ADAPTER)], **kw, gzip_outputs=("output",),
                             gzip_outputs2=())
    with pytest.raises(ValueError, match="alike"):
        bad.process_chunk_split(d1, d2)
    ads = lambda: [BackAdapter(ADAPTER, name="x"), FrontAdapter("ACGTTGCA", name="y")]  # noqa: E731
    p = PairedFastqTrimmer(ads(), ads(), options1=OPTS, options2=OPTS)
    g = PairedFastqTrimmer(ads(), ads(), options1=OPTS, options2=OPTS, gzip_outputs=("output",))
    want, got = p.process_chunk_demux(d1, d2, combinatorial=True), g.process_chunk_demux(d1, d2, combinatorial=True)
    for key in want:
        for k in (0, 1):
            same_member_bytes(got[key][k], want[key][k])


def test_mask_errors_and_the_buffer_bound():
    with pytest.raises(ValueError):
        FastqTrimmer(None, gzip_outputs=("nope",))
    t = FastqTrimmer(None)
    t.params.gzip_outputs = 16
    with pytest.raises(ValueError, match="gzip_outputs"):
        t.process_chunk(reads(10))
    # random sequences compress to stored members: the bound is then reached exactly and still fits
    rng = np.random.default_rng(9)
    n = 3000
    seq = rng.choice(np.frombuffer(b"ACGT", np.uint8), (n, 150))
    qual = rng.integers(33, 75, (n, 150), dtype=np.uint8)
    data = b"".join(b"@r%d\n" % i + seq[i].tobytes() + b"\n+\n" + qual[i].tobytes() + b"\n" for i in range(n))
    t = FastqTrimmer(None, gzip_outputs=("output",))
    out = t.process_chunk(data)
    assert gzip.decompress(out) == data
    # the "buffer too small" contract: the compressed size is reported, a retry with it succeeds
    tr = FastqTrimmer(None, gzip_outputs=("output",))
    slot, size, _ = tr._submit(data)
    buf = np.empty(100, dtype=np.uint8)
    res = _lib.cg_fastq_result()
    import ctypes as C

    rc = _lib.lib().cg_fastq_collect(tr.ctx.handle, slot, None, C.byref(tr.params), buf.ctypes.data, buf.size,
                                     C.byref(res))
    assert rc != 0 and res.out_bytes == len(out) and res.out_bytes_plain == len(data) and res.n_written == n
    slot, _, _ = tr._submit(data)
    buf = np.empty(res.out_bytes, dtype=np.uint8)
    assert _lib.lib().cg_fastq_collect(tr.ctx.handle, slot, None, C.byref(tr.params), buf.ctypes.data, buf.size,
                                       C.byref(res)) == 0
    assert buf.tobytes() == out


@pytest.mark.parametrize("g1,g2", [(("output",), ("output",)), ((), ("output",))])
def test_pair_adapters(g1, g2):
    d1, d2, _ = _pairs(1500, 5)
    ads1 = [BackAdapter(ADAPTER, name="p"), BackAdapter("ACGTTGCA", name="q")]
    ads2 = [BackAdapter("TTGCATTGCA", name="p"), BackAdapter(ADAPTER, name="q")]
    plain = PairedFastqTrimmer(ads1, ads2, OPTS, OPTS, pair_adapters=True, collect_statistics=True)
    gz = PairedFastqTrimmer(ads1, ads2, OPTS, OPTS, pair_adapters=True, collect_statistics=True, gzip_outputs=g1,
                            gzip_outputs2=g2)
    for w, g, names in zip(plain.process_chunk(d1, d2), gz.process_chunk(d1, d2), (g1, g2)):
        if names:
            same_member_bytes(g, w)
        else:
            assert g == w
    for a, b in zip(plain.statistics, gz.statistics):
        assert counters(a) == counters(b)
    for (v1, _, _), (v2, _, _) in zip(plain.statistics_vector(), gz.statistics_vector()):
        assert (v1 == v2).all()


def test_two_million_records_in_one_chunk():
    from cutadapt_b200.synth import make_read_tensor

    n = 2_000_000
    seq, qual = make_read_tensor(n, config=2, device="cpu", with_qualities=True, seed=11)
    rec = np.empty((n, 1 + 15 + 1 + 150 + 3 + 150 + 1), dtype=np.uint8)
    rec[:, 0] = ord("@")
    idx = np.arange(n)
    rec[:, 1:6] = np.frombuffer(b"SIM2:", dtype=np.uint8)
    for d in range(10):
        rec[:, 15 - d] = 48 + (idx // 10 ** d) % 10
    rec[:, 16] = 10
    rec[:, 17:167] = seq.numpy()
    rec[:, 167:170] = np.frombuffer(b"\n+\n", dtype=np.uint8)
    rec[:, 170:320] = qual.numpy()
    rec[:, 320] = 10
    data = rec.tobytes()
    del rec, seq, qual
    want = FastqTrimmer([BackAdapter(ADAPTER)], **OPTS).process_chunk(data)
    t = FastqTrimmer([BackAdapter(ADAPTER)], **OPTS, gzip_outputs=("output",))
    got = t.process_chunk(data)
    assert len(want) > 300 * 65280
    assert t.statistics["out_bytes_plain"] == len(want) and t.statistics["out_bytes"] == len(got)
    same_member_bytes(got, want)


def test_many_members_slots_in_flight_alternating_and_deterministic():
    data = reads(200_000, seed=6)
    chunks = [data[: len(data) // 2], data[len(data) // 2:]]
    cut = chunks[0].rfind(b"\n@SIM2:") + 1
    chunks = [data[:cut], data[cut:]]
    gz = FastqTrimmer([BackAdapter(ADAPTER)], gzip_outputs=("output",))
    plain = FastqTrimmer([BackAdapter(ADAPTER)])
    outs = list(gz.process_chunks(chunks))
    wants = list(plain.process_chunks(chunks))
    for o, w in zip(outs, wants):
        assert len(members(o)) == (len(w) + 65279) // 65280 > 50
        same_member_bytes(o, w)
    assert list(gz.process_chunks(chunks)) == outs                     # the same bytes again
    mixed = []
    for k in range(4):                                                 # gzip and plain calls on one context
        t = gz if k % 2 == 0 else plain
        mixed.append(t.process_chunk(chunks[k % 2]))
    assert mixed[0] == outs[0] and mixed[2] == outs[0] and mixed[1] == wants[1]
    total = b"".join(wants)
    assert sum(len(o) for o in outs) <= 1.15 * zlib1(total)


def test_tool_end_to_end(tmp_path):
    d1, d2, _ = _pairs(2000, 7)
    (tmp_path / "in.1.fastq.gz").write_bytes(gzip.compress(d1))
    (tmp_path / "in.2.fastq").write_bytes(d2)
    tool = [sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py")]

    def run(*argv):
        subprocess.run(tool + [str(a) for a in argv], check=True, capture_output=True)

    run("-a", ADAPTER, "-A", ADAPTER, "-m", 50, "-o", tmp_path / "gz.1.fastq.gz", "-p", tmp_path / "gz.2.fastq",
        "--too-short-output", tmp_path / "s.1.fastq.gz", "--too-short-paired-output", tmp_path / "s.2.fastq.gz",
        tmp_path / "in.1.fastq.gz", tmp_path / "in.2.fastq")
    (tmp_path / "in.1.fastq").write_bytes(d1)
    run("-a", ADAPTER, "-A", ADAPTER, "-m", 50, "-o", tmp_path / "p.1.fastq", "-p", tmp_path / "p.2.fastq",
        "--too-short-output", tmp_path / "ps.1.fastq", "--too-short-paired-output", tmp_path / "ps.2.fastq",
        tmp_path / "in.1.fastq", tmp_path / "in.2.fastq")
    assert gzip.decompress((tmp_path / "gz.1.fastq.gz").read_bytes()) == (tmp_path / "p.1.fastq").read_bytes()
    assert (tmp_path / "gz.2.fastq").read_bytes() == (tmp_path / "p.2.fastq").read_bytes()
    assert gzip.decompress((tmp_path / "s.2.fastq.gz").read_bytes()) == (tmp_path / "ps.2.fastq").read_bytes()
    run("-g", "x=^ACGTTGCA", "-g", "y=^TTGCATTGCA", "-o", str(tmp_path / "{name}.fastq.gz"), tmp_path / "in.1.fastq")
    run("-g", "x=^ACGTTGCA", "-g", "y=^TTGCATTGCA", "-o", str(tmp_path / "{name}.fastq"), tmp_path / "in.1.fastq")
    for name in ("x", "y", "unknown"):
        gzp, pp = tmp_path / f"{name}.fastq.gz", tmp_path / f"{name}.fastq"
        assert gzp.exists() == pp.exists()
        if pp.exists():
            assert gzip.decompress(gzp.read_bytes()) == pp.read_bytes()
