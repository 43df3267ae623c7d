"""
GPU tests (-m gpu) of interleaved paired-end data on the device (cg_fastq_submit_interleaved,
cg_fastq_collect_paired_interleaved; --interleaved): the reference's known answers (tests/golden/interleaved_kat.json.gz),
interleaved input against the same pairs as two chunks on every paired collect, interleaved outputs against a host
interleave of the two-file outputs, the errors, a large chunk, an empty one and slots shared with two-file pairs.
"""
import ctypes as C
import itertools
import os
import random
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cutadapt_b200.adapters as PA  # noqa: E402
import fasta_oracle as FO  # noqa: E402
import interleaved_oracle as IO  # noqa: E402
from cutadapt_b200 import _lib  # noqa: E402
from cutadapt_b200.pipeline import PairedFastqTrimmer  # noqa: E402
from oracle import oracle  # noqa: E402
from test_gpu_fastq import synthetic_fastq  # noqa: E402
from test_interleaved_host import oracle_case  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUTPUTS = ("output", "too_short", "too_long", "untrimmed")


def random_pairs(n, seed, fasta=False):
    """(R1 chunk, R2 chunk, interleaved chunk) of n seeded random pairs whose mates have matching names."""
    recs = [oracle.parse_fastq(synthetic_fastq(n, seed + k)) for k in (0, 1)]
    mates = ([], [])
    for i, pair in enumerate(zip(*recs)):
        for k, (_, seq, qual) in enumerate(pair):
            name = f"p{seed}_{i}/{k + 1} c{k}"
            mates[k].append(f">{name}\n{seq}\n" if fasta else f"@{name}\n{seq}\n+\n{qual}\n")
    return "".join(mates[0]).encode(), "".join(mates[1]).encode(), "".join(a + b for a, b in zip(*mates)).encode()


def adapters(tag, k=2):
    seqs = ("AGATCGGAAGAGC", "TTAGACATATCTCC", "CAGTGGAGTA")
    return [PA.BackAdapter(seqs[(i + tag) % 3], max_errors=0.1, name=f"{tag}_{i}") for i in range(k)]


def stats_of(t):
    return [(v.tolist(), m, k) for v, m, k in t.statistics_vector()] if t.collect_statistics else None


# ---- the reference's answers ------------------------------------------------------------------------------------------

def test_kat_cases_on_the_device():
    for c in IO.interleaved_kat()["cases"]:
        o = c["options"]
        data = [IO.kat_file(k) for k in c["inputs"]]
        fmt = "fasta" if data[0][:1] in (b">", b"#") else "fastq"
        kw1, kw2 = IO.kat_trimmer_kwargs(o)
        t = PairedFastqTrimmer(FO.kat_adapters(o, "specs1"), FO.kat_adapters(o, "specs2"), kw1, kw2, input_format=fmt,
                               redirect=o.get("redirect", ()), interleaved_outputs=IO.kat_interleaved_outputs(c))
        got = t.process_chunk_split(data[0], data[1] if len(data) == 2 else None)
        for name, files in c["expected"].items():
            want = tuple(IO.kat_file(k) for k in files) + ((b"",) if len(files) == 1 else ())
            assert got[name] == want, (c["name"], name)
        _, c1, c2 = oracle_case(c)
        for st, cc in zip(t.statistics, (c1, c2)):
            for k, v in cc.items():
                assert st[k] == v, (c["name"], k)


def test_kat_cases_through_the_tool(tmp_path):
    kat = IO.interleaved_kat()
    picked = [c for c in kat["cases"] if not c["name"].startswith("separate")] + \
        [c for c in kat["cases"] if c["name"].startswith("separate")][::7]
    for c in picked:
        ins = []
        for k in c["inputs"]:
            p = tmp_path / k.replace("/", "_")
            p.write_bytes(IO.kat_file(k))
            ins.append(str(p))
        if "argv" in c:
            argv = c["argv"]
        else:
            argv = ["-q", "20", "-a", "TTAGACATAT", "-A", "CAGTGGAGTA", "-m", "14", "-M", "90", "--interleaved"]
            if c["name"] == "interleaved_untrimmed_output":
                argv = ["--interleaved", "-a", "XXXX", "--untrimmed-output", str(tmp_path / "u.fastq")]
        outs = {"output": [str(tmp_path / "o1.out"), str(tmp_path / "o2.out")]}
        argv = argv + ["-o", outs["output"][0]]
        if len(c["expected"].get("output", [None, None])) == 2:
            argv += ["-p", outs["output"][1]]
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py")] + argv + ins,
                           capture_output=True, text=True)
        assert r.returncode == 0, (c["name"], r.stderr)
        for name, files in c["expected"].items():
            paths = outs["output"] if name == "output" else [str(tmp_path / "u.fastq")]
            for path, k in zip(paths, files):
                assert open(path, "rb").read() == IO.kat_file(k), (c["name"], name)


# ---- input equivalence: one interleaved chunk == the same pairs as two chunks ---------------------------------------

CONFIGS = {
    "plain": dict(),
    "statistics": dict(collect_statistics=True),
    "cut_qual": dict(options1=dict(cut=[3, -2], quality_cutoff=(5, 20)), options2=dict(cut=[4], quality_cutoff=(0, 15)),
                     collect_statistics=True),
    "pair_filter_both": dict(options1=dict(minimum_length=30), options2=dict(minimum_length=40), pair_filter="both"),
    "pair_filter_first": dict(options1=dict(maximum_length=100, discard_untrimmed=True),
                              options2=dict(maximum_length=100, discard_untrimmed=True), pair_filter="first"),
    "pair_filter_any": dict(options1=dict(minimum_length=20, max_n=2), options2=dict(minimum_length=25)),
    "fasta": dict(fasta=True, options1=dict(minimum_length=10), options2=dict(minimum_length=10), collect_statistics=True),
    "fastq_to_fasta": dict(output_format="fasta", options1=dict(minimum_length=10), options2=dict(maximum_length=120)),
    "pair_adapters": dict(pair_adapters=True, collect_statistics=True),
    "one_mate_adapters": dict(adapters2=False, options1=dict(discard_untrimmed=True), options2=dict(discard_untrimmed=True)),
}
for _r in range(1, 8):
    _names = tuple(n for i, n in enumerate(("too_short", "too_long", "untrimmed")) if _r >> i & 1)
    CONFIGS[f"split_{'_'.join(_names)}"] = dict(
        redirect=_names, options1=dict(minimum_length=40, maximum_length=140), options2=dict(minimum_length=30,
                                                                                               maximum_length=150),
        collect_statistics=True, method="split")


def _trimmer(cfg, interleaved_outputs=()):
    a1 = adapters(0)
    a2 = adapters(1) if cfg.get("adapters2", True) else None
    fmt = "fasta" if cfg.get("fasta") else "fastq"
    return PairedFastqTrimmer(a1, a2, cfg.get("options1", {}), cfg.get("options2", {}), cfg.get("pair_filter", "any"),
                              pair_adapters=cfg.get("pair_adapters", False), input_format=fmt,
                              output_format=cfg.get("output_format"), collect_statistics=cfg.get("collect_statistics", False),
                              redirect=cfg.get("redirect", ()), interleaved_outputs=interleaved_outputs)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_interleaved_input_equals_two_chunks(name):
    cfg = CONFIGS[name]
    d1, d2, dil = random_pairs(700, 11, fasta=cfg.get("fasta", False))
    results = []
    for chunks in ((d1, d2), (dil, None)):
        t = _trimmer(cfg)
        if cfg.get("method") == "split":
            got = t.process_chunk_split(*chunks)
        else:
            got = t.process_chunk(*chunks)
        results.append((got, [dict(s) for s in t.statistics], stats_of(t)))
    assert results[0] == results[1]
    assert results[0][1][0]["n_records"] == 700


@pytest.mark.parametrize("combinatorial", [False, True])
def test_interleaved_input_equals_two_chunks_demux(combinatorial):
    d1, d2, dil = random_pairs(600, 5)
    got = []
    for chunks in ((d1, d2), (dil, None)):
        t = _trimmer(dict(collect_statistics=True))
        got.append((t.process_chunk_demux(*chunks, combinatorial=combinatorial), [dict(s) for s in t.statistics],
                    stats_of(t)))
    assert got[0] == got[1]
    assert sum(len(a) for a, _ in got[0][0].values()) > 0


# ---- output equivalence: every set of interleaved destinations == a host interleave of the two-file outputs ----------

@pytest.mark.parametrize("subset", [s for k in range(len(OUTPUTS) + 1) for s in itertools.combinations(OUTPUTS, k)],
                         ids=lambda s: "-".join(s) or "none")
@pytest.mark.parametrize("interleaved_input", [False, True])
def test_interleaved_outputs_equal_a_host_interleave(subset, interleaved_input):
    d1, d2, dil = random_pairs(800, 23)
    cfg = dict(redirect=("too_short", "too_long", "untrimmed"), options1=dict(minimum_length=40, maximum_length=140),
               options2=dict(minimum_length=30, maximum_length=150))
    formats = {"too_short": "fasta", "untrimmed": "fasta"}
    chunks = (dil, None) if interleaved_input else (d1, d2)
    ref = PairedFastqTrimmer(adapters(0), adapters(1), cfg["options1"], cfg["options2"], redirect=cfg["redirect"],
                             collect_statistics=True, redirect_formats=formats)
    t = PairedFastqTrimmer(adapters(0), adapters(1), cfg["options1"], cfg["options2"], redirect=cfg["redirect"],
                           collect_statistics=True, redirect_formats=formats, interleaved_outputs=subset)
    want, got = ref.process_chunk_split(*chunks), t.process_chunk_split(*chunks)
    for name in OUTPUTS:
        fmt = formats.get(name, "fastq")
        a, b = want[name]
        assert got[name] == ((IO.interleave(a, b, fmt), b"") if name in subset else (a, b)), name
    assert sum(len(a) for a, _ in got.values()) > 0 and all(want[n][0] for n in OUTPUTS)
    st_want = [dict(s) for s in ref.statistics]
    st_got = [dict(s) for s in t.statistics]
    if subset:
        # res1.out_bytes holds both mates of the interleaved outputs, res2.out_bytes the rest
        total = sum(len(a) + len(b) for a, b in want.values())
        assert st_got[0]["out_bytes"] + st_got[1]["out_bytes"] == total
    for s in st_want + st_got:
        s.pop("out_bytes")
    assert st_got == st_want
    assert stats_of(t) == stats_of(ref)


def _raw_collect_interleaved(t, chunk, cap1, cap2, ilv):
    """cg_fastq_submit_interleaved + cg_fastq_collect_paired_interleaved with given capacities: (rc, res1, res2)."""
    buf = np.frombuffer(chunk, dtype=np.uint8)
    s1, s2 = C.c_int32(-1), C.c_int32(-1)
    lib = _lib.lib()
    _lib.check(lib.cg_fastq_submit_interleaved(t.ctx.handle, buf.ctypes.data, buf.size, 0, C.byref(s1), C.byref(s2)))
    out1, out2 = np.empty(max(cap1, 1), dtype=np.uint8), np.empty(max(cap2, 1), dtype=np.uint8)
    r1, r2 = _lib.cg_fastq_result(), _lib.cg_fastq_result()
    seg1, seg2 = np.zeros(5, dtype=np.int64), np.zeros(5, dtype=np.int64)
    rc = lib.cg_fastq_collect_paired_interleaved(
        t.ctx.handle, s1.value, s2.value, t._set1.handle, t._set2.handle, C.byref(t.params1), C.byref(t.params2), 0, 0, 0,
        ilv, out1.ctypes.data, cap1, out2.ctypes.data, cap2, C.byref(r1), C.byref(r2), seg1.ctypes.data, seg2.ctypes.data)
    return rc, r1, r2


def test_too_small_output_reports_out_bytes_and_adds_no_statistics():
    _, _, dil = random_pairs(300, 3)
    t = _trimmer(dict(collect_statistics=True))
    before = stats_of(t)
    want = t.process_chunk(dil)
    after = stats_of(t)
    for cap1, cap2, ilv in ((10, 1 << 20, 8), (len(want[0]) - 1, 1 << 20, 0), (1 << 20, len(want[1]) - 1, 0)):
        rc, r1, r2 = _raw_collect_interleaved(t, dil, cap1, cap2, ilv)
        assert rc != 0 and "too small" in _lib.lib().cg_last_error().decode()
        if ilv:
            assert r1.out_bytes == len(want[0]) + len(want[1]) and r2.out_bytes == 0
        else:
            assert (r1.out_bytes, r2.out_bytes) == (len(want[0]), len(want[1]))
        assert stats_of(t) == after
    assert after != before


# ---- errors ------------------------------------------------------------------------------------------------------------

def test_errors_name_what_was_found():
    d1, d2, dil = random_pairs(50, 7)
    recs = IO.records(dil, "fastq")
    t = _trimmer(dict())
    with pytest.raises(ValueError, match="Interleaved input file incomplete"):
        t.process_chunk(b"".join(recs[:-1]))
    # the first improper pair is named by its record numbers
    bad = list(recs)
    bad[21] = bad[21].replace(b"/2 c1", b"x/2 c1", 1)
    bad[33] = bad[33].replace(b"/2 c1", b"y/2 c1", 1)
    with pytest.raises(ValueError, match="improperly paired: records 20 and 21 "):
        t.process_chunk(b"".join(bad))
    # a FASTQ format error names the record of the interleaved chunk
    for k in (13, 14):
        bad = list(recs)
        bad[k] = bad[k].replace(b"\n+", b"\n-", 1)
        with pytest.raises(ValueError, match=f"FASTQ format error in record {k}:"):
            t.process_chunk(b"".join(bad))
    # FASTA: format errors name lines of the interleaved chunk
    f1, f2, fil = random_pairs(4, 8, fasta=True)
    tf = _trimmer(dict(fasta=True))
    lines = fil.split(b"\n")
    with pytest.raises(ValueError, match="FASTA format error in line 4:"):
        tf.process_chunk(b"\n".join(lines[:3] + [b"#late"] + lines[3:]))
    # the slots of an interleaved submission belong together
    buf = np.frombuffer(dil, dtype=np.uint8)
    s1, s2 = C.c_int32(-1), C.c_int32(-1)
    lib = _lib.lib()
    _lib.check(lib.cg_fastq_submit_interleaved(t.ctx.handle, buf.ctypes.data, buf.size, 0, C.byref(s1), C.byref(s2)))
    res = _lib.cg_fastq_result()
    out = np.empty(len(dil) * 2, dtype=np.uint8)
    assert lib.cg_fastq_collect(t.ctx.handle, s1.value, t._set1.handle, C.byref(t.params1), out.ctypes.data, out.size,
                                C.byref(res)) != 0
    r2 = _lib.cg_fastq_result()
    assert lib.cg_fastq_collect_paired(t.ctx.handle, s2.value, s1.value, t._set1.handle, t._set2.handle,
                                       C.byref(t.params1), C.byref(t.params2), 0, out.ctypes.data, out.size,
                                       out.ctypes.data, out.size, C.byref(res), C.byref(r2)) != 0
    out2 = np.empty(len(dil) * 2, dtype=np.uint8)
    _lib.check(lib.cg_fastq_collect_paired(t.ctx.handle, s1.value, s2.value, t._set1.handle, t._set2.handle,
                                           C.byref(t.params1), C.byref(t.params2), 0, out.ctypes.data, out.size,
                                           out2.ctypes.data, out2.size, C.byref(res), C.byref(r2)))
    assert res.n_records == 50


def test_refused_combinations():
    with pytest.raises(ValueError, match="interleaved outputs.*pair-adapters"):
        PairedFastqTrimmer(adapters(0), adapters(1), pair_adapters=True, interleaved_outputs=("output",))
    t = _trimmer(dict(), interleaved_outputs=("output",))
    _, _, dil = random_pairs(10, 1)
    with pytest.raises(ValueError, match="interleaved outputs.*demultiplexing"):
        t.process_chunk_demux(dil)
    with pytest.raises(ValueError, match="unknown output"):
        _trimmer(dict(), interleaved_outputs=("main",))


# ---- scale and slots ---------------------------------------------------------------------------------------------------

def test_two_million_pairs_in_one_chunk():
    rng = random.Random(2)
    n = 2_000_000
    seqs = ["".join(rng.choice("ACGT") for _ in range(58 + k % 7)) + "AGATCGGAAGAGC" * (k % 2) for k in range(64)]
    m1 = [b"@q%d/1\n%s\n+\n%s\n" % (i, seqs[i % 64].encode(), b"I" * len(seqs[i % 64])) for i in range(n)]
    m2 = [b"@q%d/2\n%s\n+\n%s\n" % (i, seqs[(i * 7) % 64].encode(), b"I" * len(seqs[(i * 7) % 64])) for i in range(n)]
    d1, d2 = b"".join(m1), b"".join(m2)
    dil = b"".join(x for pair in zip(m1, m2) for x in pair)
    del m1, m2
    opts = dict(minimum_length=61)
    a = PairedFastqTrimmer(adapters(0), adapters(1), opts, opts).process_chunk(d1, d2)
    b = PairedFastqTrimmer(adapters(0), adapters(1), opts, opts).process_chunk(dil)
    assert a == b and 0 < len(a[0]) < len(d1)


def test_empty_chunk():
    t = _trimmer(dict(collect_statistics=True), interleaved_outputs=("output",))
    assert t.process_chunk(b"") == (b"", b"")
    assert t.process_chunk_split(b"")["output"] == (b"", b"")
    assert t.statistics[0]["n_records"] == 0


def test_one_pair_in_flight_alternating_interleaved_and_two_file_chunks():
    items, want = [], []
    ref = _trimmer(dict(redirect=("too_short",), options1=dict(minimum_length=50), options2=dict(minimum_length=50),
                        collect_statistics=True))
    for k in range(9):
        d1, d2, dil = random_pairs(100 + 37 * k, 100 + k)
        items.append((d1, d2) if k % 3 == 1 else dil)
        want.append(ref.process_chunk_split(d1, d2))
    t = _trimmer(dict(redirect=("too_short",), options1=dict(minimum_length=50), options2=dict(minimum_length=50),
                      collect_statistics=True))
    assert list(t.process_chunks_split(items)) == want
    assert [dict(s) for s in t.statistics] == [dict(s) for s in ref.statistics]
    assert stats_of(t) == stats_of(ref)
