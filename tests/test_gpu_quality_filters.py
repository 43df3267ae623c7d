"""
--max-aer (TooHighAverageErrorRate) and -z (ZeroCapper) on the device, byte for byte against the oracle extended with
both steps (tests/quality_filters_oracle.py): the reference's known answers, seeded single-end and paired chunks, filter
outputs, single / paired / combinatorial demultiplexing, interleaved and gzip outputs, info rows, FASTQ -> FASTA, the
result counter and statistics slot 15, the argument errors of the C ABI, and tools/trim_fastq.py.
"""
import ctypes as C
import gzip
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import fasta_oracle as FO
import filter_outputs_oracle as RO
import interleaved_oracle as IO
import quality_filters_oracle as QO
import rows_oracle as RW
from test_quality_filters_host import ADAPTER, synthetic_chunk

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COUNTERS = ("n_written", "bp_out", "too_short", "too_long", "too_many_n", "too_many_expected_errors", "discarded",
            "casava_filtered", "too_high_average_error_rate")


def _ads(names=("a1", "a2")):
    import cutadapt_b200.adapters as PA

    return [PA.BackAdapter(ADAPTER, max_errors=0.1, min_overlap=3, name=names[0]),
            PA.FrontAdapter("TTGACNNACG", max_errors=0.1, min_overlap=3, name=names[1])]


def _okw(kw):
    """The oracle's keywords for FastqTrimmer's."""
    o = dict(kw)
    if "quality_cutoff" in o:
        qc = o.pop("quality_cutoff")
        o.update(quality_trim=True, cutoff_front=qc[0], cutoff_back=qc[1])
    return o


def _check_counters(stats, c):
    for k in COUNTERS:
        assert stats[k] == c[k], (k, stats[k], c[k])


VARIANTS = {
    "aer_cap": dict(max_average_error_rate=0.05, zero_cap=True, minimum_length=5),
    "aer_only": dict(max_average_error_rate=0.01),
    "cap_ee_qtrim": dict(zero_cap=True, max_expected_errors=1.5, quality_cutoff=(5, 20), trim_n=True),
    "all": dict(zero_cap=True, max_expected_errors=2.0, max_average_error_rate=0.02, discard_casava=True,
                minimum_length=10, max_n=3),
    "base64": dict(quality_base=64, zero_cap=True, max_average_error_rate=0.0004, quality_cutoff=(0, 15)),
}
BELOW = {"aer_only": False}


def _chunk(name, seed, n=3000):
    kw = VARIANTS[name]
    return synthetic_chunk(random.Random(seed), n, base=kw.get("quality_base", 33), below=BELOW.get(name, True))


# ---- the reference's known answers -------------------------------------------------------------------------------

def test_known_answers_of_the_reference():
    from cutadapt_b200.pipeline import FastqTrimmer

    kat = QO.quality_filters_kat()
    for case in kat["too_high_average_error_rate"]:
        q = case["qualities"]
        data = f"@r\n{'A' * len(q)}\n+\n{q}\n".encode()
        t = FastqTrimmer(max_average_error_rate=float.fromhex(case["rate"]), collect_statistics=True)
        out = t.process_chunk(data)
        assert (out == b"") == case["expected"], case
        assert t.statistics["too_high_average_error_rate"] == int(case["expected"])
        assert int(t.statistics_vector()[0][15]) == int(case["expected"])
    z = kat["zero_capper"]
    t = FastqTrimmer(zero_cap=True, quality_base=z["quality_base"])
    data = f"@r1\n{z['sequence']}\n+\n{z['qualities']}\n".encode()
    assert t.process_chunk(data) == f"@r1\n{z['sequence']}\n+\n{z['expected']}\n".encode()


# ---- seeded chunks -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(VARIANTS))
@pytest.mark.parametrize("adapters", [False, True])
def test_single_end_chunks_against_the_oracle(name, adapters):
    from cutadapt_b200.pipeline import FastqTrimmer

    kw = VARIANTS[name]
    data = _chunk(name, 100 + len(name) + adapters)
    ads = _ads() if adapters else None
    t = FastqTrimmer(ads, collect_statistics=True, **kw)
    got = t.process_chunk(data)
    with QO.extended() as orc:
        want, c = orc.oracle_fastq_trim(data, *(FO.descriptors(ads) if ads else (None, None)), **_okw(kw))
    assert got == want
    _check_counters(t.statistics, c)
    assert int(t.statistics_vector()[0][15]) == c["too_high_average_error_rate"]
    if kw.get("max_average_error_rate"):
        assert c["too_high_average_error_rate"] > 0


@pytest.mark.parametrize("pair_filter", ["any", "both", "first"])
@pytest.mark.parametrize("which", ["both", "r1", "r2"])
def test_paired_chunks_against_the_oracle(pair_filter, which):
    from cutadapt_b200.pipeline import PairedFastqTrimmer

    rng = random.Random(7)
    data1, data2 = synthetic_chunk(rng, 2000), synthetic_chunk(rng, 2000)
    aer = dict(max_average_error_rate=0.03, zero_cap=True, minimum_length=5)
    kw1 = aer if which in ("both", "r1") else dict(zero_cap=True, minimum_length=5)
    kw2 = aer if which in ("both", "r2") else dict(zero_cap=True, minimum_length=5)
    t = PairedFastqTrimmer(_ads(), None, kw1, kw2, pair_filter, collect_statistics=True)
    got = t.process_chunk(data1, data2)
    with QO.extended() as orc:
        o1, o2, c1, c2 = orc.oracle_fastq_trim_paired(data1, data2, *FO.descriptors(_ads()), None, None, kw1, kw2,
                                                      pair_filter)
    assert got == (o1, o2)
    for st, c in zip(t.statistics, (c1, c2)):
        _check_counters(st, c)
    vecs = t.statistics_vector()
    assert int(vecs[0][0][15]) == int(vecs[1][0][15]) == c1["too_high_average_error_rate"] > 0


# ---- filter outputs, demultiplexing, interleaved and gzip outputs ------------------------------------------------

def test_split_outputs_carry_capped_qualities_and_drop_max_aer_reads():
    from cutadapt_b200.pipeline import FastqTrimmer

    kw = dict(minimum_length=30, maximum_length=70, max_average_error_rate=0.04, zero_cap=True)
    data = _chunk("aer_cap", 31)
    t = FastqTrimmer(_ads(), redirect=("too_short", "too_long", "untrimmed"), **kw)
    got = t.process_chunk_split(data)
    with QO.extended():
        want, c = RO.redirect_trim(data, *FO.descriptors(_ads()), redirect=("too_short", "too_long", "untrimmed"), **kw)
    assert got == want
    _check_counters(t.statistics, c)
    assert c["too_high_average_error_rate"] > 0 and c["too_short"] > 0
    assert all(min(line) >= 33 for line in got["too_short"].split(b"\n")[3::4] if line)
    written = sum(len(v.split(b"\n")) // 4 for v in got.values())
    assert written + c["too_high_average_error_rate"] == data.count(b"\n") // 4


def test_single_end_demultiplexing():
    from cutadapt_b200.pipeline import FastqTrimmer

    kw = dict(max_average_error_rate=0.05, zero_cap=True)
    data = _chunk("aer_cap", 41)
    t = FastqTrimmer(_ads(), **kw)
    got = t.process_chunk_demux(data)
    with QO.extended() as orc:
        want = orc.oracle_fastq_demux(data, *FO.descriptors(_ads()), ["a1", "a2"], **kw)
    assert {k: v for k, v in got.items() if v} == {k: v for k, v in want.items() if v}
    assert t.statistics["too_high_average_error_rate"] > 0


@pytest.mark.parametrize("combinatorial", [False, True])
def test_paired_demultiplexing(combinatorial):
    from cutadapt_b200.pipeline import PairedFastqTrimmer

    rng = random.Random(51 + combinatorial)
    data1, data2 = synthetic_chunk(rng, 2000), synthetic_chunk(rng, 2000)
    ads1, ads2 = _ads(("x0", "x1")), _ads(("y0", "y1"))
    kw1 = dict(max_average_error_rate=0.04, zero_cap=True)
    kw2 = dict(zero_cap=True, max_expected_errors=3.0)
    t = PairedFastqTrimmer(ads1, ads2, kw1, kw2, "any")
    got = t.process_chunk_demux(data1, data2, combinatorial=combinatorial)
    names1, names2 = [a.name for a in ads1], [a.name for a in ads2]

    def route(last1, last2):
        k1 = names1[last1] if last1 >= 0 else None
        k2 = names2[last2] if last2 >= 0 else None
        return (k1, k2) if combinatorial else (k1 if k1 is not None else "unknown")
    with QO.extended() as orc:
        e1, e2, c1, c2 = orc.oracle_fastq_trim_paired(data1, data2, *FO.descriptors(ads1), *FO.descriptors(ads2), kw1,
                                                      kw2, "any", route=route)
    assert set(e1) <= set(got)
    for key, (g1, g2) in got.items():
        assert g1 == e1.get(key, b"") and g2 == e2.get(key, b""), key
    for st, c in zip(t.statistics, (c1, c2)):
        _check_counters(st, c)
    assert c1["too_high_average_error_rate"] > 0


def test_interleaved_and_gzip_outputs():
    from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer

    rng = random.Random(61)
    data1, data2 = synthetic_chunk(rng, 2000), synthetic_chunk(rng, 2000)
    kw = dict(max_average_error_rate=0.03, zero_cap=True, minimum_length=20)
    t = PairedFastqTrimmer(_ads(), None, kw, kw, "any", interleaved_outputs=("output", "too_short"),
                           redirect=("too_short",), gzip_outputs=("output", "too_short"))
    got = t.process_chunk_split(data1, data2)
    with QO.extended():
        want, c1, c2 = RO.redirect_trim_paired(data1, data2, *FO.descriptors(_ads()), None, None, kw, kw, "any",
                                               redirect=("too_short",))
    for name in ("output", "too_short"):
        assert got[name][1] == b""
        assert gzip.decompress(got[name][0]) == IO.interleave(*want[name], "fastq"), name
    _check_counters(t.statistics[0], c1)
    single = FastqTrimmer(_ads(), gzip_outputs=("output",), **kw)
    with QO.extended() as orc:
        plain, c = orc.oracle_fastq_trim(data1, *FO.descriptors(_ads()), **kw)
    assert gzip.decompress(single.process_chunk(data1)) == plain
    _check_counters(single.statistics, c)


# ---- info rows and FASTA output --------------------------------------------------------------------------------

@pytest.mark.parametrize("paired", [False, True])
def test_info_rows_capped_when_unmatched_original_when_matched(paired):
    from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer

    rng = random.Random(71 + paired)
    data1, data2 = synthetic_chunk(rng, 1500), synthetic_chunk(rng, 1500)
    kw = dict(zero_cap=True, max_average_error_rate=0.05)
    with QO.extended() as orc:
        if paired:
            t = PairedFastqTrimmer(_ads(), _ads(("b1", "b2")), kw, kw, rows=("info",), rows2=("info",))
            out = t.process_chunk(data1, data2)
            o1, o2, c1, c2, r1, r2 = RW.oracle_rows_paired(orc, data1, data2, _ads(), _ads(("b1", "b2")), kw, kw,
                                                           kinds1=("info",), kinds2=("info",))
            assert out == (o1, o2)
            assert t.last_rows["info"] == (r1["info"], r2["info"])
            rows = r1["info"]
        else:
            t = FastqTrimmer(_ads(), rows=("info",), **kw)
            out = t.process_chunk(data1)
            o1, c1, r1 = RW.oracle_rows_single(orc, data1, _ads(), kw, kinds=("info",))
            assert out == o1
            assert t.last_rows["info"] == r1["info"]
            rows = r1["info"]
    unmatched = [r.split(b"\t") for r in rows.split(b"\n") if r.count(b"\t") == 3]
    matched = [r.split(b"\t") for r in rows.split(b"\n") if r.count(b"\t") > 3]
    assert unmatched and all(min(f[3], default=33) >= 33 for f in unmatched)
    assert any(min(f[8] + f[9] + f[10], default=33) < 33 for f in matched)


def test_fastq_to_fasta():
    from cutadapt_b200.pipeline import FastqTrimmer

    kw = dict(zero_cap=True, max_average_error_rate=0.05, minimum_length=5)
    data = _chunk("aer_cap", 81)
    t = FastqTrimmer(_ads(), output_format="fasta", **kw)
    got = t.process_chunk(data)
    with QO.extended():
        want, c = FO.fasta_trim(data, *FO.descriptors(_ads()), input_format="fastq", output_format="fasta", **kw)
    assert got == want
    _check_counters(t.statistics, c)


# ---- the C ABI -------------------------------------------------------------------------------------------------

def _collect(ctx, data, params):
    from cutadapt_b200 import _lib

    buf = np.frombuffer(data, dtype=np.uint8)
    slot = C.c_int32(-1)
    _lib.check(_lib.lib().cg_fastq_submit(ctx.handle, buf.ctypes.data, buf.size, C.byref(slot)))
    out = np.zeros(2 * len(data) + 64, dtype=np.uint8)
    res = _lib.cg_fastq_result()
    rc = _lib.lib().cg_fastq_collect(ctx.handle, slot.value, None, C.byref(params), out.ctypes.data, out.size,
                                     C.byref(res))
    return rc, out[:res.out_bytes].tobytes() if rc == 0 else b"", res


def test_invalid_arguments_through_the_abi():
    from cutadapt_b200 import _lib
    from cutadapt_b200.pipeline import _fastq_params

    ctx = _lib.default_context()
    fastq = b"@r\nACGT\n+\nIIII\n"
    fasta = b">r\nACGT\n"
    for rate in (-0.1, 1.0, 1.5, float("nan")):
        p = _fastq_params()
        p.max_average_error_rate = rate
        assert _collect(ctx, fastq, p)[0] == _lib.CG_EINVAL, rate
    p = _fastq_params()
    p.zero_cap = 2
    assert _collect(ctx, fastq, p)[0] == _lib.CG_EINVAL
    for extra in (dict(zero_cap=True), dict(max_average_error_rate=0.1)):
        assert _collect(ctx, fasta, _fastq_params(input_format="fasta", **extra))[0] == _lib.CG_EINVAL, extra
        rc, out, _ = _collect(ctx, fastq, _fastq_params(output_format="fasta", **extra))
        assert rc == 0 and out == b">r\nACGT\n"
    rc, out, res = _collect(ctx, fastq, _fastq_params())            # 0 is off
    assert rc == 0 and out == fastq and res.too_high_average_error_rate == 0
    assert _collect(ctx, fasta, _fastq_params(input_format="fasta"))[0] == 0


def test_quality_below_the_base_with_max_ee():
    """A quality character below '!' makes --max-ee fail the chunk; with -z it is capped first and the read passes."""
    from cutadapt_b200.pipeline import FastqTrimmer

    data = b"@r\nACGT\n+\nII I\n"
    with pytest.raises(Exception):
        FastqTrimmer(max_expected_errors=1.5).process_chunk(data)
    with pytest.raises(Exception):
        FastqTrimmer(max_average_error_rate=0.5).process_chunk(data)
    t = FastqTrimmer(max_expected_errors=1.5, max_average_error_rate=0.5, zero_cap=True)
    assert t.process_chunk(data) == b"@r\nACGT\n+\nII!I\n"
    assert t.process_chunk(data) == b"@r\nACGT\n+\nII!I\n"      # the context stays usable


# ---- tools/trim_fastq.py ---------------------------------------------------------------------------------------

def test_trim_fastq_tool(tmp_path):
    import json

    data = synthetic_chunk(random.Random(91), 3000)
    (tmp_path / "in.fastq").write_bytes(data)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), "--max-aer", "0.01", "-z", "-q", "20",
                        "-a", ADAPTER, "-o", "out.fastq.gz", "--json", "report.json", "in.fastq"],
                       capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    import cutadapt_b200.adapters as PA

    ads = [PA.BackAdapter(ADAPTER, max_errors=0.1, min_overlap=3, name="back1")]
    with QO.extended() as orc:
        want, c = orc.oracle_fastq_trim(data, *FO.descriptors(ads), quality_trim=True, cutoff_back=20,
                                        max_average_error_rate=0.01, zero_cap=True)
    assert gzip.decompress((tmp_path / "out.fastq.gz").read_bytes()) == want
    report = json.loads((tmp_path / "report.json").read_text())
    assert report["counters"]["too_high_average_error_rate"] == c["too_high_average_error_rate"] > 0
    # FASTA input: --max-aer is dropped with a warning
    (tmp_path / "in.fasta").write_bytes(b">r\nACGTACGT\n")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), "--max-aer", "0.01", "-o", "o.fasta",
                        "in.fasta"], capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0 and "Ignoring option --max-aer" in r.stderr
    assert (tmp_path / "o.fasta").read_bytes() == b">r\nACGTACGT\n"
