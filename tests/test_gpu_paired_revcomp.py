"""
GPU tests (-m gpu) of --revcomp on pairs in the device FASTQ path (PairedReverseComplementer, modifiers.py:311-400):
the reference's three known answers through PairedFastqTrimmer, interleaved input and tools/trim_fastq.py; seeded
random pairs against the test-side oracle (tests/paired_revcomp_oracle.py) on every paired collect, with gzip outputs,
gzip device input, FASTA, rest and wildcard rows and the statistics; and the refusals.
"""
import ctypes as C
import gzip
import os
import random
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cutadapt_b200.adapters as PA  # noqa: E402
import fasta_oracle as FO  # noqa: E402
import filter_outputs_oracle as FOO  # noqa: E402
import interleaved_oracle as IO  # noqa: E402
import paired_revcomp_oracle as PRO  # noqa: E402
import rows_oracle as RO  # noqa: E402
from cutadapt_b200 import _lib, pipeline  # noqa: E402
from cutadapt_b200.pipeline import PairedFastqTrimmer  # noqa: E402
from test_paired_revcomp_host import descs_of, kat_cases  # noqa: E402
from util import fastq_file  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def interleave(d1: bytes, d2: bytes, fmt="fastq") -> bytes:
    return IO.interleave(d1, d2, fmt)


# ---- the reference's known answers ------------------------------------------------------------------------------------

def test_kat_cases_through_the_trimmer_and_interleaved_input():
    in1, in2 = fastq_file("revcomp.in.fastq"), fastq_file("revcomp.in2.fastq")
    for name, a1, a2, swap_inputs, want1, want2, n_swapped in kat_cases():
        d1, d2 = (in2, in1) if swap_inputs else (in1, in2)
        for chunk2 in (d2, None):
            t = PairedFastqTrimmer(a1, a2, revcomp=True)
            got = t.process_chunk(d1, chunk2) if chunk2 is not None else t.process_chunk(interleave(d1, d2))
            assert got == (want1, want2), (name, chunk2 is None)
            st1, st2 = t.statistics
            assert st1["reverse_complemented"] == st2["reverse_complemented"]
            if n_swapped is not None:
                assert st1["reverse_complemented"] == n_swapped


def test_kat_cases_through_trim_fastq(tmp_path):
    in1, in2 = tmp_path / "in.1.fastq", tmp_path / "in.2.fastq"
    in1.write_bytes(fastq_file("revcomp.in.fastq"))
    in2.write_bytes(fastq_file("revcomp.in2.fastq"))
    tool = [sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), "--revcomp"]
    o1, o2, js = tmp_path / "o1.fastq", tmp_path / "o2.fastq", tmp_path / "r.json"
    subprocess.run(tool + ["-g", "^TTATTTGTCT", "-G", "^TCCGCACTGGC", "--json", str(js), "-o", str(o1), "-p", str(o2),
                           str(in1), str(in2)], check=True, capture_output=True)
    assert o1.read_bytes() == fastq_file("revcomp_r1r2.out1.fastq")
    assert o2.read_bytes() == fastq_file("revcomp_r1r2.out2.fastq")
    import json

    report = json.loads(js.read_text())
    assert report["read1"]["counters"]["reverse_complemented"] == 2
    subprocess.run(tool + ["-g", "^TTATTTGTCT", "-g", "^TCCGCACTGGC", "-o", str(o1), "-p", str(o2), str(in1), str(in2)],
                   check=True, capture_output=True)
    assert (o1.read_bytes(), o2.read_bytes()) == (fastq_file("revcomp_one_mate.out1.fastq"),
                                                  fastq_file("revcomp_one_mate.out2.fastq"))
    # single-end --revcomp (ReverseComplementer) and the interleaved output
    subprocess.run(tool + ["-g", "^TTATTTGTCT", "-g", "^TCCGCACTGG", "-o", str(o1), str(in1)], check=True,
                   capture_output=True)
    assert o1.read_bytes() == fastq_file("revcomp.out.fastq")
    ilv = tmp_path / "in.ilv.fastq"
    ilv.write_bytes(interleave(in1.read_bytes(), in2.read_bytes()))
    subprocess.run(tool + ["--interleaved", "-g", "^TTATTTGTCT", "-G", "^TCCGCACTGGC", "-o", str(o1), str(ilv)],
                   check=True, capture_output=True)
    assert o1.read_bytes() == interleave(fastq_file("revcomp_r1r2.out1.fastq"), fastq_file("revcomp_r1r2.out2.fastq"))


# ---- seeded random pairs against the oracle ---------------------------------------------------------------------------

BACK1, FRONT1, BACK2, FRONT2 = "AGATCGGAAGAGC", "TTATTTGTCTCA", "CAGTGGAGTAACTC", "TCCGCACTGGCA"


def random_pairs(n, seed, fasta=False):
    """Pairs whose mates carry the -a adapters (BACK1 / FRONT1) or the -A adapters (BACK2 / FRONT2), each in either mate,
    and some identical mates (a tie: the input order stays)."""
    rng = random.Random(seed)

    def body():
        return "".join(rng.choice("ACGT") for _ in range(rng.randint(15, 70)))

    def plant(seq, back, front):
        r = rng.random()
        if r < 0.3:
            cut = rng.randint(4, len(back))
            return seq + back[:cut] + body()[:rng.randint(0, 5)]
        if r < 0.5:
            return front + seq
        return seq
    m1, m2 = [], []
    for i in range(n):
        s1, s2 = body(), body()
        if rng.random() < 0.5:
            s1, s2 = plant(s1, BACK1, FRONT1), plant(s2, BACK2, FRONT2)
        else:                                               # the adapters in the other mates
            s1, s2 = plant(s1, BACK2, FRONT2), plant(s2, BACK1, FRONT1)
        if rng.random() < 0.1:
            s2 = s1
        for k, s in ((0, s1), (1, s2)):
            name = f"p{seed}_{i}/{k + 1}"
            q = "".join(rng.choice("#+5?I") for _ in s)
            (m1, m2)[k].append(f">{name}\n{s}\n" if fasta else f"@{name}\n{s}\n+\n{q}\n")
    return "".join(m1).encode(), "".join(m2).encode()


def adapters(which, linked=False):
    if which == 1:
        ads = [PA.BackAdapter(BACK1, max_errors=0.1, name="b1"), PA.FrontAdapter(FRONT1, max_errors=0.1, name="f1")]
        if linked:
            ads = [PA.LinkedAdapter(PA.PrefixAdapter(FRONT1, name="lf"), PA.BackAdapter(BACK1, name="lb"), False, False,
                                    "l1"), PA.BackAdapter("GGGGCCCCAAAA", name="x1")]
        return ads
    return [PA.BackAdapter(BACK2, max_errors=0.1, name="b2"), PA.FrontAdapter(FRONT2, max_errors=0.1, name="f2")]


def okw(o):
    """FastqTrimmer keywords -> oracle options"""
    o = dict(o)
    if "quality_cutoff" in o:
        c = o.pop("quality_cutoff")
        o.update(quality_trim=True, cutoff_front=c[0], cutoff_back=c[1])
    return o


def n_flat(ads):
    return len(PA.MultipleAdapters(ads)._flatten()[0]) if ads else 0


CASES = {
    "qual_cut_min": (dict(quality_cutoff=(0, 20), cut=[3], minimum_length=10),
                     dict(quality_cutoff=(5, 10), cut=[-2], minimum_length=20), "any", True, (1, 2), False),
    "times2_polya_both": (dict(times=2, poly_a=True, minimum_length=10), dict(times=2, poly_a=True), "both", False,
                          (1, 2), False),
    "linked_mask_first": (dict(action="mask", maximum_length=70), dict(action="mask", maximum_length=70), "first", True,
                          (1, 2), True),
    "lowercase_maxn": (dict(action="lowercase", max_n=1), dict(action="lowercase", max_n=1), "any", True, (1, 2), False),
    "none_untrimmed": (dict(action="none", discard_untrimmed=True), dict(action="none", discard_untrimmed=True), "any",
                       True, (1, 2), False),
    "set1_only_trimmed": (dict(discard_trimmed=True, nextseq_cutoff=20), dict(quality_cutoff=(0, 15)), "any", True,
                          (1,), False),
    "set2_only": (dict(cut=[-4]), dict(minimum_length=25, trim_n=True), "both", True, (2,), False),
}


def case_adapters(sets, linked):
    return (adapters(1, linked) if 1 in sets else None), (adapters(2) if 2 in sets else None)


def oracle_paired(d1, d2, a1, a2, o1, o2, pf, rc_suffix, **kw):
    return PRO.paired_revcomp_trim(d1, d2, *descs_of(a1), *descs_of(a2), okw(o1), okw(o2), pf, 1 if rc_suffix else 2,
                                   n_adapters=(n_flat(a1), n_flat(a2)), **kw)


@pytest.mark.parametrize("name", sorted(CASES))
def test_random_pairs_against_oracle_with_statistics(name):
    o1, o2, pf, rc_suffix, sets, linked = CASES[name]
    a1, a2 = case_adapters(sets, linked)
    d1, d2 = random_pairs(3000, 100 + sorted(CASES).index(name))
    t = PairedFastqTrimmer(a1, a2, o1, o2, pf, revcomp=True, rc_suffix=rc_suffix, collect_statistics=True)
    got = t.process_chunk(d1, d2)
    e1, e2, c1, c2, extra = oracle_paired(d1, d2, a1, a2, o1, o2, pf, rc_suffix)
    assert got == (e1, e2)
    assert 0 < extra["swapped"].sum() < len(extra["swapped"])
    for st, c in zip(t.statistics, (c1, c2)):
        for k, v in c.items():
            assert st[k] == v, (k, st[k], v)
    for (vec, max_len, kmax), rc in zip(t.statistics_vector(), extra["adapter_rc"]):
        lay = pipeline.fastq_stats_layout(len(rc), max_len, kmax)
        assert vec[5] == extra["swapped"].sum()
        assert vec[lay["reverse_complemented"]:lay["reverse_complemented"] + len(rc)].tolist() == rc
    # interleaved input gives the same
    t2 = PairedFastqTrimmer(a1, a2, o1, o2, pf, revcomp=True, rc_suffix=rc_suffix)
    assert t2.process_chunk(interleave(d1, d2)) == (e1, e2)


def test_fasta_input():
    a1, a2 = adapters(1), adapters(2)
    d1, d2 = random_pairs(2000, 71, fasta=True)
    o = dict(minimum_length=12)
    t = PairedFastqTrimmer(a1, a2, o, o, revcomp=True, input_format="fasta")
    got = t.process_chunk(d1, d2)
    e1, e2, c1, c2, _ = oracle_paired(FO.as_fastq(d1), FO.as_fastq(d2), a1, a2, o, o, "any", True)
    assert got == (FO.fastq_as_fasta(e1), FO.fastq_as_fasta(e2))
    assert t.statistics[0]["reverse_complemented"] == c1["reverse_complemented"] > 0


def split_oracle(d1, d2, a1, a2, o1, o2, pf, redirect, formats=None, output_format=None):
    s1, s2, so1, so2, extra = PRO.swapped_pairs(d1, d2, *descs_of(a1), *descs_of(a2), okw(o1), okw(o2))
    outs, c1, c2 = FOO.redirect_trim_paired(s1, s2, *descs_of(a1), *descs_of(a2), so1, so2, pf, redirect, formats,
                                            "fastq", output_format)
    PRO.fix_counters(c1, c2, extra)
    return outs, c1, c2


@pytest.mark.parametrize("gz", [False, True])
def test_split_and_interleaved_outputs(gz):
    a1, a2 = adapters(1), adapters(2)
    d1, d2 = random_pairs(3000, 5 + gz)
    o = dict(minimum_length=25, maximum_length=75)
    redirect = ("too_short", "too_long", "untrimmed")
    formats = {"too_long": "fasta"}
    names = ("output",) + redirect
    want, c1, c2 = split_oracle(d1, d2, a1, a2, o, o, "any", redirect, formats)
    gzk = dict(gzip_outputs=names) if gz else {}
    t = PairedFastqTrimmer(a1, a2, o, o, revcomp=True, redirect=redirect, redirect_formats=formats, **gzk)
    got = t.process_chunk_split(d1, d2)
    unz = (lambda b: gzip.decompress(b) if b else b) if gz else (lambda b: b)
    assert {k: (unz(v[0]), unz(v[1])) for k, v in got.items()} == want
    for st, c in zip(t.statistics, (c1, c2)):
        for k in FOO.COUNTER_NAMES + ("reverse_complemented", "bp_in", "with_adapters"):
            assert st[k] == c[k], k
    ti = PairedFastqTrimmer(a1, a2, o, o, revcomp=True, redirect=redirect, redirect_formats=formats,
                            interleaved_outputs=("output", "too_short"), **gzk)
    got = ti.process_chunk_split(interleave(d1, d2))
    assert unz(got["output"][0]) == interleave(*want["output"])
    assert unz(got["too_short"][0]) == interleave(*want["too_short"])
    assert (unz(got["too_long"][0]), unz(got["too_long"][1])) == want["too_long"]


@pytest.mark.parametrize("combinatorial", [False, True])
def test_demultiplexing(combinatorial):
    a1, a2 = adapters(1), adapters(2)
    d1, d2 = random_pairs(3000, 11 + combinatorial)
    o = dict(minimum_length=10)
    t = PairedFastqTrimmer(a1, a2, o, o, revcomp=True)
    got = t.process_chunk_demux(d1, d2, combinatorial=combinatorial)
    names1, names2 = [a.name for a in a1], [a.name for a in a2]

    def route(l1, l2):
        k1 = names1[l1] if l1 >= 0 else None
        k2 = names2[l2] if l2 >= 0 else None
        return (k1, k2) if combinatorial else (k1 if k1 is not None else "unknown")
    e1, e2, c1, c2, _ = oracle_paired(d1, d2, a1, a2, o, o, "any", True, route=route)
    assert set(e1) <= set(got)
    for key, (g1, g2) in got.items():
        assert (g1, g2) == (e1.get(key, b""), e2.get(key, b"")), key
    for st, c in zip(t.statistics, (c1, c2)):
        for k, v in c.items():
            assert st[k] == v, k


def test_gzip_device_input(tmp_path):
    a1, a2 = adapters(1), adapters(2)
    d1, d2 = random_pairs(4000, 23)
    p1, p2 = tmp_path / "a.fastq.gz", tmp_path / "b.fastq.gz"
    for p, d in ((p1, d1), (p2, d2)):                       # short concatenated members: the device inflates them
        recs = d.split(b"\n")
        parts = [b"\n".join(recs[k:k + 400]) + b"\n" for k in range(0, len(recs) - 1, 400)]
        p.write_bytes(b"".join(gzip.compress(x) for x in parts))
    o = dict(minimum_length=10)
    t = PairedFastqTrimmer(a1, a2, o, o, revcomp=True)
    out1, out2 = [], []
    with open(p1, "rb") as f1, open(p2, "rb") as f2:
        for c1_, c2_ in pipeline.read_gzip_device_paired_chunks(f1, f2, t, 1 << 16):
            g1, g2 = t.process_chunk(c1_, c2_)
            out1.append(g1)
            out2.append(g2)
    e1, e2, c1, _, _ = oracle_paired(d1, d2, a1, a2, o, o, "any", True)
    assert (b"".join(out1), b"".join(out2)) == (e1, e2)
    assert t.statistics[0]["reverse_complemented"] == c1["reverse_complemented"] > 0


def test_rest_and_wildcard_rows():
    a1 = [PA.BackAdapter(BACK1, max_errors=0.1, name="b1"), PA.FrontAdapter("NNTTATTTGTCTCA", max_errors=0.1, name="w1")]
    a2 = adapters(2)
    d1, d2 = random_pairs(3000, 31)
    t = PairedFastqTrimmer(a1, a2, revcomp=True, rows=("rest", "wildcard"), rows2=("rest",))
    got = t.process_chunk(d1, d2)
    ro1, l1 = RO.row_options(a1, ("rest", "wildcard"))
    ro2, l2 = RO.row_options(a2, ("rest",))
    e1, e2, _, _, extra = PRO.paired_revcomp_trim(d1, d2, *descs_of(a1), *descs_of(a2), ro1, ro2)
    assert got == (e1, e2) and extra["swapped"].any()
    assert t.last_rows["rest"] == (RO._text(l1)["rest"], RO._text(l2)["rest"])
    assert t.last_rows["wildcard"][0] == RO._text(l1)["wildcard"]


# ---- refusals and the unchanged path ---------------------------------------------------------------------------------

def collect_raw(t, d1, d2, p1, p2):
    s1, s2 = pipeline._submit_chunk(t.ctx, d1), pipeline._submit_chunk(t.ctx, d2)
    out1, out2 = np.empty(1 << 20, np.uint8), np.empty(1 << 20, np.uint8)
    r1, r2 = _lib.cg_fastq_result(), _lib.cg_fastq_result()
    rc = _lib.lib().cg_fastq_collect_paired(t.ctx.handle, s1[0], s2[0], t._set1.handle, t._set2.handle, C.byref(p1),
                                            C.byref(p2), 0, out1.ctypes.data, out1.size, out2.ctypes.data, out2.size,
                                            C.byref(r1), C.byref(r2))
    return rc, s1[0], s2[0]


def test_refusals():
    a1, a2 = adapters(1), adapters(2)
    d1, d2 = random_pairs(50, 3)
    t = PairedFastqTrimmer(a1, a2)
    p1 = pipeline._fastq_params(revcomp=True)
    p2 = pipeline._fastq_params()
    rc, s1, s2 = collect_raw(t, d1, d2, p1, p2)
    assert rc == _lib.CG_EINVAL and b"must be equal" in _lib.lib().cg_last_error()
    # the slots stay submitted: they can still be collected
    out = np.empty(1 << 20, np.uint8)
    assert _lib.lib().cg_fastq_collect_paired(t.ctx.handle, s1, s2, t._set1.handle, t._set2.handle, C.byref(p2),
                                              C.byref(p2), 0, out.ctypes.data, out.size, out.ctypes.data, out.size,
                                              C.byref(_lib.cg_fastq_result()), C.byref(_lib.cg_fastq_result())) == 0
    # an info-row request on a paired revcomp collect
    s1, _ = pipeline._submit_chunk(t.ctx, d1)
    s2, _ = pipeline._submit_chunk(t.ctx, d2)
    texts = pipeline._row_text(t.adapters1, "info")
    pipeline._request_rows(t.ctx, s1, ("info",), {"info": texts}, ())
    pr = pipeline._fastq_params(revcomp=True)
    rc = _lib.lib().cg_fastq_collect_paired(t.ctx.handle, s1, s2, t._set1.handle, t._set2.handle, C.byref(pr),
                                            C.byref(pr), 0, out.ctypes.data, out.size, out.ctypes.data, out.size,
                                            C.byref(_lib.cg_fastq_result()), C.byref(_lib.cg_fastq_result()))
    assert rc == _lib.CG_EINVAL and b"info rows" in _lib.lib().cg_last_error()
    with pytest.raises(ValueError, match="Cannot use --revcomp with --pair-adapters"):
        PairedFastqTrimmer(a1, a2, pair_adapters=True, revcomp=True)
