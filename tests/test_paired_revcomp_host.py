"""
--revcomp on pairs without a GPU: the host build of the pair decision (fq_pair_swap_core via tests/hostsim) against a
restatement of PairedReverseComplementer's rule, the test-side oracle (tests/paired_revcomp_oracle.py) against the
reference's three known answers (test_paired.py:786-833, tests/golden/fastq_kat.json.gz), and the argument errors of
PairedFastqTrimmer and tools/trim_fastq.py.
"""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import paired_revcomp_oracle as PRO
from oracle import oracle
from util import fastq_file, spec_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def descs_of(adapters):
    import cutadapt_b200.adapters as PA

    if not adapters:
        return None, None
    spec = spec_of(PA.MultipleAdapters(adapters))
    return spec.adapters, spec.groups


# ---- the pair decision ---------------------------------------------------------------------------------------------

def hostsim_swap(m11, m22, m12, m21, per1, per2):
    from util import hostsim_lib

    lib = hostsim_lib()
    lib.hs_pair_swap.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    n = next(len(m) for m in (m11, m22, m12, m21) if m is not None)
    arrays = [None if m is None else np.ascontiguousarray(m) for m in (m11, m22, m12, m21)]
    out = np.zeros(n, dtype=np.int32)
    lib.hs_pair_swap(n, *[None if a is None else a.ctypes.data for a in arrays], per1, per2, out.ctypes.data)
    return out.astype(bool)


def random_records(rng, n, times, slots):
    m = np.zeros((n, times, slots), dtype=oracle.MATCH_DTYPE)
    m["adapter"] = -1
    for i in range(n):
        for t in range(times):
            for s in range(slots):                   # slot 1: the back part of a linked match
                if rng.random() < 0.45:
                    m[i, t, s]["adapter"] = rng.randrange(3)
                    m[i, t, s]["score"] = rng.choice([0, 1, 3, 5, 8, 12])
                elif rng.random() < 0.2:
                    m[i, t, s]["score"] = rng.choice([7, 100])    # a score on an empty record never counts
    return m


def restated(m11, m22, m12, m21):
    def score(m, i):
        if m is None:
            return 0
        return sum(int(r["score"]) for r in m[i].reshape(-1) if r["adapter"] >= 0)
    n = next(len(m) for m in (m11, m22, m12, m21) if m is not None)
    return np.array([score(m12, i) + score(m21, i) > score(m11, i) + score(m22, i) for i in range(n)])


@pytest.mark.parametrize("times1,slots1,times2,slots2", [(1, 1, 1, 1), (2, 1, 1, 2), (1, 2, 3, 1), (3, 2, 2, 2)])
@pytest.mark.parametrize("absent", [None, 1, 2])
def test_pair_decision_against_restatement(times1, slots1, times2, slots2, absent):
    rng = random.Random(times1 * 100 + slots1 * 10 + times2 + (absent or 0) * 1000)
    n = 4000
    m11, m12 = random_records(rng, n, times1, slots1), random_records(rng, n, times1, slots1)
    m22, m21 = random_records(rng, n, times2, slots2), random_records(rng, n, times2, slots2)
    ties = rng.sample(range(n), n // 5)              # identical mates: both pairings score the same
    for i in ties:
        m12[i], m21[i] = m11[i], m22[i]
    if absent == 1:
        m11 = m12 = None
    elif absent == 2:
        m22 = m21 = None
    want = restated(m11, m22, m12, m21)
    got = hostsim_swap(m11, m22, m12, m21, times1 * slots1, times2 * slots2)
    assert (got == want).all()
    assert (got == PRO.pair_swapped(m11, m22, m12, m21)).all()
    assert not got[ties].any()                        # a tie keeps the input order
    assert 0 < got.sum() < n


# ---- the reference's known answers through the oracle ------------------------------------------------------------------

def kat_cases():
    """(name, adapters1, adapters2, swap inputs, expected out1, out2, swapped pairs) of test_paired.py:786-833."""
    import cutadapt_b200.adapters as PA

    g = [PA.PrefixAdapter("TTATTTGTCT", name="a"), PA.PrefixAdapter("TCCGCACTGGC", name="b")]
    one = (fastq_file("revcomp_one_mate.out1.fastq"), fastq_file("revcomp_one_mate.out2.fastq"))
    return [("one_mate_g", g, None, False, one[0], one[1], None),
            ("one_mate_G", None, g, True, one[1], one[0], None),
            ("r1r2", [PA.PrefixAdapter("TTATTTGTCT", name="a")], [PA.PrefixAdapter("TCCGCACTGGC", name="b")], False,
             fastq_file("revcomp_r1r2.out1.fastq"), fastq_file("revcomp_r1r2.out2.fastq"), 2)]


def test_oracle_reproduces_the_known_answers():
    in1, in2 = fastq_file("revcomp.in.fastq"), fastq_file("revcomp.in2.fastq")
    for name, a1, a2, swap_inputs, want1, want2, n_swapped in kat_cases():
        d1, d2 = (in2, in1) if swap_inputs else (in1, in2)
        out1, out2, c1, c2, extra = PRO.paired_revcomp_trim(d1, d2, *descs_of(a1), *descs_of(a2), {}, {},
                                                            n_adapters=(len(a1 or []), len(a2 or [])))
        assert (out1, out2) == (want1, want2), name
        assert c1["reverse_complemented"] == c2["reverse_complemented"] == int(extra["swapped"].sum())
        if n_swapped is not None:
            assert c1["reverse_complemented"] == n_swapped


def test_oracle_without_revcomp_effect_matches_the_plain_oracle():
    """Per-mate -u / -q stay with the input mate: a pair that is not swapped is trimmed exactly as without --revcomp,
    and bp_in / quality_trimmed_bp are the input mates' own."""
    import cutadapt_b200.adapters as PA

    in1, in2 = fastq_file("revcomp.in.fastq"), fastq_file("revcomp.in2.fastq")
    o1 = dict(quality_trim=True, cutoff_front=0, cutoff_back=20, cut=(2,))
    o2 = dict(quality_trim=True, cutoff_front=0, cutoff_back=5, cut=(-1,))
    a1 = [PA.BackAdapter("GGGGGGGGGGGGGG", name="never")]
    e1, e2, ec1, ec2 = oracle.oracle_fastq_trim_paired(in1, in2, *descs_of(a1), None, None, o1, o2)
    g1, g2, gc1, gc2, extra = PRO.paired_revcomp_trim(in1, in2, *descs_of(a1), None, None, o1, o2, n_adapters=(1, 0))
    assert not extra["swapped"].any()
    assert (g1, g2) == (e1, e2)
    for k in ec1:
        assert gc1[k] == ec1[k] and gc2[k] == ec2[k], k


def test_oracle_swap_keeps_each_mates_own_quality_trimming():
    """A swapped record is trimmed with its input mate's -q only (rc names, no second quality pass)."""
    import cutadapt_b200.adapters as PA

    r1 = "@p/1\nACGTACGTACGTAAAAAAAA\n+\nIIIIIIIIIIII########\n"
    r2 = "@p/2\nTTATTTGTCTGGGGCCCCAAAA\n+\nIIIIIIIIIIIIIIIIIIIIII\n"
    a1 = [PA.PrefixAdapter("TTATTTGTCT", name="a")]
    out1, out2, c1, c2, extra = PRO.paired_revcomp_trim(
        r1.encode(), r2.encode(), *descs_of(a1), None, None,
        dict(quality_trim=True, cutoff_front=0, cutoff_back=30), dict(quality_trim=True, cutoff_front=0, cutoff_back=30),
        n_adapters=(1, 0))
    assert extra["swapped"].tolist() == [True]
    assert out1 == b"@p/2 rc\nGGGGCCCCAAAA\n+\nIIIIIIIIIIII\n"
    assert out2 == b"@p/1 rc\nACGTACGTACGT\n+\nIIIIIIIIIIII\n"
    assert c1["quality_trimmed_bp"] == 8 and c2["quality_trimmed_bp"] == 0
    assert c1["bp_in"] == 20 and c2["bp_in"] == 22
    assert extra["adapter_rc"] == ([1], [])


# ---- argument errors -------------------------------------------------------------------------------------------------

def test_paired_trimmer_argument_errors():
    import cutadapt_b200.adapters as PA
    from cutadapt_b200.pipeline import PairedFastqTrimmer

    a = [PA.BackAdapter("ACGTACGT", name="a")]
    for key in ("revcomp", "rc_suffix"):
        with pytest.raises(ValueError, match="one option for the pair"):
            PairedFastqTrimmer(a, a, {key: True}, {})
        with pytest.raises(ValueError, match="one option for the pair"):
            PairedFastqTrimmer(a, a, {}, {key: True})
    with pytest.raises(ValueError, match="Cannot use --revcomp with --pair-adapters"):
        PairedFastqTrimmer(a, a, {}, {}, pair_adapters=True, revcomp=True)
    with pytest.raises(ValueError, match="info rows"):
        PairedFastqTrimmer(a, a, {}, {}, revcomp=True, rows=("info",))
    with pytest.raises(ValueError, match="info rows"):
        PairedFastqTrimmer(a, a, {}, {}, revcomp=True, rows2=("info",))


def test_trim_fastq_refuses_info_file_with_paired_revcomp(tmp_path):
    in1, in2 = tmp_path / "in.1.fastq", tmp_path / "in.2.fastq"
    in1.write_bytes(fastq_file("revcomp.in.fastq"))
    in2.write_bytes(fastq_file("revcomp.in2.fastq"))
    for extra in (["-p", str(tmp_path / "o2.fastq"), str(in1), str(in2)], ["--interleaved", str(in1)]):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), "--revcomp", "-g", "^TTATTTGTCT",
                            "--info-file", str(tmp_path / "info.txt"), "-o", str(tmp_path / "o1.fastq")] + extra,
                           capture_output=True, text=True)
        assert r.returncode == 2
        assert "--info-file cannot be combined with --revcomp on paired-end data" in r.stderr
