"""
--max-aer (TooHighAverageErrorRate) and -z (ZeroCapper) without a GPU: the host build of the per-record logic of the
FASTQ kernels (fq_evaluate_core + fq_finish_core via tests/hostsim) against the oracle extended with both steps
(tests/quality_filters_oracle.py), the reference's known answers (tests/golden/quality_filters_kat.json.gz), the chain
order of the quality filters, the pair filter modes, and the argument errors of the Python layer and of
tools/trim_fastq.py.
"""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import quality_filters_oracle as QO
from oracle import oracle
from test_hostsim import _fastq_table, _finish

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADAPTER = "AGATCGGAAGAGC"
# fail-mask bit -> the counter of cg_fastq_result it goes to
COUNTER_OF_BIT = {0: "too_short", 1: "too_long", 2: "too_many_n", 3: "too_many_expected_errors", 4: "casava_filtered",
                  5: "discarded", 6: "discarded", 7: "too_high_average_error_rate"}


def synthetic_chunk(rng, n, base=33, below=True, empty=0.05):
    """FASTQ chunk with the adapter in some reads, N bases, casava flags, reads of length 0 and -- with below --
    quality characters under chr(base) (never a line break)."""
    lo = max(20, base - 12) if below else base
    alphabet = [chr(c) for c in range(lo, min(126, base + 41) + 1) if c not in (10, 13)]
    out = []
    for i in range(n):
        length = 0 if rng.random() < empty else rng.randint(1, 90)
        seq = "".join(rng.choice("ACGTACGTACGTN") for _ in range(length))
        if length > 20 and rng.random() < 0.4:
            k = rng.randint(0, length - 5)
            seq = (seq[:k] + ADAPTER + seq[k:])[:length]
        mode = rng.random()
        if mode < 0.3:                                   # good reads
            qual = "".join(rng.choice(alphabet[-15:]) for _ in range(length))
        elif mode < 0.5:                                 # poor reads
            qual = "".join(rng.choice(alphabet[:15]) for _ in range(length))
        else:
            qual = "".join(rng.choice(alphabet) for _ in range(length))
        flag = "Y" if rng.random() < 0.2 else "N"
        out.append(f"@r{i} 1:{flag}:0:ACGT\n{seq}\n+\n{qual}\n")
    return "".join(out).encode("latin-1")


def hostsim_quality(data, kw, adapters=False, second_mate=False):
    """fq_evaluate_core with both new fields on one mate (hostsim_quality.cpp), after the host build of the trimming
    pass: (record table, intervals, masks, enabled filters, cap character)."""
    from cutadapt_b200.pipeline import _fastq_params
    import cutadapt_b200.adapters as PA
    from util import hostsim_lib, hostsim_process, spec_of

    fp = _fastq_params(**kw)
    rec, lens = _fastq_table(data, kw.get("cut", ()))
    buf = np.frombuffer(data, dtype=np.uint8)
    seqs = [data[int(r[2]):int(r[2]) + int(n)].decode("latin-1") for r, n in zip(rec, lens)]
    quals = [data[int(r[3]):int(r[3]) + int(n)].decode("latin-1") for r, n in zip(rec, lens)]
    want_q = bool(fp.trim.quality_trim)
    matches = qtrim = None
    slots = 1
    if adapters:
        spec = spec_of(PA.MultipleAdapters([PA.BackAdapter(ADAPTER, max_errors=0.1, min_overlap=3)]))
        matches, qtrim = hostsim_process(spec, seqs, quals if want_q else None, fp.trim)
        slots = spec.slots
        if not want_q:
            qtrim = None
    elif want_q:
        qtrim = np.array([oracle.quality_trim_index(q, fp.trim.cutoff_front, fp.trim.cutoff_back, fp.trim.quality_base)
                          for q in quals], dtype=np.int32).reshape(-1, 2)
    n = len(seqs)
    cap = fp.trim.quality_base if fp.zero_cap else 0
    ip = np.array([fp.minimum_length, fp.maximum_length, fp.discard_trimmed, fp.discard_untrimmed,
                   (2 if second_mate else 1) if fp.poly_a else 0, 0, fp.trim_n, fp.discard_casava, 0, cap], dtype=np.int32)
    dp = np.array([fp.max_n, fp.max_expected_errors, fp.max_average_error_rate], dtype=np.float64)
    interval = np.zeros((n, 2), dtype=np.int32)
    mask = np.zeros(n, dtype=np.int32)
    lib = hostsim_lib()
    lib.hs_fastq_evaluate_quality.restype = C.c_int
    lib.hs_fastq_evaluate_quality.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    bad = lib.hs_fastq_evaluate_quality(buf.ctypes.data, n, rec.ctypes.data, lens.ctypes.data,
                                        matches.ctypes.data if matches is not None else None, max(1, fp.trim.times), slots,
                                        qtrim.ctypes.data if qtrim is not None else None, ip.ctypes.data, dp.ctypes.data,
                                        interval.ctypes.data, mask.ctypes.data)
    enabled = (1 if fp.minimum_length > 0 else 0) | (2 if fp.maximum_length >= 0 else 0) | (4 if fp.max_n >= 0 else 0) | \
        (8 if fp.max_expected_errors >= 0 else 0) | (16 if fp.discard_casava else 0) | (32 if fp.discard_trimmed else 0) | \
        (64 if fp.discard_untrimmed else 0) | (128 if fp.max_average_error_rate > 0 else 0)
    return dict(data=data, rec=rec, interval=interval, mask=mask, enabled=enabled, cap=cap, bad=bad)


def formatted(ev, fired):
    """fq_write_kernel in Python for the surviving records, qualities capped at ev["cap"]."""
    data, cap, out = ev["data"], ev["cap"], []
    for r in range(len(ev["mask"])):
        if fired[r] >= 0:
            continue
        hs, hl, ss, qs = (int(x) for x in ev["rec"][r])
        a, b = (int(x) for x in ev["interval"][r])
        q = bytes(max(c, cap) for c in data[qs + a:qs + b])
        out.append(b"@" + data[hs:hs + hl] + b"\n" + data[ss + a:ss + b] + b"\n+\n" + q + b"\n")
    return b"".join(out)


def counters(fired):
    c = {name: 0 for name in COUNTER_OF_BIT.values()}
    for k in fired:
        if k >= 0:
            c[COUNTER_OF_BIT[int(k)]] += 1
    return c


def oracle_single(data, kw, adapters=False):
    descs, groups = None, None
    if adapters:
        import cutadapt_b200.adapters as PA
        import fasta_oracle as FO

        descs, groups = FO.descriptors([PA.BackAdapter(ADAPTER, max_errors=0.1, min_overlap=3)])
    opts = dict(kw)
    if "quality_cutoff" in opts:
        qc = opts.pop("quality_cutoff")
        opts.update(quality_trim=True, cutoff_front=qc[0], cutoff_back=qc[1])
    if "maximum_length" in opts and opts["maximum_length"] is None:
        opts["maximum_length"] = -1
    with QO.extended() as orc:
        return orc.oracle_fastq_trim(data, descs, groups, **opts)


VARIANTS = [
    ("aer", 33, True, dict(max_average_error_rate=0.05, zero_cap=True)),
    ("aer_only", 33, False, dict(max_average_error_rate=0.01)),
    ("cap_only", 33, True, dict(zero_cap=True, minimum_length=1)),
    ("ee_cap", 33, True, dict(max_expected_errors=1.5, zero_cap=True)),
    ("all_quality", 33, True, dict(max_expected_errors=2.0, max_average_error_rate=0.02, zero_cap=True,
                                    discard_casava=True, minimum_length=10, max_n=3)),
    ("qtrim", 33, True, dict(quality_cutoff=(5, 20), max_average_error_rate=0.03, zero_cap=True, trim_n=True)),
    ("base64", 64, True, dict(quality_base=64, zero_cap=True, max_average_error_rate=0.0004, max_expected_errors=0.04)),
    ("base64_qtrim", 64, True, dict(quality_base=64, quality_cutoff=(0, 15), zero_cap=True, max_average_error_rate=0.0004)),
    ("base64_aer", 64, False, dict(quality_base=64, max_average_error_rate=0.0002)),
]


@pytest.mark.parametrize("name,base,below,kw", VARIANTS, ids=[v[0] for v in VARIANTS])
@pytest.mark.parametrize("adapters", [False, True])
def test_evaluate_and_finish_against_the_oracle(name, base, below, kw, adapters):
    rng = random.Random(hash((name, adapters)) & 0xFFFF)
    data = synthetic_chunk(rng, 1200, base=base, below=below)
    ev = hostsim_quality(data, kw, adapters)
    assert ev["bad"] == 0
    fired = _finish(ev)
    out, c = oracle_single(data, kw, adapters)
    assert formatted(ev, fired) == out
    got = counters(fired)
    for k, v in got.items():
        assert c[k] == v, (k, v, c[k])
    if kw.get("max_average_error_rate"):
        assert got["too_high_average_error_rate"] > 0


def test_reads_of_length_zero_pass_max_aer():
    data = b"@a\n\n+\n\n@b\nAC\n+\n!!\n@c\n\n+\n\n"
    ev = hostsim_quality(data, dict(max_average_error_rate=0.001))
    assert list(ev["mask"] & 128) == [0, 128, 0]
    ev = hostsim_quality(data, dict(max_average_error_rate=0.001, minimum_length=1))
    assert list(_finish(ev)) == [0, 7, 0]


def test_known_answers_of_the_reference():
    from util import hostsim_lib

    kat = QO.quality_filters_kat()
    lib = hostsim_lib()
    lib.hs_expected_errors_capped.restype = C.c_double
    lib.hs_expected_errors_capped.argtypes = [C.c_char_p, C.c_int, C.c_int]
    for case in kat["too_high_average_error_rate"]:
        q = case["qualities"].encode("latin-1")
        for cap in (0, 33):
            assert lib.hs_expected_errors_capped(q, len(q), cap).hex() == case["expected_errors"], case
        rate = float.fromhex(case["rate"])
        data = b"@r\n" + b"A" * len(q) + b"\n+\n" + q + b"\n"
        ev = hostsim_quality(data, dict(max_average_error_rate=rate))
        assert bool(ev["mask"][0] & 128) == case["expected"], case
        assert QO.too_high_average_error_rate(case["qualities"], rate) == case["expected"]
    z = kat["zero_capper"]
    assert QO.cap_qualities(z["qualities"], z["quality_base"]) == z["expected"]
    data = f"@r1\n{z['sequence']}\n+\n{z['qualities']}\n".encode()
    ev = hostsim_quality(data, dict(zero_cap=True, quality_base=z["quality_base"]))
    assert formatted(ev, _finish(ev)) == f"@r1\n{z['sequence']}\n+\n{z['expected']}\n".encode()
    q = z["qualities"].encode()
    assert lib.hs_expected_errors_capped(q, len(q), 33) == oracle.expected_errors(z["expected"])
    assert lib.hs_expected_errors_capped(q, len(q), 0) < 0          # ' ' is outside [33, 126] without the cap


def test_quality_below_the_base_with_max_ee():
    """With base 33 a character below '!' makes --max-ee fail the chunk; -z caps it first, so it passes."""
    data = b"@r\nACGT\n+\nII I\n"
    assert hostsim_quality(data, dict(max_expected_errors=1.5))["bad"] == 1
    assert hostsim_quality(data, dict(max_average_error_rate=0.5))["bad"] == 1
    ev = hostsim_quality(data, dict(max_expected_errors=1.5, max_average_error_rate=0.5, zero_cap=True))
    assert ev["bad"] == 0 and ev["mask"][0] & (8 | 128) == 0
    with pytest.raises(ValueError):
        oracle_single(data, dict(max_expected_errors=1.5))
    out, _ = oracle_single(data, dict(max_expected_errors=1.5, zero_cap=True))
    assert out == b"@r\nACGT\n+\nII!I\n"


def test_chain_order_of_the_quality_filters():
    """A read that fails --max-ee, --max-aer and --discard-casava is counted by the first in the reference's chain
    (TooManyExpectedErrors, TooHighAverageErrorRate, CasavaFiltered)."""
    data = b"@r 1:Y:0:A\nACGTACGTAC\n+\n!!!!!!!!!!\n"
    for kw, bit, counter in ((dict(max_expected_errors=1.0, max_average_error_rate=0.5, discard_casava=True), 3,
                              "too_many_expected_errors"),
                             (dict(max_expected_errors=20.0, max_average_error_rate=0.5, discard_casava=True), 7,
                              "too_high_average_error_rate"),
                             (dict(max_average_error_rate=0.5, discard_casava=True), 7, "too_high_average_error_rate"),
                             (dict(max_average_error_rate=0.5, discard_casava=True, max_n=0), 7,
                              "too_high_average_error_rate"),
                             (dict(max_average_error_rate=0.5, discard_casava=True, minimum_length=11), 0, "too_short"),
                             (dict(discard_casava=True), 4, "casava_filtered")):
        ev = hostsim_quality(data, kw)
        assert ev["mask"][0] & (8 | 16 | 128) == (8 if "max_expected_errors" in kw and kw["max_expected_errors"] < 10 else 0) \
            | 16 | (128 if "max_average_error_rate" in kw else 0)
        assert list(_finish(ev)) == [bit], kw
        _, c = oracle_single(data, kw)
        assert c[counter] == 1 and c["n_written"] == 0, kw


def _paired_oracle(data1, data2, kw1, kw2, pair_filter):
    with QO.extended() as orc:
        return orc.oracle_fastq_trim_paired(data1, data2, options1=kw1, options2=kw2, pair_filter=pair_filter)


@pytest.mark.parametrize("pair_filter,mode", [("any", 0), ("both", 1), ("first", 2)])
@pytest.mark.parametrize("which", ["both", "r1", "r2"])
def test_pair_filter_modes(pair_filter, mode, which):
    rng = random.Random(11 + mode)
    data1 = synthetic_chunk(rng, 800)
    data2 = synthetic_chunk(rng, 800).replace(b"@r", b"@r")
    aer = dict(max_average_error_rate=0.03, zero_cap=True)
    kw1 = dict(aer if which in ("both", "r1") else dict(zero_cap=True), minimum_length=5)
    kw2 = dict(aer if which in ("both", "r2") else dict(zero_cap=True), minimum_length=5)
    ev1, ev2 = hostsim_quality(data1, kw1), hostsim_quality(data2, kw2, second_mate=True)
    fired = _finish(ev1, ev2, mode=mode, mode_untrimmed=mode)
    out1, out2, c1, c2 = _paired_oracle(data1, data2, kw1, kw2, pair_filter)
    assert formatted(ev1, fired) == out1 and formatted(ev2, fired) == out2
    got = counters(fired)
    for c in (c1, c2):
        for k, v in got.items():
            assert c[k] == v, (k, v, c[k])
    assert got["too_high_average_error_rate"] > 0


# ---- argument errors -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rate", [0.0, 1.0, -0.1, 1.5])
def test_rate_outside_the_open_interval_is_rejected(rate):
    from cutadapt_b200.pipeline import _fastq_params

    with pytest.raises(ValueError, match="max_error_rate must be between 0.0 and 1.0"):
        _fastq_params(max_average_error_rate=rate)
    with pytest.raises(ValueError, match="max_error_rate must be between 0.0 and 1.0"):
        QO.evaluate(b"", None, None, max_average_error_rate=rate)


def test_params_defaults_leave_both_off():
    from cutadapt_b200.pipeline import _fastq_params

    fp = _fastq_params()
    assert fp.max_average_error_rate == 0.0 and fp.zero_cap == 0
    fp = _fastq_params(max_average_error_rate=0.25, zero_cap=True)
    assert fp.max_average_error_rate == 0.25 and fp.zero_cap == 1


def run_tool(tmp_path, args, content=b"@r\nACGT\n+\nIIII\n"):
    p = tmp_path / "in.fastq"
    p.write_bytes(content)
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), *args, str(p)],
                          capture_output=True, text=True, cwd=tmp_path)


@pytest.mark.parametrize("args,content,message", [
    (["-z", "-o", "o.fasta"], b">r\nACGT\n", "-z/--zero-cap needs quality values"),
    (["--max-aer", "1.0", "-o", "o.fastq"], b"@r\nACGT\n+\nIIII\n", "max_error_rate must be between 0.0 and 1.0"),
    (["--max-average-error-rate", "0", "-o", "o.fastq"], b"@r\nACGT\n+\nIIII\n",
     "max_error_rate must be between 0.0 and 1.0"),
])
def test_trim_fastq_argument_errors(tmp_path, args, content, message):
    r = run_tool(tmp_path, args, content)
    assert r.returncode == 2, r.stderr
    assert message in r.stderr
    assert not any(p.name.startswith("o.") for p in tmp_path.iterdir())
