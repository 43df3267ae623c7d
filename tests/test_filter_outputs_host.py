"""
Filter outputs (--too-short-output, --too-long-output, --untrimmed-output and their paired forms) without a GPU:
the host build of the device's routing (fq_finish_core + fq_route_core via tests/hostsim) against a model of the
reference's filter chain, the test-side redirect oracle (tests/filter_outputs_oracle.py) against the reference's known
answers (tests/golden/filter_outputs_kat.json.gz), and the argument errors of tools/trim_fastq.py.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import fasta_oracle as FO
import filter_outputs_oracle as RO
from oracle import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_KAT_CASES = 9


# ---- the routing core ------------------------------------------------------------------------------------------------

def model_route(m1, m2, pair, enabled1, enabled2, mode, mode_untrimmed, redirect):
    """(fired filter, destination) per record from the reference's chain (oracle.FILTER_CHAIN), PairedEndFilter's
    modes and the outputs of the filters (steps.py:70-180)."""
    if redirect & 4:                                    # --untrimmed-output: IsUntrimmed with a writer
        enabled1, enabled2 = enabled1 | 64, enabled2 | 64
    n = len(m1)
    fired = np.full(n, -1, dtype=np.int32)
    open_ = np.ones(n, dtype=bool)
    for k, name in enumerate(oracle.FILTER_CHAIN):
        bit = 1 << k
        e1, e2 = bool(enabled1 & bit), pair and bool(enabled2 & bit)
        if not e1 and not e2:
            continue
        f1, f2 = (m1 & bit) != 0, (m2 & bit) != 0
        md = mode_untrimmed if name == "discard_untrimmed" else mode
        if not e2:
            hit = f1
        elif not e1:
            hit = f2
        else:
            hit = (f1 | f2) if md == 0 else (f1 & f2) if md == 1 else f1
        fired[open_ & hit] = k
        open_ &= ~hit
    dest = np.where(fired < 0, 0, -1).astype(np.int32)
    for k, name in enumerate(oracle.FILTER_CHAIN):
        out = RO.OUTPUT_OF.get(name)
        if out is not None and redirect & (1 << RO.REDIRECT_NAMES.index(out)):
            dest[fired == k] = 1 + RO.REDIRECT_NAMES.index(out)
    return fired, dest


def hostsim_route(m1, m2, enabled1, enabled2, mode, mode_untrimmed, redirect):
    from util import hostsim_lib

    lib = hostsim_lib()
    lib.hs_fastq_route.argtypes = [C.c_int64, C.c_void_p, C.c_void_p] + [C.c_int] * 5 + [C.c_void_p, C.c_void_p]
    n = len(m1)
    fired, dest = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    lib.hs_fastq_route(n, m1.ctypes.data, m2.ctypes.data if m2 is not None else None, enabled1, enabled2, mode,
                       mode_untrimmed, redirect, fired.ctypes.data, dest.ctypes.data)
    return fired, dest


def test_routing_core_single_end_every_mask_and_filter_set():
    masks = np.arange(128, dtype=np.int32)
    for enabled in range(128):
        for redirect in range(8):
            got = hostsim_route(masks, None, enabled, 0, 0, 0, redirect)
            exp = model_route(masks, masks * 0, False, enabled, 0, 0, 0, redirect)
            assert (got[0] == exp[0]).all() and (got[1] == exp[1]).all(), (enabled, redirect)


def test_routing_core_pairs_every_mask_pair():
    """Every pair of failed-filter masks; every filter set of R1 with R2's equal to it, empty or its complement; every
    pair filter mode, the untrimmed override to "both" and every set of outputs."""
    m1, m2 = (a.ravel().astype(np.int32) for a in np.meshgrid(np.arange(128), np.arange(128), indexing="ij"))
    for enabled1 in range(128):
        for enabled2 in {enabled1, 0, 127 & ~enabled1}:
            for mode in range(3):
                for mode_untrimmed in {mode, 1}:
                    for redirect in range(8):
                        got = hostsim_route(m1, m2, enabled1, enabled2, mode, mode_untrimmed, redirect)
                        exp = model_route(m1, m2, True, enabled1, enabled2, mode, mode_untrimmed, redirect)
                        assert (got[0] == exp[0]).all() and (got[1] == exp[1]).all(), \
                            (enabled1, enabled2, mode, mode_untrimmed, redirect)


# ---- the redirect oracle against the reference's answers ----------------------------------------------------------------

def oracle_case(c):
    """({output: bytes or (bytes1, bytes2)}, counters of R1) of a filter_outputs_kat case from the redirect oracle."""
    o = c["options"]
    data = [RO.kat_file(k) for k in c["inputs"]]
    fmt = RO.input_format_of(data[0])
    if c["kind"] == "paired":
        sets = [FO.descriptors(FO.kat_adapters(o, key)) for key in ("specs1", "specs2")]
        kw = RO.kat_trimmer_kwargs(o)
        outs, c1, _ = RO.redirect_trim_paired(data[0], data[1], *sets[0], *sets[1], kw, kw,
                                              o.get("pair_filter", "any"), o.get("redirect", ()), input_format=fmt)
        return outs, c1
    descs, groups = FO.descriptors(FO.kat_adapters(o))
    return RO.redirect_trim(data[0], descs, groups, o.get("redirect", ()), input_format=fmt,
                            **RO.kat_trimmer_kwargs(o))


def test_kat_has_every_case():
    assert len(RO.filter_outputs_kat()["cases"]) == N_KAT_CASES


@pytest.mark.parametrize("case", [c["name"] for c in RO.filter_outputs_kat()["cases"]])
def test_redirect_oracle_reproduces_the_reference(case):
    c = next(x for x in RO.filter_outputs_kat()["cases"] if x["name"] == case)
    outs, counters = oracle_case(c)
    for name, exp in c["expected"].items():
        if c["kind"] == "paired":
            assert outs[name] == (RO.kat_file(exp[0]), RO.kat_file(exp[1])), name
        else:
            assert outs[name] == RO.kat_file(exp), name
    for k, v in c["counters"].items():
        assert counters[k] == v, k


def test_redirecting_changes_no_counter():
    """test_too_short_statistics[False / True] of the reference: the same counters with and without the output."""
    cases = {c["name"]: c for c in RO.filter_outputs_kat()["cases"]}
    assert oracle_case(cases["too_short_statistics"])[1] == oracle_case(cases["too_short_statistics_redirect"])[1]


# ---- tools/trim_fastq.py: the reference's command-line errors -------------------------------------------------------

def run_tool(tmp_path, args, inputs=1):
    files = []
    for i in range(inputs):
        p = tmp_path / f"in.{i + 1}.fastq"
        p.write_bytes(b"@r\nACGT\n+\nIIII\n")
        files.append(str(p))
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), *args, *files],
                          capture_output=True, text=True, cwd=tmp_path)


@pytest.mark.parametrize("args,inputs,message", [
    (["--too-short-output", "s.fastq", "-o", "o.fastq"], 1, "a minimum length must be provided with -m"),
    (["--too-long-output", "l.fastq", "-o", "o.fastq"], 1, "a maximum length must be provided with -M"),
    (["-m", "5", "--too-short-output", "s.fastq", "-o", "o.1.fastq", "-p", "o.2.fastq"], 2,
     "either none or both of the --too-short-output/--too-short-paired-output"),
    (["-M", "5", "--too-long-paired-output", "l.fastq", "-o", "o.1.fastq", "-p", "o.2.fastq"], 2,
     "either none or both of the --too-long-output/--too-long-paired-output"),
    (["--untrimmed-output", "u.fastq", "-o", "o.1.fastq", "-p", "o.2.fastq", "-a", "ACGT"], 2,
     "either none or both of the --untrimmed-output/--untrimmed-paired-output"),
    (["-m", "5", "--too-short-paired-output", "s.fastq", "-o", "o.fastq"], 1,
     "--too-short/long-paired-output cannot be used with single-end data"),
    (["--untrimmed-paired-output", "u.fastq", "-o", "o.fastq"], 1,
     "--untrimmed-paired-output can only be used when trimming paired-end reads"),
    (["--discard-trimmed", "--untrimmed-output", "u.fastq", "-o", "o.fastq"], 1,
     "Only one of the --discard-trimmed, --discard-untrimmed and --untrimmed-output"),
    (["--discard-untrimmed", "--untrimmed-output", "u.fastq", "-o", "o.fastq"], 1,
     "Only one of the --discard-trimmed, --discard-untrimmed and --untrimmed-output"),
    (["--discard-trimmed", "--discard-untrimmed", "-o", "o.fastq"], 1,
     "Only one of the --discard-trimmed, --discard-untrimmed and --untrimmed-output"),
    (["-m", "5", "--too-short-output", "s.fastq", "-a", "x=ACGT", "-o", "{name}.fastq"], 1,
     "--too-short-output and --too-long-output cannot be combined with demultiplexing"),
])
def test_trim_fastq_argument_errors(tmp_path, args, inputs, message):
    r = run_tool(tmp_path, args, inputs)
    assert r.returncode == 2, r.stderr
    assert message in r.stderr
    assert not any(p.name.startswith(("o.", "s.", "l.", "u.")) for p in tmp_path.iterdir())
