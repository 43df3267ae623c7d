"""
Filter outputs on top of the FASTQ oracle (test infrastructure): --too-short-output, --too-long-output,
--untrimmed-output and their paired forms, as SingleEndFilter / PairedEndFilter with a writer do it (steps.py:70-180).
oracle._fastq_evaluate gives every read as modified and the verdict of every filter; the first enabled filter in chain
order that fires counts the read, and writes it to its output when it has one.  Each output has its own format.
"""
from oracle import oracle

import fasta_oracle

# filter of the chain -> the output that keeps what it removes; the outputs in the order of the CG_REDIRECT_* bits
OUTPUT_OF = {"too_short": "too_short", "too_long": "too_long", "discard_untrimmed": "untrimmed"}
REDIRECT_NAMES = ("too_short", "too_long", "untrimmed")
COUNTER_NAMES = ("n_written", "bp_out", "too_short", "too_long", "too_many_n", "too_many_expected_errors", "discarded",
                 "casava_filtered")


def _record(fmt, name, ts, tq):
    return fasta_oracle.fasta_record(name, ts) if fmt == "fasta" else oracle._fastq_record(name, ts, tq)


def _formats(redirect, formats, input_format, output_format):
    main = output_format or input_format
    return {"output": main, **{name: (formats or {}).get(name, main) for name in redirect}}


def _destination(fired, redirect):
    """The output a removed read goes to, or None (dropped)."""
    out = OUTPUT_OF.get(fired)
    return out if out in redirect else None


def redirect_trim(data: bytes, adapters=None, groups=None, redirect=(), formats=None, input_format="fastq",
                  output_format=None, **options):
    """({"output": bytes, <redirected output>: bytes}, counters) of one single-end chunk."""
    options = dict(options)
    if "untrimmed" in redirect:
        options["discard_untrimmed"] = True                 # the untrimmed output is IsUntrimmed with a writer
    fmt = _formats(redirect, formats, input_format, output_format)
    evaluated, enabled, c = oracle._fastq_evaluate(fasta_oracle._input(data, input_format, options), adapters, groups,
                                                   **options)
    c.update({k: 0 for k in COUNTER_NAMES})
    outs = {name: [] for name in fmt}
    for name, ts, tq, fails in evaluated:
        fired = next((f for f in enabled if fails[f]), None)
        if fired is not None:
            c[oracle._FILTER_COUNTER.get(fired, fired)] += 1
            dest = _destination(fired, redirect)
            if dest is not None:
                outs[dest].append(_record(fmt[dest], name, ts, tq))
            continue
        c["n_written"] += 1
        c["bp_out"] += len(ts)
        outs["output"].append(_record(fmt["output"], name, ts, tq))
    return {k: b"".join(v) for k, v in outs.items()}, c


def redirect_trim_paired(data1: bytes, data2: bytes, adapters1=None, groups1=None, adapters2=None, groups2=None,
                         options1=None, options2=None, pair_filter="any", redirect=(), formats=None,
                         input_format="fastq", output_format=None):
    """({"output": (bytes1, bytes2), <redirected output>: (bytes1, bytes2)}, counters1, counters2) of a paired chunk.
    With adapters on one mate only, the untrimmed filter tests "both" (cli.py:859-893)."""
    options1, options2 = dict(options1 or {}), dict(options2 or {})
    if "untrimmed" in redirect:
        options1["discard_untrimmed"] = options2["discard_untrimmed"] = True
    fmt = _formats(redirect, formats, input_format, output_format)
    ev1, en1, c1 = oracle._fastq_evaluate(fasta_oracle._input(data1, input_format, options1), adapters1, groups1,
                                          **options1)
    ev2, en2, c2 = oracle._fastq_evaluate(fasta_oracle._input(data2, input_format, options2), adapters2, groups2,
                                          second_mate=True, **options2)
    assert len(ev1) == len(ev2)
    for c in (c1, c2):
        c.update({k: 0 for k in COUNTER_NAMES})
    outs = {name: ([], []) for name in fmt}
    for (n1, s1, q1, f1), (n2, s2, q2, f2) in zip(ev1, ev2):
        fired = None
        for flt in oracle.FILTER_CHAIN:
            e1, e2 = flt in en1, flt in en2
            if not e1 and not e2:
                continue
            mode = "both" if flt == "discard_untrimmed" and (not adapters1 or not adapters2) else pair_filter
            if not e2:
                hit = f1[flt]
            elif not e1:
                hit = f2[flt]
            else:
                hit = {"any": f1[flt] or f2[flt], "both": f1[flt] and f2[flt], "first": f1[flt]}[mode]
            if hit:
                fired = flt
                break
        dest = "output"
        if fired is not None:
            for c in (c1, c2):
                c[oracle._FILTER_COUNTER.get(fired, fired)] += 1
            dest = _destination(fired, redirect)
            if dest is None:
                continue
        else:
            for c in (c1, c2):
                c["n_written"] += 1
            c1["bp_out"] += len(s1)
            c2["bp_out"] += len(s2)
        outs[dest][0].append(_record(fmt[dest], n1, s1, q1))
        outs[dest][1].append(_record(fmt[dest], n2, s2, q2))
    return {k: (b"".join(a), b"".join(b)) for k, (a, b) in outs.items()}, c1, c2


# ---- the known-answer cases of tests/golden/filter_outputs_kat.json.gz (make_filter_outputs_golden.py) -------------

_KAT = None


def filter_outputs_kat():
    global _KAT
    if _KAT is None:
        from util import golden

        _KAT = golden("filter_outputs_kat.json.gz")
    return _KAT


def kat_file(key) -> bytes:
    return filter_outputs_kat()["files"][key].encode("latin-1")


def input_format_of(data: bytes) -> str:
    """"fasta" or "fastq" from the first byte, as the reference detects it (files.py:314-333)."""
    return "fasta" if data[:1] in (b">", b"#") else "fastq"


TRIMMER_KEYS = ("minimum_length", "maximum_length")


def kat_trimmer_kwargs(options) -> dict:
    return {k: options[k] for k in TRIMMER_KEYS if k in options}
