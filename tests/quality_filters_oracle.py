"""
--max-aer (TooHighAverageErrorRate, predicates.py:74-95) and -z (ZeroCapper, modifiers.py:806-822) on top of the FASTQ
oracle (test infrastructure).  oracle._fastq_evaluate runs the modifier chain up to NEndTrimmer; evaluate() puts
ZeroCapper behind it (the last modifier, cli.py:1129-1146), judges --max-ee on the capped qualities, puts the new
predicate behind --max-ee in the chain (cli.py:756-783) and caps the quality column of the info rows of reads without a
match (those print the modified read, steps.py:249-251; rows of a match print the original read, steps.py:232-246).
extended() installs evaluate() and the longer chain in the oracle module for the duration of a with block, so that
every oracle built on it -- single-end, paired, demultiplexing, filter outputs, interleaved, rows, FASTQ -> FASTA --
takes the two options.  Also the known answers of tests/golden/quality_filters_kat.json.gz.
"""
import contextlib

from oracle import oracle

_CHAIN, _evaluate = oracle.FILTER_CHAIN, oracle._fastq_evaluate
FILTER_CHAIN = _CHAIN[:4] + ("too_high_average_error_rate",) + _CHAIN[4:]


def cap_qualities(qualities: str, base: int = 33) -> str:
    """ZeroCapper: every character below chr(base) becomes chr(base)."""
    return qualities.translate(str.maketrans("".join(map(chr, range(base))), chr(base) * base))


def _expected_errors(qualities: str) -> float:
    ee = oracle.expected_errors(qualities)
    if ee < 0:                                  # the reference's expected_errors raises
        raise ValueError(f"quality character outside [33, 126] in {qualities!r}")
    return ee


def too_high_average_error_rate(qualities: str, rate: float) -> bool:
    """TooHighAverageErrorRate.test: a read of length 0 passes."""
    if not qualities:
        return False
    return _expected_errors(qualities) / len(qualities) > rate


def evaluate(data, adapters, groups, max_average_error_rate=None, zero_cap=False, max_expected_errors=-1.0,
             quality_base=33, info_rows=None, **options):
    """oracle._fastq_evaluate with the two options (defaults off).  Raises ValueError for a rate outside (0, 1), and
    for a quality character outside [33, 126] when a quality filter is on, as the reference does."""
    rate = max_average_error_rate
    if rate is not None and not 0.0 < rate < 1.0:
        raise ValueError(f"max_error_rate must be between 0.0 and 1.0, got {rate}.")
    rows = [] if info_rows is not None else None
    chain, oracle.FILTER_CHAIN = oracle.FILTER_CHAIN, _CHAIN       # the chain _fastq_evaluate names its filters by
    try:
        out, enabled, c = _evaluate(data, adapters, groups, quality_base=quality_base, info_rows=rows, **options)
    finally:
        oracle.FILTER_CHAIN = chain
    on = set(enabled)
    if max_expected_errors >= 0:
        on.add("too_many_expected_errors")
    if rate is not None:
        on.add("too_high_average_error_rate")
    enabled = [name for name in FILTER_CHAIN if name in on]
    c["too_high_average_error_rate"] = 0
    result = []
    for name, ts, tq, fails, *rest in out:
        if zero_cap:
            tq = cap_qualities(tq, quality_base)
        fails = dict(fails)
        fails["too_many_expected_errors"] = max_expected_errors >= 0 and _expected_errors(tq) > max_expected_errors
        fails["too_high_average_error_rate"] = rate is not None and too_high_average_error_rate(tq, rate)
        result.append((name, ts, tq, fails, *rest))
    if info_rows is not None:
        for row in rows:
            fields = row.split("\t")
            if zero_cap and len(fields) == 4 and fields[1] == "-1":     # a read without a match: name, -1, seq, qual
                fields[3] = cap_qualities(fields[3], quality_base)
            info_rows.append("\t".join(fields))
    return result, enabled, c


@contextlib.contextmanager
def extended():
    """The oracle module with evaluate() and FILTER_CHAIN in place of its own, within the with block."""
    saved = oracle._fastq_evaluate, oracle.FILTER_CHAIN
    oracle._fastq_evaluate, oracle.FILTER_CHAIN = evaluate, FILTER_CHAIN
    try:
        yield oracle
    finally:
        oracle._fastq_evaluate, oracle.FILTER_CHAIN = saved


def quality_filters_kat():
    from util import golden

    return golden("quality_filters_kat.json.gz")
