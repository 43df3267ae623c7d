#!/usr/bin/env python3
"""
Known answers of the reference for --max-aer (TooHighAverageErrorRate, predicates.py:74-95) and -z (ZeroCapper,
modifiers.py:806-822): tests/golden/quality_filters_kat.json.gz.

Needs $CUTADAPT_REFERENCE, a checkout of the reference (builds oracle/_ref on the fly):

    python tests/golden/make_quality_filters_golden.py

The cases are the reference's own tests, restated as data: the five parameter sets of test_too_high_average_error_rate
(tests/test_predicates.py:58-72, one of them the "3 x 0.1 > 0.3 in floating point" edge) and test_zero_capper
(tests/test_modifiers.py:72-77).  For every quality string the file also stores what the reference's
qualtrim.expected_errors returns, as float.hex(), so the device's sum can be compared at 0 ulp.  Boundary cases (a
rate equal to a string's average error rate, and one ulp below it) are added with the reference's expected_errors and
the predicate's comparison, ee / len > rate.  Re-running reproduces the file byte for byte.
"""
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import build_ref  # noqa: E402

build_ref.import_ref()
from cutadapt.qualtrim import expected_errors  # noqa: E402
from make_golden import dump  # noqa: E402

# tests/test_predicates.py:58-72: (qualities, rate, expected)
PREDICATE_CASES = [
    (chr(43) * 3, 0.1, True),               # 3 * 0.1 is larger than 0.3 due to floating point rounding
    (chr(43) * 3 + chr(33), 0.1, True),     # 3 * 0.1 + 1
    (chr(43) * 3 + chr(33), 0.33, False),
    (chr(43) * 3 + chr(33), 0.32, True),
    (chr(126) * 9 + chr(33), 0.1, True),    # 9 * 10^-9.3 + 1
]
# tests/test_modifiers.py:72-77: ZeroCapper() (quality base 33) on ("r1", "ACGT", "# !%")
ZERO_CAPPER_CASE = {"sequence": "ACGT", "qualities": "# !%", "quality_base": 33, "expected": "#!!%"}


def boundary_cases():
    """Rates at the average error rate of a string and one ulp below it: only the rate below fails the read."""
    out = []
    for quals in ("+" * 10, "+" * 7, "5" * 5, "?" * 4, "+" * 5 + "5" * 3, "#$%&'()*+,-./0123456789"):
        ee = expected_errors(quals)
        at = ee / len(quals)
        assert 0.0 < at < 1.0
        out.append((quals, at, False))
        out.append((quals, math.nextafter(at, 0.0), True))
    return out


def main():
    cases = []
    for quals, rate, expected in PREDICATE_CASES + boundary_cases():
        ee = expected_errors(quals)
        assert (ee / len(quals) > rate) == expected, (quals, rate)
        cases.append({"qualities": quals, "rate": rate.hex(), "expected": expected, "expected_errors": ee.hex()})
    dump("quality_filters_kat.json.gz", {"too_high_average_error_rate": cases, "zero_capper": ZERO_CAPPER_CASE})


if __name__ == "__main__":
    main()
