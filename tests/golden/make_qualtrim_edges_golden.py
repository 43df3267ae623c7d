#!/usr/bin/env python3
"""
Quality strings at the edges of the device's quality scans, with the REFERENCE's answers:
tests/golden/qualtrim_edges_kat.json.gz.

Needs $CUTADAPT_REFERENCE, a checkout of the reference (builds oracle/_ref on the fly):

    python tests/golden/make_qualtrim_edges_golden.py

For every string it stores what the reference's quality_trim_index(q, cf, cb, base) returns; for the --nextseq-trim
entries nextseq_trim_index and then quality_trim_index on what is left (modifiers.py:834-858).  Families, each built
for both ends: bad tails of 0 .. 256 characters across the 32-character steps of the warp scan (trim_scan_warp,
cg_pscan.cuh), ties of the running maximum across a step, maxima on lane 0 / lane 31 / the last character, zero
increments, a partial sum of exactly 0 before the first negative one, windows that close, quality characters below the
base and bytes >= 128, for every cutoff pair and base of tests/quality_windows.py.  Which edges the corpus reaches is
counted with that module's restatement of qualtrim.pyx:22-73 and asserted here (and again by the CPU test).
Seeds are fixed; re-running reproduces the file byte for byte.
"""
import os
import random
import sys
from types import SimpleNamespace

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import build_ref  # noqa: E402

build_ref.import_ref()
from cutadapt.qualtrim import quality_trim_index, nextseq_trim_index  # noqa: E402
import quality_windows as QW  # noqa: E402
from make_golden import dump  # noqa: E402


def chars(incs, cutoff, base):
    """Quality string whose scan increments (cutoff - quality) are `incs`, in scan order from the 5' end; increments
    the printable range cannot express are clamped."""
    out = []
    for d in incs:
        v = base + cutoff - d
        out.append(chr(min(126, max(1, v))))
    return "".join(out)


def profiles(rng):
    """(family, increments in scan order) for one end; positive = worse than the cutoff."""
    out = []
    for t in QW.TAILS:
        out.append(("bad_tail", [rng.randint(1, 6) for _ in range(t)]))
        if t >= 31:
            out.append(("bad_tail_mixed", [rng.choice([3, 3, 2, -1, -2, 4]) for _ in range(t - 1)] + [40]))
    for k in (1, 2, 4, 7):                        # first maximum in step k - 1, the same sum again in step k
        i1 = 32 * (k - 1) + rng.randint(0, 31)
        i2 = 32 * k + rng.randint(0, 31)
        if (i2 - i1) % 2:
            i2 += 1
        a = (i2 - i1) // 2
        out.append(("max_tie", [1] * (i1 + 1) + [-1] * a + [1] * a + [-30]))
        out.append(("max_tie", [1] * (i1 + 1) + [0] * (32 * k - i1) + [-1, 1] * 3 + [-30]))
    for i in (32, 64, 96, 128, 160, 224):
        out.append(("max_lane0", [2] * (i + 1) + [-60]))
        out.append(("max_lane31", [2] * (i + 32) + [-60]))
    out.append(("max_last", [1] * 40))
    out.append(("max_last", [2] * 100))
    out.append(("zero_first", [0] + [3] * 10))
    out.append(("zero_first", [0, 0, 0] + [2] * 40))
    out.append(("zero_first", [0] + [-1]))
    out.append(("zero_run", [1] * 20 + [0] * 20 + [2] * 10))
    out.append(("zero_run", [2] * 30 + [0] * 40 + [-80]))
    out.append(("zero_run", [1] * 60 + [0] * 10 + [1] * 5))
    for b in (32, 64, 96):                        # sum 0 just before the first negative one on lane 0
        h = b // 2
        out.append(("zero_then_negative", [1] * h + [-1] * h + [-1]))
    for b in (63, 95, 127):                       # ... on lane 31
        h = (b - 1) // 2
        out.append(("zero_then_negative", [1] * h + [-1] * h + [0] + [-1]))
    for b in (32, 63, 64, 95):                    # first negative sum on lane 0 / 31 of a later step
        out.append(("negative_lane", [1] * (b - 5) + [-(b - 5) - 1]))
    return out


def quality_entries():
    rng = random.Random(2101)
    out = []
    for cf, cb in QW.CUTOFFS:
        for base in QW.BASES:
            def good(k):
                return chars([-30] * k, max(cf, cb), base)

            for fam, incs in profiles(rng):
                for end in "53":
                    cutoff = cf if end == "5" else cb
                    tail = chars(incs, cutoff, base)
                    lengths = {len(tail), len(tail) + 1, len(tail) + 5, 150, 160, 161, 200, 256, 257, 300}
                    if fam != "bad_tail":
                        lengths = {len(tail) + 3, max(len(tail) + 1, rng.choice([150, 200, 256, 290]))}
                    for n in sorted(x for x in lengths if x >= len(tail)):
                        mid = good(n - len(tail))
                        q = tail + mid if end == "5" else mid + tail[::-1]
                        out.append([f"{fam}{end}", q, cf, cb, base])
            # windows that close: bad from both ends, and (cf > cb) 5' and 3' trims that meet or cross
            for n in (1, 33, 100, 256):
                out.append(["closed_both", chars([max(cf, cb) + 5] * n, 0, base), cf, cb, base])
            for _ in range(400 if cf > cb else 60):
                n = rng.randint(2, 70)
                q = "".join(chr(base + rng.choice([cb - 8, cb + 2, (cf + cb) // 2, cf + 5, cf - 3])) for _ in range(n))
                q = "".join(c if 1 <= ord(c) <= 126 else chr(base) for c in q)
                s, e = QW.raw_trim(q, cf, cb, base)
                if s >= e and not (s == n and e == 0):
                    out.append(["closed_cross", q, cf, cb, base])
            # below the base, bytes >= 128 (read as signed char: very bad qualities)
            for n in (20, 40, 70, 150, 260):
                q = "".join(chr(max(1, base - rng.randint(1, 20))) if rng.random() < 0.6 else chr(base + 40) for _ in range(n))
                out.append(["below_base", q, cf, cb, base])
            for t in (1, 32, 33, 70):
                for end in "53":
                    tail = "".join(chr(rng.randint(128, 255)) for _ in range(t))
                    mid = good(rng.choice([40, 120]))
                    out.append(["byte>=128" + end, tail + mid if end == "5" else mid + tail, cf, cb, base])
            for _ in range(40):                     # random strings around the cutoffs
                n = rng.randint(0, 300)
                c = rng.choice([cf, cb])
                q = "".join(chr(min(126, max(1, base + c + rng.choice([-3, -1, 0, 1, 2, 10])))) for _ in range(n))
                out.append(["random", q, cf, cb, base])
    for e in out:
        e.extend(quality_trim_index(e[1], e[2], e[3], e[4]))
    return out


def nextseq_entries():
    rng = random.Random(2102)
    out = []
    for ns_cut in QW.NEXTSEQ_CUTOFFS:
        for base in QW.BASES:
            for cf, cb in ((0, 30), (20, 30)):     # -q above the NextSeq cutoff: the tail is left to -q
                for g in (0, 1, 5, 30, 40):
                    for t in (0, 31, 32, 33, 64, 65, 128):
                        body = rng.randint(10, 90)
                        seq = "".join(rng.choice("ACT") for _ in range(body + t)) + "G" * g
                        q = (chr(base + 38) * body + "".join(chr(base + rng.randint(26, 29)) for _ in range(t))
                             + chr(base + 40) * g)
                        stop = nextseq_trim_index(SimpleNamespace(sequence=seq, qualities=q), ns_cut, base)
                        s, e = quality_trim_index(q[:stop], cf, cb, base)
                        out.append(["nextseq", seq, q, ns_cut, cf, cb, base, stop, s, e])
    return out


def main():
    corpus = {"quality": quality_entries(), "nextseq": nextseq_entries()}
    for fam, q, cf, cb, base, s, e in corpus["quality"]:
        assert QW.trim_index(q, cf, cb, base) == (s, e), (fam, q, cf, cb, base)
    for fam, seq, q, ns_cut, cf, cb, base, stop, s, e in corpus["nextseq"]:
        assert QW.nextseq_index(seq, q, ns_cut, base) == stop
    missing = QW.missing(corpus)
    assert not missing, missing
    dump("qualtrim_edges_kat.json.gz", corpus)


if __name__ == "__main__":
    main()
