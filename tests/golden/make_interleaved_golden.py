#!/usr/bin/env python3
"""
Copies the known-answer cases of the reference's interleaved paired-end data (--interleaved) from its own tests
($CUTADAPT_REFERENCE/tests) into tests/golden/interleaved_kat.json.gz: the input and expected files as they are, the
case list, which restates each command line in terms of cutadapt_b200's PairedFastqTrimmer, and the command-line
errors the reference's tests pin.  These are test vectors, not source code.

    python tests/golden/make_interleaved_golden.py  (needs $CUTADAPT_REFERENCE, a checkout of the reference; run once,
                                                      results committed)

Every case: "inputs" = one interleaved file or two mate files; "expected" maps an output ("output" = -o / -p,
"untrimmed") to one file (written interleaved) or two (R1, R2).  Options: "specs1" / "specs2" = the command line's
[-a kind, adapter string] values, "options1" / "options2" = the trimmer's keyword arguments of each mate, "redirect" =
the filter outputs given.  test_separate_minmaxlength (test_paired.py:614-654) writes its input and expected FASTA files
itself; its 96 parameter sets are restated here from the test's own parametrization and stored under "gen/...".
"errors": command lines tools/trim_fastq.py must refuse as the reference does (argv names stored files by key).
"""
import gzip
import json
import os
from itertools import product

REF = os.path.join(os.environ.get("CUTADAPT_REFERENCE", ""), "tests")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "interleaved_kat.json.gz")
FILES = {}     # "data/<name>" / "cut/<name>" / "gen/<name>" -> content (latin-1 text)


def store(rel):
    """The reference file tests/<rel> under the key <rel>."""
    with open(os.path.join(REF, rel), "rb") as f:
        FILES[rel] = f.read().decode("latin-1")
    return rel


PL = "tests/test_paired.py"
QMM = dict(quality_cutoff=[0, 20], minimum_length=14, maximum_length=90)
ADAPTERS = dict(specs1=[["back", "TTAGACATAT"]], specs2=[["back", "CAGTGGAGTA"]], options1=QMM, options2=QMM)
CASES = [
    ("interleaved_in_and_out", f"{PL}:429", "-q 20 -a TTAGACATAT -A CAGTGGAGTA -m 14 -M 90 --interleaved",
     ["data/interleaved.fastq"], dict(output=["cut/interleaved.fastq"]), ADAPTERS),
    ("interleaved_in", f"{PL}:439", "-q 20 -a TTAGACATAT -A CAGTGGAGTA -m 14 -M 90 --interleaved (-o, -p)",
     ["data/interleaved.fastq"], dict(output=["cut/pairedq.1.fastq", "cut/pairedq.2.fastq"]), ADAPTERS),
    ("interleaved_out", f"{PL}:450", "-q 20 -a TTAGACATAT -A CAGTGGAGTA -m 14 -M 90 --interleaved (two inputs, -o)",
     ["data/paired.1.fastq", "data/paired.2.fastq"], dict(output=["cut/interleaved.fastq"]), ADAPTERS),
    # the main outputs are two files; the untrimmed output has no paired path and is interleaved
    ("interleaved_untrimmed_output", f"{PL}:471", "--interleaved -a XXXX -o o1 -p o2 --untrimmed-output untrimmed",
     ["data/interleaved.fastq"], dict(untrimmed=["data/interleaved.fastq"]),
     dict(specs1=[["back", "XXXX"]], specs2=[], options1={}, options2={}, redirect=["untrimmed"])),
]


def separate_minmaxlength():
    """test_separate_minmaxlength[name_op, l1, l2, m]: one pair r{l1}:{l2} of A-runs; kept iff each mate with a length
    passes its -m / -M.  The files are written as the test writes them (print adds the final newline)."""
    ops = (("m", lambda x, y: x >= y), ("M", lambda x, y: x <= y))
    out = []
    for (name, func), l1, l2, (m1, m2) in product(ops, range(1, 5), range(1, 5), [(2, 3), (2, None), (None, 3)]):
        record = ">r{}:{}\n{}\n".format(l1, l2, "A" * l1) + ">r{}:{}\n{}".format(l1, l2, "A" * l2)
        keep = (m1 is None or func(l1, m1)) and (m2 is None or func(l2, m2))
        ident = f"{name}-{l1}-{l2}-{m1}-{m2}"
        FILES[f"gen/{ident}.in.fasta"] = record + "\n"
        FILES[f"gen/{ident}.expected.fasta"] = record + "\n" if keep else ""
        key = "minimum_length" if name == "m" else "maximum_length"
        arg = "{}:{}".format("" if m1 is None else m1, "" if m2 is None else m2)
        out.append(dict(name=f"separate_minmaxlength[{ident}]", reference_test=f"{PL}:614",
                        command=f"--interleaved -o out.fasta -{name} {arg} in.fasta",
                        inputs=[f"gen/{ident}.in.fasta"], expected=dict(output=[f"gen/{ident}.expected.fasta"]),
                        options=dict(specs1=[], specs2=[], options1={} if m1 is None else {key: m1},
                                     options2={} if m2 is None else {key: m2}),
                        argv=["--interleaved", f"-{name}", arg]))
    return out


ERRORS = [
    # two inputs, -o and -p, and --interleaved: neither interleaved input nor interleaved output (cli.py:568-575)
    dict(name="interleaved_neither_nor", reference_test=f"{PL}:461",
         argv=["-a", "XX", "--interleaved", "-o", "{out1}", "-p", "{out2}", "data/paired.1.fastq", "data/paired.2.fastq"]),
    # -m LEN:LEN2 on single-end data (cli.py:731-735)
    dict(name="separate_minlength_single", reference_test=f"{PL}:657", argv=["-m", "5:7", "-o", "{out1}",
                                                                              "data/small.fastq"]),
]


def main():
    cases = []
    for name, test, cmd, inputs, exp, opts in CASES:
        cases.append(dict(name=name, reference_test=test, command=cmd, inputs=[store(p) for p in inputs],
                          expected={k: [store(p) for p in v] for k, v in exp.items()}, options=opts))
    cases += separate_minmaxlength()
    store("data/paired.1.fastq")
    store("data/paired.2.fastq")
    store("data/small.fastq")
    for c in cases:
        print(f"{c['name']:40s} {c['reference_test']:26s} {c['command']}")
    blob = json.dumps(dict(cases=cases, errors=ERRORS, files=FILES), sort_keys=True).encode()
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:     # mtime=0: the same bytes on every run
        f.write(blob)
    print(len(cases), "cases,", len(ERRORS), "errors,", len(FILES), "fixture files ->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
