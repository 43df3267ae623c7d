#!/usr/bin/env python3
"""
Copies the known-answer cases of the reference's filter outputs (--too-short-output, --too-long-output,
--untrimmed-output and their paired forms) from its own tests ($CUTADAPT_REFERENCE/tests) into
tests/golden/filter_outputs_kat.json.gz: the input and expected files as they are, plus the case list, which restates
each command line in terms of cutadapt_b200's FastqTrimmer / PairedFastqTrimmer, and the counters the reference's test
asserts.  These are test vectors, not source code.

    python tests/golden/make_filter_outputs_golden.py  (needs $CUTADAPT_REFERENCE, a checkout of the reference; run once,
                                                        results committed)

Case kinds: "single" and "paired".  "expected" maps an output ("output" = -o / -p, "too_short", "too_long",
"untrimmed") to its expected file (a list of two for pairs).  Options: "specs" (single-end) or "specs1" / "specs2"
(paired) = the command line's [-a/-g/-b kind, adapter string] values, "redirect" = the filter outputs given, and the
trimmer's keyword arguments ("pair_filter" for pairs).  "counters": what the reference's test asserts, in the names of
cg_fastq_result (n_written = stats.written, bp_out = stats.written_bp[0], discarded = stats.filtered["discard_untrimmed"]).
"""
import gzip
import json
import os

REF = os.path.join(os.environ.get("CUTADAPT_REFERENCE", ""), "tests")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "filter_outputs_kat.json.gz")
FILES = {}     # "data/<name>" / "cut/<name>" -> content (latin-1 text)


def store(rel):
    """The reference file tests/<rel> under the key <rel>."""
    with open(os.path.join(REF, rel), "rb") as f:
        FILES[rel] = f.read().decode("latin-1")
    return rel


CL = "tests/test_commandline.py"
PL = "tests/test_paired.py"
A = "TTAGACATATCTCCGTCG"
SINGLE = [
    ("untrimmed_output", f"{CL}:523", f"-a {A} --untrimmed-output untrimmed.fastq", "data/small.fastq",
     dict(output="cut/small.trimmed.fastq", untrimmed="cut/small.untrimmed.fastq"),
     dict(specs=[["back", A]], redirect=["untrimmed"]), dict(with_adapters=2, n_written=2, bp_out=46)),
    ("too_short", f"{CL}:141", f"-m 5 -a {A} --too-short-output tooshort.fa", "data/lengths.fa",
     dict(output="cut/minlen.fa", too_short="data/tooshort.fa"),
     dict(specs=[["back", A]], minimum_length=5, redirect=["too_short"]), dict(too_short=5)),
    ("too_long", f"{CL}:189", f"-M 5 -a {A} --too-long-output toolong.fa", "data/lengths.fa",
     dict(output="cut/maxlen.fa", too_long="data/toolong.fa"),
     dict(specs=[["back", A]], maximum_length=5, redirect=["too_long"]), dict(too_long=5)),
    # test_too_short_statistics[False / True]: redirecting changes no counter
    ("too_short_statistics", f"{CL}:165", f"-a {A} -m 24", "data/small.fastq", dict(),
     dict(specs=[["back", A]], minimum_length=24), dict(with_adapters=2, n_written=2, bp_out=58, too_short=1)),
    ("too_short_statistics_redirect", f"{CL}:165", f"--too-short-output /dev/null -a {A} -m 24", "data/small.fastq",
     dict(), dict(specs=[["back", A]], minimum_length=24, redirect=["too_short"]),
     dict(with_adapters=2, n_written=2, bp_out=58, too_short=1)),
]
PAIRED = [
    ("paired_too_short", f"{PL}:515", "-a TTAGACATAT -A CAGTGGAGTA -m 14 --too-short-output 1 --too-short-paired-output 2",
     dict(output=["cut/paired.1.fastq", "cut/paired.2.fastq"],
          too_short=["cut/paired-too-short.1.fastq", "cut/paired-too-short.2.fastq"]),
     dict(specs1=[["back", "TTAGACATAT"]], specs2=[["back", "CAGTGGAGTA"]], minimum_length=14, redirect=["too_short"])),
    ("paired_too_long", f"{PL}:531", "-a TTAGACATAT -A CAGTGGAGTA -M 14 --too-long-output 1 --too-long-paired-output 2",
     dict(output=["cut/paired-too-short.1.fastq", "cut/paired-too-short.2.fastq"],
          too_long=["cut/paired.1.fastq", "cut/paired.2.fastq"]),
     dict(specs1=[["back", "TTAGACATAT"]], specs2=[["back", "CAGTGGAGTA"]], maximum_length=14, redirect=["too_long"])),
    ("paired_untrimmed_first", f"{PL}:58",
     "-a TTAGACATAT --pair-filter=first --untrimmed-output 1 --untrimmed-paired-output 2",
     dict(output=["cut/paired-trimmed.1.fastq", "cut/paired-trimmed.2.fastq"],
          untrimmed=["cut/paired-untrimmed.1.fastq", "cut/paired-untrimmed.2.fastq"]),
     dict(specs1=[["back", "TTAGACATAT"]], specs2=[], pair_filter="first", redirect=["untrimmed"])),
    # no R2 adapters: the pair filter of the untrimmed output is "both" whatever --pair-filter says
    ("paired_untrimmed_automatic", f"{PL}:81", "-a TTAGACATAT --untrimmed-output 1 --untrimmed-paired-output 2",
     dict(output=["cut/paired-trimmed.1.fastq", "cut/paired-trimmed.2.fastq"],
          untrimmed=["cut/paired-untrimmed.1.fastq", "cut/paired-untrimmed.2.fastq"]),
     dict(specs1=[["back", "TTAGACATAT"]], specs2=[], redirect=["untrimmed"])),
]


def main():
    cases = []
    for name, test, cmd, inp, exp, opts, counters in SINGLE:
        cases.append(dict(name=name, kind="single", reference_test=test, command=cmd, inputs=[store(inp)],
                          expected={k: store(v) for k, v in exp.items()}, options=opts, counters=counters))
    for name, test, cmd, exp, opts in PAIRED:
        cases.append(dict(name=name, kind="paired", reference_test=test, command=cmd,
                          inputs=[store("data/paired.1.fastq"), store("data/paired.2.fastq")],
                          expected={k: [store(v[0]), store(v[1])] for k, v in exp.items()}, options=opts, counters={}))
    for c in cases:
        print(f"{c['kind']:7s} {c['name']:30s} {c['reference_test']:30s} {c['command']}")
    with gzip.open(OUT, "wt", compresslevel=9) as f:
        json.dump(dict(cases=cases, files=FILES), f, sort_keys=True)
    print(len(cases), "cases,", len(FILES), "fixture files ->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
