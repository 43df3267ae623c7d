#!/usr/bin/env python3
"""
Copies the known answer of the reference's paired-end info files (--info-file with --info-file-paired) from its own
tests ($CUTADAPT_REFERENCE/tests) into tests/golden/paired_rows_kat.json.gz: the two input files and the four expected
files as they are, and the case, which restates the command line in terms of cutadapt_b200's PairedFastqTrimmer.
These are test vectors, not source code.

    python tests/golden/make_paired_rows_golden.py  (needs $CUTADAPT_REFERENCE, a checkout of the reference; run once,
                                                      results committed)

The case: "inputs" = the two mate files, "expected" = {"output": [R1, R2], "info": [R1's rows, R2's rows]}; "specs1" /
"specs2" = the command line's [-a kind, adapter string] values, "options1" / "options2" = the trimmer's keyword
arguments of each mate, "argv" = the options of tools/trim_fastq.py (the file arguments are added by the test).  The
reference compares the info files ignoring trailing whitespace (assert_files_equal(..., ignore_trailing_space=True)).
"""
import gzip
import json
import os

REF = os.path.join(os.environ.get("CUTADAPT_REFERENCE", ""), "tests")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "paired_rows_kat.json.gz")
FILES = {}     # "data/<name>" / "cut/<name>" -> content (latin-1 text)


def store(rel):
    """The reference file tests/<rel> under the key <rel>."""
    with open(os.path.join(REF, rel), "rb") as f:
        FILES[rel] = f.read().decode("latin-1")
    return rel


CASES = [
    dict(name="paired_info_file", reference_test="tests/test_info_file.py:174",
         command="--info-file info1 --info-file-paired info2 -a r1adapt=TTAGACATAT -A r2adapt=CAGTGGAGTA -m 14",
         inputs=["data/paired.1.fastq", "data/paired.2.fastq"],
         expected=dict(output=["cut/paired.1.fastq", "cut/paired.2.fastq"],
                       info=["cut/paired.info1.txt", "cut/paired.info2.txt"]),
         options=dict(specs1=[["back", "r1adapt=TTAGACATAT"]], specs2=[["back", "r2adapt=CAGTGGAGTA"]],
                      options1=dict(minimum_length=14), options2=dict(minimum_length=14)),
         argv=["-a", "r1adapt=TTAGACATAT", "-A", "r2adapt=CAGTGGAGTA", "-m", "14"]),
]


def main():
    for c in CASES:
        for p in c["inputs"] + [p for v in c["expected"].values() for p in v]:
            store(p)
        print(f"{c['name']:24s} {c['reference_test']:32s} {c['command']}")
    blob = json.dumps(dict(cases=CASES, files=FILES), sort_keys=True).encode()
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:     # mtime=0: the same bytes on every run
        f.write(blob)
    print(len(CASES), "case,", len(FILES), "fixture files ->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
