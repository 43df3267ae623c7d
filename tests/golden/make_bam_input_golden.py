#!/usr/bin/env python3
"""
Copies the reference's unaligned BAM input ($CUTADAPT_REFERENCE/tests/data/small.bam) as raw bytes, and the command line
and expected file of the reference case that reads it, into tests/golden/bam_input_kat.json.gz.  The BAM file is stored
as it is (BGZF members and EOF block included), so that the device reader inflates and decodes exactly the reference's
bytes.  These are test vectors, not source code.

    python tests/golden/make_bam_input_golden.py    (needs $CUTADAPT_REFERENCE, a checkout of the reference; run once,
                                                     results committed)

The case: name, reference test, command line, input, expected output (tests/cut/...) and the options: "adapters" as
[kind, sequence, name or None] plus the error rate / overlap defaults of the command line.  The output is written sorted
by key, so the file is deterministic.
"""
import gzip
import io
import json
import os

REF = os.path.join(os.environ.get("CUTADAPT_REFERENCE", ""), "tests")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bam_input_kat.json.gz")
CASES = [
    ("small_bam", "tests/test_commandline.py:82", "-a TTAGACATATCTCCGTCG", "small.bam", "small_from_bam.fastq",
     [["back", "TTAGACATATCTCCGTCG", None]]),
]


def read(rel):
    with open(os.path.join(REF, rel), "rb") as f:
        return f.read().decode("latin-1")


def main():
    files, cases = {}, []
    for name, where, cmd, inp, expected, adapters in CASES:
        files["data/" + inp] = read("data/" + inp)
        files["cut/" + expected] = read("cut/" + expected)
        cases.append(dict(name=name, reference=where, command=cmd, input="data/" + inp, expected="cut/" + expected,
                          adapters=adapters, error_rate=0.1, min_overlap=3))
    text = json.dumps({"files": files, "cases": cases}, sort_keys=True, indent=0).encode()
    buf = io.BytesIO()
    with gzip.GzipFile(fileobj=buf, mode="wb", mtime=0, filename="") as g:
        g.write(text)
    with open(OUT, "wb") as f:
        f.write(buf.getvalue())
    print(f"{OUT}: {len(cases)} cases, {len(files)} files")


if __name__ == "__main__":
    main()
