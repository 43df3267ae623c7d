#!/usr/bin/env python3
"""
Copies the reference's six gzip-compressed inputs ($CUTADAPT_REFERENCE/tests/data/*.gz) as raw bytes, and the command
line and expected files of every reference case that reads one of them, into tests/golden/gzip_input_kat.json.gz.  The
inputs are stored compressed, header fields (FNAME) included, so that the device reader inflates exactly the reference's
bytes: all are single members except multiblock.fastq.gz.  These are test vectors, not source code.

    python tests/golden/make_gzip_input_golden.py   (needs $CUTADAPT_REFERENCE, a checkout of the reference; run once,
                                                     results committed)

Each case: name, reference test, command line, input, expected output (tests/cut/...), "info" (the expected
--info-file text, or None) and the options: "adapters" as [kind, sequence, name or None] plus the error rate / overlap
defaults of the command line.  The output is written sorted by key, so the file is deterministic.
"""
import gzip
import io
import json
import os

REF = os.path.join(os.environ.get("CUTADAPT_REFERENCE", ""), "tests")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gzip_input_kat.json.gz")
INPUTS = ["illumina.fastq.gz", "multiblock.fastq.gz", "s_1_sequence.txt.gz", "simple.fasta.gz", "small.fastq.gz",
          "underscore_fastq.gz"]
TC, CL, TI = "tests/test_compression.py", "tests/test_commandline.py", "tests/test_info_file.py"
ANY = ["anywhere", "TTAGACATATCTCCGTCG", None]
CASES = [
    ("multiblock", f"{TC}:7", "-b TTAGACATATCTCCGTCG", "multiblock.fastq.gz", "small.fastq", None, [ANY]),
    ("extension_txt_gz", f"{TC}:12", "-b TTAGACATATCTCCGTCG", "s_1_sequence.txt.gz", "s_1_sequence.txt", None, [ANY]),
    ("compressed_fasta", f"{TC}:17", "", "simple.fasta.gz", "simple.fasta", None, []),
    ("underscore_fastq_gz", f"{TC}:64", "-b TTAGACATATCTCCGTCG", "underscore_fastq.gz", "small.fastq", None, [ANY]),
    ("cores_autodetect", f"{CL}:775", "--cores 0 -b TTAGACATATCTCCGTCG", "small.fastq.gz", "small.fastq", None, [ANY]),
    ("iupac", f"{CL}:375", "-a VCCGAMCYUCKHRKDCUBBCNUWNSGHCGU", "illumina.fastq.gz", "illumina.fastq", None,
     [["back", "VCCGAMCYUCKHRKDCUBBCNUWNSGHCGU", None]]),
    ("named_adapter", f"{CL}:447", "-a MY_ADAPTER=GCCGAACTTCTTAGACTGCCTTAAGGACGT", "illumina.fastq.gz", "illumina.fastq",
     None, [["back", "GCCGAACTTCTTAGACTGCCTTAAGGACGT", "MY_ADAPTER"]]),
    ("rna", f"{CL}:455", "-a GCCGAACUUCUUAGACUGCCUUAAGGACGU", "illumina.fastq.gz", "illumina.fastq", None,
     [["back", "GCCGAACUUCUUAGACUGCCUUAAGGACGU", None]]),
    ("info_file", f"{TI}:14", "--info-file info.txt -a adapt=GCCGAACTTCTTAGACTGCCTTAAGGACGT", "illumina.fastq.gz",
     "illumina.fastq", "illumina.info.txt", [["back", "GCCGAACTTCTTAGACTGCCTTAAGGACGT", "adapt"]]),
]


def read(rel):
    with open(os.path.join(REF, rel), "rb") as f:
        return f.read().decode("latin-1")


def main():
    files = {"data/" + name: read("data/" + name) for name in INPUTS}
    cases = []
    for name, where, cmd, inp, expected, info, adapters in CASES:
        files["cut/" + expected] = read("cut/" + expected)
        if info:
            files["cut/" + info] = read("cut/" + info)
        cases.append(dict(name=name, reference=where, command=cmd, input="data/" + inp, expected="cut/" + expected,
                          info="cut/" + info if info else None, adapters=adapters, error_rate=0.1, min_overlap=3))
    text = json.dumps({"files": files, "cases": cases}, sort_keys=True, indent=0).encode()
    buf = io.BytesIO()
    with gzip.GzipFile(fileobj=buf, mode="wb", mtime=0, filename="") as g:
        g.write(text)
    with open(OUT, "wb") as f:
        f.write(buf.getvalue())
    print(f"{OUT}: {len(cases)} cases, {len(files)} files")


if __name__ == "__main__":
    main()
