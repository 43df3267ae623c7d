#!/usr/bin/env python3
"""
Copies the FASTA known-answer cases of the reference's own tests ($CUTADAPT_REFERENCE/tests: run(params, expected,
input) compares cutadapt's output with tests/cut/<expected>) into tests/golden/fasta_kat.json.gz.  Inputs and expected
files are stored as they are (FASTA, comments and line-wrapped sequences included), plus the case list, which restates
each command line in terms of cutadapt_b200's FASTQ/FASTA entry point.  These are test vectors, not source code.

    python tests/golden/make_fasta_golden.py      (needs $CUTADAPT_REFERENCE, a checkout of the reference; run once, results committed)

Case kinds: "trim" (single-end), "demux" (-o {name}.fasta), "rows" (--rest-file / --wildcard-file / --info-file: "rows"
names the expected text of that option; "expected" holds the expected trimmed output, or None where the test does not
check it), "paired".  Options: "specs" = the command line's [-a/-g/-b kind, adapter string] values, plus -e / -O / -N /
--no-indels / --match-read-wildcards and the trimmer's keyword arguments.  Cases that need options this project does
not implement (454.fa: --length-tag; the --rename cases) are left out.
"""
import gzip
import json
import os

REF = os.path.join(os.environ.get("CUTADAPT_REFERENCE", ""), "tests")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fasta_kat.json.gz")
FILES = {}     # "data/<name>" / "cut/<name>" -> content (latin-1 text)


def store(rel):
    """The reference file tests/<rel> (gzip-compressed ones decompressed) under the key <rel>."""
    path = os.path.join(REF, rel)
    with (gzip.open(path, "rb") if rel.endswith(".gz") else open(path, "rb")) as f:
        FILES[rel] = f.read().decode("latin-1")
    return rel


CL = "tests/test_commandline.py"
# single-end: name, reference test, command line, input, expected output, options
TRIM = [
    ("action_lowercase", f"{CL}:309", "-b CAAG -n 3 --action=lowercase", "action_lowercase.fasta", "action_lowercase.fasta",
     dict(specs=[["anywhere", "CAAG"]], times=3, action="lowercase")),
    ("action_retain", f"{CL}:317", "-g GGTTAACC -a CAAG --action=retain", "action_retain.fasta", "action_retain.fasta",
     dict(specs=[["front", "GGTTAACC"], ["back", "CAAG"]], action="retain")),
    ("action_crop", f"{CL}:330", "-g GGTTAA -a CAAG --action=crop --discard-untrimmed", "action_retain.fasta",
     "action_crop.fasta", dict(specs=[["front", "GGTTAA"], ["back", "CAAG"]], action="crop", discard_untrimmed=True)),
    ("example", f"{CL}:75", "-N -b ADAPTER", "example.fa", "example.fa", dict(specs=[["anywhere", "ADAPTER"]], no_wildcards=True)),
    ("minlen", f"{CL}:139", "-m 5 -a TTAGACATATCTCCGTCG", "lengths.fa", "minlen.fa",
     dict(specs=[["back", "TTAGACATATCTCCGTCG"]], minimum_length=5)),
    ("maxlen", f"{CL}:186", "-M 5 -a TTAGACATATCTCCGTCG", "lengths.fa", "maxlen.fa",
     dict(specs=[["back", "TTAGACATATCTCCGTCG"]], maximum_length=5)),
    ("overlapb", f"{CL}:239", "-O 10 -b TTAGACATATCTCCGTCG", "overlapb.fa", "overlapb.fa",
     dict(specs=[["anywhere", "TTAGACATATCTCCGTCG"]], min_overlap=10)),
    ("trim_n", f"{CL}:243", "--trim-n", "trim-n.fasta", "trim-n.fasta", dict(specs=[], trim_n=True)),
    ("twoadapters", f"{CL}:263", "-a AATTTCAGGAATT -a GTTCTCTAGTTCT", "twoadapters.fasta", "twoadapters.fasta",
     dict(specs=[["back", "AATTTCAGGAATT"], ["back", "GTTCTCTAGTTCT"]])),
    ("polya_legacy", f"{CL}:277", "-O 10 -a A{35}", "polya.1.fasta", "polya.legacy.1.fasta",
     dict(specs=[["back", "A{35}"]], min_overlap=10)),
    ("polya", f"{CL}:281", "--poly-a", "polya.1.fasta", "polya.1.fasta", dict(specs=[], poly_a=True)),
    ("read_wildcard", f"{CL}:339", "--match-read-wildcards -b ACGTACGT", "wildcard.fa", "wildcard.fa",
     dict(specs=[["anywhere", "ACGTACGT"]], read_wildcards=True)),
    ("wildcard_n", f"{CL}:372", "-e 0 -a GGGGGGG --match-read-wildcards", "wildcardN.fa", "wildcardN.fa",
     dict(specs=[["back", "GGGGGGG"]], error_rate=0, read_wildcards=True)),
    ("examplefront", f"{CL}:381", "--front ADAPTER -N", "example.fa", "examplefront.fa",
     dict(specs=[["front", "ADAPTER"]], no_wildcards=True)),
    ("literal_n3", f"{CL}:386", "-N -e 0.2 -a NNNNNNNNNNNNNN", "trimN3.fasta", "trimN3.fasta",
     dict(specs=[["back", "NNNNNNNNNNNNNN"]], no_wildcards=True, error_rate=0.2)),
    ("literal_n5", f"{CL}:390", "-N -O 1 -g NNNNNNNNNNNNNN", "trimN5.fasta", "trimN5.fasta",
     dict(specs=[["front", "N{14}"]], no_wildcards=True, min_overlap=1)),
    ("anchored_front", f"{CL}:403", "-g ^FRONTADAPT -N", "anchored.fasta", "anchored.fasta",
     dict(specs=[["front", "^FRONTADAPT"]], no_wildcards=True)),
    ("anchored_front_ellipsis", f"{CL}:407", "-a ^FRONTADAPT... -N", "anchored.fasta", "anchored.fasta",
     dict(specs=[["back", "^FRONTADAPT..."]], no_wildcards=True)),
    ("anchored_back", f"{CL}:411", "-a BACKADAPTER$ -N", "anchored-back.fasta", "anchored-back.fasta",
     dict(specs=[["back", "BACKADAPTER$"]], no_wildcards=True)),
    ("anchored_back_ellipsis", f"{CL}:415", "-a ...BACKADAPTER$ -N", "anchored-back.fasta", "anchored-back.fasta",
     dict(specs=[["back", "...BACKADAPTER$"]], no_wildcards=True)),
    ("anchored_back_no_indels", f"{CL}:419", "-a BACKADAPTER$ -N --no-indels", "anchored-back.fasta", "anchored-back.fasta",
     dict(specs=[["back", "BACKADAPTER$"]], no_wildcards=True, no_indels=True)),
    ("no_indels", f"{CL}:423", "-a TTAGACATAT -g GAGATTGCCA --no-indels", "no_indels.fasta", "no_indels.fasta",
     dict(specs=[["back", "TTAGACATAT"], ["front", "GAGATTGCCA"]], no_indels=True)),
    ("multiprefix", f"{CL}:615", "-g ^GTACGGATTGTTCAGTA -g ^TATTAAGCTCATTC", "multi.fasta", "multiprefix.fasta",
     dict(specs=[["front", "^GTACGGATTGTTCAGTA"], ["front", "^TATTAAGCTCATTC"]])),
    ("maxn0", f"{CL}:635", "--max-n 0", "maxn.fasta", "maxn0.fasta", dict(specs=[], max_n=0)),
    ("maxn1", f"{CL}:636", "--max-n 1", "maxn.fasta", "maxn1.fasta", dict(specs=[], max_n=1)),
    ("maxn2", f"{CL}:637", "--max-n 2", "maxn.fasta", "maxn2.fasta", dict(specs=[], max_n=2)),
    ("maxn0_2", f"{CL}:638", "--max-n 0.2", "maxn.fasta", "maxn0.2.fasta", dict(specs=[], max_n=0.2)),
    ("maxn0_4", f"{CL}:639", "--max-n 0.4", "maxn.fasta", "maxn0.4.fasta", dict(specs=[], max_n=0.4)),
    ("linked", f"{CL}:671", "-a ^AAAAAAAAAA...TTTTTTTTTT", "linked.fasta", "linked.fasta",
     dict(specs=[["back", "^AAAAAAAAAA...TTTTTTTTTT"]])),
    ("linked_anchored", f"{CL}:683", "-a ^AAAAAAAAAA...TTTTT$", "linked.fasta", "linked-anchored.fasta",
     dict(specs=[["back", "^AAAAAAAAAA...TTTTT$"]])),
    ("linked_not_anchored", f"{CL}:687", "-g AAAAAAAAAA...TTTTTTTTTT", "linked.fasta", "linked-not-anchored.fasta",
     dict(specs=[["front", "AAAAAAAAAA...TTTTTTTTTT"]])),
    ("xadapter", f"{CL}:746", "-g XTCCGAATAGA", "xadapterx.fasta", "xadapter.fasta", dict(specs=[["front", "XTCCGAATAGA"]])),
    ("adapterx", f"{CL}:750", "-a TCCGAATAGAX", "xadapterx.fasta", "adapterx.fasta", dict(specs=[["back", "TCCGAATAGAX"]])),
    ("adapterorder_ga", f"{CL}:799", "-g ^AAACC -a CCGGG", "adapterorder.fasta", "adapterorder-ga.fasta",
     dict(specs=[["front", "^AAACC"], ["back", "CCGGG"]])),
    ("adapterorder_ag", f"{CL}:800", "-a CCGGG -g ^AAACC", "adapterorder.fasta", "adapterorder-ag.fasta",
     dict(specs=[["back", "CCGGG"], ["front", "^AAACC"]])),
    # FASTA syntax: '#' comments and a sequence over two lines; comments alone; nothing
    ("simple", "tests/test_compression.py:17", "(no options)", "simple.fasta.gz", "simple.fasta", dict(specs=[])),
    ("onlycomment", f"{CL}:98", "(no options)", "onlycomment.fasta", "empty.fasta", dict(specs=[])),
    ("empty", f"{CL}:94", "(no options)", "empty.fasta", "empty.fasta", dict(specs=[])),
    # FASTQ in, FASTA out
    ("small_to_fasta", "tests/test_command.py:142", "--fasta -a TTAGACATATCTCCGTCG", "small.fastq", "small.fasta",
     dict(specs=[["back", "TTAGACATATCTCCGTCG"]], input_format="fastq", output_format="fasta")),
]

# --rest-file / --wildcard-file / --info-file: name, test, command line, input, expected output (or None), expected
# rows (a reference file, or the text the test asserts), row kind (0 info, 1 rest, 2 wildcard), options
WILDCARD_ROWS = "AAA 1\nGGG 2\nCCC 3b\nTTT 4b\n"     # test_commandline.py:362-364 (the lines the test compares)
ROWS = [
    ("rest", f"{CL}:112", "-b ADAPTER -N -r rest.txt", "rest.fa", "rest.fa", "data/rest.txt", 1,
     dict(specs=[["anywhere", "ADAPTER"]], no_wildcards=True)),
    ("restfront", f"{CL}:121", "-g ADAPTER -N -r rest.txt", "rest.fa", "restfront.fa", "data/restfront.txt", 1,
     dict(specs=[["front", "ADAPTER"]], no_wildcards=True)),
    ("wildcard_adapter", f"{CL}:349", "--wildcard-file wildcards.txt -a ACGTNNNACGT", "wildcard_adapter.fa",
     "wildcard_adapter.fa", WILDCARD_ROWS, 2, dict(specs=[["back", "ACGTNNNACGT"]])),
    ("wildcard_adapter_anywhere", f"{CL}:349", "--wildcard-file wildcards.txt -b ACGTNNNACGT", "wildcard_adapter.fa",
     "wildcard_adapter_anywhere.fa", WILDCARD_ROWS, 2, dict(specs=[["anywhere", "ACGTNNNACGT"]])),
    ("info_rc", "tests/test_info_file.py:78", "--info-file info-rc.txt -a adapt=GAGTCG --revcomp --rename={header}",
     "info-rc.fasta", None, "cut/info-rc.txt", 0,
     dict(specs=[["back", "adapt=GAGTCG"]], revcomp=True, rc_suffix=False)),
]

PL = "tests/test_paired.py"
PAIRED = [
    ("anchored_back_no_indels", f"{PL}:282", "-a BACKADAPTER$ -A BACKADAPTER$ -N --no-indels",
     ["anchored-back.fasta", "anchored-back.fasta"], ["anchored-back.fasta", "anchored-back.fasta"],
     dict(specs1=[["back", "BACKADAPTER$"]], specs2=[["back", "BACKADAPTER$"]], no_wildcards=True, no_indels=True)),
    ("poly_a_poly_t", f"{PL}:775", "--poly-a", ["polya.1.fasta", "polya.2.fasta"], ["polya.1.fasta", "polya.2.fasta"],
     dict(specs1=[], specs2=[], options1=dict(poly_a=True), options2=dict(poly_a=True))),
]


def main():
    cases = []
    for name, test, cmd, inp, exp, opts in TRIM:
        cases.append(dict(name=name, kind="trim", reference_test=test, command=cmd, inputs=[store("data/" + inp)],
                          expected=[store("cut/" + exp)], options=opts))
    # demultiplexing (test_commandline.py:581-601): -a first=AATTTCAGGAATT -a second=GTTCTCTAGTTCT -o {name}.fasta
    cases.append(dict(name="demux_twoadapters", kind="demux", reference_test=f"{CL}:581",
                      command="-a first=AATTTCAGGAATT -a second=GTTCTCTAGTTCT -o {name}.fasta",
                      inputs=[store("data/twoadapters.fasta")],
                      expected={n: store(f"cut/twoadapters.{n}.fasta") for n in ("first", "second", "unknown")},
                      options=dict(specs=[["back", "first=AATTTCAGGAATT"], ["back", "second=GTTCTCTAGTTCT"]])))
    for name, test, cmd, inp, exp, rows, kind, opts in ROWS:
        if rows.startswith(("data/", "cut/")):
            rows_key = store(rows)
        else:
            rows_key = f"text/{name}.rows"
            FILES[rows_key] = rows
        cases.append(dict(name=name, kind="rows", row_kind=kind, reference_test=test, command=cmd,
                          inputs=[store("data/" + inp)], expected=[store("cut/" + exp) if exp else None],
                          rows=rows_key, options=opts))
    for name, test, cmd, inps, exps, opts in PAIRED:
        cases.append(dict(name=name, kind="paired", reference_test=test, command=cmd,
                          inputs=[store("data/" + i) for i in inps], expected=[store("cut/" + e) for e in exps],
                          options=opts))
    for c in cases:
        print(f"{c['kind']:7s} {c['name']:28s} {c['reference_test']:34s} {c['command']}")
    with gzip.open(OUT, "wt", compresslevel=9) as f:
        json.dump(dict(cases=cases, files=FILES), f, sort_keys=True)
    print(len(cases), "cases,", len(FILES), "fixture files ->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
