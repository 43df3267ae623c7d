#!/usr/bin/env python3
"""
Copies the FASTQ known-answer cases of the reference's own command-line tests
($CUTADAPT_REFERENCE/tests/test_commandline.py: run(params, expected, input) compares cutadapt's output
with tests/cut/<expected>) into tests/golden/fastq_kat.json.gz: the (<case>.in.fastq, <case>.out.fastq) pairs as
text plus the case lists, which restate each command line in terms of cutadapt_b200's FASTQ entry point.
These are test vectors (inputs and expected outputs), not source code.

    python tests/golden/make_fastq_golden.py      (needs $CUTADAPT_REFERENCE, a checkout of the reference; run once, results committed)
"""
import gzip
import json
import os
import shutil

REF = os.path.join(os.environ.get("CUTADAPT_REFERENCE", ""), "tests")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fastq_kat.json.gz")
FILES = {}     # fixture name -> content (latin-1 text)


def put(name, data):
    FILES[name] = (data if isinstance(data, bytes) else data.encode()).decode("latin-1")


def copy(src, name):
    with open(src, "rb") as f:
        put(name, f.read())

# name, reference test (test_commandline.py line), command line, input, expected, options for the product
CASES = [
    ("small", 79, "-a TTAGACATATCTCCGTCG", "small.fastq", "small.fastq",
     dict(adapters=[["back", "TTAGACATATCTCCGTCG"]])),
    ("empty", 91, "-a TTAGACATATCTCCGTCG", "empty.fastq", "empty.fastq",
     dict(adapters=[["back", "TTAGACATATCTCCGTCG"]])),
    ("dos", 104, "-e 0.12 -a TTAGACATATCTCCGTCG", "dos.fastq", "dos.fastq",
     dict(adapters=[["back", "TTAGACATATCTCCGTCG"]], error_rate=0.12)),
    ("lowercase", 109, "-a ttagacatatctccgtcg", "small.fastq", "lowercase.fastq",
     dict(adapters=[["back", "ttagacatatctccgtcg"]])),
    ("discard", 129, "-b TTAGACATATCTCCGTCG --discard", "small.fastq", "discard.fastq",
     dict(adapters=[["anywhere", "TTAGACATATCTCCGTCG"]], discard_trimmed=True)),
    ("discard_untrimmed", 134, "-b CAAGAT --discard-untrimmed", "small.fastq", "discard-untrimmed.fastq",
     dict(adapters=[["anywhere", "CAAGAT"]], discard_untrimmed=True)),
    ("lowqual", 248, "-q 10 -a XXXXXX", "lowqual.fastq", "lowqual.fastq",
     dict(adapters=[["back", "XXXXXX"]], quality_cutoff=[0, 10])),
    ("illumina64", 253, "-q 10 --quality-base 64 -a XXXXXX", "illumina64.fastq", "illumina64.fastq",
     dict(adapters=[["back", "XXXXXX"]], quality_cutoff=[0, 10], quality_base=64)),
    ("illumina64_no_adapter", 258, "-q 10 --quality-base 64", "illumina64.fastq", "illumina64.fastq",
     dict(adapters=[], quality_cutoff=[0, 10], quality_base=64)),
    ("iupac", 376, "-a VCCGAMCYUCKHRKDCUBBCNUWNSGHCGU", "illumina.fastq.gz", "illumina.fastq",
     dict(adapters=[["back", "VCCGAMCYUCKHRKDCUBBCNUWNSGHCGU"]])),
    ("rna", 456, "-a GCCGAACUUCUUAGACUGCCUUAAGGACGU", "illumina.fastq.gz", "illumina.fastq",
     dict(adapters=[["back", "GCCGAACUUCUUAGACUGCCUUAAGGACGU"]])),
    ("nextseq", 667, "--nextseq-trim 22", "nextseq.fastq", "nextseq.fastq",
     dict(adapters=[], nextseq_cutoff=22)),
    ("anywhere_small", 780, "-b TTAGACATATCTCCGTCG", "small.fastq", "small.fastq",
     dict(adapters=[["anywhere", "TTAGACATATCTCCGTCG"]])),
    ("paired_separate_1", 785, "-a TTAGACATAT", "paired.1.fastq", "paired-separate.1.fastq",
     dict(adapters=[["back", "TTAGACATAT"]])),
    ("paired_separate_2", 786, "-a CAGTGGAGTA", "paired.2.fastq", "paired-separate.2.fastq",
     dict(adapters=[["back", "CAGTGGAGTA"]])),
    ("front_empty", 790, "-g CWC", "empty.fastq", "empty.fastq",
     dict(adapters=[["front", "CWC"]])),
    ("unconditional_front", 502, "-u 5", "small.fastq", "unconditional-front.fastq", dict(adapters=[], cut=[5])),
    ("unconditional_back", 506, "-u -5", "small.fastq", "unconditional-back.fastq", dict(adapters=[], cut=[-5])),
    ("unconditional_both", 510, "-u -5 -u 5", "small.fastq", "unconditional-both.fastq",
     dict(adapters=[], cut=[-5, 5])),
    ("shortened", 738, "--length 5", "small.fastq", "shortened.fastq", dict(adapters=[], length=5)),
    ("shortened_negative", 742, "--length -5", "small.fastq", "shortened-negative.fastq",
     dict(adapters=[], length=-5)),
    ("casava", 770, "--discard-casava", "casava.fastq", "casava.fastq", dict(adapters=[], discard_casava=True)),
    ("action_none", 291, "--action=none --discard-untrimmed -a CCCTAGTTAAAC", "small.fastq", "no-trim.fastq",
     dict(adapters=[["back", "CCCTAGTTAAAC"]], action="none", discard_untrimmed=True)),
    ("action_mask", 305, "-b CAAG -n 3 --action=mask", "anywhere_repeat.fastq", "anywhere_repeat.fastq",
     dict(adapters=[["anywhere", "CAAG"]], times=3, action="mask")),
    # FASTA vectors of the reference, stored as FASTQ with constant qualities (single-line records: 1:1)
    ("action_lowercase", 309, "-b CAAG -n 3 --action=lowercase", "action_lowercase.fasta", "action_lowercase.fasta",
     dict(adapters=[["anywhere", "CAAG"]], times=3, action="lowercase")),
    ("action_retain", 317, "-g GGTTAACC -a CAAG --action=retain", "action_retain.fasta", "action_retain.fasta",
     dict(adapters=[["front", "GGTTAACC"], ["back", "CAAG"]], action="retain")),
    ("action_crop", 330, "-g GGTTAA -a CAAG --action=crop --discard-untrimmed", "action_retain.fasta",
     "action_crop.fasta", dict(adapters=[["front", "GGTTAA"], ["back", "CAAG"]], action="crop", discard_untrimmed=True)),
    ("maxee", 838, "--max-ee=0.9", "maxee.fastq", "maxee.fastq",
     dict(adapters=[], max_expected_errors=0.9)),
]


# More single-end known answers of test_commandline.py whose vectors are FASTA: stored as FASTQ with constant qualities
# and checked against the oracle on the CPU (tests/test_oracle.py).  "specs" are the command line's -a/-g/-b values.
FASTA_CASES = [
    ("example", 75, "-N -b ADAPTER", "example.fa", "example.fa", dict(specs=[["anywhere", "ADAPTER"]], no_wildcards=True)),
    ("minlen", 139, "-m 5 -a TTAGACATATCTCCGTCG", "lengths.fa", "minlen.fa",
     dict(specs=[["back", "TTAGACATATCTCCGTCG"]], minimum_length=5)),
    ("maxlen", 186, "-M 5 -a TTAGACATATCTCCGTCG", "lengths.fa", "maxlen.fa",
     dict(specs=[["back", "TTAGACATATCTCCGTCG"]], maximum_length=5)),
    ("overlapb", 239, "-O 10 -b TTAGACATATCTCCGTCG", "overlapb.fa", "overlapb.fa",
     dict(specs=[["anywhere", "TTAGACATATCTCCGTCG"]], min_overlap=10)),
    ("trim_n", 243, "--trim-n", "trim-n.fasta", "trim-n.fasta", dict(specs=[], trim_n=True)),
    ("twoadapters", 263, "-a AATTTCAGGAATT -a GTTCTCTAGTTCT", "twoadapters.fasta", "twoadapters.fasta",
     dict(specs=[["back", "AATTTCAGGAATT"], ["back", "GTTCTCTAGTTCT"]])),
    ("polya_legacy", 277, "-O 10 -a A{35}", "polya.1.fasta", "polya.legacy.1.fasta",
     dict(specs=[["back", "A{35}"]], min_overlap=10)),
    ("polya", 281, "--poly-a", "polya.1.fasta", "polya.1.fasta", dict(specs=[], poly_a=True)),
    ("read_wildcard", 339, "--match-read-wildcards -b ACGTACGT", "wildcard.fa", "wildcard.fa",
     dict(specs=[["anywhere", "ACGTACGT"]], read_wildcards=True)),
    ("wildcard_n", 372, "-e 0 -a GGGGGGG --match-read-wildcards", "wildcardN.fa", "wildcardN.fa",
     dict(specs=[["back", "GGGGGGG"]], error_rate=0, read_wildcards=True)),
    ("examplefront", 381, "--front ADAPTER -N", "example.fa", "examplefront.fa",
     dict(specs=[["front", "ADAPTER"]], no_wildcards=True)),
    ("literal_n3", 386, "-N -e 0.2 -a NNNNNNNNNNNNNN", "trimN3.fasta", "trimN3.fasta",
     dict(specs=[["back", "NNNNNNNNNNNNNN"]], no_wildcards=True, error_rate=0.2)),
    ("literal_n5", 390, "-N -O 1 -g NNNNNNNNNNNNNN", "trimN5.fasta", "trimN5.fasta",
     dict(specs=[["front", "N{14}"]], no_wildcards=True, min_overlap=1)),
    ("anchored_front", 403, "-g ^FRONTADAPT -N", "anchored.fasta", "anchored.fasta",
     dict(specs=[["front", "^FRONTADAPT"]], no_wildcards=True)),
    ("anchored_front_ellipsis", 407, "-a ^FRONTADAPT... -N", "anchored.fasta", "anchored.fasta",
     dict(specs=[["back", "^FRONTADAPT..."]], no_wildcards=True)),
    ("anchored_back", 411, "-a BACKADAPTER$ -N", "anchored-back.fasta", "anchored-back.fasta",
     dict(specs=[["back", "BACKADAPTER$"]], no_wildcards=True)),
    ("anchored_back_ellipsis", 415, "-a ...BACKADAPTER$ -N", "anchored-back.fasta", "anchored-back.fasta",
     dict(specs=[["back", "...BACKADAPTER$"]], no_wildcards=True)),
    ("anchored_back_no_indels", 419, "-a BACKADAPTER$ -N --no-indels", "anchored-back.fasta", "anchored-back.fasta",
     dict(specs=[["back", "BACKADAPTER$"]], no_wildcards=True, no_indels=True)),
    ("no_indels", 423, "-a TTAGACATAT -g GAGATTGCCA --no-indels", "no_indels.fasta", "no_indels.fasta",
     dict(specs=[["back", "TTAGACATAT"], ["front", "GAGATTGCCA"]], no_indels=True)),
    ("multiprefix", 615, "-g ^GTACGGATTGTTCAGTA -g ^TATTAAGCTCATTC", "multi.fasta", "multiprefix.fasta",
     dict(specs=[["front", "^GTACGGATTGTTCAGTA"], ["front", "^TATTAAGCTCATTC"]])),
    ("maxn0", 635, "--max-n 0", "maxn.fasta", "maxn0.fasta", dict(specs=[], max_n=0)),
    ("maxn1", 636, "--max-n 1", "maxn.fasta", "maxn1.fasta", dict(specs=[], max_n=1)),
    ("maxn2", 637, "--max-n 2", "maxn.fasta", "maxn2.fasta", dict(specs=[], max_n=2)),
    ("maxn0_2", 638, "--max-n 0.2", "maxn.fasta", "maxn0.2.fasta", dict(specs=[], max_n=0.2)),
    ("maxn0_4", 639, "--max-n 0.4", "maxn.fasta", "maxn0.4.fasta", dict(specs=[], max_n=0.4)),
    ("linked", 671, "-a ^AAAAAAAAAA...TTTTTTTTTT", "linked.fasta", "linked.fasta",
     dict(specs=[["back", "^AAAAAAAAAA...TTTTTTTTTT"]])),
    ("linked_anchored", 683, "-a ^AAAAAAAAAA...TTTTT$", "linked.fasta", "linked-anchored.fasta",
     dict(specs=[["back", "^AAAAAAAAAA...TTTTT$"]])),
    ("linked_not_anchored", 687, "-g AAAAAAAAAA...TTTTTTTTTT", "linked.fasta", "linked-not-anchored.fasta",
     dict(specs=[["front", "AAAAAAAAAA...TTTTTTTTTT"]])),
    ("xadapter", 746, "-g XTCCGAATAGA", "xadapterx.fasta", "xadapter.fasta", dict(specs=[["front", "XTCCGAATAGA"]])),
    ("adapterx", 750, "-a TCCGAATAGAX", "xadapterx.fasta", "adapterx.fasta", dict(specs=[["back", "TCCGAATAGAX"]])),
    ("adapterorder_ga", 799, "-g ^AAACC -a CCGGG", "adapterorder.fasta", "adapterorder-ga.fasta",
     dict(specs=[["front", "^AAACC"], ["back", "CCGGG"]])),
    ("adapterorder_ag", 800, "-a CCGGG -g ^AAACC", "adapterorder.fasta", "adapterorder-ag.fasta",
     dict(specs=[["back", "CCGGG"], ["front", "^AAACC"]])),
]

# paired-end: name, reference test (test_paired.py line), command line, in1, in2, expected1, expected2, options
Q10 = dict(quality_cutoff=[0, 10])
Q20 = dict(quality_cutoff=[0, 20])
PAIRED = [
    ("m14", 48, "-a TTAGACATAT -m 14 -q 10", "paired.1.fastq", "paired.2.fastq", "paired.m14.1.fastq", "paired.m14.2.fastq",
     dict(adapters1=[["back", "TTAGACATAT"]], adapters2=[], options1=dict(minimum_length=14, **Q10),
          options2=dict(minimum_length=14, **Q10))),
    ("m27", 260, "-a XXX -m 27", "paired.1.fastq", "paired.2.fastq", "paired-m27.1.fastq", "paired-m27.2.fastq",
     dict(adapters1=[["back", "XXX"]], adapters2=[], options1=dict(minimum_length=27), options2=dict(minimum_length=27))),
    ("both_adapters", 272, "-a TTAGACATAT -A CAGTGGAGTA -m 14", "paired.1.fastq", "paired.2.fastq", "paired.1.fastq",
     "paired.2.fastq", dict(adapters1=[["back", "TTAGACATAT"]], adapters2=[["back", "CAGTGGAGTA"]],
                            options1=dict(minimum_length=14), options2=dict(minimum_length=14))),
    ("qualtrim", 295, "-q 20 -a TTAGACATAT -A CAGTGGAGTA -m 14 -M 90", "paired.1.fastq", "paired.2.fastq",
     "pairedq.1.fastq", "pairedq.2.fastq",
     dict(adapters1=[["back", "TTAGACATAT"]], adapters2=[["back", "CAGTGGAGTA"]],
          options1=dict(minimum_length=14, maximum_length=90, **Q20),
          options2=dict(minimum_length=14, maximum_length=90, **Q20))),
    ("qualtrim_swapped", 307, "-q 20 -a CAGTGGAGTA -A TTAGACATAT -m 14", "paired.2.fastq", "paired.1.fastq",
     "pairedq.2.fastq", "pairedq.1.fastq",
     dict(adapters1=[["back", "CAGTGGAGTA"]], adapters2=[["back", "TTAGACATAT"]],
          options1=dict(minimum_length=14, **Q20), options2=dict(minimum_length=14, **Q20))),
    ("q10_Q0", 325, "-q 10 -Q 0", "lowqual.fastq", "lowqual.fastq", "lowqual.fastq", "lowqual.unchanged.fastq",
     dict(adapters1=[], adapters2=[], options1=dict(**Q10), options2=dict())),
    ("Q10_only", 323, "-Q 10", "lowqual.fastq", "lowqual.fastq", "lowqual.unchanged.fastq", "lowqual.fastq",
     dict(adapters1=[], adapters2=[], options1=dict(), options2=dict(**Q10))),
    ("cut", 340, "-u 3 -u -1 -U 4 -U -2", "paired.1.fastq", "paired.2.fastq", "pairedu.1.fastq", "pairedu.2.fastq",
     dict(adapters1=[], adapters2=[], options1=dict(cut=[3, -1]), options2=dict(cut=[4, -2]))),
    ("length5", 351, "--length 5", "paired.1.fastq", "paired.2.fastq", "length5.1.fastq", "length5.2.fastq",
     dict(adapters1=[], adapters2=[], options1=dict(length=5), options2=dict(length=5))),
    ("length_neg5", 362, "--length -5", "paired.1.fastq", "paired.2.fastq", "length-5.1.fastq", "length-5.2.fastq",
     dict(adapters1=[], adapters2=[], options1=dict(length=-5), options2=dict(length=-5))),
    ("L5_only", 384, "-L 5", "paired.1.fastq", "paired.2.fastq", "paired-unchanged.1.fastq", "length5.2.fastq",
     dict(adapters1=[], adapters2=[], options1=dict(), options2=dict(length=5))),
    ("only_A", 396, "-A CAGTGGAGTA", "paired.1.fastq", "paired.2.fastq", "paired-onlyA.1.fastq", "paired-onlyA.2.fastq",
     dict(adapters1=[], adapters2=[["back", "CAGTGGAGTA"]], options1=dict(), options2=dict())),
    ("discard_untrimmed", 408, "-a CTCCAGCTTAGACATATC -A XXXXXXXX --discard-untrimmed", "paired.1.fastq",
     "paired.2.fastq", "empty.fastq", "empty.fastq",
     dict(adapters1=[["back", "CTCCAGCTTAGACATATC"]], adapters2=[["back", "XXXXXXXX"]],
          options1=dict(discard_untrimmed=True), options2=dict(discard_untrimmed=True))),
    ("discard_trimmed", 419, "-A C -O 1 --discard-trimmed", "paired.1.fastq", "paired.2.fastq", "empty.fastq",
     "empty.fastq", dict(adapters1=[], adapters2=[["back", "C"]], min_overlap=1,
                         options1=dict(discard_trimmed=True), options2=dict(discard_trimmed=True))),
    ("filter_both", 493, "--pair-filter=both -a TTAGACATAT -A GGAGTA -m 14", "paired.1.fastq", "paired.2.fastq",
     "paired-filterboth.1.fastq", "paired-filterboth.2.fastq",
     dict(adapters1=[["back", "TTAGACATAT"]], adapters2=[["back", "GGAGTA"]], pair_filter="both",
          options1=dict(minimum_length=14), options2=dict(minimum_length=14))),
    ("filter_first", 504, "--pair-filter=first -a TTAGACATAT -A GGAGTA -m 14", "paired.1.fastq", "paired.2.fastq",
     "paired-filterfirst.1.fastq", "paired-filterfirst.2.fastq",
     dict(adapters1=[["back", "TTAGACATAT"]], adapters2=[["back", "GGAGTA"]], pair_filter="first",
          options1=dict(minimum_length=14), options2=dict(minimum_length=14))),
]


def fasta_to_fastq(path):
    """FASTA records (sequences may span lines) as FASTQ with constant qualities 'I'."""
    recs, name, seq = [], None, []
    for line in open(path).read().split("\n"):
        if line.startswith(">"):
            if name is not None:
                recs.append((name, "".join(seq)))
            name, seq = line[1:], []
        elif name is not None:
            seq.append(line.strip())
    if name is not None:
        recs.append((name, "".join(seq)))
    return "".join("@%s\n%s\n+\n%s\n" % (n, s, "I" * len(s)) for n, s in recs).encode()


def main():
    index = []
    for name, line, cmd, inp, exp, opts in CASES:
        src = os.path.join(REF, "data", inp)
        if inp.endswith(".gz"):
            with gzip.open(src, "rb") as f:
                put(f"{name}.in.fastq", f.read())
        elif inp.endswith(".fasta"):
            put(f"{name}.in.fastq", fasta_to_fastq(src))
        else:
            copy(src, f"{name}.in.fastq")
        if exp.endswith(".fasta"):
            put(f"{name}.out.fastq", fasta_to_fastq(os.path.join(REF, "cut", exp)))
        else:
            copy(os.path.join(REF, "cut", exp), f"{name}.out.fastq")
        index.append(dict(name=name, reference_test=f"tests/test_commandline.py:{line}", command=cmd,
                          input=f"tests/data/{inp}", expected=f"tests/cut/{exp}", options=opts))
    print(len(index), "cases")
    findex = []
    for name, line, cmd, inp, exp, opts in FASTA_CASES:
        put(f"fa_{name}.in.fastq", fasta_to_fastq(os.path.join(REF, "data", inp)))
        put(f"fa_{name}.out.fastq", fasta_to_fastq(os.path.join(REF, "cut", exp)))
        findex.append(dict(name=name, reference_test=f"tests/test_commandline.py:{line}", command=cmd,
                           input=f"tests/data/{inp}", expected=f"tests/cut/{exp}", options=opts))
    print(len(findex), "FASTA cases")
    pindex = []
    for name, line, cmd, in1, in2, exp1, exp2, opts in PAIRED:
        for k, (inp, exp) in enumerate(((in1, exp1), (in2, exp2)), 1):
            copy(os.path.join(REF, "data", inp), f"paired_{name}.in{k}.fastq")
            copy(os.path.join(REF, "cut", exp), f"paired_{name}.out{k}.fastq")
        pindex.append(dict(name=name, reference_test=f"tests/test_paired.py:{line}", command=cmd,
                           inputs=[f"tests/data/{in1}", f"tests/data/{in2}"],
                           expected=[f"tests/cut/{exp1}", f"tests/cut/{exp2}"], options=opts))
    print(len(pindex), "paired cases")
    # demultiplexing (test_commandline.py:581-601: -a first=AATTTCAGGAATT -a second=GTTCTCTAGTTCT -o {name}.fasta
    # twoadapters.fasta): the reference's vectors are FASTA; they are stored as FASTQ with constant qualities 'I'
    # (single-line records, so the conversion is 1:1 and the expected sequences are untouched)
    put("demux_twoadapters.in.fastq", fasta_to_fastq(os.path.join(REF, "data", "twoadapters.fasta")))
    for name in ("first", "second", "unknown"):
        put(f"demux_twoadapters.{name}.out.fastq", fasta_to_fastq(os.path.join(REF, "cut", f"twoadapters.{name}.fasta")))
    # --info-file known answers (tests/test_info_file.py:14-55): the text files
    for src, dst in (("cut/illumina.info.txt", "info_illumina.txt"), ("cut/illumina5.info.txt", "info_illumina5.txt"),
                     ("data/illumina5.fastq", "info_illumina5.in.fastq")):
        copy(os.path.join(REF, src), dst)
    # --pair-adapters known answer (test_paired.py:668-676)
    for k in (1, 2):
        copy(os.path.join(REF, "data", f"paired.{k}.fastq"), f"pair_adapters.in{k}.fastq")
        copy(os.path.join(REF, "cut", f"pair-adapters.{k}.fastq"), f"pair_adapters.out{k}.fastq")
    # --revcomp known answer (test_commandline.py:827-835)
    copy(os.path.join(REF, "data", "revcomp.1.fastq"), "revcomp.in.fastq")
    copy(os.path.join(REF, "cut", "revcomp-single-normalize.fastq"), "revcomp.out.fastq")
    # --revcomp on pairs (test_paired.py:786-833): adapters on one mate only (either one), adapters on both
    copy(os.path.join(REF, "data", "revcomp.2.fastq"), "revcomp.in2.fastq")
    for k in (1, 2):
        copy(os.path.join(REF, "cut", f"revcomp.{k}.fastq"), f"revcomp_one_mate.out{k}.fastq")
        copy(os.path.join(REF, "cut", f"revcomp-r1r2.{k}.fastq"), f"revcomp_r1r2.out{k}.fastq")
    # --rest-file / --wildcard-file known answers (test_commandline.py:110-122, 345-367)
    for src, dst in (("data/rest.fa", "rest.in.fasta"), ("data/rest.txt", "rest.txt"),
                     ("data/restfront.txt", "restfront.txt"), ("data/wildcard_adapter.fa", "wildcard_adapter.in.fasta")):
        copy(os.path.join(REF, src), dst)
    with gzip.open(OUT, "wt", compresslevel=9) as f:
        json.dump(dict(cases=index, fasta_cases=findex, paired_cases=pindex, files=FILES), f)
    print(len(FILES), "fixture files ->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
