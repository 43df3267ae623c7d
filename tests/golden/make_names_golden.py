#!/usr/bin/env python3
"""
Known answers of the reference for the read-name modifiers (--length-tag, --strip-suffix, -x / -y, --rename):
tests/golden/names_kat.json.gz.

Needs $CUTADAPT_REFERENCE, a checkout of the reference (builds oracle/_ref on the fly):

    python tests/golden/make_names_golden.py

Three groups, as data:
  cli        the reference's command-line cases (tests/test_commandline.py test_length_tag, test_strip_suffix,
             test_suffix, test_rename, test_rename_comment_without_id, test_reverse_complement_no_rc_suffix;
             tests/test_paired.py test_rename): the argument list, the input files and the expected output files of its
             test-suite (tests/data, tests/cut); test_reverse_complement_no_rc_suffix stores what that test asserts.
  modifiers  the Renamer / PairedEndRenamer cases of tests/test_modifiers.py: template, names, what the
             ModificationInfo holds, and the expected names (or that the pair is refused).
  edges      generated names answered by the reference's own LengthTagModifier, SuffixRemover, PrefixSuffixAdder and
             Renamer.parse_name (modifiers.py of $CUTADAPT_REFERENCE, loaded next to oracle/_ref's compiled modules;
             dnaio's SequenceRecord is replaced by a plain record, which is all these four use).
Re-running reproduces the file byte for byte.
"""
import importlib.util
import os
import random
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import build_ref  # noqa: E402
from make_golden import dump  # noqa: E402

REF = os.environ.get("CUTADAPT_REFERENCE", "")


def _text(*parts):
    with open(os.path.join(REF, "tests", *parts), "rb") as f:
        return f.read().decode("ascii")


CLI = [
    ("test_length_tag", ["-n", "3", "-e", "0.1", "--length-tag", "length=",
                         "-b", "TGAGACACGCAACAGGGGAAAGGCAAGGCACACAGGGGATAGG",
                         "-b", "TCCATCTCATCCCTGCGTGTCCCATCTGTTCCCTCCCTGTCTCA"], ["454.fa"], ["454.fa"]),
    ("test_strip_suffix", ["--strip-suffix", "_sequence", "-a", "XXXXXXX"], ["simple.fasta"], ["stripped.fasta"]),
    ("test_suffix", ["-y", " {name}", "-e", "0", "-a", "OnlyT=TTTTTTTT", "-a", "OnlyG=GGGGGGGG"], ["suffix.fastq"],
     ["suffix.fastq"]),
    ("test_rename", ["--rename={id}_{cut_suffix} {header} {adapter_name}", "--cut=-4", "-a", "OnlyT=TTTTTT", "-a",
                     "OnlyG=GGGGGG"], ["suffix.fastq"], ["rename.fastq"]),
    ("test_rename_comment_without_id", ["--rename={adapter_name};{comment}", "-a", "adapter=TTTTTT"], ["suffix.fastq"],
     ["rename_comment_without_id.fastq"]),
    ("test_paired_rename", ["--rename={id} {r1.cut_prefix} {cut_prefix} {comment} {adapter_name} {r2.adapter_name}",
                            "--cut=4", "-a", "R1adapter=GTCTCCAGCT", "-A", "R2adapter=GACAAATAAC"],
     ["paired.1.fastq", "paired.2.fastq"], ["rename.1.fastq", "rename.2.fastq"]),
]
# test_reverse_complement_no_rc_suffix (tests/test_commandline.py:803-822): six reads, read 1 is read2/1 with this sequence
REVCOMP = ("test_reverse_complement_no_rc_suffix", ["--revcomp", "--rename", "{header}", "-g", "^TTATTTGTCT", "-g",
                                                    "^TCCGCACTGG"], ["revcomp.1.fastq"])

# tests/test_modifiers.py TestRenamer / TestPairedEndRenamer: (template, paired, [(name, info)], expected names or None)
MODIFIERS = [
    ("{header} extra", False, [("theid thecomment", {})], ["theid thecomment extra"]),
    ("{id} extra", False, [("theid thecomment", {})], ["theid extra"]),
    ("{id} extra\\tand a tab", False, [("theid thecomment", {})], ["theid extra\tand a tab"]),
    ("{id}_extra {comment}", False, [("theid thecomment", {})], ["theid_extra thecomment"]),
    ("{id}_extra {comment}", False, [("theid", {})], ["theid_extra "]),
    ("{id}_{cut_prefix} {comment}", False, [("theid thecomment", {"cut_prefix": "TTAAGG"})], ["theid_TTAAGG thecomment"]),
    ("{id}_{cut_suffix} {comment}", False, [("theid thecomment", {"cut_suffix": "TTAAGG"})], ["theid_TTAAGG thecomment"]),
    ("{id} rc={rc} {comment}", False, [("theid thecomment", {})], ["theid rc= thecomment"]),
    ("{id} rc={rc} {comment}", False, [("theid thecomment", {"is_rc": True})], ["theid rc=rc thecomment"]),
    ("{header} match={match_sequence}", False, [("theid thecomment", {"adapter": "AGGT", "match_sequence": "ACGT"})],
     ["theid thecomment match=ACGT"]),
    ("{header} match={match_sequence}", False,
     [("theid thecomment", {"adapter": "name", "match_sequence": "TATT,ACGT", "linked": True})],
     ["theid thecomment match=TATT,ACGT"]),
    ("{id} {comment}\\tand a tab", True, [("theid comment1", {}), ("theid comment2", {})],
     ["theid comment1\tand a tab", "theid comment2\tand a tab"]),
    ("{id} abc {comment} xyz", True, [("theid_a cmtx", {}), ("theid_b cmty", {})], None),
    ("{id} abc {comment} xyz", True, [("theid cmtx", {}), ("theid cmty", {})], ["theid abc cmtx xyz", "theid abc cmty xyz"]),
    ("{id} abc {r1.comment} xyz", True, [("theid cmtx", {}), ("theid cmty", {})],
     ["theid abc cmtx xyz", "theid abc cmtx xyz"]),
    ("{id} abc {r2.comment} xyz", True, [("theid cmtx", {}), ("theid cmty", {})],
     ["theid abc cmty xyz", "theid abc cmty xyz"]),
    ("{id} read no. is: {rn}", True, [("theid cmtx", {}), ("theid cmty", {})],
     ["theid read no. is: 1", "theid read no. is: 2"]),
    ("{header} s={match_sequence}", True, [("theid first", {"adapter": "1", "match_sequence": "AC"}),
                                           ("theid second", {"adapter": "2", "match_sequence": "GT"})],
     ["theid first s=AC", "theid second s=GT"]),
    ("{header} s={r1.match_sequence}", True, [("theid first", {"adapter": "1", "match_sequence": "AC"}),
                                              ("theid second", {"adapter": "2", "match_sequence": "GT"})],
     ["theid first s=AC", "theid second s=AC"]),
    ("{header} s={r2.match_sequence}", True, [("theid first", {"adapter": "1", "match_sequence": "AC"}),
                                              ("theid second", {"adapter": "2", "match_sequence": "GT"})],
     ["theid first s=GT", "theid second s=GT"]),
]


class _Record:
    """What the four modifiers use of dnaio.SequenceRecord: name, sequence, a copy by read[:]"""

    def __init__(self, name, sequence, qualities=None):
        self.name, self.sequence, self.qualities = name, sequence, qualities

    def __getitem__(self, key):
        return _Record(self.name, self.sequence[key], self.qualities[key] if self.qualities else None)


def reference_modifiers():
    build_ref.import_ref()
    stub = types.ModuleType("dnaio")
    stub.SequenceRecord = _Record

    def unused(*_):
        raise AssertionError("record_names_match is not part of these answers")

    stub.record_names_match = unused
    sys.modules.setdefault("dnaio", stub)
    for mod in ("tokenizer", "modifiers"):
        spec = importlib.util.spec_from_file_location(f"cutadapt.{mod}", os.path.join(REF, "src", "cutadapt", f"{mod}.py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules[f"cutadapt.{mod}"] = m
        spec.loader.exec_module(m)
    return sys.modules["cutadapt.modifiers"]


class _Adapter:
    def __init__(self, name):
        self.name = name


class _Match:
    def __init__(self, name):
        self.adapter = _Adapter(name)


class _Info:
    def __init__(self, adapter):
        self.matches = [_Match(adapter)] if adapter is not None else []


WS = [" ", "\t", "\x0b", "\x0c", "\x1c", "\x1d", "\x1e", "\x1f", "\r", "\n"]
PIECES = ["read", "length=", "length=12", "12ab", "length=7x", "x", "/1", "_", "=", ";", ":", "len", "length",
          "length=3.5", "length=99_", "9", "a=b", "-", "@"]


def edges(M):
    rng = random.Random(20261018)
    names = ["", " ", "a ", " a", "a b", "  a  b  ", "a\tb", "length=", "length=12ab", "xlength=5", "_length=5",
             "=length=5", "length=5length=6", "length=1 length=22 length=333", "r length=", "read/1"]
    names += ["a" + w + "b" for w in WS] + [w + "a" + w for w in WS]
    for _ in range(150):
        names.append("".join(rng.choice(PIECES + WS) for _ in range(rng.randint(0, 6))))
    tags = ["length=", "length", "=", "x", "_1", "12", "a=b", ";", "@len", "len-", "~"]
    out = {"length_tag": [], "strip_suffix": [], "affix": [], "parse_name": []}
    for name in names:
        for tag in tags:
            length = rng.choice([0, 7, 150, 1000])
            got = M.LengthTagModifier(tag)(_Record(name, "A" * length), None).name
            out["length_tag"].append([name, tag, length, got])
        for suffix in ["", "/1", "b", " ", name, "x" + name, name[1:]]:
            out["strip_suffix"].append([name, suffix, M.SuffixRemover(suffix)(_Record(name, ""), None).name])
        id_, comment = M.Renamer.parse_name(name)
        out["parse_name"].append([name, id_, comment])
    for prefix, suffix in [("{name}_", ""), ("", " {name}"), ("p{name}{name}", "{nam}s"), ("{{name}}", "{name")]:
        for adapter in (None, "ad1"):
            for name in names[:20]:
                got = M.PrefixSuffixAdder(prefix, suffix)(_Record(name, ""), _Info(adapter)).name
                out["affix"].append([name, prefix, suffix, adapter, got])
    return out


def main():
    if not os.path.isdir(os.path.join(REF, "src", "cutadapt")):
        sys.exit("set $CUTADAPT_REFERENCE to a checkout of the reference")
    M = reference_modifiers()
    cli = []
    for name, argv, inputs, expected in CLI:
        cli.append({"name": name, "argv": argv, "inputs": {k: _text("data", k) for k in inputs},
                    "expected": [_text("cut", k) for k in expected], "input_order": inputs})
    name, argv, inputs = REVCOMP
    cli.append({"name": name, "argv": argv, "inputs": {k: _text("data", k) for k in inputs}, "input_order": inputs,
                "expected": None, "n_reads": 6, "read1": ["read2/1", "ACCATCCGATATGTCTAATGTGGCCTGTTG"]})
    mods = [{"template": t, "paired": p, "reads": r, "expected": e} for t, p, r, e in MODIFIERS]
    dump("names_kat.json.gz", {"cli": cli, "modifiers": mods, "edges": edges(M)})


if __name__ == "__main__":
    main()
