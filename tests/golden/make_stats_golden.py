#!/usr/bin/env python3
"""
Generate tests/golden/stats_kat.json.gz: the statistics the REFERENCE's own modifiers collect for its report
(AdapterCutter / ReverseComplementer .adapter_statistics, modifiers.py:109, 200-207, 301-306;
PairedAdapterCutter.adapter_statistics, modifiers.py:437-461; PolyATrimmer.trimmed_bases, modifiers.py:861-879;
QualityTrimmer / NextseqQualityTrimmer .trimmed_bases) on:
  - the single-end and paired known-answer cases of fastq_kat.json.gz (inputs referenced by case name),
  - seeded synthetic chunks (stored in the file): several adapters, times > 1, actions, --revcomp, linked, anywhere,
    rightmost and indexed (96 barcodes) adapters, -u, --nextseq-trim, --poly-a, --pair-adapters.

    python tests/golden/make_stats_golden.py --reference DIR      (or $CUTADAPT_REFERENCE; needs Cython)

The reference's hot path comes from oracle/build_ref.py (oracle/_ref, built if missing and left as it is); its
`tokenizer` and `modifiers` are compiled the same way into a temporary directory that joins the package's path.
`modifiers` imports dnaio, which is replaced by the small stand-in below (SequenceRecord, record_names_match).
The file records the SHA-256 of every reference source involved.  Before writing, every single-end answer is
checked against the independent recount of tests/stats_cases.py (the oracle's records + the repository's
AdapterStatistics; not for the indexed cases, which the C oracle does not implement), so a drift between the
reference and the recount fails here.
"""
import argparse
import gzip
import hashlib
import json
import os
import subprocess
import sys
import sysconfig
import tempfile
import types

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)

from stats_cases import adapter_list, answer, recount, reverse_complement, synthetic_fastq  # noqa: E402
from util import canonical, fastq_cases, fastq_paired_cases  # noqa: E402

SOURCES = ["adapters.py", "modifiers.py", "tokenizer.py", "qualtrim.pyx", "_align.pyx", "_kmer_finder.pyx", "info.pyx",
           "align.py", "_match_tables.py", "kmer_heuristic.py"]


class SequenceRecord:
    """Test-side stand-in for dnaio.SequenceRecord: what the modifiers use of it."""

    def __init__(self, name, sequence, qualities=None):
        self.name, self.sequence, self.qualities = name, sequence, qualities

    def __len__(self):
        return len(self.sequence)

    def __getitem__(self, key):
        return SequenceRecord(self.name, self.sequence[key], self.qualities[key] if self.qualities is not None else None)

    def reverse_complement(self):
        return SequenceRecord(self.name, reverse_complement(self.sequence),
                              self.qualities[::-1] if self.qualities is not None else None)


def record_names_match(a, b):
    return a.split()[0] == b.split()[0]


def load_reference(reference):
    os.environ["CUTADAPT_REFERENCE"] = reference
    sys.modules["dnaio"] = types.SimpleNamespace(SequenceRecord=SequenceRecord, record_names_match=record_names_match)
    from oracle import build_ref

    cutadapt = build_ref.import_ref()
    from Cython.Compiler.Main import compile as cy_compile
    from Cython.Compiler.Options import CompilationOptions, default_options

    src = os.path.join(reference, "src", "cutadapt")
    tmp = tempfile.mkdtemp(prefix="cutadapt_ref_modifiers_")
    for mod in ("tokenizer", "modifiers"):
        c_file = os.path.join(tmp, mod + ".c")
        opts = CompilationOptions(default_options, output_file=c_file, language_level=3, include_path=[src])
        if cy_compile(os.path.join(src, mod + ".py"), opts, full_module_name="cutadapt." + mod).num_errors:
            raise RuntimeError(f"cython failed on {mod}")
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-fwrapv", "-Wno-unused-function",
                               "-I", sysconfig.get_paths()["include"], "-I", src, c_file, "-o",
                               os.path.join(tmp, mod + sysconfig.get_config_var("EXT_SUFFIX"))])
    cutadapt.__path__.append(tmp)
    import cutadapt.adapters as RA
    import cutadapt.modifiers as M
    from cutadapt.info import ModificationInfo

    provenance = {name: hashlib.sha256(open(os.path.join(src, name), "rb").read()).hexdigest() for name in SOURCES}
    return RA, M, ModificationInfo, provenance


def parse(data: bytes):
    lines = data.decode("latin-1").replace("\r\n", "\n").split("\n")
    return [(lines[i][1:], lines[i + 1], lines[i + 3]) for i in range(0, len(lines) - 3, 4)]


def front_modifiers(M, o):
    """UnconditionalCutter, NextseqQualityTrimmer, QualityTrimmer in the order cli.py:937-955 builds them."""
    mods = [M.UnconditionalCutter(c) for c in o.get("cut", ())]
    base = o.get("quality_base", 33)
    if o.get("nextseq_cutoff") is not None:
        mods.append(M.NextseqQualityTrimmer(o["nextseq_cutoff"], base))
    if o.get("quality_cutoff"):
        mods.append(M.QualityTrimmer(o["quality_cutoff"][0], o["quality_cutoff"][1], base))
    return mods


def qbp(mods, M):
    return sum(m.trimmed_bases for m in mods if isinstance(m, (M.QualityTrimmer, M.NextseqQualityTrimmer)))


def run_single(RA, M, Info, o, data, second_mate=False):
    """One mate through the reference's chain; the statistics its report would show."""
    mods = front_modifiers(M, o)
    adapters = adapter_list(RA, o.get("adapters", []), o)
    cutter = None
    if adapters:
        action = o.get("action", "trim")
        cutter = M.AdapterCutter(adapters, o.get("times", 1), None if action == "none" else action)
        mods.append(M.ReverseComplementer(cutter) if o.get("revcomp") else cutter)
    poly = M.PolyATrimmer(revcomp=second_mate) if o.get("poly_a") else None
    if poly is not None:
        mods.append(poly)
    for name, seq, qual in parse(data):
        rec = SequenceRecord(name, seq, qual)
        info = Info(rec)
        for m in mods:
            rec = m(rec, info)
    return {"adapters": answer(list(cutter.adapter_statistics.values())) if cutter else [],
            "poly_a": {str(k): v for k, v in sorted(poly.trimmed_bases.items())} if poly else {},
            "quality_trimmed_bp": qbp(mods, M)}


def run_pair_adapters(RA, M, Info, o1, o2, a1, a2, data1, data2, action="trim"):
    mods1, mods2 = front_modifiers(M, o1), front_modifiers(M, o2)
    cutter = M.PairedAdapterCutter(adapter_list(RA, a1, o1), adapter_list(RA, a2, o2), action)
    poly1 = M.PolyATrimmer() if o1.get("poly_a") else None
    poly2 = M.PolyATrimmer(revcomp=True) if o2.get("poly_a") else None
    for (n1, s1, q1), (n2, s2, q2) in zip(parse(data1), parse(data2)):
        r1, r2 = SequenceRecord(n1, s1, q1), SequenceRecord(n2, s2, q2)
        i1, i2 = Info(r1), Info(r2)
        for m in mods1:
            r1 = m(r1, i1)
        for m in mods2:
            r2 = m(r2, i2)
        r1, r2 = cutter(r1, r2, i1, i2)
        if poly1:
            r1 = poly1(r1, i1)
        if poly2:
            r2 = poly2(r2, i2)
    out = []
    for k, (mods, poly) in enumerate(((mods1, poly1), (mods2, poly2))):
        out.append({"adapters": answer(list(cutter.adapter_statistics[k].values())),
                    "poly_a": {str(k2): v for k2, v in sorted(poly.trimmed_bases.items())} if poly else {},
                    "quality_trimmed_bp": qbp(mods, M)})
    return out


def synthetic_cases():
    from cutadapt_b200.configs import config5_barcodes

    bcs = config5_barcodes()
    A, F, L2 = "AGATCGGAAGAGC", "TTGACTGACG", "CACGTCTGAACTC"
    single = [
        ("syn_times2_poly_a", dict(adapters=[["back", A], ["front", F]], quality_cutoff=[5, 20], times=2, poly_a=True),
         dict(seed=1)),
        ("syn_revcomp_linked_mask", dict(adapters=[["linked", F, A], ["back", L2]], revcomp=True, action="mask",
                                         times=2, poly_a=True), dict(seed=2, adapters=(A, F, L2), flip=True)),
        ("syn_revcomp_quality", dict(adapters=[["back", A], ["front", F]], revcomp=True, quality_cutoff=[0, 20],
                                     cut=[2, -3]), dict(seed=3, flip=True)),
        ("syn_lowercase_anywhere", dict(adapters=[["anywhere", A], ["back", L2]], action="lowercase", times=3,
                                        cut=[3, -2], nextseq_cutoff=20), dict(seed=4, adapters=(A, L2))),
        ("syn_retain_linked", dict(adapters=[["linked", F, A], ["back", L2]], action="retain", quality_cutoff=[0, 15]),
         dict(seed=5, adapters=(A, F, L2))),
        ("syn_crop", dict(adapters=[["back", A], ["front", F]], action="crop"), dict(seed=6)),
        ("syn_none", dict(adapters=[["back", A]], action="none", poly_a=True), dict(seed=7)),
        ("syn_rightmost", dict(adapters=[["rightmost_front", F], ["rightmost_back", A]]), dict(seed=8)),
        ("syn_index96", dict(adapters=[["prefix", b] for b in bcs], index=True, quality_cutoff=[0, 20]),
         dict(seed=9, barcodes=bcs)),
        ("syn_index96_back", dict(adapters=[["prefix", b] for b in bcs[:24]] + [["back", A]], index=True, times=2),
         dict(seed=10, barcodes=bcs[:24])),
    ]
    paired = [
        ("syn_paired_poly", dict(adapters1=[["back", A]], adapters2=[["back", F], ["front", L2]],
                                 options1=dict(quality_cutoff=[0, 20], times=2, poly_a=True),
                                 options2=dict(poly_a=True, cut=[2])), dict(seed=11)),
        ("syn_pair_adapters", dict(adapters1=[["back", A], ["back", L2]], adapters2=[["back", F], ["back", A]],
                                   pair_adapters=True, options1=dict(quality_cutoff=[0, 20], poly_a=True),
                                   options2=dict(poly_a=True)), dict(seed=12, adapters=(A, F, L2))),
    ]
    return single, paired


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("CUTADAPT_REFERENCE"))
    ap.add_argument("--out", default=os.path.join(HERE, "stats_kat.json.gz"))
    ap.add_argument("--reads", type=int, default=800)
    a = ap.parse_args()
    RA, M, Info, provenance = load_reference(a.reference)
    out = {"provenance": provenance, "cases": [], "paired_cases": [], "inputs": {}}
    for c in fastq_cases():
        o = dict(c["options"])
        got = run_single(RA, M, Info, o, c["input_bytes"])
        out["cases"].append(dict(name=c["name"], source="fastq_kat", options=o, **got))
    for c in fastq_paired_cases():
        opts = c["options"]
        mates = []
        for k in (1, 2):
            o = dict(opts[f"options{k}"], adapters=opts[f"adapters{k}"])
            for key in ("error_rate", "min_overlap"):
                if key in opts:
                    o[key] = opts[key]
            mates.append(run_single(RA, M, Info, o, c["input_bytes"][k - 1], second_mate=k == 2))
        out["paired_cases"].append(dict(name=c["name"], source="fastq_kat", options=opts, mates=mates))
    single, paired = synthetic_cases()
    for name, o, gen in single:
        gen = dict(gen)
        data = synthetic_fastq(a.reads, **gen)
        out["inputs"][name] = data.decode("latin-1")
        out["cases"].append(dict(name=name, source="synthetic", options=o, **run_single(RA, M, Info, o, data)))
    for name, opts, gen in paired:
        gen = dict(gen)
        seed = gen.pop("seed")
        d1, d2 = synthetic_fastq(a.reads, seed=seed, **gen), synthetic_fastq(a.reads, seed=seed + 1000, **gen)
        out["inputs"][name + ".1"], out["inputs"][name + ".2"] = d1.decode("latin-1"), d2.decode("latin-1")
        o1 = dict(opts["options1"], adapters=opts["adapters1"])
        o2 = dict(opts["options2"], adapters=opts["adapters2"])
        if opts.get("pair_adapters"):
            mates = run_pair_adapters(RA, M, Info, o1, o2, opts["adapters1"], opts["adapters2"], d1, d2)
        else:
            mates = [run_single(RA, M, Info, o1, d1), run_single(RA, M, Info, o2, d2, second_mate=True)]
        out["paired_cases"].append(dict(name=name, source="synthetic", options=opts, mates=mates))
    # drift check: the independent recount must agree with the reference on every single-end case
    inputs = {c["name"]: c["input_bytes"] for c in fastq_cases()}
    for c in out["cases"]:
        if c["options"].get("index"):       # the C oracle has no IndexedPrefixAdapters; the reference's answer stands
            print(f"{c['name']}: {len(c['adapters'])} adapters (indexed)")
            continue
        data = inputs[c["name"]] if c["source"] == "fastq_kat" else out["inputs"][c["name"]].encode("latin-1")
        got, q = recount(c["options"], data)
        assert canonical(got) == canonical(c["adapters"]), c["name"]
        assert q == c["quality_trimmed_bp"], c["name"]
        print(f"{c['name']}: {len(c['adapters'])} adapters, poly-A keys {len(c['poly_a'])}")
    for c in out["paired_cases"]:
        print(f"{c['name']}: paired")
    blob = json.dumps(canonical(out), sort_keys=True, separators=(",", ":")).encode()
    with gzip.GzipFile(a.out, "wb", mtime=0) as f:
        f.write(blob)
    print(f"wrote {a.out}: {len(blob)} bytes before compression")


if __name__ == "__main__":
    main()
