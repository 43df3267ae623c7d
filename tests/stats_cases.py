"""
Cases of tests/golden/stats_kat.json.gz (make_stats_golden.py) and the test side of the FASTQ path's statistics:
adapters from a case's specs, seeded synthetic chunks, and an independent recount -- the oracle's match records on
the reads the adapter cutter saw, fed into the repository's AdapterStatistics (create_statistics / add_match).

Adapter specs: ["back" | "front" | "anywhere" | "prefix" | "rightmost_front" | "rightmost_back", sequence] or
["linked", front sequence, back sequence]; with "index": true in the options, the prefix adapters form one
IndexedPrefixAdapters, as the reference's AdapterCutter groups them (modifiers.py:127-143).
"""
import collections
import random

import numpy as np

_COMP = bytes.maketrans(b"ACGTUMRWSYKVHDBNacgtumrwsykvhdbn", b"TGCAAKYWSRMBDHVNtgcaakywsrmbdhvn")

KINDS = {"back": "BackAdapter", "front": "FrontAdapter", "anywhere": "AnywhereAdapter", "prefix": "PrefixAdapter",
         "rightmost_front": "RightmostFrontAdapter", "rightmost_back": "RightmostBackAdapter"}


def reverse_complement(s: str) -> str:
    return s.encode("latin-1").translate(_COMP)[::-1].decode("latin-1")


def adapter_list(module, specs, options):
    """The adapters of `specs` as objects of `module` (cutadapt_b200.adapters or the reference's adapters)."""
    e = options.get("error_rate", 0.1)
    o = options.get("min_overlap", 3)
    out = []
    for i, spec in enumerate(specs):
        if spec[0] == "linked":
            out.append(module.LinkedAdapter(module.FrontAdapter(spec[1], max_errors=e, min_overlap=o, name=f"a{i}f"),
                                            module.BackAdapter(spec[2], max_errors=e, min_overlap=o, name=f"a{i}b"),
                                            False, False, f"a{i}"))
        else:
            out.append(getattr(module, KINDS[spec[0]])(spec[1], max_errors=e, min_overlap=o, name=f"a{i}"))
    return out


def repo_adapters(specs, options):
    """cutadapt_b200 adapters of a case, or None."""
    import cutadapt_b200.adapters as PA

    ads = adapter_list(PA, specs, options)
    if not ads:
        return None
    if options.get("index"):
        prefix = [a for a in ads if type(a) is PA.PrefixAdapter]
        return PA.MultipleAdapters([a for a in ads if type(a) is not PA.PrefixAdapter] + [PA.IndexedPrefixAdapters(prefix)])
    return PA.MultipleAdapters(ads)


def trimmer_kwargs(options):
    """FastqTrimmer keyword arguments of one mate's options."""
    kw = {k: options[k] for k in ("quality_base", "nextseq_cutoff", "max_expected_errors", "discard_trimmed",
                                  "discard_untrimmed", "minimum_length", "maximum_length", "max_n", "times", "cut",
                                  "poly_a", "length", "trim_n", "discard_casava", "action", "revcomp") if k in options}
    if "quality_cutoff" in options:
        kw["quality_cutoff"] = tuple(options["quality_cutoff"])
    return kw


def synthetic_fastq(n, seed, adapters=("AGATCGGAAGAGC", "TTGACTGACG"), barcodes=(), poly_a=True, flip=False):
    """Seeded FASTQ reads: adapters at random places, barcodes in front (with errors), poly-A tails, N, lower case,
    optionally every other read reverse-complemented."""
    rng = random.Random(seed)
    out = []
    for i in range(n):
        ln = rng.choice((0, 3, 20, 60, 100, 150, 150, 151))
        seq = "".join(rng.choice("ACGT") for _ in range(ln))
        if ln > 20 and rng.random() < 0.6:
            a = rng.choice(adapters)
            if rng.random() < 0.2:
                k = rng.randrange(len(a))
                a = a[:k] + rng.choice("ACGT") + a[k + 1:]
            cut = rng.randrange(0, ln)
            seq = (seq[:cut] + a + seq[cut:])[:ln] if rng.random() < 0.7 else (a + seq)[:ln]
        if barcodes and rng.random() < 0.8:
            b = rng.choice(barcodes)
            if rng.random() < 0.3:
                k = rng.randrange(len(b))
                b = b[:k] + rng.choice("ACGTN") + b[k + 1:]
            seq = b + seq
        if poly_a and ln > 20 and rng.random() < 0.2:
            tail = rng.randrange(2, 20)
            seq = seq[:len(seq) - tail] + "".join("A" if rng.random() < 0.93 else "C" for _ in range(tail))
        if rng.random() < 0.05 and seq:
            seq = "".join(c if rng.random() > 0.1 else "N" for c in seq)
        if rng.random() < 0.03:
            seq = seq.lower()
        if flip and rng.random() < 0.5:
            seq = reverse_complement(seq)
        qual = "".join(chr(33 + min(41, max(2, int(rng.gauss(32 - 25 * (j / max(len(seq), 1)) ** 2, 6)))))
                       for j in range(len(seq)))
        out.append(f"@r{i}\n{seq}\n+\n{qual}\n")
    return "".join(out).encode("latin-1")


def written_lengths_of(output: bytes, fasta: bool = False) -> dict:
    lines = output.split(b"\n")
    step = 2 if fasta else 4
    return dict(collections.Counter(len(lines[i]) for i in range(1, len(lines) - 1, step)))


def answer(stats_list):
    """[(end statistics answer, reverse_complemented)] of a list of AdapterStatistics."""
    from util import end_statistics_answer

    return [[end_statistics_answer(st), int(st.reverse_complemented)] for st in stats_list]


def cutter_records(options, data):
    """(adapters, match records, reads, (start, stop) windows, is_rc, quality-trimmed bp): the oracle's records on the
    reads the adapter cutter saw -- after -u, the quality trimmers and, with --revcomp, in the orientation with the
    higher score sum; `reads` are upper-cased for --action=lowercase (modifiers.py:222-223)."""
    from oracle import oracle
    from util import spec_of

    multi = repo_adapters(options["adapters"], options)
    times = options.get("times", 1)
    q = options.get("quality_cutoff")
    base = options.get("quality_base", 33)
    records = oracle._apply_cuts(oracle.parse_fastq(data), options.get("cut", ()))
    quals_in = [r[2] for r in records]
    records_q, qbp = oracle._quality_trimmed(records, q is not None, q[0] if q else 0, q[1] if q else 0, base,
                                             options.get("nextseq_cutoff"))
    if multi is None:
        return None, None, None, None, None, qbp
    spec = spec_of(multi)
    is_rc = [False] * len(records)
    if options.get("revcomp"):
        seqs = [r[1] for r in records_q]
        rc_seqs = [reverse_complement(s) for s in seqs]
        fwd, _ = oracle.oracle_process(spec.adapters, spec.groups, seqs, None, False, 0, 0, base, times, None)
        rev, _ = oracle.oracle_process(spec.adapters, spec.groups, rc_seqs, None, False, 0, 0, base, times, None)
        matches = fwd.copy()
        for i in range(len(seqs)):
            if int(rev[i]["score"][rev[i]["adapter"] >= 0].sum()) > int(fwd[i]["score"][fwd[i]["adapter"] >= 0].sum()):
                matches[i], seqs[i], is_rc[i] = rev[i], rc_seqs[i], True
        windows = [(0, len(x)) for x in seqs]
    else:
        seqs = [r[1] for r in records]
        matches, qtrim = oracle.oracle_process(spec.adapters, spec.groups, seqs, quals_in, q is not None,
                                               q[0] if q else 0, q[1] if q else 0, base, times,
                                               options.get("nextseq_cutoff"))
        windows = [(int(qtrim[i, 0]), int(qtrim[i, 1])) for i in range(len(seqs))]
    if options.get("action") == "lowercase":
        seqs = [x.upper() for x in seqs]
    return multi, matches, seqs, windows, is_rc, qbp


def statistics_members(multi):
    """The adapters that get an AdapterStatistics, in the order adapter_statistics_from_vector lists them."""
    from cutadapt_b200.adapters import LinkedAdapter, SingleAdapter

    members = []
    for o in multi._device_set[2]:
        members += [o] if isinstance(o, (SingleAdapter, LinkedAdapter)) else list(o._index._adapters)
    return members


def recount(options, data):
    """What the adapter cutter adds per adapter, recounted independently of the device and of the reference: every
    round's Match (on what the previous round left) fed to add_match of its adapter's statistics.
    Returns (answer, quality-trimmed bp)."""
    multi, matches, seqs, windows, is_rc, qbp = cutter_records(options, data)
    if multi is None:
        return [], qbp
    members = statistics_members(multi)
    stats = {id(a): a.create_statistics() for a in members}
    for i, (s, e) in enumerate(windows):
        cur = seqs[i][s:e]
        for r in range(matches.shape[1]):
            m = multi.matches_from_records(matches[i, r], cur)
            if m is None:
                break
            stats[id(m.adapter)].add_match(m)
            stats[id(m.adapter)].reverse_complemented += is_rc[i]
            cur = m.trimmed(cur)
    return answer([stats[id(a)] for a in members]), qbp


def repo_order(options, answers):
    """The reference lists statistics in the order the adapters were given; with "index" the repository lists the
    other adapters first, then the indexed ones (the order in which the reference's AdapterCutter matches them)."""
    if not options.get("index"):
        return answers
    kinds = [s[0] for s in options["adapters"]]
    return [a for a, k in zip(answers, kinds) if k != "prefix"] + [a for a, k in zip(answers, kinds) if k == "prefix"]


def poly_a_recount(options, data, second_mate=False) -> dict:
    """PolyATrimmer.trimmed_bases from the oracle's modifier chain with and without it (nothing behind it)."""
    from oracle import oracle
    from util import spec_of

    multi = repo_adapters(options["adapters"], options)
    descs = groups = None
    if multi is not None:
        spec = spec_of(multi)
        descs, groups = spec.adapters, spec.groups
    kw = {k: v for k, v in trimmer_kwargs(options).items()
          if k in ("quality_base", "nextseq_cutoff", "times", "cut", "action", "revcomp")}
    q = options.get("quality_cutoff")
    if q:
        kw.update(quality_trim=True, cutoff_front=q[0], cutoff_back=q[1])
    a, _, _ = oracle._fastq_evaluate(data, descs, groups, poly_a=True, second_mate=second_mate, **kw)
    b, _, _ = oracle._fastq_evaluate(data, descs, groups, poly_a=False, second_mate=second_mate, **kw)
    return dict(collections.Counter(len(y[1]) - len(x[1]) for x, y in zip(a, b)))


def np_dict(d):
    return {int(k): int(v) for k, v in d.items()}


__all__ = ["adapter_list", "repo_adapters", "trimmer_kwargs", "synthetic_fastq", "written_lengths_of", "answer",
           "recount", "cutter_records", "statistics_members", "repo_order", "poly_a_recount", "reverse_complement", "np_dict", "np"]
