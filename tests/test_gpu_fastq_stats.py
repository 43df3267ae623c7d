"""
GPU tests (-m gpu) of the statistics the FASTQ path collects for the report (cg_fastq_stats_*, FastqTrimmer /
PairedFastqTrimmer(collect_statistics=True)): per-adapter statistics, reverse_complemented per adapter, the poly-A and
written-length histograms and the scalars, against an independent recount -- the oracle's match records on what the
adapter cutter saw, fed into the repository's AdapterStatistics (create_statistics / add_match) -- and the oracle's
output.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cutadapt_b200.adapters as PA  # noqa: E402
from cutadapt_b200 import _lib  # noqa: E402
from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer, fastq_stats_layout  # noqa: E402
from oracle import oracle  # noqa: E402
from test_gpu_fastq import flip_records, synthetic_fastq, trimmer_for  # noqa: E402
from util import end_statistics_answer, fastq_case_adapters, fastq_case_kwargs, spec_of  # noqa: E402

_COMP = bytes.maketrans(b"ACGTUMRWSYKVHDBNacgtumrwsykvhdbn", b"TGCAAKYWSRMBDHVNtgcaakywsrmbdhvn")


def recount(options, data, **extra):
    """[(end statistics answer, reverse_complemented)] per adapter: the oracle's records on the reads the cutter saw
    (after -u, the quality trimmers and, with --revcomp, in the orientation that wins), upper-cased for
    --action=lowercase (modifiers.py:222-223), every round on what the previous one left (modifiers.py:225-231)."""
    kw = fastq_case_kwargs(options)
    kw.update(extra)
    multi = PA.MultipleAdapters(fastq_case_adapters(options))
    spec = spec_of(multi)
    times = kw.get("times", 1)
    records = oracle._apply_cuts(oracle.parse_fastq(data), kw.get("cut", ()))
    is_rc = [False] * len(records)
    if kw.get("revcomp"):
        records, _ = oracle._quality_trimmed(records, kw.get("quality_trim", False), kw.get("cutoff_front", 0),
                                             kw.get("cutoff_back", 0), kw.get("quality_base", 33),
                                             kw.get("nextseq_cutoff"))
        seqs = [r[1] for r in records]
        rc_seqs = [s.encode("latin-1").translate(_COMP)[::-1].decode("latin-1") for s in seqs]
        fwd, _ = oracle.oracle_process(spec.adapters, spec.groups, seqs, None, False, 0, 0, 33, times, None)
        rev, _ = oracle.oracle_process(spec.adapters, spec.groups, rc_seqs, None, False, 0, 0, 33, times, None)
        matches = fwd.copy()
        windows = list(seqs)
        for i in range(len(seqs)):
            if int(rev[i]["score"][rev[i]["adapter"] >= 0].sum()) > int(fwd[i]["score"][fwd[i]["adapter"] >= 0].sum()):
                matches[i], windows[i], is_rc[i] = rev[i], rc_seqs[i], True
    else:
        seqs, quals = [r[1] for r in records], [r[2] for r in records]
        matches, qtrim = oracle.oracle_process(spec.adapters, spec.groups, seqs, quals, kw.get("quality_trim", False),
                                               kw.get("cutoff_front", 0), kw.get("cutoff_back", 0),
                                               kw.get("quality_base", 33), times, kw.get("nextseq_cutoff"))
        windows = [s[int(qtrim[i, 0]):int(qtrim[i, 1])] for i, s in enumerate(seqs)]
    owners = multi._device_set[2]
    stats = {id(o): o.create_statistics() for o in owners}
    for i, cur in enumerate(windows):
        if kw.get("action") == "lowercase":
            cur = cur.upper()
        for r in range(times):
            m = multi.matches_from_records(matches[i, r], cur)
            if m is None:
                break
            stats[id(m.adapter)].add_match(m)
            stats[id(m.adapter)].reverse_complemented += is_rc[i]
            cur = m.trimmed(cur)
    return [(end_statistics_answer(stats[id(o)]), stats[id(o)].reverse_complemented) for o in owners]


def expected_lengths(options, data, **extra):
    """(written lengths, poly-A lengths) from the oracle: the output records, and the modifier chain with and without
    PolyATrimmer (the variants that use --poly-a have no modifier behind it)."""
    import collections

    kw = fastq_case_kwargs(options)
    kw.update(extra)
    ads = fastq_case_adapters(options)
    descs = groups = None
    if ads:
        spec = spec_of(PA.MultipleAdapters(ads))
        descs, groups = spec.adapters, spec.groups
    out, counters = oracle.oracle_fastq_trim(data, descs, groups, **kw)
    lines = out.split(b"\n")
    written = collections.Counter(len(lines[i]) for i in range(1, len(lines) - 1, 4))
    poly = {}
    if kw.get("poly_a"):
        with_poly, _, _ = oracle._fastq_evaluate(data, descs, groups, **kw)
        without, _, _ = oracle._fastq_evaluate(data, descs, groups, **{**kw, "poly_a": False})
        poly = collections.Counter(len(a[1]) - len(b[1]) for a, b in zip(without, with_poly))
    return dict(written), dict(poly), counters


def check_trimmer(t, options, data, **extra):
    got = [(end_statistics_answer(st), st.reverse_complemented) for st in t.adapter_statistics()]
    assert got == recount(options, data, **extra)
    written, poly, counters = expected_lengths(options, data, **extra)
    assert t.written_lengths == written
    assert t.poly_a_trimmed_lengths == poly
    vec, max_len, kmax = t.statistics_vector()
    assert vec.size == fastq_stats_layout(t._stats.n_adapters, max_len, kmax)["size"]
    for i, k in enumerate(("n_records", "bp_in", "with_adapters", "quality_trimmed_bp")):
        assert vec[i] == counters[k], k
    assert vec[5] == counters["reverse_complemented"]
    assert vec[6] == t.statistics["n_written"] and vec[7] == t.statistics["bp_out"]
    assert vec[6] == sum(written.values())


VARIANTS = {
    "plain": ({}, {}),
    "times3": ({}, dict(times=3, minimum_length=20)),
    "mask": ({}, dict(action="mask", times=2)),
    "lowercase": ({}, dict(action="lowercase", times=2, poly_a=True)),
    "none": ({}, dict(action="none", discard_untrimmed=True)),
    "retain_linked": (dict(adapters=[["linked", "TTGACNNACG", "AGATCGGAAGAGC"], ["back", "CACGTCTGAACTC"],
                                     ["front", "ACGTACGTAC"]], quality_cutoff=[0, 15]), dict(action="retain")),
    "crop_anywhere": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["anywhere", "CACGTCTGAA"]]),
                      dict(action="crop", discard_untrimmed=True)),
    "cut_poly_a": ({}, dict(cut=[3, -2], poly_a=True, discard_casava=True, max_n=2)),
    "nextseq": ({}, dict(nextseq_cutoff=20, times=2)),
    "revcomp": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]]), dict(revcomp=True)),
    "revcomp_linked": (dict(adapters=[["linked", "TTGACNNACG", "AGATCGGAAGAGC"], ["back", "CACGTCTGAACTC"]],
                            quality_cutoff=[0, 15]), dict(revcomp=True, action="mask", poly_a=True, times=2)),
    "quality_only": (dict(adapters=[], quality_cutoff=[0, 25]), dict(poly_a=True, minimum_length=1)),
}


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_random_chunks_against_recount(variant):
    options = dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]], quality_cutoff=[5, 20])
    over, extra = VARIANTS[variant]
    options.update(over)
    seed = sorted(VARIANTS).index(variant) + 100
    data = synthetic_fastq(6000, seed=seed)
    if variant.startswith("revcomp"):
        data = flip_records(data, seed)
    t = trimmer_for(options, collect_statistics=True, **extra)
    plain = trimmer_for(options, **extra)
    assert t.process_chunk(data) == plain.process_chunk(data)
    check_trimmer(t, options, data, **extra)
    if variant.startswith("revcomp"):
        assert sum(st.reverse_complemented for st in t.adapter_statistics()) > 0


def test_fastq_to_fasta_output():
    options = dict(adapters=[["back", "AGATCGGAAGAGC"]], quality_cutoff=[0, 20])
    data = synthetic_fastq(3000, seed=41)
    t = trimmer_for(options, collect_statistics=True, output_format="fasta", poly_a=True)
    out = t.process_chunk(data)
    lines = out.split(b"\n")
    import collections

    assert t.written_lengths == dict(collections.Counter(len(lines[i]) for i in range(1, len(lines) - 1, 2)))
    assert [(end_statistics_answer(st), st.reverse_complemented) for st in t.adapter_statistics()] == \
        recount(options, data)


def test_chunks_in_flight_add_up():
    options = dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]], quality_cutoff=[5, 20])
    chunks = [synthetic_fastq(2000, seed=200 + i) for i in range(5)]
    t = trimmer_for(options, collect_statistics=True, times=2, poly_a=True)
    list(t.process_chunks(chunks))
    total, max_len, kmax = t.statistics_vector()
    parts = []
    for c in chunks:
        one = trimmer_for(options, collect_statistics=True, times=2, poly_a=True)
        one.process_chunk(c)
        parts.append(one.statistics_vector())
    from cutadapt_b200.pipeline import relayout_statistics

    n = t._stats.n_adapters
    expect = sum(relayout_statistics(v, n, L, K, max_len, kmax) for v, L, K in parts)
    assert (total == expect).all()


def test_long_read_grows_max_len():
    options = dict(adapters=[["back", "AGATCGGAAGAGC"]])
    short = synthetic_fastq(3000, seed=300)
    long_seq = ("ACGT" * 2500)[:9980] + "AGATCGGAAGAGCAAAAAAAAAAAAAAAAAAA"
    long = short + f"@long\n{long_seq}\n+\n{'I' * len(long_seq)}\n".encode()
    t = trimmer_for(options, collect_statistics=True, poly_a=True)
    t.process_chunk(short)
    _, len0, _ = t.statistics_vector()
    t.process_chunk(long)
    vec, len1, _ = t.statistics_vector()
    assert len0 < 10000 <= len1
    both = short + long
    assert [(end_statistics_answer(st), st.reverse_complemented) for st in t.adapter_statistics()] == \
        recount(options, both)
    written, poly, _ = expected_lengths(options, both, poly_a=True)
    assert t.written_lengths == written
    assert t.poly_a_trimmed_lengths == poly


def test_statistics_off_changes_nothing():
    options = dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]], quality_cutoff=[5, 20])
    data = synthetic_fastq(4000, seed=400)
    ctx = _lib.default_context()
    runs = []
    for collect in (False, False, True):
        t = trimmer_for(options, collect_statistics=collect, poly_a=True, times=2)
        before = ctx.launch_count()
        out = t.process_chunk(data)
        runs.append((out, dict(t.statistics), ctx.launch_count() - before))
    assert runs[0] == runs[1]
    assert runs[2][:2] == runs[0][:2]
    # statistics on adds exactly its two launches (cg_stats_kernel, fq_stats_tail_kernel); everything else is the same
    # sequence of launches, so the off path launches what the path without the feature launched
    assert runs[2][2] - runs[0][2] == 2


def test_serial_runner_returns_the_vector(tmp_path):
    import io
    import json
    import subprocess
    import sys

    from cutadapt_b200.runners import SerialRunner

    options = dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]], quality_cutoff=[5, 20])
    data = b"".join(synthetic_fastq(1500, seed=800 + i) for i in range(3))
    t = trimmer_for(options, collect_statistics=True, poly_a=True)
    res = SerialRunner(t, buffer_size=1 << 18).run(data, io.BytesIO())
    vec, max_len, kmax = res["statistics_vector"]
    one = trimmer_for(options, collect_statistics=True, poly_a=True)
    one.process_chunk(data)
    v1, l1, k1 = one.statistics_vector()
    assert (max_len, kmax) == (l1, k1) and (vec == v1).all()
    t.close()
    # tools/trim_fastq.py --json writes the same statistics
    inp, out, js = tmp_path / "in.fastq", tmp_path / "out.fastq", tmp_path / "report.json"
    inp.write_bytes(data)
    root = __file__.rsplit("/", 2)[0]
    subprocess.check_call([sys.executable, f"{root}/tools/trim_fastq.py", "-a", "AGATCGGAAGAGC", "-g", "TTGACNNACG",
                           "-q", "5,20", "--poly-a", "-o", str(out), "--json", str(js), str(inp)])
    report = json.loads(js.read_text())
    assert report["written_lengths"] == {str(k): v for k, v in sorted(one.written_lengths.items())}
    assert report["poly_a_trimmed_lengths"] == {str(k): v for k, v in sorted(one.poly_a_trimmed_lengths.items())}
    stats = one.adapter_statistics()
    assert [a["three_prime_end"]["adjacent_bases"] for a in report["adapters"][:1]] == [stats[0].back.adjacent_bases]
    assert report["counters"]["n_written"] == one.statistics["n_written"]


def test_fasta_retry_is_counted_once():
    # "> rc" names of one-base reads make the FASTA output larger than the first buffer: the chunk runs again
    data = b">\nT\n" * 20000
    adapters = [PA.BackAdapter("A", max_errors=0.0, min_overlap=1, name="a")]
    t = FastqTrimmer(adapters, revcomp=True, action="none", input_format="fasta", collect_statistics=True)
    out = t.process_chunk(data)
    assert out == b"> rc\nA\n" * 20000
    vec, _, _ = t.statistics_vector()
    assert vec[0] == 20000 and vec[6] == 20000
    (st,) = t.adapter_statistics()
    assert st.reverse_complemented == 20000
    assert sum(st.back.lengths.values()) == 20000


def test_paired_mates_have_their_own_statistics():
    o1 = dict(adapters=[["back", "AGATCGGAAGAGC"]], quality_cutoff=[0, 20])
    o2 = dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]])
    d1, d2 = synthetic_fastq(3000, seed=500), synthetic_fastq(3000, seed=501)
    for mode in ("any", "both", "first"):
        opts1 = dict(quality_cutoff=(0, 20), minimum_length=30, times=2)
        opts2 = dict(minimum_length=30, poly_a=True)
        t = PairedFastqTrimmer(fastq_case_adapters(o1), fastq_case_adapters(o2), opts1, opts2, pair_filter=mode,
                               collect_statistics=True)
        t.process_chunk(d1, d2)
        s1, s2 = t.adapter_statistics()
        assert [(end_statistics_answer(st), st.reverse_complemented) for st in s1] == recount(o1, d1, times=2)
        assert [(end_statistics_answer(st), st.reverse_complemented) for st in s2] == recount(o2, d2)
        (v1, _, _), (v2, _, _) = t.statistics_vector()
        assert v1[6] == v2[6] == t.statistics[0]["n_written"]
        assert sum(t.written_lengths[0].values()) == sum(t.written_lengths[1].values()) == v1[6]
        assert sum(t.poly_a_trimmed_lengths[1].values()) == 3000 and t.poly_a_trimmed_lengths[0] == {}


def test_pair_adapters_count_pairs():
    a1 = [PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1, name="x"), PA.BackAdapter("CACGTCTGAACTC", name="y")]
    a2 = [PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1, name="x2"), PA.BackAdapter("TTGACNNACG", name="y2")]
    d1, d2 = synthetic_fastq(3000, seed=600), synthetic_fastq(3000, seed=601)
    t = PairedFastqTrimmer(a1, a2, pair_adapters=True, collect_statistics=True)
    t.process_chunk(d1, d2)
    s1, s2 = t.adapter_statistics()
    assert len(s1) == len(s2) == 2
    n1 = [sum(st.back.lengths.values()) for st in s1]
    n2 = [sum(st.back.lengths.values()) for st in s2]
    assert n1 == n2                                  # a pair counts only when both mates match
    assert sum(n1) == t.statistics[0]["with_adapters"] > 0


def test_bad_arguments():
    options = dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]])
    data = synthetic_fastq(100, seed=700)
    t = trimmer_for(options)
    t.params.stats = 12345
    with pytest.raises(ValueError):
        t.process_chunk(data)
    wrong = _lib.FastqStatistics(t.ctx, 3)
    t.params.stats = wrong.handle
    with pytest.raises(ValueError):
        t.process_chunk(data)
    wrong.close()
    p = PairedFastqTrimmer(fastq_case_adapters(options), fastq_case_adapters(options), collect_statistics=True)
    p.params2.stats = p.params1.stats
    with pytest.raises(ValueError):
        p.process_chunk(data, data)
