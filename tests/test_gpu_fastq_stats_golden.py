"""
GPU tests (-m gpu): every case of tests/golden/stats_kat.json.gz -- the statistics the reference's own modifiers
collect -- through a collect entry point of the device FASTQ path with statistics on.  Each adapter's end statistics
and reverse_complemented, the poly-A histogram and the quality-trimmed bases must equal the reference's exactly; the
written-length histogram must equal the lengths of the records written.
"""
import pytest

pytestmark = pytest.mark.gpu

import cutadapt_b200.adapters as PA  # noqa: E402
from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer  # noqa: E402
from stats_cases import adapter_list, answer, repo_adapters, repo_order, trimmer_kwargs, written_lengths_of  # noqa: E402
from util import canonical, fastq_cases, fastq_paired_cases, golden  # noqa: E402

GOLDEN = golden("stats_kat.json.gz")
ENTRY = ("collect", "demux", "info", "rest")


def poly(d):
    return {int(k): v for k, v in d.items()}


def single_input(case):
    if case["source"] == "synthetic":
        return GOLDEN["inputs"][case["name"]].encode("latin-1"), None
    c = {c["name"]: c for c in fastq_cases()}[case["name"]]
    return c["input_bytes"], c["expected_bytes"]


def check_mate(t_answer, t_poly, vec, mate, options):
    assert canonical(t_answer) == canonical(repo_order(options, mate["adapters"]))
    assert t_poly == poly(mate["poly_a"])
    assert vec[3] == mate["quality_trimmed_bp"]


@pytest.mark.parametrize("i", range(len(GOLDEN["cases"])), ids=[c["name"] for c in GOLDEN["cases"]])
def test_single_end_case(i):
    case = GOLDEN["cases"][i]
    o = case["options"]
    data, expected = single_input(case)
    t = FastqTrimmer(repo_adapters(o["adapters"], o), collect_statistics=True, **trimmer_kwargs(o))
    entry = ENTRY[i % len(ENTRY)] if o["adapters"] else "collect"
    if entry == "rest" and any(s[0] == "linked" for s in o["adapters"]):
        entry = "info"                       # the rest file is undefined for linked adapters
    if entry == "collect":
        out = t.process_chunk(data)
    elif entry == "demux":
        out = b"".join(t.process_chunk_demux(data).values())
    elif entry == "info":
        out, _ = t.process_chunk_info(data)
    else:
        out, _ = t.process_chunk_rest(data)
    vec, _, _ = t.statistics_vector()
    check_mate(answer(t.adapter_statistics()), t.poly_a_trimmed_lengths, vec, case, o)
    assert t.written_lengths == written_lengths_of(out)
    if expected is not None and entry != "demux":
        assert out == expected
        assert t.written_lengths == written_lengths_of(expected)
    assert vec[6] == sum(t.written_lengths.values()) == t.statistics["n_written"]


def paired_inputs(case):
    if case["source"] == "synthetic":
        return [GOLDEN["inputs"][f"{case['name']}.{k}"].encode("latin-1") for k in (1, 2)], None
    c = {c["name"]: c for c in fastq_paired_cases()}[case["name"]]
    return c["input_bytes"], c["expected_bytes"]


@pytest.mark.parametrize("i", range(len(GOLDEN["paired_cases"])), ids=[c["name"] for c in GOLDEN["paired_cases"]])
def test_paired_case(i):
    case = GOLDEN["paired_cases"][i]
    opts = case["options"]
    (d1, d2), expected = paired_inputs(case)
    top = {k: opts[k] for k in ("error_rate", "min_overlap") if k in opts}
    o1, o2 = dict(opts["options1"], **top), dict(opts["options2"], **top)
    a1, a2 = adapter_list(PA, opts["adapters1"], o1), adapter_list(PA, opts["adapters2"], o2)
    t = PairedFastqTrimmer(a1, a2, trimmer_kwargs(o1), trimmer_kwargs(o2), pair_filter=opts.get("pair_filter", "any"),
                           pair_adapters=bool(opts.get("pair_adapters")), collect_statistics=True)
    entry = "collect" if opts.get("pair_adapters") or not a1 else ("demux", "combinatorial", "collect")[i % 3]
    if entry == "combinatorial" and not a2:
        entry = "demux"
    if entry == "collect":
        out1, out2 = t.process_chunk(d1, d2)
    else:
        # combinatorial with discard_untrimmed: pairs without a writer are dropped and not counted
        outs = t.process_chunk_demux(d1, d2, combinatorial=entry == "combinatorial",
                                     discard_untrimmed=entry == "combinatorial")
        out1, out2 = b"".join(v[0] for v in outs.values()), b"".join(v[1] for v in outs.values())
    vecs = t.statistics_vector()
    stats = t.adapter_statistics()
    for k, (mate, o, out) in enumerate(zip(case["mates"], (o1, o2), (out1, out2))):
        check_mate(answer(stats[k]), t.poly_a_trimmed_lengths[k], vecs[k][0], mate, dict(o, adapters=[]))
        assert t.written_lengths[k] == written_lengths_of(out)
        assert vecs[k][0][6] == sum(t.written_lengths[k].values())
    if expected is not None and entry == "collect":
        assert [out1, out2] == list(expected)
