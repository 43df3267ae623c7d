"""
CPU tests of tests/golden/stats_kat.json.gz, the statistics the reference's own modifiers collect
(make_stats_golden.py): an independent recount (the oracle's records on what the cutter saw + the repository's
create_statistics / add_match) agrees with every stored case, and the host build of stats_read_core -- what
cg_stats_kernel runs on the device -- reproduces every stored case from the same records.
"""
import numpy as np
import pytest

from cutadapt_b200.pipeline import adapter_statistics_from_vector
from stats_cases import answer, cutter_records, recount, repo_order, statistics_members
from util import canonical, fastq_cases, golden, hostsim_statistics

GOLDEN = golden("stats_kat.json.gz")


def case_input(case):
    if case["source"] == "synthetic":
        return GOLDEN["inputs"][case["name"]].encode("latin-1")
    return {c["name"]: c["input_bytes"] for c in fastq_cases()}[case["name"]]


def recountable():
    return [c for c in GOLDEN["cases"] if not c["options"].get("index")]


def test_golden_covers_the_cases():
    names = {c["name"] for c in GOLDEN["cases"]}
    assert {c["name"] for c in fastq_cases()} <= names
    assert {"syn_index96", "syn_rightmost", "syn_revcomp_linked_mask", "syn_lowercase_anywhere"} <= names
    assert {"syn_pair_adapters", "syn_paired_poly"} <= {c["name"] for c in GOLDEN["paired_cases"]}
    assert sum(rc for c in GOLDEN["cases"] for _, rc in c["adapters"]) > 0
    assert set(GOLDEN["provenance"]) >= {"modifiers.py", "adapters.py"}


@pytest.mark.parametrize("case", recountable(), ids=lambda c: c["name"])
def test_recount_agrees_with_the_reference(case):
    got, qbp = recount(case["options"], case_input(case))
    assert canonical(got) == canonical(case["adapters"])
    assert qbp == case["quality_trimmed_bp"]


@pytest.mark.parametrize("case", [c for c in recountable() if c["options"]["adapters"]], ids=lambda c: c["name"])
def test_host_stats_read_core_reproduces_the_reference(case):
    multi, matches, seqs, windows, is_rc, _ = cutter_records(case["options"], case_input(case))
    n = len(multi._flatten()[0])
    max_len = max([len(s) for s in seqs] + [1])
    vec = hostsim_statistics(seqs, matches, np.array(windows, dtype=np.int32).reshape(-1, 2), n, max_len, 8)
    stats = adapter_statistics_from_vector(vec, multi, max_len, 8)
    for st, a in zip(stats, statistics_members(multi)):
        assert st.adapter is a
    got = [ans[0] for ans in answer(stats)]
    assert canonical(got) == canonical([a[0] for a in repo_order(case["options"], case["adapters"])])
