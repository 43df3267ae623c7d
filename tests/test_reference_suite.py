"""
The cases of the reference's own tests/test_kmer_heuristic.py, run against this package's kmer_heuristic: the
reference's answers on those inputs (and on real adapters) are stored in tests/golden/reference_kat.json.gz
(make_reference_golden.py), so nothing of the reference is needed here.
"""
import os
import sys
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sorted_sets(items):
    return sorted(([a, b, sorted(k)] for a, b, k in items), key=repr)


@pytest.mark.parametrize("name,extra", [("test_kmer_heuristic.py", [])])
def test_reference_test_file_passes_against_this_package(name, extra):
    from util import canonical, reference_answers

    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import cutadapt_b200.kmer_heuristic as K

    kat = reference_answers("kmer_heuristic")
    for seq, chunks, expected in kat["chunks"]:
        assert sorted(K.kmer_chunks(seq, chunks)) == expected, (seq, chunks)
    for lst, expected in kat["minimize"]:
        got = K.minimize_kmer_search_list([tuple(x) for x in lst])
        assert sorted(canonical(got), key=repr) == expected, lst
    for adapter, min_overlap, rate, expected in kat["searchsets"]:
        assert _sorted_sets(K.create_back_overlap_searchsets(adapter, min_overlap, rate)) == expected, adapter
    for seq, kw, expected in kat["positions"]:
        assert _sorted_sets(K.create_positions_and_kmers(seq, error_rate=0.1, **kw)) == expected, (seq, kw)
    # no quadratic or exponential algorithm: a 1000-base adapter is handled in well under a second
    t0 = time.perf_counter()
    K.create_positions_and_kmers("A" * 1000, min_overlap=3, error_rate=0.1, back_adapter=True, front_adapter=False,
                                 internal=True)
    assert time.perf_counter() - t0 < 0.5
