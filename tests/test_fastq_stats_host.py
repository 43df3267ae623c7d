"""
CPU tests of the statistics vector of the FASTQ path (include/cutadapt_b200.h: cg_fastq_stats_read): its layout, the
re-layout to a larger (max_len, kmax) and the merge of ranks whose layouts differ.
"""
import socket

import numpy as np

from cutadapt_b200.pipeline import (end_block, fastq_stats_layout, poly_a_trimmed_lengths, relayout_statistics,
                                    stats_layout, written_lengths)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def test_layout_extends_the_stats_layout():
    for n, max_len, kmax in ((0, 0, 0), (1, 150, 3), (96, 151, 1), (4, 10000, 7)):
        base, lay = stats_layout(n, max_len, kmax), fastq_stats_layout(n, max_len, kmax)
        assert lay["reverse_complemented"] == base["size"]
        assert lay["poly_a"] == base["size"] + n
        assert lay["size"] == base["size"] + n + max_len + 1


def test_relayout_is_lossless():
    rng = np.random.default_rng(5)
    for n, (l0, k0), (l1, k1) in ((3, (20, 2), (35, 4)), (1, (150, 3), (150, 3)), (2, (0, 0), (7, 1)),
                                  (4, (12, 5), (12, 9))):
        v = rng.integers(0, 10 ** 6, fastq_stats_layout(n, l0, k0)["size"]).astype(np.int64)
        w = relayout_statistics(v, n, l0, k0, l1, k1)
        assert w.size == fastq_stats_layout(n, l1, k1)["size"]
        assert w.sum() == v.sum()                                       # nothing lost, nothing invented
        assert (w[:16] == v[:16]).all()
        assert written_lengths(w, l1) == written_lengths(v, l0)
        assert poly_a_trimmed_lengths(w, n, l1, k1) == poly_a_trimmed_lengths(v, n, l0, k0)
        old, new = fastq_stats_layout(n, l0, k0), fastq_stats_layout(n, l1, k1)
        for a in range(n):
            for end in (0, 1):
                adj0, h0 = end_block(v, old, a, end)
                adj1, h1 = end_block(w, new, a, end)
                assert (adj0 == adj1).all()
                assert (h1[:l0 + 1, :k0 + 1] == h0).all() and h1.sum() == h0.sum()
        r = new["reverse_complemented"]
        assert (w[r:r + n] == v[old["reverse_complemented"]:old["reverse_complemented"] + n]).all()
        # growing in two steps is growing once
        mid = relayout_statistics(v, n, l0, k0, (l0 + l1) // 2, (k0 + k1) // 2)
        assert (relayout_statistics(mid, n, (l0 + l1) // 2, (k0 + k1) // 2, l1, k1) == w).all()
    try:
        relayout_statistics(np.zeros(fastq_stats_layout(1, 10, 2)["size"], np.int64), 1, 10, 2, 9, 2)
    except ValueError:
        pass
    else:
        raise AssertionError("shrinking must be refused")


def test_two_ranks_with_different_layouts_merge_to_the_sum(tmp_path):
    import torch.multiprocessing as mp
    import _fastq_stats_worker as w

    mp.spawn(w.run, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    m0, m1 = np.load(tmp_path / "merged0.npy"), np.load(tmp_path / "merged1.npy")
    assert (m0 == m1).all()
    assert list(np.load(tmp_path / "shape0.npy")) == [150, 4] == list(np.load(tmp_path / "shape1.npy"))
    expect = 0
    for rank in (0, 1):
        v, n, max_len, kmax = w.vector(rank)
        expect = expect + relayout_statistics(v, n, max_len, kmax, 150, 4)
    assert (m0 == expect).all()
