"""The quality-window corpus (tests/golden/qualtrim_edges_kat.json.gz) and the batches tests/quality_windows.py builds
from it, checked without a device: the restatement and the oracle give the reference's answers, the corpus reaches
every edge it is meant to, the poison can tell a leaking window from a clean one, and the host build of the device
functions gives the oracle's records and windows on every batch."""
import ctypes as C

import numpy as np
import pytest

import quality_windows as QW
from oracle import oracle


@pytest.fixture(scope="module")
def corpus():
    return QW.corpus()


def test_restatement_and_oracle_equal_the_reference(corpus):
    for fam, q, cf, cb, base, s, e in corpus["quality"]:
        assert QW.trim_index(q, cf, cb, base) == (s, e), (fam, q, cf, cb, base)
        assert oracle.quality_trim_index(q.encode("latin-1"), cf, cb, base) == (s, e), (fam, q, cf, cb, base)
    for fam, seq, q, ns_cut, cf, cb, base, stop, s, e in corpus["nextseq"]:
        assert QW.nextseq_index(seq, q, ns_cut, base) == stop
        assert oracle.nextseq_trim_index(seq, q, ns_cut, base) == stop
        assert oracle.quality_trim_index(q[:stop], cf, cb, base) == (s, e)


def test_corpus_reaches_every_edge(corpus):
    cov = QW.coverage(corpus)
    assert not QW.missing(corpus), "edges the corpus does not reach: " + ", ".join(QW.missing(corpus))
    # the step boundaries of the warp scan, at both ends, each by several strings
    for e in "53":
        for t in (32, 33, 64, 65, 96, 97, 128, 129, 255, 256):
            assert cov[f"tail{e}:{t}"] >= 2, (e, t)
    assert len(corpus["quality"]) > 5000 and len(corpus["nextseq"]) > 200


def test_poisoned_windows_discriminate(corpus):
    """For a clear share of the poisoned reads the adapter's bytes outside the window change the match: a kernel that
    let them in would give another record."""
    import cutadapt_b200.adapters as PA

    b = QW.batch(corpus, (5, 20, 33), max_len=256, seed=1)
    idx = [i for i, p in enumerate(b.poison) if p is not None]
    assert len(idx) > 500
    for cls in (PA.BackAdapter, PA.FrontAdapter, PA.AnywhereAdapter):
        d = cls(QW.ADAPTER, max_errors=0.1, name="a").descriptor()
        clean = [b.seqs[i][b.windows[i][0]:b.windows[i][1]] for i in idx]
        leaky = [QW.leaky_view(b, i) for i in idx]
        m_clean, _ = oracle.oracle_process([d], None, clean)
        m_leaky, _ = oracle.oracle_process([d], None, leaky)
        hit = m_clean["adapter"][:, 0, 0] >= 0
        length = lambda m: m["rstop"][:, 0, 0] - m["rstart"][:, 0, 0]  # noqa: E731
        differ = hit & ((m_leaky["adapter"][:, 0, 0] < 0) | (length(m_clean) != length(m_leaky)))
        assert differ.sum() > 0.3 * len(idx), (cls.__name__, int(hit.sum()), int(differ.sum()), len(idx))


def _hostsim(spec, data, qd, offsets, params, mode):
    from cutadapt_b200 import _lib as L
    from util import hostsim_lib

    arr, n, garr, ng = spec.to_ctypes()
    iarr, ni = spec.index_ctypes()
    nr = offsets.size - 1
    out = np.zeros((nr, max(1, params.times), spec.slots), dtype=L.MATCH_DTYPE)
    qt = np.zeros((nr, 2), dtype=np.int32)
    rc = hostsim_lib().hs_process_batch_indexed(arr, n, garr, ng, iarr, ni, data.ctypes.data, qd.ctypes.data,
                                                offsets.ctypes.data, nr, C.byref(params), out.ctypes.data,
                                                qt.ctypes.data, mode)
    assert rc == 0, hostsim_lib().hs_last_error()
    return out, qt


@pytest.mark.parametrize("mode", [0, 2, 64, 256])
def test_hostsim_gives_the_oracles_records_on_every_batch(corpus, mode):
    """The host build of the first stage's per-read functions (pre_trim_core, then the scan the mode selects) on every
    parameter set's batch, and on the --nextseq-trim batches: records and windows equal the oracle's, and the windows
    equal the reference's answers stored with the corpus."""
    import cutadapt_b200.adapters as PA
    from cutadapt_b200 import _lib as L
    from util import spec_of

    spec = spec_of(PA.MultipleAdapters([PA.BackAdapter(QW.ADAPTER, max_errors=0.1, name="a")]))
    cases = [(p, False) for p in QW.param_sets(corpus)]
    cases += [((ns, 0, 30, b), True) for ns in QW.NEXTSEQ_CUTOFFS for b in QW.BASES]
    for params, nextseq in cases:
        b = QW.batch(corpus, params, max_len=256 if mode >= 64 else None, seed=2, nextseq=nextseq)
        data, offsets, qd = b.packed()
        ns_cut, cf, cb, base = params if nextseq else (None,) + params
        p = L.make_params(quality_trim=True, cutoff_front=cf, cutoff_back=cb, quality_base=base, nextseq_cutoff=ns_cut)
        got, gqt = _hostsim(spec, data, qd, offsets, p, mode)
        exp, eqt = oracle.oracle_process_packed(spec.adapters, spec.groups, data, offsets, qd, True, cf, cb, base, 1,
                                                ns_cut)
        assert (gqt == eqt).all(), (params, mode, np.nonzero((gqt != eqt).any(axis=1))[0][:5])
        assert (got == exp).all(), (params, mode, np.nonzero(got != exp)[0][:5])
        known = [i for i, w in enumerate(b.windows) if w is not None]
        assert [tuple(eqt[i]) for i in known] == [b.windows[i] for i in known], params
