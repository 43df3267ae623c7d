"""
The quality-trimmed window on every device path that computes it or searches inside it, against the oracle
(-m gpu): the corpus of tests/golden/qualtrim_edges_kat.json.gz (the warp quality scan of the bit-plane first stage at
its 32-character steps, ties, zero sums, closing windows, bytes below the base and >= 128) in the read batches of
tests/quality_windows.py (whole tiles that need the warp scan, a 256-character tail on lane 0 or lane 31 only, empty
reads, a ragged count, a shuffled copy; adapters that straddle the window's edges with the missing part just outside).
Records and windows must equal the oracle's bit for bit; FASTQ output byte for byte.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import quality_windows as QW  # noqa: E402
from cutadapt_b200 import _lib as L  # noqa: E402
from oracle import oracle  # noqa: E402

SHORT, MID = 160, 256          # bit-plane widths: 5 words up to 160 characters, 8 up to 256


@pytest.fixture(scope="module")
def corpus():
    return QW.corpus()


def _adapters(kind):
    import cutadapt_b200.adapters as PA

    a = dict(max_errors=0.1, name="a")
    if kind == "back":
        return [PA.BackAdapter(QW.ADAPTER, **a)]
    if kind == "two":
        return [PA.BackAdapter(QW.ADAPTER, **a), PA.FrontAdapter(QW.ADAPTER[::-1], max_errors=0.1, name="f")]
    if kind == "anywhere":
        return [PA.AnywhereAdapter(QW.ADAPTER, **a)]
    if kind == "front":
        return [PA.FrontAdapter(QW.ADAPTER, **a)]
    assert kind == "linked"
    return [PA.BackAdapter(QW.ADAPTER, **a),
            PA.LinkedAdapter(PA.FrontAdapter(QW.ADAPTER[:14], max_errors=0.1, name="lf"),
                             PA.BackAdapter(QW.LINKED_BACK, max_errors=0.1, name="lb"), False, False, "l")]


def _set(kind):
    import cutadapt_b200.adapters as PA
    from util import spec_of

    spec = spec_of(PA.MultipleAdapters(_adapters(kind)))
    return spec, L.AdapterSet(L.AdapterSetSpec(spec.adapters, spec.groups))


def _split(params, nextseq):
    return params if nextseq else (None,) + tuple(params)


def _first_difference(b, got, gqt, exp, eqt):
    bad = np.nonzero((gqt != eqt).any(axis=1) | (got != exp).reshape(len(b), -1).any(axis=1))[0]
    if not bad.size:
        return None
    i = int(bad[0])
    return dict(read=i, n_bad=int(bad.size), quality=b.quals[i][:80], window=b.windows[i], poison=b.poison[i],
                got=(gqt[i].tolist(), got[i].tolist()), want=(eqt[i].tolist(), exp[i].tolist()))


def _check(label, aset, spec, b, times=1):
    """Run batch b on aset (cg_process_batch) and compare with oracle_process_packed on the same bytes."""
    ns_cut, cf, cb, base = _split(b.params, len(b.params) == 4)
    data, offsets, qd = b.packed()
    p = L.make_params(quality_trim=True, cutoff_front=cf, cutoff_back=cb, quality_base=base, times=times,
                      nextseq_cutoff=ns_cut)
    got, gqt = aset.process(data, offsets, qd, p)
    exp, eqt = oracle.oracle_process_packed(spec.adapters, spec.groups, data, offsets, qd, True, cf, cb, base, times, ns_cut)
    diff = _first_difference(b, got, gqt, exp, eqt)
    assert diff is None, (label, b.params, diff)
    return got, gqt


def _batches(corpus, max_len, nextseq=False, ascii_only=False):
    if nextseq:
        return [QW.batch(corpus, (ns, 0, 30, base), max_len, seed=7, nextseq=True, ascii_only=ascii_only)
                for ns in QW.NEXTSEQ_CUTOFFS for base in QW.BASES]
    return [QW.batch(corpus, p, max_len, seed=5, ascii_only=ascii_only) for p in QW.param_sets(corpus)]


@pytest.mark.parametrize("jit", ["0", "1"])
@pytest.mark.parametrize("max_len", [SHORT, MID])
@pytest.mark.parametrize("nextseq", [False, True])
def test_bitplane_first_stage(corpus, max_len, jit, nextseq, monkeypatch):
    """cg_pscan_kernel (warp quality scan, plane loads that blank the bytes in front of the window, TMA tiles with a
    margin, the plan stage's 16-byte window fetches), interpreted and specialised, W = 5 and W = 8."""
    monkeypatch.setenv("CUTADAPT_B200_JIT", jit)
    spec, aset = _set("back")
    for b in _batches(corpus, max_len, nextseq):
        _check(("bitplane", max_len, jit, nextseq), aset, spec, b)
    if jit == "1":
        assert aset.jit_status() == 1, L.last_error()


@pytest.mark.parametrize("max_len", [MID, None])
def test_shiftand_first_stage(corpus, max_len, monkeypatch):
    """The shift-and first stage: forced, and chosen by the batch itself for reads longer than 256."""
    if max_len is not None:
        monkeypatch.setenv("CUTADAPT_B200_SCAN", "shiftand")
    spec, aset = _set("back")
    for b in _batches(corpus, max_len) + _batches(corpus, max_len, nextseq=True):
        _check(("shiftand", max_len), aset, spec, b)


@pytest.mark.parametrize("kernel, times", [("general", 1), ("block", 1), ("warp", 1), ("general", 2)])
def test_one_phase_kernels(corpus, kernel, times, monkeypatch):
    monkeypatch.setenv("CUTADAPT_B200_KERNEL", kernel)
    spec, aset = _set("back")
    for b in _batches(corpus, MID):
        _check(("one-phase", kernel, times), aset, spec, b, times=times)


@pytest.mark.parametrize("kind", ["two", "linked", "anywhere", "front"])
@pytest.mark.parametrize("sub", [None, "1100"])
def test_multi_pass_schedule_and_seams(corpus, kind, sub, monkeypatch):
    """Several adapters (the first pass trims, every later pass searches a view), a linked adapter, and single 5' /
    anywhere adapters; with sub-batches of 1100 reads the seams fall inside 32-read tiles."""
    if sub:
        monkeypatch.setenv("CUTADAPT_B200_SUB_READS", sub)
    spec, aset = _set(kind)
    for b in _batches(corpus, None):
        _check(("multi-pass", kind, sub), aset, spec, b)


def test_split_pipeline_sub_batch_seams(corpus, monkeypatch):
    monkeypatch.setenv("CUTADAPT_B200_SUB_READS", "1100")
    spec, aset = _set("back")
    for max_len in (SHORT, MID):
        for b in _batches(corpus, max_len) + _batches(corpus, max_len, nextseq=True):
            _check(("split seams", max_len), aset, spec, b)


def test_host_facing_batch_at_size_and_without_qtrim(corpus):
    """cg_process_batch with >= 65536 reads (compressed transfer, both lanes); passing NULL for qtrim through the
    ctypes handle must not change the records."""
    spec, aset = _set("back")
    for params in ((5, 20, 33), (20, 20, 64)):
        one = QW.batch(corpus, params, MID, seed=9)
        reps = -(-65536 // len(one)) + 1
        b = QW.Batch(one.seqs * reps, one.quals * reps, one.windows * reps, one.poison * reps, params)
        got, _ = _check(("host-facing", params), aset, spec, b)
        data, offsets, qd = b.packed()
        p = L.make_params(quality_trim=True, cutoff_front=params[0], cutoff_back=params[1], quality_base=params[2])
        m = np.empty_like(got)
        L.check(L.lib().cg_process_batch(aset.ctx.handle, aset.handle, data.ctypes.data, qd.ctypes.data,
                                         offsets.ctypes.data, len(b), C.byref(p), m.ctypes.data, None))
        assert (m == got).all(), params


def test_standalone_batch_functions(corpus):
    from cutadapt_b200.qualtrim import quality_trim_index_batch, nextseq_trim_index_batch

    by = {}
    for _, q, cf, cb, base, s, e in corpus["quality"]:
        by.setdefault((cf, cb, base), []).append((q, [s, e]))
    for (cf, cb, base), rows in by.items():
        got = quality_trim_index_batch([q for q, _ in rows], cf, cb, base)
        bad = [i for i, (g, (_, w)) in enumerate(zip(got.tolist(), rows)) if g != w]
        assert not bad, ((cf, cb, base), rows[bad[0]], got[bad[0]].tolist())
    by = {}
    for _, seq, q, ns_cut, cf, cb, base, stop, _, _ in corpus["nextseq"]:
        by.setdefault((ns_cut, base), []).append((seq, q, stop))
    for (ns_cut, base), rows in by.items():
        got = nextseq_trim_index_batch([r[0] for r in rows], [r[1] for r in rows], ns_cut, base)
        assert got.tolist() == [r[2] for r in rows], (ns_cut, base)


@pytest.mark.parametrize("jit", ["0", "1"])
def test_statistics_on_quality_windows(corpus, jit, monkeypatch):
    """run_with_statistics with 5' and 3' cutoffs: the vector equals the host build of stats_read_core on the device's
    own records, which equal the oracle's; some 3' matches start exactly at the window's start (adjacent base "")."""
    import torch
    from cutadapt_b200.pipeline import DeviceBatch
    from util import hostsim_statistics

    monkeypatch.setenv("CUTADAPT_B200_JIT", jit)
    for params in ((5, 20, 33), (20, 20, 33), (0, 20, 64)):
        cf, cb, base = params
        b = QW.batch(corpus, params, MID, seed=11)
        data, offsets, qd = b.packed()
        batch = DeviceBatch(_adapters("back"), quality_cutoff=(cf, cb), quality_base=base)
        pad = np.zeros(64, dtype=np.uint8)
        d_seq = torch.from_numpy(np.concatenate([data, pad])).cuda()
        d_qual = torch.from_numpy(np.concatenate([qd, pad])).cuda()
        d_off = torch.from_numpy(offsets).cuda()
        res, stats = batch.run_with_statistics(d_seq, d_off, d_qual, max_read_len=MID, max_len=MID, kmax=3)
        recs = res.matches.cpu().numpy().view(L.MATCH_DTYPE).reshape(len(b), 1, 1)
        qt = res.qtrim.cpu().numpy().reshape(len(b), 2)
        spec = batch.spec
        exp, eqt = oracle.oracle_process_packed(spec.adapters, spec.groups, data, offsets, qd, True, cf, cb, base)
        diff = _first_difference(b, recs, qt, exp, eqt)
        assert diff is None, ("statistics records", params, diff)
        want = hostsim_statistics(b.seqs, recs, qt, 1, MID, 3)
        got = stats.cpu().numpy()
        assert (got == want).all(), (params, np.nonzero(got != want)[0][:8].tolist())
        at_start = (recs["adapter"][:, 0, 0] >= 0) & (recs["rstart"][:, 0, 0] == 0)
        assert at_start.sum() > 0, params


def _fastq_oracle(b, ads, **kw):
    import cutadapt_b200.adapters as PA
    from util import spec_of

    descs = groups = None
    if ads:
        spec = spec_of(PA.MultipleAdapters(ads))
        descs, groups = spec.adapters, spec.groups
    return oracle.oracle_fastq_trim(b.fastq(), descs, groups, **kw)


@pytest.mark.parametrize("variant", ["one", "two", "none", "nextseq", "revcomp"])
def test_fastq_path(corpus, variant):
    """The same reads as FASTQ chunks through FastqTrimmer with quality_cutoff: the split pipeline (one adapter), two
    adapters, no adapters (fq_pretrim_kernel), --nextseq-trim, --revcomp (fq_fold_qtrim_kernel)."""
    from cutadapt_b200.pipeline import FastqTrimmer

    ads = {"one": _adapters("back"), "two": _adapters("two"), "none": None, "nextseq": _adapters("back"),
           "revcomp": _adapters("back")}[variant]
    nextseq = variant == "nextseq"
    for b in _batches(corpus, None, nextseq=nextseq, ascii_only=True):
        ns_cut, cf, cb, base = _split(b.params, nextseq)
        kw = dict(quality_base=base)
        if ns_cut is not None:
            kw["nextseq_cutoff"] = ns_cut
        t = FastqTrimmer(ads, quality_cutoff=(cf, cb), revcomp=variant == "revcomp", **kw)
        got = t.process_chunk(b.fastq())
        want, counters = _fastq_oracle(b, ads, quality_trim=True, cutoff_front=cf, cutoff_back=cb,
                                       revcomp=variant == "revcomp", **kw)
        if got != want:
            g, w = got.split(b"\n"), want.split(b"\n")
            k = next(i for i, (x, y) in enumerate(zip(g, w)) if x != y)
            pytest.fail(f"{variant} {b.params}: record {k // 4} differs: {g[k][:80]!r} != {w[k][:80]!r}")
        for key, v in counters.items():
            assert t.statistics[key] == v, (variant, b.params, key)


def test_paired_fastq_config4_shape(corpus):
    """PairedFastqTrimmer in the shape of config 4: -q on both mates, one 3' adapter per mate."""
    import cutadapt_b200.adapters as PA
    from cutadapt_b200.configs import CONFIG4_R1
    from cutadapt_b200.pipeline import PairedFastqTrimmer
    from util import spec_of

    r2 = "AGATCGGAAGAGCGTCGTGTAGGGAAAGAGTGT"
    for params in ((0, 20, 33), (5, 20, 33), (20, 20, 64)):
        cf, cb, base = params
        b1 = QW.batch(corpus, params, MID, seed=13, adapter=CONFIG4_R1, ascii_only=True)
        b2 = QW.batch(corpus, params, MID, seed=14, adapter=r2, ascii_only=True)
        n = min(len(b1), len(b2))
        c1 = QW.Batch(b1.seqs[:n], b1.quals[:n], b1.windows[:n], b1.poison[:n], params).fastq()
        c2 = QW.Batch(b2.seqs[:n], b2.quals[:n], b2.windows[:n], b2.poison[:n], params).fastq()
        a1, a2 = [PA.BackAdapter(CONFIG4_R1, max_errors=0.1, name="r1")], [PA.BackAdapter(r2, max_errors=0.1, name="r2")]
        o = dict(quality_cutoff=(cf, cb), quality_base=base)
        t = PairedFastqTrimmer(a1, a2, o, o, "any")
        g1, g2 = t.process_chunk(c1, c2)
        s1, s2 = spec_of(PA.MultipleAdapters(a1)), spec_of(PA.MultipleAdapters(a2))
        ko = dict(quality_trim=True, cutoff_front=cf, cutoff_back=cb, quality_base=base)
        e1, e2, _, _ = oracle.oracle_fastq_trim_paired(c1, c2, s1.adapters, s1.groups, s2.adapters, s2.groups, ko, ko, "any")
        assert g1 == e1 and g2 == e2, params
