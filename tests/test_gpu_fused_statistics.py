"""Trim statistics counted inside the trimming pass (cg_process_batch_device_stats, the default for one plain adapter)
against the standalone statistics kernel on the records (run + statistics): bit for bit, with the interpreted and the
run-time specialised first stage, at the benchmark's config-2 and config-4 shapes."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 150_000
SUB = 40_000          # reads per sub-batch of the split pipeline: four sub-batches, the last one short


def _reads(config, seed, read_len=150):
    """Reads of a configuration (config 4: read 1 and its qualities) with ragged lengths up to read_len, the adapter
    planted behind N, lower-case and upper-case bases, as 16-byte aligned device buffers with their offsets."""
    import torch
    from cutadapt_b200.configs import CONFIG2_ADAPTER, CONFIG4_R1, make_config_batch

    b = make_config_batch(config, N, seed=seed, device="cpu")
    seq = b["seq"].numpy().copy()
    qual = b["qual"].numpy().copy() if b["qual"] is not None else None
    rng = np.random.default_rng(seed)
    adapter = np.frombuffer((CONFIG4_R1 if config == 4 else CONFIG2_ADAPTER).encode(), dtype=np.uint8)
    # every fifth read: the adapter (or its start, at the end of the read) at a random place, behind a chosen base
    rows = np.arange(0, N, 5)
    pos = rng.integers(1, 150 - 5, rows.size)
    before = np.frombuffer(b"NacgtnACGT", dtype=np.uint8)[rng.integers(0, 10, rows.size)]
    for r, p, c in zip(rows, pos, before):
        k = min(adapter.size, 150 - p)
        seq[r, p:p + k] = adapter[:k]
        seq[r, p - 1] = c
    lens = rng.integers(0, read_len + 1, N)
    lens[::3] = read_len
    keep = np.arange(150)[None, :] < lens[:, None]
    offsets = np.zeros(N + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    pad = np.zeros(64, dtype=np.uint8)
    d_seq = torch.from_numpy(np.concatenate([seq[keep], pad])).cuda()
    d_qual = torch.from_numpy(np.concatenate([qual[keep], pad])).cuda() if qual is not None else None
    return d_seq, d_qual, torch.from_numpy(offsets).cuda()


def _batch(config):
    from cutadapt_b200.configs import config_adapters
    from cutadapt_b200.pipeline import DeviceBatch

    return DeviceBatch(config_adapters(config)[0], quality_cutoff=(0, 20) if config == 4 else None)


def _both(batch, seq, qual, offs, max_len, kmax, read_len=150):
    """(run + statistics, run_with_statistics) on the same reads, and the launches each made."""
    ctx = batch.ctx
    l0 = ctx.launch_count()
    res = batch.run(seq, offs, qual, max_read_len=read_len)
    want = batch.statistics(res, max_len, kmax)
    l1 = ctx.launch_count()
    res2, got = batch.run_with_statistics(seq, offs, qual, max_read_len=read_len, max_len=max_len, kmax=kmax)
    l2 = ctx.launch_count()
    return (res, want, l1 - l0), (res2, got, l2 - l1)


def _assert_same(a, b):
    import torch

    (res, want, _), (res2, got, _) = a, b
    assert torch.equal(res.matches, res2.matches)
    if res.qtrim is not None:
        assert torch.equal(res.qtrim, res2.qtrim)
    assert torch.equal(got, want), torch.nonzero(got != want)[:8].tolist()


@pytest.mark.parametrize("jit", ["0", "1"])
@pytest.mark.parametrize("config, read_len", [(2, 150), (2, 64), (4, 150)])
def test_statistics_in_the_pass_equal_the_statistics_kernel(config, read_len, jit, monkeypatch):
    """Records, quality-trim intervals and vector of run_with_statistics equal run + statistics: ragged reads, N and
    lower-case bases in front of the adapter, histograms narrower than the reads, four sub-batches.  Without quality
    trimming the statistics are counted in the pass; config 4 (-q 20) keeps the statistics kernel."""
    monkeypatch.setenv("CUTADAPT_B200_JIT", jit)
    monkeypatch.setenv("CUTADAPT_B200_SUB_READS", str(SUB))
    batch = _batch(config)
    seq, qual, offs = _reads(config, seed=11 + config, read_len=read_len)
    for max_len, kmax in ((150, 3), (100, 2), (40, 1)):
        plain, fused = _both(batch, seq, qual, offs, max_len, kmax, read_len)
        _assert_same(plain, fused)
        if config == 2:
            # counted in the pass: one statistics launch per sub-batch (the reads the first stage handed on) instead
            # of one over all records
            subs = -(-N // SUB)
            assert fused[2] - plain[2] == subs - 1, (plain[2], fused[2])
        else:
            assert fused[2] == plain[2]
    assert batch.adapter_set.jit_status() == (1 if jit == "1" else 0)


def test_interleaved_calls_on_one_set_each_use_their_kernel(monkeypatch):
    """With the specialised first stage active, run() and run_with_statistics() alternate on one adapter set; each
    call compiles / picks its own variant and stays correct."""
    import torch

    monkeypatch.setenv("CUTADAPT_B200_JIT", "1")
    batch = _batch(2)
    seq, qual, offs = _reads(2, seed=3)
    first, _ = batch.run_with_statistics(seq, offs, max_read_len=150, max_len=150, kmax=3)
    ref = first.matches.clone()
    want = batch.statistics(first, 150, 3)
    for _ in range(3):
        res = batch.run(seq, offs, max_read_len=150)
        assert torch.equal(res.matches, ref)
        res2, got = batch.run_with_statistics(seq, offs, max_read_len=150, max_len=150, kmax=3)
        assert torch.equal(res2.matches, ref) and torch.equal(got, want)
    assert batch.adapter_set.jit_status() == 1
    assert "StaticPlaneProg, true>" in batch.adapter_set.jit_source(5, False, statistics=True)
    assert "StaticPlaneProg>" in batch.adapter_set.jit_source(5, False)


@pytest.mark.parametrize("case", ["two_adapters", "wide_histogram"])
def test_sets_outside_the_fused_conditions_take_the_statistics_kernel(case, monkeypatch):
    """Two adapters (multi-pass schedule) or max_len > 4096: one standalone statistics launch after the pass, with
    the same vector as run + statistics."""
    import cutadapt_b200.adapters as PA
    from cutadapt_b200.pipeline import DeviceBatch

    monkeypatch.setenv("CUTADAPT_B200_SUB_READS", str(SUB))
    if case == "two_adapters":
        batch = DeviceBatch(PA.MultipleAdapters([PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1, name="a"),
                                                 PA.BackAdapter("CACGTCTGAACTC", max_errors=0.1, name="b")]))
        max_len, kmax = 150, 3
    else:
        batch = _batch(2)
        max_len, kmax = 5000, 1
    seq, _, offs = _reads(2, seed=5)
    plain, fused = _both(batch, seq, None, offs, max_len, kmax)
    _assert_same(plain, fused)
    assert fused[2] == plain[2]
