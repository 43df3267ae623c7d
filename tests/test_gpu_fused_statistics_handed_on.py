"""Trim statistics of the reads the first stage hands on, listed where the plan stage, its second launch (windows with
other letters than A/C/G/T) or a DP round writes their final records and counted once per sub-batch, against the
standalone statistics kernel on the records: bit for bit, with the interpreted and the run-time specialised first
stage, over sub-batch seams."""
import numpy as np
import pytest

import test_gpu_fused_statistics as F

pytestmark = pytest.mark.gpu

N = 60_000
ADAPTER = b"AGATCGGAAGAGC"


def _handed_on_reads(seed, read_len, five_prime=False):
    """Reads the first stage cannot settle: the adapter (or its start, at the 3' end) with one substitution, deletion
    or insertion at every position of the read, some without an error, N inside some windows, each behind a chosen
    base.  Fixed-length reads of a multiple of 16 bases keep every window's first character 16-byte aligned.  Device
    buffers and offsets."""
    import torch

    rng = np.random.default_rng(seed)
    seq = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, (N, read_len))]
    ad = np.frombuffer(ADAPTER, dtype=np.uint8)
    for r in range(N):
        a = ad.copy()
        kind = r % 4
        j = int(rng.integers(0, a.size))
        if kind == 1:
            a[j] = b"ACGT"[(b"ACGT".index(bytes([a[j]])) + 1) % 4]
        elif kind == 2:
            a = np.delete(a, j)
        elif kind == 3:
            a = np.insert(a, j, np.uint8(ord("ACGT"[r % 4])))
        if five_prime:
            # the 5' adapter ends at p (possibly cut off at the start of the read)
            p = int(rng.integers(3, read_len - 20))
            k = min(a.size, p)
            seq[r, p - k:p] = a[a.size - k:]
        else:
            p = r % (read_len - 3)              # every start position, including 0 and the last ones
            k = min(a.size, read_len - p)
            seq[r, p:p + k] = a[:k]
            if p > 0:
                seq[r, p - 1] = b"ACGTNa"[r % 6]
        if r % 7 == 0:
            seq[r, int(rng.integers(0, read_len))] = ord("N")
    lens = np.full(N, read_len, dtype=np.int64)
    lens[1::5] = rng.integers(1, read_len + 1, lens[1::5].size)        # and some ragged reads between them
    keep = np.arange(read_len)[None, :] < lens[:, None]
    offsets = np.zeros(N + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    pad = np.zeros(64, dtype=np.uint8)
    return torch.from_numpy(np.concatenate([seq[keep], pad])).cuda(), torch.from_numpy(offsets).cuda()


@pytest.mark.parametrize("jit", ["0", "1"])
@pytest.mark.parametrize("sub", [4096, 40_000])
@pytest.mark.parametrize("read_len", [128, 144])
def test_handed_on_reads_counted_in_the_pass(read_len, sub, jit, monkeypatch):
    """3' adapter with 0 or 1 error at every start of aligned and ragged reads (matches that begin at the first
    column of a DP run, so the base in front of them lies outside the staged run), N inside windows: the in-pass vector
    equals the statistics kernel's, with one counting launch per sub-batch in place of the one over all records."""
    from cutadapt_b200.configs import config_adapters
    from cutadapt_b200.pipeline import DeviceBatch

    monkeypatch.setenv("CUTADAPT_B200_JIT", jit)
    monkeypatch.setenv("CUTADAPT_B200_SUB_READS", str(sub))
    batch = DeviceBatch(config_adapters(2)[0])
    seq, offs = _handed_on_reads(seed=read_len + sub, read_len=read_len)
    for max_len, kmax in ((read_len, 3), (100, 1)):
        plain, fused = F._both(batch, seq, None, offs, max_len, kmax, read_len)
        F._assert_same(plain, fused)
        assert fused[2] - plain[2] == -(-N // sub) - 1, (plain[2], fused[2])
    res, want, _ = plain
    m = res.matches.view(-1, 8)
    errors = m[:, 6][m[:, 0] >= 0]
    assert int((errors == 1).sum()) > N // 10          # the DP rounds finished reads with one error


@pytest.mark.parametrize("jit", ["0", "1"])
def test_five_prime_adapter_counted_in_the_pass(jit, monkeypatch):
    """A 5' adapter (remove before, the read searched from its other end): removed lengths, length bins and the
    vector as the statistics kernel counts them."""
    import cutadapt_b200.adapters as PA
    from cutadapt_b200.pipeline import DeviceBatch

    monkeypatch.setenv("CUTADAPT_B200_JIT", jit)
    monkeypatch.setenv("CUTADAPT_B200_SUB_READS", "4096")
    batch = DeviceBatch(PA.MultipleAdapters([PA.FrontAdapter(ADAPTER.decode(), max_errors=0.1, min_overlap=3, name="f")]))
    seq, offs = _handed_on_reads(seed=5, read_len=144, five_prime=True)
    plain, fused = F._both(batch, seq, None, offs, 144, 3, 144)
    F._assert_same(plain, fused)
    assert int(plain[1][2]) > N // 2      # reads with an adapter
