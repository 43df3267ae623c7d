"""Worker of tests/test_fastq_stats_host.py (gloo, world_size 2; CPU only)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def vector(rank):
    """A FASTQ-path statistics vector of 3 adapters whose layout differs per rank: (max_len, kmax) = (150, 2) / (90, 4)."""
    from cutadapt_b200.pipeline import fastq_stats_layout

    n, max_len, kmax = 3, (150, 90)[rank], (2, 4)[rank]
    rng = np.random.default_rng(rank)
    return rng.integers(0, 1000, fastq_stats_layout(n, max_len, kmax)["size"]).astype(np.int64), n, max_len, kmax


def run(rank, world, port, out_dir):
    import torch.distributed as dist
    from cutadapt_b200.pipeline import allreduce_fastq_statistics_vector

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        v, n, max_len, kmax = vector(rank)
        merged, new_len, new_kmax = allreduce_fastq_statistics_vector(v, n, max_len, kmax)
        np.save(os.path.join(out_dir, f"merged{rank}.npy"), merged)
        np.save(os.path.join(out_dir, f"shape{rank}.npy"), np.array([new_len, new_kmax]))
    finally:
        dist.destroy_process_group()
