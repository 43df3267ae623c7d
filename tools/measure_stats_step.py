#!/usr/bin/env python3
"""
measure_stats_step.py -- where the time of bench.py's step goes when it also yields the trim statistics.

    python tools/measure_stats_step.py [--rounds R] [--reads2 N] [--pairs4 N]

For config 2 (one 3' adapter, 100 M resident reads of 150 bp) and config 4 (50 M pairs, one adapter per mate, -q 20),
with the run-time specialised first stage active, it alternates two ways of getting records plus statistics:
  (a) run() then statistics(): the trimming pass, then cg_stats_kernel over every record;
  (b) run_with_statistics(): the statistics counted inside the pass (cg_process_batch_device_stats).
Per variant and round: the step time (CUDA events around the calls of every mate) and ctx.kernel_time (the events the
library records around each call).  Then, in runs of their own: the stage split of the split pipeline
(CUTADAPT_B200_STAGE_TIMES=1) for (a) and (b), and the standalone cg_stats_kernel (statistics() on the records
alone).  Records, quality-trim intervals and vectors of (a) and (b) are compared bit for bit.  The card's name, power
limit and SM clocks are read in the same run.  Prints one JSON line per configuration.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
READ_LEN = 150


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:      # the numbers are then reported without their card
        out = f"nvidia-smi failed: {e}"
    return dict(zip(q.split(","), [p.strip() for p in out.split(",")]))


def measure(config, n, rounds):
    import torch
    from cutadapt_b200 import _lib
    from cutadapt_b200.configs import config_adapters, make_config_batch
    from cutadapt_b200.pipeline import DeviceBatch

    dev = torch.device("cuda", 0)
    data = make_config_batch(config, n, device=str(dev))
    offsets = torch.arange(n + 1, device=dev, dtype=torch.int64) * READ_LEN
    qc = (0, 20) if config == 4 else None
    mates = []
    for key, qkey, ads in (("seq", "qual", config_adapters(config)[0]), ("seq2", "qual2", config_adapters(config)[1])):
        if ads is None:
            continue
        batch = DeviceBatch(ads, quality_cutoff=qc)
        size = int(_lib.lib().cg_stats_size(batch.n_adapters, READ_LEN, 3))
        mates.append({"batch": batch, "seq": data[key].reshape(-1), "qual": data[qkey].reshape(-1) if qc else None,
                      "out": [torch.empty((n, 8), dtype=torch.int32, device=dev) for _ in range(2)],
                      "qt": [torch.empty((n, 2), dtype=torch.int32, device=dev) if qc else None for _ in range(2)],
                      "stats": [torch.zeros(size, dtype=torch.int64, device=dev) for _ in range(2)]})
    del data

    def step(variant):
        res = []
        for m in mates:
            m["stats"][variant].zero_()
            if variant == 0:
                r = m["batch"].run(m["seq"], offsets, m["qual"], max_read_len=READ_LEN, out=m["out"][0], qtrim_out=m["qt"][0])
                m["batch"].statistics(r, READ_LEN, 3, into=m["stats"][0])
            else:
                r, _ = m["batch"].run_with_statistics(m["seq"], offsets, m["qual"], max_read_len=READ_LEN, out=m["out"][1],
                                                      qtrim_out=m["qt"][1], max_len=READ_LEN, kmax=3, into=m["stats"][1])
            res.append(r)
        return res

    def kernel_ms():
        return sum(m["batch"].ctx.kernel_time(reset=True)[0] for m in mates)

    for _ in range(2):                 # warm-up: compiles the specialised kernels of both variants
        step(0)
        step(1)
    torch.cuda.synchronize()
    kernel_ms()
    jit = [m["batch"].adapter_set.jit_status() for m in mates]
    times = {0: [], 1: []}
    kern = {0: [], 1: []}
    for _ in range(rounds):
        for v in (0, 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            step(v)
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1))
            kern[v].append(kernel_ms())
    same = all(torch.equal(m["out"][0], m["out"][1]) and torch.equal(m["stats"][0], m["stats"][1]) and
               (m["qt"][0] is None or torch.equal(m["qt"][0], m["qt"][1])) for m in mates)
    # stage split, each variant in a run of its own
    stages = {}
    os.environ["CUTADAPT_B200_STAGE_TIMES"] = "1"
    for v in (0, 1):
        for m in mates:
            m["batch"].ctx.stage_times(reset=True)
        step(v)
        torch.cuda.synchronize()
        st = [m["batch"].ctx.stage_times(reset=True) for m in mates]
        stages["ab"[v]] = {k: sum(s[k] for s in st) for k in st[0]}
    del os.environ["CUTADAPT_B200_STAGE_TIMES"]
    kernel_ms()
    # the standalone statistics kernel over all records (what variant (a) adds to the pass)
    res = step(0)
    torch.cuda.synchronize()
    stats_ms = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for m, r in zip(mates, res):
            m["batch"].statistics(r, READ_LEN, 3, into=m["stats"][0])
        e1.record()
        torch.cuda.synchronize()
        stats_ms.append(e0.elapsed_time(e1))
    reads = n * len(mates)

    def med(x):
        return sorted(x)[len(x) // 2]

    return {
        "config": config, "reads_per_step": reads, "first_stage_specialised": jit, "rounds": rounds,
        "a_run_then_statistics": {"step_ms": times[0], "kernel_time_ms": kern[0], "reads_per_s_median": reads / med(times[0]) * 1e3},
        "b_run_with_statistics": {"step_ms": times[1], "kernel_time_ms": kern[1], "reads_per_s_median": reads / med(times[1]) * 1e3},
        "stage_ms": stages, "standalone_stats_kernel_ms": stats_ms,
        "records_and_vectors_equal": bool(same),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reads2", type=int, default=100_000_000, help="config 2: reads")
    ap.add_argument("--pairs4", type=int, default=50_000_000, help="config 4: pairs")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 2
    os.environ.setdefault("CUTADAPT_B200_JIT", "1")
    print(json.dumps({"card": card()}), flush=True)
    ok = True
    for config, n in ((2, args.reads2), (4, args.pairs4)):
        r = measure(config, n, args.rounds)
        ok = ok and r["records_and_vectors_equal"]
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    print(json.dumps({"card": card()}), flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
