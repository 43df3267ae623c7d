"""End-to-end throughput of the FASTQ entry point (not a bench line; see DESIGN.md sections 4.6, 4.7).

  python tools/measure_fastq.py [n_reads] [chunk_megabytes] [fastq | fasta | fasta60 | barcodes | paired | interleaved]
                                [--statistics] [--redirect]

Builds n_reads synthetic FASTQ records of BASELINE configs[1]'s shape (150 bp, Phred+33 qualities, names
"@SIM2:000000123") in pinned host memory, cuts the buffer into chunks of whole records and streams them
through FastqTrimmer.process_chunks (-a AGATCGGAAGAGC -q 20 -m 20): raw FASTQ bytes in, trimmed FASTQ bytes
out, host -> device -> host inside the timed region.  Prints one JSON line.  "fasta" / "fasta60": the same reads as
FASTA (">SIM2:000000123" and the sequence on one line / wrapped at 60 columns) through the FASTA path
(input_format="fasta", -a AGATCGGAAGAGC -m 20: FASTA has no qualities to trim).  "barcodes": the FASTQ reads with
the 96 anchored 5' barcodes of config 5 (-g ^BARCODE..., IndexedPrefixAdapters) instead of the 3' adapter.
--statistics: the trimmer also collects the report's statistics (collect_statistics=True; cg_fastq_stats_*).
--redirect: the filters keep what they remove (--too-short-output --untrimmed-output: process_chunks_split,
cg_fastq_collect_split); the output bytes are those of all three outputs.
"paired" / "interleaved": the same n_reads records as n_reads / 2 pairs (-a / -A AGATCGGAAGAGC -q 20 -m 20 on both
mates; the mates of a pair share their name): "paired" streams them as two mate chunks per step
(PairedFastqTrimmer.process_chunks_split, two uploads, two outputs), "interleaved" as one interleaved chunk in and out
(cg_fastq_submit_interleaved, interleaved_outputs=("output",)); each step holds the same pairs, chunk_megabytes in all.
--gzip: the FASTQ variant in three arms, alternating over three rounds in one process: plain output, gzip output
compressed on the device (gzip_outputs=("output",)), and plain output compressed on the host by zlib level 1 on one
thread (one stream over the run).  Per arm: host-to-host reads/s, output bytes, compression ratio and device-to-host
bytes per chunk (Context.transfer_bytes); the card's name and power limit are read in the same run (nvidia-smi, a
read-only query).  A second line: the device time of gz_compress_kernel and gz_gather_kernel per MiB of plain output
and per chunk, from torch.profiler's CUDA activity in a run of its own over the warmed chunks, next to the wall time
per chunk that gzip adds, so that kernel time and the host round trip of the compaction can be told apart.
"""
import json
import subprocess
import sys
import time
import zlib

import numpy as np
import torch

sys.path.insert(0, __file__.rsplit("/", 2)[0])
import cutadapt_b200.adapters as PA  # noqa: E402
from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer  # noqa: E402
from cutadapt_b200.synth import make_read_tensor  # noqa: E402


def build_fastq(n, pinned=True, pair_names=False):
    """n records; pair_names: records 2p and 2p + 1 are named after pair p (the two mates of an interleaved file)."""
    seq, qual = make_read_tensor(n, config=2, device="cuda", with_qualities=True)
    name_len = 6 + 9
    rec_len = 1 + name_len + 1 + 150 + 3 + 150 + 1
    rec = torch.empty((n, rec_len), dtype=torch.uint8, device="cuda")
    rec[:, 0] = ord("@")
    rec[:, 1:6] = torch.tensor(list(b"SIM2:"), dtype=torch.uint8, device="cuda")
    idx = torch.arange(n, device="cuda") // (2 if pair_names else 1)
    for d in range(10):
        rec[:, 6 + 9 - d] = (48 + (idx // 10 ** d) % 10).to(torch.uint8)
    o = 1 + name_len
    rec[:, o] = 10
    rec[:, o + 1:o + 151] = seq
    rec[:, o + 151] = 10
    rec[:, o + 152] = ord("+")
    rec[:, o + 153] = 10
    rec[:, o + 154:o + 304] = qual
    rec[:, o + 304] = 10
    host = torch.empty(n * rec_len, dtype=torch.uint8, pin_memory=pinned)
    host.copy_(rec.view(-1))
    torch.cuda.synchronize()
    return host.numpy(), rec_len


def build_fasta(n, wrap=None, pinned=True):
    """The reads of build_fastq as FASTA records of equal size: one sequence line, or lines of `wrap` columns."""
    seq, _ = make_read_tensor(n, config=2, device="cuda", with_qualities=True)
    name_len = 6 + 9
    cuts = list(range(0, 150, wrap or 150))
    rec_len = 1 + name_len + 1 + 150 + len(cuts)
    rec = torch.empty((n, rec_len), dtype=torch.uint8, device="cuda")
    rec[:, 0] = ord(">")
    rec[:, 1:6] = torch.tensor(list(b"SIM2:"), dtype=torch.uint8, device="cuda")
    idx = torch.arange(n, device="cuda")
    for d in range(10):
        rec[:, 6 + 9 - d] = (48 + (idx // 10 ** d) % 10).to(torch.uint8)
    o = 1 + name_len
    rec[:, o] = 10
    o += 1
    for c in cuts:
        w = min(150, c + (wrap or 150)) - c
        rec[:, o:o + w] = seq[:, c:c + w]
        rec[:, o + w] = 10
        o += w + 1
    host = torch.empty(n * rec_len, dtype=torch.uint8, pin_memory=pinned)
    host.copy_(rec.view(-1))
    torch.cuda.synchronize()
    return host.numpy(), rec_len


def measure_gzip(n, chunk_mb):
    data, rec_len = build_fastq(n)
    per_chunk = max(1, (chunk_mb << 20) // rec_len)
    chunks = [data[i * rec_len:min(n, i + per_chunk) * rec_len] for i in range(0, n, per_chunk)]
    adapters = [PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1)]
    opts = dict(quality_cutoff=(0, 20), minimum_length=20)
    arms = {"plain": FastqTrimmer(adapters, **opts), "device_gzip": FastqTrimmer(adapters, **opts, gzip_outputs=("output",)),
            "host_zlib1": FastqTrimmer(adapters, **opts)}

    def run(name, cs):
        t = arms[name]
        if name != "host_zlib1":
            return sum(len(o) for o in t.process_chunks(cs, copy=False)), 0
        z = zlib.compressobj(1, zlib.DEFLATED, 31)
        plain = out = 0
        for o in t.process_chunks(cs, copy=False):
            plain += len(o)
            out += len(z.compress(o))
        return out + len(z.flush()), plain

    for name in arms:
        run(name, chunks[:3])                     # warm-up: buffers, module load
    res = {name: {"wall_s": 0.0, "out_bytes": 0, "d2h_bytes": 0} for name in arms}
    for _ in range(3):
        for name in arms:
            ctx = arms[name].ctx
            ctx.transfer_bytes(reset=True)
            t0 = time.perf_counter()
            out, _ = run(name, chunks)
            res[name]["wall_s"] += time.perf_counter() - t0
            res[name]["out_bytes"] = out
            res[name]["d2h_bytes"] = ctx.transfer_bytes()[1]
    plain_bytes = res["plain"]["out_bytes"]
    for name, r in res.items():
        r["reads_per_s"] = 3 * n / r["wall_s"]
        r["ratio"] = plain_bytes / r["out_bytes"]
        r["d2h_bytes_per_chunk"] = r["d2h_bytes"] / len(chunks)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"what": "FASTQ -> trimmed FASTQ (-a AGATCGGAAGAGC -q 20 -m 20), host to host: plain, device gzip, "
                              "plain + host zlib level 1 (one thread)", "reads": n, "chunk_mb": chunk_mb,
                      "chunks": len(chunks), "gpu": torch.cuda.get_device_name(), "card_and_power_limit": card,
                      "arms": res}))

    # the compressor's kernels alone, in a profiled run of their own
    from torch.profiler import ProfilerActivity, profile

    rounds = 3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            run("device_gzip", chunks)
        torch.cuda.synchronize()
    ms = {"gz_compress_kernel": 0.0, "gz_gather_kernel": 0.0}
    launches = {k: 0 for k in ms}
    for ev in prof.key_averages():
        for k in ms:
            if k in ev.key:
                ms[k] += ev.device_time_total / 1000.0
                launches[k] += ev.count
    if not launches["gz_compress_kernel"]:
        raise RuntimeError("the profiler saw no gz_compress_kernel launch")
    mib = rounds * plain_bytes / 2**20
    n_chunks = rounds * len(chunks)
    added = (res["device_gzip"]["wall_s"] - res["plain"]["wall_s"]) / (3 * len(chunks)) * 1000
    print(json.dumps({"what": "gzip kernels' device time (torch.profiler, CUDA activity)",
                      "card_and_power_limit": card,
                      "ms_per_MiB_plain": {k: v / mib for k, v in ms.items()},
                      "ms_per_chunk": {k: v / n_chunks for k, v in ms.items()},
                      "launches": launches, "chunk_MiB_plain": plain_bytes / len(chunks) / 2**20,
                      "wall_ms_per_chunk_added_by_gzip": added}))


def main():
    if "--gzip" in sys.argv:
        argv = [a for a in sys.argv if a != "--gzip"]
        return measure_gzip(int(argv[1]) if len(argv) > 1 else 4_000_000, int(argv[2]) if len(argv) > 2 else 64)
    collect = "--statistics" in sys.argv
    redirect = ("too_short", "untrimmed") if "--redirect" in sys.argv else ()
    argv = [a for a in sys.argv if a not in ("--statistics", "--redirect")]
    n = int(argv[1]) if len(argv) > 1 else 4_000_000
    chunk_mb = int(argv[2]) if len(argv) > 2 else 64
    variant = argv[3] if len(argv) > 3 else "fastq"
    if variant in ("paired", "interleaved"):
        n -= n % 2
        data, rec_len = build_fastq(n, pair_names=True)
    elif variant in ("fastq", "barcodes"):
        data, rec_len = build_fastq(n)
    else:
        data, rec_len = build_fasta(n, wrap=60 if variant == "fasta60" else None)
    per_chunk = max(1, (chunk_mb << 20) // rec_len)
    if variant in ("paired", "interleaved"):
        per_chunk = max(2, per_chunk // 2 * 2)         # whole pairs
    chunks = [data[i * rec_len:min(n, i + per_chunk) * rec_len] for i in range(0, n, per_chunk)]
    adapters = [PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1)]
    split = dict(redirect=redirect) if redirect else {}
    if variant in ("paired", "interleaved"):
        opts = dict(quality_cutoff=(0, 20), minimum_length=20)
        t = PairedFastqTrimmer(adapters, adapters, opts, opts, collect_statistics=collect, **split,
                               interleaved_outputs=("output",) if variant == "interleaved" else ())
        what = (f"paired FASTQ ({variant}) bytes in -> trimmed bytes out (-a/-A AGATCGGAAGAGC -q 20 -m 20), host to host")
        if variant == "paired":
            # the mates as two files: the same pairs, two chunks of chunk_megabytes per step
            mates = [np.ascontiguousarray(data.reshape(n // 2, 2, rec_len)[:, k]).reshape(-1) for k in (0, 1)]
            mates = [torch.from_numpy(m).pin_memory().numpy() for m in mates]
            half = per_chunk // 2                           # the pairs of one interleaved chunk
            chunks = [tuple(m[i * rec_len:min(n // 2, i + half) * rec_len] for m in mates) for i in range(0, n // 2, half)]
    elif variant == "fastq":
        t = FastqTrimmer(adapters, quality_cutoff=(0, 20), minimum_length=20, collect_statistics=collect, **split)
        what = "FASTQ bytes in -> trimmed FASTQ bytes out (-a AGATCGGAAGAGC -q 20 -m 20), host to host"
    elif variant == "barcodes":
        from cutadapt_b200.configs import config5_barcodes

        barcodes = [PA.PrefixAdapter(b, max_errors=0.1, min_overlap=3, indels=True, name=f"bc{i}")
                    for i, b in enumerate(config5_barcodes())]
        t = FastqTrimmer(PA.MultipleAdapters([PA.IndexedPrefixAdapters(barcodes)]), quality_cutoff=(0, 20),
                         minimum_length=20, collect_statistics=collect, **split)
        what = "FASTQ bytes in -> trimmed FASTQ bytes out (96 barcodes -g ^BC -q 20 -m 20), host to host"
    else:
        t = FastqTrimmer(adapters, minimum_length=20, input_format="fasta", collect_statistics=collect, **split)
        what = f"FASTA ({variant}) bytes in -> trimmed FASTA bytes out (-a AGATCGGAAGAGC -m 20), host to host"
    if redirect:
        what += ", --too-short-output --untrimmed-output"
    if variant in ("paired", "interleaved"):
        def run(cs):
            return sum(len(a) + len(b) for parts in t.process_chunks_split(cs) for a, b in parts.values())
    elif redirect:
        def run(cs):
            return sum(len(o) for parts in t.process_chunks_split(cs, copy=False) for o in parts.values())
    else:
        def run(cs):
            return sum(len(o) for o in t.process_chunks(cs, copy=False))
    run(chunks[:9])                    # warm-up: every slot's buffers, pool
    for st in (t.statistics if isinstance(t.statistics, tuple) else (t.statistics,)):
        st.clear()
    t0 = time.perf_counter()
    out_bytes = run(chunks)
    wall = time.perf_counter() - t0
    st = t.statistics[0] if isinstance(t.statistics, tuple) else t.statistics
    print(json.dumps({
        "what": what,
        "variant": variant, "reads": n, "chunk_mb": chunk_mb, "collect_statistics": collect, "redirect": list(redirect), "chunks": len(chunks),
        "reads_per_s": n / wall,
        "in_GB_per_s": data.size / wall / 1e9, "out_GB_per_s": out_bytes / wall / 1e9,
        "in_bytes": int(data.size),
        "gpu": torch.cuda.get_device_name(), "out_bytes": out_bytes, "wall_s": wall,
        "statistics": {k: int(v) for k, v in st.items()},
    }))


if __name__ == "__main__":
    main()
