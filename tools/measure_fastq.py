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
--gzip-input [n_reads] [submission_megabytes]: gzip input, three arms alternating over three rounds in one process on
each of two inputs of the same reads (-a AGATCGGAAGAGC -q 20 -m 20, plain output): "plain" (read_fastq_chunks on the
plain bytes), "host_gzip" (Python's gzip module on one core, the tool's path for single-member files) and "device"
(read_gzip_device_chunks: the compressed bytes are uploaded and inflated on the device).  Inputs: "multi_member"
(members of 65 280 plain bytes at zlib level 6), "mib_members" (members of 2 MiB plain, about 1 MiB compressed: the
tool's threshold) and "single_member" (one zlib level 6 member), whose device arm reads the whole input on a split
stream (split_members=True: the member inflated block-parallel).  Per arm: host-to-host reads/s and MiB/s of plain
input, and the bytes uploaded.  Then, on the single member: the stride sweep (CUTADAPT_B200_GZIN_STRIDE of 32, 64, 128
and 256 KiB, two rounds alternating), with the chunks decoded again because their speculative start was wrong
(cg_gzin_result.respeculated, from an untimed pass per stride) against the chunks searched; the file-size sweep of the
tool's rule (prefixes of the reads compressed as one member of about 4 to 64 MiB, host gzip against the split stream,
three rounds alternating) and the smallest size from which the device wins at every larger size.  Last lines: the
inflate kernels' device time per MiB of plain output from torch.profiler, in runs of their own, on the multi-member
input and on the split stream.  The card's name and power limit are read in the run.
--revcomp [n_reads] [chunk_megabytes]: the "paired" variant without and with --revcomp (the pair swap on the device), the
two arms alternating over three rounds in one process; pairs per second of each and the card's name and power limit.
--rows [n_reads] [chunk_megabytes] [--baseline-tree DIR]: the "paired" variant with the info rows of both mates
(--info-file and --info-file-paired), four arms alternating over three rounds in one process: no rows, plain rows, rows
compressed on the device (gzip_rows), and plain rows compressed by host zlib level 1 (one stream per mate, one thread).
Per arm: host-to-host reads/s and the row bytes downloaded.  With --baseline-tree (a built checkout of another commit):
its "paired" run and this tree's, both without rows, in alternating processes, three each.  The card's name and power
limit are read in the run.
--bam-input [n_reads] [submission_megabytes]: unaligned BAM input.  The same reads (-a AGATCGGAAGAGC -q 20 -m 20, plain
output) in two forms, alternating over three rounds in one process, host to host: a BGZF uBAM read through the BAM path
(FastqTrimmer(input_format="bam"), read_gzip_device_chunks: inflated, records decoded into FASTQ on the device) and the
same reads as BGZF FASTQ through the member path.  Per arm: reads/s and the compressed bytes; for the BAM arm the tiles
of the record-boundary walk and those walked again.  A second line: the BAM kernels' device time per MiB of BAM from
torch.profiler, in a run of its own.  The card's name and power limit are read in the run.
"""
import json
import os
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


def measure_gzip_input(n, submit_mb):
    import gzip
    import io
    from concurrent.futures import ThreadPoolExecutor

    from cutadapt_b200.pipeline import read_fastq_chunks, read_gzip_device_chunks

    data, rec_len = build_fastq(n, pinned=False)
    plain = data.tobytes()
    pieces = [plain[i:i + 65280] for i in range(0, len(plain), 65280)]
    with ThreadPoolExecutor(16) as ex:
        multi = b"".join(ex.map(lambda p: gzip.compress(p, 6, mtime=0), pieces))
    single = gzip.compress(plain, 6, mtime=0)
    big = [plain[i:i + (2 << 20)] for i in range(0, len(plain), 2 << 20)]
    with ThreadPoolExecutor(16) as ex:
        mib = b"".join(ex.map(lambda p: gzip.compress(p, 6, mtime=0), big))
    inputs = {"multi_member": (multi, plain), "mib_members": (mib, plain), "single_member": (single, plain)}
    adapters = [PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1)]
    opts = dict(quality_cutoff=(0, 20), minimum_length=20)
    chunk = 64 << 20

    def run(arm, gz, pl):
        t = FastqTrimmer(adapters, **opts)
        if arm == "plain":
            src = read_fastq_chunks(io.BytesIO(pl), chunk)
        elif arm == "host_gzip":
            src = read_fastq_chunks(gzip.GzipFile(fileobj=io.BytesIO(gz)), chunk)
        else:
            src = read_gzip_device_chunks(io.BytesIO(gz), t, submit_mb << 20, split_members=arm == "split")
        t.ctx.transfer_bytes(reset=True)
        t0 = time.perf_counter()
        out = sum(len(o) for o in t.process_chunks(src, copy=False))
        return time.perf_counter() - t0, out, t.ctx.transfer_bytes()[0]

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    res = {}
    for name, (gz, pl) in inputs.items():
        dev = "split" if name == "single_member" else "device"
        arms = {"plain": (gz, pl), "host_gzip": (gz, pl), dev: (gz, pl)}
        warm = plain[:rec_len * 1000]
        for arm in arms:                          # warm-up: buffers, module load
            run(arm, gzip.compress(warm, 6), warm)
        r = {arm: {"wall_s": 0.0, "plain_bytes": len(p), "gz_bytes": len(g)} for arm, (g, p) in arms.items()}
        outs = {}
        for _ in range(3):
            for arm, (g, p) in arms.items():
                w, out, up = run(arm, g, p)
                r[arm]["wall_s"] += w
                r[arm]["h2d_bytes"] = up
                outs.setdefault(len(p), set()).add(out)
        for arm, x in r.items():
            reads = x["plain_bytes"] // rec_len
            x["M_reads_per_s"] = 3 * reads / x["wall_s"] / 1e6
            x["plain_MiB_per_s"] = 3 * x["plain_bytes"] / x["wall_s"] / 2**20
        assert all(len(v) == 1 for v in outs.values()), "the arms wrote different amounts"
        res[name] = r
    print(json.dumps({"what": "gzip input -> trimmed FASTQ (-a AGATCGGAAGAGC -q 20 -m 20), host to host", "reads": n,
                      "submission_MiB": submit_mb, "gpu": torch.cuda.get_device_name(), "card_and_power_limit": card,
                      "inputs": res}))

    # the stride sweep on the single member
    import os

    from cutadapt_b200 import _lib
    from cutadapt_b200.pipeline import DeviceChunk

    def respeculated(gz):
        """(chunks decoded again, chunks searched) of one untimed pass, submissions as the reader makes them."""
        import ctypes as C

        stride = int(os.environ["CUTADAPT_B200_GZIN_STRIDE"])
        t = FastqTrimmer(adapters, **opts)
        h = C.c_int32(0)
        _lib.check(_lib.lib().cg_gzin_create_ex(t.ctx.handle, _lib.CG_GZIN_SPLIT_MEMBERS, C.byref(h)))
        pos, buf, again, searched = 0, b"", 0, 0
        try:
            while True:
                take = gz[pos:pos + (submit_mb << 20) - len(buf)]
                pos += len(take)
                buf += take
                final = pos >= len(gz)
                slot, r = C.c_int32(-1), _lib.cg_gzin_result()
                _lib.check(_lib.lib().cg_fastq_submit_gzip(t.ctx.handle, h.value, buf, len(buf), 0, int(final),
                                                           C.byref(slot), C.byref(r)))
                again += r.respeculated
                searched += max(0, (len(buf) + stride - 1) // stride - 1)
                if slot.value >= 0:
                    t.process_chunk(DeviceChunk(slot.value, r.chunk_bytes))
                buf = buf[r.consumed:]
                if final and not buf:
                    return again, searched
        finally:
            _lib.check(_lib.lib().cg_gzin_destroy(t.ctx.handle, h.value))

    strides = [32 << 10, 64 << 10, 128 << 10, 256 << 10]
    sweep = {s: {"wall_s": 0.0} for s in strides}
    for _ in range(2):
        for s in strides:
            os.environ["CUTADAPT_B200_GZIN_STRIDE"] = str(s)
            w, out, _ = run("split", single, plain)
            sweep[s]["wall_s"] += w
            outs.setdefault(len(plain), set()).add(out)
    for s in strides:
        os.environ["CUTADAPT_B200_GZIN_STRIDE"] = str(s)
        again, searched = respeculated(single)
        sweep[s].update(M_reads_per_s=2 * n / sweep[s]["wall_s"] / 1e6, respeculated=again, chunks_searched=searched,
                        false_start_rate=again / max(searched, 1))
    os.environ.pop("CUTADAPT_B200_GZIN_STRIDE")
    assert all(len(v) == 1 for v in outs.values()), "the arms wrote different amounts"
    print(json.dumps({"what": "split stream on the single member by stride S (bytes)", "reads": n,
                      "card_and_power_limit": card, "strides": sweep}))

    # the file-size sweep of the tool's rule: one member of about `mib` MiB compressed
    ratio = len(single) / len(plain)
    sizes = {}
    for mib_gz in (4, 8, 16, 32, 64):
        k = min(len(plain), int((mib_gz << 20) / ratio) // rec_len * rec_len)
        sizes[mib_gz] = (gzip.compress(plain[:k], 6, mtime=0), plain[:k])
    size_res = {m: {"host_gzip": 0.0, "split": 0.0, "gz_bytes": len(g)} for m, (g, _) in sizes.items()}
    for _ in range(3):
        for m, (g, p) in sizes.items():
            for arm in ("host_gzip", "split"):
                size_res[m][arm] += run(arm, g, p)[0]
    win = None
    for m in sorted(size_res, reverse=True):
        x = size_res[m]
        x["speedup"] = x["host_gzip"] / x["split"]
        if x["speedup"] > 1:
            win = m
        else:
            break
    print(json.dumps({"what": "one member by compressed size: host gzip against the split stream (wall s, 3 rounds)",
                      "card_and_power_limit": card, "sizes_MiB": size_res,
                      "device_wins_from_MiB": win}))

    from torch.profiler import ProfilerActivity, profile

    kernels = ("gu_cand_count", "gu_cand_write", "gu_parse", "gu_chain", "gu_place", "gu_crc", "gu_flag", "gu_select",
               "gu_search", "gu_spec", "gu_walk", "gu_window", "gu_resolve", "gu_crc_piece", "gu_crc_fold")
    for name, arm, gz in (("multi-member input", "device", multi), ("single member, split stream", "split", single)):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(arm, gz, plain)
            torch.cuda.synchronize()
        ms, launches = {}, {}
        for ev in prof.key_averages():
            for k in kernels:
                if "::" + k + "_kernel" in ev.key or ev.key.startswith(k + "_kernel"):
                    ms[k] = ms.get(k, 0.0) + ev.device_time_total / 1000.0
                    launches[k] = launches.get(k, 0) + ev.count
        if not ms:
            raise RuntimeError("the profiler saw no inflate kernel launch")
        mib = len(plain) / 2**20
        print(json.dumps({"what": "inflate kernels' device time on the %s (torch.profiler, CUDA activity)" % name,
                          "card_and_power_limit": card, "ms_per_MiB_plain": {k: v / mib for k, v in ms.items()},
                          "ms_per_MiB_plain_total": sum(ms.values()) / mib, "launches": launches}))


def _bgzf(plain, level=6):
    """plain as BGZF members of 65 280 plain bytes (BC extra field), compressed on 16 threads, and the EOF block."""
    import struct
    from concurrent.futures import ThreadPoolExecutor

    def member(piece):
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        data = c.compress(piece) + c.flush()
        return (b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\x00BC\x02\x00" + struct.pack("<H", 25 + len(data)) + data
                + struct.pack("<II", zlib.crc32(piece), len(piece)))
    with ThreadPoolExecutor(16) as ex:
        parts = list(ex.map(member, [plain[i:i + 65280] for i in range(0, len(plain), 65280)]))
    return b"".join(parts) + bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def _bam_of_fastq(data, rec_len):
    """The unaligned BAM stream (header and records, flag 4) of fixed-size FASTQ records "@name\nSEQ\n+\nQUAL\n"."""
    import struct

    fq = np.frombuffer(data, dtype=np.uint8).reshape(-1, rec_len)
    name_len = int(np.argmax(fq[0] == ord("\n"))) - 1
    read_len = (rec_len - name_len - 5) // 2
    n = fq.shape[0]
    lrn, half = name_len + 1, (read_len + 1) // 2
    body = 32 + lrn + half + read_len
    rec = np.zeros((n, 4 + body), dtype=np.uint8)
    rec[:, :36] = np.frombuffer(struct.pack("<iiiBBHHHiiii", body, -1, -1, lrn, 255, 4680, 0, 4, read_len, -1, -1, 0),
                                dtype=np.uint8)
    rec[:, 36:36 + name_len] = fq[:, 1:1 + name_len]
    code = np.full(256, 15, dtype=np.uint8)
    for i, ch in enumerate("=ACMGRSVTWYHKDBN"):
        code[ord(ch)] = i
    seq = code[fq[:, 2 + name_len:2 + name_len + read_len]]
    if read_len & 1:
        seq = np.concatenate([seq, np.zeros((n, 1), dtype=np.uint8)], axis=1)
    rec[:, 36 + lrn:36 + lrn + half] = (seq[:, 0::2] << 4) | seq[:, 1::2]
    q0 = 2 + name_len + read_len + 3
    rec[:, 36 + lrn + half:] = fq[:, q0:q0 + read_len] - 33
    text = b"@HD\tVN:1.6\tSO:unsorted\n"
    return b"BAM\x01" + struct.pack("<i", len(text)) + text + struct.pack("<i", 0) + rec.tobytes()


def measure_bam_input(n, submit_mb):
    import io

    from cutadapt_b200.pipeline import read_gzip_device_chunks

    data, rec_len = build_fastq(n, pinned=False)
    plain = data.tobytes()
    forms = {"bam": _bgzf(_bam_of_fastq(plain, rec_len)), "bgzf_fastq": _bgzf(plain)}
    adapters = [PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1)]
    opts = dict(quality_cutoff=(0, 20), minimum_length=20)

    def run(arm, gz):
        t = FastqTrimmer(adapters, **opts, input_format="bam" if arm == "bam" else "fastq")
        t0 = time.perf_counter()
        out = sum(len(o) for o in t.process_chunks(read_gzip_device_chunks(io.BytesIO(gz), t, submit_mb << 20),
                                                   copy=False))
        return time.perf_counter() - t0, out, getattr(t, "bam_tiles", None)

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    warm = plain[:rec_len * 1000]
    warm_forms = {"bam": _bgzf(_bam_of_fastq(warm, rec_len)), "bgzf_fastq": _bgzf(warm)}
    for arm, gz in warm_forms.items():             # warm-up: buffers, module load
        run(arm, gz)
    res = {arm: {"wall_s": 0.0, "gz_bytes": len(gz)} for arm, gz in forms.items()}
    outs = set()
    for _ in range(3):
        for arm, gz in forms.items():
            w, out, tiles = run(arm, gz)
            res[arm]["wall_s"] += w
            outs.add(out)
            if tiles:
                res[arm]["tiles"], res[arm]["tiles_rewalked"] = tiles
    for x in res.values():
        x["M_reads_per_s"] = 3 * n / x["wall_s"] / 1e6
    assert len(outs) == 1, "the arms wrote different amounts"
    print(json.dumps({"what": "BGZF uBAM through the BAM path against the same reads as BGZF FASTQ (-a AGATCGGAAGAGC "
                      "-q 20 -m 20), host to host", "reads": n, "submission_MiB": submit_mb,
                      "gpu": torch.cuda.get_device_name(), "card_and_power_limit": card, "arms": res}))

    from torch.profiler import ProfilerActivity, profile

    kernels = ("bam_spec", "bam_resolve", "bam_count", "bam_starts", "bam_cut", "bam_emit")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run("bam", forms["bam"])
        torch.cuda.synchronize()
    ms, launches = {}, {}
    for ev in prof.key_averages():
        for k in kernels:
            if "::" + k + "_kernel" in ev.key or ev.key.startswith(k + "_kernel"):
                ms[k] = ms.get(k, 0.0) + ev.device_time_total / 1000.0
                launches[k] = launches.get(k, 0) + ev.count
    if not ms:
        raise RuntimeError("the profiler saw no BAM kernel launch")
    mib = len(_bam_of_fastq(plain, rec_len)) / 2**20
    print(json.dumps({"what": "BAM kernels' device time (torch.profiler, CUDA activity)", "card_and_power_limit": card,
                      "BAM_MiB": mib, "ms_total": ms, "ms_per_MiB_bam": {k: v / mib for k, v in ms.items()},
                      "ms_per_MiB_bam_total": sum(ms.values()) / mib, "launches": launches}))


def measure_rows(n, chunk_mb, baseline_tree=None):
    """--rows: the "paired" variant with info rows on both mates (--info-file + --info-file-paired), four arms
    alternating over three rounds in one process; then, with a baseline tree, its "paired" run without rows against
    this tree's, alternating processes."""
    n -= n % 2
    data, rec_len = build_fastq(n, pair_names=True)
    per_chunk = max(2, max(1, (chunk_mb << 20) // rec_len) // 2 * 2)
    mates = [np.ascontiguousarray(data.reshape(n // 2, 2, rec_len)[:, k]).reshape(-1) for k in (0, 1)]
    mates = [torch.from_numpy(m).pin_memory().numpy() for m in mates]
    half = per_chunk // 2
    chunks = [tuple(m[i * rec_len:min(n // 2, i + half) * rec_len] for m in mates) for i in range(0, n // 2, half)]
    adapters = [PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1, name="adapter")]
    opts = dict(quality_cutoff=(0, 20), minimum_length=20)
    info = dict(rows=("info",), rows2=("info",))
    arms = {"no_rows": PairedFastqTrimmer(adapters, adapters, opts, opts),
            "plain_rows": PairedFastqTrimmer(adapters, adapters, opts, opts, **info),
            "device_gzip_rows": PairedFastqTrimmer(adapters, adapters, opts, opts, **info, gzip_rows=("info",)),
            "host_zlib1_rows": PairedFastqTrimmer(adapters, adapters, opts, opts, **info)}

    def run(name, cs):
        t = arms[name]
        z = [zlib.compressobj(1, zlib.DEFLATED, 31) for _ in (0, 1)] if name == "host_zlib1_rows" else None
        downloaded = written = 0
        for parts in t.process_chunks_split(cs):
            for k, r in enumerate(t.last_rows.get("info", ())):
                downloaded += len(r)
                written += len(z[k].compress(r)) if z else len(r)
        if z:
            written += sum(len(x.flush()) for x in z)
        return downloaded, written

    for name in arms:
        run(name, chunks[:3])                     # warm-up: buffers, module load
    res = {name: {"wall_s": 0.0} for name in arms}
    for _ in range(3):
        for name in arms:
            t0 = time.perf_counter()
            downloaded, written = run(name, chunks)
            res[name]["wall_s"] += time.perf_counter() - t0
            res[name]["row_bytes_downloaded"], res[name]["row_bytes_written"] = downloaded, written
    for r in res.values():
        r["reads_per_s"] = 3 * n / r["wall_s"]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"what": "paired FASTQ (-a/-A AGATCGGAAGAGC -q 20 -m 20), host to host, info rows of both mates: "
                              "none, plain, device gzip, plain + host zlib level 1 (one thread per mate's stream)",
                      "reads": n, "chunk_mb": chunk_mb, "chunks": len(chunks), "gpu": torch.cuda.get_device_name(),
                      "card_and_power_limit": card, "arms": res}))
    if baseline_tree is None:
        return
    # a collect without requests: this tree against the baseline tree (library and Python), alternating processes
    runs = {"baseline": [], "this": []}
    for _ in range(3):
        for name, tree in (("baseline", baseline_tree), ("this", __file__.rsplit("/", 2)[0])):
            out = subprocess.run([sys.executable, f"{tree}/tools/measure_fastq.py", str(n), str(chunk_mb), "paired"],
                                 capture_output=True, text=True, check=True).stdout
            runs[name].append(json.loads(out.strip().split("\n")[-1])["reads_per_s"])
    print(json.dumps({"what": "paired variant without rows, this tree against the baseline tree, alternating processes",
                      "card_and_power_limit": card, "reads_per_s": runs,
                      "median": {k: sorted(v)[len(v) // 2] for k, v in runs.items()}}))


def measure_paired_revcomp(n, chunk_mb):
    """--revcomp: the "paired" variant without and with --revcomp (PairedReverseComplementer on the device), the two arms
    alternating over three rounds in one process; host-to-host pairs per second of each."""
    n -= n % 2
    data, rec_len = build_fastq(n, pair_names=True)
    per_chunk = max(2, max(1, (chunk_mb << 20) // rec_len) // 2 * 2)
    mates = [np.ascontiguousarray(data.reshape(n // 2, 2, rec_len)[:, k]).reshape(-1) for k in (0, 1)]
    mates = [torch.from_numpy(m).pin_memory().numpy() for m in mates]
    half = per_chunk // 2
    chunks = [tuple(m[i * rec_len:min(n // 2, i + half) * rec_len] for m in mates) for i in range(0, n // 2, half)]
    adapters = [PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1, name="adapter")]
    opts = dict(quality_cutoff=(0, 20), minimum_length=20)
    arms = {"paired": PairedFastqTrimmer(adapters, adapters, opts, opts),
            "paired_revcomp": PairedFastqTrimmer(adapters, adapters, opts, opts, revcomp=True)}

    def run(name, cs):
        return sum(len(a) + len(b) for parts in arms[name].process_chunks_split(cs) for a, b in parts.values())

    for name in arms:
        run(name, chunks[:3])                     # warm-up: buffers, module load
    res = {name: {"wall_s": 0.0} for name in arms}
    for _ in range(3):
        for name in arms:
            t0 = time.perf_counter()
            res[name]["out_bytes"] = run(name, chunks)
            res[name]["wall_s"] += time.perf_counter() - t0
    for name, r in res.items():
        r["pairs_per_s"] = 3 * (n // 2) / r["wall_s"]
        r["reverse_complemented"] = int(arms[name].statistics[0].get("reverse_complemented", 0))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"what": "paired FASTQ (-a/-A AGATCGGAAGAGC -q 20 -m 20), host to host, without and with --revcomp",
                      "pairs": n // 2, "chunk_mb": chunk_mb, "chunks": len(chunks), "gpu": torch.cuda.get_device_name(),
                      "card_and_power_limit": card, "arms": res,
                      "revcomp_over_plain_time": res["paired_revcomp"]["wall_s"] / res["paired"]["wall_s"]}))


def measure_names(n, chunk_mb, baseline_tree=None):
    """--names: the "fastq" variant without read names, with --rename '{id} {adapter_name} {comment}' and with
    -y ' {name}' --length-tag length=, the three arms alternating over three rounds in one process; then, with a
    baseline tree, its "fastq" run against this tree's (no names), alternating processes.  Both compile the run-time
    specialised first stage at once (CUTADAPT_B200_JIT=1): by default it is compiled (~1 s of NVRTC) once a set has seen
    4 Mi reads, which would fall inside one arm's timed round here and inside the single timed pass of a fresh process."""
    os.environ["CUTADAPT_B200_JIT"] = "1"
    data, rec_len = build_fastq(n)
    per_chunk = max(1, (chunk_mb << 20) // rec_len)
    chunks = [data[i * rec_len:min(n, i + per_chunk) * rec_len] for i in range(0, n, per_chunk)]
    adapters = [PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1, name="adapter")]
    opts = dict(quality_cutoff=(0, 20), minimum_length=20)
    arms = {"no_names": FastqTrimmer(adapters, **opts),
            "rename": FastqTrimmer(adapters, **opts, rename="{id} {adapter_name} {comment}"),
            "suffix_length_tag": FastqTrimmer(adapters, **opts, suffix=" {name}", length_tag="length=")}

    def run(name, cs):
        return sum(len(o) for o in arms[name].process_chunks(cs, copy=False))

    for name in arms:
        run(name, chunks[:3])                     # warm-up: buffers, module load
    res = {name: {"wall_s": 0.0, "round_s": []} for name in arms}
    for _ in range(3):
        for name in arms:
            t0 = time.perf_counter()
            res[name]["out_bytes"] = run(name, chunks)
            res[name]["round_s"].append(time.perf_counter() - t0)
            res[name]["wall_s"] += res[name]["round_s"][-1]
    for r in res.values():
        r["reads_per_s"] = 3 * n / r["wall_s"]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"what": "FASTQ (-a AGATCGGAAGAGC -q 20 -m 20), host to host: no read names, --rename "
                              "'{id} {adapter_name} {comment}', -y ' {name}' --length-tag length=",
                      "reads": n, "chunk_mb": chunk_mb, "chunks": len(chunks), "gpu": torch.cuda.get_device_name(),
                      "card_and_power_limit": card, "arms": res}))
    if baseline_tree is None:
        return
    runs = {"baseline": [], "this": []}
    for _ in range(3):
        for name, tree in (("baseline", baseline_tree), ("this", __file__.rsplit("/", 2)[0])):
            out = subprocess.run([sys.executable, f"{tree}/tools/measure_fastq.py", str(n), str(chunk_mb), "fastq"],
                                 capture_output=True, text=True, check=True).stdout
            runs[name].append(json.loads(out.strip().split("\n")[-1])["reads_per_s"])
    print(json.dumps({"what": "fastq variant without read names, this tree against the baseline tree, alternating "
                              "processes", "card_and_power_limit": card, "reads_per_s": runs,
                      "median": {k: sorted(v)[len(v) // 2] for k, v in runs.items()}}))


def main():
    if "--names" in sys.argv:
        argv = [a for a in sys.argv if a != "--names"]
        base = None
        if "--baseline-tree" in argv:
            i = argv.index("--baseline-tree")
            base = argv[i + 1]
            del argv[i:i + 2]
        return measure_names(int(argv[1]) if len(argv) > 1 else 4_000_000, int(argv[2]) if len(argv) > 2 else 64, base)
    if "--revcomp" in sys.argv:
        argv = [a for a in sys.argv if a != "--revcomp"]
        return measure_paired_revcomp(int(argv[1]) if len(argv) > 1 else 4_000_000,
                                      int(argv[2]) if len(argv) > 2 else 64)
    if "--rows" in sys.argv:
        argv = [a for a in sys.argv if a != "--rows"]
        base = None
        if "--baseline-tree" in argv:
            i = argv.index("--baseline-tree")
            base = argv[i + 1]
            del argv[i:i + 2]
        return measure_rows(int(argv[1]) if len(argv) > 1 else 4_000_000, int(argv[2]) if len(argv) > 2 else 64, base)
    if "--bam-input" in sys.argv:
        argv = [a for a in sys.argv if a != "--bam-input"]
        return measure_bam_input(int(argv[1]) if len(argv) > 1 else 4_000_000, int(argv[2]) if len(argv) > 2 else 64)
    if "--gzip-input" in sys.argv:
        argv = [a for a in sys.argv if a != "--gzip-input"]
        return measure_gzip_input(int(argv[1]) if len(argv) > 1 else 4_000_000, int(argv[2]) if len(argv) > 2 else 64)
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
