"""
Chunk runners: the reference's reader / worker / writer arrangement (``ReaderProcess``, ``WorkerProcess``,
``OrderedChunkWriter``, ``ParallelPipelineRunner``, runners.py:38-412) with one process per GPU.

The reference reads the input in chunks of whole records, hands chunk c to the next free worker and writes the
workers' outputs back in chunk order (runners.py:224-245); workers never talk to each other.  Here a worker is a
rank with a GPU:

* every rank reads the input itself and takes the chunks c with ``c % world == rank`` (round-robin as
  SURVEY.md section 8(e) asks; the chunker is deterministic, so all ranks agree on the chunk boundaries);
* it trims them with its ``FastqTrimmer`` (one library call per chunk, the upload of the next chunk overlapping
  the download of the previous one);
* the outputs go to rank 0 round by round (one round = ``world`` consecutive chunks) over a host-side gloo group
  -- they are host bytes already -- and rank 0 writes them in chunk order: byte for byte what a single GPU writes;
* the counters of all ranks are summed once at the end (``allreduce_fastq_statistics``), where the reference adds up
  the workers' Statistics objects (runners.py:372-373); a trimmer that collects statistics also has its statistics
  vector merged (``allreduce_fastq_statistics_vector``), returned as ``statistics_vector`` = (vector, max_len, kmax).

``SerialRunner`` is the one-GPU form (``SerialPipelineRunner``, runners.py:415-436).
"""
import io
from typing import BinaryIO, Callable, Iterable, Optional

from .pipeline import FastqTrimmer, allreduce_fastq_statistics, allreduce_fastq_statistics_vector, read_fastq_chunks


def _chunks_of(source, buffer_size: int) -> Iterable:
    """Chunks of whole records from a path, a binary file object or bytes."""
    if isinstance(source, (bytes, bytearray, memoryview)):
        return read_fastq_chunks(io.BytesIO(bytes(source)), buffer_size)
    if isinstance(source, str):
        f = open(source, "rb")

        def gen():
            with f:
                yield from read_fastq_chunks(f, buffer_size)

        return gen()
    return read_fastq_chunks(source, buffer_size)


class SerialRunner:
    """All chunks on one GPU, outputs written as they come (runners.py:415-436)."""

    def __init__(self, trimmer: FastqTrimmer, buffer_size: int = 4 * 1024 * 1024):
        self.trimmer = trimmer
        self.buffer_size = buffer_size

    def run(self, source, sink: BinaryIO) -> dict:
        n = 0
        for out in self.trimmer.process_chunks(_chunks_of(source, self.buffer_size), copy=False):
            sink.write(memoryview(out))
            n += 1
        stats = dict(self.trimmer.statistics)
        stats["chunks"] = n
        if getattr(self.trimmer, "collect_statistics", False):
            stats["statistics_vector"] = self.trimmer.statistics_vector()
        return stats


class RoundRobinRunner:
    """
    One of ``world`` ranks (torch.distributed must be initialised; ``group`` is used for the statistics, a gloo
    group created here for the host-side output merge).  ``process_chunk`` maps a chunk to its output bytes --
    by default ``FastqTrimmer.process_chunk`` of the given trimmer; the CPU tests pass their own.
    """

    def __init__(self, trimmer: Optional[FastqTrimmer] = None, buffer_size: int = 4 * 1024 * 1024, group=None,
                 process_chunk: Optional[Callable[[bytes], bytes]] = None):
        import torch.distributed as dist

        if not dist.is_initialized():
            raise RuntimeError("RoundRobinRunner needs an initialised torch.distributed process group")
        self.trimmer = trimmer
        self.buffer_size = buffer_size
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        # the outputs are host bytes: merge them over a gloo group, whatever backend carries the statistics
        self._host_group = group if dist.get_backend(group) == "gloo" else dist.new_group(backend="gloo")
        self._process = process_chunk or (lambda chunk: trimmer.process_chunk(chunk))

    def run(self, source, sink: Optional[BinaryIO]) -> dict:
        """Trims this rank's chunks; rank 0 writes every chunk's output to ``sink`` in input order.  Returns the
        counters of the whole run (on every rank)."""
        import numpy as np
        import torch
        import torch.distributed as dist

        mine = []                      # outputs of this rank's chunks of the current round (0 or 1)
        n_chunks = 0

        def flush_round(first_chunk: int, in_round: int):
            # lengths first, then the payloads padded to the longest; rank 0 writes them in chunk order
            length = torch.tensor([len(mine[0]) if mine else -1], dtype=torch.int64)
            lengths = [torch.zeros(1, dtype=torch.int64) for _ in range(self.world)]
            dist.all_gather(lengths, length, group=self._host_group)
            longest = max(1, max(int(t.item()) for t in lengths))
            payload = torch.zeros(longest, dtype=torch.uint8)
            if mine:
                payload[: len(mine[0])] = torch.frombuffer(bytearray(mine[0]), dtype=torch.uint8) if len(mine[0]) else payload[:0]
            gathered = [torch.zeros(longest, dtype=torch.uint8) for _ in range(self.world)] if self.rank == 0 else None
            dist.gather(payload, gathered, dst=0, group=self._host_group)
            if self.rank == 0 and sink is not None:
                for r in range(in_round):            # chunk first_chunk + r was trimmed by rank r
                    n = int(lengths[r].item())
                    if n > 0:
                        sink.write(gathered[r][:n].numpy().tobytes())
            mine.clear()

        round_start = 0
        for c, chunk in enumerate(_chunks_of(source, self.buffer_size)):
            if c % self.world == 0 and c > 0:
                flush_round(round_start, self.world)
                round_start = c
            if c % self.world == self.rank:
                mine.append(self._process(bytes(chunk) if not isinstance(chunk, (bytes, bytearray)) else chunk))
            n_chunks = c + 1
        if n_chunks > round_start:
            flush_round(round_start, n_chunks - round_start)
        local = dict(self.trimmer.statistics) if self.trimmer is not None else {}
        total = allreduce_fastq_statistics(local, self._host_group)
        total["chunks"] = n_chunks
        if getattr(self.trimmer, "collect_statistics", False):
            vector, max_len, kmax = self.trimmer.statistics_vector()
            total["statistics_vector"] = allreduce_fastq_statistics_vector(
                vector, self.trimmer.statistics_adapters, max_len, kmax, self._host_group)
        return total
