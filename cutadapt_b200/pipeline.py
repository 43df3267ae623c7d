"""
Batched per-chunk dispatch: what replaces the per-read loop of the reference's worker.

In the reference every chunk of ~4 MB FASTQ is processed read by read
(``WorkerProcess.run -> Pipeline.process_reads``, runners.py:174-214, pipeline.py:47-73) and for
each read ``QualityTrimmer.__call__`` (modifiers.py:853-858) and
``AdapterCutter.match_and_trim`` (modifiers.py:225-231) call into the native code.  Here one
chunk is one fused kernel launch:

``BatchTrimmer``   host-side chunks (lists of str or packed uint8 arrays): pack -> C ABI
                   (H2D, fused kernel, D2H pipelined in the library) -> kept intervals, match
                   records, optional reference-style Match objects and AdapterStatistics.
``DeviceBatch``    the same on torch CUDA tensors that are already resident in HBM (this is what
                   bench.py times for the roofline number and what multi-GPU runs use).
``allreduce_statistics``  the end-of-run merge of the trim statistics across GPUs: the fixed-layout
                   int64 vector is summed with one all-reduce (NCCL over NVLink for CUDA tensors,
                   gloo in the CPU tests).  It stands where the reference merges per-worker
                   ``Statistics`` objects in the parent (runners.py:372-373, report.py:81-126).

Reads shard across ranks by contiguous ranges (``shard_range``); no read ever needs another rank.
"""
import ctypes as C
import re
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .adapters import LinkedAdapter, Matchable, MultipleAdapters


# ---- statistics vector layout (include/cutadapt_b200.h: cg_stats_accumulate_device) ----------

STAT_N_READS, STAT_TOTAL_BP, STAT_WITH_ADAPTERS, STAT_QUALITY_TRIMMED_BP, STAT_ADAPTER_BP = 0, 1, 2, 3, 4
STAT_REVERSE_COMPLEMENTED, STAT_N_WRITTEN, STAT_BP_WRITTEN, STAT_FILTERED = 5, 6, 7, 8
FILTER_NAMES = ("too_short", "too_long", "too_many_n", "too_many_expected_errors", "casava_filtered", "discard_trimmed",
                "discard_untrimmed", "too_high_average_error_rate")     # slots STAT_FILTERED .. STAT_FILTERED + 7
_SCALARS, _ADJ = 16, 8


def stats_layout(n_adapters: int, max_len: int, kmax: int) -> dict:
    """Where the parts of the statistics vector are (cg_types.h: cg_stats_*)."""
    end = _ADJ + (max_len + 1) * (kmax + 1)
    adapters = _SCALARS + max_len + 1
    return {
        "size": adapters + 2 * n_adapters * end,
        "lengths": _SCALARS,                 # read-length histogram: max_len + 1 entries
        "adapters": adapters,                # per adapter, per end (0: 5' side, 1: 3' side): adjacent[8] + hist
        "end_size": end,
        "hist_shape": (max_len + 1, kmax + 1),
    }


def end_block(stats, layout: dict, adapter: int, end: int):
    """(adjacent[5], hist[max_len + 1, kmax + 1]) of one end of one adapter: views into the vector."""
    off = layout["adapters"] + (2 * adapter + end) * layout["end_size"]
    return stats[off:off + 5], stats[off + _ADJ:off + layout["end_size"]].reshape(layout["hist_shape"])


def adapter_statistics_from_vector(stats, adapters, max_len: int, kmax: int):
    """
    The reference-style AdapterStatistics objects of every adapter of ``adapters`` (a Matchable), rebuilt from the
    (all-reduced) statistics vector: what the reference gets by adding up the workers' Statistics objects
    (adapters.py:96-111, report.py:81-126).  Removed lengths above ``max_len`` and error counts above ``kmax``
    were clamped when counting.
    """
    from .adapters import LinkedAdapter, SingleAdapter

    stats = np.asarray(stats)
    singles, _, owners = adapters._flatten()
    number = {id(s): i for i, s in enumerate(singles)}
    lay = stats_layout(len(singles), max_len, kmax)
    out = []
    seen = set()
    for owner in owners:
        if id(owner) in seen:
            continue
        seen.add(id(owner))
        members = [owner] if isinstance(owner, (SingleAdapter, LinkedAdapter)) else list(owner._index._adapters)
        for adapter in members:
            st = adapter.create_statistics()
            if isinstance(adapter, LinkedAdapter):
                parts = ((st.front, adapter.front_adapter, 0), (st.back, adapter.back_adapter, 1))
            else:
                parts = ((st.front, adapter, 0), (st.back, adapter, 1))
            for end_stats, single, end in parts:
                if end_stats is None:
                    continue
                adjacent, hist = end_block(stats, lay, number[id(single)], end)
                end_stats.add_counts(hist, adjacent if end == 1 else None)
            out.append(st)
    return out


# ---- statistics of the FASTQ path (include/cutadapt_b200.h: cg_fastq_stats_read) ----------------------------------

def fastq_stats_layout(n_adapters: int, max_len: int, kmax: int) -> dict:
    """``stats_layout`` plus the tail of the FASTQ path's vector: reverse_complemented per adapter, then the poly-A
    histogram (max_len + 1 entries)."""
    lay = stats_layout(n_adapters, max_len, kmax)
    lay["reverse_complemented"] = lay["size"]
    lay["poly_a"] = lay["size"] + n_adapters
    lay["size"] = lay["poly_a"] + max_len + 1
    return lay


def relayout_statistics(stats, n_adapters: int, max_len: int, kmax: int, new_max_len: int, new_kmax: int,
                        tail: bool = True) -> np.ndarray:
    """The statistics vector laid out at a larger (new_max_len, new_kmax): every count keeps its (length, errors)
    cell, the new cells are 0.  ``tail``: the vector of the FASTQ path (fastq_stats_layout), else stats_layout."""
    if new_max_len < max_len or new_kmax < kmax:
        raise ValueError("relayout_statistics only grows the layout")
    stats = np.asarray(stats)
    layout = fastq_stats_layout if tail else stats_layout
    old, new = layout(n_adapters, max_len, kmax), layout(n_adapters, new_max_len, new_kmax)
    if stats.size != old["size"]:
        raise ValueError(f"the vector has {stats.size} entries, the layout {old['size']}")
    out = np.zeros(new["size"], dtype=stats.dtype)
    out[:_SCALARS + max_len + 1] = stats[:_SCALARS + max_len + 1]
    for block in range(2 * n_adapters):
        src = old["adapters"] + block * old["end_size"]
        dst = new["adapters"] + block * new["end_size"]
        out[dst:dst + _ADJ] = stats[src:src + _ADJ]
        hist = stats[src + _ADJ:src + old["end_size"]].reshape(old["hist_shape"])
        out[dst + _ADJ:dst + new["end_size"]].reshape(new["hist_shape"])[:max_len + 1, :kmax + 1] = hist
    if tail:
        out[new["reverse_complemented"]:new["reverse_complemented"] + n_adapters] = \
            stats[old["reverse_complemented"]:old["reverse_complemented"] + n_adapters]
        out[new["poly_a"]:new["poly_a"] + max_len + 1] = stats[old["poly_a"]:old["poly_a"] + max_len + 1]
    return out


def _histogram(counts) -> dict:
    return {int(i): int(counts[i]) for i in np.nonzero(np.asarray(counts))[0]}


def fastq_adapter_statistics(stats, adapters, max_len: int, kmax: int):
    """AdapterStatistics of every adapter from a vector of the FASTQ path, ``reverse_complemented`` filled in from
    its tail (a linked adapter's count is on its front or back part, whichever its match starts with)."""
    from .adapters import LinkedAdapter

    stats = np.asarray(stats)
    singles = adapters._flatten()[0]
    number = {id(s): i for i, s in enumerate(singles)}
    rc = stats[fastq_stats_layout(len(singles), max_len, kmax)["reverse_complemented"]:][:len(singles)]
    out = adapter_statistics_from_vector(stats, adapters, max_len, kmax)
    for st in out:
        a = st.adapter
        parts = (a.front_adapter, a.back_adapter) if isinstance(a, LinkedAdapter) else (a,)
        st.reverse_complemented = int(sum(rc[number[id(p)]] for p in parts))
    return out


def pair_adapter_statistics_from_vector(stats, adapters: Sequence, max_len: int, kmax: int):
    """One mate's AdapterStatistics under --pair-adapters (PairedAdapterCutter.adapter_statistics[i],
    modifiers.py:437-442): adapter i of the list is block i of the vector."""
    stats = np.asarray(stats)
    lay = stats_layout(len(adapters), max_len, kmax)
    out = []
    for i, adapter in enumerate(adapters):
        st = adapter.create_statistics()
        for end_stats, end in ((st.front, 0), (st.back, 1)):
            if end_stats is not None:
                adjacent, hist = end_block(stats, lay, i, end)
                end_stats.add_counts(hist, adjacent if end == 1 else None)
        out.append(st)
    return out


def poly_a_trimmed_lengths(stats, n_adapters: int, max_len: int, kmax: int) -> dict:
    """{bases removed: reads} of PolyATrimmer (its trimmed_bases, modifiers.py:861-879), from a FASTQ-path vector."""
    off = fastq_stats_layout(n_adapters, max_len, kmax)["poly_a"]
    return _histogram(np.asarray(stats)[off:off + max_len + 1])


def written_lengths(stats, max_len: int) -> dict:
    """{length: records} of the written records (ReadLengthStatistics, statistics.py:5-48)."""
    return _histogram(np.asarray(stats)[_SCALARS:_SCALARS + max_len + 1])


def allreduce_fastq_statistics_vector(stats, n_adapters: int, max_len: int, kmax: int, group=None, device=None):
    """Merge the FASTQ-path statistics vectors of all ranks: one MAX all-reduce of (max_len, kmax), every rank lays
    its vector out at the result, then one SUM all-reduce.  Returns (vector, max_len, kmax)."""
    import torch
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        shape = torch.tensor([max_len, kmax], dtype=torch.int64, device=device)
        dist.all_reduce(shape, op=dist.ReduceOp.MAX, group=group)
        new_len, new_kmax = (int(x) for x in shape.tolist())
    else:
        new_len, new_kmax = max_len, kmax
    t = torch.from_numpy(relayout_statistics(stats, n_adapters, max_len, kmax, new_len, new_kmax)).to(device)
    allreduce_statistics(t, group)
    return t.cpu().numpy(), new_len, new_kmax


def shard_range(n_items: int, rank: int, world_size: int) -> Tuple[int, int]:
    """Contiguous, near-equal split of ``n_items`` reads over ``world_size`` ranks."""
    base, extra = divmod(n_items, world_size)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def allreduce_statistics(stats, group=None):
    """
    Sum the statistics vector over all ranks in place (torch tensor on any device).
    One small all-reduce per run: latency-bound, nothing to fuse it with.
    """
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(stats, op=dist.ReduceOp.SUM, group=group)
    return stats


FASTQ_COUNTERS = ("n_records", "n_written", "bp_in", "bp_out", "out_bytes", "with_adapters", "quality_trimmed_bp",
                  "too_short", "too_long", "too_many_n", "too_many_expected_errors", "discarded", "casava_filtered",
                  "reverse_complemented", "too_high_average_error_rate")


def allreduce_fastq_statistics(statistics: dict, group=None, device=None) -> dict:
    """
    Sum the counters of ``FastqTrimmer.statistics`` (``cg_fastq_result``) over all ranks: every rank trims its own
    FASTQ chunks, the totals of the run are one small all-reduce at the end -- where the reference adds the
    per-worker ``Statistics`` in the parent (runners.py:372-373, report.py:81-126).  Returns a new dict.
    """
    import torch

    t = torch.tensor([int(statistics.get(k, 0)) for k in FASTQ_COUNTERS], dtype=torch.int64, device=device)
    allreduce_statistics(t, group)
    return dict(zip(FASTQ_COUNTERS, (int(x) for x in t.tolist())))


def kept_intervals(matches: np.ndarray, qtrim: Optional[np.ndarray], lengths: np.ndarray) -> np.ndarray:
    """
    (n, 2) array of the part of every read that survives quality trimming and all rounds of
    adapter removal, relative to the original read -- i.e. the composition of
    ``read[start:stop]`` (modifiers.py:858) and ``match.trimmed(read)`` (adapters.py:453-454,
    486-487, 1132-1137) for each round.
    """
    n = matches.shape[0]
    if qtrim is not None:
        start = qtrim[:, 0].astype(np.int64)
        stop = qtrim[:, 1].astype(np.int64)
    else:
        start = np.zeros(n, dtype=np.int64)
        stop = lengths.astype(np.int64).copy()
    for r in range(matches.shape[1]):
        for s in range(matches.shape[2]):
            rec = matches[:, r, s]
            present = rec["adapter"] >= 0
            after = ((rec["info"] >> 8) & 1).astype(bool)
            # read[:rstart] / read[rstop:] with Python's slice clamping (an index match on a read shorter than
            # the matched key reports rstop > len or rstart < 0, adapters.py:1342-1365)
            cur = stop - start
            rs = rec["rstart"].astype(np.int64)
            new_stop = start + np.where(rs >= 0, np.minimum(rs, cur), np.maximum(cur + rs, 0))
            new_start = start + np.minimum(rec["rstop"].astype(np.int64), cur)
            stop = np.where(present & after, new_stop, stop)
            start = np.where(present & ~after, new_start, start)
    return np.stack([start, stop], axis=1)


def action_intervals(matches: np.ndarray, qtrim: Optional[np.ndarray], lengths: np.ndarray,
                     action: Optional[str] = "trim") -> Tuple[np.ndarray, np.ndarray]:
    """
    What ``AdapterCutter`` writes for each read under its ``action`` (modifiers.py:214-251), from the match
    records: ``(out, keep)``, two (n, 2) arrays relative to the original read.  The output is
    ``read[out[i, 0]:out[i, 1]]``; under "mask" the characters outside ``keep`` become ``N``, under "lowercase"
    the read is upper-cased inside ``keep`` and lower-cased outside (``apply_action`` does that).
    The same rules as ``fq_evaluate_kernel``.
    """
    n = matches.shape[0]
    kept = kept_intervals(matches, qtrim, lengths)
    if action == "trim":
        return kept, kept.copy()
    if qtrim is not None:
        base = qtrim.astype(np.int64)
    else:
        base = np.stack([np.zeros(n, dtype=np.int64), lengths.astype(np.int64)], axis=1)
    matched = (matches["adapter"] >= 0).any(axis=(1, 2))
    out, keep = base.copy(), base.copy()
    if action in ("mask", "lowercase"):
        keep[matched] = kept[matched]
    elif action in ("retain", "crop"):
        if matches.shape[1] != 1:
            raise ValueError("'retain' and 'crop' cannot be combined with times > 1")       # modifiers.py:117-118
        m0 = matches[:, 0, 0]
        has0 = m0["adapter"] >= 0
        if matches.shape[2] > 1:
            m1 = matches[:, 0, 1]
            has1 = m1["adapter"] >= 0
        else:
            m1, has1 = m0, np.zeros(n, dtype=bool)
        length = base[:, 1] - base[:, 0]
        if action == "crop":                                  # read[m.rstart:m.rstop]
            a = np.where(has0, m0["rstart"], m1["rstart"]).astype(np.int64)
            b = np.where(has0, m0["rstop"], m1["rstop"]).astype(np.int64)
        else:                                                 # retained_adapter_interval, adapters.py:446-447, 479-480, 1145-1155
            after0 = has0 & (((m0["info"] >> 8) & 1) == 1)
            a = np.where(after0, 0, np.where(has0, m0["rstart"], 0)).astype(np.int64)
            offset = np.where(has0, m0["rstop"], 0).astype(np.int64)
            b = np.where(after0, m0["rstop"], np.where(has1, m1["rstop"] + offset, length)).astype(np.int64)
        a = np.clip(a, 0, length)
        b = np.maximum(np.clip(b, 0, length), a)
        cut = np.stack([base[:, 0] + a, base[:, 0] + b], axis=1)
        out[matched] = cut[matched]
        keep[matched] = cut[matched]
    elif action not in (None, "none"):
        raise ValueError(f"unknown action {action!r}")
    return out, keep


def apply_action(sequence: str, out, keep, action: Optional[str] = "trim") -> str:
    """The sequence ``AdapterCutter`` returns for one read, given its rows of ``action_intervals``."""
    o0, o1, k0, k1 = int(out[0]), int(out[1]), int(keep[0]), int(keep[1])
    if action == "mask":
        sequence = "N" * k0 + sequence[k0:k1] + "N" * (len(sequence) - k1)
    elif action == "lowercase":
        sequence = sequence[:k0].lower() + sequence[k0:k1].upper() + sequence[k1:].lower()
    return sequence[o0:o1]


def info_file_rows(names: Sequence[str], sequences: Sequence[str], qualities: Optional[Sequence[str]],
                   matches: np.ndarray, adapters: Matchable, final_reads=None) -> List[str]:
    """
    The lines ``--info-file`` gets for a chunk (InfoFileWriter.__call__, steps.py:232-253;
    SingleMatch.get_info_records, adapters.py:395-417; LinkedMatch.get_info_records, adapters.py:1157-1171),
    built from the match records: per match ``name, errors, rstart, rstop, before, match, after, adapter name,
    three quality parts, rc flag``; the parts of a linked match carry the linked adapter's name + ";1" / ";2";
    reads without a match give ``name, -1, sequence, qualities`` of the read as written.  ``sequences`` /
    ``qualities`` are the ORIGINAL reads (``info.original_read``): the reference applies the coordinates of every
    round to them as they are.  ``final_reads``: optional (sequence, qualities) per read for the unmatched rows
    (default: the originals).
    """
    singles, groups, owners = adapters._flatten()
    rows = []
    for i, name in enumerate(names):
        cur_s = sequences[i]
        cur_q = qualities[i] if qualities is not None else None
        any_match = False
        for r in range(matches.shape[1]):
            if not (matches["adapter"][i, r] >= 0).any():
                break
            any_match = True
            for slot in range(matches.shape[2]):
                m = matches[i, r, slot]
                if m["adapter"] < 0:
                    continue
                g = int(m["info"]) & 255
                if groups[g][0] == _lib.CG_GROUP_LINKED:
                    adapter_name = ("none" if owners[g].name is None else owners[g].name) + (";1", ";2")[slot]
                else:
                    adapter_name = singles[int(m["adapter"])].name
                rs, re_ = int(m["rstart"]), int(m["rstop"])
                q3 = [cur_q[0:rs], cur_q[rs:re_], cur_q[re_:]] if cur_q else ["", "", ""]
                rows.append("\t".join([name, str(int(m["errors"])), str(rs), str(re_), cur_s[0:rs], cur_s[rs:re_],
                                       cur_s[re_:], adapter_name] + q3 + [""]))
                # current_read = match.trimmed(current_read)
                if (int(m["info"]) >> 8) & 1:
                    cur_s, cur_q = cur_s[:rs], (cur_q[:rs] if cur_q is not None else None)
                else:
                    cur_s, cur_q = cur_s[re_:], (cur_q[re_:] if cur_q is not None else None)
        if not any_match:
            fs, fq = final_reads[i] if final_reads is not None else (sequences[i], qualities[i] if qualities else "")
            rows.append("\t".join([name, "-1", fs, fq or ""]))
    return rows


def _last_matches(sequences, matches):
    """Per read: (record of info.matches[-1] or None, the sequence that round searched)."""
    for i, seq in enumerate(sequences):
        cur, last = seq, None
        for r in range(matches.shape[1]):
            present = [m for m in matches[i, r] if m["adapter"] >= 0]
            if not present:
                break
            for m in present:
                last = (m, cur)
                cur = cur[:int(m["rstart"])] if (int(m["info"]) >> 8) & 1 else cur[int(m["rstop"]):]
        yield last


def rest_file_rows(names: Sequence[str], sequences: Sequence[str], matches: np.ndarray) -> List[str]:
    """The lines of ``--rest-file`` (RestFileWriter, steps.py:193-206; SingleMatch.rest, adapters.py:430-437,
    463-470): for the last match of a read, what lies before a 5' adapter / behind a 3' adapter, if not empty."""
    rows = []
    for name, last in zip(names, _last_matches(sequences, matches)):
        if last is None:
            continue
        m, cur = last
        rest = cur[int(m["rstop"]):] if (int(m["info"]) >> 8) & 1 else cur[:int(m["rstart"])]
        if rest:
            rows.append(f"{rest} {name}")
    return rows


def wildcard_file_rows(names: Sequence[str], sequences: Sequence[str], matches: np.ndarray,
                       adapters: Matchable) -> List[str]:
    """The lines of ``--wildcard-file`` (WildcardFileWriter, steps.py:209-220; SingleMatch.wildcards,
    adapters.py:378-393): the read characters under the ``N`` positions of the adapter of the last match."""
    singles, _, _ = adapters._flatten()
    rows = []
    for name, last in zip(names, _last_matches(sequences, matches)):
        if last is None:
            continue
        m, cur = last
        aseq = singles[int(m["adapter"])].sequence
        astart, rstart = int(m["astart"]), int(m["rstart"])
        chars = [cur[rstart + i] for i in range(int(m["astop"]) - astart)
                 if aseq[astart + i] == "N" and rstart + i < len(cur)]
        rows.append(f"{''.join(chars)} {name}")
    return rows


_COMPLEMENT = bytes.maketrans(b"ACGTUMRWSYKVHDBNacgtumrwsykvhdbn", b"TGCAAKYWSRMBDHVNtgcaakywsrmbdhvn")


def reverse_complement(sequence: str) -> str:
    """``SequenceRecord.reverse_complement`` of dnaio for the sequence: IUPAC-aware, case preserved, every other
    character unchanged (qualities are simply reversed)."""
    return sequence.encode("latin-1").translate(_COMPLEMENT)[::-1].decode("latin-1")


def revcomp_select(matches_forward: np.ndarray, matches_reverse: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """
    ``ReverseComplementer.__call__`` (modifiers.py:278-308) on match records: a read is replaced by its reverse
    complement iff the scores of its matches there add up to MORE than those of the forward read (a LinkedMatch
    counts with the sum of its parts, adapters.py:1113-1118).  Returns (is_rc[n] bool, the chosen records).
    """
    def total(m):
        return np.where(m["adapter"] >= 0, m["score"], 0).astype(np.int64).sum(axis=(1, 2))

    is_rc = total(matches_reverse) > total(matches_forward)
    chosen = np.where(is_rc[:, None, None], matches_reverse, matches_forward)
    return is_rc, chosen


def pair_adapters_select(per_adapter1: Sequence[np.ndarray], per_adapter2: Sequence[np.ndarray]):
    """
    ``PairedAdapterCutter._find_best_match_pair`` (modifiers.py:480-503) on match records: ``per_adapter1[i]`` /
    ``per_adapter2[i]`` are the records (n, 1, slots) of adapter pair i matched ALONE against R1 / R2.  A pair of
    reads is trimmed only by an adapter pair that matches both mates; among those the highest score sum wins, then
    the fewest errors, then the first listed.  Returns (pair index per read or -1, records for R1, records for R2).
    """
    k = len(per_adapter1)
    if k == 0 or k != len(per_adapter2):
        raise ValueError("The number of adapters to trim from R1 and R2 must be the same and not zero")
    n = per_adapter1[0].shape[0]
    best = np.full(n, -1, dtype=np.int64)
    best_score = np.zeros(n, dtype=np.int64)
    best_errors = np.zeros(n, dtype=np.int64)
    for i in range(k):
        m1, m2 = per_adapter1[i], per_adapter2[i]
        p1, p2 = m1["adapter"] >= 0, m2["adapter"] >= 0
        both = p1.any(axis=(1, 2)) & p2.any(axis=(1, 2))
        score = (np.where(p1, m1["score"], 0).sum(axis=(1, 2)) + np.where(p2, m2["score"], 0).sum(axis=(1, 2))).astype(np.int64)
        errors = (np.where(p1, m1["errors"], 0).sum(axis=(1, 2)) + np.where(p2, m2["errors"], 0).sum(axis=(1, 2))).astype(np.int64)
        better = both & ((best < 0) | (score > best_score) | ((score == best_score) & (errors < best_errors)))
        best = np.where(better, i, best)
        best_score = np.where(better, score, best_score)
        best_errors = np.where(better, errors, best_errors)
    out1 = per_adapter1[0].copy()
    out2 = per_adapter2[0].copy()
    out1["adapter"] = -1
    out2["adapter"] = -1
    for i in range(k):
        sel = best == i
        out1[sel] = per_adapter1[i][sel]
        out2[sel] = per_adapter2[i][sel]
    return best, out1, out2


class PairedAdapterBatch:
    """
    ``--pair-adapters`` for whole chunks (PairedAdapterCutter, modifiers.py:410-478): adapter i of the first list is
    only accepted together with adapter i of the second.  Every adapter runs as its own pass over its mate
    (2 k passes), ``pair_adapters_select`` combines the records.  ``process(seqs1, seqs2)`` returns
    (pair index per read pair, TrimResult for R1, TrimResult for R2); the adapter numbers in the records are the
    positions in the lists.
    """

    def __init__(self, adapters1: Sequence, adapters2: Sequence, ctx: Optional[_lib.Context] = None):
        if len(adapters1) != len(adapters2) or not adapters1:
            raise ValueError("The number of adapters to trim from R1 and R2 must be the same and not zero")
        self._trimmers1 = [BatchTrimmer([a], ctx=ctx) for a in adapters1]
        self._trimmers2 = [BatchTrimmer([a], ctx=ctx) for a in adapters2]

    def process(self, sequences1: Sequence[str], sequences2: Sequence[str]):
        s1, o1 = _lib.pack_strings(sequences1)
        s2, o2 = _lib.pack_strings(sequences2)
        m1 = [t.adapter_set.process(s1, o1, None, t.params)[0] for t in self._trimmers1]
        m2 = [t.adapter_set.process(s2, o2, None, t.params)[0] for t in self._trimmers2]
        for i, (a, b) in enumerate(zip(m1, m2)):        # adapter numbers = positions in the lists
            a["adapter"] = np.where(a["adapter"] >= 0, i, -1)
            b["adapter"] = np.where(b["adapter"] >= 0, i, -1)
        best, r1, r2 = pair_adapters_select(m1, m2)
        return (best, TrimResult(r1, None, kept_intervals(r1, None, np.diff(o1))),
                TrimResult(r2, None, kept_intervals(r2, None, np.diff(o2))))


def paired_revcomp_select(m11: Optional[np.ndarray], m22: Optional[np.ndarray], m12: Optional[np.ndarray],
                          m21: Optional[np.ndarray]):
    """
    ``PairedReverseComplementer.__call__`` (modifiers.py:334-400) on match records.  ``m11`` / ``m22``: the -a adapters
    on R1, the -A adapters on R2 (the pair as it came); ``m12`` / ``m21``: the -a adapters on R2, the -A adapters on R1
    (the pair with its mates swapped, "equivalent to reverse complementing").  None = that mate has no adapters.  A
    pair is swapped iff the scores of the swapped search add up to MORE.  Returns (swapped[n] bool, records of the new
    R1, records of the new R2); for a swapped pair the new R1 is the OLD R2 and vice versa.
    """
    def total(m):
        return 0 if m is None else np.where(m["adapter"] >= 0, m["score"], 0).astype(np.int64).sum(axis=(1, 2))

    swapped = np.asarray(total(m12) + total(m21) > total(m11) + total(m22))
    pick = lambda a, b: None if a is None else np.where(swapped[:, None, None], b, a)     # noqa: E731
    return swapped, pick(m11, m12), pick(m22, m21)


class PairedRevcompBatch:
    """
    ``--revcomp`` on pairs (PairedReverseComplementer, modifiers.py:311-400): four batched passes -- every mate against
    both adapter lists -- and ``paired_revcomp_select``.  ``process(seqs1, seqs2)`` returns (swapped[n], TrimResult of
    the new R1, TrimResult of the new R2); the caller writes old R2 as new R1 for a swapped pair and appends the
    name suffix.  (The FASTQ kernels do both forms, ``FastqTrimmer(revcomp=True)`` and
    ``PairedFastqTrimmer(revcomp=True)``; this is the record-level composition for callers that work with records.)
    """

    def __init__(self, adapters1: Optional[Sequence], adapters2: Optional[Sequence], ctx: Optional[_lib.Context] = None):
        self._t1 = BatchTrimmer(adapters1, ctx=ctx) if adapters1 else None
        self._t2 = BatchTrimmer(adapters2, ctx=ctx) if adapters2 else None
        if self._t1 is None and self._t2 is None:
            raise ValueError("no adapters given")

    def process(self, sequences1: Sequence[str], sequences2: Sequence[str]):
        s1, o1 = _lib.pack_strings(sequences1)
        s2, o2 = _lib.pack_strings(sequences2)
        run = lambda t, s, o: None if t is None else t.adapter_set.process(s, o, None, t.params)[0]   # noqa: E731
        m11, m22 = run(self._t1, s1, o1), run(self._t2, s2, o2)
        m12, m21 = run(self._t1, s2, o2), run(self._t2, s1, o1)
        swapped, r1, r2 = paired_revcomp_select(m11, m22, m12, m21)
        len1 = np.where(swapped, np.diff(o2), np.diff(o1))
        len2 = np.where(swapped, np.diff(o1), np.diff(o2))

        def result(records, lengths):
            if records is None:
                return None
            return TrimResult(records, None, kept_intervals(records, None, lengths))
        return swapped, result(r1, len1), result(r2, len2)


class TrimResult:
    """Outcome of one chunk: raw records plus the derived kept interval of every read."""

    def __init__(self, matches, qtrim, intervals):
        self.matches = matches      # structured array [n, times, slots], dtype MATCH_DTYPE
        self.qtrim = qtrim          # [n, 2] int32 or None
        self.intervals = intervals  # [n, 2] int64: read[start:stop] is what remains

    @property
    def with_adapters(self) -> int:
        return int((self.matches["adapter"] >= 0).any(axis=(1, 2)).sum())


class BatchTrimmer:
    """
    Quality trimming + adapter removal for whole chunks of reads.

    adapters          a Matchable (e.g. MultipleAdapters) or a list of adapters
    times             as AdapterCutter(times=...)          (modifiers.py:98-119)
    quality_cutoff    None or (cutoff_front, cutoff_back)  as QualityTrimmer (modifiers.py:840-851)
    nextseq_cutoff    None or the cutoff of NextseqQualityTrimmer (modifiers.py:825-837), applied first
    """

    def __init__(self, adapters, times: int = 1, quality_cutoff: Optional[Tuple[int, int]] = None,
                 quality_base: int = 33, ctx: Optional[_lib.Context] = None, nextseq_cutoff: Optional[int] = None):
        self.adapters: Matchable = adapters if isinstance(adapters, Matchable) else MultipleAdapters(list(adapters))
        self.times = int(times)
        self.quality_cutoff = quality_cutoff
        self.nextseq_cutoff = nextseq_cutoff
        self.quality_base = quality_base
        self._ctx = ctx
        self.params = _lib.make_params(
            quality_trim=quality_cutoff is not None,
            cutoff_front=quality_cutoff[0] if quality_cutoff else 0,
            cutoff_back=quality_cutoff[1] if quality_cutoff else 0,
            quality_base=quality_base,
            times=times,
            nextseq_cutoff=nextseq_cutoff,
        )

    @property
    def adapter_set(self) -> _lib.AdapterSet:
        return self.adapters.adapter_set()

    def process_packed(self, seq: np.ndarray, offsets: np.ndarray, qual: Optional[np.ndarray] = None) -> TrimResult:
        matches, qtrim = self.adapter_set.process(seq, offsets, qual, self.params)
        lengths = np.diff(offsets)
        return TrimResult(matches, qtrim, kept_intervals(matches, qtrim, lengths))

    def process(self, sequences: Sequence[str], qualities: Optional[Sequence[str]] = None) -> TrimResult:
        seq, offsets = _lib.pack_strings(sequences)
        qual = None
        if self.quality_cutoff is not None or self.nextseq_cutoff is not None:
            if qualities is None or any(q is None for q in qualities):
                from .qualtrim import HasNoQualities

                raise HasNoQualities("Cannot do quality trimming when no qualities are available")
            qual, _ = _lib.pack_strings(qualities, "Quality data")
        return self.process_packed(seq, offsets, qual)

    def process_revcomp(self, sequences: Sequence[str], qualities: Optional[Sequence[str]] = None):
        """
        ``--revcomp``: every read and its reverse complement go through the same pass (two batches); the better
        orientation wins (``revcomp_select``).  Returns (TrimResult of the chosen orientation, is_rc[n]); intervals
        and records of reads with ``is_rc`` refer to ``reverse_complement(read)`` and its reversed qualities.
        As in the reference, quality trimming has to happen before (ReverseComplementer wraps only the AdapterCutter).
        """
        if self.quality_cutoff is not None or self.nextseq_cutoff is not None:
            raise ValueError("process_revcomp searches adapters only; quality-trim the reads first")
        forward = self.process(sequences)
        reverse = self.process([reverse_complement(s) for s in sequences])
        is_rc, chosen = revcomp_select(forward.matches, reverse.matches)
        lengths = np.array([len(s) for s in sequences], dtype=np.int64)
        return TrimResult(chosen, None, kept_intervals(chosen, None, lengths)), is_rc

    def match_objects(self, result: TrimResult, sequences: Sequence[str]) -> List[List]:
        """Per read, the list of reference-style Match objects of its rounds (info.matches)."""
        self.adapter_set  # make sure the bookkeeping for matches_from_records exists
        out = []
        qt = result.qtrim
        for i, seq in enumerate(sequences):
            cur = seq if qt is None else seq[qt[i, 0]:qt[i, 1]]
            found = []
            for r in range(result.matches.shape[1]):
                m = self.adapters.matches_from_records(result.matches[i, r], cur)
                if m is None:
                    break
                found.append(m)
                cur = m.trimmed(cur)
            out.append(found)
        return out

    def adapter_statistics(self, result: TrimResult, sequences: Sequence[str]):
        """AdapterStatistics per adapter, filled like AdapterCutter.__call__ does (modifiers.py:200-207)."""
        _, _, owners = self.adapters._device_set if self.adapters._device_set else (None, None, None)
        self.adapter_set
        _, _, owners = self.adapters._device_set
        stats = {id(o): o.create_statistics() for o in owners}
        for matches in self.match_objects(result, sequences):
            for m in matches:
                stats[id(m.adapter)].add_match(m)
        return [stats[id(o)] for o in owners]


def _fastq_head(buf, end: int, lines: int = 4) -> int:
    """Length of the longest prefix of buf[:end] that consists of complete 4-line records (the buffer starts at a
    record; same counting rule as dnaio's chunk reader, which the reference uses at runners.py:116-126).  lines=8:
    complete pairs of interleaved records."""
    linebreaks = buf.count(b"\n", 0, end)
    right = end
    for _ in range(linebreaks % lines + 1):
        right = buf.rfind(b"\n", 0, right)
        if right < 0:
            return 0
    return right + 1


def _cut_records(buf, end: int, n_records: int) -> int:
    """Offset just behind the first n_records records of buf[:end]."""
    pos = 0
    for _ in range(4 * n_records):
        pos = buf.find(b"\n", pos, end) + 1
    return pos


def read_fastq_chunks(f, buffer_size: int = 4 * 1024 * 1024):
    """
    Chunks of complete FASTQ records from a binary file object -- what ``dnaio.read_chunks`` hands the reference's
    workers (runners.py:116-126) and what ``FastqTrimmer.process_chunk(s)`` takes.  The last chunk may lack the
    final newline.  A record larger than the buffer makes the buffer grow.
    """
    return _read_chunks(f, buffer_size, _fastq_head)


def _read_chunks(f, buffer_size: int, head_of):
    """Chunks of buf[:head_of(buf, end)] from a binary file object; the buffer grows when it holds no complete chunk,
    whatever is left at the end of the file is the last chunk."""
    buf = bytearray(buffer_size)
    start = 0
    while True:
        if start == len(buf):
            buf.extend(bytes(len(buf)))
        n = f.readinto(memoryview(buf)[start:])
        if not n:
            break
        end = start + n
        head = head_of(buf, end)
        if head:
            yield bytes(buf[:head])
            buf[0:end - head] = buf[head:end]
            start = end - head
        else:
            start = end
    if start:
        yield bytes(buf[:start])


def read_interleaved_fastq_chunks(f, buffer_size: int = 4 * 1024 * 1024):
    """
    Chunks of whole pairs of an interleaved FASTQ file (R1 and R2 of each pair one after the other, ``--interleaved``):
    every chunk ends after a multiple of 8 lines, for ``PairedFastqTrimmer``'s chunk methods with ``chunk2=None``.  A
    record larger than the buffer makes the buffer grow.  An odd number of records at the end of the file stays in the
    last chunk, which the device then rejects ("Interleaved input file incomplete").
    """
    return _read_chunks(f, buffer_size, lambda buf, end: _fastq_head(buf, end, 8))


def read_paired_fastq_chunks(f1, f2, buffer_size: int = 4 * 1024 * 1024):
    """Pairs of chunks with the same number of complete records each (``dnaio.read_paired_chunks``)."""
    return _read_paired_chunks(f1, f2, buffer_size, lambda buf, end: buf.count(b"\n", 0, _fastq_head(buf, end)) // 4,
                               _cut_records)


def _read_paired_chunks(f1, f2, buffer_size: int, count, cut):
    """Pairs of chunks with the same number of complete records each: count(buf, end) is the number of complete
    records in buf[:end], cut(buf, end, n) the offset just behind the first n of them.  Whatever is left at the end of
    the files is the last pair."""
    bufs = [bytearray(buffer_size), bytearray(buffer_size)]
    starts = [0, 0]
    files = (f1, f2)
    eof = [False, False]
    while True:
        ends = list(starts)
        for k in (0, 1):
            if starts[k] == len(bufs[k]):
                bufs[k].extend(bytes(len(bufs[k])))
            n = 0 if eof[k] else files[k].readinto(memoryview(bufs[k])[starts[k]:])
            eof[k] = eof[k] or not n
            ends[k] = starts[k] + (n or 0)
        if eof[0] and eof[1]:
            break
        records = min(count(bufs[k], ends[k]) for k in (0, 1))
        if records:
            cuts = [cut(bufs[k], ends[k], records) for k in (0, 1)]
            yield bytes(bufs[0][:cuts[0]]), bytes(bufs[1][:cuts[1]])
            for k in (0, 1):
                bufs[k][0:ends[k] - cuts[k]] = bufs[k][cuts[k]:ends[k]]
                starts[k] = ends[k] - cuts[k]
        else:
            starts = ends
    if starts[0] or starts[1]:
        yield bytes(bufs[0][:starts[0]]), bytes(bufs[1][:starts[1]])


def _fasta_head(buf, end: int) -> int:
    """Length of the longest prefix of buf[:end] that ends in front of a header line (a line starting with '>'),
    not counting a header at offset 0: the complete records of a FASTA buffer (plus any leading '#' lines)."""
    return buf.rfind(b"\n>", 0, end) + 1


def _fasta_headers(buf, end: int) -> int:
    """Number of header lines that start in buf[:end]."""
    return (1 if end and buf[:1] == b">" else 0) + buf.count(b"\n>", 0, end)


def _fasta_cut(buf, end: int, n_records: int) -> int:
    """Offset of header number n_records (0-based) of buf[:end]: just behind the first n_records records."""
    pos = 0 if buf[:1] == b">" else buf.find(b"\n>", 0, end) + 1
    for _ in range(n_records):
        pos = buf.find(b"\n>", pos, end) + 1
    return pos


def read_fasta_chunks(f, buffer_size: int = 4 * 1024 * 1024):
    """
    Chunks of complete FASTA records from a binary file object, for ``FastqTrimmer(input_format="fasta")``.  A chunk
    ends in front of a line that starts with '>'; the first chunk carries any '#' lines in front of the first record.
    A record larger than the buffer makes the buffer grow.
    """
    return _read_chunks(f, buffer_size, _fasta_head)


def _fasta_pairs_head(buf, end: int) -> int:
    """The longest prefix of complete FASTA records that holds an even number of them (0 without a complete pair)."""
    records = _fasta_headers(buf, _fasta_head(buf, end))
    return _fasta_cut(buf, end, records - records % 2) if records >= 2 else 0


def read_interleaved_fasta_chunks(f, buffer_size: int = 4 * 1024 * 1024):
    """Chunks of whole pairs of an interleaved FASTA file: every chunk ends in front of every second header (see
    read_interleaved_fastq_chunks)."""
    return _read_chunks(f, buffer_size, _fasta_pairs_head)


def read_paired_fasta_chunks(f1, f2, buffer_size: int = 4 * 1024 * 1024):
    """Pairs of FASTA chunks with the same number of complete records each (see read_fasta_chunks)."""
    return _read_paired_chunks(f1, f2, buffer_size, lambda buf, end: _fasta_headers(buf, _fasta_head(buf, end)),
                               _fasta_cut)


class DeviceChunk:
    """A chunk that a device gzip reader (read_gzip_device_chunks and its paired / interleaved twins) has already
    submitted: its plain bytes are in ``slot`` of the trimmer's context (``slot2``: mate 2 of an interleaved chunk).
    The trimmers' chunk methods take it in place of bytes; ``size`` / ``len()`` is its plain size."""

    def __init__(self, slot: int, size: int, slot2: int = -1):
        self.slot, self.size, self.slot2 = slot, size, slot2

    def __len__(self) -> int:
        return self.size


def _submit_chunk(ctx, chunk):
    """(slot, chunk) for the trimmers' collects: bytes or a uint8 array are uploaded (``cg_fastq_submit``) and come back
    as the array, which has to stay alive until the collect; a DeviceChunk is in its slot already."""
    if isinstance(chunk, DeviceChunk):
        return chunk.slot, chunk
    buf = np.frombuffer(chunk, dtype=np.uint8) if not isinstance(chunk, np.ndarray) else chunk
    slot = C.c_int32(-1)
    _lib.check(_lib.lib().cg_fastq_submit(ctx.handle, buf.ctypes.data if buf.size else None, buf.size, C.byref(slot)))
    return slot.value, buf


def _one_in_flight(items, submit, collect):
    """collect(submit(item)) of every item in order, item i+1 submitted before item i is collected: its upload
    overlaps the work on item i."""
    pending = None
    for item in items:
        ticket = submit(item)
        if pending is not None:
            yield collect(pending)
        pending = ticket
    if pending is not None:
        yield collect(pending)


class _GzipInput:
    """One compressed input file on a context (cg_gzin_create): the bytes read but not yet consumed, and the carry."""

    def __init__(self, ctx, f, buffer_size: int, split_members: bool = False):
        h = C.c_int32(0)
        if split_members:
            _lib.check(_lib.lib().cg_gzin_create_ex(ctx.handle, _lib.CG_GZIN_SPLIT_MEMBERS, C.byref(h)))
        else:
            _lib.check(_lib.lib().cg_gzin_create(ctx.handle, C.byref(h)))
        self.ctx, self.handle, self.f = ctx, h.value, f
        self.buf, self.end, self.eof = bytearray(buffer_size), 0, False

    def fill(self):
        """Read more of the file; the buffer doubles when it is full (nothing consumed from a whole buffer)."""
        if self.eof:
            return
        if self.end == len(self.buf):
            self.buf.extend(bytes(len(self.buf)))
        n = self.f.readinto(memoryview(self.buf)[self.end:])
        self.eof = not n
        self.end += n or 0

    def pointer(self):
        a = np.frombuffer(self.buf, dtype=np.uint8)
        return a.ctypes.data if self.end else None

    def consume(self, n: int):
        self.buf[0:self.end - n] = self.buf[n:self.end]
        self.end -= n

    @property
    def done(self) -> bool:
        return self.eof and self.end == 0

    def close(self):
        if self.handle:
            _lib.check(_lib.lib().cg_gzin_destroy(self.ctx.handle, self.handle))
            self.handle = 0


def _add_gzip_bytes(statistics: dict, n: int):
    statistics["in_bytes_gzip"] = statistics.get("in_bytes_gzip", 0) + n


def read_gzip_device_chunks(f, trimmer, buffer_size: int = 4 * 1024 * 1024, split_members: bool = False):
    """
    Chunks of a gzip file (a binary file object of the compressed bytes) inflated on the device
    (``cg_fastq_submit_gzip``): every member is inflated on the GPU and the plain bytes never cross PCIe.  Yields
    ``DeviceChunk`` objects for ``trimmer`` (a FastqTrimmer; its context and format decide how the chunks are cut: the
    records of read_fastq_chunks / read_fasta_chunks).  A trimmer with ``input_format="bam"`` reads unaligned BAM
    (``CG_FORMAT_BAM``): the records are decoded on the device into FASTQ chunks, and afterwards ``trimmer.bam_tiles``
    holds (tiles of the record-boundary walk, tiles walked again).  A chunk is submitted when the generator is advanced, so the
    trimmer's one chunk in flight stays as it is.  ``trimmer.statistics["in_bytes_gzip"]`` counts the compressed bytes
    consumed.  Meant for files of many members (BGZF, concatenated .gz files, this project's gzip outputs); a member
    that does not fit one submission makes the buffer grow.  ``split_members=True`` (``CG_GZIN_SPLIT_MEMBERS``) inflates
    a long member -- the one member of a file from ``gzip`` or ``pigz`` -- block-parallel instead, over as many
    submissions as it takes.
    """
    g = _GzipInput(trimmer.ctx, f, buffer_size, split_members)
    bam = getattr(trimmer, "input_format", None) == "bam"
    fmt = _lib.CG_FORMAT_BAM if bam else trimmer.params.format
    carry = 0
    try:
        # BAM: a last chunk that reaches the 2 GiB chunk limit leaves a carry behind, submitted again
        while not g.done or carry:
            g.fill()
            slot, res = C.c_int32(-1), _lib.cg_gzin_result()
            _lib.check(_lib.lib().cg_fastq_submit_gzip(trimmer.ctx.handle, g.handle, g.pointer(), g.end, fmt,
                                                       int(g.eof), C.byref(slot), C.byref(res)))
            _add_gzip_bytes(trimmer.statistics, res.consumed)
            g.consume(res.consumed)
            carry = res.carry_bytes if bam and g.done else 0
            if slot.value >= 0:
                yield DeviceChunk(slot.value, res.chunk_bytes)
        if bam:
            tiles, rewalked = C.c_int64(), C.c_int64()
            _lib.check(_lib.lib().cg_gzin_bam_tiles(trimmer.ctx.handle, g.handle, C.byref(tiles), C.byref(rewalked)))
            trimmer.bam_tiles = (tiles.value, rewalked.value)
    finally:
        g.close()


def read_gzip_device_interleaved_chunks(f, trimmer, buffer_size: int = 4 * 1024 * 1024, split_members: bool = False):
    """read_gzip_device_chunks for an interleaved file and a PairedFastqTrimmer: every chunk holds whole pairs (the
    cuts of read_interleaved_fastq_chunks / read_interleaved_fasta_chunks) and is split on the device as
    ``cg_fastq_submit_interleaved`` splits it.  Pass each chunk with ``chunk2=None``."""
    g = _GzipInput(trimmer.ctx, f, buffer_size, split_members)
    try:
        while not g.done:
            g.fill()
            s1, s2, res = C.c_int32(-1), C.c_int32(-1), _lib.cg_gzin_result()
            _lib.check(_lib.lib().cg_fastq_submit_gzip_interleaved(
                trimmer.ctx.handle, g.handle, g.pointer(), g.end, trimmer.params1.format, int(g.eof), C.byref(s1),
                C.byref(s2), C.byref(res)))
            _add_gzip_bytes(trimmer.statistics[0], res.consumed)
            g.consume(res.consumed)
            if s1.value >= 0:
                yield DeviceChunk(s1.value, res.chunk_bytes, s2.value)
    finally:
        g.close()


def read_gzip_device_paired_chunks(f1, f2, trimmer, buffer_size: int = 4 * 1024 * 1024, split_members=False):
    """read_gzip_device_chunks for the two files of a pair and a PairedFastqTrimmer: yields (chunk1, chunk2) with the
    same number of records (read_paired_fastq_chunks / read_paired_fasta_chunks).  split_members: a bool for both
    files, or a pair of them."""
    sp1, sp2 = split_members if isinstance(split_members, (tuple, list)) else (split_members, split_members)
    g1, g2 = _GzipInput(trimmer.ctx, f1, buffer_size, sp1), _GzipInput(trimmer.ctx, f2, buffer_size, sp2)
    try:
        while not (g1.done and g2.done):
            g1.fill()
            g2.fill()
            s1, s2, r1, r2 = C.c_int32(-1), C.c_int32(-1), _lib.cg_gzin_result(), _lib.cg_gzin_result()
            _lib.check(_lib.lib().cg_fastq_submit_gzip_paired(
                trimmer.ctx.handle, g1.handle, g2.handle, g1.pointer(), g1.end, g2.pointer(), g2.end,
                trimmer.params1.format, int(g1.eof and g2.eof), C.byref(s1), C.byref(s2), C.byref(r1), C.byref(r2)))
            for st, g, r in ((trimmer.statistics[0], g1, r1), (trimmer.statistics[1], g2, r2)):
                _add_gzip_bytes(st, r.consumed)
                g.consume(r.consumed)
            if s1.value >= 0:
                yield DeviceChunk(s1.value, r1.chunk_bytes), DeviceChunk(s2.value, r2.chunk_bytes)
    finally:
        g1.close()
        g2.close()


_FORMATS = {("fastq", None): _lib.CG_FORMAT_FASTQ, ("fastq", "fastq"): _lib.CG_FORMAT_FASTQ,
            ("fasta", None): _lib.CG_FORMAT_FASTA, ("fasta", "fasta"): _lib.CG_FORMAT_FASTA,
            ("fastq", "fasta"): _lib.CG_FORMAT_FASTQ_TO_FASTA,
            # BAM arrives as FASTQ chunks (read_gzip_device_chunks), so the collects see FASTQ
            ("bam", None): _lib.CG_FORMAT_FASTQ, ("bam", "fastq"): _lib.CG_FORMAT_FASTQ,
            ("bam", "fasta"): _lib.CG_FORMAT_FASTQ_TO_FASTA}


def _format_code(input_format: str, output_format: Optional[str]) -> int:
    """cg_fastq_params.format of (input format, output format or None for the input's)."""
    if (input_format, output_format) not in _FORMATS:
        raise ValueError(f"unsupported formats: {input_format!r} in, {output_format!r} out "
                         "(input 'fastq', 'fasta' or 'bam'; output None, 'fasta', or 'fastq' for FASTQ or BAM input)")
    return _FORMATS[(input_format, output_format)]


def _output_capacity(n_bytes: int, fmt: int, gzip: bool = False, n_dest: int = 4, rc_suffixes: bool = False) -> int:
    """Output bytes a chunk of n_bytes can need: trimming only shortens a record ("\\r\\n" -> "\\n" and "+name" -> "+"
    too), except for the newline a chunk without a final one gets and, in FASTA, the empty line of a record without
    sequence (">a\\n" -> ">a\\n\\n", at most 1.5 x).  rc_suffixes: FASTA output that may append " rc" to every
    record, at most 3 x (">\\n" -> "> rc\\n\\n").  gzip outputs: a member adds at most 23 bytes to its 65 280, and
    each of the n_dest outputs can end in a short member."""
    if rc_suffixes and fmt != _lib.CG_FORMAT_FASTQ:
        plain = 3 * n_bytes + 16
    else:
        plain = (n_bytes + n_bytes // 2 if fmt == _lib.CG_FORMAT_FASTA else n_bytes) + 16
    return plain + (_lib.GZ_OVERHEAD * (plain // _lib.GZ_MEMBER + n_dest) if gzip else 0)


def _fastq_params(times=1, quality_cutoff=None, quality_base=33, nextseq_cutoff=None, minimum_length=0,
                  maximum_length=None, max_n=None, max_expected_errors=None, discard_trimmed=False,
                  discard_untrimmed=False, cut=(), poly_a=False, length=None, trim_n=False,
                  discard_casava=False, action="trim", revcomp=False, rc_suffix=True, input_format="fastq",
                  output_format=None, max_average_error_rate=None, zero_cap=False) -> "_lib.cg_fastq_params":
    fp = _lib.cg_fastq_params()
    fp.format = _format_code(input_format, output_format)
    fp.trim = _lib.make_params(
        quality_trim=quality_cutoff is not None,
        cutoff_front=quality_cutoff[0] if quality_cutoff else 0,
        cutoff_back=quality_cutoff[1] if quality_cutoff else 0,
        quality_base=quality_base, times=times, nextseq_cutoff=nextseq_cutoff)
    fp.minimum_length = int(minimum_length or 0)
    fp.maximum_length = -1 if maximum_length is None else int(maximum_length)
    fp.max_n = -1.0 if max_n is None else float(max_n)
    fp.max_expected_errors = -1.0 if max_expected_errors is None else float(max_expected_errors)
    fp.discard_trimmed = int(bool(discard_trimmed))
    fp.discard_untrimmed = int(bool(discard_untrimmed))
    # -u N removes N bases from the 5' end, -u -N from the 3' end; several values add up per end
    fp.cut_front = sum(int(c) for c in cut if c > 0)
    fp.cut_back = sum(-int(c) for c in cut if c < 0)
    fp.poly_a = int(bool(poly_a))
    fp.shorten = int(length is not None)
    fp.shorten_length = int(length or 0)
    fp.trim_n = int(bool(trim_n))
    fp.discard_casava = int(bool(discard_casava))
    actions = {"trim": 0, None: 1, "none": 1, "mask": 2, "lowercase": 3, "retain": 4, "crop": 5}
    if action not in actions:
        raise ValueError(f"unknown action {action!r}")
    if action in ("retain", "crop") and times > 1:
        raise ValueError("'retain' and 'crop' cannot be combined with times > 1")     # modifiers.py:117-118
    fp.action = actions[action]
    fp.revcomp = 0 if not revcomp else (1 if rc_suffix else 2)
    if max_average_error_rate is not None:
        rate = float(max_average_error_rate)
        if not 0.0 < rate < 1.0:                                                         # predicates.py:81-85
            raise ValueError(f"max_error_rate must be between 0.0 and 1.0, got {rate}.")
        fp.max_average_error_rate = rate
    fp.zero_cap = int(bool(zero_cap))
    return fp


REDIRECT_OUTPUTS = ("too_short", "too_long", "untrimmed")     # destinations 1, 2, 3 of cg_fastq_collect_split


# the outputs cg_fastq_collect_paired_interleaved can interleave, and their bits
INTERLEAVE_BITS = {"output": _lib.CG_INTERLEAVE_MAIN, "too_short": _lib.CG_REDIRECT_TOO_SHORT,
                   "too_long": _lib.CG_REDIRECT_TOO_LONG, "untrimmed": _lib.CG_REDIRECT_UNTRIMMED}


def _gzip_bits(names) -> int:
    """cg_fastq_params.gzip_outputs of output names out of ("output",) + REDIRECT_OUTPUTS."""
    bits = 0
    for name in names or ():
        if name not in INTERLEAVE_BITS:
            raise ValueError(f"unknown output {name!r} to compress (one of {', '.join(INTERLEAVE_BITS)})")
        bits |= _lib.CG_GZIP_MAIN if name == "output" else INTERLEAVE_BITS[name]
    return bits


def _redirect_bits(redirect, redirect_formats, params) -> Tuple[int, int]:
    """(redirect, fasta_outputs) bits of cg_fastq_collect_split from output names and {name: "fasta" / "fastq"} (default:
    the main output's format).  FASTA input can only be written as FASTA."""
    redirect = tuple(redirect or ())
    formats = dict(redirect_formats or {})
    for name in list(redirect) + list(formats):
        if name not in REDIRECT_OUTPUTS:
            raise ValueError(f"unknown filter output {name!r} (one of {', '.join(REDIRECT_OUTPUTS)})")
    main = "fastq" if params.format == _lib.CG_FORMAT_FASTQ else "fasta"
    bits = fasta = 0
    for i, name in enumerate(REDIRECT_OUTPUTS):
        fmt = formats.get(name, main)
        if fmt not in ("fastq", "fasta"):
            raise ValueError(f"format of the {name} output must be 'fastq' or 'fasta', not {fmt!r}")
        if name in redirect:
            if fmt == "fastq" and params.format == _lib.CG_FORMAT_FASTA:
                raise ValueError(f"FASTA input cannot be written as FASTQ (the {name} output)")
            bits |= 1 << i
        if fmt == "fasta":
            fasta |= 1 << i
    if bits & _lib.CG_REDIRECT_UNTRIMMED and params.discard_trimmed:
        raise ValueError("the untrimmed output cannot be combined with discard_trimmed")
    return bits, fasta


def _device_set(adapters, ctx):
    if adapters is not None and not isinstance(adapters, Matchable):
        adapters = MultipleAdapters(list(adapters)) if len(adapters) else None
    if adapters is None:
        return None, None
    singles, groups, _ = adapters._flatten()
    spec = _lib.AdapterSetSpec([s.descriptor() for s in singles], groups, adapters._flatten_indexes())
    return adapters, _lib.AdapterSet(spec, ctx)


def _demux_names(adapters):
    """(names of the outputs, destination number of every adapter): the name of the adapter of a read's most
    recent match selects its output (Demultiplexer, steps.py:397-409); a LinkedAdapter's parts share its name."""
    if adapters is None:
        raise ValueError("demultiplexing needs adapters")
    singles, groups, owners = adapters._flatten()
    names = [s.name for s in singles]
    for (typ, a0, a1, _, _), owner in zip(groups, owners):
        if typ == _lib.CG_GROUP_LINKED:
            names[a0] = names[a1] = owner.name
    outputs = list(dict.fromkeys(names))
    number = {name: i for i, name in enumerate(outputs)}
    return outputs, np.array([number[n] for n in names], dtype=np.int32)


# the per-read text outputs (cg_fastq_request_rows): --info-file, --rest-file, --wildcard-file
ROW_KINDS = ("info", "rest", "wildcard")


def _row_kinds(rows, gzip_rows, what: str = "rows") -> Tuple[tuple, tuple]:
    """(kinds, compressed kinds) from names out of ROW_KINDS; a compressed kind must be requested."""
    rows = tuple(dict.fromkeys(rows or ()))
    gzip_rows = tuple(dict.fromkeys(gzip_rows or ()))
    for name in rows + gzip_rows:
        if name not in ROW_KINDS:
            raise ValueError(f"unknown row output {name!r} (one of {', '.join(ROW_KINDS)})")
    for name in gzip_rows:
        if name not in rows:
            raise ValueError(f"the {name} rows are to be compressed but are not in {what}")
    return rows, gzip_rows


def _text_blob(texts) -> Tuple[bytes, np.ndarray]:
    blobs = [t.encode("latin-1") for t in texts]
    offsets = np.zeros(len(blobs) + 1, dtype=np.int32)
    offsets[1:] = np.cumsum([len(b) for b in blobs])
    return b"".join(blobs), offsets


def _row_text(adapters, kind: str, pair_list: bool = False) -> Tuple[bytes, np.ndarray]:
    """(text, offsets) a kind of rows needs for the adapters of a mate: names as the info file shows them (the parts
    of a linked adapter are "name;1" / "name;2", LinkedMatch.get_info_records, adapters.py:1157-1171), nothing for
    rest rows, the sequences for wildcard rows.  pair_list: the -a or -A list of --pair-adapters, whose matches name
    the pair; no adapters: no entries."""
    if adapters is None:
        return b"", np.zeros(1, dtype=np.int32)
    if pair_list:
        singles = list(adapters)
        names = [a.name for a in singles]
    else:
        singles, groups, owners = adapters._flatten()
        names = [s.name for s in singles]
        for (typ, a0, a1, _, _), owner in zip(groups, owners):
            if typ == _lib.CG_GROUP_LINKED:
                base = "none" if owner.name is None else owner.name
                names[a0], names[a1] = base + ";1", base + ";2"
    if kind == "info":
        return _text_blob(names)
    if kind == "rest":
        return _text_blob([""] * len(singles))
    return _text_blob([s.sequence for s in singles])


def _request_rows(ctx, slot: int, kinds, texts: dict, gzip_rows) -> None:
    for kind in kinds:
        blob, offsets = texts[kind]
        _lib.check(_lib.lib().cg_fastq_request_rows(ctx.handle, slot, ROW_KINDS.index(kind), blob, offsets.ctypes.data,
                                                    offsets.size - 1, int(kind in gzip_rows)))


def _read_rows(ctx, slot: int, kinds) -> dict:
    """{kind: bytes} of the collect that took ``slot`` (cg_fastq_read_rows)."""
    rows = {}
    for kind in kinds:
        k, n, plain = ROW_KINDS.index(kind), C.c_int64(0), C.c_int64(0)
        _lib.check(_lib.lib().cg_fastq_read_rows(ctx.handle, slot, k, None, 0, C.byref(n), C.byref(plain)))
        buf = np.empty(n.value, dtype=np.uint8)
        if n.value:
            _lib.check(_lib.lib().cg_fastq_read_rows(ctx.handle, slot, k, buf.ctypes.data, buf.size, C.byref(n),
                                                     C.byref(plain)))
        rows[kind] = buf.tobytes()
    return rows


# ---- read names (cg_names_*): --length-tag, --strip-suffix, -x / -y, --rename ----
RENAME_VARIABLES = ("header", "id", "comment", "cut_prefix", "cut_suffix", "adapter_name", "rc", "match_sequence")
_NAME_KINDS = {v: i + 1 for i, v in enumerate(RENAME_VARIABLES)}
_NAME_KINDS["rn"] = 9
LENGTH_TAG_CHARACTERS = "_=:,;/-@#%!~"


def _tokenize_braces(text: str):
    """tokenize_braces of the reference: (is a variable, value) in order; a stray brace is an error."""
    for value in re.split(r"(\{[^}]*\})", text):
        if value == "":
            continue
        brace = value.startswith("{") and value.endswith("}")
        if brace:
            value = value[1:-1]
        for ch in "{}":
            if ch in value:
                raise ValueError(f"Unexpected '{ch}' encountered")
        yield brace, value


def rename_tokens(template: str, paired: bool = False) -> list:
    """The --rename template as (kind, mate, literal text) tokens for cg_names_create, with the reference's errors as
    ValueError (Renamer / PairedEndRenamer.__init__, modifiers.py:620-633, 706-711): the single-end template has "\\t"
    replaced by a tab before it is tokenized, the paired one after."""
    if not paired:
        template = template.replace(r"\t", "\t")
    try:
        tokens = list(_tokenize_braces(template))
    except ValueError as e:
        raise ValueError(f"Error in template '{template}': {e}") from None
    allowed = set(RENAME_VARIABLES)
    if paired:
        allowed = (allowed - {"rc"}) | {"rn"}
        for v in set(RENAME_VARIABLES) - {"id", "rc"}:
            allowed |= {"r1." + v, "r2." + v}
    for brace, value in tokens:
        if brace and value not in allowed:
            raise ValueError(f"Error in template: Variable '{value}' not recognized")
    out = []
    for brace, value in tokens:
        if not brace:
            out.append((0, 0, value.replace(r"\t", "\t") if paired else value))
        elif value[:3] in ("r1.", "r2."):
            out.append((_NAME_KINDS[value[3:]], int(value[1]), ""))
        else:
            out.append((_NAME_KINDS[value], 0, ""))
    return out


def check_length_tag(tag: str) -> None:
    """The length tags the device takes: literal text without regular-expression meaning."""
    if tag == "":
        raise ValueError("the length tag must not be empty")
    for ch in tag:
        if not (ch.isascii() and ch.isalnum()) and ch not in LENGTH_TAG_CHARACTERS:
            raise ValueError(f"length tag {tag!r}: the character {ch!r} has a meaning in the reference's regular "
                             f"expression; only letters, digits and {' '.join(LENGTH_TAG_CHARACTERS)} are accepted")


def _names_wanted(rename, prefix, suffix, strip_suffix, length_tag) -> bool:
    return rename is not None or bool(prefix) or bool(suffix) or bool(strip_suffix) or length_tag is not None


def _make_names(ctx, rename, prefix, suffix, strip_suffix, length_tag, paired: bool):
    """A names handle, or None when nothing changes a name.  An empty template is no --rename, and --rename '{header}'
    installs no renamer (cli.py:982-990 test the template for truth and for "{header}")."""
    rename = rename or None
    if rename is not None and (prefix or suffix):
        raise ValueError("Option --rename cannot be combined with --prefix (-x) or --suffix (-y)")
    if rename is not None:
        rename_tokens(rename, paired)           # the reference's template errors, "{header}" included
    if rename == "{header}":
        rename = None
    if not _names_wanted(rename, prefix, suffix, strip_suffix, length_tag):
        return None
    if length_tag is not None:
        check_length_tag(length_tag)
    tokens = rename_tokens(rename, paired) if rename is not None else None
    return _lib.Names(ctx, length_tag, tuple(strip_suffix or ()), prefix or "", suffix or "", tokens, paired)


def _name_table(adapters, pair_list: bool = False):
    """(adapter names by match-record index, linked flags): a linked adapter's parts carry its own name, as for
    demultiplexing; with --pair-adapters, pair i of the list."""
    if adapters is None:
        return [], []
    if pair_list:
        return [str(a.name) for a in adapters], [0] * len(adapters)
    singles, groups, owners = adapters._flatten()
    names = [str(s.name) for s in singles]
    linked = [0] * len(singles)
    for (typ, a0, a1, _, _), owner in zip(groups, owners):
        if typ == _lib.CG_GROUP_LINKED:
            names[a0] = names[a1] = str(owner.name)
            linked[a0] = linked[a1] = 1
    return names, linked


def _last_cuts(cut) -> Tuple[int, int]:
    """The last -u value of each end: the bases {cut_prefix} / {cut_suffix} show."""
    front = [int(c) for c in cut if c > 0]
    back = [-int(c) for c in cut if c < 0]
    return (front[-1] if front else 0), (back[-1] if back else 0)


def _keep_chunk(ctx, chunk):
    """The plain bytes of a chunk, read back from its slot when the device holds it: a collect with read names may
    have to run the chunk again with a larger output buffer."""
    if not isinstance(chunk, DeviceChunk):
        return chunk
    n = C.c_int64(0)
    buf = np.empty(chunk.size, dtype=np.uint8)
    _lib.check(_lib.lib().cg_fastq_slot_read(ctx.handle, chunk.slot, buf.ctypes.data if buf.size else None, buf.size,
                                             C.byref(n)))
    return buf[: n.value]


class FastqTrimmer:
    """
    FASTQ chunks in, trimmed FASTQ chunks out -- the per-chunk worker of the reference
    (``WorkerProcess.run``, runners.py:174-214: parse, modifiers, filters, format) as one library call
    per chunk (``cg_fastq_submit`` / ``cg_fastq_collect``): the chunk is indexed, trimmed, filtered and
    formatted on the device.

    adapters            a Matchable / list of adapters, or None / [] for quality trimming and filters only
    quality_cutoff      None or (cutoff_front, cutoff_back)        -q        (modifiers.py:840-858)
    nextseq_cutoff      None or the --nextseq-trim cutoff                    (modifiers.py:825-837)
    times               -n                                                   (modifiers.py:225-231)
    minimum_length, maximum_length   -m / -M                                 (predicates.py:29-53)
    max_n, max_expected_errors       --max-n / --max-ee                      (predicates.py:56-122)
    max_average_error_rate           --max-aer: expected errors per base     (predicates.py:74-95), counted in
                                     ``too_high_average_error_rate``
    zero_cap            -z: quality characters below quality_base are written as quality_base, last in the modifier
                        chain, so the quality filters see them capped (ZeroCapper, modifiers.py:806-822)
    discard_trimmed, discard_untrimmed                                       (predicates.py:127-160)
    cut                 -u values (UnconditionalCutter, modifiers.py:66-95), applied first
    poly_a, length, trim_n           --poly-a / --length / --trim-n, after the adapters (modifiers.py:861-918)
    discard_casava      --discard-casava                                     (predicates.py:125-139)
    action              --action: "trim" (default), "none"/None, "mask", "lowercase", "retain", "crop"
                        (AdapterCutter, modifiers.py:175-249)
    revcomp, rc_suffix  --revcomp: adapters are searched on the read and on its reverse complement and the better
                        orientation is written (" rc" appended to the name unless rc_suffix is False;
                        ReverseComplementer, modifiers.py:264-308), all on the device
    input_format        "fastq" (default), "fasta" (read_fasta_chunks; no quality options then) or "bam" (unaligned
                        BAM, single-end: chunks only from read_gzip_device_chunks, which decodes the records on the
                        device; bytes are refused)
    output_format       None (the input's format; FASTQ for BAM) or "fasta" (FASTQ or BAM in, FASTA out: a .fasta / .fa
                        output or --fasta)
    collect_statistics  also collect what the report needs beyond the counters (cg_fastq_stats_*): per-adapter
                        statistics, the poly-A and written-length histograms; ``statistics_vector()``,
                        ``adapter_statistics()``, ``poly_a_trimmed_lengths``, ``written_lengths``
    redirect            filter outputs: names out of REDIRECT_OUTPUTS ("too_short", "too_long", "untrimmed") --
                        --too-short-output / --too-long-output / --untrimmed-output.  The reads these filters remove
                        are written to their own output, trimmed like the main output (``process_chunk_split``);
                        "untrimmed" switches the untrimmed filter on and counts its reads in ``discarded``
    redirect_formats    {output name: "fastq" or "fasta"}; an output not named has the main output's format
    gzip_outputs        names out of ("output",) + REDIRECT_OUTPUTS written as gzip, compressed on the device: every
                        method then returns gzip members (65 280 plain bytes each, see cg_fastq_params.gzip_outputs;
                        "output" covers every demultiplexed output), which concatenate into one gzip file, and
                        ``statistics`` gains ``out_bytes_plain``, the uncompressed size
    rows                names out of ROW_KINDS ("info", "rest", "wildcard") -- --info-file / --rest-file /
                        --wildcard-file: every chunk method also formats these rows of the chunk's reads on the device
                        (every read, filtered or not, in input order; cg_fastq_request_rows) and leaves them in
                        ``last_rows`` = {kind: bytes} for the chunk it just returned or yielded
    gzip_rows           names out of ``rows`` whose rows are compressed on the device (gzip members as for
                        gzip_outputs)
    length_tag, strip_suffix, prefix, suffix, rename
                        --length-tag / --strip-suffix / -x / -y / --rename, last in the chain and on the device
                        (cg_names_*): every output and row gets the new names.  A length tag may hold letters, digits and
                        _ = : , ; / - @ # % ! ~ only; template and tag errors are ValueError, with the reference's
                        messages; --rename '{header}' renames nothing.  Pass rc_suffix=False with rename, as the
                        command line does

    ``process_chunk(bytes) -> bytes``; ``process_chunks(iterable)`` keeps one chunk in flight so that the
    upload of chunk i+1 overlaps the download of chunk i.  With ``redirect``: ``process_chunk_split(bytes) ->
    {"output": bytes, <redirected output>: bytes, ...}`` and ``process_chunks_split(iterable)``.  ``statistics``
    accumulates the counters of ``cg_fastq_result`` over all chunks.  Chunks must consist of complete records (what
    ``dnaio.read_chunks`` yields; read_fastq_chunks / read_fasta_chunks).
    """

    def __init__(self, adapters=None, times: int = 1, quality_cutoff: Optional[Tuple[int, int]] = None,
                 quality_base: int = 33, nextseq_cutoff: Optional[int] = None, minimum_length: int = 0,
                 maximum_length: Optional[int] = None, max_n: Optional[float] = None,
                 max_expected_errors: Optional[float] = None, discard_trimmed: bool = False,
                 discard_untrimmed: bool = False, cut: Sequence[int] = (), poly_a: bool = False,
                 length: Optional[int] = None, trim_n: bool = False, discard_casava: bool = False,
                 action: Optional[str] = "trim", revcomp: bool = False, rc_suffix: bool = True,
                 input_format: str = "fastq", output_format: Optional[str] = None,
                 ctx: Optional[_lib.Context] = None, collect_statistics: bool = False,
                 redirect: Sequence[str] = (), redirect_formats: Optional[dict] = None,
                 gzip_outputs: Sequence[str] = (), rows: Sequence[str] = (), gzip_rows: Sequence[str] = (),
                 max_average_error_rate: Optional[float] = None, zero_cap: bool = False,
                 rename: Optional[str] = None, prefix: str = "", suffix: str = "", strip_suffix: Sequence[str] = (),
                 length_tag: Optional[str] = None):
        self.rows, self.gzip_rows = _row_kinds(rows, gzip_rows)
        self.input_format = input_format
        self.params = _fastq_params(times, quality_cutoff, quality_base, nextseq_cutoff, minimum_length, maximum_length,
                                    max_n, max_expected_errors, discard_trimmed, discard_untrimmed, cut, poly_a, length,
                                    trim_n, discard_casava, action, revcomp, rc_suffix, input_format, output_format,
                                    max_average_error_rate, zero_cap)
        self.gzip_outputs = tuple(dict.fromkeys(gzip_outputs or ()))
        self.params.gzip_outputs = _gzip_bits(self.gzip_outputs)
        self.redirect = tuple(dict.fromkeys(redirect or ()))
        self._redirect, self._fasta_outputs = _redirect_bits(self.redirect, redirect_formats, self.params)
        self.ctx = ctx or _lib.default_context()
        self.adapters, self._set = _device_set(adapters, self.ctx)
        self._names = _make_names(self.ctx, rename, prefix, suffix, strip_suffix, length_tag, False)
        if self._names is not None:
            self._names.set_mate(0, *_name_table(self.adapters), *_last_cuts(cut))
            self.params.names = self._names.handle
        self._stats = None
        if collect_statistics:
            n = len(self.adapters._flatten()[0]) if self.adapters is not None else 0
            self._stats = _lib.FastqStatistics(self.ctx, n)
            self.params.stats = self._stats.handle
        self.statistics = {}
        self._out_bufs, self._out_keep = {}, {}
        self._row_texts = {}
        self._slot_rows = {}          # slot -> the kinds requested for the chunk in it
        self._rows_taken = {}
        self.last_rows = {}

    def _texts(self, kinds) -> dict:
        for kind in kinds:
            if kind not in self._row_texts:
                self._row_texts[kind] = _row_text(self.adapters, kind)
        return self._row_texts

    def _submit(self, chunk, rows: Optional[tuple] = None) -> Tuple[int, int, object]:
        """Upload a chunk and request its rows (``rows``: kinds, default the trimmer's)."""
        if self.input_format == "bam" and not isinstance(chunk, DeviceChunk):
            raise ValueError("a BAM trimmer takes the chunks of read_gzip_device_chunks, not bytes: BAM records are "
                             "decoded on the device")
        slot, buf = _submit_chunk(self.ctx, chunk)
        kinds = self.rows if rows is None else rows
        _request_rows(self.ctx, slot, kinds, self._texts(kinds), self.gzip_rows)
        self._slot_rows[slot] = kinds
        return slot, buf.size, buf

    def _take_rows(self, slot: int) -> None:
        """The rows of the collect that just took ``slot``: every kind requested for it, and the trimmer's kinds in
        last_rows."""
        self._rows_taken = _read_rows(self.ctx, slot, self._slot_rows.pop(slot, ()))
        self.last_rows = {kind: self._rows_taken[kind] for kind in self.rows}

    def _capacity(self, n_bytes: int, n_dest: int = 4, chunk=None) -> int:
        # a device chunk cannot be submitted again, so FASTA output with " rc" suffixes gets room for all of them
        rc = isinstance(chunk, DeviceChunk) and self.params.revcomp != 0
        return _output_capacity(n_bytes, self.params.format, self.params.gzip_outputs != 0, n_dest, rc)

    def _account(self, res) -> None:
        for k, v in res.as_dict(self.params.gzip_outputs != 0).items():
            self.statistics[k] = self.statistics.get(k, 0) + v

    def _out_buffer(self, slot: int, n_bytes: int) -> np.ndarray:
        """Per-slot output buffer, pinned when torch can provide it (the download then needs no bounce)."""
        buf = self._out_bufs.get(slot)
        if buf is None or buf.size < n_bytes:
            size = max(n_bytes + n_bytes // 4, 1 << 20)
            try:
                import torch

                self._out_keep[slot] = torch.empty(size, dtype=torch.uint8, pin_memory=True)
                buf = self._out_keep[slot].numpy()
            except Exception:
                buf = np.empty(size, dtype=np.uint8)
            self._out_bufs[slot] = buf
        return buf

    def _keep(self, chunk):
        """A device chunk as bytes when read names may make a collect run it again (see _again)."""
        return _keep_chunk(self.ctx, chunk) if self._names is not None else chunk

    def _again(self, rc: int, res, out, chunk, slot):
        """After a collect that failed because its output did not fit (" rc" suffixes in FASTA, longer read names;
        the call says how much it needs): the ticket of the chunk submitted again, else None."""
        grows = self._names is not None or self.params.format != _lib.CG_FORMAT_FASTQ
        if rc == 0 or not grows or res.out_bytes <= out.size or isinstance(chunk, DeviceChunk):
            return None
        kinds = self._slot_rows.pop(slot, None)
        if self.input_format == "bam":              # the slot held the decoded records as FASTQ text
            slot, buf = _submit_chunk(self.ctx, chunk)
            _request_rows(self.ctx, slot, kinds, self._texts(kinds), self.gzip_rows)
            self._slot_rows[slot] = kinds
            return slot, buf.size, buf
        return self._submit(chunk, kinds)

    def _collect(self, ticket, copy: bool = True):
        slot, n_bytes, chunk = ticket
        chunk = self._keep(chunk)
        out = self._out_buffer(slot, self._capacity(n_bytes, chunk=ticket[2]))
        while True:
            res = _lib.cg_fastq_result()
            rc = _lib.lib().cg_fastq_collect(
                self.ctx.handle, slot, self._set.handle if self._set is not None else None, C.byref(self.params),
                out.ctypes.data, out.size, C.byref(res))
            again = self._again(rc, res, out, chunk, slot)
            if again is not None:
                slot, _, chunk = again
                out = self._out_buffer(slot, res.out_bytes)
                continue
            _lib.check(rc)
            break
        self._account(res)
        self._take_rows(slot)
        return out[: res.out_bytes].tobytes() if copy else out[: res.out_bytes]

    def _no_redirect(self, what: str):
        if self._redirect:
            raise ValueError(f"filter outputs ({', '.join(self.redirect)}) cannot be combined with {what}; "
                             "use process_chunk_split / process_chunks_split")

    def process_chunk(self, chunk) -> bytes:
        self._no_redirect("process_chunk")
        return self._collect(self._submit(chunk))

    def _collect_split(self, ticket, copy: bool = True) -> dict:
        slot, n_bytes, chunk = ticket
        chunk = self._keep(chunk)
        out = self._out_buffer(slot, self._capacity(n_bytes, chunk=ticket[2]))
        segments = np.zeros(5, dtype=np.int64)
        while True:
            res = _lib.cg_fastq_result()
            rc = _lib.lib().cg_fastq_collect_split(
                self.ctx.handle, slot, self._set.handle if self._set is not None else None, C.byref(self.params),
                self._redirect, self._fasta_outputs, out.ctypes.data, out.size, C.byref(res), segments.ctypes.data)
            # " rc" suffixes and read names can exceed the bound; the call says how much it needs, run the chunk again
            again = self._again(rc, res, out, chunk, slot)
            if again is None and rc != 0 and res.out_bytes > out.size and not isinstance(chunk, DeviceChunk):
                again = self._submit(chunk, self._slot_rows.pop(slot, None))
            if again is not None:
                slot, _, chunk = again
                out = self._out_buffer(slot, res.out_bytes)
                continue
            _lib.check(rc)
            break
        self._account(res)
        self._take_rows(slot)
        names = ("output",) + REDIRECT_OUTPUTS
        part = (lambda a, b: out[a:b].tobytes()) if copy else (lambda a, b: out[a:b])
        return {name: part(segments[d], segments[d + 1]) for d, name in enumerate(names)
                if d == 0 or name in self.redirect}

    def process_chunk_split(self, chunk) -> dict:
        """{"output": main output, and for every name in ``redirect``: the reads that filter removed} for one chunk,
        every output in input order (``cg_fastq_collect_split``)."""
        return self._collect_split(self._submit(chunk))

    def process_chunks_split(self, chunks, copy: bool = True):
        """process_chunk_split over an iterable with one chunk in flight (see process_chunks)."""
        yield from _one_in_flight(chunks, self._submit, lambda ticket: self._collect_split(ticket, copy))

    def _demux_names(self):
        return _demux_names(self.adapters)

    def process_chunk_demux(self, chunk, unknown: str = "unknown") -> dict:
        """{adapter name: FASTQ bytes} + {unknown: reads without a match} -- what ``-o 'demux-{name}.fastq'`` writes
        for this chunk (every output in input order); ``cg_fastq_collect_demux``."""
        self._no_redirect("demultiplexing")
        outputs, dest = self._demux_names()
        slot, n_bytes, _ = self._submit(chunk)
        chunk = self._keep(chunk)
        out = self._out_buffer(slot, self._capacity(n_bytes, len(outputs) + 1))
        segments = np.zeros(len(outputs) + 2, dtype=np.int64)
        while True:
            res = _lib.cg_fastq_result()
            rc = _lib.lib().cg_fastq_collect_demux(
                self.ctx.handle, slot, self._set.handle, C.byref(self.params), dest.ctypes.data, len(outputs),
                out.ctypes.data, out.size, C.byref(res), segments.ctypes.data)
            again = self._again(rc, res, out, chunk, slot)
            if again is None:
                _lib.check(rc)
                break
            slot, _, chunk = again
            out = self._out_buffer(slot, res.out_bytes)
        self._account(res)
        self._take_rows(slot)
        return {name: out[segments[i]:segments[i + 1]].tobytes() for i, name in enumerate(outputs + [unknown])}

    def _info_names(self):
        """Adapter names as the info file shows them: the parts of a linked adapter are "name;1" / "name;2"
        (LinkedMatch.get_info_records, adapters.py:1157-1171)."""
        return _row_text(self.adapters, "info")

    def _process_chunk_rows(self, chunk, kind: str) -> Tuple[bytes, bytes]:
        """(trimmed output, the rows of one kind) of a chunk: that kind is requested next to the trimmer's rows."""
        self._no_redirect(kind + " file rows")
        if self.adapters is None:
            raise ValueError("these outputs need adapters")
        out = self._collect(self._submit(chunk, tuple(dict.fromkeys(self.rows + (kind,)))))
        return out, self._rows_taken[kind]

    def process_chunk_info(self, chunk) -> Tuple[bytes, bytes]:
        """(trimmed FASTQ, the rows ``--info-file`` gets for the chunk), both formatted on the device
        (``cg_fastq_request_rows`` CG_ROWS_INFO; InfoFileWriter, steps.py:222-253)."""
        if self.adapters is None:
            raise ValueError("the info file needs adapters")
        return self._process_chunk_rows(chunk, "info")

    def process_chunk_rest(self, chunk) -> Tuple[bytes, bytes]:
        """(trimmed FASTQ, the rows of ``--rest-file``): RestFileWriter, steps.py:193-206."""
        return self._process_chunk_rows(chunk, "rest")

    def process_chunk_wildcards(self, chunk) -> Tuple[bytes, bytes]:
        """(trimmed FASTQ, the rows of ``--wildcard-file``): WildcardFileWriter, steps.py:209-220."""
        return self._process_chunk_rows(chunk, "wildcard")

    @property
    def collect_statistics(self) -> bool:
        return self._stats is not None

    @property
    def statistics_adapters(self) -> int:
        """Number of adapters the statistics vector has blocks for (its n_adapters)."""
        if self._stats is None:
            raise ValueError("this trimmer does not collect statistics (collect_statistics=False)")
        return self._stats.n_adapters

    def close(self) -> None:
        """Release the statistics accumulator now rather than when the trimmer is collected."""
        if self._stats is not None:
            self._stats.close()

    def statistics_vector(self) -> Tuple[np.ndarray, int, int]:
        """(vector, max_len, kmax) of everything trimmed so far (layout: fastq_stats_layout)."""
        if self._stats is None:
            raise ValueError("this trimmer does not collect statistics (collect_statistics=False)")
        return self._stats.read()

    def adapter_statistics(self):
        """AdapterStatistics of every adapter (AdapterCutter.adapter_statistics / ReverseComplementer's)."""
        stats, max_len, kmax = self.statistics_vector()
        return fastq_adapter_statistics(stats, self.adapters, max_len, kmax) if self.adapters is not None else []

    @property
    def poly_a_trimmed_lengths(self) -> dict:
        stats, max_len, kmax = self.statistics_vector()
        return poly_a_trimmed_lengths(stats, self._stats.n_adapters, max_len, kmax)

    @property
    def written_lengths(self) -> dict:
        stats, max_len, _ = self.statistics_vector()
        return written_lengths(stats, max_len)

    def process_chunks(self, chunks, copy: bool = True):
        """copy=False yields uint8 array views into per-slot buffers: valid until the next-but-one result."""
        self._no_redirect("process_chunks")
        yield from _one_in_flight(chunks, self._submit, lambda ticket: self._collect(ticket, copy))


class PairedFastqTrimmer:
    """
    Paired-end FASTQ chunks (``PairedEndPipeline.process_reads``, pipeline.py:125-153): record i of the two
    chunks is one pair.  ``adapters1`` / ``adapters2`` are the -a / -A adapters (None or [] for none),
    ``options1`` / ``options2`` dicts with FastqTrimmer's keyword arguments for each mate (-q / -Q, -u / -U,
    -l / -L ...; ``max_average_error_rate`` and ``zero_cap`` go into both, as on the command line; filters such as
    ``minimum_length`` or ``discard_trimmed`` go into both unless the command line gives them for one mate only).
    ``pair_filter`` is "any" (default), "both" or "first" (PairedEndFilter, steps.py:105-180).  ``input_format`` /
    ``output_format`` as for FastqTrimmer, for both mates (read_paired_fasta_chunks).  ``process_chunk(chunk1, chunk2) -> (bytes, bytes)``;
    ``statistics`` = (dict for R1, dict for R2).  ``collect_statistics``: as for FastqTrimmer, one accumulator per
    mate; ``statistics_vector()``, ``adapter_statistics()``, ``poly_a_trimmed_lengths`` and ``written_lengths`` give
    one value per mate.  ``redirect`` / ``redirect_formats``: as for FastqTrimmer, both mates of a removed pair go to
    the filter's two outputs (--too-short-output / --too-short-paired-output, ...); with adapters on one mate only, a
    pair is untrimmed when both mates are (cli.py:859-893).  ``process_chunk_split(chunk1, chunk2) -> {name: (bytes1,
    bytes2)}`` and ``process_chunks_split(iterable of pairs)``.

    Interleaved data (``--interleaved``): every chunk method takes ``chunk2=None`` to mean that ``chunk1`` holds R1 and
    R2 of each pair one after the other (read_interleaved_fastq_chunks / read_interleaved_fasta_chunks); the device
    splits it (``cg_fastq_submit_interleaved``) and rejects an odd record count or mates whose names do not match.
    ``process_chunks_split`` takes single chunks in place of pairs.  ``interleaved_outputs``: names out of
    ``("output",) + REDIRECT_OUTPUTS`` whose output is written interleaved, R1 then R2 of each pair, returned as
    ``(bytes, b"")`` (the reference interleaves an output whose paired path is missing).  Not with ``pair_adapters``
    or demultiplexing.  ``gzip_outputs`` / ``gzip_outputs2``: as FastqTrimmer's ``gzip_outputs``, for R1's files and for
    R2's (default: the same names); an interleaved output must be named in both.

    ``rows`` / ``rows2``: FastqTrimmer's ``rows`` for R1's reads and for R2's (--info-file, --rest-file and
    --wildcard-file write R1's rows, PairedSingleEndStep, cli.py:675-696; --info-file-paired adds R2's info rows,
    PairedInfoFileWriter, steps.py:256-269); ``gzip_rows`` / ``gzip_rows2`` the kinds compressed (default for R2: those
    of ``gzip_rows`` it has).  Every chunk method leaves ``last_rows`` = {kind: (bytes of R1, bytes of R2)}, b"" for a
    mate without that kind.  With ``pair_adapters`` the info rows name adapter i of each mate's own list.

    ``revcomp`` / ``rc_suffix``: --revcomp for the pair (PairedReverseComplementer, modifiers.py:311-400), on the
    device.  After each mate's own -u / --nextseq-trim / -q, the -a set also runs on R2 and the -A set on R1; a pair
    whose swapped matches score strictly more is written swapped: R1's output gets R2's read trimmed by the -a set, R2's
    output gets R1's read trimmed by the -A set, both names with " rc" unless rc_suffix is False.  Without adapters it
    does nothing.  ``statistics[k]["reverse_complemented"]`` counts the swapped pairs; each adapter's
    ``reverse_complemented`` its matches in swapped pairs.  Not with ``pair_adapters`` or info rows.

    ``length_tag`` / ``strip_suffix`` / ``prefix`` / ``suffix`` / ``rename``: as for FastqTrimmer, on both mates; the
    template is PairedEndRenamer's ({rn}, {r1.x} / {r2.x}), and a pair whose new IDs no longer name mates fails the call
    with the reference's message.
    """

    MODES = {"any": 0, "both": 1, "first": 2}

    def __init__(self, adapters1=None, adapters2=None, options1: Optional[dict] = None,
                 options2: Optional[dict] = None, pair_filter: str = "any", pair_adapters: bool = False,
                 input_format: str = "fastq", output_format: Optional[str] = None,
                 ctx: Optional[_lib.Context] = None, collect_statistics: bool = False,
                 redirect: Sequence[str] = (), redirect_formats: Optional[dict] = None,
                 interleaved_outputs: Sequence[str] = (), gzip_outputs: Sequence[str] = (),
                 gzip_outputs2: Optional[Sequence[str]] = None, rows: Sequence[str] = (),
                 rows2: Sequence[str] = (), gzip_rows: Sequence[str] = (), gzip_rows2: Optional[Sequence[str]] = None,
                 revcomp: bool = False, rc_suffix: bool = True, rename: Optional[str] = None, prefix: str = "",
                 suffix: str = "", strip_suffix: Sequence[str] = (), length_tag: Optional[str] = None):
        if pair_filter not in self.MODES:
            raise ValueError("pair_filter must be 'any', 'both' or 'first'")
        if input_format == "bam":
            raise ValueError("BAM input is read single-end only (as the reference reads it): use FastqTrimmer")
        for options in (options1, options2):
            for key in ("revcomp", "rc_suffix"):
                if key in (options or {}):
                    raise ValueError(f"--revcomp is one option for the pair: pass {key}= to PairedFastqTrimmer, "
                                     "not in options1 / options2")
        if revcomp and "info" in tuple(rows or ()) + tuple(rows2 or ()):
            raise ValueError("info rows (--info-file) cannot be combined with --revcomp on pairs")
        self.rows, self.gzip_rows = _row_kinds(rows, gzip_rows)
        if gzip_rows2 is None:
            gzip_rows2 = [k for k in self.gzip_rows if k in (rows2 or ())]
        self.rows2, self.gzip_rows2 = _row_kinds(rows2, gzip_rows2, "rows2")
        self.last_rows = {}
        formats = dict(input_format=input_format, output_format=output_format, revcomp=revcomp, rc_suffix=rc_suffix)
        self.params1 = _fastq_params(**{**(options1 or {}), **formats})
        self.params2 = _fastq_params(**{**(options2 or {}), **formats})
        if pair_adapters and revcomp:
            raise ValueError("Cannot use --revcomp with --pair-adapters")            # cli.py:1087
        self.params1.gzip_outputs = _gzip_bits(gzip_outputs)
        self.params2.gzip_outputs = _gzip_bits(gzip_outputs if gzip_outputs2 is None else gzip_outputs2)
        self.redirect = tuple(dict.fromkeys(redirect or ()))
        self._redirect, self._fasta_outputs = _redirect_bits(self.redirect, redirect_formats, self.params1)
        _redirect_bits(self.redirect, redirect_formats, self.params2)
        if self._redirect and pair_adapters:
            raise ValueError("filter outputs cannot be combined with --pair-adapters")
        self.interleaved_outputs = tuple(dict.fromkeys(interleaved_outputs or ()))
        self._interleave = 0
        for name in self.interleaved_outputs:
            if name not in INTERLEAVE_BITS:
                raise ValueError(f"unknown output {name!r} to interleave (one of {', '.join(INTERLEAVE_BITS)})")
            self._interleave |= INTERLEAVE_BITS[name]
        if self._interleave and pair_adapters:
            raise ValueError("interleaved outputs cannot be combined with --pair-adapters")
        self.ctx = ctx or _lib.default_context()
        self.mode = self.MODES[pair_filter]
        self.statistics = ({}, {})
        self._pairs = None
        if pair_adapters:
            # --pair-adapters (PairedAdapterCutter.__init__, modifiers.py:417-442): one device set per adapter
            adapters1, adapters2 = list(adapters1 or []), list(adapters2 or [])
            if len(adapters1) != len(adapters2):
                raise ValueError("The number of adapters to trim from R1 and R2 must be the same. "
                                 f"Given: {len(adapters1)} for R1, {len(adapters2)} for R2")
            if not adapters1:
                raise ValueError("No adapters given")
            self.adapters1, self.adapters2 = adapters1, adapters2
            self._pairs = [(_device_set([a1], self.ctx)[1], _device_set([a2], self.ctx)[1])
                           for a1, a2 in zip(adapters1, adapters2)]
            self._set1 = self._set2 = None
            k = len(self._pairs)
            self._pair_handles = ((C.c_void_p * k)(*[p[0].handle for p in self._pairs]),
                                  (C.c_void_p * k)(*[p[1].handle for p in self._pairs]))
        else:
            self.adapters1, self._set1 = _device_set(adapters1, self.ctx)
            self.adapters2, self._set2 = _device_set(adapters2, self.ctx)
        self._stats = None
        if collect_statistics:
            if self._pairs is not None:
                counts = (len(self._pairs), len(self._pairs))
            else:
                counts = tuple(len(a._flatten()[0]) if a is not None else 0 for a in (self.adapters1, self.adapters2))
            self._stats = tuple(_lib.FastqStatistics(self.ctx, n) for n in counts)
            self.params1.stats, self.params2.stats = self._stats[0].handle, self._stats[1].handle
        pair_list = self._pairs is not None
        self._names = _make_names(self.ctx, rename, prefix, suffix, strip_suffix, length_tag, True)
        if self._names is not None and pair_list and rename and "match_sequence" in rename and any(
                isinstance(a, LinkedAdapter) for a in self.adapters1 + self.adapters2):
            # a linked adapter of a --pair-adapters list matches as one adapter here: its front,back form is not kept
            raise ValueError("{match_sequence} cannot be combined with linked adapters under --pair-adapters")
        if self._names is not None:
            for mate, (adapters, options) in enumerate(((self.adapters1, options1), (self.adapters2, options2))):
                self._names.set_mate(mate, *_name_table(adapters, pair_list), *_last_cuts((options or {}).get("cut", ())))
            self.params1.names = self.params2.names = self._names.handle
        self._row_texts = ({k: _row_text(self.adapters1, k, pair_list) for k in self.rows},
                           {k: _row_text(self.adapters2, k, pair_list) for k in self.rows2})

    @property
    def collect_statistics(self) -> bool:
        return self._stats is not None

    def close(self) -> None:
        """Release the two statistics accumulators now rather than when the trimmer is collected."""
        for st in self._stats or ():
            st.close()

    def statistics_vector(self):
        """((vector, max_len, kmax) of R1, the same of R2)."""
        if self._stats is None:
            raise ValueError("this trimmer does not collect statistics (collect_statistics=False)")
        return tuple(st.read() for st in self._stats)

    def adapter_statistics(self):
        """(AdapterStatistics of R1's adapters, of R2's): the two lists of PairedAdapterCutter.adapter_statistics
        under --pair-adapters, else those of the two AdapterCutters."""
        out = []
        for (stats, max_len, kmax), adapters in zip(self.statistics_vector(), (self.adapters1, self.adapters2)):
            if self._pairs is not None:
                out.append(pair_adapter_statistics_from_vector(stats, adapters, max_len, kmax))
            else:
                out.append(fastq_adapter_statistics(stats, adapters, max_len, kmax) if adapters is not None else [])
        return tuple(out)

    @property
    def poly_a_trimmed_lengths(self):
        return tuple(poly_a_trimmed_lengths(v, st.n_adapters, max_len, kmax)
                     for (v, max_len, kmax), st in zip(self.statistics_vector(), self._stats))

    @property
    def written_lengths(self):
        return tuple(written_lengths(v, max_len) for v, max_len, _ in self.statistics_vector())

    def _submit_pair(self, chunk1, chunk2):
        """((slot1, chunk), (slot2, chunk)): two chunks, or one interleaved chunk (chunk2 None) split on the device;
        the rows of each mate are requested."""
        tickets = self._upload_pair(chunk1, chunk2)
        for (slot, _), kinds, texts, gz in zip(tickets, (self.rows, self.rows2), self._row_texts,
                                                (self.gzip_rows, self.gzip_rows2)):
            _request_rows(self.ctx, slot, kinds, texts, gz)
        return tickets

    def _upload_pair(self, chunk1, chunk2):
        if chunk2 is not None:
            return _submit_chunk(self.ctx, chunk1), _submit_chunk(self.ctx, chunk2)
        if isinstance(chunk1, DeviceChunk):            # interleaved, already split into two slots
            return (chunk1.slot, chunk1), (chunk1.slot2, chunk1)
        buf = np.frombuffer(chunk1, dtype=np.uint8) if not isinstance(chunk1, np.ndarray) else chunk1
        s1, s2 = C.c_int32(-1), C.c_int32(-1)
        _lib.check(_lib.lib().cg_fastq_submit_interleaved(self.ctx.handle, buf.ctypes.data if buf.size else None,
                                                          buf.size, self.params1.format, C.byref(s1), C.byref(s2)))
        return (s1.value, buf), (s2.value, buf)

    def _take_rows(self, tickets) -> None:
        """last_rows of the pair of slots just collected: {kind: (R1's rows, R2's rows)}."""
        (s1, _), (s2, _) = tickets
        r1, r2 = _read_rows(self.ctx, s1, self.rows), _read_rows(self.ctx, s2, self.rows2)
        self.last_rows = {k: (r1.get(k, b""), r2.get(k, b"")) for k in ROW_KINDS if k in r1 or k in r2}

    def _run(self, tickets, call, n_dest: int = 4):
        """(tickets, out1, out2, r1, r2) of call(tickets, out1, out2, r1, r2) -> rc.  With read names an output can
        outgrow its bound: the call then says how much it needs and the pair is submitted and run again."""
        kept = None
        if self._names is not None:
            (_, b1), (_, b2) = tickets
            if b1 is b2:                                # one interleaved chunk (a device chunk: read from its first slot)
                kept = (_keep_chunk(self.ctx, b1), None)
            else:
                kept = (_keep_chunk(self.ctx, b1), _keep_chunk(self.ctx, b2))
        need = (0, 0)
        while True:
            out1, out2 = self._out_buffers(tickets, n_dest, need)
            r1, r2 = _lib.cg_fastq_result(), _lib.cg_fastq_result()
            rc = call(tickets, out1, out2, r1, r2)
            cap1 = out1.size - (out2.size if self._interleave else 0)
            if rc != 0 and kept is not None and (r1.out_bytes > cap1 or r2.out_bytes > out2.size):
                need = (max(r1.out_bytes, cap1), max(r2.out_bytes, out2.size))
                tickets = self._submit_pair(*kept)
                continue
            _lib.check(rc)
            return tickets, out1, out2, r1, r2

    def _out_buffers(self, tickets, n_dest: int = 4, need=(0, 0)):
        """Output buffers of a pair: out1 also holds R2 of the interleaved outputs.  With --revcomp either mate's output
        can receive the other mate's records, each with " rc" (3 bytes on a FASTQ record of at least 6)."""
        (_, b1), (_, b2) = tickets
        if self.params1.revcomp:
            both = b1.size + b2.size
            n_in = both + both // 2 if self.params1.format == _lib.CG_FORMAT_FASTQ else both
            n1 = _output_capacity(n_in, self.params1.format, self.params1.gzip_outputs != 0, n_dest, True)
            n2 = _output_capacity(n_in, self.params2.format, self.params2.gzip_outputs != 0, n_dest, True)
        else:
            n1 = _output_capacity(b1.size, self.params1.format, self.params1.gzip_outputs != 0, n_dest)
            n2 = _output_capacity(b2.size, self.params2.format, self.params2.gzip_outputs != 0, n_dest)
        n1, n2 = max(n1, need[0]), max(n2, need[1])
        return np.empty(n1 + (n2 if self._interleave else 0), dtype=np.uint8), np.empty(n2, dtype=np.uint8)

    def _no_interleave(self, what: str):
        if self._interleave:
            raise ValueError(f"interleaved outputs ({', '.join(self.interleaved_outputs)}) cannot be combined with {what}")

    def _account(self, r1, r2):
        for st, res, p in zip(self.statistics, (r1, r2), (self.params1, self.params2)):
            for k, v in res.as_dict(p.gzip_outputs != 0).items():
                st[k] = st.get(k, 0) + v

    def _no_redirect(self, what: str):
        if self._redirect:
            raise ValueError(f"filter outputs ({', '.join(self.redirect)}) cannot be combined with {what}; "
                             "use process_chunk_split / process_chunks_split")

    def _collect_split(self, tickets) -> dict:
        seg1, seg2 = np.zeros(5, dtype=np.int64), np.zeros(5, dtype=np.int64)
        sets = (self._set1.handle if self._set1 is not None else None,
                self._set2.handle if self._set2 is not None else None)

        def call(tickets, out1, out2, r1, r2):
            (s1, _), (s2, _) = tickets
            if self._interleave:
                return _lib.lib().cg_fastq_collect_paired_interleaved(
                    self.ctx.handle, s1, s2, *sets, C.byref(self.params1), C.byref(self.params2), self.mode,
                    self._redirect, self._fasta_outputs, self._interleave, out1.ctypes.data, out1.size,
                    out2.ctypes.data, out2.size, C.byref(r1), C.byref(r2), seg1.ctypes.data, seg2.ctypes.data)
            return _lib.lib().cg_fastq_collect_paired_split(
                self.ctx.handle, s1, s2, *sets, C.byref(self.params1), C.byref(self.params2), self.mode,
                self._redirect, self._fasta_outputs, out1.ctypes.data, out1.size, out2.ctypes.data, out2.size,
                C.byref(r1), C.byref(r2), seg1.ctypes.data, seg2.ctypes.data)

        tickets, out1, out2, r1, r2 = self._run(tickets, call)
        self._account(r1, r2)
        self._take_rows(tickets)
        names = ("output",) + REDIRECT_OUTPUTS
        return {name: (out1[seg1[d]:seg1[d + 1]].tobytes(), out2[seg2[d]:seg2[d + 1]].tobytes())
                for d, name in enumerate(names) if d == 0 or name in self.redirect}

    def process_chunk_split(self, chunk1, chunk2=None) -> dict:
        """{"output": (R1, R2) of the main outputs, and for every name in ``redirect``: (R1, R2) of the pairs that filter
        removed} for one pair of chunks, or one interleaved chunk (chunk2 None); an interleaved output is (R1 and R2,
        b"") (``cg_fastq_collect_paired_split`` / ``cg_fastq_collect_paired_interleaved``)."""
        return self._collect_split(self._submit_pair(chunk1, chunk2))

    def process_chunks_split(self, pairs):
        """process_chunk_split over an iterable of (chunk1, chunk2), or of interleaved chunks, with one pair in flight:
        the upload of pair i+1 overlaps the work on pair i."""
        yield from _one_in_flight(
            pairs, lambda item: self._submit_pair(*(item if isinstance(item, (tuple, list)) else (item, None))),
            self._collect_split)

    def process_chunk(self, chunk1, chunk2=None) -> Tuple[bytes, bytes]:
        """(R1, R2) of one pair of chunks or of one interleaved chunk (chunk2 None); with "output" in
        ``interleaved_outputs``: (R1 and R2 interleaved, b"")."""
        self._no_redirect("process_chunk")
        if self._interleave:
            return self._collect_split(self._submit_pair(chunk1, chunk2))["output"]
        def call(tickets, out1, out2, r1, r2):
            (s1, _), (s2, _) = tickets
            if self._pairs is not None:
                return _lib.lib().cg_fastq_collect_pair_adapters(
                    self.ctx.handle, s1, s2, self._pair_handles[0], self._pair_handles[1], len(self._pairs),
                    C.byref(self.params1), C.byref(self.params2), self.mode, out1.ctypes.data, out1.size,
                    out2.ctypes.data, out2.size, C.byref(r1), C.byref(r2))
            return _lib.lib().cg_fastq_collect_paired(
                self.ctx.handle, s1, s2, self._set1.handle if self._set1 is not None else None,
                self._set2.handle if self._set2 is not None else None, C.byref(self.params1), C.byref(self.params2),
                self.mode, out1.ctypes.data, out1.size, out2.ctypes.data, out2.size, C.byref(r1), C.byref(r2))

        tickets, out1, out2, r1, r2 = self._run(self._submit_pair(chunk1, chunk2), call)
        self._account(r1, r2)
        self._take_rows(tickets)
        return out1[: r1.out_bytes].tobytes(), out2[: r2.out_bytes].tobytes()

    def process_chunk_demux(self, chunk1, chunk2=None, combinatorial: bool = False, discard_untrimmed: bool = False,
                            unknown: str = "unknown") -> dict:
        """
        Demultiplexed pairs of one chunk on the device (``cg_fastq_collect_paired_demux``).

        combinatorial=False: ``PairedDemultiplexer`` (steps.py:422-503) -- {adapter name of R1's most recent match or
        ``unknown``: (R1 bytes, R2 bytes)}; with ``discard_untrimmed`` the ``unknown`` output is not produced.
        combinatorial=True: ``CombinatorialDemultiplexer`` (steps.py:506-581) -- keys are (name1, name2) with None for a
        mate without a match; with ``discard_untrimmed`` only pairs with matches on both mates are kept.  Pairs
        without an output are dropped without being counted, as in the reference.  chunk2 None: chunk1 is interleaved.
        """
        if self._pairs is not None:
            raise ValueError("demultiplexing with --pair-adapters is not supported")
        self._no_redirect("demultiplexing")
        self._no_interleave("demultiplexing")
        names1, dest1 = _demux_names(self.adapters1)
        n1 = len(names1)
        if combinatorial:
            names2, dest2 = _demux_names(self.adapters2)
            n2 = len(names2)
            keys = [(a, b) for a in names1 + [None] for b in names2 + [None]]
            keep = np.array([not discard_untrimmed or (a is not None and b is not None) for a, b in keys], dtype=np.uint8)
        else:
            dest2, n2 = None, 0
            keys = names1 + [unknown]
            keep = np.array([1] * n1 + [0 if discard_untrimmed else 1], dtype=np.uint8)
        seg1 = np.zeros(len(keys) + 1, dtype=np.int64)
        seg2 = np.zeros(len(keys) + 1, dtype=np.int64)

        def call(tickets, out1, out2, r1, r2):
            (s1, _), (s2, _) = tickets
            return _lib.lib().cg_fastq_collect_paired_demux(
                self.ctx.handle, s1, s2, self._set1.handle, self._set2.handle if self._set2 is not None else None,
                C.byref(self.params1), C.byref(self.params2), self.mode, dest1.ctypes.data, n1,
                dest2.ctypes.data if dest2 is not None else None, n2, keep.ctypes.data, out1.ctypes.data, out1.size,
                out2.ctypes.data, out2.size, C.byref(r1), C.byref(r2), seg1.ctypes.data, seg2.ctypes.data)

        tickets, out1, out2, r1, r2 = self._run(self._submit_pair(chunk1, chunk2), call, len(keys))
        self._account(r1, r2)
        self._take_rows(tickets)
        return {key: (out1[seg1[i]:seg1[i + 1]].tobytes(), out2[seg2[i]:seg2[i + 1]].tobytes())
                for i, key in enumerate(keys) if keep[i]}


class DeviceResult:
    def __init__(self, matches, qtrim, n_reads, offsets, seq=None):
        self.matches = matches    # torch int32 [n * times * slots, 8]
        self.qtrim = qtrim        # torch int32 [n, 2] or None
        self.n_reads = n_reads
        self.offsets = offsets
        self.seq = seq            # the reads (for the adjacent-base counts of the statistics)


class DeviceBatch:
    """The fused pass on torch CUDA tensors already resident in HBM (cg_process_batch_device)."""

    def __init__(self, adapters, times: int = 1, quality_cutoff: Optional[Tuple[int, int]] = None,
                 quality_base: int = 33, device: Optional[int] = None, nextseq_cutoff: Optional[int] = None):
        import torch

        self.adapters: Matchable = adapters if isinstance(adapters, Matchable) else MultipleAdapters(list(adapters))
        self.device = torch.cuda.current_device() if device is None else device
        # torch's default stream is the legacy stream (handle 0); cudaStreamLegacy (0x1) names it
        # explicitly so that the library launches on it instead of creating its own stream
        stream = torch.cuda.current_stream(self.device).cuda_stream or 1
        self.ctx = _lib.Context(self.device, stream)
        singles, groups, owners = self.adapters._flatten()
        self.spec = _lib.AdapterSetSpec([s.descriptor() for s in singles], groups, self.adapters._flatten_indexes())
        self.adapter_set = _lib.AdapterSet(self.spec, self.ctx)
        self.n_adapters = len(singles)
        self.times = int(times)
        self.params = _lib.make_params(
            quality_trim=quality_cutoff is not None,
            cutoff_front=quality_cutoff[0] if quality_cutoff else 0,
            cutoff_back=quality_cutoff[1] if quality_cutoff else 0,
            quality_base=quality_base,
            times=times,
            nextseq_cutoff=nextseq_cutoff,
        )

    def run(self, seq, offsets, qual=None, max_read_len: int = 0, out=None, qtrim_out=None) -> DeviceResult:
        import torch

        n = int(offsets.numel() - 1)
        slots = self.adapter_set.slots
        if out is None:
            out = torch.empty((n * self.times * slots, 8), dtype=torch.int32, device=seq.device)
        want_q = bool(self.params.quality_trim or self.params.nextseq_trim)
        if want_q and qtrim_out is None:
            qtrim_out = torch.empty((n, 2), dtype=torch.int32, device=seq.device)
        _lib.check(
            _lib.lib().cg_process_batch_device(
                self.ctx.handle, self.adapter_set.handle, seq.data_ptr(),
                qual.data_ptr() if (qual is not None and want_q) else None, offsets.data_ptr(), n,
                int(max_read_len), C.byref(self.params), out.data_ptr(),
                qtrim_out.data_ptr() if qtrim_out is not None else None,
            )
        )
        return DeviceResult(out, qtrim_out, n, offsets, seq)

    def run_with_statistics(self, seq, offsets, qual=None, max_read_len: int = 0, out=None, qtrim_out=None,
                            max_len: int = 150, kmax: int = 3, into=None):
        """``run`` + ``statistics`` as ONE library call (``cg_process_batch_device_stats``): for a set of one plain
        adapter the statistics are gathered inside the trimming pass instead of from the records afterwards; the
        resulting vector is the same.  Returns (DeviceResult, statistics vector)."""
        import torch

        n = int(offsets.numel() - 1)
        slots = self.adapter_set.slots
        if out is None:
            out = torch.empty((n * self.times * slots, 8), dtype=torch.int32, device=seq.device)
        want_q = bool(self.params.quality_trim or self.params.nextseq_trim)
        if want_q and qtrim_out is None:
            qtrim_out = torch.empty((n, 2), dtype=torch.int32, device=seq.device)
        size = int(_lib.lib().cg_stats_size(self.n_adapters, max_len, kmax))
        stats = into if into is not None else torch.zeros(size, dtype=torch.int64, device=seq.device)
        _lib.check(
            _lib.lib().cg_process_batch_device_stats(
                self.ctx.handle, self.adapter_set.handle, seq.data_ptr(),
                qual.data_ptr() if (qual is not None and want_q) else None, offsets.data_ptr(), n,
                int(max_read_len), C.byref(self.params), out.data_ptr(),
                qtrim_out.data_ptr() if qtrim_out is not None else None, max_len, kmax, stats.data_ptr(),
            )
        )
        return DeviceResult(out, qtrim_out, n, offsets, seq), stats

    def statistics(self, result: DeviceResult, max_len: int = 150, kmax: int = 3, into=None):
        """Device-side reduction of a batch into the fixed-layout int64 statistics vector."""
        import torch

        size = int(_lib.lib().cg_stats_size(self.n_adapters, max_len, kmax))
        stats = into if into is not None else torch.zeros(size, dtype=torch.int64, device=result.matches.device)
        _lib.check(
            _lib.lib().cg_stats_accumulate_device(
                self.ctx.handle, self.adapter_set.handle,
                result.seq.data_ptr() if result.seq is not None else None, result.offsets.data_ptr(), result.n_reads,
                C.byref(self.params), result.matches.data_ptr(),
                result.qtrim.data_ptr() if result.qtrim is not None else None, max_len, kmax, stats.data_ptr(),
            )
        )
        return stats
