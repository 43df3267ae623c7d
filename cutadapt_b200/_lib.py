"""
ctypes binding of ``libcutadapt_b200.so`` (include/cutadapt_b200.h).

This module is the only place that touches the C ABI.  There is no CPU fallback: if the
shared library is missing or no CUDA device is usable, the first call that needs the device
raises ``RuntimeError`` -- loudly, by design (the reference's behaviour on a broken extension
module is an ImportError, too).
"""
import ctypes as C
import os
import threading
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcutadapt_b200.so")

# ---- status codes (include/cutadapt_b200.h) ------------------------------------------------
CG_OK = 0
CG_EINVAL = -1
CG_ENONASCII = -2
CG_ECUDA = -3
CG_ENOMEM = -4
CG_EUNSUPPORTED = -5
CG_ENOQUAL = -6

CG_KIND_ALIGNER = 0
CG_KIND_PREFIX_COMPARER = 1
CG_KIND_SUFFIX_COMPARER = 2
CG_REMOVE_BEFORE = 0
CG_REMOVE_AFTER = 1
CG_REMOVE_AUTO = 2
CG_GROUP_SINGLE = 0
CG_GROUP_LINKED = 1
CG_GROUP_INDEXED = 2
CG_FORMAT_FASTQ = 0              # cg_fastq_params.format: FASTQ in, FASTQ out
CG_FORMAT_FASTA = 1              # FASTA in, FASTA out
CG_FORMAT_FASTQ_TO_FASTA = 2     # FASTQ in, FASTA out
CG_FORMAT_BAM = 3                # cg_fastq_submit_gzip only: unaligned BAM in, its records as FASTQ text in the slot
CG_GZIN_SPLIT_MEMBERS = 1        # cg_gzin_create_ex: long members inflated block-parallel, consumed in part
CG_GZIN_LONG_MEMBER = 64 * 1024  # compressed bytes above which a split stream takes a member block-parallel
CG_GZIN_STRIDE = 64 * 1024       # compressed bytes between speculative chunk starts
CG_REDIRECT_TOO_SHORT = 1        # cg_fastq_collect_split: --too-short-output (destination 1)
CG_REDIRECT_TOO_LONG = 2         # --too-long-output (destination 2)
CG_REDIRECT_UNTRIMMED = 4        # --untrimmed-output (destination 3)
CG_INTERLEAVE_MAIN = 8           # cg_fastq_collect_paired_interleaved: the main output is interleaved
CG_GZIP_MAIN = 8                 # cg_fastq_params.gzip_outputs: the main (every demultiplexed) output is gzip
CG_ROWS_INFO = 0                 # cg_fastq_request_rows: --info-file rows
CG_ROWS_REST = 1                 # --rest-file rows
CG_ROWS_WILDCARD = 2             # --wildcard-file rows
GZ_MEMBER = 65280                # plain bytes per gzip member of a gzip output ...
GZ_OVERHEAD = 23                 # ... and the most a member adds to them


class cg_kmer_entry(C.Structure):
    _fields_ = [
        ("search_start", C.c_int64),
        ("search_stop", C.c_int64),
        ("init_mask", C.c_uint64),
        ("found_mask", C.c_uint64),
    ]


class cg_adapter_desc(C.Structure):
    _fields_ = [
        ("sequence", C.c_char_p),
        ("length", C.c_int32),
        ("max_error_rate", C.c_double),
        ("flags", C.c_int32),
        ("wildcard_ref", C.c_int32),
        ("wildcard_query", C.c_int32),
        ("indel_cost", C.c_int32),
        ("min_overlap", C.c_int32),
        ("kind", C.c_int32),
        ("reverse_read", C.c_int32),
        ("remove", C.c_int32),
        ("kmer_entries", C.POINTER(cg_kmer_entry)),
        ("kmer_masks", C.POINTER(C.c_uint64)),
        ("n_kmer_entries", C.c_int32),
        ("reserved", C.c_int32),
    ]


class cg_group_desc(C.Structure):
    _fields_ = [
        ("type", C.c_int32),
        ("a0", C.c_int32),
        ("a1", C.c_int32),
        ("front_required", C.c_int32),
        ("back_required", C.c_int32),
        ("reserved", C.c_int32 * 3),
    ]


class cg_index_desc(C.Structure):
    _fields_ = [
        ("prefix", C.c_int32),
        ("n_lengths", C.c_int32),
        ("lengths", C.POINTER(C.c_int32)),
        ("n_keys", C.c_int64),
        ("keys", C.c_void_p),
        ("stride", C.c_int32),
        ("reserved", C.c_int32),
        ("adapter", C.POINTER(C.c_int32)),
        ("errors", C.POINTER(C.c_int32)),
        ("matches", C.POINTER(C.c_int32)),
    ]


class cg_params(C.Structure):
    _fields_ = [
        ("quality_trim", C.c_int32),
        ("cutoff_front", C.c_int32),
        ("cutoff_back", C.c_int32),
        ("quality_base", C.c_int32),
        ("times", C.c_int32),
        ("nextseq_trim", C.c_int32),
        ("nextseq_cutoff", C.c_int32),
        ("reserved", C.c_int32),
    ]


class cg_fastq_params(C.Structure):
    _fields_ = [
        ("trim", cg_params),
        ("minimum_length", C.c_int32),
        ("maximum_length", C.c_int32),
        ("discard_trimmed", C.c_int32),
        ("discard_untrimmed", C.c_int32),
        ("max_n", C.c_double),
        ("max_expected_errors", C.c_double),
        ("cut_front", C.c_int32),
        ("cut_back", C.c_int32),
        ("poly_a", C.c_int32),
        ("shorten", C.c_int32),
        ("shorten_length", C.c_int32),
        ("trim_n", C.c_int32),
        ("discard_casava", C.c_int32),
        ("action", C.c_int32),
        ("revcomp", C.c_int32),
        ("format", C.c_int32),
        ("stats", C.c_int32),
        ("gzip_outputs", C.c_int32),
        ("max_average_error_rate", C.c_double),
        ("zero_cap", C.c_int32),
        ("names", C.c_int32),
    ]


class cg_fastq_result(C.Structure):
    _fields_ = [(name, C.c_int64) for name in (
        "n_records", "n_written", "bp_in", "bp_out", "out_bytes", "with_adapters", "quality_trimmed_bp",
        "too_short", "too_long", "too_many_n", "too_many_expected_errors", "discarded", "casava_filtered",
        "reverse_complemented", "out_bytes_plain", "too_high_average_error_rate")]

    def as_dict(self, plain_bytes: bool = False) -> dict:
        """The counters; out_bytes_plain (the uncompressed size of gzip outputs) only with plain_bytes."""
        return {name: int(getattr(self, name)) for name, _ in self._fields_
                if plain_bytes or name != "out_bytes_plain"}


class cg_gzin_result(C.Structure):
    _fields_ = [(name, C.c_int64) for name in (
        "consumed", "members", "plain_bytes", "chunk_bytes", "carry_bytes", "n_records", "in_member", "respeculated")]


MATCH_DTYPE = np.dtype(
    [
        ("adapter", "<i4"),
        ("astart", "<i4"),
        ("astop", "<i4"),
        ("rstart", "<i4"),
        ("rstop", "<i4"),
        ("score", "<i4"),
        ("errors", "<i4"),
        ("info", "<i4"),
    ]
)
assert MATCH_DTYPE.itemsize == 32


class CutadaptB200Error(RuntimeError):
    pass


_lib = None
_lib_lock = threading.Lock()


def _declare(lib) -> None:
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    lib.cg_version.restype = C.c_int
    lib.cg_last_error.restype = C.c_char_p
    lib.cg_ctx_create.argtypes = [C.c_int, vp, C.POINTER(vp)]
    lib.cg_ctx_destroy.argtypes = [vp]
    lib.cg_ctx_synchronize.argtypes = [vp]
    lib.cg_ctx_launch_count.argtypes = [vp]
    lib.cg_ctx_launch_count.restype = i64
    lib.cg_ctx_kernel_time.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(i64), C.c_int]
    lib.cg_ctx_host_profile.argtypes = [vp, C.POINTER(C.c_double), C.c_int]
    lib.cg_ctx_transfer_bytes.argtypes = [vp, C.POINTER(i64), C.POINTER(i64), C.c_int]
    lib.cg_pack3_host.argtypes = [vp, i64, i64, i64, i64, vp, vp, i64, i32]
    lib.cg_pack3_host.restype = i64
    lib.cg_fastq_trim_chunk.argtypes = [vp, vp, vp, i64, C.POINTER(cg_fastq_params), vp, i64,
                                        C.POINTER(cg_fastq_result)]
    lib.cg_fastq_submit.argtypes = [vp, vp, i64, C.POINTER(i32)]
    lib.cg_fastq_collect_demux.argtypes = [vp, i32, vp, C.POINTER(cg_fastq_params), vp, i32, vp, i64,
                                           C.POINTER(cg_fastq_result), vp]
    lib.cg_fastq_collect_paired.argtypes = [vp, i32, i32, vp, vp, C.POINTER(cg_fastq_params), C.POINTER(cg_fastq_params),
                                            i32, vp, i64, vp, i64, C.POINTER(cg_fastq_result), C.POINTER(cg_fastq_result)]
    lib.cg_fastq_collect_info.argtypes = [vp, i32, vp, C.POINTER(cg_fastq_params), C.c_char_p, vp, vp, i64, vp, i64,
                                          C.POINTER(cg_fastq_result), C.POINTER(i64)]
    lib.cg_fastq_collect_rows.argtypes = [vp, i32, vp, C.POINTER(cg_fastq_params), i32, C.c_char_p, vp, vp, i64, vp, i64,
                                          C.POINTER(cg_fastq_result), C.POINTER(i64)]
    lib.cg_fastq_request_rows.argtypes = [vp, i32, i32, C.c_char_p, vp, i32, i32]
    lib.cg_fastq_read_rows.argtypes = [vp, i32, i32, vp, i64, C.POINTER(i64), C.POINTER(i64)]
    lib.cg_fastq_collect_pair_adapters.argtypes = [vp, i32, i32, vp, vp, i32, C.POINTER(cg_fastq_params),
                                                   C.POINTER(cg_fastq_params), i32, vp, i64, vp, i64,
                                                   C.POINTER(cg_fastq_result), C.POINTER(cg_fastq_result)]
    lib.cg_fastq_collect_paired_demux.argtypes = [vp, i32, i32, vp, vp, C.POINTER(cg_fastq_params),
                                                  C.POINTER(cg_fastq_params), i32, vp, i32, vp, i32, vp, vp, i64, vp, i64,
                                                  C.POINTER(cg_fastq_result), C.POINTER(cg_fastq_result), vp, vp]
    lib.cg_fastq_collect.argtypes = [vp, i32, vp, C.POINTER(cg_fastq_params), vp, i64, C.POINTER(cg_fastq_result)]
    lib.cg_fastq_collect_split.argtypes = [vp, i32, vp, C.POINTER(cg_fastq_params), i32, i32, vp, i64,
                                           C.POINTER(cg_fastq_result), vp]
    lib.cg_fastq_collect_paired_split.argtypes = [vp, i32, i32, vp, vp, C.POINTER(cg_fastq_params),
                                                  C.POINTER(cg_fastq_params), i32, i32, i32, vp, i64, vp, i64,
                                                  C.POINTER(cg_fastq_result), C.POINTER(cg_fastq_result), vp, vp]
    lib.cg_fastq_submit_interleaved.argtypes = [vp, vp, i64, i32, C.POINTER(i32), C.POINTER(i32)]
    lib.cg_gzin_create.argtypes = [vp, C.POINTER(i32)]
    lib.cg_gzin_create_ex.argtypes = [vp, i32, C.POINTER(i32)]
    lib.cg_fastq_slot_read.argtypes = [vp, i32, vp, i64, C.POINTER(i64)]
    lib.cg_gzin_destroy.argtypes = [vp, i32]
    lib.cg_gzin_bam_tiles.argtypes = [vp, i32, C.POINTER(i64), C.POINTER(i64)]
    lib.cg_fastq_submit_gzip.argtypes = [vp, i32, vp, i64, i32, i32, C.POINTER(i32), C.POINTER(cg_gzin_result)]
    lib.cg_fastq_submit_gzip_paired.argtypes = [vp, i32, i32, vp, i64, vp, i64, i32, i32, C.POINTER(i32), C.POINTER(i32),
                                                C.POINTER(cg_gzin_result), C.POINTER(cg_gzin_result)]
    lib.cg_fastq_submit_gzip_interleaved.argtypes = [vp, i32, vp, i64, i32, i32, C.POINTER(i32), C.POINTER(i32),
                                                     C.POINTER(cg_gzin_result)]
    lib.cg_fastq_collect_paired_interleaved.argtypes = [vp, i32, i32, vp, vp, C.POINTER(cg_fastq_params),
                                                        C.POINTER(cg_fastq_params), i32, i32, i32, i32, vp, i64, vp, i64,
                                                        C.POINTER(cg_fastq_result), C.POINTER(cg_fastq_result), vp, vp]
    lib.cg_fastq_stats_create.argtypes = [vp, i32, C.POINTER(i32)]
    lib.cg_fastq_stats_read.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32), vp, i64, C.POINTER(i64), C.c_int]
    lib.cg_fastq_stats_destroy.argtypes = [vp, i32]
    lib.cg_names_create.argtypes = [vp, C.POINTER(cg_names_desc), C.POINTER(i32)]
    lib.cg_names_set_mate.argtypes = [vp, i32, i32, C.c_char_p, vp, i32, vp, i32, i32]
    lib.cg_names_destroy.argtypes = [vp, i32]
    lib.cg_adapterset_create.argtypes = [
        vp, C.POINTER(cg_adapter_desc), i32, C.POINTER(cg_group_desc), i32, C.POINTER(vp),
    ]
    lib.cg_adapterset_create_indexed.argtypes = [
        vp, C.POINTER(cg_adapter_desc), i32, C.POINTER(cg_group_desc), i32,
        C.POINTER(cg_index_desc), i32, C.POINTER(vp),
    ]
    lib.cg_adapterset_destroy.argtypes = [vp]
    lib.cg_ctx_stage_times.argtypes = [vp, C.POINTER(C.c_double), C.c_int]
    lib.cg_adapterset_jit_status.argtypes = [vp]
    lib.cg_adapterset_jit_source.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.c_char_p, C.c_int64]
    lib.cg_adapterset_jit_source.restype = C.c_int64
    lib.cg_adapterset_slots.argtypes = [vp]
    lib.cg_adapterset_effective_length.argtypes = [vp, i32, C.POINTER(i32)]
    lib.cg_process_batch.argtypes = [vp, vp, vp, vp, vp, i64, C.POINTER(cg_params), vp, vp]
    lib.cg_process_batch_device.argtypes = [
        vp, vp, vp, vp, vp, i64, i32, C.POINTER(cg_params), vp, vp,
    ]
    lib.cg_process_batch_device_stats.argtypes = [
        vp, vp, vp, vp, vp, i64, i32, C.POINTER(cg_params), vp, vp, i32, i32, vp,
    ]
    lib.cg_kmers_present_batch.argtypes = [vp, C.POINTER(cg_kmer_entry), vp, i32, vp, vp, i64, vp]
    lib.cg_quality_trim_batch.argtypes = [vp, vp, vp, i64, i32, i32, i32, vp]
    lib.cg_nextseq_trim_batch.argtypes = [vp, vp, vp, vp, i64, i32, i32, vp]
    lib.cg_poly_a_trim_batch.argtypes = [vp, vp, vp, i64, i32, vp]
    lib.cg_expected_errors_batch.argtypes = [vp, vp, vp, i64, i32, vp]
    lib.cg_stats_size.argtypes = [i32, i32, i32]
    lib.cg_stats_size.restype = i64
    lib.cg_stats_accumulate_device.argtypes = [
        vp, vp, vp, vp, i64, C.POINTER(cg_params), vp, vp, i32, i32, vp,
    ]
    lib.cg_locate_debug.argtypes = [vp, C.POINTER(cg_adapter_desc), vp, i32, vp, vp, vp]
    lib.cg_process_batch_stats.argtypes = [vp, vp, vp, vp, vp, i64, C.POINTER(cg_params), vp, vp, i32, i32, vp]
    lib.cg_edit_environment.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp, i64]
    lib.cg_edit_environment.restype = i64
    lib.cg_hamming_environment.argtypes = [vp, i32, i32, i32, vp, vp, vp, i64]
    lib.cg_hamming_environment.restype = i64


def lib():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        with _lib_lock:
            if _lib is None:
                path = os.environ.get("CUTADAPT_B200_LIB", LIB_PATH)
                if not os.path.exists(path):
                    raise CutadaptB200Error(
                        f"{path} not found: build it with `python -c 'import __graft_entry__ as g; "
                        "g.build()'` (there is no CPU fallback)"
                    )
                handle = C.CDLL(path)
                _declare(handle)
                _lib = handle
    return _lib


_ERRORS = {
    CG_EINVAL: ValueError,
    CG_ENONASCII: ValueError,
    CG_ENOMEM: MemoryError,
    CG_ECUDA: CutadaptB200Error,
    CG_EUNSUPPORTED: CutadaptB200Error,
}


def last_error() -> str:
    message = lib().cg_last_error()
    return message.decode("utf-8", "replace") if message else ""


def check(rc: int) -> None:
    if rc >= 0:
        return
    message = lib().cg_last_error()
    text = message.decode("utf-8", "replace") if message else f"error {rc}"
    if rc == CG_ENOQUAL:
        from .qualtrim import HasNoQualities

        raise HasNoQualities(text)
    raise _ERRORS.get(rc, CutadaptB200Error)(text)


# ---- packing of Python strings into the batch layout ----------------------------------------


def pack_strings(strings: Sequence[str], what: str = "String") -> Tuple[np.ndarray, np.ndarray]:
    """
    Concatenate ASCII strings into one uint8 array + int64 offsets (n+1).
    Non-ASCII input raises ValueError like the reference's translate() (_align.pyx:44-45).
    """
    try:
        joined = "".join(strings).encode("ascii")
    except UnicodeEncodeError:
        raise ValueError(f"{what} must contain only ASCII characters") from None
    offsets = np.zeros(len(strings) + 1, dtype=np.int64)
    if len(strings):
        np.cumsum(np.fromiter((len(s) for s in strings), dtype=np.int64, count=len(strings)), out=offsets[1:])
    data = np.frombuffer(joined, dtype=np.uint8)
    if data.size == 0:
        data = np.zeros(1, dtype=np.uint8)
    return data, offsets


class AdapterSetSpec:
    """
    Plain-Python description of an adapter set: what cg_adapterset_create() consumes.
    ``adapters`` is a list of dicts with the fields of cg_adapter_desc (``sequence`` as str,
    ``kmer_entries`` as an (n,4) list / ``kmer_masks`` as uint64 array or None), ``groups`` a
    list of (type, a0, a1, front_required, back_required).  ``indexes`` (for CG_GROUP_INDEXED
    groups, whose a0 is the index number) is a list of dicts ``{"prefix": bool, "lengths": [...],
    "keys": [str], "adapter": [...], "errors": [...], "matches": [...]}`` = the dict an
    AdapterIndex builds (adapters.py:1416-1466).
    """

    def __init__(self, adapters: List[dict], groups: Optional[List[tuple]] = None,
                 indexes: Optional[List[dict]] = None):
        self.adapters = adapters
        self.indexes = indexes or []
        self.groups = groups if groups is not None else [
            (CG_GROUP_SINGLE, i, -1, 0, 0) for i in range(len(adapters))
        ]
        self._keep = []

    def to_ctypes(self):
        """Returns (adapter array, n, group array, n).  Keeps referenced buffers alive on self."""
        keep = []
        arr = (cg_adapter_desc * len(self.adapters))()
        for i, a in enumerate(self.adapters):
            try:
                seq = a["sequence"].encode("ascii")
            except UnicodeEncodeError:
                raise ValueError("String must contain only ASCII characters") from None
            keep.append(seq)
            d = arr[i]
            d.sequence = seq
            d.length = len(seq)
            d.max_error_rate = float(a["max_error_rate"])
            d.flags = int(a.get("flags", 15))
            d.wildcard_ref = int(bool(a.get("wildcard_ref", False)))
            d.wildcard_query = int(bool(a.get("wildcard_query", False)))
            d.indel_cost = int(a.get("indel_cost", 1))
            d.min_overlap = int(a.get("min_overlap", 1))
            d.kind = int(a.get("kind", CG_KIND_ALIGNER))
            d.reverse_read = int(bool(a.get("reverse_read", False)))
            d.remove = int(a.get("remove", CG_REMOVE_AFTER))
            entries = a.get("kmer_entries")
            if entries is not None and len(entries):
                ents = (cg_kmer_entry * len(entries))()
                for j, (start, stop, init, found) in enumerate(entries):
                    ents[j].search_start = start
                    ents[j].search_stop = stop
                    ents[j].init_mask = init
                    ents[j].found_mask = found
                masks = np.ascontiguousarray(a["kmer_masks"], dtype=np.uint64).reshape(-1)
                assert masks.size == 128 * len(entries)
                keep.extend([ents, masks])
                d.kmer_entries = ents
                d.kmer_masks = masks.ctypes.data_as(C.POINTER(C.c_uint64))
                d.n_kmer_entries = len(entries)
            else:
                d.kmer_entries = None
                d.kmer_masks = None
                d.n_kmer_entries = 0
        garr = (cg_group_desc * len(self.groups))()
        for i, (typ, a0, a1, freq, breq) in enumerate(self.groups):
            garr[i].type = typ
            garr[i].a0 = a0
            garr[i].a1 = a1
            garr[i].front_required = int(bool(freq))
            garr[i].back_required = int(bool(breq))
        self._keep = keep
        return arr, len(self.adapters), garr, len(self.groups)

    def index_ctypes(self):
        """Returns (cg_index_desc array or None, n)."""
        if not self.indexes:
            return None, 0
        keep = []
        iarr = (cg_index_desc * len(self.indexes))()
        for i, ix in enumerate(self.indexes):
            lengths = np.ascontiguousarray(ix["lengths"], dtype=np.int32)
            keys = ix["keys"]
            stride = max([len(k) for k in keys] + [1])
            buf = np.zeros((len(keys), stride), dtype=np.uint8)
            for j, k in enumerate(keys):
                buf[j, : len(k)] = np.frombuffer(k.encode("ascii"), dtype=np.uint8)
            ad = np.ascontiguousarray(ix["adapter"], dtype=np.int32)
            er = np.ascontiguousarray(ix["errors"], dtype=np.int32)
            ma = np.ascontiguousarray(ix["matches"], dtype=np.int32)
            keep.extend([lengths, buf, ad, er, ma])
            d = iarr[i]
            d.prefix = int(bool(ix["prefix"]))
            d.n_lengths = len(lengths)
            d.lengths = lengths.ctypes.data_as(C.POINTER(C.c_int32))
            d.n_keys = len(keys)
            d.keys = buf.ctypes.data
            d.stride = stride
            d.adapter = ad.ctypes.data_as(C.POINTER(C.c_int32))
            d.errors = er.ctypes.data_as(C.POINTER(C.c_int32))
            d.matches = ma.ctypes.data_as(C.POINTER(C.c_int32))
        self._keep_index = keep
        return iarr, len(self.indexes)

    @property
    def slots(self) -> int:
        return 2 if any(g[0] == CG_GROUP_LINKED for g in self.groups) else 1


def make_params(quality_trim=False, cutoff_front=0, cutoff_back=0, quality_base=33, times=1,
                nextseq_cutoff=None) -> cg_params:
    p = cg_params()
    p.nextseq_trim = int(nextseq_cutoff is not None)
    p.nextseq_cutoff = int(nextseq_cutoff or 0)
    p.quality_trim = int(bool(quality_trim))
    p.cutoff_front = int(cutoff_front)
    p.cutoff_back = int(cutoff_back)
    p.quality_base = int(quality_base)
    p.times = int(times)
    return p


# ---- context ---------------------------------------------------------------------------------


class cg_name_token(C.Structure):
    _fields_ = [("kind", C.c_int32), ("mate", C.c_int32), ("text", C.c_char_p), ("len", C.c_int32)]


class cg_names_desc(C.Structure):
    _fields_ = [("length_tag", C.c_char_p), ("strip_suffix", C.POINTER(C.c_char_p)), ("n_strip_suffix", C.c_int32),
                ("paired", C.c_int32), ("prefix", C.c_char_p), ("suffix", C.c_char_p),
                ("rename", C.POINTER(cg_name_token)), ("n_rename", C.c_int32)]


class Names:
    """A names handle on a context (cg_names_*): the read-name modifiers of the collects whose parameters name
    ``handle`` in ``names``.  tokens: the --rename template as (kind, mate, literal text) or None for no renamer."""

    def __init__(self, ctx: "Context", length_tag=None, strip_suffix=(), prefix="", suffix="", tokens=None,
                 paired=False):
        enc = lambda x: x.encode("latin-1")
        strips = (C.c_char_p * max(len(strip_suffix), 1))(*[enc(x) for x in strip_suffix])
        toks = (cg_name_token * max(len(tokens or ()), 1))()
        for i, (kind, mate, text) in enumerate(tokens or ()):
            toks[i].kind, toks[i].mate, toks[i].text, toks[i].len = kind, mate, enc(text), len(enc(text))
        d = cg_names_desc(enc(length_tag) if length_tag is not None else None, strips, len(strip_suffix), int(paired),
                          enc(prefix or ""), enc(suffix or ""), toks, -1 if tokens is None else len(tokens))
        h = C.c_int32(0)
        check(lib().cg_names_create(ctx.handle, C.byref(d), C.byref(h)))
        self.ctx, self.handle = ctx, h.value

    def set_mate(self, mate: int, names, linked, last_cut_front: int = 0, last_cut_back: int = 0) -> None:
        blobs = [n.encode("latin-1") for n in names]
        offsets = np.zeros(len(blobs) + 1, dtype=np.int32)
        offsets[1:] = np.cumsum([len(b) for b in blobs]) if blobs else []
        flags = np.array(linked, dtype=np.uint8).reshape(-1)
        check(lib().cg_names_set_mate(self.ctx.handle, self.handle, mate, b"".join(blobs), offsets.ctypes.data,
                                      len(blobs), flags.ctypes.data if flags.size else None, int(last_cut_front),
                                      int(last_cut_back)))

    def close(self) -> None:
        if self.handle:
            check(lib().cg_names_destroy(self.ctx.handle, self.handle))
            self.handle = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class FastqStatistics:
    """A statistics accumulator of the FASTQ path on a context (cg_fastq_stats_*): the collects whose parameters
    name ``handle`` in ``stats`` add their statistics to it."""

    def __init__(self, ctx: "Context", n_adapters: int):
        h = C.c_int32(0)
        check(lib().cg_fastq_stats_create(ctx.handle, int(n_adapters), C.byref(h)))
        self.ctx, self.handle, self.n_adapters = ctx, h.value, int(n_adapters)

    def read(self, reset: bool = False) -> Tuple[np.ndarray, int, int]:
        """(the int64 vector, max_len, kmax) of its current layout."""
        max_len, kmax, size = C.c_int32(), C.c_int32(), C.c_int64()
        check(lib().cg_fastq_stats_read(self.ctx.handle, self.handle, C.byref(max_len), C.byref(kmax), None, 0,
                                        C.byref(size), 0))
        out = np.zeros(size.value, dtype=np.int64)
        check(lib().cg_fastq_stats_read(self.ctx.handle, self.handle, C.byref(max_len), C.byref(kmax),
                                        out.ctypes.data, out.size, C.byref(size), int(reset)))
        return out, max_len.value, kmax.value

    def close(self) -> None:
        if self.handle:
            check(lib().cg_fastq_stats_destroy(self.ctx.handle, self.handle))
            self.handle = 0

    def __del__(self):
        # the accumulator keeps its context alive (self.ctx), so the handle is still valid here
        try:
            self.close()
        except Exception:
            pass



class Context:
    """One CUDA device + stream + staging buffers (cg_ctx).  Not thread-safe."""

    def __init__(self, device: Optional[int] = None, stream: Optional[int] = None):
        if device is None:
            device = int(os.environ.get("LOCAL_RANK", "0")) if "CUTADAPT_B200_DEVICE" not in os.environ \
                else int(os.environ["CUTADAPT_B200_DEVICE"])
        self.device = device
        handle = C.c_void_p()
        check(lib().cg_ctx_create(device, C.c_void_p(stream or 0), C.byref(handle)))
        self._h = handle

    @property
    def handle(self):
        return self._h

    def synchronize(self) -> None:
        check(lib().cg_ctx_synchronize(self._h))

    def launch_count(self) -> int:
        return int(lib().cg_ctx_launch_count(self._h))

    def kernel_time(self, reset: bool = False) -> Tuple[float, int]:
        total = C.c_double()
        launches = C.c_int64()
        check(lib().cg_ctx_kernel_time(self._h, C.byref(total), C.byref(launches), int(reset)))
        return total.value, launches.value

    def stage_times(self, reset: bool = False) -> dict:
        """ms per stage of the split pipeline (only recorded while CUTADAPT_B200_STAGE_TIMES is set)."""
        out = (C.c_double * 3)()
        check(lib().cg_ctx_stage_times(self._h, out, int(reset)))
        return {"first_stage_ms": out[0], "plan_ms": out[1], "dp_rounds_ms": out[2]}

    def host_profile(self, reset: bool = False) -> dict:
        """Seconds the host side of cg_process_batch spent per phase (cg_ctx_host_profile)."""
        out = (C.c_double * 8)()
        check(lib().cg_ctx_host_profile(self._h, out, int(reset)))
        return {"total_s": out[0], "offset_scan_s": out[1], "pack_s": out[2], "lane_wait_s": out[3],
                "drain_s": out[4], "chunks": int(out[5]), "packed_characters": int(out[6]),
                "pack_fraction": out[7]}

    def transfer_bytes(self, reset: bool = False) -> Tuple[int, int]:
        """Bytes cg_process_batch moved host->device and device->host on this context."""
        h2d, d2h = C.c_int64(), C.c_int64()
        check(lib().cg_ctx_transfer_bytes(self._h, C.byref(h2d), C.byref(d2h), int(reset)))
        return h2d.value, d2h.value

    def close(self) -> None:
        if self._h:
            lib().cg_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx = None
_default_pid = None


def default_context() -> Context:
    """Process-wide context (one per process, re-created after fork)."""
    global _default_ctx, _default_pid
    if _default_ctx is None or _default_pid != os.getpid():
        _default_ctx = Context()
        _default_pid = os.getpid()
    return _default_ctx


class AdapterSet:
    """Compiled adapter tables resident on the device (cg_adapterset)."""

    def __init__(self, spec: AdapterSetSpec, ctx: Optional[Context] = None):
        self.spec = spec
        self.ctx = ctx or default_context()
        arr, n, garr, ng = spec.to_ctypes()
        handle = C.c_void_p()
        iarr, ni = spec.index_ctypes()
        if ni:
            check(lib().cg_adapterset_create_indexed(self.ctx.handle, arr, n, garr, ng, iarr, ni, C.byref(handle)))
        else:
            check(lib().cg_adapterset_create(self.ctx.handle, arr, n, garr, ng, C.byref(handle)))
        self._h = handle
        self.slots = int(lib().cg_adapterset_slots(handle))

    @property
    def handle(self):
        return self._h

    def jit_status(self) -> int:
        """1: a first-stage kernel specialised for this set is in use, 0: not (yet), -1: its compilation failed
        (the precompiled kernel runs; last_error() says why)."""
        return int(lib().cg_adapterset_jit_status(self._h))

    def jit_source(self, plane_words: int = 5, has_qual: bool = False, statistics: bool = False) -> str:
        """The translation unit the run-time specialisation compiles for this set ('' if it has no plane program);
        statistics=True: the variant that counts the trim statistics inside the first stage (run_with_statistics)."""
        n = int(lib().cg_adapterset_jit_source(self._h, plane_words, int(has_qual), int(statistics), None, 0))
        if n == 0:
            return ""
        buf = C.create_string_buffer(n + 1)
        lib().cg_adapterset_jit_source(self._h, plane_words, int(has_qual), int(statistics), buf, n + 1)
        return buf.value.decode()

    def effective_length(self, adapter: int = 0) -> int:
        out = C.c_int32()
        check(lib().cg_adapterset_effective_length(self._h, adapter, C.byref(out)))
        return out.value

    def process(
        self,
        seq: np.ndarray,
        offsets: np.ndarray,
        qual: Optional[np.ndarray] = None,
        params: Optional[cg_params] = None,
        want_qtrim: bool = False,
    ):
        """Run the fused pass on host arrays; returns (matches[n, times, slots], qtrim[n,2] or None)."""
        params = params or make_params()
        n = int(offsets.size - 1)
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        if (params.quality_trim or params.nextseq_trim) and qual is None:
            from .qualtrim import HasNoQualities

            raise HasNoQualities("Cannot do quality trimming when no qualities are available")
        if qual is not None:
            qual = np.ascontiguousarray(qual, dtype=np.uint8)
        times = max(1, params.times)
        matches = np.empty((n, times, self.slots), dtype=MATCH_DTYPE)
        qtrim = np.empty((n, 2), dtype=np.int32) if (want_qtrim or params.quality_trim or params.nextseq_trim) else None
        if n:
            check(
                lib().cg_process_batch(
                    self.ctx.handle, self._h, seq.ctypes.data, qual.ctypes.data if qual is not None else None,
                    offsets.ctypes.data, n, C.byref(params), matches.ctypes.data,
                    qtrim.ctypes.data if qtrim is not None else None,
                )
            )
        return matches, qtrim

    def close(self) -> None:
        if getattr(self, "_h", None):
            try:
                lib().cg_adapterset_destroy(self._h)
            finally:
                self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
