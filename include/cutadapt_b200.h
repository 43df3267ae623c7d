/*
 * cutadapt_b200.h -- C ABI of the H100-native adapter-trimming core.
 *
 * Drop-in boundary for ONE hot path of marcelm/cutadapt:
 *     Adapter.match_to -> KmerFinder.kmers_present -> Aligner.locate   (+ quality_trim_index)
 * batched per chunk of reads.  Every entry point below states which reference interface it
 * replaces (file:line relative to the reference checkout).  Plain C types only: no torch,
 * no C++ types, no Python objects cross this boundary.  The Python host layer
 * (the modules of cutadapt_b200) binds it with ctypes; INTEGRATION.md shows the stub a cutadapt
 * maintainer would add.
 *
 * Conventions
 *   - every function returns CG_OK (0) or a negative CG_E* code; the message for the last
 *     failing call on the calling thread is returned by cg_last_error().
 *   - "no match" is never an error: it is reported as adapter == -1 in cg_match.
 *   - the caller owns all host buffers; the library owns device memory inside a cg_ctx.
 *   - a cg_ctx is bound to one CUDA device and one stream and is NOT thread-safe
 *     (mirrors "one Aligner per process", _align.pyx:172: the DP column is per-instance).
 *   - there is no CPU fallback: without a usable CUDA device cg_ctx_create fails.
 */
#ifndef CUTADAPT_B200_H
#define CUTADAPT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CG_ABI_VERSION 1

/* ---- status codes --------------------------------------------------------------------- */
#define CG_OK 0
#define CG_EINVAL (-1)    /* bad argument: the reference raises ValueError/TypeError            */
#define CG_ENONASCII (-2) /* non-ASCII byte in a read/adapter (_align.pyx:44-45, _kmer_finder.pyx:182-183) */
#define CG_ECUDA (-3)     /* CUDA runtime error                                                  */
#define CG_ENOMEM (-4)    /* host or device allocation failed (_align.pyx:252-256 MemoryError)   */
#define CG_EUNSUPPORTED (-5) /* configuration outside what the kernels implement (message says which) */
#define CG_ENOQUAL (-6)   /* quality trimming requested without qualities (qualtrim.pyx:35-36 HasNoQualities) */

/* ---- Aligner flags: EndSkip (src/cutadapt/align.py:24-34) ------------------------------ */
#define CG_START_IN_REFERENCE 1
#define CG_START_IN_QUERY 2
#define CG_STOP_IN_REFERENCE 4
#define CG_STOP_IN_QUERY 8

/* ---- what locates the adapter (adapters.py:601-614 vs 1031-1041,1068-1078) ------------- */
#define CG_KIND_ALIGNER 0        /* Aligner.locate            (_align.pyx:298-587) */
#define CG_KIND_PREFIX_COMPARER 1 /* PrefixComparer.locate     (_align.pyx:651-693) */
#define CG_KIND_SUFFIX_COMPARER 2 /* SuffixComparer.locate     (_align.pyx:708-714) */

/* ---- which Match class wraps the alignment (adapters.py:427-493, 925-935) -------------- */
#define CG_REMOVE_BEFORE 0   /* RemoveBeforeMatch: 5' adapters, keep read[rstop:]      */
#define CG_REMOVE_AFTER 1    /* RemoveAfterMatch:  3' adapters, keep read[:rstart]     */
#define CG_REMOVE_AUTO 2     /* AnywhereAdapter: BEFORE iff rstart == 0 else AFTER      */

/* ---- composition of adapters (adapters.py:1181-1286) ----------------------------------- */
#define CG_GROUP_SINGLE 0   /* one SingleAdapter                                            */
#define CG_GROUP_LINKED 1   /* LinkedAdapter(front=a0, back=a1)   adapters.py:1215-1227      */
#define CG_GROUP_INDEXED 2  /* IndexedPrefixAdapters / IndexedSuffixAdapters (adapters.py:1289-1571):
                               a0 = index number in the cg_index_desc array                    */

typedef struct cg_ctx cg_ctx;               /* device, stream, staging buffers            */
typedef struct cg_adapterset cg_adapterset; /* immutable compiled adapter tables on device */

/* One search word of a KmerFinder, exactly the reference's KmerSearchEntry
 * (_kmer_finder.pyx:58-63) minus mask_offset: the 128 x uint64 needle-mask table of entry e
 * is masks[128*e .. 128*e+127] (_kmer_finder.pyx:153-154, 226-238). */
typedef struct cg_kmer_entry {
    int64_t search_start; /* negative = relative to the end of the read                     */
    int64_t search_stop;  /* 0 = up to the end; negative = relative to the end               */
    uint64_t init_mask;   /* one bit at the first character of every packed k-mer           */
    uint64_t found_mask;  /* one bit at the last character of every packed k-mer            */
} cg_kmer_entry;

/* One SingleAdapter = the arguments of Aligner.__cinit__ (_align.pyx:195-204) or
 * PrefixComparer.__init__ (_align.pyx:615-622) plus its KmerFinder tables and the few
 * attributes adapters.py needs to build the Match (adapters.py:564-599, 684-1089). */
typedef struct cg_adapter_desc {
    const uint8_t *sequence;  /* adapter as given to the aligner (ASCII; already reversed
                                 for Rightmost* adapters, adapters.py:746-750,849-854)      */
    int32_t length;           /* m                                                          */
    double max_error_rate;
    int32_t flags;            /* CG_START_IN_* / CG_STOP_IN_* bits (aligner only)           */
    int32_t wildcard_ref;     /* IUPAC characters in the adapter are wildcards              */
    int32_t wildcard_query;   /* IUPAC characters in the read are wildcards                 */
    int32_t indel_cost;       /* 1, or 100000 for --no-indels (adapters.py:605)             */
    int32_t min_overlap;
    int32_t kind;             /* CG_KIND_*                                                  */
    int32_t reverse_read;     /* 1: match against the reversed read and mirror the
                                 coordinates back (adapters.py:766-786, 870-890)            */
    int32_t remove;           /* CG_REMOVE_*                                                */
    const cg_kmer_entry *kmer_entries; /* NULL / 0 entries = MockKmerFinder (adapters.py:29-31) */
    const uint64_t *kmer_masks;        /* 128 * n_kmer_entries words                        */
    int32_t n_kmer_entries;
    int32_t reserved;
} cg_adapter_desc;

/* One Matchable in MultipleAdapters order (adapters.py:1265-1286). */
typedef struct cg_group_desc {
    int32_t type;            /* CG_GROUP_*                                                  */
    int32_t a0;              /* adapter index (SINGLE) / front adapter (LINKED)             */
    int32_t a1;              /* back adapter (LINKED), else -1                              */
    int32_t front_required;  /* LINKED only                                                 */
    int32_t back_required;   /* LINKED only                                                 */
    int32_t reserved[3];
} cg_group_desc;

/* The dict of an AdapterIndex (adapters.py:1416-1466), built on the host with
 * cg_edit_environment / cg_hamming_environment: every key is an ACGT string of at most 32
 * characters that maps to (adapter, errors, matches).  `lengths` are the distinct key lengths in
 * descending order (AdapterIndex._lengths).  The device keeps it as an open-addressing hash table in
 * HBM; lookups follow _match_to_one_length/_match_to_multiple_lengths/_lookup_with_n
 * (adapters.py:1474-1551) exactly. */
typedef struct cg_index_desc {
    int32_t prefix;            /* 1: IndexedPrefixAdapters, 0: IndexedSuffixAdapters            */
    int32_t n_lengths;
    const int32_t *lengths;
    int64_t n_keys;
    const uint8_t *keys;       /* n_keys strings, `stride` bytes apart, NUL padded                */
    int32_t stride;
    int32_t reserved;
    const int32_t *adapter;    /* per key: index into the adapter array                          */
    const int32_t *errors;
    const int32_t *matches;
} cg_index_desc;

/* Per-batch parameters of the fused pass (modifiers.py:825-858 then 200-261). */
typedef struct cg_params {
    int32_t quality_trim;    /* 0 = off; 1 = run quality_trim_index first and search read[start:stop] */
    int32_t cutoff_front;
    int32_t cutoff_back;
    int32_t quality_base;    /* 33 or 64                                                     */
    int32_t times;           /* AdapterCutter(times=...) rounds, >= 1 (modifiers.py:225-231) */
    int32_t nextseq_trim;    /* 1 = NextseqQualityTrimmer first (modifiers.py:825-837, cli.py:940-945):
                                the read is cut at nextseq_trim_index(read, nextseq_cutoff, quality_base)
                                before quality_trim_index (if enabled) runs on what is left               */
    int32_t nextseq_cutoff;
    int32_t reserved;
} cg_params;

/* One match record (32 bytes).  For round r of read i the records are at
 *     out[(i * times + r) * slots + s],  slots = cg_adapterset_slots(set)
 * s = 0 for single adapters; LINKED groups use s = 0 (front) and s = 1 (back), either of
 * which may be absent (adapter == -1) while the other is present.
 * Coordinates are those of SingleMatch (adapters.py:334-356): relative to the sequence
 * that was searched in that round (after quality trimming and earlier rounds). */
typedef struct cg_match {
    int32_t adapter; /* index into the adapter array, -1 = no match                         */
    int32_t astart, astop;
    int32_t rstart, rstop;
    int32_t score, errors;
    int32_t info;    /* bits 0..7: group index; bit 8: RemoveBefore(0)/RemoveAfter(1);
                        bits 16..31: length of the sequence that was searched (mod 65536)   */
} cg_match;

/* ---- library ---------------------------------------------------------------------------- */
int cg_version(void);
const char *cg_last_error(void);

/* ---- context ---------------------------------------------------------------------------- */
/* device: CUDA ordinal.  stream: a cudaStream_t to run on (e.g. torch's current stream),
 * or NULL to let the context create its own. */
int cg_ctx_create(int device, void *stream, cg_ctx **out);
int cg_ctx_destroy(cg_ctx *ctx);
int cg_ctx_synchronize(cg_ctx *ctx);
/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
int64_t cg_ctx_launch_count(cg_ctx *ctx);
/* Average device time in ms of the fused trimming kernel since the last reset, measured with
 * CUDA events on the launching stream; launches = number of samples. */
int cg_ctx_kernel_time(cg_ctx *ctx, double *total_ms, int64_t *launches, int reset);
/* Device time (ms) of the three stages of the split pipeline -- first stage, plan, DP rounds -- since the last reset;
 * recorded only while CUTADAPT_B200_STAGE_TIMES is set in the environment (measurement aid, no reference counterpart). */
int cg_ctx_stage_times(cg_ctx *ctx, double *out3, int reset);

/* Bytes cg_process_batch has copied host->device / device->host on this context so far (what actually
 * crossed PCIe: the compressed read stream + exceptions, qualities, irregular offsets; the records back). */
int cg_ctx_transfer_bytes(cg_ctx *ctx, int64_t *h2d, int64_t *d2h, int reset);

/* CPUs this process may use (affinity mask, cut down by a cgroup CPU quota) and the number of worker
 * threads the library's host side will start (CUTADAPT_B200_HOST_THREADS overrides). */
int cg_host_cpus_available(void);
int cg_host_threads(void);
/* NUMA node the context's worker threads were bound to (the node holding the first packed read buffer), -1 = none */
int cg_ctx_numa_node(cg_ctx *ctx);

/* Where the host side of cg_process_batch spent its time, in seconds, accumulated over calls:
 * out[0] total, [1] scanning the offsets, [2] packing reads for the compressed transfer, [3] waiting for a
 * free lane (= the device or PCIe is the bottleneck), [4] draining the lanes at the end, [5] chunks,
 * [6] characters sent compressed, [7] the current compressed share of a chunk; out must hold 8 doubles. */
int cg_ctx_host_profile(cg_ctx *ctx, double *out, int reset);

/* ---- adapter set (replaces Aligner.__cinit__/_set_reference _align.pyx:195-277 and
 *      KmerFinder.__cinit__ _kmer_finder.pyx:106-165 for every adapter at once) ----------- */
int cg_adapterset_create(cg_ctx *ctx, const cg_adapter_desc *adapters, int32_t n_adapters,
                         const cg_group_desc *groups, int32_t n_groups, cg_adapterset **out);
/* Same, with anchored-adapter indexes for CG_GROUP_INDEXED groups. */
int cg_adapterset_create_indexed(cg_ctx *ctx, const cg_adapter_desc *adapters, int32_t n_adapters,
                                 const cg_group_desc *groups, int32_t n_groups,
                                 const cg_index_desc *indexes, int32_t n_indexes, cg_adapterset **out);
/* Aligner.enable_debug() / .dpmatrix / .scorematrix (_align.pyx:279-296): the dynamic-programming matrices of ONE
 * read against ONE aligner adapter as the search fills them -- (m + 1) x (n + 1) int32 each, row-major, CG_DEBUG_NONE
 * where a cell was never computed (outside the Ukkonen band or after the early exit).  result8 = found (0/1) and the
 * six numbers of Aligner.locate().  A triage aid (one device thread, exact cells, no prefilter). */
#define CG_DEBUG_NONE (-2147483647 - 1)
int cg_locate_debug(cg_ctx *ctx, const cg_adapter_desc *adapter, const uint8_t *query, int32_t n,
                    int32_t *cost, int32_t *score, int32_t *result8);

int cg_adapterset_destroy(cg_adapterset *set);

/* Run-time specialisation of the bit-plane first stage for this adapter set (compiled with NVRTC once the set has
 * processed a few million reads; CUTADAPT_B200_JIT=1 at once, =0 never).  1 = in use, 0 = not (yet), -1 = the
 * compilation failed and the precompiled kernel keeps running (cg_last_error() then says why).  There is no
 * counterpart in the reference; results do not depend on it. */
int cg_adapterset_jit_status(const cg_adapterset *set);
/* The generated translation unit (for inspection).  Returns its length; copies at most cap - 1 characters. */
int64_t cg_adapterset_jit_source(const cg_adapterset *set, int32_t plane_words, int32_t has_qual, int32_t stats,
                                 char *buf, int64_t cap);
int cg_adapterset_slots(const cg_adapterset *set); /* 1, or 2 if any group is LINKED */
/* Aligner.effective_length / PrefixComparer.effective_length (_align.pyx:188,268-271,626-630) */
int cg_adapterset_effective_length(const cg_adapterset *set, int32_t adapter, int32_t *out);

/* ---- the batched hot path ---------------------------------------------------------------
 * Replaces, for a whole chunk of reads, the per-read loop
 *     QualityTrimmer.__call__ (modifiers.py:853-858) -> quality_trim_index (qualtrim.pyx:22-73)
 *     AdapterCutter.match_and_trim (modifiers.py:225-231)
 *       -> MultipleAdapters.match_to (adapters.py:1265-1286)
 *         -> <Adapter>.match_to (adapters.py:707-724, 815-832, ...)
 *           -> KmerFinder.kmers_present (_kmer_finder.pyx:170-213)
 *           -> Aligner.locate (_align.pyx:298-587)
 *
 * Layout: read i occupies seq[offsets[i] .. offsets[i+1]) (and the same range of qual).
 *   matches : n_reads * times * slots records
 *   qtrim   : 2 * n_reads int32 (start, stop) of quality_trim_index; may be NULL
 *
 * cg_process_batch: HOST pointers (pageable or pinned); the library overlaps H2D / kernels / D2H in
 *   sub-batches on its streams.  Batches of >= 65536 reads travel partly compressed: worker threads of the
 *   library (CUTADAPT_B200_HOST_THREADS; default: the CPUs the process may use, cgroup quota included, at
 *   most 32) pack reads three characters per byte (A C G T N; every other byte goes verbatim into an
 *   exception list) and a device kernel restores the caller's bytes exactly, so results do not depend on
 *   it.  The share of each chunk that is packed follows a feedback rule (pack more while PCIe is the
 *   bottleneck, less while the host threads are); CUTADAPT_B200_H2D_PACK=0 sends raw bytes only, =all
 *   compresses everything.
 * cg_process_batch_device: DEVICE pointers (16-byte aligned seq/qual, readable up to the next
 *   16-byte boundary past offsets[n_reads]); runs asynchronously on the context stream.
 *   max_read_len must be >= the longest read in the batch (pass 0 to let the library
 *   compute it with a reduction kernel).
 */
int cg_process_batch(cg_ctx *ctx, const cg_adapterset *set, const uint8_t *seq,
                     const uint8_t *qual, const int64_t *offsets, int64_t n_reads,
                     const cg_params *params, cg_match *matches, int32_t *qtrim);
int cg_process_batch_device(cg_ctx *ctx, const cg_adapterset *set, const uint8_t *d_seq,
                            const uint8_t *d_qual, const int64_t *d_offsets, int64_t n_reads,
                            int32_t max_read_len, const cg_params *params, cg_match *d_matches,
                            int32_t *d_qtrim);
/* The same plus the statistics of these reads ADDED to d_stats (int64[cg_stats_size(n_adapters, stats_max_len,
 * stats_kmax)], device memory; what cg_stats_accumulate_device computes from the records, bit for bit).  For a set
 * of one plain adapter, one round, no quality trimming and stats_max_len <= 4096 the split pipeline counts the reads
 * its first stage settles while they are in shared memory (a variant of that kernel compiled with the statistics
 * code) and the rest from its task list, so the records are not read back; otherwise the statistics kernel runs after
 * the pass.
 * With quality trimming d_qtrim is required. */
int cg_process_batch_device_stats(cg_ctx *ctx, const cg_adapterset *set, const uint8_t *d_seq, const uint8_t *d_qual,
                                  const int64_t *d_offsets, int64_t n_reads, int32_t max_read_len, const cg_params *params,
                                  cg_match *d_matches, int32_t *d_qtrim, int32_t stats_max_len, int32_t stats_kmax,
                                  int64_t *d_stats);

/* The host half of that compressed transfer, callable without a device (tests): packs the characters
 * at absolute positions a0 .. a0 + 3 * n_stream of `seq` (positions outside [lo, hi) are not read and
 * count as 'A') into n_stream bytes, base 6, first character most significant; writes up to `capacity`
 * exceptions (position - a0) << 8 | byte and returns how many there are. */
int64_t cg_pack3_host(const uint8_t *seq, int64_t a0, int64_t lo, int64_t hi, int64_t n_stream,
                      uint8_t *packed, uint64_t *exceptions, int64_t capacity, int32_t n_threads);

/* ---- stand-alone batched versions of the native functions -------------------------
 * KmerFinder.kmers_present (_kmer_finder.pyx:170-213): out[i] = 1/0.  Host pointers. */
int cg_kmers_present_batch(cg_ctx *ctx, const cg_kmer_entry *entries, const uint64_t *masks,
                           int32_t n_entries, const uint8_t *seq, const int64_t *offsets,
                           int64_t n_reads, uint8_t *out);
/* quality_trim_index (qualtrim.pyx:22-73): out[2i], out[2i+1] = start, stop.  Host pointers. */
int cg_quality_trim_batch(cg_ctx *ctx, const uint8_t *qual, const int64_t *offsets,
                          int64_t n_reads, int32_t cutoff_front, int32_t cutoff_back,
                          int32_t base, int32_t *out);
/* nextseq_trim_index (qualtrim.pyx:76-117; NextseqQualityTrimmer, modifiers.py:825-837): out[i] = the
 * index at which read i is cut at its 3' end ('G' counted as quality cutoff - 1).  Host pointers. */
int cg_nextseq_trim_batch(cg_ctx *ctx, const uint8_t *seq, const uint8_t *qual, const int64_t *offsets,
                          int64_t n_reads, int32_t cutoff, int32_t base, int32_t *out);
/* expected_errors (qualtrim.pyx:172-197; expected_errors.h:95-140): out[i] = the FP64 sum of 10^(-q/10)
 * over read i's qualities, accumulated in the reference's order (bit-identical doubles); -1.0 marks a
 * quality character outside [base, 126] (the reference raises ValueError).  Host pointers. */
int cg_expected_errors_batch(cg_ctx *ctx, const uint8_t *qual, const int64_t *offsets, int64_t n_reads,
                             int32_t base, double *out);
/* poly_a_trim_index (qualtrim.pyx:120-169; PolyATrimmer, modifiers.py:861-918): out[i] = start of the
 * poly-A tail of read i, or with revcomp != 0 the end of its poly-T head.  Host pointers. */
int cg_poly_a_trim_batch(cg_ctx *ctx, const uint8_t *seq, const int64_t *offsets, int64_t n_reads,
                         int32_t revcomp, int32_t *out);

/* ---- FASTQ chunks in, trimmed FASTQ out (SURVEY.md section 8(f) N1) ---------------------------------
 * The per-chunk worker of the reference as one call: WorkerProcess.run (runners.py:174-214) parses a chunk of
 * complete 4-line records (dnaio.read_chunks, runners.py:116-126), runs the modifiers per read
 * (pipeline.py:47-73, in the order cli.py:937-975 builds them: UnconditionalCutter, NextseqQualityTrimmer,
 * QualityTrimmer, AdapterCutter with its action, PolyATrimmer, Shortener, NEndTrimmer, ZeroCapper), the filters
 * (TooShort, TooLong, TooManyN, TooManyExpectedErrors, TooHighAverageErrorRate, CasavaFiltered, then DiscardTrimmed /
 * DiscardUntrimmed: predicates.py:29-160 in the order of cli.py:700-830) and formats the surviving records
 * ("@name\nsequence\n+\nqualities\n", SingleEndSink steps.py:299-319).  Here the chunk is indexed, packed,
 * trimmed, filtered and formatted on the device; it crosses PCIe once in each direction.
 * "\r\n" line ends are accepted (and written back as "\n", like dnaio). */
/* What AdapterCutter does with a read that has matches (modifiers.py:175-249) */
#define CG_ACTION_TRIM 0       /* remove the adapters (default)                                            */
#define CG_ACTION_NONE 1       /* leave the read as it is (matches still drive --discard-(un)trimmed)       */
#define CG_ACTION_MASK 2       /* N outside the part that would remain                                      */
#define CG_ACTION_LOWERCASE 3  /* whole read upper case, lower case outside the part that would remain      */
#define CG_ACTION_RETAIN 4     /* trim but keep the adapter itself (times must be 1)                        */
#define CG_ACTION_CROP 5       /* keep only the matched part read[rstart:rstop] (times must be 1)           */
typedef struct cg_fastq_params {
    cg_params trim;
    int32_t minimum_length;      /* -m; 0 = off                                                       */
    int32_t maximum_length;      /* -M; negative = off                                                */
    int32_t discard_trimmed;     /* --discard-trimmed                                                 */
    int32_t discard_untrimmed;   /* --discard-untrimmed                                               */
    double max_n;                /* --max-n; negative = off; below 1: proportion of the read length   */
    double max_expected_errors;  /* --max-ee; negative = off                                          */
    int32_t cut_front, cut_back; /* -u N / -u -N (UnconditionalCutter, modifiers.py:66-95): bases removed from
                                    the 5' / 3' end before anything else; both >= 0                    */
    int32_t poly_a;              /* --poly-a (PolyATrimmer, modifiers.py:861-879), after the adapters */
    int32_t shorten;             /* 1 = --length given (Shortener, modifiers.py:882-899) ...          */
    int32_t shorten_length;      /* ... its value: >= 0 keeps read[:L], < 0 keeps read[L:]            */
    int32_t trim_n;              /* --trim-n (NEndTrimmer, modifiers.py:902-918)                      */
    int32_t discard_casava;      /* --discard-casava (CasavaFiltered, predicates.py:125-139)          */
    int32_t action;              /* CG_ACTION_*: --action of the AdapterCutter (modifiers.py:236-249)   */
    int32_t revcomp;             /* --revcomp.  Single-end collects (ReverseComplementer, modifiers.py:264-308): the
                                    adapters are searched on the read and on its reverse complement, the better
                                    orientation is kept.  Paired collects (PairedReverseComplementer, modifiers.py:
                                    311-400; both mates' values must be equal, not with --pair-adapters): each mate's
                                    set also runs on the other mate's read, and a pair whose swapped matches score
                                    strictly more is written swapped (R1's output gets r2 trimmed by the -a set, R2's
                                    gets r1 trimmed by the -A set); no info rows then.  1 = append " rc" to the name
                                    of a replaced read (both mates of a swapped pair), 2 = do not (--rename given,
                                    cli.py:1082-1116)                                                   */
    int32_t format;              /* CG_FORMAT_*: what the chunk is and what is written (below); 0 = FASTQ    */
    int32_t stats;               /* 0 = off, else a handle of cg_fastq_stats_create: the call ADDS this mate's
                                    statistics to that accumulator if it succeeds (cg_fastq_stats_read, below) */
    int32_t gzip_outputs;        /* CG_GZIP_MAIN / CG_REDIRECT_* bits: the outputs written as gzip (below); 0 = plain */
    double max_average_error_rate; /* --max-aer (TooHighAverageErrorRate, predicates.py:74-95): a read of length > 0 is
                                    removed when expected errors / length > this rate (FP64); 0 = off, else it must lie
                                    in (0, 1).  Its count: cg_fastq_result.too_high_average_error_rate          */
    int32_t zero_cap;            /* -z / --zero-cap (ZeroCapper, modifiers.py:806-822), the last modifier: quality
                                    characters below trim.quality_base become trim.quality_base, for the filters and in
                                    every output; info rows of reads with a match keep the original qualities.  0 / 1 */
    int32_t names;               /* 0 = off, else a handle of cg_names_create (below): the read-name modifiers
                                    (--length-tag, --strip-suffix, -x / -y, --rename) run on this mate's records.  Both
                                    mates of a paired collect must give the same handle.  Without it a collect launches
                                    exactly what it launches with 0 here. */
} cg_fastq_params;
typedef struct cg_fastq_result {
    int64_t n_records, n_written;
    int64_t bp_in, bp_out;       /* bases read / bases written                                        */
    int64_t out_bytes;           /* size of the formatted output                                      */
    int64_t with_adapters, quality_trimmed_bp;
    int64_t too_short, too_long, too_many_n, too_many_expected_errors, discarded, casava_filtered;
    int64_t reverse_complemented; /* --revcomp: reads replaced by their reverse complement; pairs: the swapped
                                     pairs, in both mates' results                                      */
    int64_t out_bytes_plain;     /* size of the same outputs uncompressed (== out_bytes without gzip outputs) */
    int64_t too_high_average_error_rate; /* reads (pairs) removed by --max-aer                               */
} cg_fastq_result;
/* Formats (cg_fastq_params.format; both mates of a pair must have the same one, else CG_EINVAL):
 *   CG_FORMAT_FASTQ           FASTQ in, FASTQ out (zeroed parameters)
 *   CG_FORMAT_FASTA           FASTA in, FASTA out
 *   CG_FORMAT_FASTQ_TO_FASTA  FASTQ in, FASTA out (what the reference writes to a .fasta / .fa path or with --fasta,
 *                             files.py:238-285, cli.py:925-931)
 * A FASTA chunk is a sequence of records: a header line that starts with '>' (the name is the rest of the line)
 * followed by any number of sequence lines, which are joined without separator; a record may have no sequence line
 * at all (">a\n>b\n" is two empty reads).  Lines end in "\n" or "\r\n", the last one may lack its terminator.  Lines
 * that start with '#' in front of the first header are comments and are skipped (a chunk of comments alone holds no
 * record).  Rejected with CG_EINVAL, the message naming the line (1-based, within the chunk): any other line in front
 * of the first header (an empty one included), and a '#' line after the first header (the reference's test vectors
 * do not say what dnaio does with it).  A chunk must start at a header or at those comments.  FASTA has no qualities:
 * with CG_FORMAT_FASTA, quality_trim, nextseq_trim, max_expected_errors >= 0, max_average_error_rate != 0 and zero_cap are
 * CG_EINVAL (the reference's CLI drops --max-ee and --max-aer with a warning, cli.py:756-776; that is the caller's
 * decision), the info-file rows have empty quality
 * columns (adapters.py:408-415, steps.py:250).  FASTA output is ">name\nsequence\n", the sequence on one line.  It can
 * be LARGER than the input: a record without sequence line (">a" plus a line break) is written as ">a\n\n", so the
 * output of a FASTA chunk is at most 1.5 x its size plus 2 bytes; FASTQ -> FASTA output is never larger than the
 * FASTQ bound below. */
#define CG_FORMAT_FASTQ 0
#define CG_FORMAT_FASTA 1
#define CG_FORMAT_FASTQ_TO_FASTA 2
/* set may be NULL: quality trimming and filters only.  fastq / out: HOST pointers (pinned or pageable).
 * Errors: CG_EINVAL for malformed FASTQ (message names the record) or FASTA (names the line), a too small output buffer (out_bytes in
 * *res says what is needed), CG_ENONASCII like cg_process_batch. */
int cg_fastq_trim_chunk(cg_ctx *ctx, const cg_adapterset *set, const uint8_t *fastq, int64_t n_bytes,
                        const cg_fastq_params *params, uint8_t *out, int64_t out_capacity, cg_fastq_result *res);
/* The same in two halves so that the upload of the next chunk overlaps the download of this one (two slots):
 * submit starts the upload and the line index; collect does the rest and returns the output. */
int cg_fastq_submit(cg_ctx *ctx, const uint8_t *fastq, int64_t n_bytes, int32_t *slot);
int cg_fastq_collect(cg_ctx *ctx, int32_t slot, const cg_adapterset *set, const cg_fastq_params *params,
                     uint8_t *out, int64_t out_capacity, cg_fastq_result *res);

/* gzip input, inflated on the device.  A stream per input file (cg_gzin_create) keeps on the device the plain bytes
 * that do not yet form a whole record (the carry) and counts the compressed bytes consumed, so that errors can name an
 * offset in the file.  cg_fastq_submit_gzip takes the next compressed bytes of the file (host memory, starting at a
 * member boundary), uploads them, inflates every whole member they hold (zero bytes after a member are skipped), appends
 * the plain bytes to the carry and cuts the longest prefix of whole records into a slot -- the rules of read_fastq_chunks
 * / read_fasta_chunks (format CG_FORMAT_FASTQ_TO_FASTA cuts as FASTQ).  The caller passes the bytes not consumed again,
 * in front of the next ones.  No whole record yet: no slot is taken, *slot = -1.  final: every byte must be consumed and
 * the carry becomes the last chunk, which may lack its final newline.  The slot is indistinguishable from cg_fastq_submit
 * of the same plain bytes: every collect accepts it.
 * Errors: CG_EINVAL for what Python's gzip module rejects (the message names the byte offset of the bad member in the
 * file; no slot is taken and the stream is unchanged); CG_EUNSUPPORTED when not even one member fits under the 2 GiB
 * plain-size limit of a submission (the chain otherwise stops early to stay under it; `consumed` says where).  The
 * paired call's messages name the mate (first or second input). */
typedef struct cg_gzin_result {
    int64_t consumed;      /* compressed bytes of whole members (and the zeros behind them) used */
    int64_t members;       /* members inflated */
    int64_t plain_bytes;   /* their plain bytes */
    int64_t chunk_bytes;   /* bytes of the chunk in the slot (0 without a slot) */
    int64_t carry_bytes;   /* plain bytes kept for the next submission */
    int64_t n_records;     /* records of the chunk (pairs count two) */
    int64_t in_member;     /* split streams: 1 when `consumed` stopped inside a member (else 0) */
    int64_t respeculated;  /* split streams: chunks decoded again because their speculative start was wrong */
} cg_gzin_result;
int cg_gzin_create(cg_ctx *ctx, int32_t *handle);
/* cg_gzin_create with flags.  CG_GZIN_SPLIT_MEMBERS: a member that runs past the bytes given, or that is longer than
 * CG_GZIN_LONG_MEMBER compressed bytes, is inflated block-parallel (speculative block starts every CG_GZIN_STRIDE
 * compressed bytes, back-references into the unknown window resolved afterwards) and may be consumed in part: then
 * `consumed` stops at a deflate block boundary inside it and in_member is 1.  The stream keeps the bit offset into the
 * first byte passed again, the member's last 32 KiB of plain bytes, its running CRC-32 and length, and its offset in
 * the file; the caller still passes the unconsumed bytes again.  Such a member may exceed 2 GiB (it streams over
 * submissions); CG_EUNSUPPORTED remains for a stretch of deflate blocks that alone reaches the limit.  Every other
 * member, and every result field, is as on a default stream.  Any other flag bit is CG_EINVAL.
 * The environment variable CUTADAPT_B200_GZIN_STRIDE, read when a split stream is created, replaces CG_GZIN_STRIDE
 * (in bytes, at least 32 KiB) for that stream; tools/measure_fastq.py --gzip-input sweeps it.
 * Device memory of a split stream, held until cg_gzin_destroy: 16 bytes of symbol room per compressed byte of the
 * largest submission (grown for chunks that inflate further), 32 KiB of window per chunk, and the plain bytes. */
#define CG_GZIN_SPLIT_MEMBERS 1
#define CG_GZIN_LONG_MEMBER (64 * 1024)
#define CG_GZIN_STRIDE (64 * 1024)
int cg_gzin_create_ex(cg_ctx *ctx, int32_t flags, int32_t *handle);
int cg_gzin_destroy(cg_ctx *ctx, int32_t handle);
int cg_fastq_submit_gzip(cg_ctx *ctx, int32_t handle, const uint8_t *gz, int64_t n_bytes, int32_t format, int32_t final,
                         int32_t *slot, cg_gzin_result *res);
/* Unaligned BAM input (what the reference reads single-end since v4.7 through dnaio): format CG_FORMAT_BAM, accepted only
 * by cg_fastq_submit_gzip (default and split streams alike; CG_EINVAL in every other submit and as
 * cg_fastq_params.format).  A BAM file is BGZF, so its members inflate like any gzip input; the plain stream is the BAM
 * header ("BAM\1", l_text, text, n_ref, n_ref x (l_name, name, l_ref)), skipped, then records.  The slot holds the FASTQ
 * text of the whole records cut so far -- per record "@" + name + "\n" + the sequence decoded with "=ACMGRSVTWYHKDBN" +
 * "\n+\n" + every quality byte + 33 + "\n"; CIGAR and aux tags are skipped -- and is indistinguishable from
 * cg_fastq_submit of that text: cg_fastq_slot_read returns it and every single-end collect takes it (params.format
 * CG_FORMAT_FASTQ or CG_FORMAT_FASTQ_TO_FASTA).  Result: chunk_bytes is the FASTQ size of the slot, n_records its
 * records, plain_bytes and carry_bytes count BAM bytes.  The cut keeps the FASTQ text under the 2 GiB chunk limit (FASTQ
 * is at most 4/3 of its BAM bytes); at `final` a chunk that reaches it leaves carry_bytes > 0: submit again (final, no
 * bytes) until the carry is empty.  A stream takes one format for its whole life: CG_FORMAT_BAM after another format,
 * or another after CG_FORMAT_BAM, is CG_EINVAL.
 * A record is structurally valid when l_read_name >= 1, its name ends in NUL, l_seq >= 0 and
 * 32 + l_read_name + 4 n_cigar_op + (l_seq + 1) / 2 + l_seq <= block_size.  Where dnaio refuses a record or its answer
 * is not known, the record is refused rather than guessed:
 *   CG_EINVAL        not "BAM\1" or a negative length in the header ("not a BAM file"); a header or record still
 *                    incomplete at `final` ("BAM file ends inside record N"); a structurally invalid record; a quality
 *                    value above 93; a name byte outside 0x21..0x7E (the SAM specification's [!-?A-~]);
 *   CG_EUNSUPPORTED  flag != 4 (dnaio reads unmapped single reads only); no qualities (l_seq > 0 and the first quality
 *                    byte 0xFF); one record whose FASTQ text alone reaches 2 GiB.
 * Messages name the record by its number in the file (0-based) and its offset in the decompressed stream.  As for gzip
 * errors, no slot is taken, the stream is unchanged and the context stays usable. */
#define CG_FORMAT_BAM 3
/* The tiles of the BAM record-boundary walk a stream ran and those walked again because their speculative start was
 * not on the true chain, over the stream's life. */
int cg_gzin_bam_tiles(cg_ctx *ctx, int32_t handle, int64_t *tiles, int64_t *rewalked);
/* The plain chunk of a submitted, not yet collected slot, copied to host memory (the first slot of an interleaved chunk
 * returns the whole interleaved chunk; its second slot holds none):
 * what a caller keeps to submit a chunk from cg_fastq_submit_gzip again (a collect that needs a larger row buffer).
 * *n_bytes: its size; CG_EINVAL when capacity is smaller. */
int cg_fastq_slot_read(cg_ctx *ctx, int32_t slot, uint8_t *dst, int64_t capacity, int64_t *n_bytes);
/* Two files of a pair: both chunks hold the same number of records (read_paired_fastq_chunks / read_paired_fasta_chunks);
 * slots -1 until both have one. */
int cg_fastq_submit_gzip_paired(cg_ctx *ctx, int32_t handle1, int32_t handle2, const uint8_t *gz1, int64_t n_bytes1,
                                const uint8_t *gz2, int64_t n_bytes2, int32_t format, int32_t final, int32_t *slot1,
                                int32_t *slot2, cg_gzin_result *res1, cg_gzin_result *res2);
/* An interleaved file: the chunk holds whole pairs (8 lines, or an even number of FASTA records) and becomes the two
 * slots cg_fastq_submit_interleaved gives for it. */
int cg_fastq_submit_gzip_interleaved(cg_ctx *ctx, int32_t handle, const uint8_t *gz, int64_t n_bytes, int32_t format,
                                     int32_t final, int32_t *slot1, int32_t *slot2, cg_gzin_result *res);

/* Demultiplexing (Demultiplexer.__call__, steps.py:397-409; SURVEY.md section 8(f) N4): every surviving record
 * goes to the output of the adapter of its most recent match, records without a match to the last output
 * ("unknown"; combine with discard_untrimmed to drop them).  adapter_dest[a] in [0, n_named) names the output of
 * adapter a (adapters that share a file share a number).  `out` receives the n_named + 1 outputs back to back, each
 * in input order: output d is out[segments[d] .. segments[d + 1]); segments must hold n_named + 2 values. */
int cg_fastq_collect_demux(cg_ctx *ctx, int32_t slot, const cg_adapterset *set, const cg_fastq_params *params,
                           const int32_t *adapter_dest, int32_t n_named, uint8_t *out, int64_t out_capacity,
                           cg_fastq_result *res, int64_t *segments);

/* Paired-end chunks (PairedEndPipeline.process_reads, pipeline.py:125-153): record i of the two chunks is one
 * pair.  Each mate has its own adapter set (-a / -A; NULL = none) and parameters (-q / -Q, -u / -U, ...); --poly-a
 * trims the poly-T head of the second mate (PolyATrimmer(revcomp=True), cli.py:968-971).  Filters work on the
 * pair like PairedEndFilter (steps.py:105-180): pair_filter_mode 0 "any" (default), 1 "both", 2 "first"; a filter
 * enabled in only one mate's parameters tests that mate alone; with adapters on one mate only,
 * --discard-untrimmed tests "both" (cli.py:859-893).  Pair-level counters (n_written, too_short, ...) are
 * reported in both results, per-mate ones (bp_in, bp_out, with_adapters, quality_trimmed_bp) in their own. */
int cg_fastq_collect_paired(cg_ctx *ctx, int32_t slot1, int32_t slot2, const cg_adapterset *set1,
                            const cg_adapterset *set2, const cg_fastq_params *params1, const cg_fastq_params *params2,
                            int32_t pair_filter_mode, uint8_t *out1, int64_t out_capacity1, uint8_t *out2,
                            int64_t out_capacity2, cg_fastq_result *res1, cg_fastq_result *res2);

/* cg_fastq_collect plus the rows --info-file gets for the chunk (InfoFileWriter.__call__, steps.py:222-253;
 * SingleMatch / LinkedMatch.get_info_records, adapters.py:395-417, 1157-1171), formatted on the device: one row per
 * match (name, errors, rstart, rstop, the three parts of the read and of its qualities, adapter name, "1" / "0" if
 * --revcomp is on), coordinates applied to the read as it came; reads without a match: name, -1, the read as written.
 * Rows of ALL records, filtered or not (the writer sits in front of the filters).  adapter_names: the names of the
 * set's adapters back to back (the parts of a linked adapter as "name;1" / "name;2"), name_offsets: n_adapters + 1
 * offsets into it.  *info_bytes: size of the rows; CG_EINVAL if info_capacity is too small (nothing is then added
 * to the statistics accumulator).  The same as cg_fastq_request_rows(CG_ROWS_INFO) + cg_fastq_collect +
 * cg_fastq_read_rows. */
int cg_fastq_collect_info(cg_ctx *ctx, int32_t slot, const cg_adapterset *set, const cg_fastq_params *params,
                          const char *adapter_names, const int32_t *name_offsets, uint8_t *out, int64_t out_capacity,
                          uint8_t *info_out, int64_t info_capacity, cg_fastq_result *res, int64_t *info_bytes);

/* The same for the other per-read text outputs.  kind 0: --info-file (as above); 1: --rest-file (RestFileWriter,
 * steps.py:193-206; SingleMatch.rest, adapters.py:430-437, 463-470): for the last match of a read, what lies behind a
 * 3' adapter / in front of a 5' adapter, if not empty, then " name"; 2: --wildcard-file (WildcardFileWriter,
 * steps.py:209-220; SingleMatch.wildcards, adapters.py:378-393): the read characters under the N positions of the adapter
 * of the last match, then " name" -- adapter_text holds the adapters' SEQUENCES for kind 2 (their names for kind 0,
 * anything for kind 1).  Linked adapters: undefined, as in the reference (its writers fail on a LinkedMatch). */
int cg_fastq_collect_rows(cg_ctx *ctx, int32_t slot, const cg_adapterset *set, const cg_fastq_params *params, int32_t kind,
                          const char *adapter_text, const int32_t *text_offsets, uint8_t *out, int64_t out_capacity,
                          uint8_t *rows_out, int64_t rows_capacity, cg_fastq_result *res, int64_t *rows_bytes);

/* Rows from any collect.  A row request belongs to a submitted slot (from any cg_fastq_submit*, a mate of an
 * interleaved chunk included) and is honoured by whatever collect takes that slot, next to its usual outputs: the
 * plain, split, demultiplexing and paired collects all format the rows of each of their slots that has requests, after
 * the adapters were matched and before the filters, so the rows cover every record of the slot, filtered or not, in
 * input order -- the row writers sit in front of the filters in the reference (steps.py:193-269).  On pairs this is
 * PairedSingleEndStep (cli.py:675-696: --info-file, --rest-file and --wildcard-file write R1's rows) and
 * PairedInfoFileWriter (steps.py:256-269: --info-file-paired adds R2's info rows): request the kinds on each mate's
 * slot.  The rows and their format are those of cg_fastq_collect_info / cg_fastq_collect_rows; the coordinates of info
 * rows apply to the read as it came (before -u and the quality trimmers) on every path.  With --pair-adapters,
 * `adapter` of a match is the number of the pair, so the text of each mate is that mate's list (R1: the -a adapters, R2:
 * the -A adapters; PairedAdapterCutter, modifiers.py:476-477).
 *
 * cg_fastq_request_rows: ask the next collect that takes `slot` for the rows of `kind` as well.  adapter_text /
 * text_offsets as for cg_fastq_collect_rows (names for CG_ROWS_INFO, anything for CG_ROWS_REST, sequences for
 * CG_ROWS_WILDCARD), n_entries + 1 offsets; both are copied before the call returns.  gzip != 0: the rows are
 * compressed on the device in the member format of cg_fastq_params.gzip_outputs (members of at most 65 280 plain
 * bytes).  At most one request per kind and slot; a request applies to one collect.  The collect fails with CG_EINVAL
 * when n_entries is not the number of adapters of its set for that slot (the number of pairs with --pair-adapters, 0
 * without a set).  A collect without requests does what it did without this call. */
#define CG_ROWS_INFO 0          /* --info-file      (InfoFileWriter)     */
#define CG_ROWS_REST 1          /* --rest-file      (RestFileWriter)     */
#define CG_ROWS_WILDCARD 2      /* --wildcard-file  (WildcardFileWriter) */
int cg_fastq_request_rows(cg_ctx *ctx, int32_t slot, int32_t kind, const char *adapter_text, const int32_t *text_offsets,
                          int32_t n_entries, int32_t gzip);
/* After the collect that took `slot` returned CG_OK: the rows of `kind` into dst (dst == NULL: the sizes only).  They
 * stay on the device until the slot is submitted again.  *n_bytes: the bytes delivered (compressed if requested),
 * *n_bytes_plain: the size of the text; CG_EINVAL if capacity < *n_bytes, if that kind was not requested, or before
 * the collect or after a failed one. */
int cg_fastq_read_rows(cg_ctx *ctx, int32_t slot, int32_t kind, uint8_t *dst, int64_t capacity, int64_t *n_bytes,
                       int64_t *n_bytes_plain);

/* --pair-adapters (PairedAdapterCutter, modifiers.py:412-503): adapter i of the -a list is removed from R1 only
 * together with adapter i of the -A list from R2.  sets1[i] / sets2[i] hold adapter i alone (one group each); every
 * pair is matched against both mates on the device and the best pair that matches BOTH mates wins (highest score
 * sum, then fewest errors, then the first listed).  `adapter` of the resulting matches is the pair's number.  The
 * quality trimmers of params1 / params2 run first, times is 1; actions: trim, none, mask, retain. */
int cg_fastq_collect_pair_adapters(cg_ctx *ctx, int32_t slot1, int32_t slot2, const cg_adapterset *const *sets1,
                                   const cg_adapterset *const *sets2, int32_t n_pairs, const cg_fastq_params *params1,
                                   const cg_fastq_params *params2, int32_t pair_filter_mode, uint8_t *out1,
                                   int64_t out_capacity1, uint8_t *out2, int64_t out_capacity2, cg_fastq_result *res1,
                                   cg_fastq_result *res2);

/* Paired-end demultiplexing.  adapter_dest2 == NULL: PairedDemultiplexer (steps.py:422-503), both mates go to the
 * output of the adapter of R1's most recent match, destinations 0 .. n_named1 (the last = no match).  Otherwise
 * CombinatorialDemultiplexer (steps.py:506-581): destination d1 * (n_named2 + 1) + d2 from the matches on both mates.
 * dest_keep (optional, one byte per destination): pairs routed to a destination with 0 are dropped without being
 * counted (a combination without a writer, steps.py:574-577).  out1 / out2 receive the destinations back to back;
 * segments1 / segments2 (n_dest + 1 values each) say where each starts. */
int cg_fastq_collect_paired_demux(cg_ctx *ctx, int32_t slot1, int32_t slot2, const cg_adapterset *set1,
                                  const cg_adapterset *set2, const cg_fastq_params *params1, const cg_fastq_params *params2,
                                  int32_t pair_filter_mode, const int32_t *adapter_dest1, int32_t n_named1,
                                  const int32_t *adapter_dest2, int32_t n_named2, const uint8_t *dest_keep, uint8_t *out1,
                                  int64_t out_capacity1, uint8_t *out2, int64_t out_capacity2, cg_fastq_result *res1,
                                  cg_fastq_result *res2, int64_t *segments1, int64_t *segments2);

/* Filter outputs: --too-short-output, --too-long-output, --untrimmed-output and their paired forms (SingleEndFilter /
 * PairedEndFilter with a writer, steps.py:70-180).  A read (or pair) that one of these filters removes is written to
 * that filter's output instead of being dropped: trimmed and modified exactly as the main output would have it.  The
 * first filter in chain order that fires decides, as in cg_fastq_collect; filters without an output still drop.
 * Destinations: 0 main, 1 too-short, 2 too-long, 3 untrimmed.  `out` holds them back to back, each in input order:
 * output d is out[segments[d] .. segments[d + 1]) (5 values; outputs not redirected are empty).
 *   redirect       CG_REDIRECT_* bits.  CG_REDIRECT_UNTRIMMED switches the untrimmed filter on for both mates (with
 *                  adapters on one mate only, a pair is untrimmed when both mates are, cli.py:859-893); combined
 *                  with discard_trimmed it is CG_EINVAL.  redirect == 0 gives what cg_fastq_collect(_paired) gives.
 *   fasta_outputs  the same bits: a set bit writes that output as FASTA (">name\nsequence\n"), a clear one as FASTQ;
 *                  the main output follows params.format.  With CG_FORMAT_FASTA input every redirect bit must be set.
 * Counters: the filter counters count every removed read as before (the untrimmed output in `discarded`); n_written,
 * bp_out and the written-length histogram of params.stats count the main output only.  The output bound and the
 * "buffer too small -> out_bytes" contract are those of cg_fastq_collect (every record is written at most once). */
#define CG_REDIRECT_TOO_SHORT 1
#define CG_REDIRECT_TOO_LONG 2
#define CG_REDIRECT_UNTRIMMED 4
int cg_fastq_collect_split(cg_ctx *ctx, int32_t slot, const cg_adapterset *set, const cg_fastq_params *params,
                           int32_t redirect, int32_t fasta_outputs, uint8_t *out, int64_t out_capacity,
                           cg_fastq_result *res, int64_t *segments);
/* Paired-end: cg_fastq_collect_paired's arguments; both mates of a pair go to the same destination. */
int cg_fastq_collect_paired_split(cg_ctx *ctx, int32_t slot1, int32_t slot2, const cg_adapterset *set1,
                                  const cg_adapterset *set2, const cg_fastq_params *params1, const cg_fastq_params *params2,
                                  int32_t pair_filter_mode, int32_t redirect, int32_t fasta_outputs, uint8_t *out1,
                                  int64_t out_capacity1, uint8_t *out2, int64_t out_capacity2, cg_fastq_result *res1,
                                  cg_fastq_result *res2, int64_t *segments1, int64_t *segments2);

/* Interleaved paired-end input (--interleaved with one input; what `fastq-dump --split-spot` writes): R1 and R2 of each
 * pair follow each other in one chunk.  The chunk is uploaded once and split on the device into two slots that look
 * exactly like two submitted mate chunks: record 2p of the chunk is record p of mate 1 (*slot1), record 2p + 1 record p
 * of mate 2 (*slot2).  Every paired collect (cg_fastq_collect_paired, _paired_split, _paired_demux, _pair_adapters,
 * _paired_interleaved) then takes (*slot1, *slot2) in that order; any other use of these slots is CG_EINVAL.  format is
 * the input format as cg_fastq_params.format gives it: CG_FORMAT_FASTQ or CG_FORMAT_FASTQ_TO_FASTA for FASTQ,
 * CG_FORMAT_FASTA for FASTA (a chunk of whole records); the collect's params must have the same input format.  The split runs when the pair is
 * collected; these are then CG_EINVAL, the message naming what was found:
 *   - an odd number of records (the last one has no mate: "Interleaved input file incomplete");
 *   - mate names that do not match ("Reads are improperly paired"; the rule of dnaio's readers, doc/reference.rst:
 *     925-950: the IDs up to the first space or tab, a final 1, 2 or 3 of both ignored), naming the first such pair by
 *     its record numbers in the chunk;
 *   - a FASTQ format error, naming the record number in the chunk (2p or 2p + 1); FASTA format errors name the line of
 *     the chunk.
 * The split takes two of the four slots, like a two-file pair, so one pair can stay in flight while the next uploads. */
int cg_fastq_submit_interleaved(cg_ctx *ctx, const uint8_t *chunk, int64_t n_bytes, int32_t format, int32_t *slot1,
                                int32_t *slot2);

/* Interleaved outputs: cg_fastq_collect_paired_split plus interleaved_outputs, the destinations written interleaved
 * (CG_INTERLEAVE_MAIN for the main output, the CG_REDIRECT_* bits for the too-short, too-long and untrimmed outputs; the
 * reference interleaves each output whose paired path is missing, cli.py:650-661, 913-921).  An interleaved destination
 * d holds both mates in out1's segment d, R1 then R2 of each pair in input order, and out2's segment d is empty.
 * interleaved_outputs == 0 gives what cg_fastq_collect_paired_split gives, byte for byte.  The bound and the "buffer too
 * small -> out_bytes" contract hold per buffer (out1 must hold both mates of every interleaved destination; out_bytes of
 * res1 counts them); fasta_outputs applies per destination.  Counters, n_written, bp_out and the statistics vectors are
 * those of the two-file call.  Works on two submitted mate chunks and on an interleaved submission alike. */
#define CG_INTERLEAVE_MAIN 8
int cg_fastq_collect_paired_interleaved(cg_ctx *ctx, int32_t slot1, int32_t slot2, const cg_adapterset *set1,
                                        const cg_adapterset *set2, const cg_fastq_params *params1,
                                        const cg_fastq_params *params2, int32_t pair_filter_mode, int32_t redirect,
                                        int32_t fasta_outputs, int32_t interleaved_outputs, uint8_t *out1,
                                        int64_t out_capacity1, uint8_t *out2, int64_t out_capacity2, cg_fastq_result *res1,
                                        cg_fastq_result *res2, int64_t *segments1, int64_t *segments2);

/* gzip outputs: cg_fastq_params.gzip_outputs names the outputs that every call writing records (cg_fastq_trim_chunk,
 * cg_fastq_collect, _demux, _info, _rows, _paired, _pair_adapters, _paired_demux, _split, _paired_split,
 * _paired_interleaved) writes as gzip, compressed on the device before the download:
 *   CG_GZIP_MAIN      the main output; in the demultiplexing collects every demultiplexed output, "unknown" included;
 *   CG_REDIRECT_*     the filter outputs of the split collects (a bit for an output that is not redirected compresses
 *                     nothing).
 * Any other bit is CG_EINVAL.  params1 governs out1's outputs and params2 out2's; an interleaved output needs its bit set
 * alike in both, else CG_EINVAL.  The row outputs of _info / _rows stay plain.
 * Format: each output is cut into pieces of 65 280 bytes (0xff00) from its start, the last one shorter, and every piece is
 * one gzip member: the header 1f 8b 08 00 00 00 00 00 00 ff (no name, mtime 0, OS unknown), one final deflate block
 * (dynamic Huffman codes, or stored when that is not larger), CRC-32 and ISIZE.  An empty output is 0 bytes.  The members
 * follow each other, which is one valid gzip file (RFC 1952 2.2), so chunk outputs can be concatenated.  The bytes depend
 * on the plain bytes alone.  A member is at most 23 bytes larger than its piece, so an output of n plain bytes needs at
 * most n + 23 * ceil(n / 65280) bytes.
 * segments and out_bytes then describe the compressed outputs, out_bytes_plain the plain ones.  "Buffer too small" is
 * judged on the compressed size (out_bytes says what is needed); counters, n_written, bp_out and the statistics vectors
 * are those of the same call without compression. */
#define CG_GZIP_MAIN 8

/* ---- trim statistics (the payload of the end-of-run all-reduce, report.py:81-126) --------
 * Device-side reduction of a batch's match records into a fixed-layout int64 vector that carries everything the
 * reference's Statistics.__iadd__ adds up (report.py:81-126), so that one all-reduce merges the ranks:
 *   [0] n_reads  [1] total_bp  [2] reads_with_adapters  [3] quality_trimmed_bp  [4] bp_removed_by_adapters
 *   [5] reverse_complemented  [6] n_written  [7] bp_written
 *   [8..14] filtered: too_short, too_long, too_many_n, too_many_expected_errors, casava_filtered, discard_trimmed,
 *           discard_untrimmed   [15] too_high_average_error_rate
 *       ([5..15] are produced by steps outside the match records; this function leaves them alone)
 *   [16 .. 16 + max_len]  read-length histogram after trimming (ReadLengthStatistics, statistics.py:5-48)
 *   then per adapter a and end e (0: matches removing what precedes them, 1: what follows them), i.e. the two
 *   EndStatistics of AdapterStatistics.end_statistics() (adapters.py:142-289):
 *       adjacent[8]: A C G T other (EndStatistics.adjacent_bases; only filled when d_seq is given), 3 unused
 *       hist[removed_len (0..max_len)][errors (0..kmax)]                        (EndStatistics.errors)
 * cg_stats_size() returns the vector length for given (n_adapters, max_len, kmax).  d_seq may be NULL. */
int64_t cg_stats_size(int32_t n_adapters, int32_t max_len, int32_t kmax);
int cg_stats_accumulate_device(cg_ctx *ctx, const cg_adapterset *set, const uint8_t *d_seq, const int64_t *d_offsets,
                               int64_t n_reads, const cg_params *params,
                               const cg_match *d_matches, const int32_t *d_qtrim,
                               int32_t max_len, int32_t kmax, int64_t *d_stats);
/* cg_process_batch plus the statistics vector of the batch (same layout), reduced on the device chunk by chunk and
 * ADDED to the caller's host vector `stats` (cg_stats_size(n_adapters, max_len, kmax) entries) at the end: what a
 * worker of the reference accumulates in its Statistics object while it processes a chunk (pipeline.py:60-69,
 * modifiers.py:202-205), ready for the end-of-run merge. */
int cg_process_batch_stats(cg_ctx *ctx, const cg_adapterset *set, const uint8_t *seq, const uint8_t *qual,
                           const int64_t *offsets, int64_t n_reads, const cg_params *params,
                           cg_match *matches, int32_t *qtrim, int32_t max_len, int32_t kmax, int64_t *stats);

/* ---- statistics of the FASTQ path ------------------------------------------------------------------------
 * What a worker of the reference collects for its report while it runs a chunk (Statistics.collect, report.py:128-208):
 * AdapterCutter.adapter_statistics (modifiers.py:109, 200-207), ReverseComplementer's per-adapter reverse_complemented
 * (modifiers.py:301-306), PolyATrimmer.trimmed_bases (modifiers.py:861-879) and the ReadLengthStatistics of the
 * writers (report.py:155-157).  An accumulator belongs to a context; a collect adds to the one named by
 * cg_fastq_params.stats when it returns CG_OK (a failed call, e.g. "output buffer too small", adds nothing).  Every
 * collect honours it; paired calls take params1.stats / params2.stats, one accumulator per mate (the same handle on
 * both is CG_EINVAL).  n_adapters must be the number of adapters of the set (cg_adapter_desc entries; 0 without a
 * set), for --pair-adapters the number of pairs (`adapter` = pair number); otherwise the collect is CG_EINVAL.
 * Nothing is clamped: max_len grows to the longest read (after -u) seen, kmax to the largest error count any adapter
 * of the sets can report ((int)(max_error_rate * length)); the vector is laid out anew when they grow.
 * Vector (int64): the cg_stats_* layout below at (n_adapters, max_len, kmax), with
 *   [0] n_records [1] bp_in [2] with_adapters [3] quality_trimmed_bp [4] bases removed by the adapter matches
 *   [5] reverse_complemented [6] n_written [7] bp_out [8..14] the filter counts of the result struct; discarded goes
 *   to [13] with discard_trimmed, else to [14]; [15] too_high_average_error_rate
 *   read-length histogram: WRITTEN records by written length, all outputs of a demultiplexing call together (pairs
 *   dropped through dest_keep are not counted)
 *   per adapter and end: every match of every read that went through the cutter, filtered or not; adjacent bases
 *   as the reference reads them (upper-cased read with CG_ACTION_LOWERCASE)
 * then the tail: reverse_complemented[n_adapters] (matches on reads that were replaced by their reverse complement),
 * poly_a[max_len + 1] (bases PolyATrimmer removed per read, 0 included; empty without --poly-a).
 * cg_fastq_stats_read reports (max_len, kmax) and the size; with out != NULL it copies the vector (capacity must
 * hold it) and with reset != 0 then zeroes it. */
int cg_fastq_stats_create(cg_ctx *ctx, int32_t n_adapters, int32_t *handle);   /* handle > 0 */
int cg_fastq_stats_read(cg_ctx *ctx, int32_t handle, int32_t *max_len, int32_t *kmax, int64_t *out, int64_t capacity,
                        int64_t *size, int reset);
int cg_fastq_stats_destroy(cg_ctx *ctx, int32_t handle);

/* ---- read names: --length-tag, --strip-suffix, -x / -y and --rename on the device ----
 * The reference's name modifiers (LengthTagModifier, SuffixRemover, PrefixSuffixAdder, Renamer / PairedEndRenamer,
 * modifiers.py:529-760) run last in its chain (cli.py:937-991, 1136-1146), after the adapters, --poly-a, --length and
 * --trim-n; in pairs the first three run on each mate with that mate's own match.  A collect whose params name a names
 * handle runs one name stage per mate once the matches and the written part of every read are final: after --revcomp,
 * the pair swap, --pair-adapters and the filters' evaluation, before the rows and the sizing of the records.  Every
 * output then carries the new name: main, filter, demultiplexed, interleaved and gzip outputs, FASTA output, and the
 * info, rest and wildcard rows.  The name the chain starts from already carries the " rc" of --revcomp (revcomp = 1).
 *   length_tag   TAG (NULL = off): when TAG occurs in the name, every non-overlapping match of \bTAG[0-9]*\b (Python
 *                re, left to right; the longest digit run followed by a word boundary, possibly empty) becomes TAG
 *                followed by the length of the sequence as written.  TAG is a literal here: only letters, digits and
 *                _ = : , ; / - @ # % ! ~ are accepted (CG_EINVAL names any other character); "" is refused.
 *   strip_suffix each value in order: removed once if the name ends with it ("" empties the name, as name[:-0] does)
 *   prefix / suffix  (NULL = ""): prefix + name + suffix, "{name}" in either replaced by the adapter name of the read's
 *                last match or "no_adapter"; no other brace is special.
 *   rename / n_rename  the --rename template tokenized (tokenize_braces; the caller reports the reference's errors and
 *                replaces a two-character \t by a tab in the literals); n_rename < 0: no renamer.  Variables:
 *                header, id, comment (name.split(maxsplit=1) with Python's whitespace: one field or none gives the id
 *                the whole name and an empty comment), cut_prefix / cut_suffix (the bases the last -u value of that end
 *                removed; the 5' values are applied first), adapter_name, rc ("rc" / ""), match_sequence (the last
 *                match's sequence[rstart:rstop] of the sequence its round searched, front + "," + back for a linked
 *                match, "" without a match).  paired != 0 (PairedEndRenamer): rc is refused, rn (1 / 2) and the
 *                mate forms (mate 1 = r1., 2 = r2.) of every variable but id and rc are allowed; each mate is
 *                evaluated on its own record.  A pair whose step-1 names do not name mates (dnaio's rule) fails the
 *                collect with "Input read IDs not identical: ..." (R1's ID and R1's comment, as the reference prints
 *                them), a pair whose new IDs no longer do with "After renaming R1 and R2, ...", each naming the first
 *                such pair.  Neither prefix nor suffix may be
 *                given with a renamer.
 * cg_names_set_mate: the adapter names of a mate's list, indexed as the match records index it (a linked adapter's
 * parts both carry the linked adapter's name; with --pair-adapters, pair i of that mate's list), with linked[a] != 0
 * for the parts of a linked adapter, and the last -u value of each end of that mate (>= 0).  A mate not set has no
 * names ("no_adapter") and no -u cutter. */
#define CG_NT_LITERAL 0
#define CG_NT_HEADER 1
#define CG_NT_ID 2
#define CG_NT_COMMENT 3
#define CG_NT_CUT_PREFIX 4
#define CG_NT_CUT_SUFFIX 5
#define CG_NT_ADAPTER_NAME 6
#define CG_NT_RC 7
#define CG_NT_MATCH_SEQUENCE 8
#define CG_NT_RN 9
typedef struct cg_name_token {
    int32_t kind;                /* CG_NT_*                                                           */
    int32_t mate;                /* 0 the record's own value, 1 {r1.x}, 2 {r2.x}                       */
    const char *text;            /* CG_NT_LITERAL: the text (len bytes)                               */
    int32_t len;
} cg_name_token;
typedef struct cg_names_desc {
    const char *length_tag;
    const char *const *strip_suffix;
    int32_t n_strip_suffix;
    int32_t paired;
    const char *prefix, *suffix;
    const cg_name_token *rename;
    int32_t n_rename;
} cg_names_desc;
int cg_names_create(cg_ctx *ctx, const cg_names_desc *desc, int32_t *handle);   /* handle > 0 */
int cg_names_set_mate(cg_ctx *ctx, int32_t handle, int32_t mate, const char *names, const int32_t *offsets,
                      int32_t n_names, const uint8_t *linked, int32_t last_cut_front, int32_t last_cut_back);
int cg_names_destroy(cg_ctx *ctx, int32_t handle);

/* ---- host-side index helpers (adapters.py:1416-1442 use these to build AdapterIndex) ----
 * edit_environment (_align.pyx:785-882) / hamming_sphere-based environment
 * (align.py hamming_environment): enumerate into a caller buffer.
 * Each record: length byte-string of `stride` bytes (NUL padded), then errors, matches.
 * Returns the number of records (>= 0) or a negative code; if it exceeds `capacity` only the
 * first `capacity` are written and the full count is still returned. */
int64_t cg_edit_environment(const uint8_t *s, int32_t n, int32_t k, int32_t stride,
                            uint8_t *strings, int32_t *lengths, int32_t *errors,
                            int32_t *matches, int64_t capacity);
int64_t cg_hamming_environment(const uint8_t *s, int32_t n, int32_t k, int32_t stride,
                               uint8_t *strings, int32_t *errors, int32_t *matches,
                               int64_t capacity);

#ifdef __cplusplus
}
#endif
#endif /* CUTADAPT_B200_H */
