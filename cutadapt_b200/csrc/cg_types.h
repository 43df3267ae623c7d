// cg_types.h -- plain-old-data tables shared by the host-side adapter-set compiler and the kernels.
//
// An adapter set is compiled once on the host (cg_api.cu: cg_adapterset_create) into one
// contiguous, position-independent blob:
//
//   CgSetHeader | CgAdapter[n_adapters] | CgGroup[n_groups] | CgEntry[n_entries] | pool bytes
//
// The blob is copied to HBM once and, at the start of every fused kernel, from HBM into the
// CTA's shared memory (it is a few hundred bytes to a few KB: adapters are <= a few hundred
// bases).  The 128 x uint64 needle masks of the k-mer prefilter live in a second HBM array
// (L1/L2 resident; 1 KiB per search word).
#pragma once
#if defined(__CUDACC_RTC__)      // NVRTC (cg_jit.cpp): no host headers
typedef signed char int8_t;
typedef unsigned char uint8_t;
typedef short int16_t;
typedef unsigned short uint16_t;
typedef int int32_t;
typedef unsigned int uint32_t;
typedef long long int64_t;
typedef unsigned long long uint64_t;
typedef unsigned long long uintptr_t;
#else
#include <stdint.h>
#endif

#if defined(__CUDACC__)
#define CG_HD __host__ __device__ __forceinline__
#define CG_HD_NOINLINE __host__ __device__ __noinline__
#else
#define CG_HD inline
#define CG_HD_NOINLINE
#endif

enum { CG_CELL_PACKED32 = 0, CG_CELL_WIDE = 1 };

struct CgAdapter {          // 80 bytes
    int32_t m;              // adapter length
    int32_t k;              // (int)(max_error_rate * m)                  _align.pyx:343
    int32_t flags;          // EndSkip bits                               align.py:24-34
    int32_t min_overlap;
    int32_t indel_cost;
    int32_t kind;           // CG_KIND_*
    int32_t reverse;        // scan the read back to front                adapters.py:766,870
    int32_t remove;         // CG_REMOVE_*
    int32_t compare_ascii;  // 1: upper-cased ASCII equality, 0: (a & b) != 0   _align.pyx:442-445
    int32_t query_enc;      // read encoding table: 0 upper, 1 acgt, 2 iupac     _align.pyx:322-328
    int32_t wildcard_ref;
    int32_t effective_length;
    int32_t max_k_cmp;      // comparers: int(rate * effective_length)    _align.pyx:633
    int32_t cell_mode;      // CG_CELL_*
    int32_t pf_first;       // first prefilter entry
    int32_t pf_count;       // number of prefilter entries; 0 = always pass (MockKmerFinder)
    uint32_t ref_off;       // pool offset: encoded adapter bytes [m]
    uint32_t ncount_off;    // pool offset (4-aligned): int32 n_counts[m+1]  _align.pyx:260-266
    uint32_t maxcost_off;   // pool offset (4-aligned): int32 maxcost[m+1] = floor(L * rate)
    uint32_t peq_off;       // pool offset (4-aligned): uint32 peq_lo[128], peq_hi[128]: bit r of
                            //   peq[c] = adapter row r matches read character c (m <= 64), else 0
};

struct CgEntry {            // 32 bytes; the reference's KmerSearchEntry  _kmer_finder.pyx:58-63
    int32_t start;
    int32_t stop;
    uint32_t mask_index;    // masks64[128 * mask_index + c]
    uint32_t pad;
    uint64_t init_mask;
    uint64_t found_mask;
};

struct CgGroup {            // 32 bytes
    int32_t type, a0, a1, front_required, back_required, pad[3];
};

// One 32-bit shift-and word of the fused scan stage (two-phase kernel).  The host re-packs the
// reference-form k-mer entries of an adapter, plus the "locator" chunks that drive the windowed
// DP, into 32-bit words grouped by window type (cg_setbuild.cpp: build_scan_program).
enum { CG_SCAN_WHOLE = 0, CG_SCAN_SUFFIX = 1, CG_SCAN_PREFIX = 2 };
struct CgScanWord {         // 32 bytes
    uint32_t type;          // CG_SCAN_*
    uint32_t span;          // SUFFIX/PREFIX: window length in characters
    uint32_t init;          // WHOLE: init mask (one bit at the first character of every k-mer)
    uint32_t pass_found;    // found bits of k-mers that belong to the KmerFinder (prefilter verdict)
    uint32_t loc_found;     // found bits of locator chunks (they place the DP windows)
    uint32_t mask_off;      // pool offset (4-aligned): uint32 mask[128] by ASCII code
    uint32_t pos_off;       // pool offset (4-aligned): SUFFIX: {init, found}[span + 1] by distance
                            //   from the end; PREFIX: {init, found}[span] by position
    uint32_t loc_off;       // pool offset: uint8 {bmin, bmax}[32] per bit: adapter offsets at which the
                            //   locator chunk ending in that bit may end (WHOLE words with loc_found)
};

struct CgSetHeader {        // 80 bytes
    int32_t n_adapters, n_groups, n_entries, slots;
    int32_t max_m;          // longest adapter (DP column height - 1)
    int32_t any_wide;       // some adapter needs the wide-cell path
    uint32_t adapters_off, groups_off, entries_off, pool_off;
    uint32_t total_bytes;   // size of the blob, multiple of 16
    // two-phase ("simple") program: one SINGLE aligner adapter with packed cells
    int32_t simple_ok;      // 1: the two-phase kernel may be used (times == 1)
    int32_t scan_count;     // number of CgScanWord
    uint32_t scan_off;      // blob offset of CgScanWord[scan_count]
    int32_t windowed;       // 1: DP may be restricted to windows around locator hits
    int32_t exact_ok;       // 1: an exact, leftmost occurrence found by the locator needs no DP at all
    int32_t myers;          // 1: the plan stage finds the DP runs with a bit-vector edit-distance pass over the
                            //    read instead of locator chunks (adapters whose chunks would hit everywhere)
    // bit-plane scan program (plane_scan_core): the same k-mers as 2-bit codes, matched word-parallel
    int32_t plane_count;    // number of op words (0: the adapter does not qualify)
    uint32_t plane_off;     // blob offset of uint32 ops[plane_count], then (8-aligned) CgPlaneEmit[n_emits]
    int32_t plane_flags;    // bit 0: an exact occurrence found by the planes may be reported without DP;
                            // bit 1: the program holds the end analysis (guard pieces + overlap emits; the
                            //        uint64 after the emits marks the overlap lengths whose string alone
                            //        makes KmerFinder.kmers_present true); bits 8-15: n_emits
};

// Bit-plane scan program.  Characters are 2-bit codes taken from bits 1 and 2 of the ASCII code
// (A = 0, C = 1, T = 2, G = 3; the same for lower case); only k-mers whose every position matches exactly
// one of A/C/G/T (either case) can be expressed, which the host checks.  The k-mers are laid out as
// CHAINS of one-character steps, acc = (acc << 1) & plane[code], so that k-mers sharing a prefix
// (AGA, AGAT, AGATC, AGATCGG) share the steps; a step may EMIT up to two k-mers that end with it.
//   op word: bits 0-1 code, bit 2 first step of a chain, bits 8-15 / 16-23: emit index + 1 (0 = none)
#define CG_PLANE_PASS 1u    // a k-mer of the KmerFinder (prefilter verdict)
#define CG_PLANE_LOC 2u     // a locator chunk (one of the k+1 pieces of the adapter)
#define CG_PLANE_GUARD 4u   // a piece of an adapter prefix, searched at the end of the read: if none occurs, no
                            // cell of the last column with errors can be acceptable (see plane_decide)
#define CG_PLANE_OP_NEW 4u
#define CG_SCAN_OVERLAP 3   // emit type: the adapter's first `len` characters; does the read END with them?
struct CgPlaneEmit {        // 8 bytes
    uint8_t len;            // 1..32
    uint8_t type;           // CG_SCAN_WHOLE or CG_SCAN_SUFFIX
    uint8_t flags;          // CG_PLANE_*
    uint8_t bend;           // locator chunk: adapter offset (exclusive) at which it ends
    uint16_t window;        // SUFFIX: the k-mer must lie within the last `window` characters (<= 64)
    uint16_t pad;
};
static_assert(sizeof(CgPlaneEmit) == 8, "CgPlaneEmit layout");
// host-side form of one k-mer (cg_setbuild.cpp)
struct CgPlaneKmer {
    uint64_t codes;         // 2 bits per character, first character in the low bits
    uint8_t len, type, flags, bend;
    uint16_t window, pad;
};

// Anchored-adapter index (AdapterIndex, adapters.py:1289-1551) as an open-addressing hash table.
struct CgIndexEntry {       // 16 bytes; len == 0 marks an empty slot
    uint64_t bases;         // 2 bits per character (A=0 C=1 G=2 T=3), first character in the low bits
    uint32_t len;           // key length (1..32)
    uint32_t val;           // adapter (16) | errors (8) | matches (8)
};
struct CgIndexHeader {      // 64 bytes, one per index, followed in the same array by its table
    int32_t prefix;
    int32_t n_lengths;
    uint8_t lengths[32];    // descending (keys are 1..32 characters, so at most 32 distinct lengths)
    uint32_t table_off;     // first CgIndexEntry of this index (in entries) within the index array
    uint32_t table_mask;    // capacity - 1 (power of two)
    uint32_t pad[4];
};
static_assert(sizeof(CgIndexHeader) == 64, "CgIndexHeader layout");

// Multi-pass schedule: which pass holds which component of which group (see cg_setbuild.h).
#define CG_MAX_PASSES 16
struct CgSelectTables {
    int32_t n_groups, slots;
    int32_t map_off[CG_MAX_PASSES];                 // per pass: first entry in pass_map
    int8_t gtype[CG_MAX_PASSES], pass0[CG_MAX_PASSES], pass1[CG_MAX_PASSES];      // per group
    int8_t front_required[CG_MAX_PASSES], back_required[CG_MAX_PASSES];
};

// Trim statistics vector (cg_stats_accumulate_device; the payload of the end-of-run all-reduce):
//   [0] n_reads  [1] total_bp  [2] reads_with_adapters  [3] quality_trimmed_bp  [4] bp_removed_by_adapters
//   [5] reverse_complemented  [6] n_written  [7] bp_written  [8..14] filtered[7]: too_short, too_long,
//   too_many_n, too_many_expected_errors, casava_filtered, discard_trimmed, discard_untrimmed
//   [15] too_high_average_error_rate (filtered, but not in filtered[7]: the reference's report does not list it)
//       ([5..15] belong to steps outside the match records -- ReverseComplementer, the filters, the writer -- and are
//        filled by whoever runs those steps; they are part of the vector so that ONE all-reduce carries everything
//        Statistics.__iadd__ adds up, report.py:81-126)
//   [16 .. 16 + max_len]   read-length histogram: final length of every read after all trimming
//                          (ReadLengthStatistics, statistics.py:5-48, before filters)
//   then per adapter a, per end (0 = 5' side: matches that remove what precedes them, 1 = 3' side):
//       adjacent[8]: counts of the base in front of a 3' match, order A C G T other (EndStatistics.adjacent_bases,
//                    adapters.py:84, 193-199); [5..7] unused
//       hist[removed_len (0..max_len)][errors (0..kmax)]          (EndStatistics.errors, adapters.py:82)
#define CG_STATS_SCALARS 16
#define CG_STATS_ADJ 8
CG_HD long long cg_stats_end_size(int max_len, int kmax) { return CG_STATS_ADJ + (long long)(max_len + 1) * (kmax + 1); }
CG_HD long long cg_stats_lengths_off() { return CG_STATS_SCALARS; }
CG_HD long long cg_stats_adapters_off(int max_len) { return CG_STATS_SCALARS + (max_len + 1); }
CG_HD long long cg_stats_total(int n_adapters, int max_len, int kmax)
{
    return cg_stats_adapters_off(max_len) + 2LL * n_adapters * cg_stats_end_size(max_len, kmax);
}

// One result of locating a single adapter in a (sub)sequence; coordinates as SingleMatch.
struct CgHit {
    int32_t adapter;        // -1 = none
    int32_t astart, astop, rstart, rstop, score, errors;
    int32_t remove;         // resolved CG_REMOVE_BEFORE / CG_REMOVE_AFTER
};

// Packed-cell limits (see cg_core.cuh, struct Packed32)
#define CG_PACKED_MAX_K 29
#define CG_PACKED_MAX_M 447
#define CG_PACKED_MAX_N 32255
