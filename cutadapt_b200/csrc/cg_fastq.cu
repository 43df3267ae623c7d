// cg_fastq.cu -- the steps either side of the hot path, on the device (SURVEY.md section 8(f) N1):
//
//   raw FASTQ chunk  ->  record index  ->  packed reads (what the trimming kernels consume)
//   match records    ->  kept intervals + filters  ->  trimmed FASTQ bytes
//
// In the reference these are dnaio's chunk parser and record writer around the per-read loop
// (runners.py:116-126 read_chunks, pipeline.py:47-73 process_reads, steps.py:299-319 SingleEndSink,
// files.py:164-188 ProxyRecordWriter) plus the length / trimmed filters (predicates.py:29-66, 127-160).
// Everything here is HBM-bound byte shuffling; the chunk crosses PCIe once in each direction.
#include <cuda_runtime.h>
#include <stdint.h>

#include "cg_kernels.cuh"

namespace {

constexpr int FQ_TILE = 8192;        // bytes per CTA in the newline passes
constexpr int FQ_THREADS = 256;      // 32 bytes per thread

__device__ __forceinline__ uint32_t newline_mask16(uint4 v)
{
    // bit i set iff byte i of the 16-byte vector is '\n'
    uint32_t m = 0;
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint32_t x = w[k] ^ 0x0A0A0A0Au;                        // zero byte where '\n'
        const uint32_t z = __vcmpeq4(x, 0u);                          // 0xFF per matching byte
        m |= ((z & 1u) | ((z >> 7) & 2u) | ((z >> 14) & 4u) | ((z >> 21) & 8u)) << (4 * k);
    }
    return m;
}

// bytes [n, padded end) of the last vector are masked off
__device__ __forceinline__ uint32_t load_mask(const uint8_t *buf, long long n, long long pos)
{
    if (pos >= n) return 0;
    const uint4 v = __ldg((const uint4 *)(buf + pos));
    uint32_t m = newline_mask16(v);
    if (pos + 16 > n) m &= (1u << (int)(n - pos)) - 1u;
    return m;
}

// pass 1: newlines per tile
__global__ void __launch_bounds__(FQ_THREADS) fq_count_kernel(const uint8_t *buf, long long n, uint32_t *tile_counts)
{
    const long long base = (long long)blockIdx.x * FQ_TILE + threadIdx.x * 32;
    int c = __popc(load_mask(buf, n, base)) + __popc(load_mask(buf, n, base + 16));
    __shared__ int warp_sums[FQ_THREADS / 32];
    c = __reduce_add_sync(0xFFFFFFFFu, c);
    if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int i = 0; i < FQ_THREADS / 32; ++i) t += warp_sums[i];
        tile_counts[blockIdx.x] = (uint32_t)t;
    }
}

// exclusive scan of up to a few hundred thousand uint32 values by ONE CTA (in place); total -> *total
__global__ void __launch_bounds__(1024) scan_u32_single_cta_kernel(uint32_t *vals, long long n, unsigned long long *total)
{
    __shared__ unsigned long long warp_tot[32];
    __shared__ unsigned long long carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (long long base = 0; base < n; base += 1024) {
        const long long i = base + threadIdx.x;
        const unsigned long long v = i < n ? vals[i] : 0;
        unsigned long long x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) warp_tot[warp] = x;
        __syncthreads();
        if (warp == 0) {
            unsigned long long w = warp_tot[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, w, d);
                if (lane >= d) w += y;
            }
            warp_tot[lane] = w;   // inclusive
        }
        __syncthreads();
        const unsigned long long carry = carry_s;
        const unsigned long long before = carry + (warp ? warp_tot[warp - 1] : 0) + (x - v);
        if (i < n) vals[i] = (uint32_t)before;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = carry + warp_tot[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry_s;
}

// pass 2: positions of all newlines, in order
__global__ void __launch_bounds__(FQ_THREADS) fq_index_kernel(const uint8_t *buf, long long n, const uint32_t *tile_offsets,
                                                               uint32_t *nl_pos)
{
    const long long base = (long long)blockIdx.x * FQ_TILE + threadIdx.x * 32;
    const uint32_t m = load_mask(buf, n, base) | (load_mask(buf, n, base + 16) << 16);
    const int c = __popc(m);
    __shared__ int warp_sums[FQ_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xFFFFFFFFu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    int before = x - c;
    for (int w = 0; w < warp; ++w) before += warp_sums[w];
    uint32_t out = tile_offsets[blockIdx.x] + (uint32_t)before;
    uint32_t mm = m;
    while (mm) {
        const int b = __ffs(mm) - 1;
        mm &= mm - 1;
        nl_pos[out++] = (uint32_t)(base + b);
    }
}

// record r = lines 4r .. 4r+3: fq_record_core (cg_fastq_core.cuh) builds the table entry and checks the format
__global__ void fq_records_kernel(const uint8_t *buf, long long n, const uint32_t *nl_pos, long long n_nl,
                                  long long n_records, int cut_front, int cut_back, CgFastqRecord *rec,
                                  int32_t *seq_len, int32_t *origin, unsigned long long *counters, int *err)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned bp = 0;
    if (r < n_records) {
        CgFastqRecord o;
        int len, full, cf;
        const int bad = fq_record_core(buf, n, nl_pos, n_nl, r, cut_front, cut_back, &o, &len, &full, &cf);
        // where the record lies in the read as it came: (bases in front of it, length of the whole read)
        if (origin) { origin[2 * r] = cf; origin[2 * r + 1] = full; }
        if (bad) {
            // report the first bad record: err[0] = code, err[1] = record number (smallest; initialised to INT_MAX)
            atomicMin((unsigned int *)&err[1], (unsigned int)r);
            atomicMax(&err[0], bad);
        }
        rec[r] = o;
        seq_len[r] = len;
        bp = (unsigned)full;
    }
    // bases read: the length before any modifier (pipeline.py:58-64)
    unsigned long long sum = bp;
    for (int d = 16; d; d >>= 1) sum += __shfl_down_sync(0xFFFFFFFFu, sum, d);
    if ((threadIdx.x & 31) == 0 && sum && counters) atomicAdd(&counters[1], sum);
}

// ---- exclusive scan int32 -> int64 (n+1 outputs), any n: tile sums, one-CTA scan of the sums, apply ----
constexpr int SC_TILE = 2048;     // elements per CTA (256 threads x 8)

__global__ void __launch_bounds__(256) scan_tile_sums_kernel(const int32_t *in, long long n, unsigned long long *tile_sums)
{
    const long long base = (long long)blockIdx.x * SC_TILE;
    long long s = 0;
    for (int k = 0; k < 8; ++k) {
        const long long i = base + k * 256 + threadIdx.x;
        if (i < n) s += in[i];
    }
    __shared__ long long ws[8];
    for (int d = 16; d; d >>= 1) s += __shfl_down_sync(0xFFFFFFFFu, s, d);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long t = 0;
        for (int i = 0; i < 8; ++i) t += ws[i];
        tile_sums[blockIdx.x] = (unsigned long long)t;
    }
}
__global__ void __launch_bounds__(1024) scan_u64_single_cta_kernel(unsigned long long *vals, long long n)
{
    __shared__ unsigned long long warp_tot[32];
    __shared__ unsigned long long carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (long long base = 0; base < n; base += 1024) {
        const long long i = base + threadIdx.x;
        const unsigned long long v = i < n ? vals[i] : 0;
        unsigned long long x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) warp_tot[warp] = x;
        __syncthreads();
        if (warp == 0) {
            unsigned long long w = warp_tot[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, w, d);
                if (lane >= d) w += y;
            }
            warp_tot[lane] = w;
        }
        __syncthreads();
        const unsigned long long carry = carry_s;
        if (i < n) vals[i] = carry + (warp ? warp_tot[warp - 1] : 0) + (x - v);
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = carry + warp_tot[31];
        __syncthreads();
    }
}
__global__ void __launch_bounds__(256) scan_apply_kernel(const int32_t *in, long long n, const unsigned long long *tile_offsets,
                                                          int64_t *out)
{
    // thread t owns 8 consecutive elements of the tile
    const long long base = (long long)blockIdx.x * SC_TILE + threadIdx.x * 8;
    int32_t v[8];
    long long s = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        v[k] = base + k < n ? in[base + k] : 0;
        s += v[k];
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long x = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const long long y = __shfl_up_sync(0xFFFFFFFFu, x, d);
        if (lane >= d) x += y;
    }
    __shared__ long long ws[8];
    if (lane == 31) ws[warp] = x;
    __syncthreads();
    long long before = (long long)tile_offsets[blockIdx.x] + (x - s);
    for (int w = 0; w < warp; ++w) before += ws[w];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        if (base + k < n) out[base + k] = before;
        before += v[k];
        if (base + k == n - 1) out[n] = before;
    }
}

// packed reads for the trimming kernels: read r at offsets[r] in seq_out / qual_out; rc: its reverse complement
__global__ void __launch_bounds__(256) fq_gather_kernel(const uint8_t *buf, const CgFastqRecord *rec, const int64_t *offsets,
                                                         long long n_records, uint8_t *seq_out, uint8_t *qual_out, int rc)
{
    const int lane = threadIdx.x & 31;
    const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_records; r += warps) {
        const CgFastqRecord m = rec[r];
        const long long o = offsets[r];
        const int len = (int)(offsets[r + 1] - o);
        if (rc) {
            for (int j = lane; j < len; j += 32) seq_out[o + j] = fq_complement(buf[m.seq_start + len - 1 - j]);
            if (qual_out)
                for (int j = lane; j < len; j += 32) qual_out[o + j] = buf[m.qual_start + len - 1 - j];
            continue;
        }
        for (int j = lane; j < len; j += 32) seq_out[o + j] = buf[m.seq_start + j];
        if (qual_out)
            for (int j = lane; j < len; j += 32) qual_out[o + j] = buf[m.qual_start + j];
    }
}

// The quality-trimmed interval becomes the record (like -u in fq_record_core): the modifiers after the quality
// trimmers then see the read they see in the reference (used where a later step needs the trimmed read as an
// object of its own: --revcomp, --pair-adapters).  counters[6] += bases removed.
__global__ void fq_fold_qtrim_kernel(CgFastqRecord *rec, int32_t *seq_len, const int32_t *qtrim, long long n_records,
                                     int32_t *origin, unsigned long long *counters)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long removed = 0;
    if (r < n_records) {
        const int n = seq_len[r], qs = qtrim[2 * r], qe = qtrim[2 * r + 1];
        rec[r].seq_start += (uint32_t)qs;
        rec[r].qual_start += (uint32_t)qs;
        seq_len[r] = qe - qs;
        if (origin) origin[2 * r] += qs;
        removed = (unsigned long long)(n - (qe - qs));
    }
    for (int d = 16; d; d >>= 1) removed += __shfl_down_sync(0xFFFFFFFFu, removed, d);
    if ((threadIdx.x & 31) == 0 && removed) atomicAdd(&counters[6], removed);
}

// ReverseComplementer.__call__ (modifiers.py:278-308), one warp per record: the reverse complement replaces the
// read iff the scores of its matches add up to MORE than those of the forward read (a linked match counts with
// both parts).  The replacement happens IN the chunk: the WHOLE read as it came is reverse-complemented in place
// (qualities reversed), so that the part the modifiers in front of the cutter left -- the record -- is the reverse
// complement of what it was and the rest still surrounds it (info.original_read.reverse_complement() of the info
// file, steps.py:233-235); the record table follows, the reverse matches become the record's matches,
// is_rc[r] = 1.  Every later kernel works on the chosen orientation without knowing about it (the writer appends
// the name suffix).  counters[11] += replaced.
__global__ void __launch_bounds__(256) fq_revcomp_commit_kernel(uint8_t *buf, CgFastqRecord *rec, const int32_t *seq_len,
                                                                 int32_t *origin, long long n_records, cg_match_rec *matches,
                                                                 const cg_match_rec *matches_rc, int per_read,
                                                                 uint8_t *is_rc, unsigned long long *counters)
{
    const int lane = threadIdx.x & 31;
    const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
    unsigned replaced = 0;
    for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_records; r += warps) {
        long long fwd = 0, rev = 0;
        for (int k = lane; k < per_read; k += 32) {
            const cg_match_rec a = matches[(size_t)r * per_read + k], b = matches_rc[(size_t)r * per_read + k];
            if (a.adapter >= 0) fwd += a.score;
            if (b.adapter >= 0) rev += b.score;
        }
        for (int d = 16; d; d >>= 1) {
            fwd += __shfl_xor_sync(0xFFFFFFFFu, fwd, d);
            rev += __shfl_xor_sync(0xFFFFFFFFu, rev, d);
        }
        const bool use = rev > fwd;
        if (lane == 0) is_rc[r] = use;
        if (!use) continue;
        replaced += lane == 0;
        const CgFastqRecord m = rec[r];
        const int front = origin[2 * r], full = origin[2 * r + 1];
        uint8_t *sq = buf + m.seq_start - front, *ql = buf + m.qual_start - front;
        for (int j = lane; 2 * j < full; j += 32) {      // pair (j, full-1-j); the middle of an odd length meets itself
            const int k = full - 1 - j;
            const uint8_t a = sq[j], b = sq[k], qa = ql[j], qb = ql[k];
            sq[j] = fq_complement(b); sq[k] = fq_complement(a);
            ql[j] = qb; ql[k] = qa;
        }
        __syncwarp();
        if (lane == 0) {
            const int new_front = full - front - seq_len[r];
            CgFastqRecord o = m;
            o.seq_start = m.seq_start - (uint32_t)front + (uint32_t)new_front;
            o.qual_start = m.qual_start - (uint32_t)front + (uint32_t)new_front;
            rec[r] = o;
            origin[2 * r] = new_front;
        }
        const int words = per_read * (int)(sizeof(cg_match_rec) / sizeof(int32_t));
        int32_t *dst = (int32_t *)(matches + (size_t)r * per_read);
        const int32_t *src = (const int32_t *)(matches_rc + (size_t)r * per_read);
        for (int k = lane; k < words; k += 32) dst[k] = src[k];
    }
    if (lane == 0 && replaced) atomicAdd(&counters[11], (unsigned long long)replaced);
}

// quality-driven trimming only (no adapter set): NextseqQualityTrimmer + QualityTrimmer straight on the chunk
__global__ void fq_pretrim_kernel(const uint8_t *buf, const CgFastqRecord *rec, const int32_t *seq_len, long long n_records,
                                  int flags, int cutoff_front, int cutoff_back, int qbase, int32_t *qtrim)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_records) return;
    const CgFastqRecord m = rec[r];
    int s = 0, e = seq_len[r];
    if (flags) pre_trim_core(buf + m.seq_start, buf + m.qual_start, e, flags, cutoff_front, cutoff_back, qbase, &s, &e);
    qtrim[2 * r] = s;
    qtrim[2 * r + 1] = e;
}

// kept interval + failed filters of every record: fq_evaluate_core (cg_fastq_core.cuh); per-read counters
__global__ void fq_evaluate_kernel(const uint8_t *buf, const CgFastqRecord *rec, const int32_t *seq_len, long long n_records,
                                   const cg_match_rec *matches, int times, int slots, const int32_t *qtrim,
                                   CgFastqFilter f, const double *phred, const uint8_t *is_rc, int32_t *interval,
                                   int32_t *keep_interval, int32_t *fail_mask, unsigned long long *counters, int *err)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long c_adapt = 0, c_qbp = 0;
    if (r < n_records) {
        const int n = seq_len[r];
        const int qs = qtrim ? qtrim[2 * r] : 0, qe = qtrim ? qtrim[2 * r + 1] : n;
        c_qbp = (unsigned long long)(n - (qe - qs));
        const FqVerdict v = fq_evaluate_core(buf, rec[r], n, matches ? matches + (size_t)r * times * slots : nullptr, times,
                                             slots, qtrim != nullptr, qs, qe, f, phred);
        if (v.bad_quality) { atomicMin((unsigned int *)&err[1], (unsigned int)r); atomicMax(&err[0], 4); }
        interval[2 * r] = v.start;
        interval[2 * r + 1] = v.stop;
        if (keep_interval) { keep_interval[2 * r] = v.k0; keep_interval[2 * r + 1] = v.k1; }
        fail_mask[r] = v.mask | ((v.last_adapter + 1) << 8) | ((is_rc && is_rc[r]) ? CG_FQ_MASK_RC : 0);
        c_adapt = v.matched;
    }
    c_adapt = __reduce_add_sync(0xFFFFFFFFu, (unsigned)c_adapt);
    for (int d = 16; d; d >>= 1) c_qbp += __shfl_down_sync(0xFFFFFFFFu, c_qbp, d);
    if ((threadIdx.x & 31) == 0) {
        if (c_adapt) atomicAdd(&counters[3], c_adapt);
        if (c_qbp) atomicAdd(&counters[6], c_qbp);
    }
}

// counter slot of filter bit k (the layout of cg_fastq_result): 4 too_short, 5 too_long, 8 too_many_n,
// 9 too_many_expected_errors, 10 casava_filtered, 7 discarded (trimmed / untrimmed)
__device__ __constant__ int kFilterCounter[7] = {4, 5, 8, 9, 10, 7, 7};

// The verdict on a read (mask2 == nullptr) or a pair.  For every enabled filter, in chain order, the pair is
// filtered according to PairedEndFilter (steps.py:105-180): a filter given for one mate only tests that mate;
// otherwise mode 0 "any", 1 "both", 2 "first" (mode_untrimmed: cli.py:859-893 overrides the mode of
// --discard-untrimmed to "both" when only one mate has adapters).  The first filter that fires gets the count.
// out_len = size of the formatted record ("@" name "\n" sequence "\n+\n" qualities "\n") or 0.
__global__ void fq_finish_kernel(long long n_records, const CgFastqRecord *rec1, const int32_t *interval1,
                                 const int32_t *mask1, int enabled1, int32_t *out_len1, unsigned long long *counters1,
                                 const CgFastqRecord *rec2, const int32_t *interval2, const int32_t *mask2, int enabled2,
                                 int32_t *out_len2, unsigned long long *counters2, int mode, int mode_untrimmed,
                                 int rc_suffix, const int32_t *dest, const uint8_t *dest_keep)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int fired = -1;
    unsigned long long bp1 = 0, bp2 = 0;
    unsigned written = 0;
    if (r < n_records) {
        fired = fq_finish_core(mask1[r], mask2 ? mask2[r] : 0, mask2 != nullptr, enabled1, enabled2, mode, mode_untrimmed);
        // a demultiplexer without a writer for this destination drops the pair without counting it (steps.py:574-577)
        if (fired < 0 && dest_keep && !dest_keep[dest[r]]) fired = 7;
        const int left1 = interval1[2 * r + 1] - interval1[2 * r];
        // a reverse-complemented read gets " rc" appended to its name (modifiers.py:295-296)
        const int extra1 = (rc_suffix && (mask1[r] & CG_FQ_MASK_RC)) ? 3 : 0;
        out_len1[r] = fired < 0 ? rec1[r].hdr_len + extra1 + 2 * left1 + 6 : 0;
        if (mask2) {
            const int left2 = interval2[2 * r + 1] - interval2[2 * r];
            const int extra2 = (rc_suffix && (mask2[r] & CG_FQ_MASK_RC)) ? 3 : 0;
            out_len2[r] = fired < 0 ? rec2[r].hdr_len + extra2 + 2 * left2 + 6 : 0;
            bp2 = fired < 0 ? left2 : 0;
        }
        written = fired < 0;
        bp1 = fired < 0 ? left1 : 0;
    }
    const unsigned w = __reduce_add_sync(0xFFFFFFFFu, written);
    for (int d = 16; d; d >>= 1) {
        bp1 += __shfl_down_sync(0xFFFFFFFFu, bp1, d);
        bp2 += __shfl_down_sync(0xFFFFFFFFu, bp2, d);
    }
    // filter counters: one atomic per warp and filter that fired
    for (int k = 0; k < 7; ++k) {
        const unsigned cnt = __popc(__ballot_sync(0xFFFFFFFFu, fired == k));
        if (cnt && (threadIdx.x & 31) == 0) {
            atomicAdd(&counters1[kFilterCounter[k]], (unsigned long long)cnt);
            if (counters2) atomicAdd(&counters2[kFilterCounter[k]], (unsigned long long)cnt);
        }
    }
    if ((threadIdx.x & 31) == 0) {
        if (w) { atomicAdd(&counters1[0], (unsigned long long)w); if (counters2) atomicAdd(&counters2[0], (unsigned long long)w); }
        if (bp1) atomicAdd(&counters1[2], bp1);
        if (bp2 && counters2) atomicAdd(&counters2[2], bp2);
    }
}

// the trimmed records, one warp per record
__global__ void __launch_bounds__(256) fq_write_kernel(const uint8_t *buf, const CgFastqRecord *rec, const int32_t *interval,
                                                        const int64_t *out_off, const int32_t *out_len,
                                                        long long n_records, uint8_t *out, int action,
                                                        const int32_t *keep_interval, const int32_t *mask, int rc_suffix)
{
    const int lane = threadIdx.x & 31;
    const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_records; r += warps) {
        if (out_len[r] == 0) continue;         // filtered
        const long long o = out_off[r];
        const CgFastqRecord m = rec[r];
        const int start = interval[2 * r], left = interval[2 * r + 1] - start;
        uint8_t *p = out + o;
        if (lane == 0) p[0] = '@';
        for (int j = lane; j < m.hdr_len; j += 32) p[1 + j] = buf[m.hdr_start + j];
        p += 1 + m.hdr_len;
        if (rc_suffix && (mask[r] & CG_FQ_MASK_RC)) {
            if (lane < 3) p[lane] = lane == 0 ? ' ' : (lane == 1 ? 'r' : 'c');
            p += 3;
        }
        if (lane == 0) p[0] = '\n';
        if (action == CG_FQ_ACTION_MASK || action == CG_FQ_ACTION_LOWERCASE) {
            // --action=mask / lowercase (modifiers.py:175-193): N / lower case outside the remainder
            const int k0 = keep_interval[2 * r], k1 = keep_interval[2 * r + 1];
            for (int j = lane; j < left; j += 32) {
                uint8_t c = buf[m.seq_start + start + j];
                const bool in = start + j >= k0 && start + j < k1;
                if (action == CG_FQ_ACTION_MASK) c = in ? c : (uint8_t)'N';
                else if ((uint8_t)((c | 0x20) - 'a') < 26) c = in ? (uint8_t)(c & ~0x20) : (uint8_t)(c | 0x20);
                p[1 + j] = c;
            }
        } else {
            for (int j = lane; j < left; j += 32) p[1 + j] = buf[m.seq_start + start + j];
        }
        p += 1 + left;
        if (lane < 3) p[lane] = lane == 1 ? '+' : '\n';
        for (int j = lane; j < left; j += 32) p[3 + j] = buf[m.qual_start + start + j];
        if (lane == 0) p[3 + left] = '\n';
    }
}

// ---- --info-file rows (InfoFileWriter.__call__, steps.py:222-253; SingleMatch.get_info_records, adapters.py:395-417;
// LinkedMatch.get_info_records, adapters.py:1157-1171) --------------------------------------------------------------
// Per match: name, errors, rstart, rstop, before, match, after, adapter name, three quality parts, rc flag; the
// coordinates of every round are applied to info.original_read -- the read AS IT CAME (before -u and the quality
// trimmers; reverse-complemented if the reverse complement was chosen) -- from its first base, and the read is then
// cut the way the match cuts it.  Reads without a match: name, -1, sequence and qualities of the read as written.
// The same walk runs twice: with a counting sink (row bytes per record) and, after a scan, with a writing sink.
struct InfoCountSink {
    long long n = 0;
    __device__ void bytes(const uint8_t *, int len, bool = false) { n += len; }
    __device__ void ch(uint8_t) { n += 1; }
    __device__ void number(int v)
    {
        unsigned u = v < 0 ? 0u - (unsigned)v : (unsigned)v;
        int d = 1;
        while (u >= 10u) { u /= 10u; ++d; }
        n += d + (v < 0 ? 1 : 0);
    }
};
struct InfoWriteSink {                  // all 32 lanes of a warp walk together
    uint8_t *p;
    int lane;
    __device__ void bytes(const uint8_t *src, int len, bool upper = false)
    {
        for (int j = lane; j < len; j += 32) {
            uint8_t c = src[j];
            if (upper && (uint8_t)(c - 'a') < 26) c = (uint8_t)(c & ~0x20);
            p[j] = c;
        }
        p += len;
    }
    __device__ void ch(uint8_t c) { if (lane == 0) *p = c; ++p; }
    __device__ void number(int v)
    {
        unsigned u = v < 0 ? 0u - (unsigned)v : (unsigned)v;
        int d = 1;
        for (unsigned t = u; t >= 10u; t /= 10u) ++d;
        const int total = d + (v < 0 ? 1 : 0);
        if (lane == 0) {
            if (v < 0) p[0] = '-';
            for (int k = total - 1; k >= (v < 0 ? 1 : 0); --k) { p[k] = (uint8_t)('0' + u % 10u); u /= 10u; }
        }
        p += total;
    }
};

// Python's seq[a:b] for a sequence of length len: (start, count)
__device__ __forceinline__ void py_slice(int a, int b, int len, int *start, int *count)
{
    if (a < 0) { a += len; if (a < 0) a = 0; } else if (a > len) a = len;
    if (b < 0) { b += len; if (b < 0) b = 0; } else if (b > len) b = len;
    *start = a;
    *count = b > a ? b - a : 0;
}

struct InfoArgs {
    const uint8_t *buf;
    const CgFastqRecord *rec;
    const int32_t *origin;       // (bases of the read in front of the record, length of the whole read)
    const int32_t *interval;     // the read as written, relative to the record
    const int32_t *mask;
    const cg_match_rec *matches;
    int times, slots;
    const uint8_t *names;        // adapter names, back to back
    const int32_t *name_off;     // n_adapters + 1 offsets into names
    int revcomp;                 // 0: no rc column content; else "1" / "0"
    int rc_suffix;
    int upper_unmatched;         // --action=lowercase writes reads without a match in upper case (modifiers.py:222-223)
    int kind;                    // 0: --info-file rows; 1: --rest-file rows; 2: --wildcard-file rows (names = the adapters' sequences)
    const int32_t *qtrim;        // quality-trimmed interval of the record (the read the cutter saw), or null
    const int32_t *seq_len;
};

template <class Sink>
__device__ void info_rows(const InfoArgs &a, long long r, Sink &out)
{
    const CgFastqRecord m = a.rec[r];
    const int front = a.origin[2 * r], full = a.origin[2 * r + 1];
    const uint8_t *sq = a.buf + m.seq_start - front, *ql = a.buf + m.qual_start - front;
    const bool is_rc = (a.mask[r] & CG_FQ_MASK_RC) != 0;
    auto name = [&]() {
        out.bytes(a.buf + m.hdr_start, m.hdr_len);
        if (is_rc && a.rc_suffix) { out.ch(' '); out.ch('r'); out.ch('c'); }
    };
    int ws = 0, we = full;                              // current_read = original_read[ws:we]
    bool any = false;
    if (a.matches) {
        const cg_match_rec *mr = a.matches + (size_t)r * a.times * a.slots;
        for (int t = 0; t < a.times; ++t) {
            bool round_hit = false;
            for (int k = 0; k < a.slots; ++k) round_hit |= mr[t * a.slots + k].adapter >= 0;
            if (!round_hit) break;
            any = true;
            for (int k = 0; k < a.slots; ++k) {
                const cg_match_rec h = mr[t * a.slots + k];
                if (h.adapter < 0) continue;
                const int cur = we - ws;
                int s0, c0, s1, c1, s2, c2;
                py_slice(0, h.rstart, cur, &s0, &c0);
                py_slice(h.rstart, h.rstop, cur, &s1, &c1);
                py_slice(h.rstop, cur, cur, &s2, &c2);
                name();
                out.ch('\t'); out.number(h.errors);
                out.ch('\t'); out.number(h.rstart);
                out.ch('\t'); out.number(h.rstop);
                out.ch('\t'); out.bytes(sq + ws + s0, c0);
                out.ch('\t'); out.bytes(sq + ws + s1, c1);
                out.ch('\t'); out.bytes(sq + ws + s2, c2);
                out.ch('\t'); out.bytes(a.names + a.name_off[h.adapter], a.name_off[h.adapter + 1] - a.name_off[h.adapter]);
                out.ch('\t'); out.bytes(ql + ws + s0, c0);
                out.ch('\t'); out.bytes(ql + ws + s1, c1);
                out.ch('\t'); out.bytes(ql + ws + s2, c2);
                out.ch('\t');
                if (a.revcomp) out.ch(is_rc ? '1' : '0');
                out.ch('\n');
                // current_read = match.trimmed(current_read)
                if (h.info & 256) { int s, c; py_slice(0, h.rstart, cur, &s, &c); we = ws + c; }
                else { int s, c; py_slice(h.rstop, cur, cur, &s, &c); ws += s; }
            }
        }
    }
    if (!any) {
        const int start = a.interval[2 * r], left = a.interval[2 * r + 1] - start;
        name();
        out.ch('\t'); out.ch('-'); out.ch('1');
        out.ch('\t'); out.bytes(a.buf + m.seq_start + start, left, a.upper_unmatched != 0);
        out.ch('\t'); out.bytes(a.buf + m.qual_start + start, left);
        out.ch('\n');
    }
}

// --rest-file (RestFileWriter, steps.py:193-206; SingleMatch.rest, adapters.py:430-437, 463-470) and --wildcard-file
// rows (WildcardFileWriter, steps.py:209-220; SingleMatch.wildcards, adapters.py:378-393): both look at the LAST match
// of a read and at the sequence that match's round searched (the read after the earlier rounds).
//   rest:     what lies behind a 3' adapter / in front of a 5' adapter, if not empty, then " name"
//   wildcard: the read characters under the adapter's N positions (alignment-free, like the reference), then " name"
template <class Sink>
__device__ void aux_rows(const InfoArgs &a, long long r, Sink &out)
{
    if (!a.matches) return;
    const CgFastqRecord m = a.rec[r];
    int ws = a.qtrim ? a.qtrim[2 * r] : 0, we = a.qtrim ? a.qtrim[2 * r + 1] : a.seq_len[r];
    cg_match_rec last; last.adapter = -1;
    int last_ws = 0, last_we = 0;
    const cg_match_rec *mr = a.matches + (size_t)r * a.times * a.slots;
    for (int t = 0; t < a.times; ++t) {
        bool round_hit = false;
        for (int k = 0; k < a.slots; ++k) {
            const cg_match_rec h = mr[t * a.slots + k];
            if (h.adapter < 0) continue;
            round_hit = true;
            last = h; last_ws = ws; last_we = we;
            const int cur = we - ws;
            int s, c;
            if (h.info & 256) { py_slice(0, h.rstart, cur, &s, &c); we = ws + c; }
            else { py_slice(h.rstop, cur, cur, &s, &c); ws += s; }
        }
        if (!round_hit) break;
    }
    if (last.adapter < 0) return;
    const uint8_t *cur_p = a.buf + m.seq_start + last_ws;
    const int cur = last_we - last_ws;
    const bool is_rc = (a.mask[r] & CG_FQ_MASK_RC) != 0;
    if (a.kind == 1) {
        int s, c;
        if (last.info & 256) py_slice(last.rstop, cur, cur, &s, &c);
        else py_slice(0, last.rstart, cur, &s, &c);
        if (c == 0) return;
        out.bytes(cur_p + s, c);
    } else {
        const uint8_t *aseq = a.names + a.name_off[last.adapter];
        const int alen = a.name_off[last.adapter + 1] - a.name_off[last.adapter];
        for (int i = 0; i < last.astop - last.astart; ++i) {
            const int ai = last.astart + i, ri = last.rstart + i;
            if (ai < 0 || ai >= alen || aseq[ai] != 'N' || ri >= cur) continue;
            const int idx = ri < 0 ? ri + cur : ri;          // Python indexing
            if (idx >= 0) out.ch(cur_p[idx]);
        }
    }
    out.ch(' ');
    out.bytes(a.buf + m.hdr_start, m.hdr_len);
    if (is_rc && a.rc_suffix) { out.ch(' '); out.ch('r'); out.ch('c'); }
    out.ch('\n');
}

__global__ void fq_info_count_kernel(InfoArgs a, long long n_records, int32_t *row_bytes)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_records) return;
    InfoCountSink sink;
    if (a.kind == 0) info_rows(a, r, sink); else aux_rows(a, r, sink);
    row_bytes[r] = (int32_t)sink.n;
}

__global__ void __launch_bounds__(256) fq_info_write_kernel(InfoArgs a, long long n_records, const int64_t *row_off, uint8_t *out)
{
    const int lane = threadIdx.x & 31;
    const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_records; r += warps) {
        InfoWriteSink sink;
        sink.p = out + row_off[r];
        sink.lane = lane;
        if (a.kind == 0) info_rows(a, r, sink); else aux_rows(a, r, sink);
    }
}

// ---- demultiplexing (Demultiplexer.__call__, steps.py:397-409): records go to the output of the adapter of
// their most recent match, reads without a match to "unknown"; inside every output the input order is kept.
// A stable partition of the OUTPUT BYTES: per tile of 256 records the bytes per destination, an exclusive scan
// over (destination-major, tile-minor), then every record's offset = base(destination, tile) + bytes of the
// earlier records of its tile with the same destination.
constexpr int DM_TILE = 256;

// destination of every record: by the adapter of the most recent match of the read (Demultiplexer / PairedDemultiplexer:
// of R1), or of both mates (CombinatorialDemultiplexer, steps.py:565-577): d1 * (n_named2 + 1) + d2; "no match" is the
// last value of its dimension.
__global__ void fq_dest_kernel(const int32_t *mask1, const int32_t *mask2, long long n, const int32_t *adapter_dest1,
                               int n_named1, const int32_t *adapter_dest2, int n_named2, int32_t *dest)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int a1 = CG_FQ_MASK_ADAPTER(mask1[r]);
    int d = a1 < 0 ? n_named1 : adapter_dest1[a1];
    if (mask2) {
        const int a2 = CG_FQ_MASK_ADAPTER(mask2[r]);
        d = d * (n_named2 + 1) + (a2 < 0 ? n_named2 : adapter_dest2[a2]);
    }
    dest[r] = d;
}

__global__ void __launch_bounds__(DM_TILE) fq_demux_hist_kernel(const int32_t *out_len, const int32_t *dest, long long n,
                                                                 int n_dest, long long n_tiles, int32_t *bytes)
{
    extern __shared__ int hist[];
    for (int d = threadIdx.x; d < n_dest; d += DM_TILE) hist[d] = 0;
    __syncthreads();
    const long long r = (long long)blockIdx.x * DM_TILE + threadIdx.x;
    if (r < n && out_len[r] > 0) atomicAdd(&hist[dest[r]], out_len[r]);
    __syncthreads();
    for (int d = threadIdx.x; d < n_dest; d += DM_TILE) bytes[(long long)d * n_tiles + blockIdx.x] = hist[d];
}

__global__ void __launch_bounds__(DM_TILE) fq_demux_offsets_kernel(const int32_t *out_len, const int32_t *dest_of, long long n,
                                                                    long long n_tiles, const int64_t *base, int64_t *out_off)
{
    __shared__ int s_dest[DM_TILE], s_len[DM_TILE];
    const long long r = (long long)blockIdx.x * DM_TILE + threadIdx.x;
    const int len = r < n ? out_len[r] : 0;
    const int dest = len > 0 ? dest_of[r] : -1;
    s_dest[threadIdx.x] = dest;
    s_len[threadIdx.x] = len;
    __syncthreads();
    if (len > 0) {
        long long before = 0;
        for (int j = 0; j < (int)threadIdx.x; ++j) before += s_dest[j] == dest ? s_len[j] : 0;
        out_off[r] = base[(long long)dest * n_tiles + blockIdx.x] + before;
    }
}

// ---- --pair-adapters (PairedAdapterCutter._find_best_match_pair, modifiers.py:480-503) ----
// After adapter pair `pair` was matched alone against both mates (cur1 / cur2, slots1 / slots2 records per read):
// a pair that matches BOTH mates replaces the best pair so far if its score sum is higher, or equal with fewer
// errors.  best1 / best2 hold `slots` records per read (adapter = the pair's number), best_key = (score, errors).
__global__ void fq_pair_select_kernel(long long n, int pair, const cg_match_rec *cur1, int slots1, const cg_match_rec *cur2,
                                      int slots2, cg_match_rec *best1, cg_match_rec *best2, int slots, int32_t *best_key)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    if (pair == 0) {
        for (int k = 0; k < slots; ++k) { best1[r * slots + k].adapter = -1; best2[r * slots + k].adapter = -1; }
        best_key[2 * r] = 0; best_key[2 * r + 1] = 0;
    }
    int score = 0, errors = 0;
    bool has1 = false, has2 = false;
    for (int k = 0; k < slots1; ++k) {
        const cg_match_rec m = cur1[r * slots1 + k];
        if (m.adapter >= 0) { has1 = true; score += m.score; errors += m.errors; }
    }
    for (int k = 0; k < slots2; ++k) {
        const cg_match_rec m = cur2[r * slots2 + k];
        if (m.adapter >= 0) { has2 = true; score += m.score; errors += m.errors; }
    }
    if (!has1 || !has2) return;
    const bool have = best1[r * slots].adapter >= 0 || (slots > 1 && best1[r * slots + 1].adapter >= 0);
    if (have && !(score > best_key[2 * r] || (score == best_key[2 * r] && errors < best_key[2 * r + 1]))) return;
    best_key[2 * r] = score; best_key[2 * r + 1] = errors;
    for (int k = 0; k < slots; ++k) {
        cg_match_rec m; m.adapter = -1; m.astart = m.astop = m.rstart = m.rstop = m.score = m.errors = m.info = 0;
        cg_match_rec a = m, b = m;
        if (k < slots1) { a = cur1[r * slots1 + k]; if (a.adapter >= 0) a.adapter = pair; }
        if (k < slots2) { b = cur2[r * slots2 + k]; if (b.adapter >= 0) b.adapter = pair; }
        best1[r * slots + k] = a;
        best2[r * slots + k] = b;
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
long long cg_fastq_tiles(long long n_bytes) { return (n_bytes + FQ_TILE - 1) / FQ_TILE; }

cudaError_t cg_launch_fastq_index(const uint8_t *d_buf, long long n_bytes, uint32_t *d_tile_counts,
                                  unsigned long long *d_total, uint32_t *d_nl_pos, int phase, cudaStream_t st)
{
    const long long tiles = cg_fastq_tiles(n_bytes);
    if (tiles <= 0) return cudaSuccess;
    if (phase == 0) {
        fq_count_kernel<<<(unsigned)tiles, FQ_THREADS, 0, st>>>(d_buf, n_bytes, d_tile_counts);
        scan_u32_single_cta_kernel<<<1, 1024, 0, st>>>(d_tile_counts, tiles, d_total);
    } else {
        fq_index_kernel<<<(unsigned)tiles, FQ_THREADS, 0, st>>>(d_buf, n_bytes, d_tile_counts, d_nl_pos);
    }
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_records(const uint8_t *d_buf, long long n_bytes, const uint32_t *d_nl_pos, long long n_newlines,
                                    long long n_records, int cut_front, int cut_back, CgFastqRecord *d_rec,
                                    int32_t *d_seq_len, int32_t *d_origin, unsigned long long *d_counters, int *d_err,
                                    cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    fq_records_kernel<<<(unsigned)((n_records + 255) / 256), 256, 0, st>>>(d_buf, n_bytes, d_nl_pos, n_newlines, n_records,
                                                                          cut_front, cut_back, d_rec, d_seq_len, d_origin,
                                                                          d_counters, d_err);
    return cudaGetLastError();
}

long long cg_scan_tiles(long long n) { return (n + SC_TILE - 1) / SC_TILE; }

cudaError_t cg_launch_scan_i32(const int32_t *d_in, long long n, unsigned long long *d_tile_scratch, int64_t *d_out,
                               cudaStream_t st)
{
    if (n <= 0) return cudaMemsetAsync(d_out, 0, sizeof(int64_t), st);
    const long long tiles = cg_scan_tiles(n);
    scan_tile_sums_kernel<<<(unsigned)tiles, 256, 0, st>>>(d_in, n, d_tile_scratch);
    scan_u64_single_cta_kernel<<<1, 1024, 0, st>>>(d_tile_scratch, tiles);
    scan_apply_kernel<<<(unsigned)tiles, 256, 0, st>>>(d_in, n, d_tile_scratch, d_out);
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_gather(const uint8_t *d_buf, const CgFastqRecord *d_rec, const int64_t *d_offsets,
                                   long long n_records, uint8_t *d_seq, uint8_t *d_qual, int rc, cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    long long grid = (n_records + 7) / 8;
    grid = cg_grid_cap(grid, 16);
    fq_gather_kernel<<<(unsigned)grid, 256, 0, st>>>(d_buf, d_rec, d_offsets, n_records, d_seq, d_qual, rc);
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_fold_qtrim(CgFastqRecord *d_rec, int32_t *d_seq_len, const int32_t *d_qtrim, long long n_records,
                                       int32_t *d_origin, unsigned long long *d_counters, cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    fq_fold_qtrim_kernel<<<(unsigned)((n_records + 255) / 256), 256, 0, st>>>(d_rec, d_seq_len, d_qtrim, n_records, d_origin,
                                                                             d_counters);
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_revcomp_commit(uint8_t *d_buf, CgFastqRecord *d_rec, const int32_t *d_seq_len, int32_t *d_origin,
                                           long long n_records, cg_match_rec *d_matches, const cg_match_rec *d_matches_rc,
                                           int per_read, uint8_t *d_is_rc, unsigned long long *d_counters, cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    long long grid = (n_records + 7) / 8;
    grid = cg_grid_cap(grid, 16);
    fq_revcomp_commit_kernel<<<(unsigned)grid, 256, 0, st>>>(d_buf, d_rec, d_seq_len, d_origin, n_records, d_matches,
                                                             d_matches_rc, per_read, d_is_rc, d_counters);
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_pretrim(const uint8_t *d_buf, const CgFastqRecord *d_rec, const int32_t *d_seq_len,
                                    long long n_records, int flags, int cutoff_front, int cutoff_back, int qbase,
                                    int32_t *d_qtrim, cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    fq_pretrim_kernel<<<(unsigned)((n_records + 127) / 128), 128, 0, st>>>(d_buf, d_rec, d_seq_len, n_records, flags,
                                                                          cutoff_front, cutoff_back, qbase, d_qtrim);
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_evaluate(const uint8_t *d_buf, const CgFastqRecord *d_rec, const int32_t *d_seq_len,
                                     long long n_records, const cg_match_rec *d_matches, int times, int slots,
                                     const int32_t *d_qtrim, CgFastqFilter f, const double *d_phred, const uint8_t *d_is_rc,
                                     int32_t *d_interval, int32_t *d_keep_interval, int32_t *d_fail_mask,
                                     unsigned long long *d_counters, int *d_err, cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    fq_evaluate_kernel<<<(unsigned)((n_records + 255) / 256), 256, 0, st>>>(d_buf, d_rec, d_seq_len, n_records, d_matches,
                                                                           times, slots, d_qtrim, f, d_phred, d_is_rc,
                                                                           d_interval, d_keep_interval, d_fail_mask,
                                                                           d_counters, d_err);
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_finish(long long n_records, const CgFastqRecord *d_rec1, const int32_t *d_interval1,
                                   const int32_t *d_mask1, int enabled1, int32_t *d_out_len1,
                                   unsigned long long *d_counters1, const CgFastqRecord *d_rec2,
                                   const int32_t *d_interval2, const int32_t *d_mask2, int enabled2, int32_t *d_out_len2,
                                   unsigned long long *d_counters2, int mode, int mode_untrimmed, int rc_suffix,
                                   const int32_t *d_dest, const uint8_t *d_dest_keep, cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    fq_finish_kernel<<<(unsigned)((n_records + 255) / 256), 256, 0, st>>>(n_records, d_rec1, d_interval1, d_mask1, enabled1,
                                                                         d_out_len1, d_counters1, d_rec2, d_interval2,
                                                                         d_mask2, enabled2, d_out_len2, d_counters2, mode,
                                                                         mode_untrimmed, rc_suffix, d_dest, d_dest_keep);
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_write(const uint8_t *d_buf, const CgFastqRecord *d_rec, const int32_t *d_interval,
                                  const int64_t *d_out_off, const int32_t *d_out_len, long long n_records,
                                  uint8_t *d_out, int action, const int32_t *d_keep_interval, const int32_t *d_mask,
                                  int rc_suffix, cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    long long grid = (n_records + 7) / 8;
    grid = cg_grid_cap(grid, 16);
    fq_write_kernel<<<(unsigned)grid, 256, 0, st>>>(d_buf, d_rec, d_interval, d_out_off, d_out_len, n_records, d_out, action,
                                                    d_keep_interval, d_mask, rc_suffix);
    return cudaGetLastError();
}

long long cg_demux_tiles(long long n_records) { return (n_records + DM_TILE - 1) / DM_TILE; }

cudaError_t cg_launch_fastq_dest(const int32_t *d_mask1, const int32_t *d_mask2, long long n_records,
                                 const int32_t *d_adapter_dest1, int n_named1, const int32_t *d_adapter_dest2, int n_named2,
                                 int32_t *d_dest, cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    fq_dest_kernel<<<(unsigned)((n_records + 255) / 256), 256, 0, st>>>(d_mask1, d_mask2, n_records, d_adapter_dest1, n_named1,
                                                                       d_adapter_dest2, n_named2, d_dest);
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_demux(int phase, const int32_t *d_out_len, const int32_t *d_dest, long long n_records,
                                  int n_dest, int32_t *d_bytes, const int64_t *d_base, int64_t *d_out_off, cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    const long long tiles = cg_demux_tiles(n_records);
    if (phase == 0)
        fq_demux_hist_kernel<<<(unsigned)tiles, DM_TILE, (size_t)n_dest * sizeof(int), st>>>(d_out_len, d_dest, n_records,
                                                                                           n_dest, tiles, d_bytes);
    else
        fq_demux_offsets_kernel<<<(unsigned)tiles, DM_TILE, 0, st>>>(d_out_len, d_dest, n_records, tiles, d_base, d_out_off);
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_pair_select(long long n_records, int pair, const cg_match_rec *d_cur1, int slots1,
                                        const cg_match_rec *d_cur2, int slots2, cg_match_rec *d_best1, cg_match_rec *d_best2,
                                        int slots, int32_t *d_best_key, cudaStream_t st)
{
    if (n_records <= 0) return cudaSuccess;
    fq_pair_select_kernel<<<(unsigned)((n_records + 255) / 256), 256, 0, st>>>(n_records, pair, d_cur1, slots1, d_cur2, slots2,
                                                                              d_best1, d_best2, slots, d_best_key);
    return cudaGetLastError();
}

cudaError_t cg_launch_fastq_info(int phase, const uint8_t *d_buf, const CgFastqRecord *d_rec, const int32_t *d_origin,
                                 const int32_t *d_interval, const int32_t *d_mask, const cg_match_rec *d_matches, int times,
                                 int slots, const uint8_t *d_names, const int32_t *d_name_off, int revcomp, int rc_suffix,
                                 int upper_unmatched, long long n_records, int32_t *d_row_bytes, const int64_t *d_row_off,
                                 uint8_t *d_out, cudaStream_t st, int kind, const int32_t *d_qtrim, const int32_t *d_seq_len)
{
    if (n_records <= 0) return cudaSuccess;
    InfoArgs a;
    a.kind = kind; a.qtrim = d_qtrim; a.seq_len = d_seq_len;
    a.buf = d_buf; a.rec = d_rec; a.origin = d_origin; a.interval = d_interval; a.mask = d_mask; a.matches = d_matches;
    a.times = times; a.slots = slots; a.names = d_names; a.name_off = d_name_off; a.revcomp = revcomp;
    a.rc_suffix = rc_suffix; a.upper_unmatched = upper_unmatched;
    if (phase == 0) {
        fq_info_count_kernel<<<(unsigned)((n_records + 127) / 128), 128, 0, st>>>(a, n_records, d_row_bytes);
    } else {
        long long grid = (n_records + 7) / 8;
        grid = cg_grid_cap(grid, 16);
        fq_info_write_kernel<<<(unsigned)grid, 256, 0, st>>>(a, n_records, d_row_off, d_out);
    }
    return cudaGetLastError();
}
