// cg_pscan.cuh -- body of the bit-plane first stage of the split pipeline.
//
// Included twice: by cg_kernels.cu, which instantiates it with RuntimePlaneProg (the interpreter of the op list
// in the adapter blob: any adapter, compiled ahead of time), and by the translation unit cg_jit.cpp builds per
// adapter set for NVRTC, where the program is a sequence of plane_chain_step / plane_emit calls with literal
// arguments that the compiler folds into straight-line code.
#pragma once
#include "cg_core.cuh"
#include "cg_args.h"
#include "cg_device.cuh"

struct ScanSmem { size_t blob_off, enc_off, stats_off, warp_off, warp_stride, bar_rel, seq_rel, qual_rel, total; };

// ------------------------------------------------------------------------------------------
// cg_pscan_kernel -- the bit-plane first stage (plane_scan_core in cg_core.cuh) in the frame of
// cg_scan_kernel: per-warp TMA-staged mini-tiles of 32 reads, one lane per read.  Reads it settles
// ("no match": 47 % of the benchmark's reads; exact occurrence: 41 %) get their record here; the rest
// (12 %) append a CG_TASK_PLANES task with the hit mask M, from which cg_list_kernel<plan> derives the DP runs
// (reads the planes cannot represent -- empty or longer than 32 W -- go as CG_TASK_RESCAN).
// A margin in front of every warp's tile keeps the right-aligned plane loads of the tile's first read
// inside shared memory.
// ------------------------------------------------------------------------------------------
#define CG_PSCAN_MARGIN 272
#ifndef CG_PSCAN_BLOCKS
#define CG_PSCAN_BLOCKS 8     // resident CTAs per SM the 5-word variant is compiled for (64 registers)
#endif
#define CG_TASK_RESCAN 0x100u     // the plan stage must scan the read itself (shift-and scan_core)
#define CG_TASK_BYTES 0x400u      // the task carries the read window itself: 2 W + 1 16-byte pieces after the four header
                                  // words (the aligned stretch of shared memory that covers the 32 W characters in front
                                  // of the window's end); td.y = offset of the window's first character in them.  The
                                  // plan stage then streams its input instead of gathering windows from all over HBM.
#define CG_TASK_PLANES 0x200u     // a 4 x uint4 task of cg_pscan_kernel: {read, window offset hi, lo, length},
                                  // {M0, flags, M1, M2}, {M3 .. M6}, {M7, window offset, 0, 0} with M = PlaneOut::M (+ CG_TASK_BYTES);
                                  // flags bits 12-15: plane words W, bit 20: PlaneOut::end_hit, bit 21: PlaneOut::no_end
// ------------------------------------------------------------------------------------------
// Fused statistics (one plain adapter, one round, one slot: the passes choose_schedule fuses them into): per-CTA
// histograms in shared memory, flushed once at the end of the CTA.  Layout: read lengths (max_len + 1), removed
// lengths for 5' then for 3' matches ((max_len + 1) x cols each: cols = 1 keeps 0 errors only, kmax + 1 every error
// count), adjacent bases (8), then 8 64-bit scalars (reads, matches, bases, quality-trimmed, adapter bases).
// ------------------------------------------------------------------------------------------
struct StatsSmem { uint32_t *hlen, *hrem, *hadj; unsigned long long *scal; };
__host__ __device__ inline size_t stats_smem_bytes(int max_len, int cols)
{
    return cg_align_up((size_t)((1 + 2 * cols) * (max_len + 1) + 8) * sizeof(uint32_t), 8) + 8 * sizeof(unsigned long long);
}
__device__ __forceinline__ StatsSmem stats_smem_view(uint8_t *base, int max_len, int cols)
{
    StatsSmem H;
    H.hlen = (uint32_t *)base;
    H.hrem = H.hlen + (max_len + 1);
    H.hadj = H.hrem + 2 * cols * (max_len + 1);
    H.scal = (unsigned long long *)(base + stats_smem_bytes(max_len, cols) - 8 * sizeof(unsigned long long));
    return H;
}
// (before the CTA's first __syncthreads)
__device__ __forceinline__ void stats_smem_zero(const StatsSmem &H, int max_len, int cols)
{
    for (int i = threadIdx.x; i < (1 + 2 * cols) * (max_len + 1) + 8; i += CG_NT) H.hlen[i] = 0;
    if (threadIdx.x < 8) H.scal[threadIdx.x] = 0;
}
// One warp's reads.  fin: this lane's final-length bin (-1 = nothing to count); its contributions to the scalars,
// packed for three warp sums: p1 = bases | quality-trimmed bases << 16, p2 = adapter bases | read << 16 | match << 22,
// p3 = one 6-bit count per adjacent-base class (the fields hold the sums of 32 reads of at most 256 bases).  The
// removed-length bins are the caller's.  All 32 lanes call it.
__device__ __forceinline__ void stats_warp_add(const StatsSmem &H, int fin, uint32_t p1, uint32_t p2, uint32_t p3)
{
    const int lane = threadIdx.x & 31;
    // most reads of a tile end in the same length bin: one shared-memory atomic for the bin of the first
    // counted lane and its peers, one each for the others
    const uint32_t counted = __ballot_sync(0xffffffffu, fin >= 0);
    if (!counted) return;
    const int leader = __ffs(counted) - 1;
    const int common = __shfl_sync(0xffffffffu, fin, leader);
    const uint32_t same = __ballot_sync(0xffffffffu, fin == common);
    if (lane == leader) atomicAdd(&H.hlen[common], (uint32_t)__popc(same));
    else if (fin >= 0 && fin != common) atomicAdd(&H.hlen[fin], 1u);
    const uint32_t s1 = __reduce_add_sync(0xffffffffu, p1);
    const uint32_t s2 = __reduce_add_sync(0xffffffffu, p2);
    const uint32_t s3 = __reduce_add_sync(0xffffffffu, p3);
    // lane L adds scalar L of the warp to the CTA's counters (no register held across the tile loop):
    // reads, matches, bases, quality-trimmed, adapter bases, adjacent x 5
    uint32_t mine_add = 0;
    switch (lane) {
    case 0: mine_add = (s2 >> 16) & 63u; break;
    case 1: mine_add = s2 >> 22; break;
    case 2: mine_add = s1 & 0xffffu; break;
    case 3: mine_add = s1 >> 16; break;
    case 4: mine_add = s2 & 0xffffu; break;
    default: if (lane < 10) mine_add = (s3 >> (6 * (lane - 5))) & 63u; break;
    }
    if (mine_add) {
        if (lane < 5) atomicAdd(&H.scal[lane], (unsigned long long)mine_add);
        else atomicAdd(&H.hadj[lane - 5], mine_add);
    }
}
// The CTA's counters into the vector (one adapter: lengths, then its 5' block and its 3' block); after a __syncthreads.
__device__ __forceinline__ void stats_cta_flush(const StatsSmem &H, int max_len, int kmax, int cols, unsigned long long *stats)
{
    // reads, matches, bases, quality-trimmed, adapter bases -> stats[0, 2, 1, 3, 4]
    if (threadIdx.x < 5 && H.scal[threadIdx.x])
        atomicAdd(&stats[threadIdx.x == 1 ? 2 : (threadIdx.x == 2 ? 1 : threadIdx.x)], H.scal[threadIdx.x]);
    unsigned long long *hist = stats + CG_STATS_SCALARS;
    const long long end_size = cg_stats_end_size(max_len, kmax);
    for (int i = threadIdx.x; i <= max_len; i += CG_NT) {
        const uint32_t v = H.hlen[i];
        if (v) atomicAdd(&hist[i], (unsigned long long)v);
    }
    for (int i = threadIdx.x; i < 2 * cols * (max_len + 1); i += CG_NT) {
        const uint32_t w = H.hrem[i];
        const int kind = i / (cols * (max_len + 1)), j = i - kind * cols * (max_len + 1);
        if (w) atomicAdd(&hist[(max_len + 1) + kind * end_size + CG_STATS_ADJ + (long long)(j / cols) * (kmax + 1) + j % cols],
                         (unsigned long long)w);
    }
    if (threadIdx.x < 8 && H.hadj[threadIdx.x])
        atomicAdd(&hist[(max_len + 1) + end_size + threadIdx.x], (unsigned long long)H.hadj[threadIdx.x]);
}

// stats_max_len >= 0: room for the per-CTA histograms of the fused statistics, removed lengths at 0 errors only
__host__ __device__ inline ScanSmem pscan_smem_layout(uint32_t blob_bytes, int mini_cap, bool has_qual, int stats_max_len = -1)
{
    ScanSmem L;
    size_t o = 0;
    L.blob_off = o; o += cg_align_up(blob_bytes, 16);
    L.enc_off = o; o += 768;
    L.stats_off = o;
    if (stats_max_len >= 0) o += stats_smem_bytes(stats_max_len, 1);
    o = cg_align_up(o, 128);
    L.warp_off = o;
    size_t w = 0;
    L.bar_rel = w; w += 16;
    w = cg_align_up(w, 128);
    w += CG_PSCAN_MARGIN;
    L.seq_rel = w; w += (size_t)mini_cap;
    L.qual_rel = w; if (has_qual) w += (size_t)mini_cap;
    L.warp_stride = cg_align_up(w, 128);
    L.total = L.warp_off + (CG_NT / 32) * L.warp_stride;
    return L;
}

// ------------------------------------------------------------------------------------------
// Quality trimming of a warp's 32 reads (quality_trim_index, qualtrim.pyx:22-73; the per-lane form is
// quality_trim_core).  The scan from an end stops at the first negative partial sum: for a good read after ONE
// character, for a read with a bad tail after the whole tail -- and a warp runs as long as its slowest lane.  So
// every lane looks at its first character itself, and the reads that go on (typically 3 of 32) are then scanned by
// the whole warp, 32 characters per step: inclusive prefix sums by shuffles, the first negative sum by ballot, the
// (first) maximum by a warp reduction -- exactly the loop's `if (s < 0) break; if (s > best) { best = s; pos = i }`.
// DIR = +1: the 5' scan (returns the new start), -1: the 3' scan (returns the new stop).  q_smem: shared-memory
// address of this lane's qualities.  All 32 lanes must call it.
// ------------------------------------------------------------------------------------------
template <int DIR>
__device__ __forceinline__ int trim_scan_warp(uint32_t q_smem, int n, int cutoff, int base, int lane)
{
#if defined(__CUDA_ARCH__)
    int res = DIR > 0 ? 0 : n;
    bool more = false;
    if (n > 0) {
        const int d0 = cutoff - ((int)(signed char)cg_lds_u8(q_smem + (uint32_t)(DIR > 0 ? 0 : n - 1)) - base);
        more = d0 >= 0;
    }
    uint32_t todo = __ballot_sync(0xffffffffu, more);
    while (todo) {
        const int T = __ffs(todo) - 1;
        todo &= todo - 1;
        const uint32_t qT = __shfl_sync(0xffffffffu, q_smem, T);
        const int nT = __shfl_sync(0xffffffffu, n, T);
        int carry = 0, best = 0, resT = DIR > 0 ? 0 : nT;
        for (int j0 = 0; j0 < nT; j0 += 32) {
            const int j = j0 + lane;
            const bool valid = j < nT;
            int P = 0;
            if (valid) P = cutoff - ((int)(signed char)cg_lds_u8(qT + (uint32_t)(DIR > 0 ? j : nT - 1 - j)) - base);
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, P, o);
                if (lane >= o) P += t;
            }
            P += carry;
            const uint32_t neg = __ballot_sync(0xffffffffu, valid && P < 0);
            const int first_neg = neg ? __ffs(neg) - 1 : 32;
            const bool ok = valid && lane < first_neg;
            const int M = __reduce_max_sync(0xffffffffu, ok ? P : (int)0x80000000);
            if (M > best) {
                best = M;
                const int w = __ffs(__ballot_sync(0xffffffffu, ok && P == M)) - 1;
                resT = DIR > 0 ? j0 + w + 1 : nT - 1 - (j0 + w);
            }
            if (first_neg < 32) break;
            carry = __shfl_sync(0xffffffffu, P, 31);
        }
        if (lane == T) res = resT;
    }
    return res;
#else
    return 0;       // (host pass of nvcc: never called)
#endif
}

// pre_trim_core for a whole warp (NextSeq trimming stays per lane; it only runs with --nextseq-trim)
__device__ __forceinline__ void pre_trim_warp(const uint8_t *seq, const uint8_t *qual, int n, int flags, int cutoff_front,
                                              int cutoff_back, int qbase, int lane, int *s_out, int *e_out)
{
    const int base = qbase & 255;
    int start = 0, stop = n;
    if (flags & 2) stop = nextseq_trim_core(seq, qual, n, qbase >> 8, base);
    if (flags & 1) {
        const uint32_t q_smem = (uint32_t)__cvta_generic_to_shared(qual);
        const int nq = stop;
        start = trim_scan_warp<+1>(q_smem, nq, cutoff_front, base, lane);
        stop = trim_scan_warp<-1>(q_smem, nq, cutoff_back, base, lane);
        if (start >= stop) { start = 0; stop = 0; }                 // qualtrim.pyx:71-72
    }
    *s_out = start; *e_out = stop;
}

// STATS: the variant that counts the statistics of the reads it settles (a.stats, see below); the other variant carries
// none of that code.
template <bool HAS_QUAL, int W, class Prog, bool STATS = false>
__device__ __forceinline__ void cg_pscan_body(const CgKernelArgs &a)
{
    extern __shared__ __align__(128) uint8_t smem[];
    const ScanSmem L = pscan_smem_layout(a.blob_bytes, a.mini_cap, HAS_QUAL, (STATS && a.stats) ? a.stats_max_len : -1);
    uint8_t *s_blob = smem + L.blob_off;
    uint8_t *s_enc = smem + L.enc_off;
    const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
    uint8_t *wbase = smem + L.warp_off + (size_t)wib * L.warp_stride;
    uint64_t *bars = (uint64_t *)(wbase + L.bar_rel);
    uint8_t *s_seq = wbase + L.seq_rel;
    uint8_t *s_qual = wbase + L.qual_rel;
    // fused statistics: per-CTA histograms, flushed at the end (stats_smem_view; the reads settled here have 0 errors).
    // Everything is re-derived from the kernel arguments where it is used: nothing of it may occupy a register across
    // the plane code.
#define CG_PSCAN_STATS_VIEW                                                                                              \
    const int st_len = a.stats_max_len;                                                                                  \
    const StatsSmem H = stats_smem_view(smem + pscan_smem_layout(a.blob_bytes, a.mini_cap, HAS_QUAL, st_len).stats_off, st_len, 1);
    if (STATS && a.stats) {
        CG_PSCAN_STATS_VIEW
        stats_smem_zero(H, st_len, 1);
    }
    for (uint32_t i = tid; i < a.blob_bytes / 16; i += CG_NT) ((uint4 *)s_blob)[i] = ((const uint4 *)a.blob)[i];
    for (uint32_t i = tid; i < 768 / 16; i += CG_NT) ((uint4 *)s_enc)[i] = ((const uint4 *)a.enc)[i];
    if (lane == 0) {
        mbar_init(&bars[0], 1);
        fence_barrier_init();
    }
    __syncthreads();
    const SetView S = make_set_view(s_blob, a.masks64, s_enc, a.index);
    const CgAdapter &A = S.ad[0];
    const uint32_t *prog = plane_program(S);
    const int n_prog = S.h->plane_count, pflags = S.h->plane_flags;
    const uint8_t *ref = S.pool + A.ref_off;
    const bool always_pass = A.pf_count == 0;

    const long long n_reads = a.n_reads;
    const long long n_mt = (n_reads + 31) / 32;
    const long long warps_total = (long long)gridDim.x * (CG_NT / 32);
    const long long wg = (long long)blockIdx.x * (CG_NT / 32) + wib;
    const uintptr_t seq_base = (uintptr_t)a.seq, qual_base = (uintptr_t)a.qual;

    auto issue = [&](long long mt) {
        const long long r0 = mt * 32;
        const long long r1 = (r0 + 32 < n_reads) ? r0 + 32 : n_reads;
        const long long b0 = a.offsets[r0], b1 = a.offsets[r1];
        if (b1 <= b0) return;
        const uintptr_t sa0 = (seq_base + b0) & ~(uintptr_t)15;
        const uint32_t bytes = (uint32_t)(((seq_base + b1 + 15) & ~(uintptr_t)15) - sa0);
        uint32_t qbytes = 0;
        uintptr_t qa0 = 0;
        if (HAS_QUAL) {
            qa0 = (qual_base + b0) & ~(uintptr_t)15;
            qbytes = (uint32_t)(((qual_base + b1 + 15) & ~(uintptr_t)15) - qa0);
        }
        mbar_expect_tx(&bars[0], bytes + qbytes);
        tma_load_1d(s_seq, (const void *)sa0, bytes, &bars[0]);
        if (HAS_QUAL) tma_load_1d(s_qual, (const void *)qa0, qbytes, &bars[0]);
    };
    if (lane == 0 && wg < n_mt) issue(wg);
    uint32_t phase0 = 0;
    for (long long mt = wg; mt < n_mt; mt += warps_total) {
        const long long r0 = mt * 32;
        const long long r1 = (r0 + 32 < n_reads) ? r0 + 32 : n_reads;
        const long long r = r0 + lane;
        const long long b0 = a.offsets[r0], b1 = a.offsets[r1];
        long long o0 = 0, o1 = 0;
        if (r < n_reads) { o0 = a.offsets[r]; o1 = a.offsets[r + 1]; }
        const uintptr_t sa0 = (seq_base + b0) & ~(uintptr_t)15;
        if (b1 > b0) { mbar_wait(&bars[0], phase0); phase0 ^= 1; }
        // quality trimming: the whole warp together (lanes without a read take part with an empty one)
        int q_ts = 0, q_te = 0;
        if (HAS_QUAL && a.quality_trim) {
            const uintptr_t qa0 = (qual_base + b0) & ~(uintptr_t)15;
            const bool has = r < n_reads;
            pre_trim_warp(s_seq + (size_t)(has ? (seq_base + o0) - sa0 : 0), s_qual + (size_t)(has ? (qual_base + o0) - qa0 : 0),
                          has ? (int)(o1 - o0) : 0, a.quality_trim, a.cutoff_front, a.cutoff_back, a.qbase, lane, &q_ts, &q_te);
        }
        int cls = CG_PLANE_NONE, s0 = 0, ts = 0, te = 0;
        int st_fin = -1;                              // fused statistics: this lane's final-length bin, -1 = none
        uint32_t st_p1 = 0, st_p2 = 0, st_p3 = 0;     // ... and its contributions to the scalars, packed (below)
        uint32_t t_flags = 4u | CG_TASK_RESCAN;
        uint32_t tm[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        uint32_t win_region = 0, win_off = 0;         // shared-memory address of the carried bytes, window offset in them
        bool mine = false;
        if (r < n_reads) {
            mine = true;
            const int n = (int)(o1 - o0);
            const uint32_t off = (uint32_t)((seq_base + o0) - sa0);
            ts = 0; te = n;
            if (HAS_QUAL && a.quality_trim) { ts = q_ts; te = q_te; }
            if (a.qtrim) { a.qtrim[2 * r] = ts; a.qtrim[2 * r + 1] = te; }
            if (a.view) { ts = a.view[2 * r]; te = a.view[2 * r + 1]; }
            const int nn = te - ts;
            if (nn >= 1 && nn <= 32 * W) {
                const PlaneOut po = plane_scan_core<W, Prog>(prog, n_prog, pflags, A.m, ref, s_seq + off + te, nn, always_pass);
                cls = po.cls; s0 = po.s0;
                if (po.bad & 0x80808080u) atomicOr(a.err_flag, 1);
                if (cls == CG_PLANE_SLOW) {
                    t_flags = 4u | CG_TASK_PLANES | (a.task_rec > 4 ? CG_TASK_BYTES : 0u) | ((uint32_t)W << 12) |
                              ((uint32_t)po.end_hit << 20) | ((uint32_t)po.no_end << 21);
                    const uint32_t wend = smem_u32(s_seq + off + te);
                    win_region = (wend - 32u * W) & ~15u;
                    win_off = (wend - (uint32_t)nn) - win_region;
#pragma unroll
                    for (int b = 0; b < 8; ++b) tm[b] = po.M[b];
                }
            } else {
                cls = CG_PLANE_SLOW;                 // (empty or over-long window: the exact path checks its bytes)
                uint32_t bad = 0;
                for (int i = ts; i < te; ++i) bad |= s_seq[off + i];
                if (bad & 0x80u) atomicOr(a.err_flag, 1);
            }
            if (cls != CG_PLANE_SLOW) {
                CgHit hit; hit.adapter = -1; hit.remove = 0;
                hit.astart = hit.astop = hit.rstart = hit.rstop = hit.score = hit.errors = 0;
                if (cls == CG_PLANE_EXACT) hit_exact(A, nn, s0, hit);
                else if (cls == CG_PLANE_OVERLAP) hit_end_overlap(A, nn, s0, hit);
                store_hit(a.out + (size_t)r * a.slots, hit, 0, nn);
                if (STATS && a.stats) {
                    // what stats_read_core adds for this read (one round, one slot), packed as stats_warp_add takes it
                    CG_PSCAN_STATS_VIEW
                    st_p1 = (uint32_t)n | ((a.quality_trim && a.qtrim) ? (uint32_t)(n - nn) << 16 : 0u);
                    st_p2 = 1u << 16;
                    int fin = nn;
                    if (hit.adapter >= 0) {
                        // (a literal where the program fixes the adapter's kind: one of the two branches is dead)
                        const int kind = Prog::remove_kind(A.remove);
                        const bool after = kind == CGK_REMOVE_AUTO ? hit.remove == CGK_REMOVE_AFTER : kind == CGK_REMOVE_AFTER;
                        int removed = after ? nn - hit.rstart : hit.rstop;
                        removed = removed < 0 ? 0 : removed;
                        st_p2 |= (uint32_t)removed | (1u << 22);
                        atomicAdd(&H.hrem[(after ? st_len + 1 : 0) + (removed > st_len ? st_len : removed)], 1u);
                        if (after) {
                            int k = 4;
                            if (hit.rstart > 0) {
                                const uint8_t c = s_seq[off + ts + hit.rstart - 1];
                                k = c == 'A' ? 0 : (c == 'C' ? 1 : (c == 'G' ? 2 : (c == 'T' ? 3 : 4)));
                            }
                            st_p3 = 1u << (6 * k);
                            fin = hit.rstart;
                        } else {
                            fin = nn - hit.rstop;
                        }
                    }
                    st_fin = fin < 0 ? 0 : (fin > st_len ? st_len : fin);
                }
            }
        }
        if (STATS && a.stats) {
            CG_PSCAN_STATS_VIEW
            stats_warp_add(H, st_fin, st_p1, st_p2, st_p3);
        }
        const bool slow = mine && cls == CG_PLANE_SLOW;
        // two lists: reads with locator hits (and everything the planes could not look at) from the front, reads
        // without from the back -- the plan stage does different work for the two kinds, and a warp is as slow as
        // its slowest lane
        const bool kind_b = slow && a.task_count_b != nullptr && (t_flags & CG_TASK_PLANES) && !(t_flags & (1u << 20)) &&
                            (tm[0] | tm[1] | tm[2] | tm[3] | tm[4] | tm[5] | tm[6] | tm[7]) == 0u;
        const uint32_t ballot_a = __ballot_sync(0xffffffffu, slow && !kind_b);
        const uint32_t ballot_b = __ballot_sync(0xffffffffu, kind_b);
        if (ballot_a | ballot_b) {
            unsigned long long base_a = 0, base_b = 0;
            if (lane == 0) {
                if (ballot_a) base_a = atomicAdd(a.task_count, (unsigned long long)__popc(ballot_a));
                if (ballot_b) base_b = atomicAdd(a.task_count_b, (unsigned long long)__popc(ballot_b));
            }
            base_a = __shfl_sync(0xffffffffu, base_a, 0);
            base_b = __shfl_sync(0xffffffffu, base_b, 0);
            if (slow) {
                const uint32_t below = (1u << lane) - 1u;
                const unsigned long long slot = kind_b
                    ? (unsigned long long)a.task_cap - 1ull - (base_b + __popc(ballot_b & below))
                    : base_a + __popc(ballot_a & below);
                uint4 *rec = a.tasks + (size_t)a.task_rec * slot;
                const unsigned long long woff = (unsigned long long)(o0 + ts);     // where the window lies in the batch
                rec[0] = make_uint4((uint32_t)r, (uint32_t)(woff >> 32), (uint32_t)woff, (uint32_t)(te - ts));
                rec[1] = make_uint4(tm[0], t_flags, tm[1], tm[2]);
                rec[2] = make_uint4(tm[3], tm[4], tm[5], tm[6]);
                rec[3] = make_uint4(tm[7], win_off, 0u, 0u);
                if (t_flags & CG_TASK_BYTES) {
#pragma unroll
                    for (int c = 0; c < 2 * W + 1; ++c) {
                        uint4 v;
                        asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(win_region + 16u * (uint32_t)c));
                        rec[4 + c] = v;
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) {
            const long long next = mt + warps_total;
            if (next < n_mt) issue(next);
        }
    }
    if (STATS && a.stats) {
        CG_PSCAN_STATS_VIEW
        __syncthreads();
        stats_cta_flush(H, st_len, a.stats_kmax, 1, a.stats);
    }
}

