// cg_kernels.cu -- sm_90a (H100) kernels of the adapter-trimming hot path.
//
// cg_trim_fast_kernel   the fused pass: quality trim -> k-mer prefilter -> banded DP ->
//                       best-adapter selection, one lane per read, persistent CTAs.
//                       Read bytes are staged HBM -> shared memory as one contiguous 16-byte
//                       aligned range per 128-read tile with TMA 1-D bulk copies
//                       (cp.async.bulk + mbarrier complete_tx), double buffered so the copy of
//                       tile t+1 overlaps the compute of tile t.  The adapter tables (a few
//                       hundred bytes) and each lane's DP column live in shared memory.
//                       No tensor cores: this is small-integer DP, not a contraction.
// cg_trim_generic_kernel  same per-read code (cg_core.cuh) for configurations the fused kernel
//                       does not cover (wide cells for --no-indels / very long reads):
//                       reads straight from HBM, DP columns in an HBM scratch.
// plus the stand-alone batched KmerFinder / quality_trim_index kernels and the statistics
// reduction.
#include <atomic>

#include "cg_kernels.cuh"
#include "cg_device.cuh"
#include "cg_pscan.cuh"   // (ScanSmem, cg_pscan_body)

// shared-memory carve-up of the fused kernel
struct FastSmem {
    size_t bar_off, cnt_off, task_off, blob_off, enc_off, seq_off, qual_off, col_off, total;
};
__host__ __device__ inline FastSmem fast_smem_layout(uint32_t blob_bytes, int tile_cap, int col_rows, bool has_qual)
{
    FastSmem L;
    size_t o = 0;
    L.bar_off = o; o += 16;
    L.cnt_off = o; o += 16;                       // two task counters (two-phase kernel)
    o = cg_align_up(o, 128);
    L.task_off = o; o += CG_NT * 32;              // compacted DP tasks (two-phase kernel): 2 x uint4
    L.blob_off = o; o += cg_align_up(blob_bytes, 16);
    L.enc_off = o; o += 768;
    o = cg_align_up(o, 128);
    L.seq_off = o; o += 2 * (size_t)tile_cap;
    L.qual_off = o; if (has_qual) o += 2 * (size_t)tile_cap;
    o = cg_align_up(o, 128);
    L.col_off = o; o += (size_t)col_rows * CG_NT * sizeof(uint32_t);
    L.total = cg_align_up(o, 128);
    return L;
}

size_t cg_fast_smem_bytes(uint32_t blob_bytes, int tile_cap, int col_rows, bool has_qual)
{
    return fast_smem_layout(blob_bytes, tile_cap, col_rows, has_qual).total;
}

// ------------------------------------------------------------------------------------------
// The fused kernel
// ------------------------------------------------------------------------------------------
// SIMPLE = false: every lane runs the complete per-read pass (any adapter set, rounds, linked).
// SIMPLE = true : two-phase schedule for one aligner adapter: phase A (scan: prefilter verdict +
//                 locator hits) on all reads of the tile, warp-ballot compaction of the reads that
//                 pass into a shared-memory task list, phase B (windowed DP) on dense lanes.
template <bool HAS_QUAL, bool SIMPLE>
__global__ void __launch_bounds__(CG_NT) cg_trim_fast_kernel(const CgKernelArgs a)
{
    extern __shared__ __align__(128) uint8_t smem[];
    const FastSmem L = fast_smem_layout(a.blob_bytes, a.tile_cap, a.col_rows, HAS_QUAL);
    uint64_t *bars = (uint64_t *)(smem + L.bar_off);
    uint8_t *s_blob = smem + L.blob_off;
    uint8_t *s_enc = smem + L.enc_off;
    uint8_t *s_seq = smem + L.seq_off;
    uint8_t *s_qual = smem + L.qual_off;
    uint32_t *s_col = (uint32_t *)(smem + L.col_off);
    uint32_t *s_cnt = (uint32_t *)(smem + L.cnt_off);
    uint4 *s_task = (uint4 *)(smem + L.task_off);
    const int tid = threadIdx.x;

    // adapter tables HBM -> smem (16-byte vectors), encoding tables
    for (uint32_t i = tid; i < a.blob_bytes / 16; i += CG_NT)
        ((uint4 *)s_blob)[i] = ((const uint4 *)a.blob)[i];
    for (uint32_t i = tid; i < 768 / 16; i += CG_NT)
        ((uint4 *)s_enc)[i] = ((const uint4 *)a.enc)[i];
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        fence_barrier_init();
        s_cnt[0] = 0; s_cnt[1] = 0;
    }
    __syncthreads();
    const SetView S = make_set_view(s_blob, a.masks64, s_enc, a.index);

    const long long n_reads = a.n_reads;
    const long long n_tiles = (n_reads + CG_NT - 1) / CG_NT;
    const uintptr_t seq_base = (uintptr_t)a.seq, qual_base = (uintptr_t)a.qual;

    // producer: one elected lane issues the bulk copies of a tile into stage `st`
    auto issue = [&](long long tile, int st) {
        const long long r0 = tile * CG_NT;
        const long long r1 = (r0 + CG_NT < n_reads) ? r0 + CG_NT : n_reads;
        const long long b0 = a.offsets[r0], b1 = a.offsets[r1];
        if (b1 <= b0) return;
        const uintptr_t sa0 = (seq_base + b0) & ~(uintptr_t)15;
        const uintptr_t sa1 = (seq_base + b1 + 15) & ~(uintptr_t)15;
        uint32_t bytes = (uint32_t)(sa1 - sa0);
        uint32_t qbytes = 0;
        uintptr_t qa0 = 0;
        if (HAS_QUAL) {
            qa0 = (qual_base + b0) & ~(uintptr_t)15;
            qbytes = (uint32_t)(((qual_base + b1 + 15) & ~(uintptr_t)15) - qa0);
        }
        mbar_expect_tx(&bars[st], bytes + qbytes);
        tma_load_1d(s_seq + (size_t)st * a.tile_cap, (const void *)sa0, bytes, &bars[st]);
        if (HAS_QUAL) tma_load_1d(s_qual + (size_t)st * a.tile_cap, (const void *)qa0, qbytes, &bars[st]);
    };

    if (tid == 0) {
        if ((long long)blockIdx.x < n_tiles) issue(blockIdx.x, 0);
        if ((long long)blockIdx.x + gridDim.x < n_tiles) issue((long long)blockIdx.x + gridDim.x, 1);
    }

    PackedCol colp; colp.base = s_col + tid; colp.stride = CG_NT;
    WideCol colw; colw.base = nullptr; colw.stride = 0;
    uint32_t phase0 = 0, phase1 = 0;
    int it = 0;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
        const int st = it & 1;
        const long long r0 = tile * CG_NT;
        const long long r1 = (r0 + CG_NT < n_reads) ? r0 + CG_NT : n_reads;
        const long long r = r0 + tid;
        const long long b0 = a.offsets[r0], b1 = a.offsets[r1];
        long long o0 = 0, o1 = 0;
        if (r < n_reads) { o0 = a.offsets[r]; o1 = a.offsets[r + 1]; }
        const uintptr_t sa0 = (seq_base + b0) & ~(uintptr_t)15;
        const uint8_t *tile_seq = s_seq + (size_t)st * a.tile_cap;
        const uint8_t *tile_qual = s_qual + (size_t)st * a.tile_cap;
        if (b1 > b0) {
            if (st == 0) { mbar_wait(&bars[0], phase0); phase0 ^= 1; }
            else { mbar_wait(&bars[1], phase1); phase1 ^= 1; }
            // ASCII check of the staged bases (the reference raises ValueError, _align.pyx:44-45)
            const uint32_t head = (uint32_t)((seq_base + b0) - sa0);
            const uint32_t body = (uint32_t)(b1 - b0);
            const uint32_t nchunks = (head + body + 15) / 16;
            uint32_t bad = 0;
            // the slack bytes of interior tiles belong to neighbouring reads of the same batch, so only
            // the very first and very last chunk of the batch need byte-exact masking
            const bool edge_first = tile == 0, edge_last = tile == n_tiles - 1;
            for (uint32_t c = tid; c < nchunks; c += CG_NT) {
                const uint4 v = ((const uint4 *)tile_seq)[c];
                if ((c == 0 && edge_first) || (c == nchunks - 1 && edge_last)) {
                    const uint8_t *pb = tile_seq + 16 * c;
                    for (uint32_t b = 0; b < 16; ++b) {
                        const uint32_t idx = 16 * c + b;
                        if (idx >= head && idx < head + body) bad |= pb[b];
                    }
                } else bad |= v.x | v.y | v.z | v.w;
            }
            if (bad & 0x80808080u) atomicOr(a.err_flag, 1);
        }
        if (!SIMPLE) {
            if (r < n_reads) {
                const int n = (int)(o1 - o0);
                const uint8_t *p = tile_seq + (size_t)((seq_base + o0) - sa0);
                const uint8_t *q = nullptr;
                if (HAS_QUAL) {
                    const uintptr_t qa0 = (qual_base + b0) & ~(uintptr_t)15;
                    q = tile_qual + (size_t)((qual_base + o0) - qa0);
                }
                process_read<false>(S, p, q, n, HAS_QUAL ? a.quality_trim : 0, a.cutoff_front, a.cutoff_back,
                                    a.qbase, a.times, colp, colw,
                                    a.out + (size_t)r * a.times * a.slots, a.qtrim ? a.qtrim + 2 * r : nullptr,
                                    a.view ? a.view + 2 * r : nullptr);
            }
        } else {
            // ---- phase A: quality trim + fused scan on every read of the tile ----------------
            // The scan reports locator hits per 16-character group plus the scan state at the start of
            // the first two hit groups.  Phase B (m <= 32, "regs"): resumes the scan there to get exact
            // end positions -> exact DP runs, DP column in registers.  Longer adapters: group-granular
            // windows and the shared-memory column.
            const bool regs = S.ad[0].m <= 32;
            bool pass = false;
            uint32_t hits = 0, t_off = 0, t_len = 0;
            int gs = 4;
            uint32_t rs0 = 0, rs1 = 0;
            if (r < n_reads) {
                const int n = (int)(o1 - o0);
                const uint32_t off = (uint32_t)((seq_base + o0) - sa0);
                int ts = 0, te = n;
                if (HAS_QUAL) {
                    const uintptr_t qa0 = (qual_base + b0) & ~(uintptr_t)15;
                    const uint8_t *q = tile_qual + (size_t)((qual_base + o0) - qa0);
                    if (a.quality_trim) pre_trim_core(tile_seq + off, q, n, a.quality_trim, a.cutoff_front, a.cutoff_back, a.qbase, &ts, &te);
                }
                if (a.qtrim) { a.qtrim[2 * r] = ts; a.qtrim[2 * r + 1] = te; }
                if (a.view) { ts = a.view[2 * r]; te = a.view[2 * r + 1]; }
                t_off = off + (uint32_t)ts; t_len = (uint32_t)(te - ts);
                const ScanOut sc = simple_scan(S, tile_seq + t_off, (int)t_len, &gs);
                pass = sc.pass; hits = sc.hits; rs0 = sc.rs0; rs1 = sc.rs1;
                if (!pass) {
                    CgHit none; none.adapter = -1; none.remove = 0;
                    none.astart = none.astop = none.rstart = none.rstop = none.score = none.errors = 0;
                    store_hit(a.out + (size_t)r * a.slots, none, 0, 0);
                }
            }
            // ---- compaction: reads that passed become dense DP tasks -------------------------
            uint32_t *cnt = &s_cnt[it & 1];
            const uint32_t ballot = __ballot_sync(0xffffffffu, pass);
            const uint32_t lane = tid & 31;
            uint32_t base = 0;
            if (lane == 0 && ballot) base = atomicAdd(cnt, __popc(ballot));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (pass) {
                const uint32_t slot = base + __popc(ballot & ((1u << lane) - 1u));
                s_task[2 * slot] = make_uint4(t_off, t_len, hits, (uint32_t)tid | ((uint32_t)gs << 16));
                s_task[2 * slot + 1] = make_uint4(rs0, rs1, 0u, 0u);
            }
            __syncthreads();
            const uint32_t n_tasks = *cnt;
            if (tid == 0) s_cnt[(it + 1) & 1] = 0;
            // ---- phase B: DP on the compacted tasks -------------------------------------------
            const bool has_task = (uint32_t)tid < n_tasks;
            const bool warp_has_task = (uint32_t)(tid & ~31) < n_tasks;
            if (regs) {
                if (warp_has_task) {     // warp collectives inside: whole warps only
                    uint4 t = make_uint4(0, 0, 0, 4u << 16), u = make_uint4(0, 0, 0, 0);
                    if (has_task) { t = s_task[2 * tid]; u = s_task[2 * tid + 1]; }
                    CgHit hit;
                    const bool found = simple_locate_regs(S, tile_seq + t.x, (int)t.y, t.z, (int)(t.w >> 16),
                                                          u.x, u.y, has_task, hit);
                    if (has_task) {
                        if (!found) {
                            hit.adapter = -1; hit.remove = 0;
                            hit.astart = hit.astop = hit.rstart = hit.rstop = hit.score = hit.errors = 0;
                        }
                        store_hit(a.out + (size_t)(r0 + (long long)(t.w & 0xFFFFu)) * a.slots, hit, 0, (int)t.y);
                    }
                }
            } else if (has_task) {
                const uint4 t = s_task[2 * tid];
                const long long rr = r0 + (long long)(t.w & 0xFFFFu);
                CgHit hit;
                if (!simple_locate(S, tile_seq + t.x, (int)t.y, t.z, (int)(t.w >> 16), colp, hit)) {
                    hit.adapter = -1; hit.remove = 0;
                    hit.astart = hit.astop = hit.rstart = hit.rstop = hit.score = hit.errors = 0;
                }
                store_hit(a.out + (size_t)rr * a.slots, hit, 0, (int)t.y);
            }
        }
        __syncthreads();   // every lane is done with stage `st`
        if (tid == 0) {
            const long long next = tile + 2LL * gridDim.x;
            if (next < n_tiles) issue(next, st);
        }
    }
}

typedef void (*fast_kernel_t)(const CgKernelArgs);
static fast_kernel_t pick_fast(bool has_qual, bool simple)
{
    if (simple) return has_qual ? cg_trim_fast_kernel<true, true> : cg_trim_fast_kernel<false, true>;
    return has_qual ? cg_trim_fast_kernel<true, false> : cg_trim_fast_kernel<false, false>;
}

cudaError_t cg_fast_occupancy(bool has_qual, bool simple, size_t smem, int *blocks_per_sm)
{
    fast_kernel_t k = pick_fast(has_qual, simple);
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, k, CG_NT, smem);
}

cudaError_t cg_launch_fast(const CgKernelArgs &a, bool has_qual, bool simple, int grid, size_t smem, cudaStream_t st)
{
    pick_fast(has_qual, simple)<<<grid, CG_NT, smem, st>>>(a);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// The warp-autonomous kernel (one aligner adapter with m <= 32, one round).
//
// Every warp is its own pipeline -- there is no block-level barrier after set-up:
//   * it stages its own mini-tiles of 32 reads (one per lane) with TMA 1-D bulk copies into a
//     private 2-stage ring (lane 0 issues, all lanes wait on the warp's mbarrier);
//   * phase A on the mini-tile: quality trim + fused scan; failing reads write "no match";
//   * passing reads become tasks.  The DP (phase B) only ever runs on FULL groups of 32 tasks:
//     tasks left over (< 32) are copied -- read bytes and scan results -- into a 31-slot carry
//     buffer and complete the next group, so every DP pass has all lanes busy and the lanes' bands
//     grow in step;
//   * a final flush pass handles what is left in the carry buffer.
// ------------------------------------------------------------------------------------------
struct WarpSmem {
    size_t blob_off, enc_off, warp_off, warp_stride;                   // per CTA
    size_t bar_rel, meta_new_rel, meta_carry_rel, seq_rel, qual_rel, carry_rel;   // inside a warp region
    size_t total;
};
__host__ __device__ inline WarpSmem warp_smem_layout(uint32_t blob_bytes, int mini_cap, int carry_slot, bool has_qual)
{
    WarpSmem L;
    size_t o = 0;
    L.blob_off = o; o += cg_align_up(blob_bytes, 16);
    L.enc_off = o; o += 768;
    o = cg_align_up(o, 128);
    L.warp_off = o;
    size_t w = 0;
    L.bar_rel = w; w += 16;
    L.meta_new_rel = w; w += 32 * 32;
    L.meta_carry_rel = w; w += 32 * 32;
    w = cg_align_up(w, 128);
    L.seq_rel = w; w += 2 * (size_t)mini_cap;
    L.qual_rel = w; if (has_qual) w += 2 * (size_t)mini_cap;
    L.carry_rel = w; w += 31 * (size_t)carry_slot;
    L.warp_stride = cg_align_up(w, 128);
    L.total = L.warp_off + 4 * L.warp_stride;
    return L;
}

size_t cg_warp_smem_bytes(uint32_t blob_bytes, int mini_cap, int carry_slot, bool has_qual)
{
    return warp_smem_layout(blob_bytes, mini_cap, carry_slot, has_qual).total;
}

// One DP pass of a warp: a single call site keeps the (large) register-DP code out of the loop body.
__device__ __noinline__ void warp_dp_pass(const SetView &S, const uint8_t *smem_base, const uint4 ma, const uint4 mb,
                                          bool has_task, cg_match_rec *out, int slots)
{
    CgHit hit;
    const bool found = simple_locate_regs(S, smem_base + ma.x, (int)ma.y, ma.z, (int)ma.w, mb.x, mb.y, has_task, hit);
    if (has_task) {
        if (!found) {
            hit.adapter = -1; hit.remove = 0;
            hit.astart = hit.astop = hit.rstart = hit.rstop = hit.score = hit.errors = 0;
        }
        const long long r = (long long)(((unsigned long long)mb.w << 32) | mb.z);
        store_hit(out + (size_t)r * slots, hit, 0, (int)ma.y);
    }
}

template <bool HAS_QUAL>
__global__ void __launch_bounds__(CG_NT) cg_trim_warp_kernel(const CgKernelArgs a)
{
    extern __shared__ __align__(128) uint8_t smem[];
    const WarpSmem L = warp_smem_layout(a.blob_bytes, a.mini_cap, a.carry_slot, HAS_QUAL);
    uint8_t *s_blob = smem + L.blob_off;
    uint8_t *s_enc = smem + L.enc_off;
    const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
    uint8_t *wbase = smem + L.warp_off + (size_t)wib * L.warp_stride;
    uint64_t *bars = (uint64_t *)(wbase + L.bar_rel);
    uint4 *meta_new = (uint4 *)(wbase + L.meta_new_rel);
    uint4 *meta_carry = (uint4 *)(wbase + L.meta_carry_rel);
    uint8_t *s_seq = wbase + L.seq_rel;
    uint8_t *s_qual = wbase + L.qual_rel;
    uint8_t *s_carry = wbase + L.carry_rel;

    for (uint32_t i = tid; i < a.blob_bytes / 16; i += CG_NT) ((uint4 *)s_blob)[i] = ((const uint4 *)a.blob)[i];
    for (uint32_t i = tid; i < 768 / 16; i += CG_NT) ((uint4 *)s_enc)[i] = ((const uint4 *)a.enc)[i];
    if (lane == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        fence_barrier_init();
    }
    __syncthreads();          // the only block-wide barrier
    const SetView S = make_set_view(s_blob, a.masks64, s_enc, a.index);

    const long long n_reads = a.n_reads;
    const long long n_mt = (n_reads + 31) / 32;
    const long long warps_total = (long long)gridDim.x * (CG_NT / 32);
    const long long wg = (long long)blockIdx.x * (CG_NT / 32) + wib;
    const uintptr_t seq_base = (uintptr_t)a.seq, qual_base = (uintptr_t)a.qual;

    auto issue = [&](long long mt, int st) {
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
        mbar_expect_tx(&bars[st], bytes + qbytes);
        tma_load_1d(s_seq + (size_t)st * a.mini_cap, (const void *)sa0, bytes, &bars[st]);
        if (HAS_QUAL) tma_load_1d(s_qual + (size_t)st * a.mini_cap, (const void *)qa0, qbytes, &bars[st]);
    };
    if (lane == 0) {
        if (wg < n_mt) issue(wg, 0);
        if (wg + warps_total < n_mt) issue(wg + warps_total, 1);
    }

    uint32_t phase0 = 0, phase1 = 0;
    int c_old = 0;                 // tasks waiting in the carry buffer (warp-uniform)
    int it = 0;
    long long mt = wg;
    while (true) {
        const bool have_tile = mt < n_mt;
        if (!have_tile && c_old == 0) break;
        const int st = it & 1;
        int c_new = 0;
        const uint8_t *tile_seq = s_seq + (size_t)st * a.mini_cap;
        if (have_tile) {
            const long long r0 = mt * 32;
            const long long r1 = (r0 + 32 < n_reads) ? r0 + 32 : n_reads;
            const long long r = r0 + lane;
            const long long b0 = a.offsets[r0], b1 = a.offsets[r1];
            long long o0 = 0, o1 = 0;
            if (r < n_reads) { o0 = a.offsets[r]; o1 = a.offsets[r + 1]; }
            const uintptr_t sa0 = (seq_base + b0) & ~(uintptr_t)15;
            const uint8_t *tile_qual = s_qual + (size_t)st * a.mini_cap;
            if (b1 > b0) {
                if (st == 0) { mbar_wait(&bars[0], phase0); phase0 ^= 1; }
                else { mbar_wait(&bars[1], phase1); phase1 ^= 1; }
                const uint32_t head = (uint32_t)((seq_base + b0) - sa0);
                const uint32_t body = (uint32_t)(b1 - b0);
                const uint32_t nchunks = (head + body + 15) / 16;
                uint32_t bad = 0;
                const bool edge_first = mt == 0, edge_last = mt == n_mt - 1;
                for (uint32_t c = lane; c < nchunks; c += 32) {
                    const uint4 v = ((const uint4 *)tile_seq)[c];
                    if ((c == 0 && edge_first) || (c == nchunks - 1 && edge_last)) {
                        const uint8_t *pb = tile_seq + 16 * c;
                        for (uint32_t b = 0; b < 16; ++b) {
                            const uint32_t idx = 16 * c + b;
                            if (idx >= head && idx < head + body) bad |= pb[b];
                        }
                    } else bad |= v.x | v.y | v.z | v.w;
                }
                if (bad & 0x80808080u) atomicOr(a.err_flag, 1);
            }
            // ---- phase A ------------------------------------------------------------------------
            bool pass = false;
            uint32_t hits = 0, rs0 = 0, rs1 = 0, t_off = 0, t_len = 0;
            int gs = 4;
            if (r < n_reads) {
                const int n = (int)(o1 - o0);
                const uint32_t off = (uint32_t)((seq_base + o0) - sa0);
                int ts = 0, te = n;
                if (HAS_QUAL) {
                    const uintptr_t qa0 = (qual_base + b0) & ~(uintptr_t)15;
                    const uint8_t *q = tile_qual + (size_t)((qual_base + o0) - qa0);
                    if (a.quality_trim) pre_trim_core(tile_seq + off, q, n, a.quality_trim, a.cutoff_front, a.cutoff_back, a.qbase, &ts, &te);
                }
                if (a.qtrim) { a.qtrim[2 * r] = ts; a.qtrim[2 * r + 1] = te; }
                if (a.view) { ts = a.view[2 * r]; te = a.view[2 * r + 1]; }
                t_off = off + (uint32_t)ts; t_len = (uint32_t)(te - ts);
                const ScanOut sc = simple_scan(S, tile_seq + t_off, (int)t_len, &gs);
                pass = sc.pass; hits = sc.hits; rs0 = sc.rs0; rs1 = sc.rs1;
                if (!pass) {
                    CgHit none; none.adapter = -1; none.remove = 0;
                    none.astart = none.astop = none.rstart = none.rstop = none.score = none.errors = 0;
                    store_hit(a.out + (size_t)r * a.slots, none, 0, 0);
                }
            }
            const uint32_t ballot = __ballot_sync(0xffffffffu, pass);
            c_new = __popc(ballot);
            if (pass) {
                const uint32_t idx = __popc(ballot & ((1u << lane) - 1u));
                meta_new[2 * idx] = make_uint4((uint32_t)(tile_seq - smem) + t_off, t_len, hits, (uint32_t)gs);
                meta_new[2 * idx + 1] = make_uint4(rs0, rs1, (uint32_t)((unsigned long long)r & 0xffffffffu),
                                                   (uint32_t)((unsigned long long)r >> 32));
            }
            __syncwarp();
        }
        // ---- phase B: only full groups of 32 tasks (or the final flush) --------------------------
        const int total = c_old + c_new;
        const bool flush = !have_tile;
        int first_left = 0, n_left = c_new;      // which new tasks go to the carry buffer afterwards
        int carry_at = c_old;                    // ... and from which carry slot on
        if (total >= 32 || flush) {
            const bool has_task = lane < total;  // total < 32 only when flushing
            uint4 ma = make_uint4(0, 0, 0, 4), mb = make_uint4(0, 0, 0, 0);
            if (has_task) {
                if (lane < c_old) { ma = meta_carry[2 * lane]; mb = meta_carry[2 * lane + 1]; }
                else { ma = meta_new[2 * (lane - c_old)]; mb = meta_new[2 * (lane - c_old) + 1]; }
            }
            warp_dp_pass(S, smem, ma, mb, has_task, a.out, a.slots);
            __syncwarp();
            first_left = 32 - c_old;             // new tasks [first_left, c_new) were not processed
            n_left = total >= 32 ? total - 32 : 0;
            carry_at = 0;
            c_old = 0;
        }
        // ---- carry the unprocessed new tasks (read bytes + scan results) -------------------------
        for (int j = 0; j < n_left; ++j) {
            const uint4 ma = meta_new[2 * (first_left + j)];
            const uint4 mb = meta_new[2 * (first_left + j) + 1];
            const uint32_t src = ma.x & ~15u;
            const uint32_t nch = ((ma.x & 15u) + ma.y + 15u) >> 4;
            uint8_t *dst = s_carry + (size_t)(carry_at + j) * a.carry_slot;
            if ((uint32_t)lane < nch) ((uint4 *)dst)[lane] = ((const uint4 *)(smem + src))[lane];
            if (lane == 0) {
                meta_carry[2 * (carry_at + j)] = make_uint4((uint32_t)(dst - smem) + (ma.x & 15u), ma.y, ma.z, ma.w);
                meta_carry[2 * (carry_at + j) + 1] = mb;
            }
        }
        c_old = carry_at + n_left;
        __syncwarp();
        if (have_tile) {
            if (lane == 0) {
                const long long next = mt + 2 * warps_total;
                if (next < n_mt) issue(next, st);
            }
            mt += warps_total;
            ++it;
        }
    }
}

cudaError_t cg_warp_occupancy(bool has_qual, size_t smem, int *blocks_per_sm)
{
    void (*k)(const CgKernelArgs) = has_qual ? cg_trim_warp_kernel<true> : cg_trim_warp_kernel<false>;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, k, CG_NT, smem);
}

cudaError_t cg_launch_warp(const CgKernelArgs &a, bool has_qual, int grid, size_t smem, cudaStream_t st)
{
    if (has_qual) cg_trim_warp_kernel<true><<<grid, CG_NT, smem, st>>>(a);
    else cg_trim_warp_kernel<false><<<grid, CG_NT, smem, st>>>(a);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Split pipeline for one aligner adapter (m <= 64), one round:
//
//   cg_scan_kernel   phase A on every read at high occupancy (few registers): per-warp TMA-staged
//                    mini-tiles of 32 reads, quality trim + fused scan; failing reads get their
//                    "no match" record, passing reads append a 32-byte task (read index, trimmed
//                    window, locator hit groups, saved scan states) to a list in HBM with one
//                    warp-aggregated atomic per mini-tile.
//   cg_dp_kernel     phase B on dense groups of 32 tasks: every lane fetches its task's read window
//                    into shared memory with its own TMA bulk copy (32 copies, one mbarrier),
//                    double buffered against the DP of the previous group; then exact runs +
//                    register-column DP with all 32 lanes busy.
//
// The two phases have opposite resource profiles (the scan needs ~40 registers and wants many warps
// to hide its dependent shift-and chain; the DP wants ~128 registers); fused in one kernel the DP's
// registers cap the scan's occupancy.  The task list costs ~35 bytes of extra HBM traffic per read,
// which is noise for a kernel that is instruction-issue bound.
// ------------------------------------------------------------------------------------------
#ifndef CG_SCAN_STAGES
#define CG_SCAN_STAGES 1     // per-warp staging depth of the scan kernel (1: more resident warps hide the TMA latency)
#endif
__host__ __device__ inline ScanSmem scan_smem_layout(uint32_t blob_bytes, int mini_cap, bool has_qual)
{
    ScanSmem L;
    size_t o = 0;
    L.blob_off = o; o += cg_align_up(blob_bytes, 16);
    L.enc_off = o; o += 768;
    o = cg_align_up(o, 128);
    L.warp_off = o;
    size_t w = 0;
    L.bar_rel = w; w += 16;
    w = cg_align_up(w, 128);
    L.seq_rel = w; w += CG_SCAN_STAGES * (size_t)mini_cap;
    L.qual_rel = w; if (has_qual) w += CG_SCAN_STAGES * (size_t)mini_cap;
    L.warp_stride = cg_align_up(w, 128);
    L.total = L.warp_off + (CG_NT / 32) * L.warp_stride;
    return L;
}
size_t cg_scan_smem_bytes(uint32_t blob_bytes, int mini_cap, bool has_qual)
{
    return scan_smem_layout(blob_bytes, mini_cap, has_qual).total;
}

template <bool HAS_QUAL>
__global__ void __launch_bounds__(CG_NT) cg_scan_kernel(const CgKernelArgs a)
{
    extern __shared__ __align__(128) uint8_t smem[];
    const ScanSmem L = scan_smem_layout(a.blob_bytes, a.mini_cap, HAS_QUAL);
    uint8_t *s_blob = smem + L.blob_off;
    uint8_t *s_enc = smem + L.enc_off;
    const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
    uint8_t *wbase = smem + L.warp_off + (size_t)wib * L.warp_stride;
    uint64_t *bars = (uint64_t *)(wbase + L.bar_rel);
    uint8_t *s_seq = wbase + L.seq_rel;
    uint8_t *s_qual = wbase + L.qual_rel;

    for (uint32_t i = tid; i < a.blob_bytes / 16; i += CG_NT) ((uint4 *)s_blob)[i] = ((const uint4 *)a.blob)[i];
    for (uint32_t i = tid; i < 768 / 16; i += CG_NT) ((uint4 *)s_enc)[i] = ((const uint4 *)a.enc)[i];
    if (lane == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        fence_barrier_init();
    }
    __syncthreads();
    const SetView S = make_set_view(s_blob, a.masks64, s_enc, a.index);

    // non-ASCII input (the reference raises ValueError): when the scan program's first word walks the
    // whole searched sequence the check rides along in the scan (the characters are in registers anyway);
    // otherwise a cooperative pass over the staged tile does it
    const bool fold_ascii = scan_checks_ascii(S.scan, S.h->scan_count);
    const long long n_reads = a.n_reads;
    const long long n_mt = (n_reads + 31) / 32;
    const long long warps_total = (long long)gridDim.x * (CG_NT / 32);
    const long long wg = (long long)blockIdx.x * (CG_NT / 32) + wib;
    const uintptr_t seq_base = (uintptr_t)a.seq, qual_base = (uintptr_t)a.qual;

    auto issue = [&](long long mt, int st) {
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
        mbar_expect_tx(&bars[st], bytes + qbytes);
        tma_load_1d(s_seq + (size_t)st * a.mini_cap, (const void *)sa0, bytes, &bars[st]);
        if (HAS_QUAL) tma_load_1d(s_qual + (size_t)st * a.mini_cap, (const void *)qa0, qbytes, &bars[st]);
    };
    if (lane == 0) {
        if (wg < n_mt) issue(wg, 0);
        if (CG_SCAN_STAGES > 1 && wg + warps_total < n_mt) issue(wg + warps_total, 1);
    }
    uint32_t phase0 = 0, phase1 = 0;
    int it = 0;
    for (long long mt = wg; mt < n_mt; mt += warps_total, ++it) {
        const int st = CG_SCAN_STAGES > 1 ? (it & 1) : 0;
        const long long r0 = mt * 32;
        const long long r1 = (r0 + 32 < n_reads) ? r0 + 32 : n_reads;
        const long long r = r0 + lane;
        const long long b0 = a.offsets[r0], b1 = a.offsets[r1];
        long long o0 = 0, o1 = 0;
        if (r < n_reads) { o0 = a.offsets[r]; o1 = a.offsets[r + 1]; }
        const uintptr_t sa0 = (seq_base + b0) & ~(uintptr_t)15;
        const uint8_t *tile_seq = s_seq + (size_t)st * a.mini_cap;
        const uint8_t *tile_qual = s_qual + (size_t)st * a.mini_cap;
        if (b1 > b0) {
            if (st == 0) { mbar_wait(&bars[0], phase0); phase0 ^= 1; }
            else { mbar_wait(&bars[1], phase1); phase1 ^= 1; }
        }
        if (b1 > b0 && !fold_ascii) {
            const uint32_t head = (uint32_t)((seq_base + b0) - sa0);
            const uint32_t body = (uint32_t)(b1 - b0);
            const uint32_t nchunks = (head + body + 15) / 16;
            uint32_t bad = 0;
            const bool edge_first = mt == 0, edge_last = mt == n_mt - 1;
            for (uint32_t c = lane; c < nchunks; c += 32) {
                const uint4 v = ((const uint4 *)tile_seq)[c];
                if ((c == 0 && edge_first) || (c == nchunks - 1 && edge_last)) {
                    const uint8_t *pb = tile_seq + 16 * c;
                    for (uint32_t b = 0; b < 16; ++b) {
                        const uint32_t idx = 16 * c + b;
                        if (idx >= head && idx < head + body) bad |= pb[b];
                    }
                } else bad |= v.x | v.y | v.z | v.w;
            }
            if (bad & 0x80808080u) atomicOr(a.err_flag, 1);
        }
        bool pass = false;
        uint32_t hits = 0, rs0 = 0, rs1 = 0;
        int gs = 4, ts = 0, te = 0;
        if (r < n_reads) {
            const int n = (int)(o1 - o0);
            const uint32_t off = (uint32_t)((seq_base + o0) - sa0);
            ts = 0; te = n;
            if (HAS_QUAL) {
                const uintptr_t qa0 = (qual_base + b0) & ~(uintptr_t)15;
                const uint8_t *q = tile_qual + (size_t)((qual_base + o0) - qa0);
                if (a.quality_trim) pre_trim_core(tile_seq + off, q, n, a.quality_trim, a.cutoff_front, a.cutoff_back, a.qbase, &ts, &te);
            }
            if (a.qtrim) { a.qtrim[2 * r] = ts; a.qtrim[2 * r + 1] = te; }
            if (a.view) { ts = a.view[2 * r]; te = a.view[2 * r + 1]; }
            const ScanOut sc = simple_scan(S, tile_seq + off + ts, te - ts, &gs);
            pass = sc.pass; hits = sc.hits; rs0 = sc.rs0; rs1 = sc.rs1;
            if (fold_ascii && (sc.bad & 0x80808080u)) atomicOr(a.err_flag, 1);
            if (!pass) {
                CgHit none; none.adapter = -1; none.remove = 0;
                none.astart = none.astop = none.rstart = none.rstop = none.score = none.errors = 0;
                store_hit(a.out + (size_t)r * a.slots, none, 0, 0);
            }
        }
        // warp-aggregated append to the task list
        const uint32_t ballot = __ballot_sync(0xffffffffu, pass);
        if (ballot) {
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(a.task_count, (unsigned long long)__popc(ballot));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (pass) {
                const unsigned long long slot = base + __popc(ballot & ((1u << lane) - 1u));
                // {read (relative to the sub-batch), byte offset of the window in the batch (hi, lo), window length}:
                // the list kernels fetch the window without a dependent load of offsets[read]
                const unsigned long long woff = (unsigned long long)(o0 + ts);
                a.tasks[2 * slot] = make_uint4((uint32_t)r, (uint32_t)(woff >> 32), (uint32_t)woff, (uint32_t)(te - ts));
                a.tasks[2 * slot + 1] = make_uint4(hits, (uint32_t)gs, rs0, rs1);
            }
        }
        __syncwarp();
        if (lane == 0) {
            const long long next = mt + (long long)CG_SCAN_STAGES * warps_total;
            if (next < n_mt) issue(next, st);
        }
    }
}

cudaError_t cg_scan_occupancy(bool has_qual, size_t smem, int *blocks_per_sm)
{
    void (*k)(const CgKernelArgs) = has_qual ? cg_scan_kernel<true> : cg_scan_kernel<false>;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, k, CG_NT, smem);
}
cudaError_t cg_launch_scan(const CgKernelArgs &a, bool has_qual, int grid, size_t smem, cudaStream_t st)
{
    if (has_qual) cg_scan_kernel<true><<<grid, CG_NT, smem, st>>>(a);
    else cg_scan_kernel<false><<<grid, CG_NT, smem, st>>>(a);
    return cudaGetLastError();
}

#include "cg_pscan.cuh"

size_t cg_pscan_smem_bytes(uint32_t blob_bytes, int mini_cap, bool has_qual, int stats_max_len)
{
    return pscan_smem_layout(blob_bytes, mini_cap, has_qual, stats_max_len).total;
}

template <bool HAS_QUAL, int W, bool STATS>
__global__ void __launch_bounds__(CG_NT, W <= 5 ? CG_PSCAN_BLOCKS : 5) cg_pscan_kernel(const CgKernelArgs a)
{
    cg_pscan_body<HAS_QUAL, W, RuntimePlaneProg, STATS>(a);
}

typedef void (*pscan_kernel_t)(const CgKernelArgs);
static pscan_kernel_t pick_pscan(bool has_qual, int w, bool stats)
{
    // (the statistics are counted in this stage only for passes without quality trimming: launch_trim_single)
    if (stats) return w <= 5 ? cg_pscan_kernel<false, 5, true> : cg_pscan_kernel<false, 8, true>;
    if (w <= 5) return has_qual ? cg_pscan_kernel<true, 5, false> : cg_pscan_kernel<false, 5, false>;
    return has_qual ? cg_pscan_kernel<true, 8, false> : cg_pscan_kernel<false, 8, false>;
}
cudaError_t cg_pscan_occupancy(bool has_qual, int w, bool stats, size_t smem, int *blocks_per_sm)
{
    pscan_kernel_t k = pick_pscan(has_qual, w, stats);
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, k, CG_NT, smem);
}
cudaError_t cg_launch_pscan(const CgKernelArgs &a, bool has_qual, int w, int grid, size_t smem, cudaStream_t st)
{
    pick_pscan(has_qual, w, a.stats != nullptr)<<<grid, CG_NT, smem, st>>>(a);
    return cudaGetLastError();
}

// Staging depth of the list kernels: 1 = fetch, wait, work (half the shared memory, twice the resident
// warps to hide the copy latency); 2 = prefetch the next group's bytes while working on this one.
#ifndef CG_LIST_STAGES
#define CG_LIST_STAGES 1
#endif
struct DpSmem { size_t blob_off, enc_off, warp_off, warp_stride, bar_rel, slot_rel, total; };
__host__ __device__ inline DpSmem dp_smem_layout(uint32_t blob_bytes, int slot_bytes)
{
    DpSmem L;
    size_t o = 0;
    L.blob_off = o; o += cg_align_up(blob_bytes, 16);
    L.enc_off = o; o += 768;
    o = cg_align_up(o, 128);
    L.warp_off = o;
    size_t w = 0;
    L.bar_rel = w; w += 16;
    w = cg_align_up(w, 128);
    L.slot_rel = w; w += CG_LIST_STAGES * 32 * (size_t)slot_bytes;
    L.warp_stride = cg_align_up(w, 128);
    L.total = L.warp_off + (CG_NT / 32) * L.warp_stride;
    return L;
}
size_t cg_dp_smem_bytes(uint32_t blob_bytes, int slot_bytes) { return dp_smem_layout(blob_bytes, slot_bytes).total; }

// Common frame of the list-driven kernels: a warp walks groups of 32 list records; every lane
// fetches the bytes its record needs into its own shared-memory slot with its own TMA bulk copy
// (SASS: one UBLKCP per lane, one mbarrier per stage), double buffered against the work on the
// previous group.
//
//  PLAN = true  (cg_plan_kernel): input = the scan kernel's list (2 x uint4).  Exact end positions of
//               the locator hits -> runs; reads finished by the exact-occurrence shortcut get their
//               record, the others append a run record (4 x uint4) for the DP rounds:
//               {r_lo, r_hi, trim_start, len}, {have, origin, cost, score},
//               {ref_stop, q_stop, run_idx, n_runs | end_idx << 8}, {lo|hi<<16 of up to 4 runs}
//  PLAN = false (cg_run_kernel<MR>): one DP run of every record of the input list; reads that are
//               finished (early exit or last run) get their record, the others move to the output
//               list with the updated selection state.
#ifndef CG_PLAN_BLOCKS
#define CG_PLAN_BLOCKS 6      // resident CTAs per SM the plan kernel is compiled for (80 registers; measured: 7 CTAs at
                              // 72 registers spill in the bit-vector loops and run 25 % slower)
#endif
#ifndef CG_RUN16_BLOCKS
#define CG_RUN16_BLOCKS 4     // same for the run kernel with a 16-row column (measured: 4 beats 5)
#endif
#ifndef CG_RUN48_BLOCKS
#define CG_RUN48_BLOCKS 3      // resident CTAs per SM of the 48-row run kernel (168 registers, some spills; 2 = 255 registers)
#endif
template <bool PLAN, int MR>
__global__ void __launch_bounds__(CG_NT, PLAN ? CG_PLAN_BLOCKS : (MR <= 16 ? CG_RUN16_BLOCKS : (MR <= 32 ? 3 : (MR <= 48 ? CG_RUN48_BLOCKS : 2)))) cg_list_kernel(const CgKernelArgs a)
{
    extern __shared__ __align__(128) uint8_t smem[];
    const int slot_bytes = a.carry_slot;
    const DpSmem L = dp_smem_layout(a.blob_bytes, slot_bytes);
    uint8_t *s_blob = smem + L.blob_off;
    uint8_t *s_enc = smem + L.enc_off;
    const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
    uint8_t *wbase = smem + L.warp_off + (size_t)wib * L.warp_stride;
    uint8_t *s_slot = wbase + L.slot_rel;

    for (uint32_t i = tid; i < a.blob_bytes / 16; i += CG_NT) ((uint4 *)s_blob)[i] = ((const uint4 *)a.blob)[i];
    for (uint32_t i = tid; i < 768 / 16; i += CG_NT) ((uint4 *)s_enc)[i] = ((const uint4 *)a.enc)[i];
    __syncthreads();
    const SetView S = make_set_view(s_blob, a.masks64, s_enc, a.index);
    const CgAdapter &A = S.ad[0];

    unsigned long long n_tasks = *a.task_count;
    if (n_tasks > (unsigned long long)a.task_cap) n_tasks = (unsigned long long)a.task_cap;
    // second input list, filed from the end of the buffer backwards: its groups follow those of the first list, so that
    // no warp mixes the two kinds (plan stage: tasks without locator hits, an experiment; first DP round: runs
    // without a band, see below)
    unsigned long long n_tasks_b = a.task_count_b ? *a.task_count_b : 0ull;
    if (n_tasks + n_tasks_b > (unsigned long long)a.task_cap) n_tasks_b = (unsigned long long)a.task_cap - n_tasks;
    const long long n_groups_a = (long long)((n_tasks + 31) / 32);
    const uint4 *list = a.tasks;
    const int rec = PLAN ? a.task_rec : 4;     // the plan stage reads the scan kernel's (2 words) or cg_pscan_kernel's
                                               // (4 + the window bytes) tasks
    const long long n_groups = n_groups_a + (long long)((n_tasks_b + 31) / 32);
    const long long warps_total = (long long)gridDim.x * (CG_NT / 32);
    const long long wg = (long long)blockIdx.x * (CG_NT / 32) + wib;
    const uintptr_t seq_base = (uintptr_t)a.seq;

    // A task is fetched in two steps so that the dependent global loads of the NEXT group (list record ->
    // offsets[read] -> address) are in flight while the current group is worked on: load_task() only issues loads
    // into registers, stage() starts the per-lane cp.async copy of the read window into this lane's slot.
    struct Task { uint4 ta, tb, tc, td; uintptr_t src; uint32_t bytes, soff; };
    // physical record of lane `lane` of group g, or -1
    auto task_index = [&](long long g) -> long long {
        if (g < n_groups_a) {
            const unsigned long long t = (unsigned long long)g * 32 + lane;
            return t < n_tasks ? (long long)t : -1;
        }
        const unsigned long long t = (unsigned long long)(g - n_groups_a) * 32 + lane;
        return t < n_tasks_b ? (long long)a.task_cap - 1 - (long long)t : -1;
    };
    auto load_task = [&](long long g, Task &T) {
        const long long t = task_index(g);
        T.ta = make_uint4(0, 0, 0, 0); T.tb = make_uint4(0, 4, 0, 0); T.tc = make_uint4(0, 0, 0, 0); T.td = make_uint4(0, 0, 0, 0);
        T.src = 0; T.bytes = 0; T.soff = 0;
        if (t < 0) return;
        T.ta = list[rec * t]; T.tb = list[rec * t + 1];
        if (!PLAN || rec >= 4) { T.tc = list[rec * t + 2]; T.td = list[rec * t + 3]; }
        if (PLAN && (T.tb.y & CG_TASK_BYTES)) {          // the window travels with the task (cg_pscan_kernel)
            T.src = (uintptr_t)(list + rec * t + 4);
            T.bytes = 16u * (uint32_t)(rec - 4);
            T.soff = T.td.y;
            return;
        }
        uintptr_t addr = seq_base + (uintptr_t)(((unsigned long long)T.ta.y << 32) | T.ta.z);
        uint32_t len = T.ta.w;
        if (!PLAN) {
            const int n = (int)T.ta.w, ri = (int)T.tc.z;
            const uint32_t pk = ri == 0 ? T.td.x : (ri == 1 ? T.td.y : (ri == 2 ? T.td.z : T.td.w));
            const int lo = (int)(pk & 0xffffu), hi = (int)(pk >> 16);
            // (flag sets without both query ends free can have an empty column range: lo > hi)
            len = hi > lo ? (uint32_t)(hi - lo) : 0u;
            if (len) addr += (uintptr_t)(A.reverse ? n - hi : lo);
        }
        T.src = addr & ~(uintptr_t)15;
        T.bytes = len ? (uint32_t)(((addr + len + 15) & ~(uintptr_t)15) - T.src) : 0u;
        T.soff = (uint32_t)(addr - T.src);
    };
    auto stage = [&](const Task &T) {
        uint8_t *dst = s_slot + (size_t)lane * slot_bytes;
        for (uint32_t o = 0; o < T.bytes; o += 16) cp_async16(dst + o, (const void *)(T.src + o));
        cp_async_commit();
    };

    Task next;
    if (wg < n_groups) load_task(wg, next);
    for (long long g = wg; g < n_groups; g += warps_total) {
        const Task cur = next;
        stage(cur);
        if (g + warps_total < n_groups) load_task(g + warps_total, next);
        cp_async_wait<0>();
        const uint4 ta = cur.ta, tb = cur.tb, tc = cur.tc, td = cur.td;
        const uint32_t soff = cur.soff;
        const int st = 0;
        const bool has_task = task_index(g) >= 0;
        const uint8_t *p = s_slot + ((size_t)st * 32 + lane) * slot_bytes + soff;
        const int n = (int)ta.w;
        const long long r = (long long)ta.x;
        CgHit hit;
        hit.adapter = -1; hit.remove = 0;
        hit.astart = hit.astop = hit.rstart = hit.rstop = hit.score = hit.errors = 0;
        bool cont = false, cont_b = false, defer = false;
        uint4 ob = make_uint4(0, 0, 0, 0), oc = make_uint4(0, 0, 0, 0), od = make_uint4(0, 0, 0, 0);
        if (PLAN) {
            if (has_task) {
                RunPlan P;
                P.n_runs = 0; P.exact = 0; P.s0 = 0; P.end_idx = -1; P.banded = 0;
                uint32_t hits = tb.x, rs0 = tb.z, rs1 = tb.w;
                int gs = (int)(tb.y & 0xffu);
                bool pass = true;
                bool planned = false;
                if (tb.y & CG_TASK_PLANES) {
                    if (window_is_plain(p, n)) {
                        const uint32_t M[8] = {tb.x, tb.z, tb.w, tc.x, tc.y, tc.z, tc.w, td.x};
                        const int W = (int)((tb.y >> 12) & 15u);
                        plan_runs_planes(S, p, n, M, W, (int)((tb.y >> 20) & 1u), (int)((tb.y >> 21) & 1u), 32 * W - n, P);
                        planned = true;
                    } else {
                        // other letters than A/C/G/T: the exact scan is still to do.  Such reads are rare (an N in
                        // 1 of 7 reads), but one per warp would make every warp walk the scan: they are collected
                        // and planned by a second launch on dense warps.
                        defer = true;
                        pass = false;
                    }
                } else if (tb.y & CG_TASK_RESCAN) {
                    const ScanOut sc = simple_scan(S, p, n, &gs);
                    pass = sc.pass; hits = sc.hits; rs0 = sc.rs0; rs1 = sc.rs1;
                }
                if (planned) {}
                else if (pass) plan_runs(S, p, n, hits, gs, rs0, rs1, P);
                if (P.exact == 2) hit_end_overlap(A, n, P.s0, hit);
                else if (P.exact) hit_exact(A, n, P.s0, hit);
                else if (P.n_runs > 0) {
                    cont = true;
                    // bit 16: the runs come from the bit-plane stage's hit mask (run_band_d applies)
                    oc = make_uint4((uint32_t)A.m, (uint32_t)n, 0u, (uint32_t)P.n_runs | ((uint32_t)(P.end_idx & 15) << 8) |
                                                                   ((P.banded && !a.no_band) ? 1u << 16 : 0u));
                    // the first DP round works on two lists: runs with a band first, the others (end windows,
                    // runs that reach the end of the read) after them -- the band is warp-uniform
                    cont_b = a.task2_count_b != nullptr &&
                             run_band_d(A, n, P.lo0, P.hi0, P.banded != 0 && !a.no_band, P.end_idx == 0) < 0;
                    od = make_uint4((uint32_t)P.lo0 | ((uint32_t)P.hi0 << 16), (uint32_t)P.lo1 | ((uint32_t)P.hi1 << 16),
                                    (uint32_t)P.lo2 | ((uint32_t)P.hi2 << 16), (uint32_t)P.lo3 | ((uint32_t)P.hi3 << 16));
                }
            }
        } else {
            const int ri = (int)tc.z, n_runs = (int)(tc.w & 255u);
            int end_idx = (int)((tc.w >> 8) & 15u);
            if (end_idx == 15) end_idx = -1;
            const uint32_t pk = ri == 0 ? td.x : (ri == 1 ? td.y : (ri == 2 ? td.z : td.w));
            const int lo = (int)(pk & 0xffffu), hi = (int)(pk >> 16);
            LocState ls;
            ls.have = (int)tb.x; ls.b_origin = (int)tb.y; ls.b_cost = (int)tb.z; ls.b_score = (int)tb.w;
            ls.b_ref_stop = (int)tc.x; ls.b_q_stop = (int)tc.y; ls.stopped = 0;
            const bool last = ri == n_runs - 1;
            const int band = has_task ? run_band_d(A, n, lo, hi, (tc.w >> 16) & 1u, ri == end_idx) : -1;
            run_pass<MR>(S, p, n, lo, hi, ri != end_idx, last, has_task, ls, band);
            if (has_task) {
                if (ls.stopped || last) hit_from_state(A, n, ls, hit);
                else {
                    cont = true;
                    ob = make_uint4((uint32_t)ls.have, (uint32_t)ls.b_origin, (uint32_t)ls.b_cost, (uint32_t)ls.b_score);
                    oc = make_uint4((uint32_t)ls.b_ref_stop, (uint32_t)ls.b_q_stop, (uint32_t)(ri + 1), tc.w);
                    od = td;
                }
            }
        }
        if (has_task && !cont && !defer) store_hit(a.out + (size_t)r * a.slots, hit, 0, n);
        if (PLAN) {
            const uint32_t dballot = __ballot_sync(0xffffffffu, defer);
            if (dballot) {
                unsigned long long base = 0;
                if (lane == 0) base = atomicAdd(a.task3_count, (unsigned long long)__popc(dballot));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (defer) {
                    const unsigned long long slot = base + __popc(dballot & ((1u << lane) - 1u));
                    a.tasks3[2 * slot] = ta;
                    a.tasks3[2 * slot + 1] = make_uint4(0u, 4u | CG_TASK_RESCAN, 0u, 0u);
                }
            }
        }
        const uint32_t ballot = __ballot_sync(0xffffffffu, cont && !cont_b);
        const uint32_t ballot_b = __ballot_sync(0xffffffffu, cont && cont_b);
        if (ballot | ballot_b) {
            unsigned long long base = 0, base_b = 0;
            if (lane == 0) {
                if (ballot) base = atomicAdd(a.task2_count, (unsigned long long)__popc(ballot));
                if (ballot_b) base_b = atomicAdd(a.task2_count_b, (unsigned long long)__popc(ballot_b));
            }
            base = __shfl_sync(0xffffffffu, base, 0);
            base_b = __shfl_sync(0xffffffffu, base_b, 0);
            if (cont) {
                const uint32_t below = (1u << lane) - 1u;
                const unsigned long long slot = cont_b ? (unsigned long long)a.task_cap - 1ull - (base_b + __popc(ballot_b & below))
                                                       : base + __popc(ballot & below);
                a.tasks2[4 * slot] = ta;
                a.tasks2[4 * slot + 1] = ob;
                a.tasks2[4 * slot + 2] = oc;
                a.tasks2[4 * slot + 3] = od;
            }
        }
        __syncwarp();
    }
}

typedef void (*list_kernel_t)(const CgKernelArgs);
static list_kernel_t pick_list(bool plan, int mr)
{
    if (plan) return cg_list_kernel<true, 16>;
    if (mr <= 16) return cg_list_kernel<false, 16>;
    if (mr <= 32) return cg_list_kernel<false, 32>;
    if (mr <= 40) return cg_list_kernel<false, 40>;      // (the 33/34-base Illumina adapters: 8 rows fewer in registers)
    return mr <= 48 ? cg_list_kernel<false, 48> : cg_list_kernel<false, 64>;
}
cudaError_t cg_list_occupancy(bool plan, int mr, size_t smem, int *blocks_per_sm)
{
    list_kernel_t k = pick_list(plan, mr);
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, k, CG_NT, smem);
}
cudaError_t cg_launch_list(const CgKernelArgs &a, bool plan, int mr, int grid, size_t smem, cudaStream_t st)
{
    pick_list(plan, mr)<<<grid, CG_NT, smem, st>>>(a);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Multi-pass schedule: view of a linked adapter's back pass, and the final selection
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ cg_match_rec load_rec(const cg_match_rec *p)
{
    const int4 a = __ldg((const int4 *)p), b = __ldg((const int4 *)p + 1);
    cg_match_rec r;
    r.adapter = a.x; r.astart = a.y; r.astop = a.z; r.rstart = a.w;
    r.rstop = b.x; r.score = b.y; r.errors = b.z; r.info = b.w;
    return r;
}
__device__ __forceinline__ void store_rec(cg_match_rec *p, const cg_match_rec &r)
{
    ((int4 *)p)[0] = make_int4(r.adapter, r.astart, r.astop, r.rstart);
    ((int4 *)p)[1] = make_int4(r.rstop, r.score, r.errors, r.info);
}

__global__ void cg_linked_view_kernel(const cg_match_rec *front, const int32_t *base_view, const int64_t *offsets,
                                      long long n_reads, int32_t *out_view)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    int s = 0, e;
    if (base_view) { s = base_view[2 * r]; e = base_view[2 * r + 1]; }
    else e = (int)(offsets[r + 1] - offsets[r]);
    linked_view(load_rec(front + r), s, e);
    *(int2 *)(out_view + 2 * r) = make_int2(s, e);
}
cudaError_t cg_launch_linked_view(const cg_match_rec *front, const int32_t *base_view, const int64_t *offsets,
                                  long long n_reads, int32_t *out_view, cudaStream_t st)
{
    const int block = 256;
    cg_linked_view_kernel<<<(unsigned)((n_reads + block - 1) / block), block, 0, st>>>(front, base_view, offsets,
                                                                                     n_reads, out_view);
    return cudaGetLastError();
}

__global__ void cg_select_kernel(const CgSelectArgs a)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.n_reads) return;
    cg_match_rec b0, b1;
    select_best(a.t, a.pass_map, [&](int pass) { return load_rec(a.tmp + (size_t)pass * a.stride + r); }, b0, b1);
    cg_match_rec *dst = a.out + (size_t)r * a.t.slots;
    store_rec(dst, b0);
    if (a.t.slots > 1) store_rec(dst + 1, b1);
}
cudaError_t cg_launch_select(const CgSelectArgs &a, cudaStream_t st)
{
    const int block = 256;
    cg_select_kernel<<<(unsigned)((a.n_reads + block - 1) / block), block, 0, st>>>(a);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Generic kernel (wide cells / long reads): no staging, columns in HBM scratch
// ------------------------------------------------------------------------------------------
__global__ void cg_trim_generic_kernel(const CgKernelArgs a)
{
    const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    const SetView S = make_set_view(a.blob, a.masks64, a.enc, a.index);
    PackedCol colp; colp.base = a.scratch_p + gtid; colp.stride = (int)a.scratch_stride;
    WideCol colw; colw.base = a.scratch_w + gtid; colw.stride = a.scratch_stride;
    for (long long r = gtid; r < a.n_reads; r += nthreads) {
        const long long o0 = a.offsets[r], o1 = a.offsets[r + 1];
        const int n = (int)(o1 - o0);
        const uint8_t *p = a.seq + o0;
        uint32_t bad = 0;
        for (int i = 0; i < n; ++i) bad |= p[i];
        if (bad & 0x80) atomicOr(a.err_flag, 1);
        process_read<true>(S, p, a.qual ? a.qual + o0 : nullptr, n, a.qual ? a.quality_trim : 0,
                           a.cutoff_front, a.cutoff_back, a.qbase, a.times, colp, colw,
                           a.out + (size_t)r * a.times * a.slots, a.qtrim ? a.qtrim + 2 * r : nullptr,
                                    a.view ? a.view + 2 * r : nullptr);
    }
}

// ------------------------------------------------------------------------------------------
// cg_trim_light_kernel -- sets made of index lookups only (demultiplexing: IndexedPrefixAdapters /
// IndexedSuffixAdapters, adapters.py:1289-1571).  A read costs a handful of characters at one of its ends, packed to
// 2 bits each, and one probe sequence in the hash table (match_indexed): nothing to stage, no tiles, no DP column
// -- one lane per read straight from HBM, the adapter tables read through L2, the column of the rare re-alignment
// (an N in the looked-up affix, _lookup_with_n) in local memory.  The other characters of the read are only touched
// by the check for non-ASCII bytes, which the warp does cooperatively with 16-byte loads over its 32 reads.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CG_NT) cg_trim_light_kernel(const CgKernelArgs a)
{
    const SetView S = make_set_view(a.blob, a.masks64, a.enc, a.index);
    uint32_t lcol[CG_LIGHT_ROWS];
    PackedCol colp; colp.base = lcol; colp.stride = 1;
    WideCol colw; colw.base = nullptr; colw.stride = 0;
    const int lane = threadIdx.x & 31;
    const long long n_reads = a.n_reads;
    const long long n_mt = (n_reads + 31) / 32;
    const long long warps_total = (long long)gridDim.x * (CG_NT / 32);
    const uintptr_t seq_base = (uintptr_t)a.seq;
    for (long long mt = (long long)blockIdx.x * (CG_NT / 32) + (threadIdx.x >> 5); mt < n_mt; mt += warps_total) {
        const long long r0 = mt * 32;
        const long long r1 = (r0 + 32 < n_reads) ? r0 + 32 : n_reads;
        const long long r = r0 + lane;
        // the reference raises on non-ASCII characters: all bytes of the warp's reads, coalesced
        const uintptr_t s = seq_base + (uintptr_t)a.offsets[r0], e = seq_base + (uintptr_t)a.offsets[r1];
        const uintptr_t as = (s + 15) & ~(uintptr_t)15, ae = e & ~(uintptr_t)15;
        uint32_t bad = 0;
        if (as >= ae) {
            for (uintptr_t q = s + lane; q < e; q += 32) bad |= *(const uint8_t *)q;
        } else {
            for (uintptr_t q = s + lane; q < as; q += 32) bad |= *(const uint8_t *)q;
            for (uintptr_t q = ae + lane; q < e; q += 32) bad |= *(const uint8_t *)q;
            for (uintptr_t q = as + 16u * lane; q < ae; q += 512) {
                const uint4 v = *(const uint4 *)q;
                bad |= v.x | v.y | v.z | v.w;
            }
        }
        if (bad & 0x80808080u) atomicOr(a.err_flag, 1);
        if (r < n_reads) {
            const long long o0 = a.offsets[r], o1 = a.offsets[r + 1];
            process_read<false>(S, a.seq + o0, nullptr, (int)(o1 - o0), 0, 0, 0, a.qbase, a.times, colp, colw,
                                a.out + (size_t)r * a.times * a.slots, nullptr, a.view ? a.view + 2 * r : nullptr);
        }
    }
}

cudaError_t cg_launch_light(const CgKernelArgs &a, int grid, cudaStream_t st)
{
    cg_trim_light_kernel<<<grid, CG_NT, 0, st>>>(a);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// cg_index_kernel -- the lookups themselves, for sets of index groups, one round, no quality trimming: what
// MultipleAdapters.match_to does over IndexedPrefixAdapters / IndexedSuffixAdapters groups (best score, then fewest
// errors, then first listed; adapters.py:1271-1286) with match_indexed per group.  No DP column and no per-read
// generality (45 registers instead of the 127 of process_read): the latency of the dependent probes is covered by
// three times as many resident warps.  The one thing it cannot do is re-align a key that was looked up with an N in
// it (_lookup_with_n): such reads (about 1 %) are listed in a.tasks (one 32-bit read number each) and go through
// cg_trim_light_kernel afterwards.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CG_NT) cg_index_kernel(const CgKernelArgs a)
{
    const SetView S = make_set_view(a.blob, a.masks64, a.enc, a.index);
    PackedCol colp; colp.base = nullptr; colp.stride = 0;
    WideCol colw; colw.base = nullptr; colw.stride = 0;
    const int lane = threadIdx.x & 31;
    const long long n_reads = a.n_reads;
    const long long n_mt = (n_reads + 31) / 32;
    const long long warps_total = (long long)gridDim.x * (CG_NT / 32);
    const uintptr_t seq_base = (uintptr_t)a.seq;
    uint32_t *slow_list = (uint32_t *)a.tasks;
    for (long long mt = (long long)blockIdx.x * (CG_NT / 32) + (threadIdx.x >> 5); mt < n_mt; mt += warps_total) {
        const long long r0 = mt * 32;
        const long long r1 = (r0 + 32 < n_reads) ? r0 + 32 : n_reads;
        const long long r = r0 + lane;
        // non-ASCII check over the warp's reads, coalesced (as in cg_trim_light_kernel)
        const uintptr_t s = seq_base + (uintptr_t)a.offsets[r0], e = seq_base + (uintptr_t)a.offsets[r1];
        const uintptr_t as = (s + 15) & ~(uintptr_t)15, ae = e & ~(uintptr_t)15;
        uint32_t bad = 0;
        if (as >= ae) {
            for (uintptr_t q = s + lane; q < e; q += 32) bad |= *(const uint8_t *)q;
        } else {
            for (uintptr_t q = s + lane; q < as; q += 32) bad |= *(const uint8_t *)q;
            for (uintptr_t q = ae + lane; q < e; q += 32) bad |= *(const uint8_t *)q;
            for (uintptr_t q = as + 16u * lane; q < ae; q += 512) {
                const uint4 v = *(const uint4 *)q;
                bad |= v.x | v.y | v.z | v.w;
            }
        }
        if (bad & 0x80808080u) atomicOr(a.err_flag, 1);
        bool slow = false;
        if (r < n_reads) {
            const long long o0 = a.offsets[r], o1 = a.offsets[r + 1];
            const int n = (int)(o1 - o0);
            CgHit best; best.adapter = -1; best.remove = 0;
            best.astart = best.astop = best.rstart = best.rstop = best.score = best.errors = 0;
            int best_group = 0;
            bool have = false;
            for (int g = 0; g < S.h->n_groups && !slow; ++g) {
                CgHit h;
                if (!match_indexed<false>(S, S.gr[g].a0, a.seq + o0, n, colp, colw, h, &slow)) continue;
                if (!have || h.score > best.score || (h.score == best.score && h.errors < best.errors)) {
                    have = true; best = h; best_group = g;
                }
            }
            if (!slow) store_hit(a.out + (size_t)r * a.slots, best, have ? best_group : 0, have ? n : 0);
        }
        const uint32_t ballot = __ballot_sync(0xffffffffu, slow);
        if (ballot) {
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(a.task_count, (unsigned long long)__popc(ballot));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (slow) slow_list[base + __popc(ballot & ((1u << lane) - 1u))] = (uint32_t)r;
        }
    }
}

// the reads cg_index_kernel listed: the general per-read pass, one lane per listed read
__global__ void __launch_bounds__(CG_NT) cg_trim_listed_kernel(const CgKernelArgs a)
{
    const SetView S = make_set_view(a.blob, a.masks64, a.enc, a.index);
    uint32_t lcol[CG_LIGHT_ROWS];
    PackedCol colp; colp.base = lcol; colp.stride = 1;
    WideCol colw; colw.base = nullptr; colw.stride = 0;
    const uint32_t *list = (const uint32_t *)a.tasks;
    const unsigned long long n_listed = *a.task_count;
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)n_listed; i += nthreads) {
        const long long r = (long long)list[i];
        const long long o0 = a.offsets[r], o1 = a.offsets[r + 1];
        process_read<false>(S, a.seq + o0, nullptr, (int)(o1 - o0), 0, 0, 0, a.qbase, 1, colp, colw,
                            a.out + (size_t)r * a.slots, nullptr, nullptr);
    }
}

int cg_device_sm_count()
{
    // queried once per device (0: not yet); a launch only asks which device is current
    static std::atomic<int> cached[64];
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 1;
    if (dev >= 0 && dev < 64 && (sms = cached[dev].load(std::memory_order_relaxed)) > 0) return sms;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1) return 1;
    if (dev >= 0 && dev < 64) cached[dev].store(sms, std::memory_order_relaxed);
    return sms;
}

cudaError_t cg_launch_index(const CgKernelArgs &a, int grid, cudaStream_t st)
{
    cg_index_kernel<<<grid, CG_NT, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    // (few reads are listed: a fixed small grid, grid-stride)
    cg_trim_listed_kernel<<<cg_device_sm_count(), CG_NT, 0, st>>>(a);
    return cudaGetLastError();
}

// One read, one aligner adapter, exact int32 cells, every computed cell recorded: Aligner.enable_debug()'s matrices.
__global__ void cg_locate_debug_kernel(const uint8_t *blob, const uint8_t *enc768, const uint8_t *query, int n,
                                       int *scratch /* 3 (m + 1) */, int32_t *cost, int32_t *score, int32_t *result8)
{
    if (threadIdx.x || blockIdx.x) return;
    const SetView S = make_set_view(blob, nullptr, enc768, nullptr);
    const CgAdapter &A = S.ad[0];
    ReadView rv; rv.p = query; rv.n = n; rv.rev = 0;
    WideCol col; col.base = scratch; col.stride = 1;
    int o[6] = {0, 0, 0, 0, 0, 0};
    const bool found = locate_core<WideCell, WideCol>(A, S.pool + A.ref_off, (const int32_t *)(S.pool + A.ncount_off),
                                                      (const int32_t *)(S.pool + A.maxcost_off), enc768 + 256 * A.query_enc,
                                                      rv, col, o, 0xFFFFFFFFu, 0, cost, score);
    result8[0] = found ? 1 : 0;
    for (int i = 0; i < 6; ++i) result8[1 + i] = o[i];
    result8[7] = 0;
}

cudaError_t cg_launch_locate_debug(const uint8_t *d_blob, const uint8_t *d_enc, const uint8_t *d_query, int n,
                                   int *d_scratch, int32_t *d_cost, int32_t *d_score, int32_t *d_result, cudaStream_t st)
{
    cg_locate_debug_kernel<<<1, 32, 0, st>>>(d_blob, d_enc, d_query, n, d_scratch, d_cost, d_score, d_result);
    return cudaGetLastError();
}

cudaError_t cg_launch_generic(const CgKernelArgs &a, int grid, int block, cudaStream_t st)
{
    cg_trim_generic_kernel<<<grid, block, 0, st>>>(a);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Stand-alone batched KmerFinder.kmers_present (_kmer_finder.pyx:170-213)
// ------------------------------------------------------------------------------------------
__global__ void cg_kmers_present_kernel(const CgEntry *ents, int n_entries, const uint64_t *masks,
                                        const uint8_t *seq, const int64_t *offsets, long long n_reads,
                                        uint8_t *out, int *err)
{
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n_reads; r += nthreads) {
        ReadView rv; rv.p = seq + offsets[r]; rv.n = (int)(offsets[r + 1] - offsets[r]); rv.rev = 0;
        uint32_t bad = 0;
        for (int i = 0; i < rv.n; ++i) bad |= rv.p[i];
        if (bad & 0x80) atomicOr(err, 1);
        out[r] = kmers_present_core(ents, n_entries, masks, rv) ? 1 : 0;
    }
}

cudaError_t cg_launch_kmers_present(const CgEntry *d_entries, int n_entries, const uint64_t *d_masks,
                                    const uint8_t *d_seq, const int64_t *d_offsets, long long n_reads,
                                    uint8_t *d_out, int *d_err, cudaStream_t st)
{
    const int block = 128;
    long long grid = (n_reads + block - 1) / block;
    grid = cg_grid_cap(grid, 16);
    if (grid < 1) grid = 1;
    cg_kmers_present_kernel<<<(int)grid, block, 0, st>>>(d_entries, n_entries, d_masks, d_seq, d_offsets,
                                                         n_reads, d_out, d_err);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Stand-alone batched quality_trim_index (qualtrim.pyx:22-73)
// ------------------------------------------------------------------------------------------
__global__ void cg_quality_trim_kernel(const uint8_t *qual, const int64_t *offsets, long long n_reads,
                                       int cutoff_front, int cutoff_back, int base, int32_t *out)
{
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n_reads; r += nthreads) {
        int s, e;
        quality_trim_core(qual + offsets[r], (int)(offsets[r + 1] - offsets[r]), cutoff_front, cutoff_back,
                          base, &s, &e);
        out[2 * r] = s; out[2 * r + 1] = e;
    }
}

cudaError_t cg_launch_quality_trim(const uint8_t *d_qual, const int64_t *d_offsets, long long n_reads,
                                   int cutoff_front, int cutoff_back, int base, int32_t *d_out,
                                   cudaStream_t st)
{
    const int block = 128;
    long long grid = (n_reads + block - 1) / block;
    grid = cg_grid_cap(grid, 16);
    if (grid < 1) grid = 1;
    cg_quality_trim_kernel<<<(int)grid, block, 0, st>>>(d_qual, d_offsets, n_reads, cutoff_front,
                                                        cutoff_back, base, d_out);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Stand-alone batched nextseq_trim_index / poly_a_trim_index (qualtrim.pyx:76-169): the other two
// per-read scans of the modifier chain (NextseqQualityTrimmer, PolyATrimmer; modifiers.py:825-837,
// 861-918).  One lane per read; the scans run from the 3' end and stop early, so most reads touch
// only their last sectors.
// ------------------------------------------------------------------------------------------
__global__ void cg_nextseq_trim_kernel(const uint8_t *seq, const uint8_t *qual, const int64_t *offsets,
                                       long long n_reads, int cutoff, int base, int32_t *out)
{
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n_reads; r += nthreads) {
        const long long o = offsets[r];
        out[r] = nextseq_trim_core(seq + o, qual + o, (int)(offsets[r + 1] - o), cutoff, base);
    }
}
__global__ void cg_poly_a_trim_kernel(const uint8_t *seq, const int64_t *offsets, long long n_reads, int revcomp,
                                      int32_t *out, int *err_flag)
{
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n_reads; r += nthreads) {
        const long long o = offsets[r];
        const int n = (int)(offsets[r + 1] - o);
        out[r] = poly_a_trim_core(seq + o, n, revcomp);
    }
    (void)err_flag;
}
__global__ void cg_expected_errors_kernel(const uint8_t *qual, const int64_t *offsets, long long n_reads, int base,
                                          const double *table, double *out)
{
    __shared__ double s_table[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_table[i] = table[i];
    __syncthreads();
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n_reads; r += nthreads) {
        const long long o = offsets[r];
        out[r] = expected_errors_core(qual + o, (int)(offsets[r + 1] - o), base, s_table);
    }
}
cudaError_t cg_launch_expected_errors(const uint8_t *d_qual, const int64_t *d_offsets, long long n_reads, int base,
                                      const double *d_table, double *d_out, cudaStream_t st)
{
    const int block = 128;
    long long grid = (n_reads + block - 1) / block;
    grid = cg_grid_cap(grid, 16);
    if (grid < 1) grid = 1;
    cg_expected_errors_kernel<<<(int)grid, block, 0, st>>>(d_qual, d_offsets, n_reads, base, d_table, d_out);
    return cudaGetLastError();
}
cudaError_t cg_launch_nextseq_trim(const uint8_t *d_seq, const uint8_t *d_qual, const int64_t *d_offsets,
                                   long long n_reads, int cutoff, int base, int32_t *d_out, cudaStream_t st)
{
    const int block = 128;
    long long grid = (n_reads + block - 1) / block;
    grid = cg_grid_cap(grid, 16);
    if (grid < 1) grid = 1;
    cg_nextseq_trim_kernel<<<(int)grid, block, 0, st>>>(d_seq, d_qual, d_offsets, n_reads, cutoff, base, d_out);
    return cudaGetLastError();
}
cudaError_t cg_launch_poly_a_trim(const uint8_t *d_seq, const int64_t *d_offsets, long long n_reads, int revcomp,
                                  int32_t *d_out, cudaStream_t st)
{
    const int block = 128;
    long long grid = (n_reads + block - 1) / block;
    grid = cg_grid_cap(grid, 16);
    if (grid < 1) grid = 1;
    cg_poly_a_trim_kernel<<<(int)grid, block, 0, st>>>(d_seq, d_offsets, n_reads, revcomp, d_out, nullptr);
    return cudaGetLastError();
}

// offsets of a chunk of equally long reads: out[i] = base + i * len
__global__ void cg_fill_offsets_kernel(int64_t *out, long long base, long long len, long long count)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) out[i] = base + i * len;
}
cudaError_t cg_launch_fill_offsets(int64_t *d_out, long long base, long long len, long long count, cudaStream_t st)
{
    const int block = 256;
    cg_fill_offsets_kernel<<<(unsigned)((count + block - 1) / block), block, 0, st>>>(d_out, base, len, count);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Expansion of the compressed host-to-device stream of cg_process_batch (cg_hostpack.h): every
// stream byte holds three characters of the alphabet {A, C, G, T, N, escape} in base 6; escaped
// positions are overwritten from the exception list afterwards, which restores the caller's
// bytes exactly.  One thread expands 16 stream bytes (one 16-byte load) into 48 characters
// (three 16-byte stores).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cg_unpack3_kernel(const uint4 *__restrict__ packed, uint4 *__restrict__ out,
                                                          long long n_vec)
{
    __shared__ uint32_t lut[256];
    {
        const uint32_t ch = 0x41u | (0x43u << 8) | (0x47u << 16) | (0x54u << 24);   // "ACGT"
        const int i = threadIdx.x;
        const int v0 = i / 36, v1 = (i / 6) % 6, v2 = i % 6;
        auto chr = [&](int v) -> uint32_t { return v < 4 ? (ch >> (8 * v)) & 0xFFu : (v == 4 ? 0x4Eu : 0x41u); };
        lut[i] = chr(v0) | (chr(v1) << 8) | (chr(v2) << 16);
    }
    __syncthreads();
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += stride) {
        const uint4 p = __ldg(packed + i);
        const uint32_t w[4] = {p.x, p.y, p.z, p.w};
        uint32_t o[12];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t t0 = lut[w[k] & 0xFFu], t1 = lut[(w[k] >> 8) & 0xFFu];
            const uint32_t t2 = lut[(w[k] >> 16) & 0xFFu], t3 = lut[w[k] >> 24];
            o[3 * k + 0] = t0 | (t1 << 24);
            o[3 * k + 1] = (t1 >> 8) | (t2 << 16);
            o[3 * k + 2] = (t2 >> 16) | (t3 << 8);
        }
        out[3 * i + 0] = make_uint4(o[0], o[1], o[2], o[3]);
        out[3 * i + 1] = make_uint4(o[4], o[5], o[6], o[7]);
        out[3 * i + 2] = make_uint4(o[8], o[9], o[10], o[11]);
    }
}
__global__ void cg_unpack_fix_kernel(const unsigned long long *__restrict__ exc, long long n_exc, uint8_t *out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_exc) {
        const unsigned long long e = exc[i];
        out[e >> 8] = (uint8_t)(e & 0xFFu);
    }
}
cudaError_t cg_launch_unpack3(const uint8_t *d_packed, long long packed_bytes, uint8_t *d_out,
                              const unsigned long long *d_exc, long long n_exc, cudaStream_t st)
{
    const long long n_vec = packed_bytes / 16;
    if (n_vec > 0) {
        const int block = 256;
        long long grid = (n_vec + block - 1) / block;
        grid = cg_grid_cap(grid, 8);
        cg_unpack3_kernel<<<(int)grid, block, 0, st>>>((const uint4 *)d_packed, (uint4 *)d_out, n_vec);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    if (n_exc > 0) {
        const int block = 256;
        cg_unpack_fix_kernel<<<(unsigned)((n_exc + block - 1) / block), block, 0, st>>>(d_exc, n_exc, d_out);
    }
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Longest read of a batch (device offsets)
// ------------------------------------------------------------------------------------------
__global__ void cg_max_len_kernel(const int64_t *offsets, long long n_reads, int *out)
{
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    int best = 0;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n_reads; r += nthreads) {
        const long long d = offsets[r + 1] - offsets[r];
        const int v = d > 2147483647LL ? 2147483647 : (int)d;
        best = v > best ? v : best;
    }
    for (int o = 16; o > 0; o >>= 1) {
        const int other = __shfl_xor_sync(0xffffffffu, best, o);
        best = other > best ? other : best;
    }
    if ((threadIdx.x & 31) == 0) atomicMax(out, best);
}

cudaError_t cg_launch_max_len(const int64_t *d_offsets, long long n_reads, int *d_out, cudaStream_t st)
{
    const int block = 256;
    long long grid = (n_reads + block - 1) / block;
    grid = cg_grid_cap(grid, 8);
    if (grid < 1) grid = 1;
    cg_max_len_kernel<<<(int)grid, block, 0, st>>>(d_offsets, n_reads, d_out);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Trim statistics: the fixed-layout int64 vector that is all-reduced across GPUs
// (Statistics.__iadd__ report.py:81-126; EndStatistics.errors adapters.py:96-111,193-199)
// ------------------------------------------------------------------------------------------
template <bool SMEM_HIST>
__global__ void cg_stats_kernel(const uint8_t *seq, const int64_t *offsets, long long n_reads, int quality_trim, int times,
                                int slots, const cg_match_rec *matches, const int32_t *qtrim,
                                int n_adapters, int max_len, int kmax, unsigned long long *stats,
                                const uint4 *task_list, int task_rec, const unsigned long long *task_count,
                                int count_lengths, int upper)
{
    // per-CTA histograms in shared memory (32-bit counts, flushed once): the read-length histogram always (every
    // read adds to it, mostly to the same few bins), the per-adapter part if it fits (SMEM_HIST); a global
    // histogram would otherwise take one contended atomic per read
    extern __shared__ unsigned int s_hist[];
    const long long nbins = cg_stats_total(n_adapters, max_len, kmax) - CG_STATS_SCALARS;
    const long long n_local = SMEM_HIST ? nbins : (count_lengths ? (long long)(max_len + 1) : 0);
    for (long long i = threadIdx.x; i < n_local; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    unsigned long long n = 0;
    StatsScalars sc; sc.bp = sc.with_adapters = sc.qtrim_bp = sc.adapter_bp = 0;
    unsigned long long *hist = stats + CG_STATS_SCALARS;
    // task_list: only the reads of a task list of the split pipeline (those its first stage did not count itself)
    long long n_items = n_reads;
    if (task_list) {
        const unsigned long long t = *task_count;
        n_items = t < (unsigned long long)n_reads ? (long long)t : n_reads;
    }
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_items; i += nthreads) {
        long long r = i;
        if (task_list) {
            const uint4 t = task_list[(size_t)task_rec * i];
            r = (long long)t.x;
        }
        const long long o0 = offsets[r];
        const int len = (int)(offsets[r + 1] - o0);
        n += 1;
        const bool hq = quality_trim && qtrim;
        stats_read_core(seq ? seq + o0 : nullptr, len, hq, hq ? qtrim[2 * r] : 0, hq ? qtrim[2 * r + 1] : len,
                        matches + (size_t)r * times * slots, times, slots, n_adapters, max_len, kmax, sc,
                        [&](long long idx, unsigned int v) {
                            if (!count_lengths && idx <= max_len) return;
                            if (idx < n_local) atomicAdd(&s_hist[idx], v);
                            else atomicAdd(&hist[idx], (unsigned long long)v);
                        },
                        upper != 0);
    }
    // warp-reduce the scalar counters, one atomic per warp
    for (int o = 16; o > 0; o >>= 1) {
        n += __shfl_xor_sync(0xffffffffu, n, o);
        sc.bp += __shfl_xor_sync(0xffffffffu, sc.bp, o);
        sc.with_adapters += __shfl_xor_sync(0xffffffffu, sc.with_adapters, o);
        sc.qtrim_bp += __shfl_xor_sync(0xffffffffu, sc.qtrim_bp, o);
        sc.adapter_bp += __shfl_xor_sync(0xffffffffu, sc.adapter_bp, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&stats[0], n); atomicAdd(&stats[1], sc.bp); atomicAdd(&stats[2], sc.with_adapters);
        atomicAdd(&stats[3], sc.qtrim_bp); atomicAdd(&stats[4], sc.adapter_bp);
    }
    __syncthreads();
    for (long long i = threadIdx.x; i < n_local; i += blockDim.x) {
        const unsigned int v = s_hist[i];
        if (v) atomicAdd(&hist[i], (unsigned long long)v);
    }
}

cudaError_t cg_launch_stats(const uint8_t *d_seq, const int64_t *d_offsets, long long n_reads, int quality_trim, int times,
                            int slots, const cg_match_rec *d_matches, const int32_t *d_qtrim,
                            int n_adapters, int max_len, int kmax, unsigned long long *d_stats,
                            cudaStream_t st, const uint4 *d_task_list, int task_rec, const unsigned long long *d_task_count,
                            int count_lengths, int upper)
{
    const int block = 256;
    long long grid = (n_reads + block - 1) / block;
    grid = cg_grid_cap(grid, 8);
    if (grid < 1) grid = 1;
    const size_t hist_bytes = (size_t)(cg_stats_total(n_adapters, max_len, kmax) - CG_STATS_SCALARS) * sizeof(unsigned int);
    const size_t len_bytes = count_lengths ? (size_t)(max_len + 1) * sizeof(unsigned int) : 0;
    if (len_bytes > 48 * 1024) return cudaErrorInvalidValue;
    // a CTA handles n_reads / grid reads, so 32-bit per-CTA counts cannot overflow below 2^32 reads per CTA
    if (hist_bytes <= 48 * 1024 && n_reads / grid < (1LL << 31))
        cg_stats_kernel<true><<<(int)grid, block, hist_bytes, st>>>(d_seq, d_offsets, n_reads, quality_trim, times, slots,
                                                                     d_matches, d_qtrim, n_adapters, max_len, kmax, d_stats,
                                                                     d_task_list, task_rec, d_task_count, count_lengths,
                                                                     upper);
    else
        cg_stats_kernel<false><<<(int)grid, block, len_bytes, st>>>(d_seq, d_offsets, n_reads, quality_trim, times, slots,
                                                                     d_matches, d_qtrim, n_adapters, max_len, kmax, d_stats,
                                                                     d_task_list, task_rec, d_task_count, count_lengths,
                                                                     upper);
    return cudaGetLastError();
}
