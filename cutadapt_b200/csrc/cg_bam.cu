// cg_bam.cu -- unaligned BAM input of the FASTQ path: the records of the inflated BAM stream become FASTQ text in a slot
// (cg_bam_core.cuh has the format and every decision; cg_fastq_submit_gzip in cg_api.cu runs the steps).
//
// bam_spec_kernel     one warp per tile: the first bam_candidate offset (a ballot per 32 offsets), then one
//                     lane walks the tile speculatively and marks its offsets.
// bam_resolve_kernel  one block: the tiles' link words are read into shared memory a window at a time, one thread
//                     follows the true chain through them and walks again the tiles whose entry is not on their walk.
// bam_count_kernel    one thread per bitmap word: the record starts it holds (from its tile's entry to the chain's end).
// bam_starts_kernel   after a scan of the counts: every start and its FASTQ size, in order.
// bam_cut_kernel      one thread, after a scan of the sizes: the longest prefix of records under the size limit.
// bam_emit_kernel     one warp per record: its refusals (every record of the chain) and its FASTQ text (the cut's).
#include <cuda_runtime.h>

#include <climits>

#include "cg_bam_core.cuh"
#include "cg_kernels.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWin = 4096;                 // link words per window of the resolve (32 KiB of shared memory)
static_assert(BAM_TILE % 32 == 0, "a tile's bitmap words must be its own");

__global__ void __launch_bounds__(kThreads) bam_spec_kernel(const uint8_t *__restrict__ b, long long n, long long T,
                                                            uint32_t *bm, uint64_t *link)
{
    const long long t = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (t >= T) return;
    const long long lo = t * BAM_TILE, hi = lo + BAM_TILE < n ? lo + BAM_TILE : n;
    long long start = t == 0 ? 0 : hi;
    for (long long base = lo; t != 0 && base < hi; base += 32) {
        const long long p = base + lane;
        const unsigned v = __ballot_sync(0xffffffffu, p < hi && bam_candidate(b, n, p));
        if (v) {
            start = base + __ffs(v) - 1;
            break;
        }
    }
    if (lane == 0) link[t] = bam_spec_walk(b, n, hi, start, bm);
}

__global__ void __launch_bounds__(kThreads) bam_resolve_kernel(const uint8_t *__restrict__ b, long long n, long long T,
                                                               uint32_t *bm, const uint64_t *link, long long *entry,
                                                               BamSum *sum)
{
    __shared__ uint64_t win[kWin];
    __shared__ long long s_p;
    __shared__ int s_on, s_done;
    long long rewalked = 0;
    if (threadIdx.x == 0) {
        s_p = 0;
        s_on = 1;                              // tile 0's walk starts at 0
        s_done = 0;
    }
    for (;;) {
        __syncthreads();
        if (s_done) break;
        const long long w0 = s_p / BAM_TILE;
        for (long long i = threadIdx.x; i < kWin && w0 + i < T; i += blockDim.x)
            win[i] = bam_link_resolve(link[w0 + i], n, bm);
        __syncthreads();
        if (threadIdx.x != 0) continue;
        long long p = s_p;
        int on = s_on;
        for (;;) {
            if (p >= n) {
                sum->end = p;
                sum->end_st = BAM_OK;
                s_done = 1;
                break;
            }
            const long long t = p / BAM_TILE;
            if (t >= w0 + kWin) break;
            entry[t] = p;
            const uint64_t w = bam_resolve_step(b, n, BAM_TILE, p, on, win[t - w0], bm, &rewalked);
            if (bam_link_st(w) != BAM_OK) {
                sum->end = bam_link_pos(w);
                sum->end_st = bam_link_st(w);
                s_done = 1;
                break;
            }
            p = bam_link_pos(w);
            on = bam_link_on(w);
        }
        s_p = p;
        s_on = on;
        if (s_done) sum->rewalked = rewalked;
    }
}

__global__ void __launch_bounds__(kThreads) bam_count_kernel(const uint32_t *__restrict__ bm, long long n_words,
                                                             const long long *entry, const BamSum *sum, int32_t *cnt)
{
    const long long w = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (w < n_words) cnt[w] = __popc(bam_word_starts(bm, w, BAM_TILE, entry, sum->end));
}

__global__ void __launch_bounds__(kThreads) bam_starts_kernel(const uint8_t *__restrict__ b, const uint32_t *__restrict__ bm,
                                                              long long n_words, const long long *entry, const BamSum *sum,
                                                              const int64_t *woff, uint32_t *start, int32_t *fsize)
{
    const long long w = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (w >= n_words) return;
    uint32_t m = bam_word_starts(bm, w, BAM_TILE, entry, sum->end);
    long long o = woff[w];
    while (m) {
        const long long p = (w << 5) + __ffs(m) - 1;
        m &= m - 1;
        const long long fs = bam_fastq_size(b + p);
        start[o] = (uint32_t)p;
        fsize[o] = fs > INT_MAX ? INT_MAX : (int32_t)fs;   // such a record never fits the limit
        ++o;
    }
}

__global__ void bam_cut_kernel(const int64_t *woff, long long n_words, const uint32_t *start, const int64_t *foff,
                               long long limit, BamSum *sum)
{
    const long long R = woff[n_words];
    long long lo = 0, hi = R;                  // the largest k with foff[k] <= limit (foff[0] = 0)
    while (lo < hi) {
        const long long mid = (lo + hi + 1) / 2;
        if (foff[mid] <= limit) lo = mid;
        else hi = mid - 1;
    }
    sum->n_rec = R;
    sum->n_cut = lo;
    sum->fq_bytes = foff[lo];
    sum->bam_cut = lo < R ? (long long)start[lo] : sum->end;
}

__global__ void __launch_bounds__(kThreads) bam_emit_kernel(const uint8_t *__restrict__ b, const uint32_t *start,
                                                            const int64_t *foff, long long n_rec, long long n_cut,
                                                            uint8_t *__restrict__ out, unsigned long long *err)
{
    const long long i = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n_rec) return;
    const uint8_t *rec = b + start[i];
    const BamFields f = bam_fields(rec);
    const bool write = i < n_cut;
    uint8_t *o = out + (write ? foff[i] : 0);
    const long long name_end = f.lrn, seq0 = name_end + 1, qual0 = seq0 + f.lseq + 3;
    bool bad_name = false, bad_qual = false;
    for (int j = lane; j + 1 < f.lrn; j += 32) {
        const uint8_t c = rec[f.name + j];
        bad_name |= !bam_name_ok(c);
        if (write) o[1 + j] = c;
    }
    for (long long j = lane; j < f.lseq; j += 32) {
        const uint8_t s = rec[f.seq + (j >> 1)];
        const uint8_t q = rec[f.qual + j];
        bad_qual |= q > 93;
        if (write) {
            o[seq0 + j] = bam_base((j & 1) ? s : s >> 4);
            o[qual0 + j] = (uint8_t)(q + 33);
        }
    }
    bad_name = __any_sync(0xffffffffu, bad_name);
    bad_qual = __any_sync(0xffffffffu, bad_qual);
    if (lane != 0) return;
    if (write) {
        o[0] = '@';
        o[name_end] = '\n';
        o[seq0 + f.lseq] = '\n';
        o[seq0 + f.lseq + 1] = '+';
        o[seq0 + f.lseq + 2] = '\n';
        o[qual0 + f.lseq] = '\n';
    }
    const int code = f.flag != 4 ? BAM_R_FLAG
                     : bad_name ? BAM_R_NAME
                     : f.lseq > 0 && rec[f.qual] == 0xFF ? BAM_R_NOQUAL
                     : bad_qual ? BAM_R_QUAL
                                : 0;
    if (code) atomicMin(err, ((unsigned long long)i << 3) | (unsigned long long)code);
}

unsigned grid(long long threads) { return (unsigned)((threads + kThreads - 1) / kThreads); }

}  // namespace

long long cg_bam_words(long long n) { return (n + 31) / 32; }
long long cg_bam_tiles(long long n) { return (n + BAM_TILE - 1) / BAM_TILE; }
long long cg_bam_max_records(long long n) { return n / BAM_MIN_RECORD + 1; }

cudaError_t cg_launch_bam_bounds(const uint8_t *d_buf, long long n, uint32_t *d_bm, uint64_t *d_link, long long *d_entry,
                                 BamSum *d_sum, int32_t *d_cnt, cudaStream_t st)
{
    const long long T = cg_bam_tiles(n), W = cg_bam_words(n);
    cudaError_t e;
    if ((e = cudaMemsetAsync(d_sum, 0, sizeof(BamSum), st)) != cudaSuccess) return e;
    if (T) {
        if ((e = cudaMemsetAsync(d_bm, 0, (size_t)W * sizeof(uint32_t), st)) != cudaSuccess) return e;
        if ((e = cudaMemsetAsync(d_entry, 0xFF, (size_t)T * sizeof(long long), st)) != cudaSuccess) return e;
        bam_spec_kernel<<<grid(T * 32), kThreads, 0, st>>>(d_buf, n, T, d_bm, d_link);
    }
    bam_resolve_kernel<<<1, kThreads, 0, st>>>(d_buf, n, T, d_bm, d_link, d_entry, d_sum);
    if (W) bam_count_kernel<<<grid(W), kThreads, 0, st>>>(d_bm, W, d_entry, d_sum, d_cnt);
    return cudaGetLastError();
}

cudaError_t cg_launch_bam_starts(const uint8_t *d_buf, long long n, const uint32_t *d_bm, const long long *d_entry,
                                 const BamSum *d_sum, const int64_t *d_woff, uint32_t *d_start, int32_t *d_fsize,
                                 cudaStream_t st)
{
    const long long W = cg_bam_words(n);
    cudaError_t e;
    if ((e = cudaMemsetAsync(d_fsize, 0, (size_t)cg_bam_max_records(n) * sizeof(int32_t), st)) != cudaSuccess) return e;
    if (W) bam_starts_kernel<<<grid(W), kThreads, 0, st>>>(d_buf, d_bm, W, d_entry, d_sum, d_woff, d_start, d_fsize);
    return cudaGetLastError();
}

cudaError_t cg_launch_bam_cut(const int64_t *d_woff, long long n, const uint32_t *d_start, const int64_t *d_foff,
                              long long limit, BamSum *d_sum, cudaStream_t st)
{
    bam_cut_kernel<<<1, 1, 0, st>>>(d_woff, cg_bam_words(n), d_start, d_foff, limit, d_sum);
    return cudaGetLastError();
}

cudaError_t cg_launch_bam_emit(const uint8_t *d_buf, const uint32_t *d_start, const int64_t *d_foff, long long n_rec,
                               long long n_cut, uint8_t *d_out, unsigned long long *d_err, cudaStream_t st)
{
    if (n_rec <= 0) return cudaSuccess;
    bam_emit_kernel<<<grid(n_rec * 32), kThreads, 0, st>>>(d_buf, d_start, d_foff, n_rec, n_cut, d_out, d_err);
    return cudaGetLastError();
}
