// cg_gzip.cu -- gzip output of the FASTQ path: the formatted destinations are cut into members of GZ_MEMBER plain bytes
// and compressed on the device before the download (cg_gzip_core.cuh has the format and every decision).
//
// gz_compress_kernel: one block per piece.  A gzip piece is a member: staged in shared memory, a CRC per sub-block
// combined by one thread, the candidate table built one round of 256 positions at a time (__match_any_sync inside a warp,
// atomicMax on the buckets between rounds, so the table does not depend on scheduling), one thread per sub-block parses
// and counts symbols, one thread builds each Huffman code, a block scan places every sub-block's bits and all threads
// write them into shared memory.  A plain piece (a destination written uncompressed) is copied as it is.
// gz_gather_kernel packs the pieces behind each other once the host has their offsets.
#include <cuda_runtime.h>

#include "cg_gzip_core.cuh"
#include "cg_kernels.cuh"

namespace {

constexpr int kThreads = 256;
// shared memory: the member (later the output bits), the candidates (later the tokens), the hash table (later the
// trees), CRC tables and per-sub-block values
constexpr int kSmData = 0;
constexpr int kSmTok = kSmData + 65536;
constexpr int kSmAux = kSmTok + GZ_MEMBER * 2;
constexpr int kAuxBytes = (1 << GZ_HASH_BITS) * 4;
constexpr int kSmTab = kSmAux + kAuxBytes;
constexpr int kSmMat = kSmTab + 256 * 4;
constexpr int kSmPart = kSmMat + 32 * 4;
constexpr int kSmNtok = kSmPart + kThreads * 4;
constexpr int kSmOff = kSmNtok + kThreads * 4;
constexpr int kSmWarp = kSmOff + kThreads * 4;
constexpr int kSmBytes = kSmWarp + 32 * 4;
static_assert(sizeof(GzTrees) + (4 * 288 + 2 * 64) * 4 <= kAuxBytes, "trees and their scratch fit where the hash table was");
static_assert(GZ_MEMBER + GZ_OVERHEAD <= GZ_SLOT && GZ_NSUB < kThreads, "layout");

__global__ void __launch_bounds__(kThreads) gz_compress_kernel(const uint8_t *__restrict__ src, const CgGzPiece *pieces,
                                                               uint8_t *slots, int32_t *sizes)
{
    extern __shared__ __align__(16) uint8_t sm[];
    uint8_t *d = sm + kSmData;
    uint32_t *ow = reinterpret_cast<uint32_t *>(sm + kSmData);
    uint16_t *tok = reinterpret_cast<uint16_t *>(sm + kSmTok);
    int *bucket = reinterpret_cast<int *>(sm + kSmAux);
    GzTrees &T = *reinterpret_cast<GzTrees *>(sm + kSmAux);
    uint32_t *scratch = reinterpret_cast<uint32_t *>(sm + kSmAux + sizeof(GzTrees));
    uint32_t *tab = reinterpret_cast<uint32_t *>(sm + kSmTab);
    uint32_t *mat = reinterpret_cast<uint32_t *>(sm + kSmMat);
    uint32_t *part = reinterpret_cast<uint32_t *>(sm + kSmPart);
    int *ntok = reinterpret_cast<int *>(sm + kSmNtok);
    uint32_t *off = reinterpret_cast<uint32_t *>(sm + kSmOff);
    uint32_t *wsum = reinterpret_cast<uint32_t *>(sm + kSmWarp);
    __shared__ uint32_t s_crc, s_total;

    const int t = threadIdx.x, lane = t & 31;
    const CgGzPiece pc = pieces[blockIdx.x];
    const int n = pc.len;
    const uint8_t *g = src + pc.src;
    uint8_t *slot = slots + (size_t)blockIdx.x * GZ_SLOT;
    if (!pc.gz) {
        for (int i = t; i < n; i += kThreads) slot[i] = g[i];
        if (t == 0) sizes[blockIdx.x] = n;
        return;
    }
    for (int i = t; i < n; i += kThreads) d[i] = g[i];
    for (int i = t; i < (1 << GZ_HASH_BITS); i += kThreads) bucket[i] = -1;
    tab[t] = gz_crc_entry((uint32_t)t);
    __syncthreads();
    if (t < 32) mat[t] = gz_crc_zeros(1u << t, GZ_SUB, tab);
    const int start = t * GZ_SUB;
    if (start + GZ_SUB <= n) part[t] = gz_crc_raw(0, d + start, GZ_SUB, tab);

    for (int r0 = 0; r0 < n; r0 += GZ_ROUND) {
        const int p = r0 + t;
        const bool ok = p + 4 <= n;
        const uint32_t h = ok ? gz_hash(d + p) : (1u << GZ_HASH_BITS) + lane;    // lanes without a hash match nobody
        const uint32_t before = __match_any_sync(0xffffffffu, h) & ((1u << lane) - 1);
        const int prev = before ? p - lane + (31 - __clz(before)) : -1;
        const int b = ok ? bucket[h] : -1;
        __syncthreads();
        if (p < n) tok[p] = gz_pick(prev, b);
        if (ok) atomicMax(bucket + h, p);
        __syncthreads();
    }
    for (int i = t; i < 288; i += kThreads) T.ll_freq[i] = i == 256;
    if (t < 32) T.d_freq[t] = 0;
    __syncthreads();

    int nt = 0;
    if (start < n) {
        nt = gz_parse_sub(d, n, tok, t);
        gz_tally_sub(tok, start, nt, T.ll_freq, T.d_freq);
    }
    ntok[t] = nt;
    if (t == kThreads - 1) {        // no sub-block of its own: combine the CRCs
        uint32_t c = 0xffffffffu;
        const int full = n / GZ_SUB;
        for (int s = 0; s < full; ++s) c = gz_gf2_times(mat, c) ^ part[s];
        s_crc = ~gz_crc_raw(c, d + full * GZ_SUB, n - full * GZ_SUB, tab);
    }
    __syncthreads();
    int *work = reinterpret_cast<int *>(scratch + 4 * 288);
    if (t == 0) gz_lengths(T.ll_freq, 286, 15, T.ll_len, scratch, scratch + 288, work);
    if (t == 32) gz_lengths(T.d_freq, 30, 15, T.d_len, scratch + 2 * 288, scratch + 3 * 288, work + 64);
    __syncthreads();
    if (t == 0) gz_tree_header(T, scratch, scratch + 288, work);
    __syncthreads();

    // exclusive scan of the sub-blocks' bits behind the header
    const uint32_t mine = nt ? gz_sub_bits(T, tok, start, nt) : 0;
    uint32_t incl = mine;
    for (int k = 1; k < 32; k <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, k);
        if (lane >= k) incl += v;
    }
    if (lane == 31) wsum[t >> 5] = incl;
    __syncthreads();
    uint32_t base = T.header_bits;
    for (int w = 0; w < (t >> 5); ++w) base += wsum[w];
    off[t] = base + incl - mine;
    if (t == kThreads - 1) s_total = base + incl + T.ll_len[256];
    __syncthreads();
    const uint32_t total = s_total;

    if (gz_use_stored(total, n)) {
        for (int i = t; i < n; i += kThreads) slot[15 + i] = d[i];
        if (t == 0) {
            gz_member_header(slot);
            gz_stored_head(slot + 10, n);
            gz_member_trailer(slot + 15 + n, s_crc, (uint32_t)n);
            sizes[blockIdx.x] = 15 + n + 8;
        }
        return;
    }
    const int words = (int)(total / 32) + 2;
    for (int i = t; i < words; i += kThreads) ow[i] = 0;
    __syncthreads();
    if (t == kThreads - 1) gz_write_header(T, ow);
    if (nt) gz_write_sub(T, tok, start, nt, ow, off[t]);
    if (t == 0) gz_write_eob(T, ow, total - T.ll_len[256]);
    __syncthreads();
    const int bytes = (int)((total + 7) / 8);
    for (int i = t; i < bytes; i += kThreads) slot[10 + i] = d[i];
    if (t == 0) {
        gz_member_header(slot);
        gz_member_trailer(slot + 10 + bytes, s_crc, (uint32_t)n);
        sizes[blockIdx.x] = 10 + bytes + 8;
    }
}

__global__ void __launch_bounds__(kThreads) gz_gather_kernel(const uint8_t *__restrict__ slots, const int32_t *sizes,
                                                             const int64_t *dst_off, uint8_t *out)
{
    const int n = sizes[blockIdx.x];
    const uint8_t *s = slots + (size_t)blockIdx.x * GZ_SLOT;
    uint8_t *o = out + dst_off[blockIdx.x];
    for (int i = threadIdx.x; i < n; i += kThreads) o[i] = s[i];
}

}  // namespace

cudaError_t cg_launch_gzip_compress(const uint8_t *d_src, const CgGzPiece *d_pieces, int n_pieces, uint8_t *d_slots,
                                    int32_t *d_sizes, cudaStream_t st)
{
    if (n_pieces <= 0) return cudaSuccess;
    // per call: the attribute belongs to the current device, and a context may run on any of them
    cudaError_t e = cudaFuncSetAttribute(gz_compress_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmBytes);
    if (e != cudaSuccess) return e;
    gz_compress_kernel<<<n_pieces, kThreads, kSmBytes, st>>>(d_src, d_pieces, d_slots, d_sizes);
    return cudaGetLastError();
}

cudaError_t cg_launch_gzip_gather(const uint8_t *d_slots, const int32_t *d_sizes, const int64_t *d_dst_off, int n_pieces,
                                  uint8_t *d_out, cudaStream_t st)
{
    if (n_pieces <= 0) return cudaSuccess;
    gz_gather_kernel<<<n_pieces, kThreads, 0, st>>>(d_slots, d_sizes, d_dst_off, d_out);
    return cudaGetLastError();
}
