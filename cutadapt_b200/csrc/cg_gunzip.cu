// cg_gunzip.cu -- gzip input of the FASTQ path: the members of an uploaded piece of a .gz file are inflated on the device
// (cg_gunzip_core.cuh has the format and every decision; cg_fastq_submit_gzip in cg_api.cu runs the steps).
//
// gu_cand_*_kernel  every position of 1f 8b 08, in order (a count per tile, a scan, a write).  Every member starts at
//                   one, so a false candidate costs a parse but never a wrong result.
// gu_parse_kernel   one thread (one block) per candidate parses its member without writing: status, size, plain
//                   length, CRC.
//                   Huffman parsing does not depend on the plain bytes, so every candidate runs at once.  The decode
//                   tables of each thread are in shared memory.
// gu_chain_kernel   one thread walks from member end to member end: which candidates are members, their plain offsets.
// gu_place_kernel   one thread per member inflates it again, now into its place behind the carry.
// gu_crc_kernel     one block per member: CRC-32 of 256 stretches, combined with the GF(2) shift (cg_gzip_core.cuh).
// gu_flag / gu_select kernels  the flagged newlines of the record cut and the one the cut lies behind.
#include <cuda_runtime.h>

#include "cg_gunzip_core.cuh"
#include "cg_gzip_core.cuh"
#include "cg_kernels.cuh"

namespace {

constexpr int kScanThreads = 256;
// One member per block: the decoders of different members branch apart at every symbol, so 32 of them in one warp run
// one after the other; one per block keeps every member on a warp of its own (up to 32 per SM at once).
constexpr int kParseThreads = 1;
constexpr int kCrcThreads = 256;

__device__ __forceinline__ bool gu_is_cand(const uint8_t *gz, long long n, long long p)
{
    return p + 3 <= n && gz[p] == 0x1f && gz[p + 1] == 0x8b && gz[p + 2] == 8;
}

__global__ void __launch_bounds__(kScanThreads) gu_cand_count_kernel(const uint8_t *__restrict__ gz, long long n,
                                                                     int32_t *counts)
{
    __shared__ int s_n;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const long long p = (long long)blockIdx.x * kScanThreads + threadIdx.x;
    const unsigned v = __ballot_sync(0xffffffffu, gu_is_cand(gz, n, p));
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(&s_n, __popc(v));
    __syncthreads();
    if (threadIdx.x == 0) counts[blockIdx.x] = s_n;
}

__global__ void __launch_bounds__(kScanThreads) gu_cand_write_kernel(const uint8_t *__restrict__ gz, long long n,
                                                                     const int64_t *offs, int32_t *cand)
{
    __shared__ int s_warp[kScanThreads / 32];
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const long long p = (long long)blockIdx.x * kScanThreads + t;
    const bool c = gu_is_cand(gz, n, p);
    const unsigned v = __ballot_sync(0xffffffffu, c);
    if (lane == 0) s_warp[w] = __popc(v);
    __syncthreads();
    if (!c) return;
    long long o = offs[blockIdx.x] + __popc(v & ((1u << lane) - 1));
    for (int k = 0; k < w; ++k) o += s_warp[k];
    cand[o] = (int32_t)p;
}

__global__ void __launch_bounds__(kParseThreads) gu_parse_kernel(const uint8_t *__restrict__ gz, long long n,
                                                                 const int32_t *cand, int n_cand, GuMember *res)
{
    extern __shared__ __align__(16) uint8_t sm[];
    GuTables &T = reinterpret_cast<GuTables *>(sm)[threadIdx.x];
    const int k = blockIdx.x * kParseThreads + threadIdx.x;
    if (k >= n_cand) return;
    const long long p = cand[k];
    res[k] = gu_member(gz + p, n - p, nullptr, T);
}

__global__ void gu_chain_kernel(const uint8_t *__restrict__ gz, long long n, const int32_t *cand, const GuMember *res,
                                int n_cand, int after_member, int final, long long base, long long limit, int32_t *members,
                                long long *moff, GuChain *out)
{
    *out = gu_chain(gz, n, cand, res, n_cand, after_member != 0, final != 0, base, limit, members, moff);
}

__global__ void __launch_bounds__(kParseThreads) gu_place_kernel(const uint8_t *__restrict__ gz, long long n,
                                                                 const int32_t *cand, const int32_t *members,
                                                                 const long long *moff, const GuChain *chain,
                                                                 uint8_t *out)
{
    extern __shared__ __align__(16) uint8_t sm[];
    GuTables &T = reinterpret_cast<GuTables *>(sm)[threadIdx.x];
    const int k = blockIdx.x * kParseThreads + threadIdx.x;
    if (k >= chain->n_members) return;
    const long long p = cand[members[k]];
    gu_member(gz + p, n - p, out + moff[k], T);
}

__global__ void __launch_bounds__(kCrcThreads) gu_crc_kernel(const uint8_t *__restrict__ plain, const int32_t *members,
                                                             const long long *moff, const GuMember *res, int *bad)
{
    __shared__ uint32_t tab[256], mat[32], part[kCrcThreads];
    const int t = threadIdx.x;
    const GuMember m = res[members[blockIdx.x]];
    const uint8_t *d = plain + moff[blockIdx.x];
    const long long len = m.plain;
    const int stretch = (int)max((long long)GZ_SUB, (len + kCrcThreads - 1) / kCrcThreads);
    tab[t] = gz_crc_entry((uint32_t)t);
    __syncthreads();
    if (t < 32) mat[t] = gz_crc_zeros(1u << t, stretch, tab);
    const long long start = (long long)t * stretch;
    if (start + stretch <= len) part[t] = gz_crc_raw(0, d + start, stretch, tab);
    __syncthreads();
    if (t == 0) {
        uint32_t c = 0xffffffffu;
        const int full = (int)(len / stretch);
        for (int s = 0; s < full; ++s) c = gz_gf2_times(mat, c) ^ part[s];
        c = ~gz_crc_raw(c, d + (long long)full * stretch, (int)(len - (long long)full * stretch), tab);
        if (c != m.crc) atomicMin(bad, (int)blockIdx.x);
    }
}

__global__ void gu_flag_kernel(const uint8_t *__restrict__ buf, long long n, const uint32_t *nl, long long n_nl, int fasta,
                               int32_t *flag)
{
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n_nl) flag[j] = gu_flag(buf, n, nl[j], fasta) ? 1 : 0;
}

__global__ void gu_select_kernel(const uint32_t *nl, long long n_nl, const int32_t *flag, const int64_t *offs, long long s,
                                 long long *cut)
{
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n_nl && flag[j] && offs[j] == s) *cut = (long long)nl[j] + 1;
}

}  // namespace

long long cg_gunzip_tiles(long long n_bytes) { return (n_bytes + kScanThreads - 1) / kScanThreads; }

cudaError_t cg_launch_gunzip_candidates(int phase, const uint8_t *d_gz, long long n, int32_t *d_counts,
                                        const int64_t *d_offs, int32_t *d_cand, cudaStream_t st)
{
    const long long tiles = cg_gunzip_tiles(n);
    if (tiles <= 0) return cudaSuccess;
    if (phase == 0) gu_cand_count_kernel<<<(unsigned)tiles, kScanThreads, 0, st>>>(d_gz, n, d_counts);
    else gu_cand_write_kernel<<<(unsigned)tiles, kScanThreads, 0, st>>>(d_gz, n, d_offs, d_cand);
    return cudaGetLastError();
}

cudaError_t cg_launch_gunzip_parse(const uint8_t *d_gz, long long n, const int32_t *d_cand, int n_cand, GuMember *d_res,
                                   cudaStream_t st)
{
    if (n_cand <= 0) return cudaSuccess;
    gu_parse_kernel<<<(n_cand + kParseThreads - 1) / kParseThreads, kParseThreads, kParseThreads * sizeof(GuTables), st>>>(
        d_gz, n, d_cand, n_cand, d_res);
    return cudaGetLastError();
}

cudaError_t cg_launch_gunzip_chain(const uint8_t *d_gz, long long n, const int32_t *d_cand, const GuMember *d_res,
                                   int n_cand, int after_member, int final, long long base, long long limit,
                                   int32_t *d_members, long long *d_moff, GuChain *d_chain, cudaStream_t st)
{
    gu_chain_kernel<<<1, 1, 0, st>>>(d_gz, n, d_cand, d_res, n_cand, after_member, final, base, limit, d_members, d_moff,
                                     d_chain);
    return cudaGetLastError();
}

cudaError_t cg_launch_gunzip_place(const uint8_t *d_gz, long long n, const int32_t *d_cand, const int32_t *d_members,
                                   const long long *d_moff, const GuChain *d_chain, int n_members, const GuMember *d_res,
                                   uint8_t *d_out, int *d_bad, cudaStream_t st)
{
    if (n_members <= 0) return cudaSuccess;
    gu_place_kernel<<<(n_members + kParseThreads - 1) / kParseThreads, kParseThreads, kParseThreads * sizeof(GuTables),
                      st>>>(d_gz, n, d_cand, d_members, d_moff, d_chain, d_out);
    gu_crc_kernel<<<n_members, kCrcThreads, 0, st>>>(d_out, d_members, d_moff, d_res, d_bad);
    return cudaGetLastError();
}

cudaError_t cg_launch_gunzip_flags(const uint8_t *d_buf, long long n, const uint32_t *d_nl, long long n_nl, int fasta,
                                   int32_t *d_flag, cudaStream_t st)
{
    if (n_nl <= 0) return cudaSuccess;
    gu_flag_kernel<<<(unsigned)((n_nl + 255) / 256), 256, 0, st>>>(d_buf, n, d_nl, n_nl, fasta, d_flag);
    return cudaGetLastError();
}

cudaError_t cg_launch_gunzip_select(const uint32_t *d_nl, long long n_nl, const int32_t *d_flag, const int64_t *d_offs,
                                    long long s, long long *d_cut, cudaStream_t st)
{
    if (n_nl <= 0) return cudaSuccess;
    gu_select_kernel<<<(unsigned)((n_nl + 255) / 256), 256, 0, st>>>(d_nl, n_nl, d_flag, d_offs, s, d_cut);
    return cudaGetLastError();
}
