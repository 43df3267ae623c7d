// tests/hostsim/hostsim_bam.cpp -- TEST-ONLY host build of the BAM input path's decisions
// (cutadapt_b200/csrc/cg_bam_core.cuh), linked into libhostsim.so so that tests/test_bam_host.py can check them against
// the Python decoder of tests/bam_oracle.py without a GPU.  The steps run in the order of cg_bam.cu: the speculative walk
// of every tile, the resolve along the true chain, the starts between each tile's entry and the chain's end, then the
// refusals and the FASTQ text per record.  Nothing in cutadapt_b200/ loads this library.
#include <string.h>

#include <vector>

#include "../../cutadapt_b200/csrc/cg_bam_core.cuh"

extern "C" int64_t hs_bam_tile() { return BAM_TILE; }

// bam_header: status; *len the header's size, *why the reason of BAM_BAD
extern "C" int hs_bam_header(const uint8_t *b, int64_t n, int64_t *len, int *why)
{
    long long l = 0;
    *why = 0;
    const int s = bam_header(b, n, &l, why);
    *len = l;
    return s;
}

// The record starts of b[0, n) by the tile walk with tiles of `tile` bytes into starts (room for n / 36 + 1); their
// number.  *end / *end_st: where and why the chain stops; *rewalked: tiles walked again.
extern "C" int64_t hs_bam_starts(const uint8_t *b, int64_t n, int64_t tile, int64_t *starts, int64_t *end, int *end_st,
                                 int64_t *rewalked)
{
    const long long T = (n + tile - 1) / tile, W = (n + 31) / 32;
    std::vector<uint32_t> bm((size_t)W + 1, 0);
    std::vector<uint64_t> link((size_t)T + 1);
    std::vector<long long> entry((size_t)T + 1, -1);
    for (long long t = 0; t < T; ++t) {
        const long long lo = t * tile, hi = lo + tile < n ? lo + tile : n;
        long long start = t == 0 ? 0 : hi;
        for (long long p = lo; t != 0 && p < hi; ++p)
            if (bam_candidate(b, n, p)) { start = p; break; }
        link[t] = bam_spec_walk(b, n, hi, start, bm.data());
    }
    for (long long t = 0; t < T; ++t) link[t] = bam_link_resolve(link[t], n, bm.data());
    long long p = 0, rew = 0;
    int on = 1;
    for (;;) {
        if (p >= n) { *end = p; *end_st = BAM_OK; break; }
        const long long t = p / tile;
        entry[t] = p;
        const uint64_t w = bam_resolve_step(b, n, tile, p, on, link[t], bm.data(), &rew);
        if (bam_link_st(w) != BAM_OK) { *end = bam_link_pos(w); *end_st = bam_link_st(w); break; }
        p = bam_link_pos(w);
        on = bam_link_on(w);
    }
    *rewalked = rew;
    long long k = 0;
    for (long long w = 0; w < W; ++w) {
        uint32_t m = bam_word_starts(bm.data(), w, tile, entry.data(), *end);
        for (int i = 0; i < 32; ++i)
            if (m >> i & 1u) starts[k++] = w * 32 + i;
    }
    return k;
}

// The FASTQ text of the records at starts[0, n_rec) of b into out (room for the sum of bam_fastq_size); its size.
// *err: the first refusal, record << 3 | BAM_R_*, or -1.
extern "C" int64_t hs_bam_fastq(const uint8_t *b, const int64_t *starts, int64_t n_rec, uint8_t *out, int64_t *err)
{
    long long o = 0;
    *err = -1;
    for (long long i = 0; i < n_rec; ++i) {
        const int code = bam_refusal(b + starts[i]);
        if (code && *err < 0) *err = (i << 3) | code;
        bam_emit(b + starts[i], out + o);
        o += bam_fastq_size(b + starts[i]);
    }
    return o;
}
