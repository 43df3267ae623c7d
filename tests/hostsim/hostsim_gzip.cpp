// tests/hostsim/hostsim_gzip.cpp -- TEST-ONLY host build of the gzip member encoder (cutadapt_b200/csrc/cg_gzip_core.cuh),
// linked into libhostsim.so so that tests/test_gzip_host.py can check the members against zlib without a GPU and
// tests/test_gpu_gzip.py can check that the device writes the same bytes.  The steps run in the order and with the
// partitioning of gz_compress_kernel (cg_gzip.cu), one after the other.  Nothing in cutadapt_b200/ loads this library.
#include <string.h>

#include <vector>

#include "../../cutadapt_b200/csrc/cg_gzip_core.cuh"

// One member of d[0, n), 1 <= n <= GZ_MEMBER, into out (at least n + GZ_OVERHEAD bytes).  Returns its size.
static int gz_member_host(const uint8_t *d, int n, uint8_t *out)
{
    uint32_t tab[256];
    for (int i = 0; i < 256; ++i) tab[i] = gz_crc_entry((uint32_t)i);
    const uint32_t crc = ~gz_crc_raw(0xffffffffu, d, n, tab);

    // candidates, one round of GZ_ROUND positions at a time; the table sees a round only once it is complete
    std::vector<uint16_t> tok((size_t)n);
    std::vector<int> bucket(1 << GZ_HASH_BITS, -1);
    for (int r0 = 0; r0 < n; r0 += GZ_ROUND) {
        const int r1 = r0 + GZ_ROUND < n ? r0 + GZ_ROUND : n;
        for (int p = r0; p < r1; ++p) {
            int prev = -1;
            if (p + 4 <= n) {
                const uint32_t h = gz_hash(d + p);
                for (int q = p - 1; q >= p - (p & 31); --q)
                    if (gz_hash(d + q) == h) { prev = q; break; }
                tok[p] = gz_pick(prev, bucket[h]);
            } else {
                tok[p] = gz_pick(-1, -1);
            }
        }
        for (int p = r0; p < r1 && p + 4 <= n; ++p) bucket[gz_hash(d + p)] = p;
    }

    GzTrees T;
    memset(&T, 0, sizeof T);
    T.ll_freq[256] = 1;
    const int nsub = (n + GZ_SUB - 1) / GZ_SUB;
    std::vector<int> ntok(nsub);
    for (int s = 0; s < nsub; ++s) {
        ntok[s] = gz_parse_sub(d, n, tok.data(), s);
        gz_tally_sub(tok.data(), s * GZ_SUB, ntok[s], T.ll_freq, T.d_freq);
    }
    uint32_t key[288], a[288];
    int work[64];
    gz_lengths(T.ll_freq, 286, 15, T.ll_len, key, a, work);
    gz_lengths(T.d_freq, 30, 15, T.d_len, key, a, work);
    gz_tree_header(T, key, a, work);
    std::vector<uint32_t> off(nsub);
    uint32_t total = T.header_bits;
    for (int s = 0; s < nsub; ++s) {
        off[s] = total;
        total += gz_sub_bits(T, tok.data(), s * GZ_SUB, ntok[s]);
    }
    const uint32_t eob = total;
    total += T.ll_len[256];

    gz_member_header(out);
    int size;
    if (gz_use_stored(total, n)) {
        gz_stored_head(out + 10, n);
        memcpy(out + 15, d, (size_t)n);
        size = 15 + n;
    } else {
        std::vector<uint32_t> w(total / 32 + 2, 0);
        gz_write_header(T, w.data());
        for (int s = 0; s < nsub; ++s) gz_write_sub(T, tok.data(), s * GZ_SUB, ntok[s], w.data(), off[s]);
        gz_write_eob(T, w.data(), eob);
        const int bytes = (int)((total + 7) / 8);
        memcpy(out + 10, w.data(), (size_t)bytes);
        size = 10 + bytes;
    }
    gz_member_trailer(out + size, crc, (uint32_t)n);
    return size + 8;
}

// d[0, n) as members of GZ_MEMBER bytes (the last may be shorter; n == 0 gives nothing) into out (at least
// n + GZ_OVERHEAD per member).  Returns the bytes written.
extern "C" int64_t hs_gzip(const uint8_t *d, int64_t n, uint8_t *out)
{
    int64_t o = 0;
    for (int64_t i = 0; i < n; i += GZ_MEMBER) {
        const int len = (int)(n - i < GZ_MEMBER ? n - i : GZ_MEMBER);
        o += gz_member_host(d + i, len, out + o);
    }
    return o;
}

// the code lengths gz_lengths gives freq[0, n) under max_bits (tests of the length limit)
extern "C" void hs_gzip_lengths(const uint32_t *freq, int n, int max_bits, uint8_t *len)
{
    uint32_t key[288], a[288];
    int work[16];
    gz_lengths(freq, n, max_bits, len, key, a, work);
}
