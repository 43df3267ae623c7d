// cg_gzip_core.cuh -- every decision that fixes the bytes of a gzip member written by cg_gzip.cu, host + device.
//
// A member holds at most GZ_MEMBER plain bytes: the fixed 10-byte header (no name, mtime 0, OS unknown), one final
// deflate block (dynamic Huffman, or stored when that is not larger), CRC-32 and ISIZE.  The encoder is LZ77 + per-member
// Huffman codes:
//   candidates  for position p, the latest earlier position with the same hash of the 4 bytes at p, where "earlier" means
//               in an earlier round of GZ_ROUND positions, or in the same group of 32 positions of p's round (the device
//               builds the table one round at a time, one position per thread, a warp per group);
//   parse       greedy, independently per sub-block of GZ_SUB bytes (one thread each on the device), matches clipped at the
//               sub-block's end, taken when at least GZ_MIN_MATCH long and at most GZ_MAX_DIST back;
//   codes       Huffman lengths (Moffat-Katajainen), limited to 15 / 7 bits by moving codes up (Kraft sum kept at 1),
//               ties broken by symbol number, canonical codes;
//   block type  stored when the dynamic block does not save a byte.
// The CUDA kernel runs these one block per member; tests/hostsim compiles them for the host so that a sequential build
// produces the same members byte for byte (test infrastructure, not a fallback).
#pragma once
#include "cg_types.h"

#define GZ_MEMBER 65280       // plain bytes per member (0xff00, BGZF's limit)
#define GZ_OVERHEAD 23        // header 10 + stored block head 5 + trailer 8: a member is at most n + 23 bytes
#define GZ_SLOT 65304         // scratch stride of one member on the device (>= GZ_MEMBER + GZ_OVERHEAD, 8-aligned)
#define GZ_SUB 256            // parse / CRC sub-block
#define GZ_NSUB (GZ_MEMBER / GZ_SUB)   // 255 sub-blocks per full member
#define GZ_ROUND 256          // positions per round of the candidate table
#define GZ_HASH_BITS 12
#define GZ_NONE 0xFFFFu       // no candidate
#define GZ_MIN_MATCH 4
#define GZ_MAX_MATCH 258
#define GZ_MAX_DIST 32768
#define GZ_TOK_MATCH 0x8000u  // token slot: a literal byte (< 256), or GZ_TOK_MATCH | (length - 3) then distance - 1

CG_HD void gz_or(uint32_t *w, uint32_t i, uint32_t v)
{
    if (!v) return;
#if defined(__CUDA_ARCH__)
    atomicOr(w + i, v);
#else
    w[i] |= v;
#endif
}

CG_HD void gz_inc(uint32_t *c)
{
#if defined(__CUDA_ARCH__)
    atomicAdd(c, 1u);
#else
    ++*c;
#endif
}

CG_HD int gz_ilog2(uint32_t v)   // v != 0
{
#if defined(__CUDA_ARCH__)
    return 31 - __clz(v);
#else
    return 31 - __builtin_clz(v);
#endif
}

CG_HD uint32_t gz_hash(const uint8_t *p)
{
    const uint32_t v = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
    return (v * 2654435761u) >> (32 - GZ_HASH_BITS);
}

// the candidate of a position: the latest earlier position of its group with the same hash (group_prev >= 0), else the
// latest one of the earlier rounds (bucket, -1 = none)
CG_HD uint16_t gz_pick(int group_prev, int bucket)
{
    const int c = group_prev >= 0 ? group_prev : bucket;
    return c < 0 ? (uint16_t)GZ_NONE : (uint16_t)c;
}

// Greedy parse of sub-block s of the member d[0, n).  tok[p] holds the candidate of position p on entry; the sub-block's
// tokens overwrite its own slots from its start (a token never passes the position it was read at).  Returns the number
// of token slots.
CG_HD int gz_parse_sub(const uint8_t *d, int n, uint16_t *tok, int s)
{
    const int start = s * GZ_SUB, end = start + GZ_SUB < n ? start + GZ_SUB : n;
    int k = start, p = start;
    while (p < end) {
        const uint32_t c = tok[p];
        int len = 0;
        if (c != GZ_NONE && p - (int)c <= GZ_MAX_DIST) {
            const int lim = end - p < GZ_MAX_MATCH ? end - p : GZ_MAX_MATCH;
            while (len < lim && d[c + len] == d[p + len]) ++len;
        }
        if (len >= GZ_MIN_MATCH) {
            tok[k++] = (uint16_t)(GZ_TOK_MATCH | (len - 3));
            tok[k++] = (uint16_t)(p - c - 1);
            p += len;
        } else {
            tok[k++] = d[p++];
        }
    }
    return k - start;
}

// length 3..258 -> lit/len symbol, extra bits, extra value
CG_HD void gz_len_sym(int len, int &sym, int &nx, int &x)
{
    const int l = len - 3;
    if (len == 258) { sym = 285; nx = 0; x = 0; }
    else if (l < 8) { sym = 257 + l; nx = 0; x = 0; }
    else {
        const int e = gz_ilog2((uint32_t)l) - 2;
        sym = 257 + 4 * (e + 1) + ((l >> e) & 3); nx = e; x = l & ((1 << e) - 1);
    }
}

// distance - 1 (0..32767) -> distance symbol, extra bits, extra value
CG_HD void gz_dist_sym(int dd, int &sym, int &nx, int &x)
{
    if (dd < 4) { sym = dd; nx = 0; x = 0; }
    else {
        const int e = gz_ilog2((uint32_t)dd) - 1;
        sym = 2 * (e + 1) + ((dd >> e) & 1); nx = e; x = dd & ((1 << e) - 1);
    }
}

// symbol counts of a sub-block's tokens
CG_HD void gz_tally_sub(const uint16_t *tok, int start, int ntok, uint32_t *ll_freq, uint32_t *d_freq)
{
    for (int k = start; k < start + ntok;) {
        const uint32_t t = tok[k];
        if (t & GZ_TOK_MATCH) {
            int sym, nx, x;
            gz_len_sym((int)(t & 0xFF) + 3, sym, nx, x);
            gz_inc(ll_freq + sym);
            gz_dist_sym(tok[k + 1], sym, nx, x);
            gz_inc(d_freq + sym);
            k += 2;
        } else {
            gz_inc(ll_freq + t);
            k += 1;
        }
    }
}

// Moffat & Katajainen's in-place minimum-redundancy code: A[0..n) ascending weights, n >= 2; on return A[i] is the code
// length of the i-th lightest symbol.
CG_HD void gz_moffat(uint32_t *A, int n)
{
    int root = 0, leaf = 2, next;
    A[0] += A[1];
    for (next = 1; next < n - 1; ++next) {
        if (leaf >= n || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = (uint32_t)next; }
        else A[next] = A[leaf++];
        if (leaf >= n || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = (uint32_t)next; }
        else A[next] += A[leaf++];
    }
    A[n - 2] = 0;
    for (next = n - 3; next >= 0; --next) A[next] = A[A[next]] + 1;
    int avbl = 1, used = 0, dpth = 0;
    root = n - 2; next = n - 1;
    while (avbl > 0) {
        while (root >= 0 && (int)A[root] == dpth) { ++used; --root; }
        while (avbl > used) { A[next--] = (uint32_t)dpth; --avbl; }
        avbl = 2 * used; ++dpth; used = 0;
    }
}

// Code lengths <= maxbits for freq[0, n) (n <= 288).  key / a: scratch of n entries, work: of 16.  A single used symbol gets a
// partner of length 1 (symbol 1, or 0 if it is symbol 1); no used symbol gives symbols 0 and 1 length 1, as zlib does
// for the distance code of a block without matches.
CG_HD void gz_lengths(const uint32_t *freq, int n, int maxbits, uint8_t *len, uint32_t *key, uint32_t *a, int *work)
{
    int m = 0;
    for (int s = 0; s < n; ++s) {
        len[s] = 0;
        if (!freq[s]) continue;
        const uint32_t kv = (freq[s] << 9) | (uint32_t)s;     // order: weight, then symbol number
        int j = m++;
        while (j > 0 && key[j - 1] > kv) { key[j] = key[j - 1]; --j; }
        key[j] = kv;
    }
    if (m < 2) {
        const int s = m ? (int)(key[0] & 511) : 0;
        len[s] = 1;
        len[s == 1 ? 0 : 1] = 1;
        return;
    }
    for (int i = 0; i < m; ++i) a[i] = key[i] >> 9;
    gz_moffat(a, m);
    int *num = work;
    for (int b = 0; b < 16; ++b) num[b] = 0;
    for (int i = 0; i < m; ++i) num[a[i] < (uint32_t)maxbits ? a[i] : maxbits] += 1;
    uint32_t total = 0;
    for (int b = maxbits; b >= 1; --b) total += (uint32_t)num[b] << (maxbits - b);
    while (total != (1u << maxbits)) {      // over-subscribed after the clamp: move one code down, split one above
        num[maxbits] -= 1;
        for (int b = maxbits - 1; b > 0; --b)
            if (num[b]) { num[b] -= 1; num[b + 1] += 2; break; }
        total -= 1;
    }
    int j = 0;
    for (int b = maxbits; b >= 1; --b)
        for (int k = 0; k < num[b]; ++k) len[key[j++] & 511] = (uint8_t)b;
}

// canonical codes, bit-reversed for deflate's LSB-first bit order; work: scratch of 32
CG_HD void gz_codes(const uint8_t *len, int n, uint16_t *code, int *work)
{
    int *cnt = work, *next = work + 16;
    for (int b = 0; b < 16; ++b) cnt[b] = 0;
    for (int s = 0; s < n; ++s) cnt[len[s]] += 1;
    cnt[0] = 0;
    int c = 0;
    next[0] = 0;
    for (int b = 1; b < 16; ++b) { c = (c + cnt[b - 1]) << 1; next[b] = c; }
    for (int s = 0; s < n; ++s) {
        const int l = len[s];
        if (!l) { code[s] = 0; continue; }
        const uint32_t v = (uint32_t)next[l]++;
        uint32_t r = 0;
        for (int i = 0; i < l; ++i) r |= ((v >> i) & 1u) << (l - 1 - i);
        code[s] = (uint16_t)r;
    }
}

// the order in which the code-length code's lengths are sent: 16 17 18 0 8 7 9 6 10 5 11 4 12 3 13 2 14 1 15
CG_HD int gz_cl_order(int i)
{
    return i < 3 ? 16 + i : i == 3 ? 0 : ((i - 4) & 1) ? 7 - ((i - 4) >> 1) : 8 + ((i - 4) >> 1);
}

struct GzTrees {
    uint32_t ll_freq[288], d_freq[32];
    uint8_t ll_len[288], d_len[32], cl_len[20];
    uint16_t ll_code[288], d_code[32], cl_code[20];
    uint16_t rle[320];         // code-length symbol | extra value << 5
    int n_rle, hlit, hdist, hclen;
    uint32_t header_bits;      // block header up to the first token
};

CG_HD int gz_code_len_at(const GzTrees &T, int i) { return i < T.hlit ? T.ll_len[i] : T.d_len[i - T.hlit]; }

// With ll_len / d_len set: HLIT, HDIST, the run-length coded lengths, the code-length code, HCLEN, every canonical code
// and the header's size in bits.  key / a: scratch of 20 entries, work: of 64.
CG_HD void gz_tree_header(GzTrees &T, uint32_t *key, uint32_t *a, int *work)
{
    int hlit = 286, hdist = 30;
    while (hlit > 257 && !T.ll_len[hlit - 1]) --hlit;
    while (hdist > 1 && !T.d_len[hdist - 1]) --hdist;
    T.hlit = hlit; T.hdist = hdist;
    uint32_t *clf = reinterpret_cast<uint32_t *>(work + 32);
    for (int s = 0; s < 19; ++s) clf[s] = 0;
    const int total = hlit + hdist;
    int nr = 0;
    for (int i = 0; i < total;) {
        const int v = gz_code_len_at(T, i);
        int r = 1;
        while (i + r < total && gz_code_len_at(T, i + r) == v) ++r;
        i += r;
        if (v == 0) {
            while (r >= 11) { const int k = r < 138 ? r : 138; T.rle[nr++] = (uint16_t)(18 | ((k - 11) << 5)); clf[18] += 1; r -= k; }
            if (r >= 3) { T.rle[nr++] = (uint16_t)(17 | ((r - 3) << 5)); clf[17] += 1; r = 0; }
            for (; r > 0; --r) { T.rle[nr++] = 0; clf[0] += 1; }
        } else {
            T.rle[nr++] = (uint16_t)v; clf[v] += 1; r -= 1;
            while (r >= 3) { const int k = r < 6 ? r : 6; T.rle[nr++] = (uint16_t)(16 | ((k - 3) << 5)); clf[16] += 1; r -= k; }
            for (; r > 0; --r) { T.rle[nr++] = (uint16_t)v; clf[v] += 1; }
        }
    }
    T.n_rle = nr;
    gz_lengths(clf, 19, 7, T.cl_len, key, a, work);
    int hclen = 19;
    while (hclen > 4 && !T.cl_len[gz_cl_order(hclen - 1)]) --hclen;
    T.hclen = hclen;
    gz_codes(T.ll_len, 286, T.ll_code, work);
    gz_codes(T.d_len, 30, T.d_code, work);
    gz_codes(T.cl_len, 19, T.cl_code, work);
    uint32_t bits = 3 + 5 + 5 + 4 + 3 * (uint32_t)hclen;
    for (int i = 0; i < nr; ++i) {
        const int s = T.rle[i] & 31;
        bits += T.cl_len[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
    }
    T.header_bits = bits;
}

// bits of a sub-block's tokens under the member's codes
CG_HD uint32_t gz_sub_bits(const GzTrees &T, const uint16_t *tok, int start, int ntok)
{
    uint32_t bits = 0;
    for (int k = start; k < start + ntok;) {
        const uint32_t t = tok[k];
        if (t & GZ_TOK_MATCH) {
            int sym, nx, x;
            gz_len_sym((int)(t & 0xFF) + 3, sym, nx, x);
            bits += T.ll_len[sym] + nx;
            gz_dist_sym(tok[k + 1], sym, nx, x);
            bits += T.d_len[sym] + nx;
            k += 2;
        } else {
            bits += T.ll_len[t];
            k += 1;
        }
    }
    return bits;
}

// ORs nb <= 32 bits of v into the zeroed word array w at bit pos (w has a spare word behind the last one written)
CG_HD void gz_put(uint32_t *w, uint32_t &pos, uint32_t v, int nb)
{
    if (!nb) return;
    const uint64_t x = (uint64_t)v << (pos & 31);
    gz_or(w, pos >> 5, (uint32_t)x);
    gz_or(w, (pos >> 5) + 1, (uint32_t)(x >> 32));
    pos += (uint32_t)nb;
}

CG_HD void gz_write_header(const GzTrees &T, uint32_t *w)
{
    uint32_t pos = 0;
    gz_put(w, pos, 1u | (2u << 1), 3);               // BFINAL = 1, BTYPE = 2
    gz_put(w, pos, (uint32_t)(T.hlit - 257), 5);
    gz_put(w, pos, (uint32_t)(T.hdist - 1), 5);
    gz_put(w, pos, (uint32_t)(T.hclen - 4), 4);
    for (int i = 0; i < T.hclen; ++i) gz_put(w, pos, T.cl_len[gz_cl_order(i)], 3);
    for (int i = 0; i < T.n_rle; ++i) {
        const int s = T.rle[i] & 31;
        gz_put(w, pos, T.cl_code[s], T.cl_len[s]);
        gz_put(w, pos, T.rle[i] >> 5, s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
    }
}

CG_HD void gz_write_sub(const GzTrees &T, const uint16_t *tok, int start, int ntok, uint32_t *w, uint32_t pos)
{
    for (int k = start; k < start + ntok;) {
        const uint32_t t = tok[k];
        if (t & GZ_TOK_MATCH) {
            int sym, nx, x;
            gz_len_sym((int)(t & 0xFF) + 3, sym, nx, x);
            gz_put(w, pos, T.ll_code[sym], T.ll_len[sym]);
            gz_put(w, pos, (uint32_t)x, nx);
            gz_dist_sym(tok[k + 1], sym, nx, x);
            gz_put(w, pos, T.d_code[sym], T.d_len[sym]);
            gz_put(w, pos, (uint32_t)x, nx);
            k += 2;
        } else {
            gz_put(w, pos, T.ll_code[t], T.ll_len[t]);
            k += 1;
        }
    }
}

CG_HD void gz_write_eob(const GzTrees &T, uint32_t *w, uint32_t pos) { gz_put(w, pos, T.ll_code[256], T.ll_len[256]); }

// stored when the dynamic block (bits long) saves no byte over the stored one (n + 5 bytes)
CG_HD bool gz_use_stored(uint32_t bits, int n) { return (bits + 7) / 8 >= (uint32_t)n + 5; }

CG_HD void gz_member_header(uint8_t *o)
{
    o[0] = 0x1f; o[1] = 0x8b; o[2] = 8;
    for (int i = 3; i < 9; ++i) o[i] = 0;
    o[9] = 0xff;
}

CG_HD void gz_stored_head(uint8_t *o, int n)
{
    o[0] = 1;                                         // BFINAL = 1, BTYPE = 0
    o[1] = (uint8_t)n; o[2] = (uint8_t)(n >> 8);
    o[3] = (uint8_t)~n; o[4] = (uint8_t)(~n >> 8);
}

CG_HD void gz_member_trailer(uint8_t *o, uint32_t crc, uint32_t n)
{
    for (int i = 0; i < 4; ++i) { o[i] = (uint8_t)(crc >> (8 * i)); o[4 + i] = (uint8_t)(n >> (8 * i)); }
}

// CRC-32 (reflected, polynomial 0xEDB88320) without pre- and post-conditioning: crc32(M) = ~gz_crc_raw(~0, M)
CG_HD uint32_t gz_crc_entry(uint32_t i)
{
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    return c;
}

CG_HD uint32_t gz_crc_raw(uint32_t c, const uint8_t *p, int n, const uint32_t *tab)
{
    for (int i = 0; i < n; ++i) c = tab[(c ^ p[i]) & 255] ^ (c >> 8);
    return c;
}

// c advanced over n zero bytes; with the columns of 1 << j this gives the GF(2) matrix that shifts a CRC by n bytes
CG_HD uint32_t gz_crc_zeros(uint32_t c, int n, const uint32_t *tab)
{
    for (int i = 0; i < n; ++i) c = tab[c & 255] ^ (c >> 8);
    return c;
}

CG_HD uint32_t gz_gf2_times(const uint32_t *mat, uint32_t v)
{
    uint32_t s = 0;
    for (int j = 0; v; ++j, v >>= 1)
        if (v & 1) s ^= mat[j];
    return s;
}
