// cg_gunzip_core.cuh -- every decision of the gzip input path (cg_gunzip.cu), host + device: the gzip member parser and
// inflater, the walk over the member chain, and where a buffer of plain bytes is cut into whole records.
//
// Accepts and rejects what Python's gzip module (3.12) and zlib do:
//   header   magic 1f 8b, method 8, reserved FLG bits ignored, FEXTRA / FNAME / FCOMMENT skipped, FHCRC skipped unchecked;
//   deflate  block type 3, stored LEN != ~NLEN, HLIT > 286 or HDIST > 30, an over-subscribed code, an incomplete code
//            (the code-length code always; the literal/length and distance codes unless they hold one code of length
//            1), a repeat of the previous length at the first length, repeats past HLIT + HDIST, no end-of-block code,
//            symbols 286 / 287, distance symbols 30 / 31 and a distance behind the member's start are invalid;
//   trailer  ISIZE must be the plain length mod 2^32 (the CRC-32 is checked where the plain bytes are, cg_gunzip.cu);
//   chain    zero bytes after a member are skipped; any other byte that does not start a member is invalid.
// A member that runs past the bytes given "needs more input".  The decoder is puff's canonical decode (count and symbol
// per code length), with the tables in the caller's memory (shared memory on the device).
#pragma once
#include "cg_types.h"

#define GU_OK 0
#define GU_INVALID 1
#define GU_MORE 2          // the member runs past the bytes given
#define GU_UNSUPPORTED 3   // chain: not even one member fits under the plain-size limit

struct GuTables {
    uint16_t lcnt[16], lsym[288], dcnt[16], dsym[32], offs[16];
    uint8_t lens[320];
};

struct GuMember {
    int32_t status;
    int32_t size;          // GU_OK: bytes of the member, header and trailer included
    long long plain;       // GU_OK: plain bytes
    uint32_t crc;          // GU_OK: the trailer's CRC-32
};

struct GuBits {
    const uint8_t *in;
    long long pos, avail;
    uint64_t buf;
    int cnt;
    bool more;             // a read ran past avail
};

CG_HD bool gu_need(GuBits &b, int n)
{
    while (b.cnt <= 56 && b.pos < b.avail) { b.buf |= (uint64_t)b.in[b.pos++] << b.cnt; b.cnt += 8; }
    if (b.cnt >= n) return true;
    b.more = true;
    return false;
}

CG_HD uint32_t gu_bits(GuBits &b, int n)
{
    if (!n) return 0;
    if (!gu_need(b, n)) return 0;
    const uint32_t v = (uint32_t)(b.buf & ((1ull << n) - 1));
    b.buf >>= n;
    b.cnt -= n;
    return v;
}

// counts and symbols of the canonical code of len[0, n); returns 0 for a complete code, > 0 for an incomplete one (the
// codes left unused at 15 bits), < 0 for an over-subscribed one
CG_HD int gu_build(uint16_t *cnt, uint16_t *sym, uint16_t *offs, const uint8_t *len, int n)
{
    for (int l = 0; l < 16; ++l) cnt[l] = 0;
    for (int s = 0; s < n; ++s) cnt[len[s]] += 1;
    int left = 1;
    for (int l = 1; l < 16; ++l) {
        left <<= 1;
        left -= cnt[l];
        if (left < 0) return left;
    }
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = (uint16_t)(offs[l] + cnt[l]);
    for (int s = 0; s < n; ++s)
        if (len[s]) sym[offs[len[s]]++] = (uint16_t)s;
    return left;
}

// zlib's rule for the literal/length and distance codes: complete, or no code at all, or a single code of length 1
CG_HD bool gu_code_ok(int left, const uint16_t *cnt)
{
    if (left == 0) return true;
    if (left < 0) return false;
    int max = 0;
    for (int l = 1; l < 16; ++l)
        if (cnt[l]) max = l;
    return max <= 1;
}

// the next symbol, -1 when the input ran out, -2 for a bit pattern without a code
CG_HD int gu_decode(GuBits &b, const uint16_t *cnt, const uint16_t *sym)
{
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; ++l) {
        if (!gu_need(b, 1)) return -1;
        code |= (int)(b.buf & 1);
        b.buf >>= 1;
        b.cnt -= 1;
        const int count = cnt[l];
        if (code - count < first) return sym[index + (code - first)];
        index += count;
        first += count;
        first <<= 1;
        code <<= 1;
    }
    return -2;
}

// The member at in[0, avail).  out != nullptr: its plain bytes are written there (the caller knows how many); else it
// is only parsed -- the parse never reads the plain bytes.
CG_HD GuMember gu_member(const uint8_t *in, long long avail, uint8_t *out, GuTables &T)
{
    GuMember m = {GU_INVALID, 0, 0, 0};
    if (avail < 3 || in[0] != 0x1f || in[1] != 0x8b || in[2] != 8) return m;     // the chain sees to shorter ones
    m.status = GU_MORE;
    if (avail < 10) return m;
    const int flg = in[3];
    long long p = 10;
    m.status = GU_MORE;
    if (flg & 4) {
        if (p + 2 > avail) return m;
        p += 2 + (in[p] | (in[p + 1] << 8));
        if (p > avail) return m;
    }
    for (int f = 8; f <= 16; f <<= 1) {
        if (!(flg & f)) continue;
        while (p < avail && in[p]) ++p;
        if (p >= avail) return m;
        ++p;
    }
    if (flg & 2) {
        p += 2;
        if (p > avail) return m;
    }
    GuBits b = {in, p, avail, 0, 0, false};
    long long o = 0;
    m.status = GU_INVALID;
    int last = 0;
    while (!last) {
        last = (int)gu_bits(b, 1);
        const int type = (int)gu_bits(b, 2);
        if (b.more) { m.status = GU_MORE; return m; }
        if (type == 3) return m;
        if (type == 0) {
            b.buf >>= b.cnt & 7;
            b.cnt -= b.cnt & 7;
            const uint32_t len = gu_bits(b, 16), nlen = gu_bits(b, 16);
            if (b.more) { m.status = GU_MORE; return m; }
            if (len != (~nlen & 0xffffu)) return m;
            b.pos -= b.cnt / 8;                 // the bytes read ahead go back
            b.buf = 0;
            b.cnt = 0;
            if (b.pos + len > avail) { m.status = GU_MORE; return m; }
            if (out)
                for (uint32_t i = 0; i < len; ++i) out[o + i] = in[b.pos + i];
            o += len;
            b.pos += len;
            continue;
        }
        int nlen = 288, ndist = 32;
        if (type == 1) {
            for (int s = 0; s < 288; ++s) T.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
            for (int s = 0; s < 32; ++s) T.lens[288 + s] = 5;
        } else {
            nlen = (int)gu_bits(b, 5) + 257;
            ndist = (int)gu_bits(b, 5) + 1;
            const int ncode = (int)gu_bits(b, 4) + 4;
            if (b.more) { m.status = GU_MORE; return m; }
            if (nlen > 286 || ndist > 30) return m;
            for (int i = 0; i < 19; ++i) {
                const int s = i < 3 ? 16 + i : i == 3 ? 0 : ((i - 4) & 1) ? 7 - ((i - 4) >> 1) : 8 + ((i - 4) >> 1);
                T.lens[s] = (uint8_t)(i < ncode ? gu_bits(b, 3) : 0);
            }
            if (b.more) { m.status = GU_MORE; return m; }
            if (gu_build(T.lcnt, T.lsym, T.offs, T.lens, 19) != 0) return m;
            for (int i = 0; i < nlen + ndist;) {
                const int s = gu_decode(b, T.lcnt, T.lsym);
                if (s == -1) { m.status = GU_MORE; return m; }
                if (s < 0) return m;
                if (s < 16) { T.lens[i++] = (uint8_t)s; continue; }
                int v = 0, r;
                if (s == 16) {
                    if (i == 0) return m;
                    v = T.lens[i - 1];
                    r = 3 + (int)gu_bits(b, 2);
                } else {
                    r = s == 17 ? 3 + (int)gu_bits(b, 3) : 11 + (int)gu_bits(b, 7);
                }
                if (b.more) { m.status = GU_MORE; return m; }
                if (i + r > nlen + ndist) return m;
                while (r--) T.lens[i++] = (uint8_t)v;
            }
            if (T.lens[256] == 0) return m;
            // the distance lengths move to T.lens + 288, where the fixed code has them (backwards: the ranges overlap)
            for (int s = ndist - 1; s >= 0; --s) T.lens[288 + s] = T.lens[nlen + s];
        }
        if (!gu_code_ok(gu_build(T.lcnt, T.lsym, T.offs, T.lens, nlen), T.lcnt)) return m;
        if (!gu_code_ok(gu_build(T.dcnt, T.dsym, T.offs, T.lens + 288, ndist), T.dcnt)) return m;
        for (;;) {
            const int s = gu_decode(b, T.lcnt, T.lsym);
            if (s == -1) { m.status = GU_MORE; return m; }
            if (s < 0) return m;
            if (s < 256) {
                if (out) out[o] = (uint8_t)s;
                ++o;
                continue;
            }
            if (s == 256) break;
            const int l = s - 257;
            if (l >= 29) return m;
            const int lx = l < 8 || l == 28 ? 0 : (l - 4) >> 2;
            const int len = (l == 28 ? 258 : l < 8 ? 3 + l : ((4 + (l & 3)) << lx) + 3) + (int)gu_bits(b, lx);
            const int d = gu_decode(b, T.dcnt, T.dsym);
            if (d == -1 || b.more) { m.status = GU_MORE; return m; }
            if (d < 0 || d >= 30) return m;
            const int dx = d < 4 ? 0 : (d - 2) >> 1;
            const long long dist = (d < 4 ? d + 1 : ((2 + (d & 1)) << dx) + 1) + (long long)gu_bits(b, dx);
            if (b.more) { m.status = GU_MORE; return m; }
            if (dist > o) return m;
            if (out)
                for (int i = 0; i < len; ++i) out[o + i] = out[o + i - dist];
            o += len;
        }
    }
    const long long t = b.pos - b.cnt / 8;      // the trailer starts at the next byte
    if (t + 8 > avail) { m.status = GU_MORE; return m; }
    const uint32_t crc = in[t] | (in[t + 1] << 8) | (in[t + 2] << 16) | ((uint32_t)in[t + 3] << 24);
    const uint32_t isize = in[t + 4] | (in[t + 5] << 8) | (in[t + 6] << 16) | ((uint32_t)in[t + 7] << 24);
    if (isize != (uint32_t)o) return m;
    m.status = GU_OK;
    m.size = (int32_t)(t + 8);
    m.plain = o;
    m.crc = crc;
    return m;
}

// ---- the member chain -------------------------------------------------------------------------------------------------
// Walks gz[0, n) from member end to member end (zero bytes skipped after a member, and at 0 when the stream already
// had a member).  cand: the sorted positions of every 1f 8b 08 with their parse results.  Stops at the end, at a member
// that needs more input (an error when final), at the first invalid position, or in front of a member that would bring
// the plain bytes (plus `base`, the carry) to `limit`.  members / moff receive the chain's candidates and their plain
// offsets behind the carry.
struct GuChain {
    int32_t status;        // GU_OK, GU_INVALID, GU_UNSUPPORTED
    int32_t n_members;
    long long consumed;    // bytes of whole members and the zeros behind them
    long long plain;       // their plain bytes
    long long err_at;      // GU_INVALID / GU_UNSUPPORTED: offset of the bad (or too large) member
};

CG_HD GuChain gu_chain(const uint8_t *gz, long long n, const int32_t *cand, const GuMember *res, int n_cand, bool after_member,
                       bool final, long long base, long long limit, int32_t *members, long long *moff)
{
    GuChain c = {GU_OK, 0, 0, 0, 0};
    long long p = 0;
    for (;;) {
        if (after_member)
            while (p < n && gz[p] == 0) ++p;
        c.consumed = p;
        if (p == n) return c;
        int lo = 0, hi = n_cand;                // the candidate at p, if any
        while (lo < hi) {
            const int mid = (lo + hi) / 2;
            if (cand[mid] < p) lo = mid + 1; else hi = mid;
        }
        GuMember m = {GU_INVALID, 0, 0, 0};
        if (lo < n_cand && cand[lo] == p) m = res[lo];
        else if (n - p < 3 && gz[p] == 0x1f && (n - p == 1 || gz[p + 1] == 0x8b)) m.status = GU_MORE;   // a header's start
        if (m.status == GU_MORE && !final) return c;
        if (m.status != GU_OK) { c.status = GU_INVALID; c.err_at = p; return c; }
        if (base + c.plain + m.plain >= limit) {
            if (!c.n_members) { c.status = GU_UNSUPPORTED; c.err_at = p; }
            return c;
        }
        members[c.n_members] = lo;
        moff[c.n_members] = base + c.plain;
        c.n_members += 1;
        c.plain += m.plain;
        p += m.size;
        after_member = true;
    }
}

// ---- record cuts ------------------------------------------------------------------------------------------------------
// A buffer of plain bytes is cut behind one of its newlines.  Flagged newlines: every newline in FASTQ, a newline
// followed by '>' in FASTA (F of them; b0: the buffer starts with '>').  gu_select_* give the index of the flagged
// newline the cut lies behind, or -1 for no cut; they restate pipeline.py's readers.
CG_HD bool gu_flag(const uint8_t *buf, long long n, long long i, int fasta)
{
    return buf[i] == '\n' && (!fasta || (i + 1 < n && buf[i + 1] == '>'));
}

// whole records (FASTQ: F / 4; FASTA: the headers in front of the last one)
CG_HD long long gu_records(int fasta, long long F, int b0) { return fasta ? (F ? F + b0 - 1 : 0) : F / 4; }

// the cut in front of record r (r >= 1, or FASTA without a header at 0)
CG_HD long long gu_select_records(int fasta, long long r, int b0) { return fasta ? (b0 ? r - 1 : r) : 4 * r - 1; }

// _fastq_head / _fasta_head (pairs = 0), and whole pairs of an interleaved buffer (pairs = 1)
CG_HD long long gu_select_single(int fasta, long long F, int b0, int pairs)
{
    const long long r = gu_records(fasta, F, b0);
    if (!pairs) {
        if (fasta) return F ? F - 1 : -1;
        return r ? 4 * r - 1 : -1;
    }
    const long long even = r - r % 2;
    return even ? gu_select_records(fasta, even, b0) : -1;
}
