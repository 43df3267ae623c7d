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
#define GU_LONG 4          // gu_member: the parse reached its compressed-byte budget; gu_chain: a member for the block path
#define GU_OVER 5          // gu_chunk: the chunk's symbols outgrew its room

#define GU_WIN 32768       // the deflate window

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

// The length of the gzip header at in[0, avail) (magic and method already checked), or 0 when it runs past avail
CG_HD long long gu_head(const uint8_t *in, long long avail)
{
    if (avail < 10) return 0;
    const int flg = in[3];
    long long p = 10;
    if (flg & 4) {
        if (p + 2 > avail) return 0;
        p += 2 + (in[p] | (in[p + 1] << 8));
        if (p > avail) return 0;
    }
    for (int f = 8; f <= 16; f <<= 1) {
        if (!(flg & f)) continue;
        while (p < avail && in[p]) ++p;
        if (p >= avail) return 0;
        ++p;
    }
    if (flg & 2) {
        p += 2;
        if (p > avail) return 0;
    }
    return p;
}

// The code tables of a fixed (type 1) or dynamic (type 2) block whose three header bits are read: GU_OK, GU_INVALID
// or GU_MORE.  Dynamic: the code-length code must be complete, the literal/length and distance codes pass gu_code_ok.
CG_HD int gu_tables(GuBits &b, int type, GuTables &T)
{
    int nlen = 288, ndist = 32;
    if (type == 1) {
        for (int s = 0; s < 288; ++s) T.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
        for (int s = 0; s < 32; ++s) T.lens[288 + s] = 5;
    } else {
        nlen = (int)gu_bits(b, 5) + 257;
        ndist = (int)gu_bits(b, 5) + 1;
        const int ncode = (int)gu_bits(b, 4) + 4;
        if (b.more) return GU_MORE;
        if (nlen > 286 || ndist > 30) return GU_INVALID;
        for (int i = 0; i < 19; ++i) {
            const int s = i < 3 ? 16 + i : i == 3 ? 0 : ((i - 4) & 1) ? 7 - ((i - 4) >> 1) : 8 + ((i - 4) >> 1);
            T.lens[s] = (uint8_t)(i < ncode ? gu_bits(b, 3) : 0);
        }
        if (b.more) return GU_MORE;
        if (gu_build(T.lcnt, T.lsym, T.offs, T.lens, 19) != 0) return GU_INVALID;
        for (int i = 0; i < nlen + ndist;) {
            const int s = gu_decode(b, T.lcnt, T.lsym);
            if (s == -1) return GU_MORE;
            if (s < 0) return GU_INVALID;
            if (s < 16) { T.lens[i++] = (uint8_t)s; continue; }
            int v = 0, r;
            if (s == 16) {
                if (i == 0) return GU_INVALID;
                v = T.lens[i - 1];
                r = 3 + (int)gu_bits(b, 2);
            } else {
                r = s == 17 ? 3 + (int)gu_bits(b, 3) : 11 + (int)gu_bits(b, 7);
            }
            if (b.more) return GU_MORE;
            if (i + r > nlen + ndist) return GU_INVALID;
            while (r--) T.lens[i++] = (uint8_t)v;
        }
        if (T.lens[256] == 0) return GU_INVALID;
        // the distance lengths move to T.lens + 288, where the fixed code has them (backwards: the ranges overlap)
        for (int s = ndist - 1; s >= 0; --s) T.lens[288 + s] = T.lens[nlen + s];
    }
    if (!gu_code_ok(gu_build(T.lcnt, T.lsym, T.offs, T.lens, nlen), T.lcnt)) return GU_INVALID;
    if (!gu_code_ok(gu_build(T.dcnt, T.dsym, T.offs, T.lens + 288, ndist), T.dcnt)) return GU_INVALID;
    return GU_OK;
}

// The member at in[0, avail).  out != nullptr: its plain bytes are written there (the caller knows how many); else it
// is only parsed -- the parse never reads the plain bytes.  budget > 0: a parse that reaches a block boundary at or
// past budget compressed bytes stops with GU_LONG.
CG_HD GuMember gu_member(const uint8_t *in, long long avail, uint8_t *out, GuTables &T, long long budget = 0)
{
    GuMember m = {GU_INVALID, 0, 0, 0};
    if (avail < 3 || in[0] != 0x1f || in[1] != 0x8b || in[2] != 8) return m;     // the chain sees to shorter ones
    m.status = GU_MORE;
    const long long p = gu_head(in, avail);
    if (!p) return m;
    GuBits b = {in, p, avail, 0, 0, false};
    long long o = 0;
    m.status = GU_INVALID;
    int last = 0;
    while (!last) {
        if (budget > 0 && b.pos - b.cnt / 8 >= budget) { m.status = GU_LONG; return m; }
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
        const int tb = gu_tables(b, type, T);
        if (tb != GU_OK) { m.status = tb; return m; }
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

// from: where the walk starts.  split (streams of CG_GZIN_SPLIT_MEMBERS): a member whose parse stopped at its budget
// (GU_LONG), or that runs past the bytes given with its whole header there, ends the walk with status GU_LONG and its
// offset in err_at -- it goes to the block path.
CG_HD GuChain gu_chain(const uint8_t *gz, long long n, const int32_t *cand, const GuMember *res, int n_cand, bool after_member,
                       bool final, long long base, long long limit, int32_t *members, long long *moff,
                       long long from = 0, bool split = false)
{
    GuChain c = {GU_OK, 0, 0, 0, 0};
    long long p = from;
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
        if (split && (m.status == GU_LONG || (m.status == GU_MORE && !final && lo < n_cand && cand[lo] == p &&
                                              gu_head(gz + p, n - p) > 0))) {
            c.status = GU_LONG;
            c.err_at = p;
            return c;
        }
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

// ---- one member, block-parallel (split streams) ------------------------------------------------------------------------
// The deflate bits of a long member are cut into chunks at a stride of S compressed bytes from its known start (chunk
// 0).  Chunk k >= 1 starts at the first bit at or after its nominal start that passes a full dynamic-block header check
// (gu_dyn_start), decodes to the first block boundary at or after the next nominal start, and writes 16-bit symbols: a
// byte (< 256), or 256 + w for position w of the unknown 32 KiB window in front of the chunk (the u16 scheme of pugz and
// rapidgzip).  gu_walk confirms chunks from chunk 0 (k counts when its start is chunk k - 1's end) and lists the chunks
// to decode again; the windows then pass from chunk to chunk (gu_win_byte) and every symbol becomes its byte (gu_sym).
// A decoder started at a false offset reads garbage, so every write is bounded by the chunk's room, every marker lies
// in [256, 256 + GU_WIN), and every loop ends when the bits run out.
struct GuChunk {
    long long start;       // bit offset of its first block in the submission's bytes; -1: the search found none
    long long end;         // bit offset behind its last whole block (where it stopped for GU_INVALID / GU_OVER)
    long long n;           // symbols up to end
    long long at;          // gu_walk: symbols of the confirmed chunks in front of it
    int32_t status;        // GU_OK, GU_MORE (the bytes ran out behind end), GU_INVALID, GU_OVER
    int32_t last;          // the block in front of end is the member's last (BFINAL)
};

// a dynamic block that is not the last starts at bit `bit` of in[0, avail)
CG_HD bool gu_dyn_start(const uint8_t *in, long long avail, long long bit, GuTables &T)
{
    GuBits b = {in, bit >> 3, avail, 0, 0, false};
    gu_bits(b, (int)(bit & 7));
    if (gu_bits(b, 3) != 4 || b.more) return false;       // BFINAL 0, BTYPE 10
    return gu_tables(b, 2, T) == GU_OK;
}

// Decode from bit `start` to the first block boundary at or after `stop` (or the member's last block) into out[0, room)
CG_HD GuChunk gu_chunk(const uint8_t *in, long long avail, long long start, long long stop, uint16_t *out, long long room,
                       GuTables &T)
{
    GuChunk c = {start, start, 0, 0, GU_OK, 0};
    if (start < 0) { c.status = GU_INVALID; return c; }
    GuBits b = {in, start >> 3, avail, 0, 0, false};
    gu_bits(b, (int)(start & 7));
    if (b.more) { c.status = GU_MORE; return c; }
    long long o = 0;
    while (!c.last) {
        c.end = b.pos * 8 - b.cnt;
        c.n = o;
        if (c.end >= stop) return c;
        const int last = (int)gu_bits(b, 1);
        const int type = (int)gu_bits(b, 2);
        if (b.more) { c.status = GU_MORE; return c; }
        if (type == 3) { c.status = GU_INVALID; return c; }
        if (type == 0) {
            b.buf >>= b.cnt & 7;
            b.cnt -= b.cnt & 7;
            const uint32_t len = gu_bits(b, 16), nlen = gu_bits(b, 16);
            if (b.more) { c.status = GU_MORE; return c; }
            if (len != (~nlen & 0xffffu)) { c.status = GU_INVALID; return c; }
            b.pos -= b.cnt / 8;
            b.buf = 0;
            b.cnt = 0;
            if (b.pos + len > avail) { c.status = GU_MORE; return c; }
            if (o + len > room) { c.status = GU_OVER; return c; }
            for (uint32_t i = 0; i < len; ++i) out[o + i] = in[b.pos + i];
            o += len;
            b.pos += len;
        } else {
            const int tb = gu_tables(b, type, T);
            if (tb != GU_OK) { c.status = tb; return c; }
            for (;;) {
                const int s = gu_decode(b, T.lcnt, T.lsym);
                if (s == -1) { c.status = GU_MORE; return c; }
                if (s < 0) { c.status = GU_INVALID; return c; }
                if (s < 256) {
                    if (o >= room) { c.status = GU_OVER; return c; }
                    out[o++] = (uint16_t)s;
                    continue;
                }
                if (s == 256) break;
                const int l = s - 257;
                if (l >= 29) { c.status = GU_INVALID; return c; }
                const int lx = l < 8 || l == 28 ? 0 : (l - 4) >> 2;
                const int len = (l == 28 ? 258 : l < 8 ? 3 + l : ((4 + (l & 3)) << lx) + 3) + (int)gu_bits(b, lx);
                const int d = gu_decode(b, T.dcnt, T.dsym);
                if (d == -1 || b.more) { c.status = GU_MORE; return c; }
                if (d < 0 || d >= 30) { c.status = GU_INVALID; return c; }
                const int dx = d < 4 ? 0 : (d - 2) >> 1;
                const long long dist = (d < 4 ? d + 1 : ((2 + (d & 1)) << dx) + 1) + (long long)gu_bits(b, dx);  // <= GU_WIN
                if (b.more) { c.status = GU_MORE; return c; }
                if (o + len > room) { c.status = GU_OVER; return c; }
                for (int i = 0; i < len; ++i) {
                    const long long q = o + i - dist;
                    out[o + i] = q >= 0 ? out[q] : (uint16_t)(256 + GU_WIN + q);
                }
                o += len;
            }
        }
        c.last = last;
    }
    c.end = b.pos * 8 - b.cnt;
    c.n = o;
    return c;
}

struct GuWalk {
    int32_t status;        // GU_OK: done; GU_MORE: redo lists n_redo chunks to decode again; GU_INVALID: confirmed chunk
                           // n_ok failed; GU_UNSUPPORTED: chunk 0 alone reaches the limit
    int32_t n_ok;          // confirmed chunks
    int32_t n_redo;
    int32_t respec;        // of them, those whose start was wrong
    int32_t last;          // the member's last block ends chunk n_ok - 1
    int32_t more;          // the bytes ran out in chunk n_ok - 1
    long long end;         // bit behind the last confirmed block
    long long plain;       // symbols of the confirmed chunks
};

// Walk the K chunks from chunk 0.  limit: the symbols this submission may still take.  Chunks to decode again go to
// redo with their new start in ch[].start: the first unconfirmed one from the confirmed end (or from its own start with
// more room when it overflowed), every later one whose start is not its decoded predecessor's end from that end.
CG_HD GuWalk gu_walk(GuChunk *ch, int K, long long limit, int32_t *redo)
{
    GuWalk w = {GU_OK, 0, 0, 0, 0, 0, ch[0].start, 0};
    int k = 0;
    for (; k < K; ++k) {
        GuChunk &c = ch[k];
        if ((k && c.start != w.end) || c.status == GU_OVER) break;
        if (c.status == GU_INVALID) { w.status = GU_INVALID; w.n_ok = k; return w; }
        if (w.plain + c.n >= limit) {
            if (!k) w.status = GU_UNSUPPORTED;
            return w;
        }
        c.at = w.plain;
        w.plain += c.n;
        w.end = c.end;
        w.n_ok = k + 1;
        if (c.status == GU_MORE) { w.more = 1; return w; }
        if (c.last) { w.last = 1; return w; }
    }
    if (k == K) return w;
    w.status = GU_MORE;
    for (int j = k; j < K; ++j) {
        GuChunk &c = ch[j];
        if (j == k) {
            if (c.status != GU_OVER || (k && c.start != w.end)) {
                c.start = w.end;
                w.respec += 1;
            }
        } else {
            const GuChunk &p = ch[j - 1];
            if (p.status != GU_OK || p.last || (c.start == p.end && c.status != GU_OVER)) continue;
            if (c.start != p.end) {
                c.start = p.end;
                w.respec += 1;
            }
        }
        redo[w.n_redo++] = j;
    }
    return w;
}

// Where the chunks of a long member whose deflate bits start at byte p end: at the first candidate behind p whose parse
// found a whole member or reached its budget -- the member that most likely follows -- or at n.  A wrong guess costs
// time only: the last chunk has no nominal end and decodes on to the member's last block.
CG_HD long long gu_member_bound(const int32_t *cand, const GuMember *res, int n_cand, long long p, long long n)
{
    int lo = 0, hi = n_cand;
    while (lo < hi) {
        const int mid = (lo + hi) / 2;
        if (cand[mid] <= p) lo = mid + 1; else hi = mid;
    }
    for (; lo < n_cand; ++lo)
        if (res[lo].status == GU_OK || res[lo].status == GU_LONG) return cand[lo];
    return n;
}

// The rounds of walk and decode one block path can take.  A round confirms at least one more chunk, or multiplies the
// room of the first unconfirmed chunk by 8 (the room never passes the limit): at most K * (1 + growths) rounds.
CG_HD long long gu_walk_rounds(int K, long long room0, long long limit)
{
    int growths = 1;
    for (long long r = room0; r < limit; r *= 8) ++growths;
    return (long long)K * (1 + growths);
}

// the byte of symbol s of a chunk whose window is win
CG_HD uint8_t gu_sym(uint16_t s, const uint8_t *win) { return s < 256 ? (uint8_t)s : win[s - 256]; }

// byte i of the window behind a chunk of n symbols whose own window is win
CG_HD uint8_t gu_win_byte(const uint8_t *win, const uint16_t *sym, long long n, int i)
{
    const long long q = n + i;                 // in (win followed by the chunk)
    return q < GU_WIN ? win[q] : gu_sym(sym[q - GU_WIN], win);
}

// a marker of a chunk that starts mpos plain bytes into its member points in front of the member's first byte
CG_HD bool gu_sym_behind(uint16_t s, long long mpos) { return s >= 256 && (long long)(s - 256) + mpos < GU_WIN; }

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
