// tests/hostsim/hostsim_gunzip_blocks.cpp -- TEST-ONLY host build of a split gzip input stream (CG_GZIN_SPLIT_MEMBERS):
// the steps of gzin_inflate_split / gzin_blocks (cutadapt_b200/csrc/cg_api.cu) in their order, on the same decisions
// (cutadapt_b200/csrc/cg_gunzip_core.cuh), with the chunk stride and the plain-size limit as parameters so that small
// inputs make many chunks and long members stream over submissions.  A stream object carries the member in progress from
// one submission to the next, as the device stream does.  Nothing in cutadapt_b200/ loads this library.
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../cutadapt_b200/csrc/cg_gunzip_core.cuh"
#include "../../cutadapt_b200/csrc/cg_gzip_core.cuh"

namespace {

struct Member { int in = 0, bitoff = 0, trailer = 0; uint32_t crc = 0; long long len = 0, start = 0; };

struct Stream {
    int split = 1;
    long long stride = 65536, long_member = 65536, consumed = 0, members = 0;
    Member mem;
    std::vector<uint8_t> win = std::vector<uint8_t>(GU_WIN, 0);
};

uint32_t le32(const uint8_t *p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }

struct Crc {
    uint32_t tab[256];
    Crc() { for (int i = 0; i < 256; ++i) tab[i] = gz_crc_entry((uint32_t)i); }
    uint32_t raw(uint32_t c, const uint8_t *p, long long n) const
    {
        while (n > 0) {
            const int k = (int)std::min(n, 1LL << 30);
            c = gz_crc_raw(c, p, k, tab);
            p += k;
            n -= k;
        }
        return c;
    }
};

// gzin_blocks: returns the walk; *placed: bytes written behind out + base
GuWalk blocks(const uint8_t *gz, long long n, long long bound, long long s0, long long stride, long long limit, Member &m,
              std::vector<uint8_t> &win, uint8_t *out, long long out_cap, long long *respec, int *over_cap)
{
    const int K = (int)std::max(1LL, (bound * 8 - s0 + stride * 8 - 1) / (stride * 8));
    const auto nominal = [&](int k) { return k >= K ? (long long)9e18 : s0 + (long long)k * stride * 8; };
    std::vector<GuChunk> ch(K);
    std::vector<long long> room(K, std::min(limit, 8 * stride));
    std::vector<std::vector<uint16_t>> sym(K);
    GuTables T;
    ch[0].start = s0;
    for (int k = 1; k < K; ++k) {
        ch[k].start = -1;
        for (long long b = nominal(k), hi = std::min(nominal(k) + stride * 8, n * 8); b < hi; ++b)
            if (gu_dyn_start(gz, n, b, T)) { ch[k].start = b; break; }
    }
    const auto decode = [&](int k) {
        sym[k].assign((size_t)room[k], 0);
        ch[k] = gu_chunk(gz, n, ch[k].start, nominal(k + 1), sym[k].data(), room[k], T);
    };
    for (int k = 0; k < K; ++k) decode(k);
    std::vector<int32_t> redo(K);
    GuWalk r;
    const long long max_rounds = gu_walk_rounds(K, room[0], limit);
    for (long long round = 0;; ++round) {
        r = gu_walk(ch.data(), K, limit, redo.data());
        if (r.status != GU_MORE) break;
        if (round >= max_rounds) { r.status = -1; return r; }
        *respec += r.respec;
        long long grown = 0;
        for (int i = 0; i < r.n_redo; ++i) {
            const int k = redo[i];
            if (ch[k].status != GU_OVER || (grown && grown >= limit)) continue;
            if (room[k] >= limit) {
                if (k != r.n_ok) continue;
                r.status = r.n_ok ? GU_OK : GU_UNSUPPORTED;
                break;
            }
            room[k] = std::min(limit, room[k] * 8);
            grown += room[k];
        }
        if (r.status != GU_MORE) break;
        for (int i = 0; i < r.n_redo; ++i) decode(redo[i]);
    }
    if (r.status != GU_OK) return r;
    if (r.plain > out_cap) { *over_cap = 1; return r; }
    std::vector<uint8_t> nx(GU_WIN);
    for (int k = 0; k < r.n_ok; ++k) {
        const GuChunk &c = ch[k];
        for (long long j = 0; j < c.n; ++j) {
            if (gu_sym_behind(sym[k][j], m.len + c.at)) r.status = GU_INVALID;
            out[c.at + j] = gu_sym(sym[k][j], win.data());
        }
        for (int i = 0; i < GU_WIN; ++i) nx[i] = gu_win_byte(win.data(), sym[k].data(), c.n, i);
        win.swap(nx);
    }
    static const Crc crc;
    m.crc = crc.raw(m.crc, out, r.plain);
    m.len += r.plain;
    return r;
}

}  // namespace

extern "C" void *hs_gzb_create(int split, int64_t stride, int64_t long_member)
{
    Stream *s = new Stream;
    s->split = split;
    s->stride = stride;
    s->long_member = long_member;
    return s;
}

extern "C" void hs_gzb_destroy(void *s) { delete (Stream *)s; }

// One submission of gz[0, n) on stream `s`: the plain bytes go to out[0, out_cap).  Returns GU_OK, GU_INVALID,
// GU_UNSUPPORTED (-1: out_cap too small).  info: consumed, plain, in_member, respeculated, err_at (file offset of the bad
// member), bit offset kept, members.  An error leaves the stream unchanged; limit: the plain-size limit of a submission.
extern "C" int hs_gzb_submit(void *sp, const uint8_t *gz, int64_t n, int final, int64_t limit, uint8_t *out,
                             int64_t out_cap, int64_t *info)
{
    Stream &s = *(Stream *)sp;
    static const Crc crc;
    std::vector<int32_t> cand;
    for (int64_t p = 0; p + 3 <= n; ++p)
        if (gz[p] == 0x1f && gz[p + 1] == 0x8b && gz[p + 2] == 8) cand.push_back((int32_t)p);
    GuTables T;
    std::vector<GuMember> res(cand.size());
    for (size_t k = 0; k < cand.size(); ++k)
        res[k] = gu_member(gz + cand[k], n - cand[k], nullptr, T, s.split ? s.long_member : 0);
    std::vector<int32_t> members(cand.size() + 1);
    std::vector<long long> moff(cand.size() + 1);
    Member m = s.mem;
    std::vector<uint8_t> win = s.win;
    long long p = 0, base = 0, nm = 0, respec = 0;
    bool after = s.members > 0;
    memset(info, 0, 7 * sizeof(int64_t));
    const auto bad = [&](long long at) { info[4] = at; return GU_INVALID; };
    for (;;) {
        if (m.in && m.trailer) {
            const long long t = p + (m.bitoff ? 1 : 0);
            if (t + 8 > n) {
                if (final) return bad(m.start);
                break;
            }
            if (le32(gz + t) != ~m.crc || le32(gz + t + 4) != (uint32_t)m.len) return bad(m.start);
            p = t + 8;
            m = Member();
            nm += 1;
            after = true;
            continue;
        }
        if (m.in) {
            int over_cap = 0;
            const long long bound = gu_member_bound(cand.data(), res.data(), (int)cand.size(), p, n);
            const GuWalk r = blocks(gz, n, bound, p * 8 + m.bitoff, s.stride, limit - base, m, win, out + base, out_cap - base,
                                    &respec, &over_cap);
            if (over_cap || r.status < 0) return -1;
            if (r.status == GU_INVALID) return bad(m.start);
            if (r.status == GU_UNSUPPORTED) {
                if (base == 0 && p == 0 && !nm) { info[4] = m.start; return GU_UNSUPPORTED; }
                break;
            }
            base += r.plain;
            p = r.end >> 3;
            m.bitoff = (int)(r.end & 7);
            if (r.last) { m.trailer = 1; continue; }
            if (r.more && final) return bad(m.start);
            break;
        }
        const GuChain c = gu_chain(gz, n, cand.data(), res.data(), (int)cand.size(), after, final != 0, base, limit,
                                   members.data(), moff.data(), p, s.split != 0);
        if (c.status == GU_INVALID) return bad(s.consumed + c.err_at);
        if (c.status == GU_UNSUPPORTED && (!s.split || (base == 0 && p == 0 && !nm))) {
            info[4] = s.consumed + c.err_at;
            return GU_UNSUPPORTED;
        }
        if (base + c.plain > out_cap) return -1;
        for (int k = 0; k < c.n_members; ++k) {
            const int32_t at = cand[members[k]];
            uint8_t *o = out + moff[k];
            gu_member(gz + at, n - at, o, T);
            if (~crc.raw(0xffffffffu, o, res[members[k]].plain) != res[members[k]].crc) return bad(s.consumed + at);
        }
        base += c.plain;
        nm += c.n_members;
        after = after || c.n_members > 0;
        p = c.consumed;
        if (c.status != GU_LONG) break;
        m = Member();
        m.in = 1;
        m.crc = 0xffffffffu;
        m.start = s.consumed + c.err_at;
        p = c.err_at + gu_head(gz + c.err_at, n - c.err_at);
    }
    s.consumed += p;
    s.members += nm;
    s.mem = m;
    if (m.in) s.win = win;
    info[0] = p;
    info[1] = base;
    info[2] = m.in;
    info[3] = respec;
    info[5] = m.bitoff;
    info[6] = nm;
    return GU_OK;
}
