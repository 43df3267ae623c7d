// cg_setbuild.cpp -- see cg_setbuild.h.
//
// This is the batched equivalent of Aligner.__cinit__/_set_reference (_align.pyx:195-277),
// PrefixComparer.__init__ (_align.pyx:615-642) and the table part of KmerFinder.__cinit__
// (_kmer_finder.pyx:106-165): it runs once per adapter set on the host; nothing here is on
// the per-read path.
#include "cg_setbuild.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <utility>

static void put2(uint8_t *t, char c, uint8_t v)
{
    t[(uint8_t)c] = v;
    t[(uint8_t)(c | 0x20)] = v;
}

void cg_build_enc_tables(uint8_t *out)
{
    uint8_t *up = out, *acgt = out + 256, *iupac = out + 512;
    for (int c = 0; c < 256; ++c) up[c] = (uint8_t)((c >= 'a' && c <= 'z') ? c - 32 : c);
    memset(acgt, 0x80, 256);
    put2(acgt, 'A', 1); put2(acgt, 'C', 2); put2(acgt, 'G', 4); put2(acgt, 'T', 8); put2(acgt, 'U', 8);
    memset(iupac, 0, 256);
    const uint8_t A = 1, C = 2, G = 4, T = 8;
    put2(iupac, 'X', 0); put2(iupac, 'A', A); put2(iupac, 'C', C); put2(iupac, 'G', G);
    put2(iupac, 'T', T); put2(iupac, 'U', T); put2(iupac, 'R', A | G); put2(iupac, 'Y', C | T);
    put2(iupac, 'S', G | C); put2(iupac, 'W', A | T); put2(iupac, 'K', G | T); put2(iupac, 'M', A | C);
    put2(iupac, 'B', C | G | T); put2(iupac, 'D', A | G | T); put2(iupac, 'H', A | C | T);
    put2(iupac, 'V', A | C | G); put2(iupac, 'N', 0x8F);
}

static uint32_t align_up(uint32_t x, uint32_t a) { return (x + a - 1) / a * a; }

// ------------------------------------------------------------------------------------------
// Two-phase program: re-pack the KmerFinder entries of ONE adapter into 32-bit scan words and
// add the locator chunks.  Returns false if the adapter does not fit the scheme (the general
// fused kernel is used instead); nothing here affects results, only which kernel runs.
// ------------------------------------------------------------------------------------------
namespace {

struct ScanKmer {
    int len = 0;
    int window = 0;                       // SUFFIX: characters from the end; PREFIX: from the start
    bool pass = false, loc = false;
    int bmin = 255, bmax = 0;             // locator: adapter offsets (exclusive end) of this chunk
    std::vector<int> bends;               // ... every one of them (equal chunks of a repetitive adapter share a pattern)
    std::vector<std::array<uint64_t, 2>> cols;   // per character: set of matching ASCII codes
    bool same_pattern(const ScanKmer &o) const { return len == o.len && cols == o.cols; }
};

void put_u32(std::vector<uint8_t> &pool, uint32_t v) { pool.insert(pool.end(), (uint8_t *)&v, (uint8_t *)&v + 4); }

// Split one reference-form entry into its k-mers (init bit .. found bit, _kmer_finder.pyx:143-147)
bool split_entry(const cg_kmer_entry &e, const uint64_t *mask128, std::vector<ScanKmer> &out, int window)
{
    int bit = 0;
    uint64_t init = e.init_mask, found = e.found_mask;
    while (init) {
        while (!((init >> bit) & 1ULL)) ++bit;
        int end = bit;
        while (end < 64 && !((found >> end) & 1ULL)) {
            if (end > bit && ((init >> end) & 1ULL)) return false;   // a second start before the end
            ++end;
        }
        if (end >= 64) return false;
        ScanKmer k;
        k.len = end - bit + 1;
        k.window = window;
        k.pass = true;
        if (k.len > 32) return false;
        k.cols.resize(k.len);
        for (int t = 0; t < k.len; ++t) {
            std::array<uint64_t, 2> set = {0, 0};
            for (int c = 0; c < 128; ++c)
                if ((mask128[c] >> (bit + t)) & 1ULL) set[c >> 6] |= 1ULL << (c & 63);
            k.cols[t] = set;
        }
        out.push_back(k);
        init &= ~(1ULL << bit);
        found &= ~(1ULL << end);
        bit = end + 1;
        if (bit >= 64 && init) return false;
    }
    return found == 0;
}

// Pack k-mers of one window type into words.  `gap` leaves one dead bit between k-mers so that the
// last bit of one cannot seed the first bit of the next while that one is not active.
void pack_words(const std::vector<ScanKmer> &kmers, uint32_t type, bool gap, std::vector<uint8_t> &pool,
                std::vector<CgScanWord> &words)
{
    size_t i = 0;
    while (i < kmers.size()) {
        CgScanWord W;
        memset(&W, 0, sizeof W);
        W.type = type;
        std::vector<uint32_t> mask(256, 0);    // 256 entries: any byte indexes it, bytes >= 128 match nothing
        std::vector<std::pair<int, int>> placed;   // (kmer index, offset)
        int used = 0;
        while (i < kmers.size()) {
            const ScanKmer &k = kmers[i];
            const int need = k.len + ((gap && used > 0) ? 1 : 0);
            if (used + need > 32) break;
            const int off = used + ((gap && used > 0) ? 1 : 0);
            for (int t = 0; t < k.len; ++t)
                for (int c = 0; c < 128; ++c)
                    if ((k.cols[t][c >> 6] >> (c & 63)) & 1ULL) mask[c] |= 1u << (off + t);
            W.init |= 1u << off;
            const uint32_t fbit = 1u << (off + k.len - 1);
            if (k.pass) W.pass_found |= fbit;
            if (k.loc) W.loc_found |= fbit;
            if ((uint32_t)k.window > W.span) W.span = (uint32_t)k.window;
            placed.emplace_back((int)i, off);
            used = off + k.len;
            ++i;
        }
        while (pool.size() % 4) pool.push_back(0);
        W.mask_off = (uint32_t)pool.size();
        for (uint32_t v : mask) put_u32(pool, v);
        if (W.loc_found) {
            W.loc_off = (uint32_t)pool.size();
            std::vector<uint8_t> tab(64, 0);
            for (auto &pl : placed) {
                const ScanKmer &k = kmers[pl.first];
                if (!k.loc) continue;
                const int fb = pl.second + k.len - 1;
                tab[2 * fb] = (uint8_t)k.bmin; tab[2 * fb + 1] = (uint8_t)k.bmax;
            }
            pool.insert(pool.end(), tab.begin(), tab.end());
        }
        if (type != CG_SCAN_WHOLE) {
            W.pos_off = (uint32_t)pool.size();
            const int rows = (type == CG_SCAN_SUFFIX) ? (int)W.span + 1 : (int)W.span;
            for (int x = 0; x < rows; ++x) {
                uint32_t init = 0, found = 0;
                for (auto &pl : placed) {
                    const ScanKmer &k = kmers[pl.first];
                    // SUFFIX: x = distance from the end, active while x <= window
                    // PREFIX: x = position, active while x < window
                    const bool active = (type == CG_SCAN_SUFFIX) ? (x >= 1 && x <= k.window) : (x < k.window);
                    if (active) { init |= 1u << pl.second; found |= 1u << (pl.second + k.len - 1); }
                }
                put_u32(pool, init);
                put_u32(pool, found);
            }
        }
        words.push_back(W);
    }
}

// 2-bit code of a k-mer position that matches exactly one of A/C/G/T in both cases, else -1
int plane_code(const std::array<uint64_t, 2> &set)
{
    for (const char *b = "ACGT"; *b; ++b) {
        std::array<uint64_t, 2> want = {0, 0};
        const int up = *b, lo = *b | 0x20;
        want[up >> 6] |= 1ULL << (up & 63);
        want[lo >> 6] |= 1ULL << (lo & 63);
        if (set == want) return (up >> 1) & 3;
    }
    return -1;
}

// The bit-plane form of the scan program (plane_scan_core in cg_core.cuh).  Empty if the adapter does not
// qualify: every k-mer position must be a plain A/C/G/T, no prefix windows, suffix windows of <= 64
// characters, a forward adapter of <= 64 characters with locator chunks.
// KmerFinder.kmers_present (_kmer_finder.pyx:170-213) of the reference-form entries on a short string, host side
bool entries_present(const cg_adapter_desc &d, const uint8_t *s, int n)
{
    for (int e = 0; e < d.n_kmer_entries; ++e) {
        const cg_kmer_entry &k = d.kmer_entries[e];
        const uint64_t *mk = d.kmer_masks + 128 * (size_t)e;
        long long start = k.search_start, stop = k.search_stop;
        if (start < 0) { start += n; if (start < 0) start = 0; }
        else if (start > n) continue;
        if (stop < 0) { stop += n; if (stop <= 0) continue; }
        else if (stop == 0) stop = n;
        if (stop > n) stop = n;
        uint64_t R = 0;
        for (long long i = start; i < stop; ++i) {
            R = ((R << 1) | k.init_mask) & mk[s[i] & 127];
            if (R & k.found_mask) return true;
        }
    }
    return false;
}

void build_plane_program(const cg_adapter_desc &d, const CgAdapter &A, const uint8_t *enc_ref, const int32_t *maxcost,
                         int windowed, int exact_ok, int myers,
                         const std::vector<ScanKmer> &whole, const std::vector<ScanKmer> &suffix,
                         const std::vector<ScanKmer> &prefix, std::vector<uint8_t> &out, int &n_ops, int &flags)
{
    out.clear();
    n_ops = 0;
    flags = 0;
    if (!windowed || myers || A.reverse || !prefix.empty() || A.m > 64 || !A.compare_ascii) return;
    std::vector<CgPlaneKmer> prog;
    bool any_loc = false, unambiguous = true;
    auto add = [&](const ScanKmer &k, uint32_t type) -> bool {
        if (k.len < 1 || k.len > 32) return false;
        CgPlaneKmer pk;
        memset(&pk, 0, sizeof pk);
        for (int t = 0; t < k.len; ++t) {
            const int code = plane_code(k.cols[t]);
            if (code < 0) return false;
            pk.codes |= (uint64_t)code << (2 * t);
        }
        pk.len = (uint8_t)k.len; pk.type = (uint8_t)type;
        pk.flags = (uint8_t)((k.pass ? CG_PLANE_PASS : 0u) | (k.loc ? CG_PLANE_LOC : 0u));
        if (type == CG_SCAN_SUFFIX) {
            if (k.window < 1 || k.window > 64) return false;
            pk.window = (uint16_t)k.window;
        }
        if (k.loc) {
            any_loc = true;
            unambiguous = unambiguous && k.bmin == k.bmax;
            // a pattern that occurs at several adapter offsets (repetitive adapter) points at several adapter ends:
            // one locator entry per offset
            for (size_t i = 0; i < k.bends.size(); ++i) {
                pk.bend = (uint8_t)k.bends[i];
                if (i > 0) pk.flags = (uint8_t)CG_PLANE_LOC;      // (the prefilter verdict is taken once)
                prog.push_back(pk);
            }
            return true;
        }
        prog.push_back(pk);
        return true;
    };
    for (auto &k : whole) if (!add(k, CG_SCAN_WHOLE)) return;
    for (auto &k : suffix) if (!add(k, CG_SCAN_SUFFIX)) return;
    if (!any_loc || prog.size() > 32) return;
    const size_t n_base = prog.size();
    (void)n_base;
    // an exact occurrence may be reported straight from the planes if the locator is unambiguous
    // (exact_ok), the adapter itself is plain A/C/G/T, and KmerFinder.kmers_present is certain to say
    // yes for a read that contains the whole adapter: some whole-read k-mer of the prefilter is a
    // substring of the adapter (or there is no prefilter at all)
    bool plain = true;
    std::vector<int> acode(A.m);
    for (int i = 0; i < A.m; ++i) {
        const uint8_t c = enc_ref[i];
        if (c != 'A' && c != 'C' && c != 'G' && c != 'T') plain = false;
        acode[i] = (c >> 1) & 3;
    }
    bool implies_pass = A.pf_count == 0;
    for (auto &pk : prog) {
        if (implies_pass || pk.type != CG_SCAN_WHOLE || !(pk.flags & CG_PLANE_PASS)) continue;
        for (int s = 0; s + pk.len <= A.m && !implies_pass; ++s) {
            bool eq = true;
            for (int t = 0; t < pk.len && eq; ++t) eq = acode[s + t] == (int)((pk.codes >> (2 * t)) & 3);
            implies_pass = eq;
        }
    }
    if (exact_ok && unambiguous && plain && implies_pass) flags |= 1;
    // End analysis for 3' adapters (flags BACK: free read ends, partial adapter allowed at the end): what can the
    // last-column scan (_align.pyx:536-572) accept?  Cell (i, n) with c errors, 1 <= c <= maxcost[i] = e: the first
    // lo_e = min{i: maxcost[i] >= e} adapter characters are aligned with <= e errors inside the last i + e characters
    // of the read, so one of e + 1 disjoint pieces of adapter[:lo_e] occurs there exactly (pigeonhole).  GUARD
    // k-mers = those pieces, searched in the last hi_e + e characters (hi_e = longest prefix with maxcost == e): if
    // none occurs, every acceptable cell is an exact overlap, and of a length < lo_1 (a longer one contains the
    // pieces of level 1).  OVERLAP emits report those exact overlaps (lengths min_overlap .. lo_1 - 1).
    uint64_t overlap_ok = 0;
    // (Measured on the benchmark shape: the two guard emits, seven overlap emits and two extra chain steps cost the
    //  first stage more (+0.43 ms per 100 M reads) than the plan stage saves, because a warp of the plan stage only
    //  gets faster when all of its 32 reads skip the end window.  Kept for adapters / data where the end of the read
    //  is where the work is; CUTADAPT_B200_END_ANALYSIS=1 turns it on.)
    const char *end_env = getenv("CUTADAPT_B200_END_ANALYSIS");
    const bool end_analysis = end_env && end_env[0] == '1';
    if (end_analysis && (A.flags & 15) == 14 && A.indel_cost == 1 && plain && (flags & 1) && A.m <= 63 && maxcost) {
        int top = 0;
        for (int i = 0; i <= A.m; ++i) top = std::max(top, (int)maxcost[i]);
        bool fits = true;
        int lo1 = A.m + 1;
        auto add_text = [&](int from, int len, uint8_t type, uint8_t fl, int window) {
            CgPlaneKmer pk;
            memset(&pk, 0, sizeof pk);
            if (len < 1 || len > 32) { fits = false; return; }
            for (int t = 0; t < len; ++t) pk.codes |= (uint64_t)acode[from + t] << (2 * t);
            pk.len = (uint8_t)len; pk.type = type; pk.flags = fl; pk.window = (uint16_t)window;
            prog.push_back(pk);
        };
        for (int e = 1; e <= top && fits; ++e) {
            int lo = -1, hi = -1;
            for (int i = A.min_overlap; i <= A.m; ++i) {
                if (maxcost[i] >= e && lo < 0) lo = i;
                if (maxcost[i] == e) hi = i;
            }
            if (lo < 0 || hi < 0) continue;               // no overlap length with exactly this budget
            if (e == 1) lo1 = lo;
            if (lo < e + 1 || hi + e > 64) { fits = false; break; }
            const int base = lo / (e + 1), extra = lo % (e + 1);
            int pos = 0;
            for (int c = 0; c <= e; ++c) {
                const int len = base + (c < extra ? 1 : 0);
                add_text(pos, len, CG_SCAN_SUFFIX, (uint8_t)CG_PLANE_GUARD, hi + e);
                pos += len;
            }
        }
        // budgets that exist but start below min_overlap would need lo = min_overlap: covered (lo is searched from it)
        for (int i = A.min_overlap; i < lo1 && i <= A.m && fits; ++i) {
            if (i > 32) { fits = false; break; }
            add_text(0, i, CG_SCAN_OVERLAP, 0, 0);
            if (A.pf_count == 0 || entries_present(d, enc_ref, i)) overlap_ok |= 1ULL << i;
        }
        if (fits && prog.size() <= 48) flags |= 2;
        else { while (!prog.empty() && (prog.back().type == CG_SCAN_OVERLAP || (prog.back().flags & CG_PLANE_GUARD))) prog.pop_back(); }
    }
    // chains: sort the k-mers by their code strings; a k-mer that extends the chain in progress adds
    // only its remaining characters
    std::vector<int> order(prog.size());
    for (size_t i = 0; i < prog.size(); ++i) order[i] = (int)i;
    auto text = [&](int i) {
        std::string t;
        for (int c = 0; c < prog[i].len; ++c) t.push_back((char)('0' + ((prog[i].codes >> (2 * c)) & 3)));
        return t;
    };
    std::sort(order.begin(), order.end(), [&](int a, int b) { return text(a) < text(b); });
    std::vector<uint32_t> ops;
    std::vector<CgPlaneEmit> emits;
    std::string chain;
    for (int idx : order) {
        const std::string t = text(idx);
        CgPlaneEmit em;
        memset(&em, 0, sizeof em);
        em.len = prog[idx].len; em.type = prog[idx].type; em.flags = prog[idx].flags; em.bend = prog[idx].bend;
        em.window = prog[idx].window;
        emits.push_back(em);
        const uint32_t eno = (uint32_t)emits.size();      // index + 1
        const bool extends = !chain.empty() && t.size() >= chain.size() && t.compare(0, chain.size(), chain) == 0;
        if (extends && t.size() == chain.size()) {         // same text: second emit slot of the last step
            if (((ops.back() >> 16) & 255u) == 0) { ops.back() |= eno << 16; continue; }
        }
        size_t from = 0;
        if (extends && t.size() > chain.size()) from = chain.size();
        for (size_t c = from; c < t.size(); ++c) {
            uint32_t op = (uint32_t)(t[c] - '0');
            if (c == 0) op |= CG_PLANE_OP_NEW;
            if (c + 1 == t.size()) op |= eno << 8;
            ops.push_back(op);
        }
        chain = t;
    }
    if (emits.size() > 255 || ops.size() > 1024) return;
    n_ops = (int)ops.size();
    flags |= (int)(emits.size() << 8);
    out.resize((ops.size() * 4 + 7) / 8 * 8 + emits.size() * sizeof(CgPlaneEmit) + 8);
    memcpy(out.data(), ops.data(), ops.size() * 4);
    memcpy(out.data() + (ops.size() * 4 + 7) / 8 * 8, emits.data(), emits.size() * sizeof(CgPlaneEmit));
    memcpy(out.data() + out.size() - 8, &overlap_ok, 8);
}

bool build_scan_program(const cg_adapter_desc &d, const CgAdapter &A, const uint8_t *enc768,
                        const uint8_t *enc_ref, std::vector<uint8_t> &pool, std::vector<CgScanWord> &words,
                        int &windowed, int &exact_ok, int &myers, std::vector<uint8_t> &planes, int &plane_ops,
                        int &plane_flags)
{
    myers = 0;
    std::vector<ScanKmer> whole, suffix, prefix;
    for (int e = 0; e < d.n_kmer_entries; ++e) {
        const cg_kmer_entry &k = d.kmer_entries[e];
        const uint64_t *mk = d.kmer_masks + 128 * (size_t)e;
        if (k.search_start == 0 && k.search_stop == 0) {
            if (!split_entry(k, mk, whole, 0)) return false;
        } else if (k.search_start < 0 && k.search_stop == 0) {
            if (-k.search_start > 100000) return false;
            if (!split_entry(k, mk, suffix, (int)-k.search_start)) return false;
        } else if (k.search_start == 0 && k.search_stop > 0) {
            if (k.search_stop > 100000) return false;
            if (!split_entry(k, mk, prefix, (int)k.search_stop)) return false;
        } else {
            return false;
        }
    }
    // locator chunks: the k+1 nearly equal pieces of the whole adapter (pigeonhole principle);
    // only for adapters whose DP spans the whole read
    windowed = 0;
    const bool full_range = (A.flags & 2) && (A.flags & 8);
    const int m = A.m, pieces = A.k + 1;
    if (full_range && A.k >= 0 && pieces > m && m <= 64) myers = 1;
    if (full_range && A.k >= 0 && pieces <= m) {
        const int base = m / pieces, extra = m % pieces;
        // Piece lengths.  Plain adapters: nearly equal pieces (the partition KmerFinder uses too, so the chunks
        // coincide with its whole-read k-mers).  Adapters with wildcard positions (N runs of UMIs, IUPAC codes): any
        // partition into k + 1 contiguous pieces serves the pigeonhole argument, so the cuts are placed where they
        // balance the INFORMATION of the pieces, log2(4 / letters matched) per position -- a piece made of Ns hits
        // everywhere and would push the adapter onto the bit-vector plan although its other pieces are selective.
        std::vector<int> piece_len(pieces);
        for (int c = 0; c < pieces; ++c) piece_len[c] = base + (c < extra ? 1 : 0);
        {
            const uint8_t *qenc0 = enc768 + 256 * A.query_enc;
            std::vector<double> info(m);
            double total = 0.0;
            bool any_wild = false;
            for (int t = 0; t < m; ++t) {
                int cnt = 0;
                for (const char *b = "ACGT"; *b; ++b) {
                    const uint8_t rc = enc_ref[t];
                    cnt += A.compare_ascii ? (rc == qenc0[(int)*b]) : ((rc & qenc0[(int)*b]) != 0);
                }
                any_wild = any_wild || cnt != 1;
                info[t] = cnt >= 1 && cnt <= 4 ? std::log2(4.0 / cnt) : 2.0;
                total += info[t];
            }
            if (any_wild && total > 0.0) {
                // cut after the position where the running information passes c / pieces of the total; every piece
                // keeps at least one position
                std::vector<int> cuts;
                double run = 0.0;
                int next = 1;
                for (int t = 0; t < m && next < pieces; ++t) {
                    run += info[t];
                    const int left_pos = m - (t + 1), left_pieces = pieces - next;
                    if (run >= total * next / pieces - 1e-9 || left_pos == left_pieces) {
                        if (left_pos >= left_pieces) { cuts.push_back(t + 1); ++next; }
                    }
                }
                if ((int)cuts.size() == pieces - 1) {
                    int prev = 0;
                    for (int c = 0; c < pieces - 1; ++c) { piece_len[c] = cuts[c] - prev; prev = cuts[c]; }
                    piece_len[pieces - 1] = m - prev;
                }
            }
        }
        std::vector<ScanKmer> chunks;
        bool ok = true;
        int pos = 0;
        for (int c = 0; c < pieces && ok; ++c) {
            const int len = piece_len[c];
            if (len > 32 || len < 1) { ok = false; break; }
            ScanKmer k;
            k.len = len; k.loc = true;
            k.cols.resize(len);
            const uint8_t *qenc = enc768 + 256 * A.query_enc;
            for (int t = 0; t < len; ++t) {
                std::array<uint64_t, 2> set = {0, 0};
                const uint8_t rc = enc_ref[pos + t];
                for (int code = 0; code < 128; ++code) {
                    const bool eq = A.compare_ascii ? (rc == qenc[code]) : ((rc & qenc[code]) != 0);
                    if (eq) set[code >> 6] |= 1ULL << (code & 63);
                }
                k.cols[t] = set;
            }
            pos += len;
            k.bmin = k.bmax = pos;
            k.bends.push_back(pos);
            bool dup = false;
            for (auto &o : chunks)
                if (o.same_pattern(k)) { dup = true; o.bmin = std::min(o.bmin, pos); o.bmax = std::max(o.bmax, pos); o.bends.push_back(pos); }
            if (!dup) chunks.push_back(k);
        }
        // How often do the chunks hit by chance?  p_hit = expected hits per read position for uniform
        // A/C/G/T reads.  A false hit costs a DP window of ~ (m + 2k) x m cells (measured: one cell costs
        // about 12 instruction slots in the run kernels); the bit-vector pass of plan_runs_myers costs ~17
        // (m <= 32) or ~34 slots per position and finds the runs exactly, so it wins once
        // p_hit * 12 m (m + 2k) exceeds that -- adapters with many wildcards, N runs, or high error rates.
        double p_hit = 0.0;
        if (ok) {
            for (auto &c : chunks) {
                double p = 1.0;
                for (auto &set : c.cols) {
                    int cnt = 0;
                    for (const char *b = "ACGT"; *b; ++b) cnt += (int)((set[(*b) >> 6] >> ((*b) & 63)) & 1ULL);
                    p *= cnt / 4.0;
                }
                p_hit += p;
            }
        }
        // (Round 2 re-measured the balance with the plan stage's candidate filter in place -- a false hit then costs a
        //  bit-vector pass over the run, not a DP window -- on BASELINE config 3: moving its 21-base linked 3' adapter
        //  and the N-run adapter from the bit-vector plan to locator chunks made the pass 14 % SLOWER (plan 86 -> 99 ms,
        //  DP rounds 42 -> 57 ms per 100 M reads): at e = 0.15 the 5-base chunks hit every second read.  The model stays.)
        const double myers_cost = m <= 32 ? 17.0 : 34.0;
        if (m <= 64 && (!ok || p_hit * 12.0 * m * (m + 2.0 * A.k) > myers_cost)) {
            myers = 1;
        } else if (ok && m <= 250) {
            for (auto &c : chunks) {
                bool merged = false;
                for (auto &w : whole)
                    if (w.same_pattern(c)) { w.loc = true; w.bmin = c.bmin; w.bmax = c.bmax; w.bends = c.bends; merged = true; break; }
                if (!merged) whole.push_back(c);
            }
            windowed = 1;
        }
    }
    // Exact-occurrence shortcut (see plan_runs in cg_core.cuh): needs an unambiguous chunk -> offset
    // map, no free adapter start, and k <= m/2.
    exact_ok = 0;
    // ... and the full-length exact match must itself be acceptable (_align.pyx:511-514)
    const bool full_ok = A.m >= A.min_overlap && floor((double)A.effective_length * d.max_error_rate) >= 0.0;
    if (windowed && full_ok && !(A.flags & 1) && A.k <= A.m / 2) {
        int loc_bits = 0;
        bool unambiguous = true;
        for (auto &w : whole)
            if (w.loc) { loc_bits += w.len; unambiguous = unambiguous && w.bmin == w.bmax; }
        // chunk patterns must be pairwise distinct (else bmin != bmax); the chunks may be spread over
        // several scan words (plan_hit_runs_dir combines them)
        if (unambiguous && loc_bits > 0) exact_ok = 1;
    }
    pack_words(whole, CG_SCAN_WHOLE, false, pool, words);
    pack_words(suffix, CG_SCAN_SUFFIX, true, pool, words);
    pack_words(prefix, CG_SCAN_PREFIX, true, pool, words);
    build_plane_program(d, A, enc_ref, (const int32_t *)(pool.data() + A.maxcost_off), windowed, exact_ok, myers, whole, suffix,
                        prefix, planes, plane_ops, plane_flags);
    return words.size() <= 64;
}

}  // namespace

static int32_t floor_to_i32(double x)
{
    if (!(x == x)) return -1;  // NaN: nothing is acceptable
    double f = floor(x);
    if (f > 2000000000.0) return 2000000000;
    if (f < -1.0) return -1;
    return (int32_t)f;
}

// AdapterIndex (adapters.py:1416-1466) -> open-addressing hash table keyed by the 2-bit packed affix.
static uint64_t index_hash(uint64_t bases, uint32_t len)
{
    uint64_t x = bases ^ ((uint64_t)len * 0x9E3779B97F4A7C15ULL);   // must equal cg_index_hash (cg_core.cuh)
    x ^= x >> 29; x *= 0xBF58476D1CE4E5B9ULL; x ^= x >> 32;
    return x;
}

static int build_indexes(const cg_index_desc *indexes, int n_indexes, int n_adapters,
                         std::vector<uint8_t> &blob, std::string &err)
{
    blob.clear();
    if (n_indexes <= 0) return CG_OK;
    if (!indexes) { err = "index array is NULL"; return CG_EINVAL; }
    std::vector<CgIndexHeader> H(n_indexes);
    std::vector<CgIndexEntry> T;
    const size_t hdr_entries = (size_t)n_indexes * sizeof(CgIndexHeader) / sizeof(CgIndexEntry);
    for (int x = 0; x < n_indexes; ++x) {
        const cg_index_desc &d = indexes[x];
        CgIndexHeader &h = H[x];
        memset(&h, 0, sizeof h);
        h.prefix = d.prefix ? 1 : 0;
        if (d.n_lengths <= 0 || d.n_lengths > 32 || !d.lengths) {
            err = "an adapter index needs 1..32 distinct key lengths"; return CG_EUNSUPPORTED;
        }
        for (int i = 0; i < d.n_lengths; ++i) {
            if (d.lengths[i] <= 0 || d.lengths[i] > 32) { err = "indexed adapters longer than 32 are not supported"; return CG_EUNSUPPORTED; }
            if (i && d.lengths[i] >= d.lengths[i - 1]) { err = "index key lengths must be strictly descending"; return CG_EINVAL; }
            h.lengths[i] = (uint8_t)d.lengths[i];
        }
        h.n_lengths = d.n_lengths;
        if (d.n_keys < 0 || (d.n_keys && (!d.keys || !d.adapter || !d.errors || !d.matches)) || d.stride <= 0) {
            err = "bad index key table"; return CG_EINVAL;
        }
        size_t cap = 16;
        while (cap < (size_t)d.n_keys * 2) cap <<= 1;
        if (cap > ((size_t)1 << 30)) { err = "adapter index too large"; return CG_EUNSUPPORTED; }
        const size_t base = T.size();
        T.resize(base + cap);
        memset(T.data() + base, 0, cap * sizeof(CgIndexEntry));
        h.table_off = (uint32_t)(hdr_entries + base);
        h.table_mask = (uint32_t)(cap - 1);
        for (int64_t k = 0; k < d.n_keys; ++k) {
            const uint8_t *s = d.keys + (size_t)k * d.stride;
            uint32_t len = 0;
            uint64_t bases = 0;
            while (len < (uint32_t)d.stride && s[len]) {
                uint64_t code;
                switch (s[len]) {
                case 'A': code = 0; break; case 'C': code = 1; break;
                case 'G': code = 2; break; case 'T': code = 3; break;
                default: err = "index keys must consist of A, C, G, T"; return CG_EINVAL;
                }
                if (len >= 32) { err = "index key longer than 32"; return CG_EUNSUPPORTED; }
                bases |= code << (2 * len);
                ++len;
            }
            if (len == 0) { err = "empty index key"; return CG_EINVAL; }
            if (d.adapter[k] < 0 || d.adapter[k] >= n_adapters || d.adapter[k] > 65535) {
                err = "index refers to an unknown adapter"; return CG_EINVAL;
            }
            if (d.errors[k] < 0 || d.errors[k] > 255 || d.matches[k] < 0 || d.matches[k] > 255) {
                err = "index errors/matches out of range"; return CG_EINVAL;
            }
            const uint32_t val = ((uint32_t)d.adapter[k] << 16) | ((uint32_t)d.errors[k] << 8) | (uint32_t)d.matches[k];
            size_t slot = (size_t)(index_hash(bases, len) & h.table_mask);
            for (;;) {
                CgIndexEntry &e = T[base + slot];
                if (e.len == 0) { e.bases = bases; e.len = len; e.val = val; break; }
                if (e.len == len && e.bases == bases) { err = "duplicate index key"; return CG_EINVAL; }
                slot = (slot + 1) & h.table_mask;
            }
        }
    }
    blob.resize(H.size() * sizeof(CgIndexHeader) + T.size() * sizeof(CgIndexEntry));
    memcpy(blob.data(), H.data(), H.size() * sizeof(CgIndexHeader));
    memcpy(blob.data() + H.size() * sizeof(CgIndexHeader), T.data(), T.size() * sizeof(CgIndexEntry));
    return CG_OK;
}

int cg_build_set(const cg_adapter_desc *ads, int n_adapters, const cg_group_desc *groups, int n_groups,
                 CgBuiltSet &out, std::string &err, const cg_index_desc *indexes, int n_indexes)
{
    {
        int rc = build_indexes(indexes, n_indexes, n_adapters, out.index_blob, err);
        if (rc != CG_OK) return rc;
    }
    if (n_adapters <= 0 || !ads) { err = "adapter set is empty"; return CG_EINVAL; }
    if (n_groups <= 0 || !groups) { err = "adapter set has no groups"; return CG_EINVAL; }
    uint8_t enc[768];
    cg_build_enc_tables(enc);

    std::vector<CgAdapter> A(n_adapters);
    std::vector<CgEntry> E;
    std::vector<uint8_t> pool;
    out.masks64.clear();
    out.effective_length.assign(n_adapters, 0);
    out.max_m = 0; out.any_wide = 0;

    for (int a = 0; a < n_adapters; ++a) {
        const cg_adapter_desc &d = ads[a];
        CgAdapter &x = A[a];
        memset(&x, 0, sizeof x);
        const int m = d.length;
        if (m < 0 || (m > 0 && !d.sequence)) { err = "adapter has no sequence"; return CG_EINVAL; }
        if (m > 65535) { err = "adapter longer than 65535 characters"; return CG_EUNSUPPORTED; }
        for (int i = 0; i < m; ++i)
            if (d.sequence[i] & 0x80) { err = "String must contain only ASCII characters"; return CG_ENONASCII; }
        if (d.kind != CG_KIND_ALIGNER && d.kind != CG_KIND_PREFIX_COMPARER && d.kind != CG_KIND_SUFFIX_COMPARER) {
            err = "unknown adapter kind"; return CG_EINVAL;
        }
        if (d.remove < 0 || d.remove > 2) { err = "unknown remove mode"; return CG_EINVAL; }
        const bool wr = d.wildcard_ref != 0, wq = d.wildcard_query != 0;
        x.m = m;
        x.flags = d.flags & 15;
        x.min_overlap = d.min_overlap;
        x.kind = d.kind;
        x.reverse = d.reverse_read ? 1 : 0;
        x.remove = d.remove;
        x.compare_ascii = (!wr && !wq) ? 1 : 0;
        x.query_enc = wq ? 2 : (wr ? 1 : 0);                  // _align.pyx:322-328, 672-678
        x.wildcard_ref = wr ? 1 : 0;
        x.indel_cost = d.indel_cost;

        // encoded adapter bytes
        x.ref_off = (uint32_t)pool.size();
        int n_upper = 0, n_lower = 0;
        for (int i = 0; i < m; ++i) { n_upper += d.sequence[i] == 'N'; n_lower += d.sequence[i] == 'n'; }
        if (d.kind == CG_KIND_ALIGNER) {
            if (d.indel_cost < 1) { err = "indel_cost must be at least 1"; return CG_EINVAL; }   // _align.pyx:217-218
            x.effective_length = m;
            if (wr) {                                          // _align.pyx:268-272
                x.effective_length = m - (n_upper + n_lower);
                if (x.effective_length == 0) { err = "Cannot have only N wildcards in the sequence"; return CG_EINVAL; }
            }
            for (int i = 0; i < m; ++i) {
                const uint8_t c = d.sequence[i];
                pool.push_back(wr ? enc[512 + c] : wq ? enc[256 + c] : c);   // _align.pyx:272-276
            }
            const double km = d.max_error_rate * (double)m;    // _align.pyx:343
            if (!(km == km) || km > 1.0e9 || km < -1.0e9) { err = "max_error_rate out of range"; return CG_EINVAL; }
            x.k = (int32_t)km;
            x.cell_mode = (d.indel_cost != 1 || x.k > CG_PACKED_MAX_K || x.k < 0 || m > CG_PACKED_MAX_M)
                              ? CG_CELL_WIDE : CG_CELL_PACKED32;
            if (x.cell_mode == CG_CELL_WIDE) out.any_wide = 1;
            // n_counts (int32, 4-aligned)                      _align.pyx:260-266
            while (pool.size() % 4) pool.push_back(0);
            x.ncount_off = (uint32_t)pool.size();
            {
                int32_t c = 0;
                for (int i = 0; i <= m; ++i) {
                    pool.insert(pool.end(), (uint8_t *)&c, (uint8_t *)&c + 4);
                    if (i < m && (d.sequence[i] == 'N' || d.sequence[i] == 'n')) ++c;
                }
            }
            // maxcost[L] = floor(L * rate): "cost <= L * rate" in IEEE double (_align.pyx:513,559)
            x.maxcost_off = (uint32_t)pool.size();
            for (int L = 0; L <= m; ++L) {
                int32_t v = floor_to_i32((double)L * d.max_error_rate);
                pool.insert(pool.end(), (uint8_t *)&v, (uint8_t *)&v + 4);
            }
            // peq[c]: which adapter rows match read character c (same test as _align.pyx:442-445)
            x.peq_off = (uint32_t)pool.size();
            {
                const uint8_t *qenc = enc + 256 * x.query_enc;
                const uint8_t *eref = pool.data() + x.ref_off;
                std::vector<uint32_t> lo(128, 0), hi(128, 0);
                for (int r = 0; r < m && r < 64; ++r)
                    for (int c = 0; c < 128; ++c) {
                        const bool eq = x.compare_ascii ? (eref[r] == qenc[c]) : ((eref[r] & qenc[c]) != 0);
                        if (eq) (r < 32 ? lo[c] : hi[c]) |= 1u << (r & 31);
                    }
                for (uint32_t v : lo) pool.insert(pool.end(), (uint8_t *)&v, (uint8_t *)&v + 4);
                for (uint32_t v : hi) pool.insert(pool.end(), (uint8_t *)&v, (uint8_t *)&v + 4);
            }
        } else {
            x.effective_length = m;
            if (wr) {                                          // _align.pyx:627-630 (sic: N minus n)
                x.effective_length -= n_upper - n_lower;
                if (x.effective_length == 0) { err = "Cannot have only N wildcards in the sequence"; return CG_EINVAL; }
            }
            if (!(d.max_error_rate >= 0.0 && d.max_error_rate <= 1.0)) {
                err = "max_error_rate must be between 0 and 1"; return CG_EINVAL;   // _align.pyx:631-632
            }
            x.max_k_cmp = (int32_t)(d.max_error_rate * (double)x.effective_length);  // _align.pyx:633
            if (d.min_overlap < 1) { err = "min_overlap must be at least 1"; return CG_EINVAL; }  // _align.pyx:634-635
            for (int i = 0; i < m; ++i) {
                const uint8_t c = d.sequence[i];
                pool.push_back(wr ? enc[512 + c] : wq ? enc[256 + c] : enc[c]);      // _align.pyx:637-642
            }
            x.cell_mode = CG_CELL_PACKED32;
        }
        out.effective_length[a] = x.effective_length;
        if (m > out.max_m) out.max_m = m;

        // prefilter entries (reference form)
        x.pf_first = (int32_t)E.size();
        x.pf_count = 0;
        if (d.n_kmer_entries > 0) {
            if (!d.kmer_entries || !d.kmer_masks) { err = "k-mer tables missing"; return CG_EINVAL; }
            for (int e = 0; e < d.n_kmer_entries; ++e) {
                const cg_kmer_entry &k = d.kmer_entries[e];
                if (k.search_start > 2000000000LL || k.search_start < -2000000000LL ||
                    k.search_stop > 2000000000LL || k.search_stop < -2000000000LL) {
                    err = "k-mer window out of range"; return CG_EINVAL;
                }
                CgEntry ce;
                memset(&ce, 0, sizeof ce);
                ce.start = (int32_t)k.search_start; ce.stop = (int32_t)k.search_stop;
                ce.mask_index = (uint32_t)(out.masks64.size() / 128);
                ce.init_mask = k.init_mask; ce.found_mask = k.found_mask;
                E.push_back(ce);
                out.masks64.insert(out.masks64.end(), d.kmer_masks + 128 * (size_t)e,
                                   d.kmer_masks + 128 * (size_t)(e + 1));
            }
            x.pf_count = d.n_kmer_entries;
        }
    }

    std::vector<CgGroup> G(n_groups);
    out.slots = 1;
    for (int g = 0; g < n_groups; ++g) {
        const cg_group_desc &d = groups[g];
        CgGroup &x = G[g];
        memset(&x, 0, sizeof x);
        x.type = d.type; x.a0 = d.a0; x.a1 = d.a1;
        x.front_required = d.front_required ? 1 : 0; x.back_required = d.back_required ? 1 : 0;
        if (d.type == CG_GROUP_SINGLE) {
            if (d.a0 < 0 || d.a0 >= n_adapters) { err = "group refers to an unknown adapter"; return CG_EINVAL; }
            x.a1 = -1;
        } else if (d.type == CG_GROUP_LINKED) {
            if (d.a0 < 0 || d.a0 >= n_adapters || d.a1 < 0 || d.a1 >= n_adapters) {
                err = "linked group refers to an unknown adapter"; return CG_EINVAL;
            }
            if (ads[d.a0].remove == CG_REMOVE_AUTO || ads[d.a1].remove == CG_REMOVE_AUTO) {
                err = "anywhere adapters cannot be linked"; return CG_EINVAL;
            }
            out.slots = 2;
        } else if (d.type == CG_GROUP_INDEXED) {
            if (d.a0 < 0 || d.a0 >= n_indexes) { err = "group refers to an unknown adapter index"; return CG_EINVAL; }
            x.a1 = -1;
        } else { err = "unknown group type"; return CG_EINVAL; }
    }
    if (n_groups > 256) { err = "more than 256 adapter groups"; return CG_EUNSUPPORTED; }

    // two-phase program for the common case: one SINGLE aligner adapter with packed cells
    std::vector<CgScanWord> scan_words;
    std::vector<uint8_t> plane_kmers;      // ops + emits of the bit-plane program
    int plane_flags = 0, plane_ops = 0;
    int simple_ok = 0, windowed = 0, exact_ok = 0, myers = 0;
    if (n_adapters == 1 && n_groups == 1 && G[0].type == CG_GROUP_SINGLE && A[0].kind == CG_KIND_ALIGNER &&
        A[0].cell_mode == CG_CELL_PACKED32) {
        std::vector<uint8_t> pool2 = pool;
        std::vector<CgScanWord> words;
        if (build_scan_program(ads[0], A[0], enc, pool.data() + A[0].ref_off, pool2, words, windowed, exact_ok, myers,
                               plane_kmers, plane_ops, plane_flags)) {
            pool.swap(pool2);
            scan_words.swap(words);
            simple_ok = 1;
        } else {
            windowed = 0; exact_ok = 0; myers = 0;
            plane_kmers.clear(); plane_flags = 0; plane_ops = 0;
        }
    }

    // assemble
    CgSetHeader H;
    memset(&H, 0, sizeof H);
    H.n_adapters = n_adapters; H.n_groups = n_groups; H.n_entries = (int32_t)E.size();
    H.slots = out.slots; H.max_m = out.max_m; H.any_wide = out.any_wide;
    uint32_t off = (uint32_t)sizeof(CgSetHeader);
    H.adapters_off = off; off += (uint32_t)(A.size() * sizeof(CgAdapter)); off = align_up(off, 16);
    H.groups_off = off; off += (uint32_t)(G.size() * sizeof(CgGroup)); off = align_up(off, 16);
    H.entries_off = off; off += (uint32_t)(E.size() * sizeof(CgEntry)); off = align_up(off, 16);
    H.scan_off = off; off += (uint32_t)(scan_words.size() * sizeof(CgScanWord)); off = align_up(off, 16);
    H.simple_ok = simple_ok; H.scan_count = (int32_t)scan_words.size(); H.windowed = windowed; H.exact_ok = exact_ok; H.myers = myers;
    H.plane_off = off; off += (uint32_t)plane_kmers.size(); off = align_up(off, 16);
    H.plane_count = plane_ops; H.plane_flags = plane_flags;
    H.pool_off = off; off += (uint32_t)pool.size(); off = align_up(off, 16);
    H.total_bytes = off;
    out.blob.assign(off, 0);
    memcpy(out.blob.data(), &H, sizeof H);
    memcpy(out.blob.data() + H.adapters_off, A.data(), A.size() * sizeof(CgAdapter));
    memcpy(out.blob.data() + H.groups_off, G.data(), G.size() * sizeof(CgGroup));
    if (!E.empty()) memcpy(out.blob.data() + H.entries_off, E.data(), E.size() * sizeof(CgEntry));
    if (!scan_words.empty())
        memcpy(out.blob.data() + H.scan_off, scan_words.data(), scan_words.size() * sizeof(CgScanWord));
    if (!plane_kmers.empty())
        memcpy(out.blob.data() + H.plane_off, plane_kmers.data(), plane_kmers.size());
    if (!pool.empty()) memcpy(out.blob.data() + H.pool_off, pool.data(), pool.size());
    out.n_adapters = n_adapters; out.n_groups = n_groups; out.simple_ok = simple_ok;
    out.max_k = 0;
    for (int a = 0; a < n_adapters; ++a) out.max_k = std::max(out.max_k, std::max(0, (int)(ads[a].max_error_rate * ads[a].length)));
    out.all_indexed = n_groups > 0;
    for (int g = 0; g < n_groups; ++g) out.all_indexed = out.all_indexed && G[g].type == CG_GROUP_INDEXED;
    if (out.masks64.empty()) out.masks64.assign(128, 0);   // never hand the kernel a null table
    return CG_OK;
}


void cg_build_phred_table(double *out256)
{
    for (int q = 0; q < 256; ++q) out256[q] = pow(10.0, -(double)q / 10.0);
}

// ---- multi-pass schedule -------------------------------------------------------------------------
int cg_plan_passes(const cg_adapter_desc *adapters, int n_adapters, const cg_group_desc *groups, int n_groups,
                   const cg_index_desc *indexes, int n_indexes, CgMultiPlan &plan, std::string &err)
{
    plan.passes.clear();
    plan.pass_map.clear();
    if (n_groups > CG_MAX_PASSES) return CG_OK;
    if (n_groups == 1 && groups[0].type != CG_GROUP_LINKED) return CG_OK;
    int total = 0;
    for (int g = 0; g < n_groups; ++g) total += groups[g].type == CG_GROUP_LINKED ? 2 : 1;
    if (total > CG_MAX_PASSES) return CG_OK;
    bool ok = true;
    for (int g = 0; g < n_groups && ok; ++g) {
        const cg_group_desc &G = groups[g];
        const int comps = G.type == CG_GROUP_LINKED ? 2 : 1;
        int front_pass = -1;
        for (int role = 0; role < comps && ok; ++role) {
            plan.passes.emplace_back();
            CgPassPlan &P = plan.passes.back();
            P.group = g; P.role = role; P.front_pass = role ? front_pass : -1;
            P.map_off = (int)plan.pass_map.size();
            if (role == 0) front_pass = (int)plan.passes.size() - 1;
            cg_group_desc G2;
            memset(&G2, 0, sizeof G2);
            G2.a1 = -1;
            if (G.type == CG_GROUP_INDEXED) {
                if (G.a0 < 0 || G.a0 >= n_indexes) { ok = false; break; }
                const cg_index_desc &X = indexes[G.a0];
                std::vector<int> local(n_adapters, -1);
                std::vector<cg_adapter_desc> sub_ads;
                std::vector<int32_t> remap((size_t)(X.n_keys > 0 ? X.n_keys : 0));
                for (int64_t k = 0; k < X.n_keys; ++k) {
                    const int ga = X.adapter[k];
                    if (ga < 0 || ga >= n_adapters) { ok = false; break; }
                    if (local[ga] < 0) {
                        local[ga] = (int)sub_ads.size();
                        sub_ads.push_back(adapters[ga]);
                        plan.pass_map.push_back(ga);
                    }
                    remap[(size_t)k] = local[ga];
                }
                if (!ok || sub_ads.empty()) { ok = false; break; }
                cg_index_desc X2 = X;
                X2.adapter = remap.data();
                G2.type = CG_GROUP_INDEXED;
                if (cg_build_set(sub_ads.data(), (int)sub_ads.size(), &G2, 1, P.set, err, &X2, 1) != CG_OK) ok = false;
            } else {
                const int ga = role ? G.a1 : G.a0;
                if (ga < 0 || ga >= n_adapters) { ok = false; break; }
                plan.pass_map.push_back(ga);
                G2.type = CG_GROUP_SINGLE;
                if (cg_build_set(adapters + ga, 1, &G2, 1, P.set, err) != CG_OK) ok = false;
                else if (adapters[ga].kind == CG_KIND_ALIGNER && !(P.set.simple_ok && P.set.max_m <= 64)) ok = false;
            }
        }
    }
    if (!ok) { plan.passes.clear(); plan.pass_map.clear(); }
    return CG_OK;
}

void cg_fill_select_tables(const CgGroup *groups, int n_groups, int slots, const std::vector<CgPassPlan> &passes,
                           CgSelectTables &t)
{
    memset(&t, 0, sizeof t);
    t.n_groups = n_groups; t.slots = slots;
    for (int g = 0; g < n_groups && g < CG_MAX_PASSES; ++g) {
        t.gtype[g] = (int8_t)groups[g].type;
        t.front_required[g] = (int8_t)groups[g].front_required;
        t.back_required[g] = (int8_t)groups[g].back_required;
    }
    for (size_t pi = 0; pi < passes.size() && pi < CG_MAX_PASSES; ++pi) {
        t.map_off[pi] = passes[pi].map_off;
        if (passes[pi].role == 0) t.pass0[passes[pi].group] = (int8_t)pi;
        else t.pass1[passes[pi].group] = (int8_t)pi;
    }
}
