// cg_core.cuh -- per-read device functions of the adapter-trimming hot path.
//
// Everything here is `__host__ __device__`: the kernels in cg_kernels.cu call it with one
// lane per read; tests/hostsim compiles the very same functions for the host so that the
// selection logic can be fuzzed against the oracle on a machine without a GPU.  (The host
// build exists only under tests/; the shipped library never runs it.)
//
// Reference semantics restated here (file:line relative to the reference checkout):
//   kmers_present_core   _kmer_finder.pyx:170-213, 241-257
//   locate_core          _align.pyx:298-587       (column-major DP with Ukkonen cut-off,
//                                                  cost/score/origin triples, cutadapt's
//                                                  "best overlap" selection, incl. the stale
//                                                  `origin` at line 565)
//   compare_core         _align.pyx:651-714       (Prefix/SuffixComparer)
//   quality_trim_core    qualtrim.pyx:22-73
//   match_single/linked/multiple   adapters.py:707-724, 758-786, 815-832, 862-890, 915-935,
//                                  1215-1227, 1265-1286
//   process_read         modifiers.py:853-858 (QualityTrimmer) + 225-231 (AdapterCutter rounds)
#pragma once
#include "cg_types.h"

#define CGK_KIND_ALIGNER 0
#define CGK_KIND_PREFIX 1
#define CGK_KIND_SUFFIX 2
#define CGK_REMOVE_BEFORE 0
#define CGK_REMOVE_AFTER 1
#define CGK_REMOVE_AUTO 2
#define CGK_GROUP_SINGLE 0
#define CGK_GROUP_LINKED 1
#define CGK_GROUP_INDEXED 2

CG_HD int cg_ctz(uint32_t x)   // x != 0
{
#if defined(__CUDA_ARCH__)
    return __ffs((int)x) - 1;
#else
    return __builtin_ctz(x);
#endif
}
CG_HD uint32_t cg_funnel_r(uint32_t lo, uint32_t hi, uint32_t shift_bits)   // (hi:lo) >> shift_bits, shift in {0,8,16,24}
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, shift_bits);
#else
    return shift_bits ? (lo >> shift_bits) | (hi << (32 - shift_bits)) : lo;
#endif
}
// Byte load through a 32-bit shared-memory address computed once (device only).  Loads through a generic
// pointer into shared memory make the compiler re-derive the shared window (S2R SR_CgaCtaId + LEA) at
// every use inside the DP column loop, on the critical path of character -> match mask -> cells.
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ uint32_t cg_lds_u8(uint32_t saddr)
{
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(saddr));
    return v;
}
// character cursor of the plan stage (its read window is always in shared memory on the device)
#define CG_CHARPTR(name, expr) uint32_t name = (uint32_t)__cvta_generic_to_shared(expr)
#define CG_CHAR(cursor) cg_lds_u8((uint32_t)(cursor))
// 32-bit table in shared memory (scan masks, peq): base converted once, entries by index
__device__ __forceinline__ uint32_t cg_lds_u32(uint32_t saddr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
    return v;
}
#define CG_TABPTR(name, expr) const uint32_t name = (uint32_t)__cvta_generic_to_shared(expr)
#define CG_TAB32(tab, i) cg_lds_u32((tab) + 4u * (uint32_t)(i))
#else
#define CG_CHARPTR(name, expr) const uint8_t *name = (expr)
#define CG_CHAR(cursor) ((uint32_t) * (cursor))
#define CG_TABPTR(name, expr) const uint32_t *name = (expr)
#define CG_TAB32(tab, i) ((tab)[i])
#endif
template <class X> CG_HD X cg_min(X a, X b) { return a < b ? a : b; }
template <class X> CG_HD X cg_max(X a, X b) { return a > b ? a : b; }

// A (sub)sequence of a read, optionally seen back to front (Rightmost* adapters search the
// reversed read, adapters.py:766,870).
struct ReadView {
    const uint8_t *p;
    int n;
    int rev;
    CG_HD uint8_t at(int j) const { return rev ? p[n - 1 - j] : p[j]; }
};

// ---------------------------------------------------------------------------------------
// DP cells.
//
// Packed32 keeps (cost, score, origin) of _align.pyx:23-26 in ONE 32-bit word so that the
// three-way tie-broken minimum of _align.pyx:462-476 is a plain unsigned min:
//
//   [31..26] cost, saturating at CAP=31     [25..24] priority tag (0 diag, 1 del, 2 ins)
//   [23..15] score + 64                     [14..0]  origin + 512
//
// Candidates get distinct tags, so min() over the words orders by (cost, tag) exactly like
// "mismatch if <= both, else deletion if <= insertion, else insertion".  Any cell whose cost
// reaches CAP collapses to the constant INF: such cells can never be part of a reported
// alignment (reported cost <= k <= 29) and never win a tie-break against a cell that can.
// Valid for indel_cost == 1, k <= 29, m <= 447, n <= 32255 (the host checks; everything else
// takes WideCell).  Invariant that keeps the score field from borrowing: score >= -2*cost.
// ---------------------------------------------------------------------------------------
struct Packed32 {
    typedef uint32_t T;
    static constexpr uint32_t CS = 26, PS = 24, SS = 15, SB = 64, OB = 512, CAP = 31;
    static constexpr uint32_t INF = CAP << CS;
    CG_HD static T make(long long cost, int score, int origin)
    {
        if (cost >= (long long)CAP) return INF;
        return ((uint32_t)cost << CS) | ((uint32_t)(score + (int)SB) << SS) | (uint32_t)(origin + (int)OB);
    }
    CG_HD static int cost(T w) { return (int)(w >> CS); }
    CG_HD static int score(T w) { return (int)((w >> SS) & 511u) - (int)SB; }
    CG_HD static int origin(T w) { return (int)(w & 32767u) - (int)OB; }
    CG_HD static bool cost_le(T w, int k) { return w < ((uint32_t)(k + 1) << CS); }
    CG_HD static T clamp(T x) { return x < INF ? x : INF; }
    CG_HD static T row0_free(T w) { return w + 1u; }                                  // origin += 1
    CG_HD static T row0_ins(T w, int) { return clamp(w + (1u << CS) - (2u << SS)); }  // cost+1, score-2
    CG_HD static T match(T d) { return clamp(d + (1u << SS)); }                       // score+1
    CG_HD static T mismatch(T d, T up, T left, int)
    {
        T cd = d + ((1u << CS) - (1u << SS));
        T cu = up + ((1u << CS) + (1u << PS) - (2u << SS));
        T cl = left + ((1u << CS) + (2u << PS) - (2u << SS));
        T b = cg_min(cd, cg_min(cu, cl));
        b &= ~(3u << PS);
        return clamp(b);
    }
    // Without saturation: only valid where costs cannot reach CAP -- free start in the read keeps
    // cost(i, j) <= i, so any adapter with m < CAP qualifies (locate_regs<MR <= 16, true>).
    CG_HD static T match_nc(T d) { return d + (1u << SS); }
    CG_HD static T mismatch_nc(T d, T up, T left)
    {
        T cd = d + ((1u << CS) - (1u << SS));
        T cu = up + ((1u << CS) + (1u << PS) - (2u << SS));
        T cl = left + ((1u << CS) + (2u << PS) - (2u << SS));
        T b = cg_min(cd, cg_min(cu, cl));
        return b & ~(3u << PS);
    }
};

// Exact int32 triples for everything Packed32 cannot hold (--no-indels' indel_cost=100000,
// very long reads/adapters, k > 29).
struct WideCell {
    struct T { int cost, score, origin; };
    CG_HD static T make(long long cost, int score, int origin)
    {
        T t;
        t.cost = (int)(cost > 1000000000LL ? 1000000000LL : cost);
        t.score = score; t.origin = origin;
        return t;
    }
    CG_HD static int cost(const T &w) { return w.cost; }
    CG_HD static int score(const T &w) { return w.score; }
    CG_HD static int origin(const T &w) { return w.origin; }
    CG_HD static bool cost_le(const T &w, int k) { return w.cost <= k; }
    CG_HD static T row0_free(T w) { w.origin += 1; return w; }
    CG_HD static T row0_ins(T w, int ic) { w.cost = w.cost > 1000000000 ? w.cost : w.cost + ic; w.score -= 2; return w; }
    CG_HD static T match(T d) { d.score += 1; return d; }
    CG_HD static T mismatch(const T &d, const T &up, const T &left, int ic)
    {
        int cd = d.cost + 1, cdel = up.cost > 1000000000 ? up.cost : up.cost + ic;
        int cins = left.cost > 1000000000 ? left.cost : left.cost + ic;
        T r;
        if (cd <= cdel && cd <= cins) { r.cost = cd; r.origin = d.origin; r.score = d.score - 1; }
        else if (cdel <= cins) { r.cost = cdel; r.origin = up.origin; r.score = up.score - 2; }
        else { r.cost = cins; r.origin = left.origin; r.score = left.score - 2; }
        return r;
    }
};

// Column stores: element i of this lane's DP column.
struct PackedCol {                // shared memory, lane-interleaved: conflict-free
    uint32_t *base; int stride;
    CG_HD uint32_t get(int i) const { return base[(size_t)i * stride]; }
    CG_HD void set(int i, uint32_t v) { base[(size_t)i * stride] = v; }
};
struct WideCol {                  // global scratch, lane-interleaved: coalesced
    int *base; long long stride;
    CG_HD WideCell::T get(int i) const
    {
        WideCell::T t;
        const int *q = base + (long long)(3 * i) * stride;
        t.cost = q[0]; t.score = q[stride]; t.origin = q[2 * stride];
        return t;
    }
    CG_HD void set(int i, const WideCell::T &t)
    {
        int *q = base + (long long)(3 * i) * stride;
        q[0] = t.cost; q[stride] = t.score; q[2 * stride] = t.origin;
    }
};

// ---------------------------------------------------------------------------------------
// KmerFinder.kmers_present  (_kmer_finder.pyx:170-213) -- reference-form entries
// ---------------------------------------------------------------------------------------
CG_HD bool kmers_present_core(const CgEntry *ents, int count, const uint64_t *masks64,
                              const ReadView &rv)
{
    const long long n = rv.n;
    for (int e = 0; e < count; ++e) {
        long long start = ents[e].start, stop = ents[e].stop;
        if (start < 0) { start += n; if (start < 0) start = 0; }
        else if (start > n) continue;
        if (stop < 0) { stop += n; if (stop <= 0) continue; }
        else if (stop == 0) stop = n;
        if (stop > n) stop = n;   // the reference would read past the string here (UB); clamp
        if (stop - start <= 0) continue;
        const uint64_t *mk = masks64 + 128u * (size_t)ents[e].mask_index;
        const uint64_t init = ents[e].init_mask, found = ents[e].found_mask;
        uint64_t R = 0;
        for (long long i = start; i < stop; ++i) {       // _kmer_finder.pyx:251-257
            R = ((R << 1) | init) & mk[rv.at((int)i) & 127];
            if (R & found) return true;
        }
    }
    return false;
}

// ---------------------------------------------------------------------------------------
// Aligner.locate  (_align.pyx:298-587)
// out6 = (ref_start, ref_stop, query_start, query_stop, score, errors)
// ---------------------------------------------------------------------------------------
//
// Windowed mode (cover != 0xFFFFFFFF; only for START_IN_QUERY|STOP_IN_QUERY adapters): the read
// is cut into 32 groups of (1 << gs) characters and only the groups whose bit is set in `cover`
// are run through the DP.  A maximal run of set groups starting at character j0 > 0 restarts the
// DP as if the read began there (column j0: cost i, score -2i, origin j0 -- the path that
// deletes i adapter characters at column j0).  Every cell of the true matrix with cost <= k whose
// optimal paths start at or after j0 comes out identical (restarted costs are >= the true ones
// and equal along those paths, so all tie-breaks agree); the caller guarantees via the locator
// k-mers (pigeonhole: an alignment with <= k errors contains one of the k+1 adapter chunks
// exactly) that every bottom-row cell with cost <= k, and the cells the last-column scan can
// accept, lie at least m + k columns to the right of their run's start.
// dbg_cost / dbg_score (optional, (m + 1) x (n + 1) row-major int32, pre-filled by the caller with the "not
// computed" marker): every cell the search computes is recorded -- the DPMatrix of Aligner.enable_debug()
// (_align.pyx:291-296, 385-390, 484-489).
template <class Cell, class Col>
CG_HD bool locate_core(const CgAdapter &A, const uint8_t *ref, const int32_t *ncnt,
                       const int32_t *maxcost, const uint8_t *enc, const ReadView &rv, Col &col,
                       int *out6, uint32_t cover = 0xFFFFFFFFu, int gs = 0, int32_t *dbg_cost = nullptr,
                       int32_t *dbg_score = nullptr)
{
    typedef typename Cell::T T;
    const int m = A.m, n = rv.n, k = A.k, ic = A.indel_cost;
    const bool sir = (A.flags & 1) != 0, siq = (A.flags & 2) != 0;
    const bool eir = (A.flags & 4) != 0, eiq = (A.flags & 8) != 0;
    const bool ascii = A.compare_ascii != 0;

    int max_n = n, min_n = 0;                                   // _align.pyx:346-352
    if (!siq) max_n = cg_min(n, m + k);
    if (!eiq) min_n = cg_max(0, n - m - k);

    bool have = false;                                          // _align.pyx:391-396
    int b_origin = 0, b_cost = 0, b_score = 0, b_ref_stop = m, b_q_stop = n;
    int last = 0, last_filled = 0;
    T stale = Cell::make(0, 0, 0);      // the C variable `origin` of _align.pyx:407 (see :565)
    const bool windowed = cover != 0xFFFFFFFFu;
    bool stopped = false;               // early exit (_align.pyx:531-533)
    int run_lo = min_n, run_hi = max_n; // columns run_lo+1 .. run_hi are computed
    uint32_t todo = cover;
    bool reached_end = !windowed;

    while (true) {
      if (windowed) {
        if (todo == 0) break;
        // next maximal run of set groups
        int ga = 0;
        while (!((todo >> ga) & 1u)) ++ga;
        int gb = ga;
        while (gb < 31 && ((todo >> (gb + 1)) & 1u)) ++gb;
        todo &= ~(((gb == 31 ? 0u : (1u << (gb + 1))) - 1u) & ~((1u << ga) - 1u));
        run_lo = ga << gs;
        if (run_lo > 0 && run_lo >= n) break;
        const long long hi_ll = ((long long)(gb + 1)) << gs;
        run_hi = hi_ll > n ? n : (int)hi_ll;
        reached_end = run_hi == n;
      }
      if (run_lo == min_n) {
        for (int i = 0; i <= m; ++i) {                          // _align.pyx:364-383
            long long c; int s, o;
            if (!sir && !siq) { s = -2 * i; c = (long long)cg_max(i, min_n) * ic; o = 0; }
            else if (sir && !siq) { s = 0; c = (long long)min_n * ic; o = cg_min(0, min_n - i); }
            else if (!sir && siq) { s = -2 * i; c = (long long)i * ic; o = cg_max(0, min_n - i); }
            else { s = 0; c = (long long)cg_min(i, min_n) * ic; o = min_n - i; }
            col.set(i, Cell::make(c, s, o));
            if (dbg_cost) {
                dbg_cost[(size_t)i * (n + 1) + min_n] = Cell::cost(col.get(i));
                dbg_score[(size_t)i * (n + 1) + min_n] = s;
            }
        }
        last = sir ? m : cg_min(m, k + 1);                      // _align.pyx:399-401
      } else {
        // restart inside the read: column run_lo of a read that begins at character run_lo
        for (int i = 0; i <= m; ++i) col.set(i, Cell::make((long long)i * ic, -2 * i, run_lo));
        last = cg_min(m, k + 1);
      }

    for (int j = run_lo + 1; j <= run_hi; ++j) {                // _align.pyx:433
        const uint8_t qc = enc[rv.at(j - 1)];
        T diag = col.get(0);
        T w0 = siq ? Cell::row0_free(diag) : Cell::row0_ins(diag, ic);   // _align.pyx:438-440
        col.set(0, w0);
        T up = w0;
        int lastok = Cell::cost_le(w0, k) ? 0 : -1;
        for (int i = 1; i <= last; ++i) {                       // _align.pyx:441-483
            const T left = col.get(i);
            const uint8_t rc = ref[i - 1];
            const bool eq = ascii ? (rc == qc) : ((rc & qc) != 0);
            const T nw = eq ? Cell::match(diag) : Cell::mismatch(diag, up, left, ic);
            col.set(i, nw);
            if (Cell::cost_le(nw, k)) lastok = i;
            diag = left;
            up = nw;
        }
        if (last >= 1) stale = up;
        last_filled = last;                                     // _align.pyx:484
        if (dbg_cost) {
            for (int i = 0; i <= last; ++i) {
                const T w = col.get(i);
                dbg_cost[(size_t)i * (n + 1) + j] = Cell::cost(w);
                dbg_score[(size_t)i * (n + 1) + j] = Cell::score(w);
            }
        }
        // `while last >= 0 and column[last].cost > k: last -= 1` == lastok   (_align.pyx:490-491)
        if (lastok < m) {
            last = lastok + 1;                                  // _align.pyx:494-495
        } else if (eiq) {                                       // _align.pyx:496-533
            stale = up;
            const int cost = Cell::cost(up), score = Cell::score(up), origin = Cell::origin(up);
            const int length = m + cg_min(origin, 0);
            int eff = length;
            if (A.wildcard_ref) eff = (length < m) ? length - (ncnt[m] - ncnt[m - length]) : A.effective_length;
            const bool ok = length >= A.min_overlap && cost <= maxcost[eff];
            const int best_len = m + cg_min(b_origin, 0);
            if (ok && (!have || (origin <= b_origin + m / 2 && score > b_score) ||
                       (length > best_len && score > b_score))) {
                have = true;
                b_score = score; b_cost = cost; b_origin = origin; b_ref_stop = m; b_q_stop = j;
                if (cost == 0 && origin >= 0) { stopped = true; break; }   // _align.pyx:531-533
            }
        }
    }
      if (stopped || !windowed) break;
    }

    if (max_n == n && (reached_end || stopped)) {               // _align.pyx:536-572
        const int first_i = eir ? 0 : m;
        const int origin_var = Cell::origin(stale);
        for (int i = last_filled; i >= first_i; --i) {
            const T w = col.get(i);
            if (!Cell::cost_le(w, k)) continue;   // cost > k can never satisfy cost <= floor(eff*rate) <= k
            const int o = Cell::origin(w), cost = Cell::cost(w), score = Cell::score(w);
            const int length = i + cg_min(o, 0);
            int eff = length;
            if (A.wildcard_ref) {
                if (length < m) eff = length - (ncnt[i] - ncnt[-cg_min(o, 0)]);
                else eff = A.effective_length;
            }
            const bool ok = length >= A.min_overlap && cost <= maxcost[eff];
            const int best_len = b_ref_stop + cg_min(b_origin, 0);
            if (ok && (!have || (origin_var <= b_origin + m / 2 && score > b_score) ||
                       (length > best_len && score > b_score))) {
                have = true;
                b_score = score; b_cost = cost; b_origin = o; b_ref_stop = i; b_q_stop = n;
            }
        }
    }
    if (!have) return false;                                    // _align.pyx:573-577
    out6[0] = b_origin >= 0 ? 0 : -b_origin;                    // _align.pyx:579-587
    out6[1] = b_ref_stop;
    out6[2] = b_origin >= 0 ? b_origin : 0;
    out6[3] = b_q_stop;
    out6[4] = b_score;
    out6[5] = b_cost;
    return true;
}

// ---------------------------------------------------------------------------------------
// PrefixComparer.locate / SuffixComparer.locate  (_align.pyx:651-714)
// `ref` holds the encoded adapter in its natural orientation for both.
// ---------------------------------------------------------------------------------------
CG_HD bool compare_core(const CgAdapter &A, const uint8_t *ref, const uint8_t *enc,
                        const ReadView &rv, int *out6)
{
    const int m = A.m, n = rv.n;
    const int length = cg_min(m, n);                            // _align.pyx:667
    const bool ascii = A.compare_ascii != 0, suffix = A.kind == CGK_KIND_SUFFIX;
    int errors = 0;
    for (int i = 0; i < length; ++i) {                          // _align.pyx:681-688
        const uint8_t rc = suffix ? ref[m - 1 - i] : ref[i];
        const uint8_t qc = enc[suffix ? rv.at(n - 1 - i) : rv.at(i)];
        errors += ascii ? (rc != qc) : ((rc & qc) == 0);
    }
    if (errors > A.max_k_cmp || length < A.min_overlap) return false;   // _align.pyx:690-691
    const int score = (length - errors) - errors;               // _align.pyx:692
    if (suffix) { out6[0] = m - length; out6[1] = m; out6[2] = n - length; out6[3] = n; }  // :714
    else { out6[0] = 0; out6[1] = length; out6[2] = 0; out6[3] = length; }                  // :693
    out6[4] = score; out6[5] = errors;
    return true;
}

// ---------------------------------------------------------------------------------------
// quality_trim_index  (qualtrim.pyx:22-73)
// ---------------------------------------------------------------------------------------
CG_HD void quality_trim_core(const uint8_t *q, int n, int cutoff_front, int cutoff_back, int base,
                             int *start_out, int *stop_out)
{
    int s = 0, best = 0, start = 0, stop = n;
    for (int i = 0; i < n; ++i) {                               // qualtrim.pyx:51-59
        s += cutoff_front - ((int)(signed char)q[i] - base);
        if (s < 0) break;
        if (s > best) { best = s; start = i + 1; }
    }
    best = 0; s = 0;
    for (int i = n - 1; i >= 0; --i) {                          // qualtrim.pyx:62-70
        s += cutoff_back - ((int)(signed char)q[i] - base);
        if (s < 0) break;
        if (s > best) { best = s; stop = i; }
    }
    if (start >= stop) { start = 0; stop = 0; }                 // qualtrim.pyx:71-72
    *start_out = start; *stop_out = stop;
}

// nextseq_trim_index (qualtrim.pyx:76-117): the 3' pass with every 'G' counted as quality cutoff - 1
CG_HD int nextseq_trim_core(const uint8_t *seq, const uint8_t *q, int n, int cutoff, int base)
{
    int s = 0, max_qual = 0, max_i = n;
    for (int i = n - 1; i >= 0; --i) {
        int v = (int)(signed char)q[i] - base;
        if (seq[i] == 'G') v = cutoff - 1;
        s += cutoff - v;
        if (s < 0) break;
        if (s > max_qual) { max_qual = s; max_i = i; }
    }
    return max_i;
}

// poly_a_trim_index (qualtrim.pyx:120-169)
CG_HD int poly_a_trim_core(const uint8_t *seq, int n, int revcomp)
{
    int best_score = 0, score = 0, errors = 0, best_index;
    if (revcomp) {
        best_index = 0;
        for (int i = 0; i < n; ++i) {
            if (seq[i] == 'T') score += 1; else { score -= 2; errors += 1; }
            if (score > best_score && errors * 5 <= i + 1) { best_score = score; best_index = i + 1; }
        }
        if (best_index < 3) best_index = 0;
    } else {
        best_index = n;
        for (int i = n - 1; i >= 0; --i) {
            if (seq[i] == 'A') score += 1; else { score -= 2; errors += 1; }
            if (score > best_score && errors * 5 <= n - i) { best_score = score; best_index = i; }
        }
        if (best_index > n - 3) best_index = n;
    }
    return best_index;
}

// expected_errors (qualtrim.pyx:172-197, expected_errors.h:95-140): FP64 sum of table[q - base] in the
// reference's order -- four accumulators over groups of four, the tail into the first, then
// ((e0 + e1) + e2) + e3 -- so the double is bit-identical.  -1.0 = a character outside [base, 126].
// `table` = 256 doubles, table[q] = 10^(-q/10) (cg_build_phred_table).
// cap (ZeroCapper, modifiers.py:806-822): every character below it counts as the cap itself; 0 = as they are.
CG_HD double expected_errors_core(const uint8_t *q, int n, int base, const double *table, int cap = 0)
{
    double e0 = 0.0, e1 = 0.0, e2 = 0.0, e3 = 0.0;
    const uint8_t b = (uint8_t)base, max_phred = (uint8_t)(126 - base), c = (uint8_t)cap;
    auto at = [&](int i) -> uint8_t { return q[i] < c ? c : q[i]; };
    int i = 0;
    for (; i + 3 < n; i += 4) {
        const uint8_t p0 = (uint8_t)(at(i) - b), p1 = (uint8_t)(at(i + 1) - b);
        const uint8_t p2 = (uint8_t)(at(i + 2) - b), p3 = (uint8_t)(at(i + 3) - b);
        if (p0 > max_phred || p1 > max_phred || p2 > max_phred || p3 > max_phred) return -1.0;
        e0 += table[p0]; e1 += table[p1]; e2 += table[p2]; e3 += table[p3];
    }
    for (; i < n; ++i) {
        const uint8_t ph = (uint8_t)(at(i) - b);
        if (ph > max_phred) return -1.0;
        e0 += table[ph];
    }
    return e0 + e1 + e2 + e3;
}

// The quality-driven modifiers in front of the adapter search, fused: NextseqQualityTrimmer
// (modifiers.py:825-837) cuts the 3' end first, then QualityTrimmer (modifiers.py:840-858) works on
// what is left -- the order cutadapt builds its modifier list in (cli.py:940-953).
//   flags  bit 0: quality_trim_index, bit 1: nextseq_trim_index
//   qbase  quality base in bits 0..7, NextSeq cutoff (signed) in bits 8..31
// Result: the searched interval [*s, *e) of the read.
CG_HD void pre_trim_core(const uint8_t *seq, const uint8_t *qual, int n, int flags, int cutoff_front,
                         int cutoff_back, int qbase, int *s, int *e)
{
    const int base = qbase & 255;
    int stop = n;
    *s = 0;
    if (flags & 2) stop = nextseq_trim_core(seq, qual, n, qbase >> 8, base);
    *e = stop;
    if (flags & 1) quality_trim_core(qual, stop, cutoff_front, cutoff_back, base, s, e);
}

// ---------------------------------------------------------------------------------------
// Fused scan stage of the two-phase kernel.
//
// The host re-packs the KmerFinder entries of the adapter into 32-bit shift-and words by window
// type (whole read / suffix / prefix) and adds the "locator" chunks (the k+1 pieces of the whole
// adapter).  One pass per word answers both questions at once:
//   * KmerFinder.kmers_present (bit-for-bit the reference's verdict, _kmer_finder.pyx:170-213):
//     any k-mer of any entry found inside that entry's window;
//   * where locator chunks end, at a granularity of (1 << gs) characters, as a 32-bit group mask.
// ---------------------------------------------------------------------------------------
struct ScanOut {
    bool pass;
    uint32_t hits;   // bit g: a locator chunk ends in characters [g << gs, (g+1) << gs)
    uint32_t rs0, rs1;   // shift-and state of the first locator word at the start of the first two
                         // hit groups: phase B resumes the scan there to get exact end positions
    uint32_t bad;        // OR of the characters the first whole-read word consumed (bit 7 of any byte set
                         // = non-ASCII input); only meaningful if scan_checks_ascii(words, n_words)
};

// true if scan_core's first word walks the entire searched sequence, so that ScanOut::bad covers it
CG_HD bool scan_checks_ascii(const CgScanWord *words, int n_words)
{
    return n_words > 0 && words[0].type == CG_SCAN_WHOLE;
}

CG_HD int scan_group_shift(int n)
{
    int gs = 4;
    while ((n >> gs) >= 32) ++gs;
    return gs;
}

// REV selects the scan direction at compile time so that character addresses are base + immediate.
// The mask tables have 256 entries (the upper half is zero), so the loaded byte indexes them directly.
// byte `i` (0 = least significant) of a word, zero-extended (SASS PRMT: one instruction, and the table
// address is then one LEA instead of shift + mask + add)
CG_HD uint32_t cg_byte(uint32_t word, int i)
{
#if defined(__CUDA_ARCH__)
    return __byte_perm(word, 0u, 0x4440u | (uint32_t)i);
#else
    return (word >> (8 * i)) & 255u;
#endif
}

template <bool REV>
CG_HD ScanOut scan_core_dir(const CgScanWord *words, int n_words, const uint8_t *pool, const uint8_t *first,
                            int n, int gs, bool always_pass)
{
    // `first` is the first character in scan order; character i is first[REV ? -i : i]
    ScanOut out; out.pass = always_pass; out.hits = 0; out.rs0 = 0; out.rs1 = 0; out.bad = 0;
    // the saved states are only meaningful when a single word carries all locator chunks
    int n_loc = 0;
    for (int w = 0; w < n_words; ++w) n_loc += (words[w].type == CG_SCAN_WHOLE && words[w].loc_found) ? 1 : 0;
    for (int w = 0; w < n_words; ++w) {
        const CgScanWord &W = words[w];
        const uint32_t *mask = (const uint32_t *)(pool + W.mask_off);
        if (W.type == CG_SCAN_WHOLE) {
            const uint32_t init = W.init, locf = W.loc_found;
            uint32_t R = 0, seen = 0;
            const uint8_t *q = first;
            if (locf) {
                const bool stash = n_loc == 1;
                int nh = 0, p0 = 0;
                if (gs == 4) {                                   // reads up to 511 characters
                    // 16 characters per step, fetched as aligned 32-bit words (4x fewer shared-memory
                    // wavefronts than byte loads; the shared-memory pipe is what limits this loop).
                    // Forward: the unaligned word at q; reverse: the unaligned word at q - 3.
                    // (pointer arithmetic on q itself, not on an integer copy, keeps the shared-memory
                    // address space visible to the compiler: LDS, not generic loads)
                    const uint8_t *uq = REV ? q - 3 : q;
                    const uint32_t mis = (uint32_t)((uintptr_t)uq & 3u);
                    const uint32_t sh = mis * 8u;
                    const uint32_t *wp = (const uint32_t *)(uq - mis);
                    uint32_t carry = (p0 + 16 <= n) ? (REV ? wp[1] : wp[0]) : 0u;
                    for (; p0 + 16 <= n; p0 += 16) {
                        const uint32_t r_start = R;
                        uint32_t g = 0;
                        uint32_t x[4];
                        if (!REV) {
                            const uint32_t w1 = wp[1], w2 = wp[2], w3 = wp[3], w4 = wp[4];
                            x[0] = cg_funnel_r(carry, w1, sh); x[1] = cg_funnel_r(w1, w2, sh);
                            x[2] = cg_funnel_r(w2, w3, sh); x[3] = cg_funnel_r(w3, w4, sh);
                            carry = w4; wp += 4;
                        } else {
                            const uint32_t w0 = wp[0], m1 = wp[-1], m2 = wp[-2], m3 = wp[-3];
                            x[0] = cg_funnel_r(w0, carry, sh); x[1] = cg_funnel_r(m1, w0, sh);
                            x[2] = cg_funnel_r(m2, m1, sh); x[3] = cg_funnel_r(m3, m2, sh);
                            carry = m3; wp -= 4;
                        }
                        if (w == 0) out.bad |= x[0] | x[1] | x[2] | x[3];
#pragma unroll
                        for (int i = 0; i < 16; ++i) {
                            const uint32_t word = x[i >> 2];
                            const uint32_t c = cg_byte(word, REV ? 3 - (i & 3) : (i & 3));
                            R = ((R << 1) | init) & mask[c];
                            g |= R;
                        }
                        q += REV ? -16 : 16;
                        seen |= g;
                        const bool hg = (g & locf) != 0;
                        out.hits |= hg ? (1u << (p0 >> 4)) : 0u;
                        out.rs0 = (hg && stash && nh == 0) ? r_start : out.rs0;
                        out.rs1 = (hg && stash && nh == 1) ? r_start : out.rs1;
                        nh += hg ? 1 : 0;
                    }
                }
                const int G = 1 << gs;
                for (; p0 < n; p0 += G) {
                    const int cnt = cg_min(n - p0, G);
                    const uint32_t r_start = R;
                    uint32_t g = 0;
                    for (int i = 0; i < cnt; ++i) {
                        const uint32_t c = q[REV ? -i : i];
                        if (w == 0) out.bad |= c;
                        R = ((R << 1) | init) & mask[c];
                        g |= R;
                    }
                    q += REV ? -cnt : cnt;
                    seen |= g;
                    const bool hg = (g & locf) != 0;
                    out.hits |= hg ? (1u << (p0 >> gs)) : 0u;
                    out.rs0 = (hg && stash && nh == 0) ? r_start : out.rs0;
                    out.rs1 = (hg && stash && nh == 1) ? r_start : out.rs1;
                    nh += hg ? 1 : 0;
                }
            } else {
                int p = 0;
                for (; p + 8 <= n; p += 8) {
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const uint32_t c = q[REV ? -i : i];
                        if (w == 0) out.bad |= c;
                        R = ((R << 1) | init) & mask[c];
                        seen |= R;
                    }
                    q += REV ? -8 : 8;
                }
                for (; p < n; ++p) {
                    const uint32_t c = *q;
                    if (w == 0) out.bad |= c;
                    R = ((R << 1) | init) & mask[c];
                    seen |= R;
                    q += REV ? -1 : 1;
                }
            }
            if (seen & W.pass_found) out.pass = true;
        } else if (W.type == CG_SCAN_SUFFIX) {
            const uint32_t *tab = (const uint32_t *)(pool + W.pos_off);   // {init, found}[span + 1]
            uint32_t R = 0, seen = 0;
            const int p_lo = cg_max(0, n - (int)W.span);
            const uint8_t *q = first + (REV ? -p_lo : p_lo);
            for (int d = n - p_lo; d >= 1; --d) {
                R = ((R << 1) | tab[2 * d]) & mask[*q];
                seen |= R & tab[2 * d + 1];
                q += REV ? -1 : 1;
            }
            if (seen & W.pass_found) out.pass = true;
        } else {
            const uint32_t *tab = (const uint32_t *)(pool + W.pos_off);   // {init, found}[span]
            uint32_t R = 0, seen = 0;
            const int stop = cg_min(n, (int)W.span);
            const uint8_t *q = first;
            for (int p = 0; p < stop; ++p) {
                R = ((R << 1) | tab[2 * p]) & mask[*q];
                seen |= R & tab[2 * p + 1];
                q += REV ? -1 : 1;
            }
            if (seen & W.pass_found) out.pass = true;
        }
    }
    return out;
}

CG_HD ScanOut scan_core(const CgScanWord *words, int n_words, const uint8_t *pool, const ReadView &rv,
                        int gs, bool always_pass)
{
    if (rv.rev) return scan_core_dir<true>(words, n_words, pool, rv.p + (rv.n - 1), rv.n, gs, always_pass);
    return scan_core_dir<false>(words, n_words, pool, rv.p, rv.n, gs, always_pass);
}

// ---------------------------------------------------------------------------------------
// Bit-plane scan (split pipeline, first stage for plain A/C/G/T adapters).
//
// The searched window of a read (n <= 32 W characters) becomes four W-word bit planes -- bit i of plane X
// is set iff character i is X or x -- and every k-mer of the scan program is matched against all
// positions at once: ends(kmer) = AND_t (plane[kmer[t]] << (len - 1 - t)), 1.5 instructions per k-mer
// character and 32 positions instead of ~7 per read character of the shift-and scan.  The window is
// RIGHT-aligned in the planes (its last character is bit 32 W - 1), so that the suffix windows of the
// KmerFinder entries of a 3' adapter (_kmer_finder.pyx:188-204 with start < 0) are the last word(s).
//
// Planes come from bits 1 and 2 of the ASCII code alone (A 00, C 01, T 10, G 11; case-insensitive),
// four characters per dp4a: sum_i ((word >> (8 i + 1)) & 1) << i.  Any other byte aliases one of the four
// letters, so the planes give a SUPERSET of the true k-mer occurrences:
//   * no occurrence of any k-mer in the planes  =>  KmerFinder.kmers_present is False  =>  no match;
//   * an exact occurrence of the whole adapter found in the planes is confirmed by comparing the read
//     bytes with the adapter; if it is also the leftmost place any locator chunk points at, the
//     reference returns (0, m, s0, s0 + m, m, 0) (proof below) -- no DP;
//   * every other read goes to the exact path (cg_list_kernel<plan> re-scans it with scan_core).
//
// Exact-occurrence rule (adapters without START_IN_REFERENCE, k <= m/2, unit costs, plain A/C/G/T).
// Let s0 be the start of an exact occurrence and assume no locator chunk occurs anywhere in the read at
// a place that implies an adapter start < s0.  Column s0 + m of the DP has bottom cell (0, m, s0): a
// cost-0 path is the diagonal, so it is unique.  A bottom-row candidate accepted at an earlier column has
// cost >= 1 (cost 0 would be an exact occurrence with a smaller start, whose chunks contradict the
// assumption), hence score < m, and by the pigeonhole principle it contains a chunk exactly; its start
// is within k of the start that chunk implies, i.e. >= s0 - k >= s0 - m/2.  So at column s0 + m the
// replacement test of _align.pyx:521-525 succeeds (origin s0 <= best.origin + m/2 and score m > best.score)
// and the search stops there (_align.pyx:531-533); the last-column scan that follows cannot beat score m.
// ---------------------------------------------------------------------------------------
CG_HD uint32_t cg_dp4a(uint32_t a, uint32_t b, uint32_t c)
{
#if defined(__CUDA_ARCH__)
    return __dp4a(a, b, c);
#else
    for (int i = 0; i < 4; ++i) c += ((a >> (8 * i)) & 255u) * ((b >> (8 * i)) & 255u);
    return c;
#endif
}
CG_HD uint32_t cg_funnel_l(uint32_t lo, uint32_t hi, uint32_t s)   // (hi:lo) << s, upper word; s in 0..31
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(lo, hi, s);
#else
    return s ? (hi << s) | (lo >> (32 - s)) : hi;
#endif
}
CG_HD uint32_t cg_funnel_rb(uint32_t lo, uint32_t hi, uint32_t s)  // (hi:lo) >> s, lower word; s in 0..31
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, s);
#else
    return s ? (lo >> s) | (hi << (32 - s)) : lo;
#endif
}

struct PlaneOut {
    int cls;         // 0: no match, 1: exact occurrence at s0, 2: undecided (exact path)
    int s0;
    uint32_t bad;    // OR of the window's bytes (bit 7 of any byte set = non-ASCII input)
    // cls 2: what the plan stage needs to go on without scanning the read again (plan_runs_planes)
    uint32_t M[8];   // bit e of word b: a locator chunk occurs where the whole adapter would end at plane index 32 b + e
    int end_hit;     // a chunk occurs so close to the end of the window that the adapter would reach beyond it
    int no_end;      // the last-column scan cannot accept anything: the plan needs no end window
};
#define CG_PLANE_NONE 0
#define CG_PLANE_EXACT 1
#define CG_PLANE_SLOW 2
#define CG_PLANE_OVERLAP 3   // the read ends with the adapter's first s0 characters and nothing else can match

// x <<= s  (multi-word, s in 0..63); returns the bits shifted out at the top (non-zero = some were)
template <int W>
CG_HD uint32_t plane_shl(uint32_t (&x)[W], uint32_t s)
{
    uint32_t lost = 0;
    if (s >= 32) {
        lost = x[W - 1];
#pragma unroll
        for (int b = W - 1; b >= 1; --b) x[b] = x[b - 1];
        x[0] = 0;
        s -= 32;
    }
    lost |= cg_funnel_l(x[W - 1], 0u, s);          // the top s bits of the last word
#pragma unroll
    for (int b = W - 1; b >= 1; --b) x[b] = cg_funnel_l(x[b - 1], x[b], s);
    x[0] <<= s;
    return lost;
}

// The stage is written as a state plus three operations -- load, chain step, emit -- and a decision, so
// that the same code serves the interpreter of the op list in the adapter blob (RuntimePlaneProg: any
// adapter, precompiled) and a program spelled out as a sequence of calls with literal arguments, which the
// compiler folds into straight-line code (cg_jit.cpp compiles that per adapter set with NVRTC).
template <int W>
struct PlaneState {
    uint32_t PA[W], PC[W], PT[W], PG[W];   // bit i: character i of the (right-aligned) window is A / C / T / G
    uint32_t acc[W];                       // ends of the chain's text so far
    uint32_t M[W], E[W];                   // locator hits / all chunks, by the end of the WHOLE adapter
    bool pass, anyhit, end_hit;
    bool guard;                            // a guard piece occurs at the end (see CG_PLANE_GUARD)
    int ovl;                               // longest exact overlap (adapter prefix = read suffix) the planes see
};

// `base` = address of plane index 0 (window end - 32 W); the bytes [base - 3, base + 32 W + 4) must be readable.
// Returns the OR of the window's bytes.
template <int W>
CG_HD uint32_t plane_load(PlaneState<W> &st, const uint8_t *base, int off0)
{
    uint32_t LO[W], HI[W];
    const uint32_t mis = (uint32_t)((uintptr_t)base & 3u);
    const uint32_t sh = 8u * mis;
    const uint32_t *wp = (const uint32_t *)(base - mis);
    uint32_t carry = wp[0];
    uint32_t bad = 0;
#pragma unroll
    for (int b = 0; b < W; ++b) {
        uint32_t x[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t nxt = wp[8 * b + j + 1];
            x[j] = cg_funnel_rb(carry, nxt, sh);
            carry = nxt;
        }
        if (off0 > 32 * b) {                     // leading block(s): blank the bytes in front of the window
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int fv = off0 - (32 * b + 4 * j);          // first valid byte of this word
                const uint32_t keep = fv <= 0 ? 0xFFFFFFFFu : (fv >= 4 ? 0u : (0xFFFFFFFFu << (8 * fv)));
                x[j] &= keep;
            }
        }
        uint32_t lo = 0, hi = 0;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const uint32_t a = x[2 * p], c = x[2 * p + 1];
            bad |= a | c;
            uint32_t pl = cg_dp4a(a & 0x02020202u, 0x08040201u, 0u);
            pl = cg_dp4a(c & 0x02020202u, 0x80402010u, pl);      // 2 x (8 plane bits)
            uint32_t ph = cg_dp4a(a & 0x04040404u, 0x08040201u, 0u);
            ph = cg_dp4a(c & 0x04040404u, 0x80402010u, ph);      // 4 x (8 plane bits)
            lo += p == 0 ? (pl >> 1) : (pl << (8 * p - 1));
            hi += p == 0 ? (ph >> 2) : (ph << (8 * p - 2));
        }
        LO[b] = lo; HI[b] = hi;
    }
    // planes of the four letters, blanked in front of the window
#pragma unroll
    for (int b = 0; b < W; ++b) {
        const int fv = off0 - 32 * b;
        const uint32_t len = fv <= 0 ? 0xFFFFFFFFu : (fv >= 32 ? 0u : (0xFFFFFFFFu << fv));
        st.PA[b] = ~LO[b] & ~HI[b] & len;
        st.PC[b] = LO[b] & ~HI[b] & len;
        st.PT[b] = ~LO[b] & HI[b] & len;
        st.PG[b] = LO[b] & HI[b] & len;
    }
#if defined(__CUDA_ARCH__)
    // keep the four planes in registers: left alone, ptxas re-derives them from LO / HI / len inside every
    // chain step (two LOP3 per word instead of one)
#pragma unroll
    for (int b = 0; b < W; ++b)
        asm volatile("" : "+r"(st.PA[b]), "+r"(st.PC[b]), "+r"(st.PT[b]), "+r"(st.PG[b]));
#endif
#pragma unroll
    for (int b = 0; b < W; ++b) { st.acc[b] = 0; st.M[b] = 0; st.E[b] = 0xFFFFFFFFu; }
    st.pass = false; st.anyhit = false; st.end_hit = false;
    st.guard = false; st.ovl = 0;
    return bad;
}

// one chain step: acc = plane (first character of a chain) or (acc << 1) & plane
#ifndef CG_CHAIN_IMAD
#define CG_CHAIN_IMAD 0             // words of the accumulator whose shift runs on the multiply pipe (bit b = word b);
                                    // measured: 0xFF was SLOWER than funnel shifts (IMAD.WIDE issues at half
                                    // rate), so the default keeps the shifts on the ALU pipe
#endif
template <int W>
CG_HD void plane_chain_apply(uint32_t (&acc)[W], const uint32_t (&P)[W], bool first)
{
    if (first) {
#pragma unroll
        for (int b = 0; b < W; ++b) acc[b] = P[b];
    } else {
#if defined(__CUDA_ARCH__) && CG_CHAIN_IMAD
        // The first stage is bound by the ALU pipe (LOP3 / SHF / compares issue every other cycle per scheduler, the
        // multiply pipe idles): for the words in CG_CHAIN_IMAD the shift is a widening multiply by two -- one
        // IMAD.WIDE.U32 on the other pipe yields x << 1 AND x >> 31 -- and the carry joins in the LOP3 that was needed
        // for the AND anyway: (lo | carry_in) & plane.
        uint32_t lo[W], hi[W];
#pragma unroll
        for (int b = 0; b < W; ++b) {
            if ((CG_CHAIN_IMAD >> b) & 1 || (b + 1 < W && ((CG_CHAIN_IMAD >> (b + 1)) & 1))) {
                unsigned long long t;
                asm("mul.wide.u32 %0, %1, 2;" : "=l"(t) : "r"(acc[b]));
                lo[b] = (uint32_t)t;
                hi[b] = (uint32_t)(t >> 32);
            }
        }
#pragma unroll
        for (int b = W - 1; b >= 1; --b) {
            if ((CG_CHAIN_IMAD >> b) & 1) acc[b] = (lo[b] | hi[b - 1]) & P[b];
            else acc[b] = cg_funnel_l(acc[b - 1], acc[b], 1) & P[b];
        }
        acc[0] = ((CG_CHAIN_IMAD & 1) ? lo[0] : (acc[0] << 1)) & P[0];
#else
#pragma unroll
        for (int b = W - 1; b >= 1; --b) acc[b] = cg_funnel_l(acc[b - 1], acc[b], 1) & P[b];
        acc[0] = (acc[0] << 1) & P[0];
#endif
    }
}
template <int W>
CG_HD void plane_chain_step(PlaneState<W> &st, uint32_t code, bool first)
{
    // (branches, not a reference picked by `code`: the planes must stay in registers)
    if (code == 0) plane_chain_apply<W>(st.acc, st.PA, first);
    else if (code == 1) plane_chain_apply<W>(st.acc, st.PC, first);
    else if (code == 2) plane_chain_apply<W>(st.acc, st.PT, first);
    else plane_chain_apply<W>(st.acc, st.PG, first);
}

// A k-mer of `len` characters ends with the step just done: acc has bit e set iff it ends at plane index e
// (occurrences reaching in front of the window are impossible: the planes are blank there).
//   type/window : CG_SCAN_SUFFIX: the occurrence must start inside the last `window` (<= 64) characters, i.e.
//                 e >= 32 W - window + len - 1, which lies in the last two words
//   flags       : CG_PLANE_PASS / CG_PLANE_LOC;  shift = m - (adapter offset at which a locator chunk ends)
template <int W>
CG_HD void plane_emit(PlaneState<W> &st, int len, int type, int flags, int shift, int window)
{
    if (type == CG_SCAN_OVERLAP) {                   // does the window END with these `len` characters?
        if ((st.acc[W - 1] >> 31) && len > st.ovl) st.ovl = len;
        return;
    }
    uint32_t x[W];
#pragma unroll
    for (int b = 0; b < W; ++b) x[b] = st.acc[b];
    uint32_t any = 0;
    if (type == CG_SCAN_SUFFIX) {
        const int e_min = 32 * W - window + len - 1;
#pragma unroll
        for (int b = 0; b < W; ++b) {
            const int fv = e_min - 32 * b;
            x[b] &= fv <= 0 ? 0xFFFFFFFFu : (fv >= 32 ? 0u : (0xFFFFFFFFu << fv));
        }
#pragma unroll
        for (int b = (W >= 3 ? W - 3 : 0); b < W; ++b) any |= x[b];      // windows of <= 64 characters + a k-mer
    } else {
#pragma unroll
        for (int b = 0; b < W; ++b) any |= x[b];
    }
    if ((flags & (int)CG_PLANE_GUARD) && any) st.guard = true;
    if ((flags & (int)CG_PLANE_PASS) && any) st.pass = true;
    if (flags & (int)CG_PLANE_LOC) {
        if (any) st.anyhit = true;
        if (plane_shl<W>(x, (uint32_t)shift)) st.end_hit = true;
#pragma unroll
        for (int b = 0; b < W; ++b) { st.M[b] |= x[b]; st.E[b] &= x[b]; }
    }
}

// The interpreter of the op list in the adapter blob (cg_types.h: CG_PLANE_OP_*, CgPlaneEmit).
struct RuntimePlaneProg {
    // do the m characters at w spell the adapter (either case)?
    CG_HD static bool same_adapter(const uint8_t *w, const uint8_t *ref, int m)
    {
        bool same = true;
        for (int i = 0; i < m; ++i) same = same && ((w[i] & 0xDFu) == ref[i]);
        return same;
    }
    CG_HD static int adapter_length(int m) { return m; }
    CG_HD static unsigned long long overlap_ok(unsigned long long from_blob) { return from_blob; }
    CG_HD static int remove_kind(int from_blob) { return from_blob; }     // CgAdapter::remove
    template <int W>
    CG_HD static void run(PlaneState<W> &st, const uint32_t *ops, int n_ops, int m)
    {
        const CgPlaneEmit *emits = (const CgPlaneEmit *)((const uint8_t *)ops + (((size_t)n_ops * 4 + 7) & ~(size_t)7));
        for (int i = 0; i < n_ops; ++i) {
            const uint32_t op = ops[i];
            plane_chain_step<W>(st, op & 3u, (op & CG_PLANE_OP_NEW) != 0);
            uint32_t em = op >> 8;
            while (em) {
                const CgPlaneEmit K = emits[(em & 255u) - 1u];
                em >>= 8;
                plane_emit<W>(st, (int)K.len, (int)K.type, (int)K.flags, m - (int)K.bend, (int)K.window);
            }
        }
    }
};

// What the planes settle, and what they hand on (see the head of this section for the rules).
//   exact_ok : plane_flags bit 0;  m, ref: the adapter;  base / off0 / n as in plane_load
template <int W, class Prog>
CG_HD void plane_decide(const PlaneState<W> &st, int plane_flags, unsigned long long overlap_ok, int m, const uint8_t *ref,
                        const uint8_t *base, int off0, int n, bool always_pass, PlaneOut &out)
{
    const bool exact_ok = (plane_flags & 1) != 0, end_ok = (plane_flags & 2) != 0;
    out.cls = CG_PLANE_SLOW; out.s0 = 0; out.end_hit = st.end_hit ? 1 : 0; out.no_end = 0;
    if (!st.pass && !always_pass) { out.cls = CG_PLANE_NONE; return; }   // no k-mer even in the superset: kmers_present is False
    if (exact_ok && st.anyhit) {
        // the leftmost adapter end any chunk points at (a chunk whose implied end lies beyond the window is
        // shifted out: it implies a larger start than anything that remains)
        bool found = false, ex = false;
        int low = 0;
#pragma unroll
        for (int b = 0; b < W; ++b) {
            if (!found && st.M[b]) {
                found = true;
                const int bit = cg_ctz(st.M[b]);
                low = 32 * b + bit;
                ex = ((st.E[b] >> bit) & 1u) != 0;
            }
        }
        const int s0 = low - (m - 1) - off0;
        if (found && ex && s0 >= 0 && s0 + m <= n) {
            if (Prog::same_adapter(base + (low - (m - 1)), ref, m)) { out.cls = CG_PLANE_EXACT; out.s0 = s0; return; }
        }
    }
    // End analysis (3' adapters, program with guard pieces and overlap emits; cg_setbuild.cpp build_plane_program).
    // No guard piece at the end => every acceptable cell of the last column is an exact overlap of one of the
    // emitted lengths, and the scan takes the longest (a shorter one scores less, _align.pyx:561-570).
    if (end_ok && !st.guard && !st.end_hit) {
        if (!st.anyhit) {
            // no locator chunk anywhere: no bottom-row candidate either, only the last column can match
            if (st.ovl == 0) { out.cls = CG_PLANE_NONE; return; }
            if (st.ovl <= n && ((overlap_ok >> st.ovl) & 1ULL) && Prog::same_adapter(base + 32 * W - st.ovl, ref, st.ovl)) {
                // (kmers_present is True for such a read: the overlap itself holds a k-mer in its window)
                out.cls = CG_PLANE_OVERLAP; out.s0 = st.ovl; return;
            }
        } else if (st.ovl == 0) {
            out.no_end = 1;                       // hits to examine, but the end of the read cannot match
        }
    }
    // handed on: the plan stage gets the hits (plan_runs_planes) -- it still has to make sure the window holds
    // plain A/C/G/T only, else the prefilter verdict of the planes is not certain (window_is_plain)
#pragma unroll
    for (int b = 0; b < 8; ++b) out.M[b] = b < W ? st.M[b] : 0u;
}

// `end` points just past the last character of the searched window; n = its length (1 <= n <= 32 W;
// the caller routes everything else to the exact path).  The bytes [end - 32 W - 3, end + 4) must be
// readable (their values outside the window do not matter).
template <int W, class Prog>
CG_HD PlaneOut plane_scan_core(const uint32_t *ops, int n_ops, int plane_flags, int m, const uint8_t *ref,
                               const uint8_t *end, int n, bool always_pass)
{
    PlaneOut out;
    PlaneState<W> st;
    const int off0 = 32 * W - n;                     // plane index of the window's first character
    const uint8_t *base = end - 32 * W;              // plane index 0
    out.bad = plane_load<W>(st, base, off0);
    m = Prog::adapter_length(m);                     // (a literal in a specialised program)
    Prog::template run<W>(st, ops, n_ops, m);
    unsigned long long overlap_ok = 0;
    if (plane_flags & 2) {
        const int n_emits = (plane_flags >> 8) & 255;
        const uint8_t *after = (const uint8_t *)ops + (((size_t)n_ops * 4 + 7) & ~(size_t)7) + (size_t)n_emits * sizeof(CgPlaneEmit);
        overlap_ok = Prog::overlap_ok(*(const unsigned long long *)after);
    }
    plane_decide<W, Prog>(st, plane_flags, overlap_ok, m, ref, base, off0, n, always_pass, out);
    return out;
}

// Groups of characters the DP must visit, given the locator hits (see locate_core).
CG_HD uint32_t window_cover(const CgAdapter &A, int n, int gs, uint32_t hits)
{
    if (n <= 0) return 0xFFFFFFFFu;
    const int reach = A.m + A.k;                 // a hit at p needs characters p+1-reach .. p+reach
    const int r = (reach + (1 << gs) - 1) >> gs; // in groups
    uint32_t cover = hits;
    for (int s = 1; s <= r && s < 32; ++s) cover |= (hits << s) | (hits >> s);
    const int g_last = (n - 1) >> gs;
    if (A.flags & 1) {                           // START_IN_REFERENCE: adapter may hang over the read start
        const int g = cg_min(g_last, (reach - 1 > 0 ? reach - 1 : 0) >> gs);
        cover |= (g >= 31) ? 0xFFFFFFFFu : ((1u << (g + 1)) - 1u);
    }
    if (A.flags & 4) {                           // STOP_IN_REFERENCE: last-column scan (partial adapter at the end)
        const int g0 = cg_max(0, n - 1 - reach) >> gs;
        cover |= ~((1u << g0) - 1u);
    }
    const uint32_t valid = (g_last >= 31) ? 0xFFFFFFFFu : ((1u << (g_last + 1)) - 1u);
    cover &= valid;
    if (cover == valid) return 0xFFFFFFFFu;      // everything: plain DP
    return cover;
}

// ---------------------------------------------------------------------------------------
// Adapter composition
// ---------------------------------------------------------------------------------------
struct SetView {
    const CgSetHeader *h;
    const CgAdapter *ad;
    const CgGroup *gr;
    const CgEntry *en;
    const uint8_t *pool;
    const uint64_t *masks64;   // HBM
    const uint8_t *enc;        // 3 x 256 bytes: upper, acgt, iupac
    const CgScanWord *scan;    // two-phase program (h->scan_count words), if h->simple_ok
    const CgIndexHeader *index_hdr;   // anchored-adapter indexes (HBM), or null
    const CgIndexEntry *index_tab;
};

CG_HD SetView make_set_view(const uint8_t *blob, const uint64_t *masks64, const uint8_t *enc,
                            const uint8_t *index_blob = nullptr)
{
    SetView S;
    S.index_hdr = (const CgIndexHeader *)index_blob;
    S.index_tab = (const CgIndexEntry *)index_blob;   // table_off counts entries from the start of the array
    S.h = (const CgSetHeader *)blob;
    S.ad = (const CgAdapter *)(blob + S.h->adapters_off);
    S.gr = (const CgGroup *)(blob + S.h->groups_off);
    S.en = (const CgEntry *)(blob + S.h->entries_off);
    S.pool = blob + S.h->pool_off;
    S.masks64 = masks64;
    S.enc = enc;
    S.scan = (const CgScanWord *)(blob + S.h->scan_off);
    return S;
}

// <SingleAdapter>.match_to: prefilter, locate, wrap (adapters.py:707-724, 758-786, 815-832,
// 862-890, 915-935, 963-975, 1000-1012).
template <bool ALLOW_WIDE>
CG_HD bool match_single(const SetView &S, int ai, const uint8_t *p, int n, PackedCol &colp,
                        WideCol &colw, CgHit &hit)
{
    const CgAdapter &A = S.ad[ai];
    ReadView rv; rv.p = p; rv.n = n; rv.rev = A.reverse;
    if (A.pf_count > 0 && !kmers_present_core(S.en + A.pf_first, A.pf_count, S.masks64, rv)) return false;
    const uint8_t *ref = S.pool + A.ref_off;
    const uint8_t *enc = S.enc + 256 * A.query_enc;
    int o[6];
    bool found;
    if (A.kind == CGK_KIND_ALIGNER) {
        const int32_t *ncnt = (const int32_t *)(S.pool + A.ncount_off);
        const int32_t *maxcost = (const int32_t *)(S.pool + A.maxcost_off);
        if (ALLOW_WIDE && (A.cell_mode == CG_CELL_WIDE || n > CG_PACKED_MAX_N))
            found = locate_core<WideCell, WideCol>(A, ref, ncnt, maxcost, enc, rv, colw, o);
        else
            found = locate_core<Packed32, PackedCol>(A, ref, ncnt, maxcost, enc, rv, colp, o);
    } else {
        found = compare_core(A, ref, enc, rv, o);
    }
    if (!found) return false;
    hit.adapter = ai;
    if (A.reverse) {                                            // adapters.py:777-785, 881-889
        hit.astart = A.m - o[1]; hit.astop = A.m - o[0];
        hit.rstart = n - o[3]; hit.rstop = n - o[2];
    } else {
        hit.astart = o[0]; hit.astop = o[1]; hit.rstart = o[2]; hit.rstop = o[3];
    }
    hit.score = o[4]; hit.errors = o[5];
    hit.remove = A.remove == CGK_REMOVE_AUTO ? (hit.rstart == 0 ? CGK_REMOVE_BEFORE : CGK_REMOVE_AFTER)
                                            : A.remove;        // adapters.py:930-935
    return true;
}

// Apply Match.trimmed() to the window [s, e)   (adapters.py:453-454, 486-487)
CG_HD void apply_trim(const CgHit &h, int &s, int &e)
{
    if (h.remove == CGK_REMOVE_BEFORE) s += h.rstop;
    else e = s + h.rstart;
}

// AdapterIndex.match_to (adapters.py:1474-1551): dict lookups of the read's prefix/suffix for every
// key length, longest first.
CG_HD uint64_t cg_index_hash(uint64_t bases, uint32_t len)
{
    uint64_t x = bases ^ ((uint64_t)len * 0x9E3779B97F4A7C15ULL);
    x ^= x >> 29; x *= 0xBF58476D1CE4E5B9ULL; x ^= x >> 32;
    return x;
}

template <bool ALLOW_WIDE>
CG_HD bool match_single(const SetView &S, int ai, const uint8_t *p, int n, PackedCol &colp,
                        WideCol &colw, CgHit &hit);

template <bool ALLOW_WIDE>
CG_HD bool match_indexed(const SetView &S, int index_no, const uint8_t *p, int n, PackedCol &colp,
                         WideCol &colw, CgHit &hit, bool *needs_realign = nullptr)
{
    const CgIndexHeader &H = S.index_hdr[index_no];
    const CgIndexEntry *tab = S.index_tab + H.table_off;
    int best_a = -1, best_len = 0, best_m = -1, best_e = 1000;
    // The affix is packed ONCE, for the longest key (the lengths are descending): 2 bits per character at bit 2 i,
    // A C G T = 0 1 2 3 (bits 1-2 of the ASCII code give A C T G = 0 1 2 3; x ^ (x >> 1) swaps the last two), either
    // case (sequence.upper()), N as A (_lookup_with_n); one bit per position for "N" and for "not a nucleotide".
    // The key of a shorter length is a mask (prefix) or a shift (suffix) away.
    const int cnt_max = cg_min((int)H.lengths[0], cg_min(n, 32));
    const uint8_t *q_max = H.prefix ? p : p + (n - cnt_max);
    uint64_t packed = 0;
    uint32_t n_mask = 0, bad_mask = 0;
    for (int i = 0; i < cnt_max; ++i) {
        const uint32_t c = q_max[i], u = c & 0xDFu, x = (c >> 1) & 3u;
        const bool is_n = u == 'N';
        const bool acgt = u == 'A' || u == 'C' || u == 'G' || u == 'T';
        const uint64_t code = is_n ? 0u : (x ^ (x >> 1));
        packed |= code << (2 * i);
        n_mask |= (is_n ? 1u : 0u) << i;
        bad_mask |= ((acgt || is_n) ? 0u : 1u) << i;
    }
    for (int li = 0; li < H.n_lengths; ++li) {
        const int L = H.lengths[li];
        if (L < best_m) break;                                   // adapters.py:1506-1508
        const int cnt = cg_min(L, n);                            // sequence[:L] / sequence[-L:]
        if (cnt > 32 || cnt <= 0) continue;
        const uint8_t *q = H.prefix ? p : p + (n - cnt);
        const int skip = H.prefix ? 0 : cnt_max - cnt;           // position of the key's first character in the packed affix
        const uint32_t span = (cnt >= 32 ? 0xFFFFFFFFu : ((1u << cnt) - 1u)) << skip;
        const uint64_t bases = (packed >> (2 * skip)) & (cnt >= 32 ? ~0ULL : ((1ULL << (2 * cnt)) - 1ULL));
        const bool has_n = (n_mask & span) != 0, valid = (bad_mask & span) == 0;
        if (!valid) continue;
        uint32_t val = 0;
        bool found = false;
        for (uint32_t slot = (uint32_t)cg_index_hash(bases, (uint32_t)cnt) & H.table_mask;;
             slot = (slot + 1) & H.table_mask) {
            const CgIndexEntry e = tab[slot];
            if (e.len == 0) break;
            if (e.len == (uint32_t)cnt && e.bases == bases) { val = e.val; found = true; break; }
        }
        if (!found) continue;
        const int a = (int)(val >> 16);
        int e = (int)((val >> 8) & 255u), m = (int)(val & 255u);
        if (has_n && needs_realign) { *needs_realign = true; return false; }   // (the caller has no DP column: cg_index_kernel)
        if (has_n) {                                             // adapters.py:1535-1551: re-align
            CgHit h;
            if (!match_single<ALLOW_WIDE>(S, a, q, cnt, colp, colw, h)) continue;
            e = h.errors; m = h.score;
        }
        if (m > best_m || (m == best_m && e < best_e)) { best_a = a; best_e = e; best_m = m; best_len = L; }
    }
    if (best_m == -1) return false;
    hit.adapter = best_a;
    hit.astart = 0; hit.astop = S.ad[best_a].m;
    if (H.prefix) { hit.rstart = 0; hit.rstop = best_len; hit.remove = CGK_REMOVE_BEFORE; }
    else { hit.rstart = n - best_len; hit.rstop = n; hit.remove = CGK_REMOVE_AFTER; }
    hit.score = best_m; hit.errors = best_e;
    return true;
}

struct GroupHit {
    CgHit h0, h1;     // SINGLE: h0.  LINKED: h0 = front (adapter -1 if absent), h1 = back.
    int score, errors;
};

// One Matchable.match_to on the window [p, p+n)
template <bool ALLOW_WIDE>
CG_HD bool match_group(const SetView &S, const CgGroup &G, const uint8_t *p, int n,
                       PackedCol &colp, WideCol &colw, GroupHit &gh)
{
    gh.h0.adapter = -1; gh.h1.adapter = -1;
    if (G.type == CGK_GROUP_INDEXED) {
        if (!match_indexed<ALLOW_WIDE>(S, G.a0, p, n, colp, colw, gh.h0)) return false;
        gh.score = gh.h0.score; gh.errors = gh.h0.errors;
        return true;
    }
    if (G.type == CGK_GROUP_SINGLE) {
        if (!match_single<ALLOW_WIDE>(S, G.a0, p, n, colp, colw, gh.h0)) return false;
        gh.score = gh.h0.score; gh.errors = gh.h0.errors;
        return true;
    }
    // LinkedAdapter.match_to  (adapters.py:1215-1227)
    const bool front = match_single<ALLOW_WIDE>(S, G.a0, p, n, colp, colw, gh.h0);
    if (!front) gh.h0.adapter = -1;
    if (G.front_required && !front) return false;
    int s = 0, e = n;
    if (front) apply_trim(gh.h0, s, e);                         // sequence[front_match.trim_slice()]
    const bool back = match_single<ALLOW_WIDE>(S, G.a1, p + s, e - s, colp, colw, gh.h1);
    if (!back) gh.h1.adapter = -1;
    if (!back && (G.back_required || !front)) return false;
    gh.score = (front ? gh.h0.score : 0) + (back ? gh.h1.score : 0);   // adapters.py:1113-1130
    gh.errors = (front ? gh.h0.errors : 0) + (back ? gh.h1.errors : 0);
    return true;
}

#ifndef CG_MATCH_STRUCT_DEFINED
#define CG_MATCH_STRUCT_DEFINED
struct cg_match_rec { int32_t adapter, astart, astop, rstart, rstop, score, errors, info; };
#endif

CG_HD void store_hit(cg_match_rec *dst, const CgHit &h, int group, int searched_len)
{
    cg_match_rec r;
    r.adapter = h.adapter;
    if (h.adapter < 0) { r.astart = r.astop = r.rstart = r.rstop = r.score = r.errors = 0; r.info = 0; }
    else {
        r.astart = h.astart; r.astop = h.astop; r.rstart = h.rstart; r.rstop = h.rstop;
        r.score = h.score; r.errors = h.errors;
        r.info = (group & 255) | (h.remove == CGK_REMOVE_AFTER ? 256 : 0) | ((searched_len & 0xFFFF) << 16);
    }
#if defined(__CUDA_ARCH__)
    // two 16-byte stores
    ((int4 *)dst)[0] = make_int4(r.adapter, r.astart, r.astop, r.rstart);
    ((int4 *)dst)[1] = make_int4(r.rstop, r.score, r.errors, r.info);
#else
    *dst = r;
#endif
}

// The whole per-read pass: optional quality trimming, then `times` rounds of
// MultipleAdapters.match_to + trim  (modifiers.py:853-858, 225-231; adapters.py:1265-1286).
//   seq/qual : this read's bytes (qual may be null when quality_trim == 0)
//   out      : times * slots records
template <bool ALLOW_WIDE>
CG_HD void process_read(const SetView &S, const uint8_t *seq, const uint8_t *qual, int n,
                        int quality_trim, int cutoff_front, int cutoff_back, int qbase, int times,
                        PackedCol &colp, WideCol &colw, cg_match_rec *out, int32_t *qtrim_out,
                        const int32_t *view = nullptr)
{
    const int slots = S.h->slots;
    int s = 0, e = n;
    if (quality_trim) pre_trim_core(seq, qual, n, quality_trim, cutoff_front, cutoff_back, qbase, &s, &e);
    if (qtrim_out) { qtrim_out[0] = s; qtrim_out[1] = e; }
    if (view) { s = view[0]; e = view[1]; }                    // per-adapter pass: search read[s:e]
    CgHit none; none.adapter = -1; none.remove = 0;
    none.astart = none.astop = none.rstart = none.rstop = none.score = none.errors = 0;
    bool alive = true;
    for (int r = 0; r < times; ++r) {
        cg_match_rec *dst = out + (size_t)r * slots;
        bool have = false;
        int best_group = -1;
        GroupHit best;
        best.h0 = none; best.h1 = none; best.score = 0; best.errors = 0;
        if (alive) {
            for (int g = 0; g < S.h->n_groups; ++g) {           // adapters.py:1271-1286
                GroupHit gh;
                if (!match_group<ALLOW_WIDE>(S, S.gr[g], seq + s, e - s, colp, colw, gh)) continue;
                if (!have || gh.score > best.score || (gh.score == best.score && gh.errors < best.errors)) {
                    have = true; best = gh; best_group = g;
                }
            }
        }
        if (!have) {
            alive = false;                                      // modifiers.py:227-229
            store_hit(dst, none, 0, 0);
            if (slots > 1) store_hit(dst + 1, none, 0, 0);
            continue;
        }
        const int searched = e - s;
        store_hit(dst, best.h0, best_group, searched);
        if (slots > 1) {
            int s2 = 0, e2 = searched;
            if (best.h0.adapter >= 0) apply_trim(best.h0, s2, e2);
            store_hit(dst + 1, best.h1, best_group, e2 - s2);
        }
        // trimmed_read = match.trimmed(trimmed_read)           (modifiers.py:231; adapters.py:1132-1137)
        if (best.h0.adapter >= 0) apply_trim(best.h0, s, e);
        if (best.h1.adapter >= 0) apply_trim(best.h1, s, e);
    }
}

// ---------------------------------------------------------------------------------------
// Statistics of one read (cg_stats_kernel; tests/hostsim runs the same function).  `add(index, n)` adds to an
// entry of the vector relative to its histogram part (index 0 = first entry of the read-length histogram);
// the five scalar sums are returned through `sc` (n is counted by the caller).
//   seq   : the read's bytes or null (then no adjacent bases are counted)
//   recs  : times x slots records of this read
// Window bookkeeping as the reference does it: the rounds work on what the previous ones left
// (modifiers.py:225-231), a linked adapter's 3' part on what its 5' part left (adapters.py:1220-1222).
// upper: the adjacent base is read from the upper-cased read (--action=lowercase upper-cases the read before
// matching, modifiers.py:222-223).
// ---------------------------------------------------------------------------------------
struct StatsScalars { unsigned long long bp, with_adapters, qtrim_bp, adapter_bp; };

template <class Add>
CG_HD void stats_read_core(const uint8_t *seq, int len, bool have_qtrim, int qs, int qe, const cg_match_rec *recs,
                           int times, int slots, int n_adapters, int max_len, int kmax, StatsScalars &sc, Add add,
                           bool upper = false)
{
    sc.bp += (unsigned long long)len;
    int ws = 0, we = len;                                   // current window [ws, we) of the original read
    if (have_qtrim) { ws = qs; we = qe; sc.qtrim_bp += (unsigned long long)(len - (qe - qs)); }
    const long long end_size = cg_stats_end_size(max_len, kmax);
    const long long adapters_rel = max_len + 1;             // relative to the read-length histogram
    bool any = false;
    for (int t = 0; t < times; ++t) {
        for (int s = 0; s < slots; ++s) {
            const cg_match_rec m = recs[(size_t)t * slots + s];
            if (m.adapter < 0) continue;
            any = true;
            const bool after = (m.info & 256) != 0;
            const int cur = we - ws;
            const int removed = after ? cur - m.rstart : m.rstop;
            sc.adapter_bp += (unsigned long long)(removed < 0 ? 0 : removed);
            if (m.adapter < n_adapters) {
                const int L = removed < 0 ? 0 : (removed > max_len ? max_len : removed);
                const int E = m.errors < 0 ? 0 : (m.errors > kmax ? kmax : m.errors);
                const long long blk = adapters_rel + (2LL * m.adapter + (after ? 1 : 0)) * end_size;
                add(blk + CG_STATS_ADJ + (long long)L * (kmax + 1) + E, 1u);
                if (after && seq) {
                    // Match.adjacent_base(): the character in front of the match, "" at the start of the read;
                    // anything but an upper-case A/C/G/T counts as "" (adapters.py:193-199, 488-489)
                    int k = 4;
                    const int pos = ws + m.rstart - 1;
                    if (m.rstart > 0 && pos >= 0 && pos < len) {
                        uint8_t c = seq[pos];
                        if (upper && c >= 'a' && c <= 'z') c = (uint8_t)(c - 32);
                        k = c == 'A' ? 0 : (c == 'C' ? 1 : (c == 'G' ? 2 : (c == 'T' ? 3 : 4)));
                    }
                    add(blk + k, 1u);
                }
            }
            // Match.trimmed(): python slice semantics (indexes beyond the window clamp)
            if (after) { const int rs = m.rstart < 0 ? 0 : (m.rstart > cur ? cur : m.rstart); we = ws + rs; }
            else { const int rp = m.rstop < 0 ? 0 : (m.rstop > cur ? cur : m.rstop); ws += rp; }
        }
    }
    sc.with_adapters += any ? 1 : 0;
    const int fin = we - ws;
    add((long long)(fin < 0 ? 0 : (fin > max_len ? max_len : fin)), 1u);
}

// ---------------------------------------------------------------------------------------
// Multi-pass schedule: every component adapter of a set is located on its own (one pass each, into
// a scratch array of records), then these two functions apply the composition rules.
// ---------------------------------------------------------------------------------------
// View of a LinkedAdapter's back adapter: sequence[front_match.trim_slice()]  (adapters.py:1220-1222)
CG_HD void linked_view(const cg_match_rec &front, int &s, int &e)
{
    if (front.adapter < 0) return;
    if (front.info & 256) e = s + front.rstart;          // RemoveAfterMatch
    else s += front.rstop;                               // RemoveBeforeMatch
}

// MultipleAdapters.match_to (adapters.py:1271-1286) over the per-pass records: highest score, then
// fewest errors, then the group listed first; LinkedAdapter.match_to (adapters.py:1215-1227) for
// LINKED groups.  `load(pass)` returns this read's record of a pass.
template <class Load>
CG_HD void select_best(const CgSelectTables &T, const int32_t *pass_map, Load load, cg_match_rec &b0,
                       cg_match_rec &b1)
{
    cg_match_rec none;
    none.adapter = -1; none.astart = none.astop = none.rstart = none.rstop = none.score = none.errors = none.info = 0;
    b0 = none; b1 = none;
    bool have = false;
    int best_score = 0, best_errors = 0;
    for (int g = 0; g < T.n_groups; ++g) {
        cg_match_rec h0 = load((int)T.pass0[g]), h1 = none;
        int score, errors;
        if (T.gtype[g] != CGK_GROUP_LINKED) {
            if (h0.adapter < 0) continue;
            h0.adapter = pass_map[T.map_off[T.pass0[g]] + h0.adapter];
            score = h0.score; errors = h0.errors;
        } else {
            const bool front = h0.adapter >= 0;
            if (T.front_required[g] && !front) continue;
            h1 = load((int)T.pass1[g]);
            const bool back = h1.adapter >= 0;
            if (!back && (T.back_required[g] || !front)) continue;
            if (front) h0.adapter = pass_map[T.map_off[T.pass0[g]] + h0.adapter]; else h0 = none;
            if (back) h1.adapter = pass_map[T.map_off[T.pass1[g]] + h1.adapter]; else h1 = none;
            score = (front ? h0.score : 0) + (back ? h1.score : 0);
            errors = (front ? h0.errors : 0) + (back ? h1.errors : 0);
        }
        if (!have || score > best_score || (score == best_score && errors < best_errors)) {
            have = true; best_score = score; best_errors = errors;
            if (h0.adapter >= 0) h0.info = (h0.info & ~255) | g;
            if (h1.adapter >= 0) h1.info = (h1.info & ~255) | g;
            b0 = h0; b1 = h1;
        }
    }
}

// ---------------------------------------------------------------------------------------
// Two-phase ("simple") path: one SINGLE aligner adapter, packed cells, one round.
//   phase A  simple_scan    prefilter verdict + locator hits        (all reads)
//   phase B  simple_locate  windowed DP + Match wrapping            (reads that passed)
// The kernel compacts the reads that pass phase A before phase B; tests/hostsim runs both
// back to back per read.  Results are identical to process_read<>() by construction of the
// windows (see locate_core) -- tests/test_hostsim.py fuzzes exactly that.
// ---------------------------------------------------------------------------------------
CG_HD ScanOut simple_scan(const SetView &S, const uint8_t *p, int n, int *gs_out)
{
    const CgAdapter &A = S.ad[0];
    ReadView rv; rv.p = p; rv.n = n; rv.rev = A.reverse;
    const int gs = scan_group_shift(n);
    *gs_out = gs;
    return scan_core(S.scan, S.h->scan_count, S.pool, rv, gs, A.pf_count == 0);
}

CG_HD bool simple_locate(const SetView &S, const uint8_t *p, int n, uint32_t hits, int gs,
                         PackedCol &colp, CgHit &hit)
{
    const CgAdapter &A = S.ad[0];
    ReadView rv; rv.p = p; rv.n = n; rv.rev = A.reverse;
    const uint8_t *ref = S.pool + A.ref_off;
    const uint8_t *enc = S.enc + 256 * A.query_enc;
    const int32_t *ncnt = (const int32_t *)(S.pool + A.ncount_off);
    const int32_t *maxcost = (const int32_t *)(S.pool + A.maxcost_off);
    const uint32_t cover = S.h->windowed ? window_cover(A, n, gs, hits) : 0xFFFFFFFFu;
    int o[6];
    if (!locate_core<Packed32, PackedCol>(A, ref, ncnt, maxcost, enc, rv, colp, o, cover, gs)) return false;
    hit.adapter = 0;
    if (A.reverse) {
        hit.astart = A.m - o[1]; hit.astop = A.m - o[0];
        hit.rstart = n - o[3]; hit.rstop = n - o[2];
    } else {
        hit.astart = o[0]; hit.astop = o[1]; hit.rstart = o[2]; hit.rstop = o[3];
    }
    hit.score = o[4]; hit.errors = o[5];
    hit.remove = A.remove == CGK_REMOVE_AUTO ? (hit.rstart == 0 ? CGK_REMOVE_BEFORE : CGK_REMOVE_AFTER)
                                            : A.remove;
    return true;
}

// ---------------------------------------------------------------------------------------
// Phase B, register-column variant (adapters with m <= 32).
//
//  * refine_runs(): the coarse locator hits of phase A (one bit per 16-character group) are
//    re-scanned to exact end positions p; a chunk that ends at adapter offset b puts the adapter
//    start at p + 1 - b, and every alignment with <= k errors through that chunk lies inside
//    columns [start - k, start + m + k] (the path consumes b adapter characters and at most
//    b + k read characters before the chunk ends; m - b adapter characters and at most
//    m - b + k read characters after it).  Runs are merged into at most three disjoint intervals.
//  * locate_regs<MR>(): the same DP as locate_core, but the packed column lives in registers and
//    the row loop is unrolled with a warp-uniform bound (max band over the warp's lanes), so there
//    is no shared-memory traffic and no per-lane trip-count divergence.  Lanes of a warp start
//    their runs k columns before their own adapter start, so their bands grow in step.
// ---------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
#define CG_WARP_MAX(x) __reduce_max_sync(0xffffffffu, (x))
#define CG_WARP_ANY(p) __any_sync(0xffffffffu, (p))
#else
#define CG_WARP_MAX(x) (x)
#define CG_WARP_ANY(p) (p)
#endif

struct RunList {
    int n;
    int lo0, hi0, lo1, hi1, lo2, hi2;   // sorted, disjoint; run r restarts at column lo_r and
                                        // computes columns lo_r + 1 .. hi_r
};

CG_HD void runs_add(RunList &R, int lo, int hi, int n_read)
{
    if (lo < 0) lo = 0;
    if (hi > n_read) hi = n_read;
    if (hi <= lo) return;
    if (R.n == 0) { R.lo0 = lo; R.hi0 = hi; R.n = 1; return; }
    if (R.n == 1) {
        if (lo <= R.hi0) { R.lo0 = cg_min(R.lo0, lo); R.hi0 = cg_max(R.hi0, hi); }
        else { R.lo1 = lo; R.hi1 = hi; R.n = 2; }
        return;
    }
    if (R.n == 2) {
        if (lo <= R.hi1) {
            R.lo1 = cg_min(R.lo1, lo); R.hi1 = cg_max(R.hi1, hi);
            if (R.lo1 <= R.hi0) { R.lo0 = cg_min(R.lo0, R.lo1); R.hi0 = cg_max(R.hi0, R.hi1); R.n = 1; }
        } else { R.lo2 = lo; R.hi2 = hi; R.n = 3; }
        return;
    }
    // three runs already: merge into the last one (a superset is always valid)
    R.lo2 = cg_min(R.lo2, lo); R.hi2 = cg_max(R.hi2, hi);
    if (R.lo2 <= R.hi1) {
        R.lo1 = cg_min(R.lo1, R.lo2); R.hi1 = cg_max(R.hi1, R.hi2); R.n = 2;
        if (R.lo1 <= R.hi0) { R.lo0 = cg_min(R.lo0, R.lo1); R.hi0 = cg_max(R.hi0, R.hi1); R.n = 1; }
    }
}

// Exact positions of the locator hits -> DP runs (windowed adapters only).  For the first locator
// word the scan resumes at the start of each hit group from the state phase A saved (rs0, rs1) or
// carries over from the previous group; otherwise it backs up 31 characters (k-mers are <= 32 long).
// Hits of one stretch of consecutive hit groups are united into one run (their windows overlap or
// nearly so; a superset of the exact windows is always valid).
template <bool REV>
CG_HD void refine_runs_dir(const CgScanWord *words, int n_words, const uint8_t *pool, const CgAdapter &A,
                           const uint8_t *first, int n, uint32_t hits, int gs, uint32_t rs0, uint32_t rs1,
                           RunList &R, bool add_end)
{
    const int m = A.m, k = A.k;
    R.n = 0;
    R.lo0 = R.hi0 = R.lo1 = R.hi1 = R.lo2 = R.hi2 = 0;
    if (A.flags & 1) runs_add(R, 0, cg_min(n, m + k), n);              // START_IN_REFERENCE
    if (hits) {
        int n_loc = 0;
        for (int w = 0; w < n_words; ++w) n_loc += (words[w].type == CG_SCAN_WHOLE && words[w].loc_found) ? 1 : 0;
        for (int w = 0; w < n_words; ++w) {
            const CgScanWord &W = words[w];
            if (W.type != CG_SCAN_WHOLE || !W.loc_found) continue;
            const uint32_t *mask = (const uint32_t *)(pool + W.mask_off);
            const uint8_t *ltab = pool + W.loc_off;
            const uint32_t init = W.init, locf = W.loc_found;
            const bool stash = n_loc == 1;
            uint32_t todo = hits, Rr = 0;
            int cur_p = -1, nh = 0;
            int wlo = 0x3fffffff, whi = -1;                      // window of the current stretch
            while (todo) {
                const int g = cg_ctz(todo);
                todo &= todo - 1;
                const int p_first = g << gs;
                const long long p_end_ll = ((long long)(g + 1)) << gs;
                const int p_end = p_end_ll > n ? n : (int)p_end_ll;
                if (cur_p != p_first) {
                    if (whi >= 0) { runs_add(R, wlo, whi, n); wlo = 0x3fffffff; whi = -1; }
                    if (stash && nh < 2) {
                        Rr = nh == 0 ? rs0 : rs1;
                    } else {
                        Rr = 0;
                        const int q0 = cg_max(0, p_first - 31);
                        const uint8_t *q = first + (REV ? -q0 : q0);
                        for (int i = q0; i < p_first; ++i) {
                            Rr = ((Rr << 1) | init) & mask[*q];
                            q += REV ? -1 : 1;
                        }
                    }
                }
                ++nh;
                const uint8_t *q = first + (REV ? -p_first : p_first);
                for (int p = p_first; p < p_end; ++p) {
                    Rr = ((Rr << 1) | init) & mask[*q];
                    q += REV ? -1 : 1;
                    uint32_t f = Rr & locf;
                    while (f) {
                        const int b = cg_ctz(f);
                        f &= f - 1;
                        wlo = cg_min(wlo, p + 1 - (int)ltab[2 * b + 1] - k);
                        whi = cg_max(whi, p + 1 - (int)ltab[2 * b] + m + k);
                    }
                }
                cur_p = p_end;
            }
            if (whi >= 0) runs_add(R, wlo, whi, n);
        }
    }
    if (add_end && (A.flags & 4)) runs_add(R, cg_max(0, n - 1 - m - k), n, n);      // STOP_IN_REFERENCE
}

CG_HD void refine_runs(const CgScanWord *words, int n_words, const uint8_t *pool, const CgAdapter &A,
                       const ReadView &rv, uint32_t hits, int gs, uint32_t rs0, uint32_t rs1, RunList &R,
                       bool add_end = true)
{
    if (rv.rev) refine_runs_dir<true>(words, n_words, pool, A, rv.p + (rv.n - 1), rv.n, hits, gs, rs0, rs1, R, add_end);
    else refine_runs_dir<false>(words, n_words, pool, A, rv.p, rv.n, hits, gs, rs0, rs1, R, add_end);
}

// Phase A for the register path: the fused scan with the locator hits turned into DP runs on
// the spot (exact end position p of a chunk -> run [p+1-b-k, p+1-b+m+k]); no second pass.
CG_HD void scan_runs_core(const CgScanWord *words, int n_words, const uint8_t *pool, const CgAdapter &A,
                          const ReadView &rv, bool always_pass, bool windowed, bool &pass_out, RunList &R)
{
    const int n = rv.n, m = A.m, k = A.k;
    bool pass = always_pass;
    R.n = 0;
    R.lo0 = R.hi0 = R.lo1 = R.hi1 = R.lo2 = R.hi2 = 0;
    if (windowed && (A.flags & 1)) runs_add(R, 0, cg_min(n, m + k), n);       // START_IN_REFERENCE
    const uint8_t *cp = rv.rev ? rv.p + (n - 1) : rv.p;
    const int cstride = rv.rev ? -1 : 1;
    for (int w = 0; w < n_words; ++w) {
        const CgScanWord &W = words[w];
        const uint32_t *mask = (const uint32_t *)(pool + W.mask_off);
        if (W.type == CG_SCAN_WHOLE) {
            const uint32_t init = W.init;
            const uint32_t locf = windowed ? W.loc_found : 0u;
            uint32_t Rr = 0, seen = 0;
            if (locf) {
                const uint8_t *ltab = pool + W.loc_off;
                for (int p = 0; p < n; ++p) {
                    Rr = ((Rr << 1) | init) & mask[cp[cstride * p] & 127];
                    seen |= Rr;
                    uint32_t f = Rr & locf;
                    while (f) {                                   // rare: a locator chunk ends at p
                        const int b = cg_ctz(f);
                        f &= f - 1;
                        runs_add(R, p + 1 - (int)ltab[2 * b + 1] - k, p + 1 - (int)ltab[2 * b] + m + k, n);
                    }
                }
            } else {
                for (int p = 0; p < n; ++p) {
                    Rr = ((Rr << 1) | init) & mask[cp[cstride * p] & 127];
                    seen |= Rr;
                }
            }
            if (seen & W.pass_found) pass = true;
        } else if (W.type == CG_SCAN_SUFFIX) {
            const uint32_t *tab = (const uint32_t *)(pool + W.pos_off);
            uint32_t Rr = 0, seen = 0;
            for (int p = cg_max(0, n - (int)W.span); p < n; ++p) {
                const int d = n - p;
                Rr = ((Rr << 1) | tab[2 * d]) & mask[cp[cstride * p] & 127];
                seen |= Rr & tab[2 * d + 1];
            }
            if (seen & W.pass_found) pass = true;
        } else {
            const uint32_t *tab = (const uint32_t *)(pool + W.pos_off);
            uint32_t Rr = 0, seen = 0;
            const int stop = cg_min(n, (int)W.span);
            for (int p = 0; p < stop; ++p) {
                Rr = ((Rr << 1) | tab[2 * p]) & mask[cp[cstride * p] & 127];
                seen |= Rr & tab[2 * p + 1];
            }
            if (seen & W.pass_found) pass = true;
        }
    }
    if (windowed && (A.flags & 4)) runs_add(R, cg_max(0, n - 1 - m - k), n, n);   // STOP_IN_REFERENCE
    pass_out = pass;
}

// Selection state of _align.pyx:391-396 (the `best` match so far); carried from the main DP pass of
// a read to its end-window pass when the two are scheduled separately.
struct LocState {
    int have, b_origin, b_cost, b_score, b_ref_stop, b_q_stop, stopped;
};
CG_HD LocState loc_state_init(int m, int n)
{
    LocState st;
    st.have = 0; st.b_origin = 0; st.b_cost = 0; st.b_score = 0; st.b_ref_stop = m; st.b_q_stop = n; st.stopped = 0;
    return st;
}
CG_HD bool loc_state_result(const LocState &st, int *out6)
{
    if (!st.have) return false;                                  // _align.pyx:573-587
    out6[0] = st.b_origin >= 0 ? 0 : -st.b_origin;
    out6[1] = st.b_ref_stop;
    out6[2] = st.b_origin >= 0 ? st.b_origin : 0;
    out6[3] = st.b_q_stop;
    out6[4] = st.b_score;
    out6[5] = st.b_cost;
    return true;
}

// Processes runs [0, n_use) of R starting from the selection state `st` and leaves the updated state
// in `st`; the last-column scan (_align.pyx:536-572) is done only when final_scan is set (i.e. when
// this call covers the read's last run).
#ifndef CG_RUN_BAND
#define CG_RUN_BAND 0       // 1: the DP runs skip the rows outside the band (run_band_d).  Exact (tests/hostsim is built
                            // with it: test_banded_dp_runs_on_crowded_reads) but measured SLOWER: DP rounds of
                            // configs 2 and 4 (33-row adapters) -- the four-row
                            // chunks above the band are few once the Ukkonen bound has cut the column, and the extra
                            // live values push the 48-row kernel into spills
#endif
#ifndef CG_BAND_SLACK
#define CG_BAND_SLACK 0     // test hook: > 0 cuts rows the band needs (tools/fuzz_band.py must then report mismatches)
#endif
template <int MR, bool NC = false, bool SMEM = false, bool BAND = false>
CG_HD void locate_regs(const CgAdapter &A, const int32_t *ncnt, const int32_t *maxcost,
                       const uint32_t *peq, const ReadView &rv, const RunList &R, int n_use, bool has_task,
                       bool final_scan, LocState &st, bool eval_bottom = true, int band_d = -1)
{
    typedef Packed32 C;
    uint32_t c[MR + 1];
    const int m = A.m, n = rv.n, k = A.k;
    const bool sir = (A.flags & 1) != 0, siq = (A.flags & 2) != 0;
    const bool eir = (A.flags & 4) != 0, eiq = (A.flags & 8) != 0;
    int max_n = n, min_n = 0;
    if (!siq) max_n = cg_min(n, m + k);
    if (!eiq) min_n = cg_max(0, n - m - k);
    const uint32_t kthr = (uint32_t)(k + 1) << C::CS;      // cost <= k  <=>  word < kthr
    // character access without a per-character branch: p[base + stride * j]
    const uint8_t *cp = rv.rev ? rv.p + (n - 1) : rv.p;
#if defined(__CUDA_ARCH__)
    const uint32_t cp_s = SMEM ? (uint32_t)__cvta_generic_to_shared(cp) : 0u;   // SMEM: the read bytes are in shared memory
#endif
    const int cstride = rv.rev ? -1 : 1;

    bool have = st.have != 0;
    int b_origin = st.b_origin, b_cost = st.b_cost, b_score = st.b_score, b_ref_stop = st.b_ref_stop, b_q_stop = st.b_q_stop;
    int last = 0, last_filled = 0;
    uint32_t stale = C::make(0, 0, 0);
    bool stopped = st.stopped != 0, reached_end = false;
    const int n_runs = has_task ? n_use : 0;
    const int max_runs = CG_WARP_MAX(n_runs);
#pragma unroll
    for (int i = 0; i <= MR; ++i) c[i] = C::INF;

    for (int run = 0; run < max_runs; ++run) {
        const bool mine = run < n_runs && !stopped;
        const int lo = run == 0 ? R.lo0 : (run == 1 ? R.lo1 : R.lo2);
        const int hi = run == 0 ? R.hi0 : (run == 1 ? R.hi1 : R.hi2);
        // ---- column `lo` of this run -----------------------------------------------------------
        if (mine) {
            if (lo == min_n) {                                  // _align.pyx:364-383
#pragma unroll
                for (int i = 0; i <= MR; ++i) {
                    long long cc; int s, o;
                    if (!sir && !siq) { s = -2 * i; cc = cg_max(i, min_n); o = 0; }
                    else if (sir && !siq) { s = 0; cc = min_n; o = cg_min(0, min_n - i); }
                    else if (!sir && siq) { s = -2 * i; cc = i; o = cg_max(0, min_n - i); }
                    else { s = 0; cc = cg_min(i, min_n); o = min_n - i; }
                    c[i] = (i <= m) ? C::make(cc, s, o) : C::INF;
                }
                last = sir ? m : cg_min(m, k + 1);              // _align.pyx:399-401
            } else {                                            // restart inside the read
#pragma unroll
                for (int i = 0; i <= MR; ++i) c[i] = (i <= m) ? C::make(i, -2 * i, lo) : C::INF;
                last = cg_min(m, k + 1);
            }
            reached_end = (hi == max_n);
        }
        const int my_len = mine ? hi - lo : 0;
        const int len = CG_WARP_MAX(my_len);
        // band (run_band_d): warp-uniform, so every lane of the warp must have one; the widest d decides
        const bool band_on = BAND && !CG_WARP_ANY(mine && band_d < 0);
        const int band_off = band_on ? CG_WARP_MAX(mine ? band_d : 0) + 2 * k : (1 << 28);
        for (int t = 0; t < len; ++t) {
            const bool act = mine && !stopped && t < my_len;
            // (all lanes stopped early: rare, so the vote is only taken every 8th column)
            if ((t & 7) == 0 && !CG_WARP_ANY(act)) break;
            const int my_last = act ? last : 0;
            const int jj = act ? lo + t : 0;
#if defined(__CUDA_ARCH__)
            int ch = 0;
            if (SMEM) { if (act) ch = (int)(cg_lds_u8(cp_s + (uint32_t)(cstride * jj)) & 127u); }
            else ch = act ? (cp[cstride * jj] & 127) : 0;
#else
            const int ch = act ? (cp[cstride * jj] & 127) : 0;
#endif
            const uint32_t pq_lo = peq[ch];
            uint32_t pq_hi = 0;
            if (MR > 32) pq_hi = peq[128 + ch];
            uint32_t diag = c[0];
            uint32_t w0 = (NC || siq) ? C::row0_free(diag) : C::row0_ins(diag, 1);   // NC implies a free read start
            w0 = act ? w0 : diag;
            c[0] = w0;
            uint32_t up = w0;
            int lastok = (act && w0 < kthr) ? 0 : -1;
            const int wmax = CG_WARP_MAX(my_last);
            // rows below `skip` were already outside the band in the previous column (their values are not needed
            // as diagonal neighbours either)
            const int skip = t - band_off + CG_BAND_SLACK;
#pragma unroll
            for (int i0 = 1; i0 <= MR; i0 += 4) {
                if (BAND && i0 + 3 < skip) {                    // warp-uniform: these four rows are dead for the rest
                    diag = C::INF;                              // of the run -- their cells are never read again,
                    up = C::INF;                                // only their place as neighbours of row i0 + 4
                } else if (i0 <= wmax) {                        // warp-uniform
#pragma unroll
                    for (int i = i0; i < i0 + 4; ++i) {
                        if (i <= MR) {
                            const uint32_t left = c[i];
                            const bool eq = (i <= 32) ? (((pq_lo >> ((i - 1) & 31)) & 1u) != 0)
                                                      : (((pq_hi >> ((i - 33) & 31)) & 1u) != 0);
                            const uint32_t mt = NC ? C::match_nc(diag) : C::match(diag);
                            const uint32_t mm = NC ? C::mismatch_nc(diag, up, left) : C::mismatch(diag, up, left, 1);
                            uint32_t nw = eq ? mt : mm;
                            const bool in = i <= my_last;
                            nw = in ? nw : left;
                            up = in ? nw : up;
                            lastok = (in && nw < kthr) ? i : lastok;
                            c[i] = nw;
                            diag = left;
                        }
                    }
                }
            }
            if (act) {
                const int j = lo + t + 1;                       // the column just computed
                if (my_last >= 1) stale = up;
                last_filled = my_last;
                if (lastok < m) {
                    last = lastok + 1;                          // _align.pyx:490-495
                } else if (eiq && eval_bottom) {                // _align.pyx:496-533
                    stale = up;
                    const int cost = C::cost(up), score = C::score(up), origin = C::origin(up);
                    const int length = m + cg_min(origin, 0);
                    int eff = length;
                    if (A.wildcard_ref) eff = (length < m) ? length - (ncnt[m] - ncnt[m - length]) : A.effective_length;
                    const bool ok = length >= A.min_overlap && cost <= maxcost[eff];
                    const int best_len = m + cg_min(b_origin, 0);
                    if (ok && (!have || (origin <= b_origin + m / 2 && score > b_score) ||
                               (length > best_len && score > b_score))) {
                        have = true;
                        b_score = score; b_cost = cost; b_origin = origin; b_ref_stop = m; b_q_stop = j;
                        if (cost == 0 && origin >= 0) stopped = true;   // _align.pyx:531-533
                    }
                }
            }
        }
    }

    if (has_task && final_scan && n_runs > 0 && max_n == n && reached_end && !stopped) {   // _align.pyx:536-572
        const int first_i = eir ? 0 : m;
        const int origin_var = C::origin(stale);
#pragma unroll
        for (int i = MR; i >= 0; --i) {
            if (i > last_filled || i < first_i) continue;
            const uint32_t w = c[i];
            if (!(w < kthr)) continue;
            const int o = C::origin(w), cost = C::cost(w), score = C::score(w);
            const int length = i + cg_min(o, 0);
            int eff = length;
            if (A.wildcard_ref) {
                if (length < m) eff = length - (ncnt[i] - ncnt[-cg_min(o, 0)]);
                else eff = A.effective_length;
            }
            const bool ok = length >= A.min_overlap && cost <= maxcost[eff];
            const int best_len = b_ref_stop + cg_min(b_origin, 0);
            if (ok && (!have || (origin_var <= b_origin + m / 2 && score > b_score) ||
                       (length > best_len && score > b_score))) {
                have = true;
                b_score = score; b_cost = cost; b_origin = o; b_ref_stop = i; b_q_stop = n;
            }
        }
    }
    st.have = have ? 1 : 0; st.b_origin = b_origin; st.b_cost = b_cost; st.b_score = b_score;
    st.b_ref_stop = b_ref_stop; st.b_q_stop = b_q_stop; st.stopped = stopped ? 1 : 0;
}

// Register path entry points.
//   simple_scan_runs    phase A: prefilter verdict + DP runs of one read
//   simple_locate_runs  phase B: ALL lanes of a warp must call it (warp collectives inside);
//                       lanes without a task pass has_task = false.
CG_HD bool simple_windowed(const SetView &S, int n)
{
    const CgAdapter &A = S.ad[0];
    return S.h->windowed && (A.flags & 2) && (A.flags & 8) && n > 0;
}

CG_HD bool simple_scan_runs(const SetView &S, const uint8_t *p, int n, RunList &R)
{
    const CgAdapter &A = S.ad[0];
    ReadView rv; rv.p = p; rv.n = n; rv.rev = A.reverse;
    bool pass;
    const bool windowed = simple_windowed(S, n);
    scan_runs_core(S.scan, S.h->scan_count, S.pool, A, rv, A.pf_count == 0, windowed, pass, R);
    if (!windowed) {
        // plain: one run over the reference's column range (_align.pyx:346-352)
        int max_n = n, min_n = 0;
        if (!(A.flags & 2)) max_n = cg_min(n, A.m + A.k);
        if (!(A.flags & 8)) min_n = cg_max(0, n - A.m - A.k);
        R.n = 1; R.lo0 = min_n; R.hi0 = max_n;
    }
    return pass;
}

CG_HD bool simple_locate_runs(const SetView &S, const uint8_t *p, int n, const RunList &R, bool has_task,
                              CgHit &hit)
{
    const CgAdapter &A = S.ad[0];
    ReadView rv; rv.p = p; rv.n = n; rv.rev = A.reverse;
    const int32_t *ncnt = (const int32_t *)(S.pool + A.ncount_off);
    const int32_t *maxcost = (const int32_t *)(S.pool + A.maxcost_off);
    const uint32_t *peq = (const uint32_t *)(S.pool + A.peq_off);
    LocState st = loc_state_init(A.m, n);
    if (A.m <= 16) locate_regs<16>(A, ncnt, maxcost, peq, rv, R, R.n, has_task, true, st);
    else locate_regs<32>(A, ncnt, maxcost, peq, rv, R, R.n, has_task, true, st);
    int o[6];
    if (!has_task || !loc_state_result(st, o)) return false;
    hit.adapter = 0;
    if (A.reverse) {
        hit.astart = A.m - o[1]; hit.astop = A.m - o[0];
        hit.rstart = n - o[3]; hit.rstop = n - o[2];
    } else {
        hit.astart = o[0]; hit.astop = o[1]; hit.rstart = o[2]; hit.rstop = o[3];
    }
    hit.score = o[4]; hit.errors = o[5];
    hit.remove = A.remove == CGK_REMOVE_AUTO ? (hit.rstart == 0 ? CGK_REMOVE_BEFORE : CGK_REMOVE_AFTER)
                                            : A.remove;
    return true;
}

// Phase B entry of the kernel for m <= 32: coarse hits (+ saved scan states) -> exact runs ->
// register DP.  ALL lanes of a warp must call it.
CG_HD bool simple_locate_regs(const SetView &S, const uint8_t *p, int n, uint32_t hits, int gs,
                              uint32_t rs0, uint32_t rs1, bool has_task, CgHit &hit)
{
    const CgAdapter &A = S.ad[0];
    ReadView rv; rv.p = p; rv.n = n; rv.rev = A.reverse;
    RunList R;
    R.n = 0; R.lo0 = R.hi0 = R.lo1 = R.hi1 = R.lo2 = R.hi2 = 0;
    if (has_task) {
        if (simple_windowed(S, n)) refine_runs(S.scan, S.h->scan_count, S.pool, A, rv, hits, gs, rs0, rs1, R);
        else {
            int max_n = n, min_n = 0;
            if (!(A.flags & 2)) max_n = cg_min(n, A.m + A.k);
            if (!(A.flags & 8)) min_n = cg_max(0, n - A.m - A.k);
            R.n = 1; R.lo0 = min_n; R.hi0 = max_n;
        }
    }
    return simple_locate_runs(S, p, n, R, has_task, hit);
}

// ---------------------------------------------------------------------------------------
// Split scheduling of one read's DP (split pipeline, cg_dp_kernel<false/true>):
//   main pass : every run except a trailing, separate end window; reads that stop early
//               (_align.pyx:531-533) or have no separate end window are finished here;
//   end pass  : the end window (restart + last-column scan) from the carried LocState.
// ---------------------------------------------------------------------------------------
CG_HD void hit_from_state(const CgAdapter &A, int n, const LocState &st, CgHit &hit)
{
    int o[6];
    hit.adapter = -1; hit.remove = 0;
    hit.astart = hit.astop = hit.rstart = hit.rstop = hit.score = hit.errors = 0;
    if (!loc_state_result(st, o)) return;
    hit.adapter = 0;
    if (A.reverse) {
        hit.astart = A.m - o[1]; hit.astop = A.m - o[0];
        hit.rstart = n - o[3]; hit.rstop = n - o[2];
    } else {
        hit.astart = o[0]; hit.astop = o[1]; hit.rstart = o[2]; hit.rstop = o[3];
    }
    hit.score = o[4]; hit.errors = o[5];
    hit.remove = A.remove == CGK_REMOVE_AUTO ? (hit.rstart == 0 ? CGK_REMOVE_BEFORE : CGK_REMOVE_AFTER)
                                            : A.remove;
}

// Main pass.  Returns true when the read is finished (hit is valid); false when its end window is
// still to be done (st carries the selection state).  ALL lanes of a warp must call it.
template <int MR>
CG_HD bool split_main_pass(const SetView &S, const uint8_t *p, int n, uint32_t hits, int gs, uint32_t rs0,
                           uint32_t rs1, bool has_task, CgHit &hit, LocState &st)
{
    const CgAdapter &A = S.ad[0];
    ReadView rv; rv.p = p; rv.n = n; rv.rev = A.reverse;
    const int32_t *ncnt = (const int32_t *)(S.pool + A.ncount_off);
    const int32_t *maxcost = (const int32_t *)(S.pool + A.maxcost_off);
    const uint32_t *peq = (const uint32_t *)(S.pool + A.peq_off);
    RunList R;
    R.n = 0; R.lo0 = R.hi0 = R.lo1 = R.hi1 = R.lo2 = R.hi2 = 0;
    bool split = false;
    if (has_task) {
        if (simple_windowed(S, n)) {
            // runs around the locator hits only; the end window (needed by the last-column scan of
            // 3' adapters) is a separate pass unless a hit run already covers it.  Every bottom-row
            // cell with cost <= k lies inside a hit run, so the end pass has none to evaluate.
            refine_runs(S.scan, S.h->scan_count, S.pool, A, rv, hits, gs, rs0, rs1, R, false);
            if (A.flags & 4) {
                const int lo_end = cg_max(0, n - 1 - A.m - A.k);
                if (R.n == 0) {
                    R.n = 1; R.lo0 = lo_end; R.hi0 = n;                  // nothing but the end window
                } else {
                    const int lo_last = R.n == 1 ? R.lo0 : (R.n == 2 ? R.lo1 : R.lo2);
                    const int hi_last = R.n == 1 ? R.hi0 : (R.n == 2 ? R.hi1 : R.hi2);
                    split = !(lo_last <= lo_end && hi_last == n);
                }
            }
        } else {
            int max_n = n, min_n = 0;
            if (!(A.flags & 2)) max_n = cg_min(n, A.m + A.k);
            if (!(A.flags & 8)) min_n = cg_max(0, n - A.m - A.k);
            R.n = 1; R.lo0 = min_n; R.hi0 = max_n;
        }
    }
    st = loc_state_init(A.m, n);
    locate_regs<MR>(A, ncnt, maxcost, peq, rv, R, R.n, has_task, !split, st);
    if (!has_task) return true;
    if (split && !st.stopped) return false;
    hit_from_state(A, n, st, hit);
    return true;
}

// End pass: `tail` points at the first byte that was fetched for the end window (read orientation:
// forward reads: byte lo_end of the trimmed read; reversed reads: byte 0).
template <int MR>
CG_HD void split_end_pass(const SetView &S, const uint8_t *tail, int n, bool has_task, LocState &st, CgHit &hit)
{
    const CgAdapter &A = S.ad[0];
    const int lo_end = cg_max(0, n - 1 - A.m - A.k);
    ReadView rv;
    rv.n = n; rv.rev = A.reverse;
    rv.p = A.reverse ? tail : tail - lo_end;       // rv.at(j) for j in [lo_end, n) stays inside the fetched bytes
    const int32_t *ncnt = (const int32_t *)(S.pool + A.ncount_off);
    const int32_t *maxcost = (const int32_t *)(S.pool + A.maxcost_off);
    const uint32_t *peq = (const uint32_t *)(S.pool + A.peq_off);
    RunList R;
    R.n = 1; R.lo0 = lo_end; R.hi0 = n; R.lo1 = R.hi1 = R.lo2 = R.hi2 = 0;
    locate_regs<MR>(A, ncnt, maxcost, peq, rv, R, 1, has_task, true, st, false);
    if (has_task) hit_from_state(A, n, st, hit);
}

CG_HD void process_read_simple(const SetView &S, const uint8_t *seq, const uint8_t *qual, int n,
                               int quality_trim, int cutoff_front, int cutoff_back, int qbase,
                               PackedCol &colp, cg_match_rec *out, int32_t *qtrim_out, int use_regs = 0)
{
    int s = 0, e = n;
    if (quality_trim) pre_trim_core(seq, qual, n, quality_trim, cutoff_front, cutoff_back, qbase, &s, &e);
    if (qtrim_out) { qtrim_out[0] = s; qtrim_out[1] = e; }
    CgHit hit; hit.adapter = -1; hit.remove = 0;
    hit.astart = hit.astop = hit.rstart = hit.rstop = hit.score = hit.errors = 0;
    if (use_regs == 3 && S.ad[0].m <= 32) {       // split scheduling: main pass, then the end pass if needed
        int gs3;
        const ScanOut sc3 = simple_scan(S, seq + s, e - s, &gs3);
        if (sc3.pass) {
            LocState st;
            const CgAdapter &A = S.ad[0];
            const int nn = e - s, lo_end = cg_max(0, nn - 1 - A.m - A.k);
            const uint8_t *tail = A.reverse ? seq + s : seq + s + lo_end;
            if (A.m <= 16) {
                if (!split_main_pass<16>(S, seq + s, nn, sc3.hits, gs3, sc3.rs0, sc3.rs1, true, hit, st))
                    split_end_pass<16>(S, tail, nn, true, st, hit);
            } else {
                if (!split_main_pass<32>(S, seq + s, nn, sc3.hits, gs3, sc3.rs0, sc3.rs1, true, hit, st))
                    split_end_pass<32>(S, tail, nn, true, st, hit);
            }
        }
        store_hit(out, hit, 0, e - s);
        return;
    }
    if (use_regs == 2 && S.ad[0].m <= 32) {
        RunList R;
        if (simple_scan_runs(S, seq + s, e - s, R)) {
            if (!simple_locate_runs(S, seq + s, e - s, R, true, hit)) hit.adapter = -1;
        }
        store_hit(out, hit, 0, e - s);
        return;
    }
    int gs;
    const ScanOut sc = simple_scan(S, seq + s, e - s, &gs);
    if (sc.pass) {
        const bool found = (use_regs && S.ad[0].m <= 32)
                               ? simple_locate_regs(S, seq + s, e - s, sc.hits, gs, sc.rs0, sc.rs1, true, hit)
                               : simple_locate(S, seq + s, e - s, sc.hits, gs, colp, hit);
        if (!found) hit.adapter = -1;
    }
    store_hit(out, hit, 0, e - s);
}




// ---------------------------------------------------------------------------------------
// Planned scheduling (split pipeline v2): scan -> plan (refine + classify) -> one DP run per round.
//
//  plan_runs()   exact end positions of the locator hits -> up to three hit runs (+ the end window
//                of 3' adapters as a separate last run unless a hit run covers it).
//                Exact-occurrence shortcut: if in the leftmost hit stretch every chunk of the adapter
//                ends at the position implied by one common start s0, and s0 is the smallest start
//                any hit of that stretch implies, the read contains the adapter exactly at s0 and the
//                reference would stop there with (0, m, s0, s0+m, m, 0): every earlier bottom-row
//                candidate contains a hit of this stretch, so it starts at >= s0 - k >= s0 - m/2 and
//                scores < m, hence is replaced at column s0+m and the exact match ends the search
//                (_align.pyx:521-533).  No DP is needed for such reads.
//  run_pass<MR>  one run of one read with the selection state carried in LocState.
// ---------------------------------------------------------------------------------------
struct RunPlan {
    int n_runs;                    // 0..4
    int lo0, hi0, lo1, hi1, lo2, hi2, lo3, hi3;
    int end_idx;                   // index of the pure end-window run (no bottom-row candidates), or -1
    int exact;                     // 1: finished by the exact-occurrence shortcut at start s0;
                                   // 2: by the end-overlap shortcut, s0 = overlap length
    int s0;
    int banded;                    // the hit runs come from the bit-plane stage's mask of ALL locator hits: run_band_d
};

// Rows of a hit run that no alignment through the run's hits can touch.  The mask M of the bit-plane stage holds every
// exact occurrence of a locator chunk, so every alignment with <= k errors in the read starts within k of a start s
// that some hit implies, and a run [lo, hi) = [s_min - k, s_max + m + k) (merged hits) holds all alignments of its
// hits.  A cell (i, j) on a path that started at read position c <= s_max + k with <= k errors has
// i >= (j - c) - k >= j - s_max - 2k: in the column computed at step t of the run (j = lo + t + 1) the rows
// i < t + 1 - d - 2k with d = s_max - lo = hi - m - k - lo cannot lie on such a path.  Their cells can neither be
// reported (a bottom-row cell with cost <= k is a full alignment, hence on such a path) nor win or tie the minimum
// of a cell that is (that would make an alignment from a later start succeed, which has a hit of its own inside
// the merged run), and the stale cells beyond the Ukkonen bound always enter with cost + 1 > k + 1: so the DP may
// treat them as infinite.  Not for runs that reach the end of the read (the last-column scan accepts partial
// adapters from any start) and not for adapters with a free adapter start.  Returns d, or -1: no band.
CG_HD int run_band_d(const CgAdapter &A, int n, int lo, int hi, bool hit_derived, bool is_end_run)
{
    const bool can = A.m <= 64 && !(A.flags & 1) && (A.flags & 2) && (A.flags & 8) && A.indel_cost == 1;
    if (!can || !hit_derived || is_end_run || hi >= n) return -1;
    const int d = hi - A.m - A.k - lo;
    return d >= 0 ? d : -1;
}

template <bool REV>
CG_HD void plan_hit_runs_dir(const CgScanWord *words, int n_words, const uint8_t *pool, const CgAdapter &A,
                             const uint8_t *first, int n, uint32_t hits, int gs, uint32_t rs0, uint32_t rs1,
                             bool want_exact, RunList &R, int &exact, int &s0_out)
{
    const int m = A.m, k = A.k;
    R.n = 0;
    R.lo0 = R.hi0 = R.lo1 = R.hi1 = R.lo2 = R.hi2 = 0;
    exact = 0; s0_out = 0;
    if (A.flags & 1) runs_add(R, 0, cg_min(n, m + k), n);              // START_IN_REFERENCE
    if (!hits) return;
    int n_loc = 0;
    for (int w = 0; w < n_words; ++w) n_loc += (words[w].type == CG_SCAN_WHOLE && words[w].loc_found) ? 1 : 0;
    // exact-occurrence shortcut over all locator words: every word's chunks must imply the same start
    // within the first stretch of hit groups
    bool ex_ok = want_exact;
    int ex_s0 = -1;
    for (int w = 0; w < n_words; ++w) {
        const CgScanWord &W = words[w];
        if (W.type != CG_SCAN_WHOLE || !W.loc_found) continue;
        CG_TABPTR(mask, (const uint32_t *)(pool + W.mask_off));
        CG_CHARPTR(ltab, pool + W.loc_off);
        const uint32_t init = W.init, locf = W.loc_found;
        const bool stash = n_loc == 1;
        uint32_t todo = hits, Rr = 0;
        int cur_p = -1, nh = 0, stretch = 0;
        int wlo = 0x3fffffff, whi = -1;
        int s0 = 0x3fffffff;           // smallest implied start in the first stretch ...
        uint32_t fm = 0;               // ... and the chunks (found bits) that imply exactly s0
        while (todo) {
            const int g = cg_ctz(todo);
            todo &= todo - 1;
            const int p_first = g << gs;
            const long long p_end_ll = ((long long)(g + 1)) << gs;
            const int p_end = p_end_ll > n ? n : (int)p_end_ll;
            if (cur_p != p_first) {
                if (cur_p >= 0) ++stretch;                       // a gap between hit groups
                if (whi >= 0) { runs_add(R, wlo, whi, n); wlo = 0x3fffffff; whi = -1; }
                if (stash && nh < 2) {
                    Rr = nh == 0 ? rs0 : rs1;
                } else {
                    Rr = 0;
                    const int q0 = cg_max(0, p_first - 31);
                    CG_CHARPTR(q, first + (REV ? -q0 : q0));
                    for (int i = q0; i < p_first; ++i) {
                        Rr = ((Rr << 1) | init) & CG_TAB32(mask, CG_CHAR(q));
                        q = REV ? q - 1 : q + 1;
                    }
                }
            }
            ++nh;
            // Chunk hits are queued (position, found bits) while the shift-and advances and handled after
            // the group, lane by lane: handled inside the character loop, the whole warp would execute the
            // handler at nearly every character because some lane always has a hit there.
            uint32_t q0 = 0, q1 = 0, q2 = 0, q3 = 0, qpa = 0, qpb = 0;
            int qn = 0;
            auto handle = [&](int p, uint32_t f) {
                while (f) {
                    const int b = cg_ctz(f);
                    f &= f - 1;
                    const int bmin = (int)CG_CHAR(ltab + 2 * b), bmax = (int)CG_CHAR(ltab + 2 * b + 1);
                    wlo = cg_min(wlo, p + 1 - bmax - k);
                    whi = cg_max(whi, p + 1 - bmin + m + k);
                    if (stretch == 0) {
                        const int s = p + 1 - bmin;
                        if (s < s0) { s0 = s; fm = 1u << b; }
                        else if (s == s0) fm |= 1u << b;
                    }
                }
            };
            auto flush = [&]() {
                for (int e = qn - 1; e >= 0; --e) {            // oldest first
                    const uint32_t f = e == 3 ? q3 : (e == 2 ? q2 : (e == 1 ? q1 : q0));
                    const uint32_t pw = e >= 2 ? qpb : qpa;
                    handle((int)((e & 1) ? (pw >> 16) : (pw & 0xffffu)), f);
                }
                qn = 0;
            };
            auto push = [&](int p, uint32_t f) {
                if (qn == 4) flush();
                q3 = q2; q2 = q1; q1 = q0; q0 = f;
                qpb = (qpb << 16) | (qpa >> 16);
                qpa = (qpa << 16) | (uint32_t)p;               // p <= 32255
                ++qn;
            };
            // (fetching the group as aligned words like the scan kernel does was measured 7 % slower here:
            // the unrolled body with its predicated queue pushes outweighs the saved byte loads)
            CG_CHARPTR(q, first + (REV ? -p_first : p_first));
            for (int p = p_first; p < p_end; ++p) {
                Rr = ((Rr << 1) | init) & CG_TAB32(mask, CG_CHAR(q));
                q = REV ? q - 1 : q + 1;
                const uint32_t f = Rr & locf;
                if (f) push(p, f);
            }
            flush();
            cur_p = p_end;
        }
        if (whi >= 0) runs_add(R, wlo, whi, n);
        if (fm == locf && s0 >= 0 && s0 + m <= n && (ex_s0 < 0 || ex_s0 == s0)) ex_s0 = s0;
        else ex_ok = false;
    }
    if (ex_ok && ex_s0 >= 0) { exact = 1; s0_out = ex_s0; }
}

// Runs from a bit-vector pass (Myers 1999, semi-global: free start in the read) over the whole
// searched sequence: D[m][j], the cost of the best alignment of the full adapter ending at column j,
// is tracked for every j; the reference evaluates a bottom-row candidate only where that cost is
// <= k (_align.pyx:496-533 with cost <= maxcost[eff] <= k), and such an alignment starts at a column
// >= j - m - k.  So the DP runs are the unions of [j - m - k, j] over the columns with D[m][j] <= k.
// The vertical deltas of the last column give cost(i, n) for every adapter prefix i, i.e. whether the
// last-column scan (_align.pyx:536-572) can accept anything; if not, no end run is needed.
template <class T>
CG_HD void plan_runs_myers_t(const CgAdapter &A, const uint32_t *peq, const int32_t *ncnt,
                             const int32_t *maxcost, const uint8_t *p, int n, RunList &R, bool &need_end)
{
    const int m = A.m, k = A.k;
    const bool sir = (A.flags & 1) != 0, eir = (A.flags & 4) != 0;
    const T mmask = m >= (int)(8 * sizeof(T)) ? (T) ~(T)0 : (T)(((T)1 << m) - 1);
    const T top = (T)1 << (m - 1);
    T Pv = sir ? (T)0 : mmask, Mv = 0;                     // column 0: cost i, or 0 (START_IN_REFERENCE)
    int score = sir ? 0 : m;
    CG_CHARPTR(cp, A.reverse ? p + (n - 1) : p);
    CG_TABPTR(peq_t, peq);
    const int cstride = A.reverse ? -1 : 1;
    int wlo = 0, whi = -1;
    for (int j = 1; j <= n; ++j) {
        const int ch = (int)(CG_CHAR(cp + cstride * (j - 1)) & 127u);
        T Eq = (T)CG_TAB32(peq_t, ch);
        if (sizeof(T) > 4) Eq |= (T)((unsigned long long)CG_TAB32(peq_t, 128 + ch) << 32);
        const T Xv = Eq | Mv;
        const T Xh = (T)((((Eq & Pv) + Pv) ^ Pv) | Eq);
        T Ph = (T)(Mv | ~(Xh | Pv));
        T Mh = Pv & Xh;
        score += (Ph & top) ? 1 : 0;
        score -= (Mh & top) ? 1 : 0;
        Ph = (T)(Ph << 1); Mh = (T)(Mh << 1);               // row 0 stays 0: START_IN_QUERY
        Pv = (T)(Mh | ~(Xv | Ph));
        Mv = Ph & Xv;
        if (score <= k) {
            const int lo = cg_max(0, j - m - k);
            if (whi < 0) wlo = lo;
            else if (lo > whi) { runs_add(R, wlo, whi, n); wlo = lo; }
            whi = j;
        }
    }
    if (whi >= 0) runs_add(R, wlo, whi, n);
    need_end = false;
    if (eir) {
        if (sir) need_end = true;                           // prefix length unknown (origin < 0 possible)
        else {
            int c = 0;
            for (int i = 1; i <= m; ++i) {
                c += (int)((Pv >> (i - 1)) & 1) - (int)((Mv >> (i - 1)) & 1);
                int eff = i;
                if (A.wildcard_ref) eff = (i < m) ? i - ncnt[i] : A.effective_length;
                if (i >= A.min_overlap && c <= maxcost[eff]) { need_end = true; break; }
            }
        }
    }
}

// End-of-read shortcut for reads without any locator hit (no full-adapter alignment with <= k errors
// exists, so only the last-column scan, _align.pyx:536-572, can produce a result).  A bit-vector pass
// over the end window [lo_end, n] (same restart as the end run) gives cost(i, n) for every adapter
// prefix i.  The scan walks i downwards with no best match yet, so the first acceptable i wins and a
// later (shorter) one replaces it only with a higher score; if every acceptable cell has cost 0 (an
// exact overlap: score = i) that never happens and the result is the longest exact overlap
// (0, i, n - i, n, i, 0).  Returns -1: some acceptable cell has errors (run the DP), 0: nothing is
// acceptable, i > 0: the result is the exact overlap of length i.
template <class T>
CG_HD int end_overlap_myers_t(const CgAdapter &A, const uint32_t *peq, const int32_t *ncnt,
                              const int32_t *maxcost, const uint8_t *p, int n, int lo_end)
{
    const int m = A.m;
    const T mmask = m >= (int)(8 * sizeof(T)) ? (T) ~(T)0 : (T)(((T)1 << m) - 1);
    T Pv = mmask, Mv = 0;                                   // restart column: cost i
    CG_CHARPTR(cp, A.reverse ? p + (n - 1) : p);
    CG_TABPTR(peq_t, peq);
    const int cstride = A.reverse ? -1 : 1;
    for (int j = lo_end + 1; j <= n; ++j) {
        const int ch = (int)(CG_CHAR(cp + cstride * (j - 1)) & 127u);
        T Eq = (T)CG_TAB32(peq_t, ch);
        if (sizeof(T) > 4) Eq |= (T)((unsigned long long)CG_TAB32(peq_t, 128 + ch) << 32);
        const T Xv = Eq | Mv;
        const T Xh = (T)((((Eq & Pv) + Pv) ^ Pv) | Eq);
        T Ph = (T)(Mv | ~(Xh | Pv));
        T Mh = Pv & Xh;
        Ph = (T)(Ph << 1); Mh = (T)(Mh << 1);               // row 0 stays 0: START_IN_QUERY
        Pv = (T)(Mh | ~(Xv | Ph));
        Mv = Ph & Xv;
    }
    int c = 0, best = 0;
    bool inexact = false;
    for (int i = 1; i <= m; ++i) {
        c += (int)((Pv >> (i - 1)) & 1) - (int)((Mv >> (i - 1)) & 1);
        int eff = i;
        if (A.wildcard_ref) eff = (i < m) ? i - ncnt[i] : A.effective_length;
        if (i >= A.min_overlap && c <= maxcost[eff]) {
            if (c == 0) best = i; else inexact = true;
        }
    }
    return inexact ? -1 : best;
}

// Does the restarted DP of the run [lo, hi] ever see a bottom-row cell with cost <= k?  The same bit-vector pass
// as plan_runs_myers_t, restarted at column lo like the run (column lo: cost i; row 0 free): D'[m][j] for
// j in (lo, hi].  The reference evaluates a bottom-row candidate only where that cost is <= k
// (_align.pyx:490-514), so a run without such a column changes nothing and can be dropped -- a locator chunk
// that occurs by chance, far from any real occurrence of the adapter.
template <class T>
CG_HD bool run_has_candidate_t(const CgAdapter &A, const uint32_t *peq, const uint8_t *p, int n, int lo, int hi)
{
    const int m = A.m, k = A.k;
    const T mmask = m >= (int)(8 * sizeof(T)) ? (T) ~(T)0 : (T)(((T)1 << m) - 1);
    const T top = (T)1 << (m - 1);
    T Pv = mmask, Mv = 0;
    int score = m;
    CG_CHARPTR(cp, A.reverse ? p + (n - 1) : p);
    CG_TABPTR(peq_t, peq);
    const int cstride = A.reverse ? -1 : 1;
    bool any = false;
    for (int j = lo + 1; j <= hi; ++j) {
        const int ch = (int)(CG_CHAR(cp + cstride * (j - 1)) & 127u);
        T Eq = (T)CG_TAB32(peq_t, ch);
        if (sizeof(T) > 4) Eq |= (T)((unsigned long long)CG_TAB32(peq_t, 128 + ch) << 32);
        const T Xv = Eq | Mv;
        const T Xh = (T)((((Eq & Pv) + Pv) ^ Pv) | Eq);
        T Ph = (T)(Mv | ~(Xh | Pv));
        T Mh = Pv & Xh;
        score += (Ph & top) ? 1 : 0;
        score -= (Mh & top) ? 1 : 0;
        Ph = (T)(Ph << 1); Mh = (T)(Mh << 1);
        Pv = (T)(Mh | ~(Xv | Ph));
        Mv = Ph & Xv;
        any = any || score <= k;
    }
    return any;
}

// Second half of the plan for windowed adapters: R = the runs around the locator hits (a superset is fine).
//   * hit runs that are not also the final run are dropped when they hold no bottom-row candidate;
//   * the end window of a 3' adapter (last-column scan, _align.pyx:536-572) is needed only if some cell
//     (i, n) is acceptable; if nothing else is left and every acceptable cell is an exact overlap, the
//     result is the longest one (end_overlap_myers_t).
CG_HD void plan_finish(const SetView &S, const uint8_t *p, int n, const RunList &R0, RunPlan &P, bool skip_end = false)
{
    const CgAdapter &A = S.ad[0];
    const int32_t *ncnt = (const int32_t *)(S.pool + A.ncount_off);
    const int32_t *maxcost = (const int32_t *)(S.pool + A.maxcost_off);
    const uint32_t *peq = (const uint32_t *)(S.pool + A.peq_off);
    const bool eir = (A.flags & 4) != 0;
    const int lo_end = cg_max(0, n - 1 - A.m - A.k);
    const bool can_filter = A.m <= 64 && !(A.flags & 1) && (A.flags & 2) && (A.flags & 8) && A.indel_cost == 1;
    RunList R;
    R.n = 0; R.lo0 = R.hi0 = R.lo1 = R.hi1 = R.lo2 = R.hi2 = 0;
    bool covered = false;                             // the last kept run is also the end window
    for (int r = 0; r < R0.n; ++r) {
        const int lo = r == 0 ? R0.lo0 : (r == 1 ? R0.lo1 : R0.lo2);
        const int hi = r == 0 ? R0.hi0 : (r == 1 ? R0.hi1 : R0.hi2);
        const bool is_final = eir && r == R0.n - 1 && lo <= lo_end && hi == n;
        bool keep = true;
        if (can_filter && !is_final)
            keep = A.m <= 32 ? run_has_candidate_t<uint32_t>(A, peq, p, n, lo, hi)
                             : run_has_candidate_t<unsigned long long>(A, peq, p, n, lo, hi);
        if (!keep) continue;
        if (R.n == 0) { R.lo0 = lo; R.hi0 = hi; }
        else if (R.n == 1) { R.lo1 = lo; R.hi1 = hi; }
        else { R.lo2 = lo; R.hi2 = hi; }
        ++R.n;
        covered = is_final;
    }
    P.n_runs = R.n; P.lo0 = R.lo0; P.hi0 = R.hi0; P.lo1 = R.lo1; P.hi1 = R.hi1; P.lo2 = R.lo2; P.hi2 = R.hi2;
    if (!eir || covered || skip_end) return;
    if (can_filter) {                                 // what can the last-column scan accept?
        const int r = A.m <= 32 ? end_overlap_myers_t<uint32_t>(A, peq, ncnt, maxcost, p, n, lo_end)
                                : end_overlap_myers_t<unsigned long long>(A, peq, ncnt, maxcost, p, n, lo_end);
        if (r == 0) return;                           // nothing: no end window
        if (r > 0 && R.n == 0) { P.exact = 2; P.s0 = r; return; }
    }
    // every bottom-row cell with cost <= k lies inside a hit run, so the separate end window has none to evaluate
    P.end_idx = R.n;
    if (R.n == 0) { P.lo0 = lo_end; P.hi0 = n; }
    else if (R.n == 1) { P.lo1 = lo_end; P.hi1 = n; }
    else if (R.n == 2) { P.lo2 = lo_end; P.hi2 = n; }
    else { P.lo3 = lo_end; P.hi3 = n; }
    P.n_runs = R.n + 1;
}

CG_HD void plan_runs(const SetView &S, const uint8_t *p, int n, uint32_t hits, int gs, uint32_t rs0,
                     uint32_t rs1, RunPlan &P)
{
    const CgAdapter &A = S.ad[0];
    P.n_runs = 0; P.lo0 = P.hi0 = P.lo1 = P.hi1 = P.lo2 = P.hi2 = P.lo3 = P.hi3 = 0;
    P.end_idx = -1; P.exact = 0; P.s0 = 0; P.banded = 0;
    if (S.h->myers && (A.flags & 2) && (A.flags & 8) && n > 0) {
        const int32_t *ncnt = (const int32_t *)(S.pool + A.ncount_off);
        const int32_t *maxcost = (const int32_t *)(S.pool + A.maxcost_off);
        const uint32_t *peq = (const uint32_t *)(S.pool + A.peq_off);
        RunList R;
        R.n = 0; R.lo0 = R.hi0 = R.lo1 = R.hi1 = R.lo2 = R.hi2 = 0;
        bool need_end;
        if (A.m <= 32) plan_runs_myers_t<uint32_t>(A, peq, ncnt, maxcost, p, n, R, need_end);
        else plan_runs_myers_t<unsigned long long>(A, peq, ncnt, maxcost, p, n, R, need_end);
        P.n_runs = R.n; P.lo0 = R.lo0; P.hi0 = R.hi0; P.lo1 = R.lo1; P.hi1 = R.hi1; P.lo2 = R.lo2; P.hi2 = R.hi2;
        if (need_end) {
            const int lo_end = cg_max(0, n - 1 - A.m - A.k);
            bool covered = false;
            if (R.n > 0) {
                const int lo_last = R.n == 1 ? R.lo0 : (R.n == 2 ? R.lo1 : R.lo2);
                const int hi_last = R.n == 1 ? R.hi0 : (R.n == 2 ? R.hi1 : R.hi2);
                covered = lo_last <= lo_end && hi_last == n;
            }
            if (!covered) {
                P.end_idx = R.n;
                if (R.n == 0) { P.lo0 = lo_end; P.hi0 = n; }
                else if (R.n == 1) { P.lo1 = lo_end; P.hi1 = n; }
                else if (R.n == 2) { P.lo2 = lo_end; P.hi2 = n; }
                else { P.lo3 = lo_end; P.hi3 = n; }
                P.n_runs = R.n + 1;
            }
        }
        return;
    }
    if (!simple_windowed(S, n)) {
        // plain: one run over the reference's column range (_align.pyx:346-352)
        int max_n = n, min_n = 0;
        if (!(A.flags & 2)) max_n = cg_min(n, A.m + A.k);
        if (!(A.flags & 8)) min_n = cg_max(0, n - A.m - A.k);
        P.n_runs = 1; P.lo0 = min_n; P.hi0 = max_n;
        return;
    }
    RunList R;
    const bool want_exact = S.h->exact_ok != 0;
    if (A.reverse) plan_hit_runs_dir<true>(S.scan, S.h->scan_count, S.pool, A, p + (n - 1), n, hits, gs, rs0, rs1, want_exact, R, P.exact, P.s0);
    else plan_hit_runs_dir<false>(S.scan, S.h->scan_count, S.pool, A, p, n, hits, gs, rs0, rs1, want_exact, R, P.exact, P.s0);
    if (P.exact) return;
    plan_finish(S, p, n, R, P);
}

// Is every character of the window a plain A/C/G/T (either case)?  Then the bit-plane stage saw the read exactly
// as KmerFinder.kmers_present and the locator do (any other byte aliases one of the four letters in the planes).
CG_HD bool window_is_plain(const uint8_t *p, int n)
{
    // Four characters per aligned word.  A byte c is one of A C G T a c g t iff
    //   bit 7 = 0, bit 3 = 0, bit 6 = 1            (bit 5 is the case bit),
    //   bit 4 = bit 2 & ~bit 1                     (only T, 101_0100, has bit 4; it is the code with bit 2 and not bit 1),
    //   bit 0 != bit 4                             (A C G end in 1, T in 0).
    // The three conditions are accumulated over the words (two ORs of violations, one AND for bit 6); the bytes
    // of the first and last word that lie outside the window are replaced by 'A'.
    if (n <= 0) return true;
    const uint32_t mis = (uint32_t)((uintptr_t)p & 3u);
    const int total = n + (int)mis;                        // bytes from the aligned start
    const int n_words = (total + 3) >> 2;
#if defined(__CUDA_ARCH__)
    const uint32_t base = (uint32_t)__cvta_generic_to_shared(p - mis);
#define CG_PLAIN_WORD(i) cg_lds_u32(base + 4u * (uint32_t)(i))
#else
    const uint8_t *base = p - mis;
#define CG_PLAIN_WORD(i) ((uint32_t)base[4 * (i)] | ((uint32_t)base[4 * (i) + 1] << 8) | ((uint32_t)base[4 * (i) + 2] << 16) | \
                          ((uint32_t)base[4 * (i) + 3] << 24))
#endif
    uint32_t hi_or = 0, lo_or = 0, six_and = 0xFFFFFFFFu;
    auto take = [&](uint32_t w) {
        const uint32_t s1 = w >> 1, s2 = w >> 2, s4 = w >> 4;
        hi_or |= w & 0x88888888u;                                      // bits 7 and 3 must be clear
        six_and &= w;                                                  // bit 6 must be set
        lo_or |= ((s2 & ~s1) ^ s4) | ~(w ^ s4);                        // bit 0 of every byte: a violation
    };
    // first and last word: the bytes outside the window count as 'A'; the words between them need no masks
    uint32_t keep0 = 0xFFFFFFFFu << (8 * mis);
    const uint32_t keep_last = (total & 3) ? 0xFFFFFFFFu >> (8 * (4 - (total & 3))) : 0xFFFFFFFFu;
    if (n_words == 1) keep0 &= keep_last;
    take((CG_PLAIN_WORD(0) & keep0) | (0x41414141u & ~keep0));
#pragma unroll 4
    for (int i = 1; i < n_words - 1; ++i) take(CG_PLAIN_WORD(i));
    if (n_words > 1) take((CG_PLAIN_WORD(n_words - 1) & keep_last) | (0x41414141u & ~keep_last));
#undef CG_PLAIN_WORD
    return hi_or == 0 && (six_and & 0x40404040u) == 0x40404040u && (lo_or & 0x01010101u) == 0;
}

// The plan of a read whose locator hits come from the bit-plane stage: M (W words, plane indices) marks the
// adapter ends the chunk hits point at, off0 is the plane index of the window's first character.  A hit that
// implies the adapter start s gives the run [s - k, s + m + k] (the same window refine_runs /
// plan_hit_runs_dir derive from a chunk's end position).
CG_HD void plan_runs_planes(const SetView &S, const uint8_t *p, int n, const uint32_t *M, int W, int end_hit,
                            int no_end, int off0, RunPlan &P)
{
    const CgAdapter &A = S.ad[0];
    P.n_runs = 0; P.lo0 = P.hi0 = P.lo1 = P.hi1 = P.lo2 = P.hi2 = P.lo3 = P.hi3 = 0;
    P.end_idx = -1; P.exact = 0; P.s0 = 0; P.banded = 1;
    RunList R;
    R.n = 0; R.lo0 = R.hi0 = R.lo1 = R.hi1 = R.lo2 = R.hi2 = 0;
    if (A.flags & 1) runs_add(R, 0, cg_min(n, A.m + A.k), n);              // START_IN_REFERENCE
#pragma unroll
    for (int b = 0; b < 8; ++b) {                  // (unrolled: M stays in registers)
        uint32_t x = b < W ? M[b] : 0u;
        while (x) {
            const int e = 32 * b + cg_ctz(x);
            x &= x - 1;
            const int s = e - (A.m - 1) - off0;
            runs_add(R, s - A.k, s + A.m + A.k, n);
        }
    }
    // a chunk so close to the end that the whole adapter would not fit: its window lies inside the end window
    if (end_hit) runs_add(R, cg_max(0, n - 1 - A.m - A.k), n, n);
    // no_end: the bit-plane stage has shown that the last-column scan cannot accept anything
    plan_finish(S, p, n, R, P, no_end != 0 && !end_hit);
}

// P.exact == 2: the exact overlap of the adapter's first `len` characters with the end of the read
CG_HD void hit_end_overlap(const CgAdapter &A, int n, int len, CgHit &hit)
{
    LocState st = loc_state_init(A.m, n);
    st.have = 1; st.b_origin = n - len; st.b_cost = 0; st.b_score = len; st.b_ref_stop = len; st.b_q_stop = n;
    hit_from_state(A, n, st, hit);
}

CG_HD void hit_exact(const CgAdapter &A, int n, int s0, CgHit &hit)
{
    // (0, m, s0, s0 + m, m, 0), mirrored for reversed reads like adapters.py:777-785
    hit.adapter = 0;
    if (A.reverse) { hit.astart = 0; hit.astop = A.m; hit.rstart = n - (s0 + A.m); hit.rstop = n - s0; }
    else { hit.astart = 0; hit.astop = A.m; hit.rstart = s0; hit.rstop = s0 + A.m; }
    hit.score = A.m; hit.errors = 0;
    hit.remove = A.remove == CGK_REMOVE_AUTO ? (hit.rstart == 0 ? CGK_REMOVE_BEFORE : CGK_REMOVE_AFTER)
                                            : A.remove;
}

// One run [lo, hi] of one read.  `bytes` points at the first fetched byte: read-orientation bytes
// [lo, hi) for forward reads, [n - hi, n - lo) for reversed reads.  ALL lanes of a warp must call it.
template <int MR>
CG_HD void run_pass(const SetView &S, const uint8_t *bytes, int n, int lo, int hi, bool eval_bottom,
                    bool final_scan, bool has_task, LocState &st, int band_d = -1)
{
    const CgAdapter &A = S.ad[0];
    ReadView rv;
    rv.n = n; rv.rev = A.reverse;
    rv.p = A.reverse ? bytes - (n - hi) : bytes - lo;
    const int32_t *ncnt = (const int32_t *)(S.pool + A.ncount_off);
    const int32_t *maxcost = (const int32_t *)(S.pool + A.maxcost_off);
    const uint32_t *peq = (const uint32_t *)(S.pool + A.peq_off);
    RunList R;
    R.n = 1; R.lo0 = lo; R.hi0 = hi; R.lo1 = R.hi1 = R.lo2 = R.hi2 = 0;
    // free start in the read bounds every cost by the row number, so short adapters never saturate
    // (run_pass is only called with the run's bytes staged in shared memory on the device)
    if (MR <= 16 && (A.flags & 2)) locate_regs<MR, true, true, CG_RUN_BAND != 0>(A, ncnt, maxcost, peq, rv, R, 1, has_task, final_scan, st, eval_bottom, band_d);
    else locate_regs<MR, false, true, CG_RUN_BAND != 0>(A, ncnt, maxcost, peq, rv, R, 1, has_task, final_scan, st, eval_bottom, band_d);
}

// The DP rounds of a planned read (what the cg_list_kernel<run> rounds do), host-sim only.
CG_HD void finish_planned(const SetView &S, const uint8_t *w, int nn, const RunPlan &P, CgHit &hit)
{
    const CgAdapter &A = S.ad[0];
    if (P.exact == 2) hit_end_overlap(A, nn, P.s0, hit);
    else if (P.exact) hit_exact(A, nn, P.s0, hit);
    else {
        LocState st = loc_state_init(A.m, nn);
        for (int r = 0; r < P.n_runs && !st.stopped; ++r) {
            const int lo = r == 0 ? P.lo0 : (r == 1 ? P.lo1 : (r == 2 ? P.lo2 : P.lo3));
            const int hi = r == 0 ? P.hi0 : (r == 1 ? P.hi1 : (r == 2 ? P.hi2 : P.hi3));
            const uint8_t *bytes = A.reverse ? w + (nn - hi) : w + lo;
            const bool last = r == P.n_runs - 1;
            const int band = run_band_d(A, nn, lo, hi, P.banded != 0, r == P.end_idx);
            if (A.m <= 16) run_pass<16>(S, bytes, nn, lo, hi, r != P.end_idx, last, true, st, band);
            else if (A.m <= 32) run_pass<32>(S, bytes, nn, lo, hi, r != P.end_idx, last, true, st, band);
            else if (A.m <= 48) run_pass<48>(S, bytes, nn, lo, hi, r != P.end_idx, last, true, st, band);
            else run_pass<64>(S, bytes, nn, lo, hi, r != P.end_idx, last, true, st, band);
        }
        hit_from_state(A, nn, st, hit);
    }
}

// Host-sim driver of the planned scheduling for one read (tests/hostsim, mode 64).
CG_HD void process_read_planned(const SetView &S, const uint8_t *seq, const uint8_t *qual, int n,
                                int quality_trim, int cutoff_front, int cutoff_back, int qbase,
                                cg_match_rec *out, int32_t *qtrim_out)
{
    int s = 0, e = n;
    if (quality_trim) pre_trim_core(seq, qual, n, quality_trim, cutoff_front, cutoff_back, qbase, &s, &e);
    if (qtrim_out) { qtrim_out[0] = s; qtrim_out[1] = e; }
    CgHit hit; hit.adapter = -1; hit.remove = 0;
    hit.astart = hit.astop = hit.rstart = hit.rstop = hit.score = hit.errors = 0;
    const CgAdapter &A = S.ad[0];
    const int nn = e - s;
    int gs;
    const ScanOut sc = simple_scan(S, seq + s, nn, &gs);
    if (sc.pass) {
        RunPlan P;
        plan_runs(S, seq + s, nn, sc.hits, gs, sc.rs0, sc.rs1, P);
        finish_planned(S, seq + s, nn, P, hit);
    }
    store_hit(out, hit, 0, nn);
}

// Host-sim driver of the bit-plane first stage (tests/hostsim, mode 256): plane_scan_core decides what it
// can, everything else takes the planned scheduling above -- exactly what cg_pscan_kernel + cg_list_kernel do.
CG_HD const uint32_t *plane_program(const SetView &S)
{
    return (const uint32_t *)((const uint8_t *)S.h + S.h->plane_off);
}

CG_HD void process_read_planes(const SetView &S, const uint8_t *seq, const uint8_t *qual, int n,
                               int quality_trim, int cutoff_front, int cutoff_back, int qbase,
                               cg_match_rec *out, int32_t *qtrim_out)
{
    int s = 0, e = n;
    if (quality_trim) pre_trim_core(seq, qual, n, quality_trim, cutoff_front, cutoff_back, qbase, &s, &e);
    if (qtrim_out) { qtrim_out[0] = s; qtrim_out[1] = e; }
    const CgAdapter &A = S.ad[0];
    const int nn = e - s;
    if (S.h->plane_count > 0 && nn >= 1 && nn <= 256) {
        const uint8_t *ref = S.pool + A.ref_off;
        const PlaneOut po = nn <= 160
            ? plane_scan_core<5, RuntimePlaneProg>(plane_program(S), S.h->plane_count, S.h->plane_flags, A.m, ref, seq + e, nn, A.pf_count == 0)
            : plane_scan_core<8, RuntimePlaneProg>(plane_program(S), S.h->plane_count, S.h->plane_flags, A.m, ref, seq + e, nn, A.pf_count == 0);
        if (po.cls != CG_PLANE_SLOW) {
            CgHit hit; hit.adapter = -1; hit.remove = 0;
            hit.astart = hit.astop = hit.rstart = hit.rstop = hit.score = hit.errors = 0;
            if (po.cls == CG_PLANE_EXACT) hit_exact(A, nn, po.s0, hit);
            else if (po.cls == CG_PLANE_OVERLAP) hit_end_overlap(A, nn, po.s0, hit);
            store_hit(out, hit, 0, nn);
            return;
        }
        if (window_is_plain(seq + s, nn)) {   // plan from the planes' hits, then the DP runs (cg_list_kernel)
            const int W = nn <= 160 ? 5 : 8;
            RunPlan P;
            plan_runs_planes(S, seq + s, nn, po.M, W, po.end_hit, po.no_end, 32 * W - nn, P);
            CgHit hit; hit.adapter = -1; hit.remove = 0;
            hit.astart = hit.astop = hit.rstart = hit.rstop = hit.score = hit.errors = 0;
            finish_planned(S, seq + s, nn, P, hit);
            store_hit(out, hit, 0, nn);
            return;
        }
    }
    process_read_planned(S, seq + s, nullptr, nn, 0, 0, 0, qbase, out, nullptr);
}
