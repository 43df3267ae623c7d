// cg_fastq_core.cuh -- per-record logic of the FASTQ path (cg_fastq.cu), host + device.
//
// What is left of a read after the modifier chain, which filters it fails, and the verdict on a read or a pair.
// The CUDA kernels call these functions one thread per record; tests/hostsim compiles them for the host so that the
// logic is fuzzed against the oracle without a GPU (test infrastructure, not a fallback).
#pragma once
#include "cg_core.cuh"

struct CgFastqRecord {       // one 4-line record of the chunk
    uint32_t hdr_start;      // first character of the name (after '@')
    int32_t hdr_len;
    uint32_t seq_start;
    uint32_t qual_start;
};
struct CgFastqFilter {
    int minimum_length;      // 0 = off
    int maximum_length;      // < 0 = off
    int discard_trimmed, discard_untrimmed;
    double max_n;            // < 0 = off; < 1: proportion of the length
    double max_ee;           // < 0 = off
    int poly_a;              // PolyATrimmer after the adapter rounds: 1 = poly-A tail (R1), 2 = poly-T head (R2)
    int shorten;             // Shortener: 0 = off, L + 1 for --length L >= 0, L for --length L < 0
    int trim_n;              // NEndTrimmer
    int discard_casava;      // CasavaFiltered
    int action;              // CG_FQ_ACTION_*: AdapterCutter's action
    double max_aer = 0.0;    // TooHighAverageErrorRate: expected errors per base above this fail; 0 = off
    int zero_cap = 0;        // ZeroCapper: quality characters below this one (the quality base) become it; 0 = off
};
#define CG_FQ_ACTION_TRIM 0
#define CG_FQ_ACTION_NONE 1
#define CG_FQ_ACTION_MASK 2
#define CG_FQ_ACTION_LOWERCASE 3
#define CG_FQ_ACTION_RETAIN 4
#define CG_FQ_ACTION_CROP 5
// fail_mask word of a record: bits 0-7 failed filters, bits 8-29 adapter of the most recent match + 1,
// bit 30: the record was replaced by its reverse complement (--revcomp)
#define CG_FQ_MASK_RC (1 << 30)
#define CG_FQ_MASK_ADAPTER(mask) ((((mask) >> 8) & 0x3FFFFF) - 1)

// SequenceRecord.reverse_complement of dnaio: IUPAC-aware, case preserved, every other character unchanged
CG_HD uint8_t fq_complement(uint8_t c)
{
    const uint8_t u = (uint8_t)(c & ~0x20), low = (uint8_t)(c & 0x20);
    uint8_t o;
    switch (u) {
    case 'A': o = 'T'; break; case 'C': o = 'G'; break; case 'G': o = 'C'; break; case 'T': o = 'A'; break;
    case 'U': o = 'A'; break; case 'M': o = 'K'; break; case 'R': o = 'Y'; break; case 'Y': o = 'R'; break;
    case 'K': o = 'M'; break; case 'V': o = 'B'; break; case 'H': o = 'D'; break; case 'D': o = 'H'; break;
    case 'B': o = 'V'; break;
    default: return c;          // W, S, N and everything that is not a nucleotide code
    }
    return (uint8_t)(o | low);
}

// line k of the chunk: [start, end) without the line terminator ("\n" or "\r\n"); nl_pos = positions of all
// newlines, n = size of the chunk (the last line may lack its newline)
CG_HD void fq_line_span(const uint8_t *buf, const uint32_t *nl_pos, long long n_nl, long long n, long long k,
                        uint32_t *start, uint32_t *end)
{
    const uint32_t s = k == 0 ? 0u : nl_pos[k - 1] + 1u;
    uint32_t e = k < n_nl ? nl_pos[k] : (uint32_t)n;
    if (e > s && buf[e - 1] == '\r') --e;
    *start = s; *end = e;
}

// Record r = lines 4r .. 4r+3.  Checks what dnaio's parser checks: 1 = the record does not start with '@',
// 2 = the third line does not start with '+', 3 = sequence and qualities differ in length, 5 = the description
// repeated after the '+' differs from the first one; 0 = fine.
// cut_front / cut_back: UnconditionalCutter (-u, modifiers.py:66-95), the first modifier of the chain: the record
// table simply describes the read without those bases (read[cut_front:] then read[:-cut_back]).
// *full_len: the length before -u (what the pipeline counts as "bp processed", pipeline.py:58-64, 142-143).
CG_HD int fq_record_core(const uint8_t *buf, long long n, const uint32_t *nl_pos, long long n_nl, long long r,
                         int cut_front, int cut_back, CgFastqRecord *rec, int *seq_len, int *full_len = nullptr,
                         int *cut_applied = nullptr)
{
    uint32_t hs, he, ss, se, ps, pe, qs, qe;
    fq_line_span(buf, nl_pos, n_nl, n, 4 * r, &hs, &he);
    fq_line_span(buf, nl_pos, n_nl, n, 4 * r + 1, &ss, &se);
    fq_line_span(buf, nl_pos, n_nl, n, 4 * r + 2, &ps, &pe);
    fq_line_span(buf, nl_pos, n_nl, n, 4 * r + 3, &qs, &qe);
    int bad = 0;
    if (he == hs || buf[hs] != '@') bad = 1;
    else if (pe == ps || buf[ps] != '+') bad = 2;
    else if (pe - ps > 1) {
        // a repeated description after the '+' must equal the first one (dnaio: "Sequence descriptions don't match")
        bool same = pe - ps == he - hs;
        for (uint32_t j = 1; same && j < pe - ps; ++j) same = buf[ps + j] == buf[hs + j];
        if (!same) bad = 5;
    }
    if (!bad && se - ss != qe - qs) bad = 3;
    int len = bad ? 0 : (int32_t)(se - ss);
    if (full_len) *full_len = len;
    const int cf = cut_front < len ? cut_front : len;
    len -= cf;
    len = cut_back < len ? len - cut_back : 0;
    if (cut_applied) *cut_applied = cf;
    rec->hdr_start = hs + 1;                    // without the '@'
    rec->hdr_len = (int32_t)(he - hs) - 1;
    rec->seq_start = ss + (uint32_t)cf;
    rec->qual_start = qs + (uint32_t)cf;
    *seq_len = len;
    return bad;
}

// ---- FASTA (cg_fastq_params.format 1) ----
// A chunk is first rewritten into a normalised buffer in which every record is ">name\n" followed by its whole
// sequence (no line breaks, no '\r'); the record table then describes that buffer with an empty quality span.
#define CG_FA_LINE_SEQUENCE 0
#define CG_FA_LINE_HEADER 1
#define CG_FA_LINE_COMMENT 2
#define CG_FA_ERR_BEFORE_HEADER 6     // a line before the first header that is not a '#' comment
#define CG_FA_ERR_LATE_COMMENT 7      // a '#' line after the first header

// Line k of a FASTA chunk: its kind and how many bytes it keeps in the normalised buffer (a header keeps itself,
// '>' included, plus '\n'; a sequence line its characters; a '#' line nothing).  [*start, *end): the line without
// its terminator ("\n" or "\r\n").
CG_HD int fa_line_core(const uint8_t *buf, const uint32_t *nl_pos, long long n_nl, long long n, long long k, uint32_t *start,
                       uint32_t *end, int *keep)
{
    fq_line_span(buf, nl_pos, n_nl, n, k, start, end);
    const int len = (int)(*end - *start);
    const uint8_t c = len ? buf[*start] : 0;
    if (c == '>') { *keep = len + 1; return CG_FA_LINE_HEADER; }
    if (c == '#') { *keep = 0; return CG_FA_LINE_COMMENT; }
    *keep = len;
    return CG_FA_LINE_SEQUENCE;
}

// Is line k (of kind `kind`) allowed, given the first header line of the chunk (first_hdr: larger than every line
// number if there is none)?  '#' lines are comments only in front of the first record; any other line there is an
// error.  Returns 0 or CG_FA_ERR_*.
CG_HD int fa_line_error(int kind, long long k, long long first_hdr)
{
    if (kind == CG_FA_LINE_COMMENT) return k > first_hdr ? CG_FA_ERR_LATE_COMMENT : 0;
    if (kind == CG_FA_LINE_SEQUENCE && k < first_hdr) return CG_FA_ERR_BEFORE_HEADER;
    return 0;
}

// Record of the normalised buffer whose name is [hdr_start, hdr_start + hdr_len) and whose sequence runs from
// hdr_start + hdr_len + 1 to seq_end; -u and the bases read as in fq_record_core.
CG_HD void fa_record_core(uint32_t hdr_start, int hdr_len, uint32_t seq_end, int cut_front, int cut_back, CgFastqRecord *rec,
                          int *seq_len, int *full_len, int *cut_applied)
{
    const uint32_t ss = hdr_start + (uint32_t)hdr_len + 1u;
    int len = (int)(seq_end - ss);
    *full_len = len;
    const int cf = cut_front < len ? cut_front : len;
    len -= cf;
    len = cut_back < len ? len - cut_back : 0;
    *cut_applied = cf;
    rec->hdr_start = hdr_start;
    rec->hdr_len = hdr_len;
    rec->seq_start = ss + (uint32_t)cf;
    rec->qual_start = rec->seq_start;           // no qualities
    *seq_len = len;
}

// CasavaFiltered (predicates.py:125-139) on a name: name.partition(" ")[2][1:4] == ":Y:"
CG_HD bool fq_casava_filtered(const uint8_t *h, int hl)
{
    int sp = 0;
    while (sp < hl && h[sp] != ' ') ++sp;
    return sp + 4 < hl && h[sp + 2] == ':' && h[sp + 3] == 'Y' && h[sp + 4] == ':';
}

struct FqVerdict {
    int start, stop;         // what is written: read[start:stop] (relative to the record's sequence after -u)
    int k0, k1;              // the part the action leaves untouched ("remainder")
    int mask;                // one bit per failed filter (see below)
    int last_adapter;        // adapter of the most recent match, -1 = none
    int poly_a_removed;      // bases PolyATrimmer removed (0 without --poly-a): its trimmed_bases key
    bool matched;
    bool bad_quality;        // --max-ee met a quality character outside [33, 126]
};

// What is left of a read (modifiers.py:858 then adapters.py:453-454, 486-487 per round; AdapterCutter's action;
// PolyATrimmer, Shortener, NEndTrimmer after the adapters) and which filters it fails, one bit per filter in the
// order cli.py:700-830 + 870-910 appends them:
//   bit 0 TooShort, 1 TooLong (predicates.py:29-53), 2 TooManyN (96-122), 3 TooManyExpectedErrors (56-71),
//   4 CasavaFiltered (125-139), 5 IsTrimmed (--discard-trimmed), 6 IsUntrimmed (--discard-untrimmed),
//   7 TooHighAverageErrorRate (74-95; it comes after bit 3 in the chain, see fq_finish_core).
// ZeroCapper (modifiers.py:806-822) runs last, after NEndTrimmer: the quality filters see the capped characters.
// Every predicate is evaluated (a pair filter may need the verdict of a filter that the mate passes).
// `matches`: the times * slots records of THIS read (or nullptr); (qs, qe): its quality-trimmed interval.
CG_HD FqVerdict fq_evaluate_core(const uint8_t *buf, const CgFastqRecord &rec, int n, const cg_match_rec *matches,
                                 int times, int slots, bool has_qtrim, int qs, int qe, const CgFastqFilter &f,
                                 const double *phred)
{
    FqVerdict v;
    v.bad_quality = false;
    v.poly_a_removed = 0;
    int start = 0, stop = n;
    if (has_qtrim) { start = qs; stop = qe; }
    bool matched = false;
    int last_adapter = -1;                 // info.matches[-1].adapter: where a demultiplexer sends the read
    if (matches) {
        for (int t = 0; t < times; ++t)
            for (int s = 0; s < slots; ++s) {
                const cg_match_rec m = matches[t * slots + s];
                if (m.adapter < 0) continue;
                matched = true;
                last_adapter = m.adapter;
                // read[:rstart] / read[rstop:] with Python's slice clamping: an index match on a read that is
                // shorter than the matched key reports rstop > len or rstart < 0 (adapters.py:1342-1365)
                const int cur = stop - start;
                if ((m.info >> 8) & 1)                             // RemoveAfterMatch
                    stop = start + (m.rstart >= 0 ? (m.rstart < cur ? m.rstart : cur)
                                                  : (cur + m.rstart > 0 ? cur + m.rstart : 0));
                else                                               // RemoveBeforeMatch
                    start = start + (m.rstop < cur ? m.rstop : cur);
            }
    }
    const uint8_t *sq0 = buf + rec.seq_start;
    // AdapterCutter's action (modifiers.py:236-249): what is written instead of the trimmed read.  [k0, k1) is
    // the part that stays as it is ("remainder"), [start, stop) from here on the part that is output; all
    // relative to the read the cutter saw (after -u and quality trimming), whose interval is [b0, b1).
    const int b0 = has_qtrim ? qs : 0, b1 = has_qtrim ? qe : n;
    int k0 = start, k1 = stop;
    if (f.action != CG_FQ_ACTION_TRIM) {
        if (!matched) { start = b0; stop = b1; k0 = b0; k1 = b1; }
        else if (f.action == CG_FQ_ACTION_RETAIN || f.action == CG_FQ_ACTION_CROP) {
            // times == 1: slot 0 = the match (or the front match of a LinkedAdapter), slot 1 = a linked back match
            const cg_match_rec m0 = matches[0];
            cg_match_rec m1; m1.adapter = -1;
            if (slots > 1) m1 = matches[1];
            const int len = b1 - b0;
            int a, b;
            if (f.action == CG_FQ_ACTION_CROP) {                   // read[m.rstart:m.rstop] (modifiers.py:195-198)
                const cg_match_rec m = m0.adapter >= 0 ? m0 : m1;
                a = m.rstart; b = m.rstop;
            } else if (m0.adapter >= 0 && ((m0.info >> 8) & 1)) {  // RemoveAfterMatch: (0, rstop)  adapters.py:479-480
                a = 0; b = m0.rstop;
            } else {                                               // RemoveBeforeMatch (adapters.py:446-447) /
                a = m0.adapter >= 0 ? m0.rstart : 0;               // LinkedMatch (adapters.py:1145-1155)
                const int offset = m0.adapter >= 0 ? m0.rstop : 0;
                b = m1.adapter >= 0 ? m1.rstop + offset : len;
            }
            a = a < 0 ? 0 : (a > len ? len : a);                   // Python slice clamping
            b = b < 0 ? 0 : (b > len ? len : b);
            if (b < a) b = a;
            start = b0 + a; stop = b0 + b; k0 = start; k1 = stop;
        } else {                                                   // none / mask / lowercase: the whole read
            start = b0; stop = b1;
            if (f.action == CG_FQ_ACTION_NONE) { k0 = b0; k1 = b1; }
        }
    }
    // the character at position j as it will be written
    const int action = f.action;
    auto ch = [&](int j) -> uint8_t {
        const uint8_t c = sq0[j];
        if (action == CG_FQ_ACTION_MASK) return (j >= k0 && j < k1) ? c : (uint8_t)'N';
        if (action == CG_FQ_ACTION_LOWERCASE) {
            const bool alpha = (uint8_t)((c | 0x20) - 'a') < 26;
            return !alpha ? c : ((j >= k0 && j < k1) ? (uint8_t)(c & ~0x20) : (uint8_t)(c | 0x20));
        }
        return c;
    };
    if (f.poly_a) {                                    // PolyATrimmer (modifiers.py:861-879), qualtrim.pyx:120-169
        const int len = stop - start;
        int best_score = 0, score = 0, errors = 0;
        if (f.poly_a == 2) {                           // poly-T head of the second mate: read[index:]
            int best_index = 0;
            for (int i = 0; i < len; ++i) {
                if (ch(start + i) == 'T') score += 1; else { score -= 2; errors += 1; }
                if (score > best_score && errors * 5 <= i + 1) { best_score = score; best_index = i + 1; }
            }
            if (best_index < 3) best_index = 0;
            start += best_index;
            v.poly_a_removed = best_index;
        } else {                                       // poly-A tail: read[:index]
            int best_index = len;
            for (int i = len - 1; i >= 0; --i) {
                if (ch(start + i) == 'A') score += 1; else { score -= 2; errors += 1; }
                if (score > best_score && errors * 5 <= len - i) { best_score = score; best_index = i; }
            }
            if (best_index > len - 3) best_index = len;
            stop = start + best_index;
            v.poly_a_removed = len - best_index;
        }
    }
    if (f.shorten > 0) {                               // Shortener (modifiers.py:882-899): read[:length]
        if (stop - start > f.shorten - 1) stop = start + (f.shorten - 1);
    } else if (f.shorten < 0) {                        //                                   read[length:]
        if (stop - start > -f.shorten) start = stop + f.shorten;
    }
    if (f.trim_n) {                                    // NEndTrimmer (modifiers.py:902-918): upper-case N only
        int a = start, b = stop;
        while (a < stop && ch(a) == 'N') ++a;
        while (b > start && ch(b - 1) == 'N') --b;
        start = a; stop = b < a ? a : b;
    }
    const int left = stop - start;
    int mask = 0;
    if (f.minimum_length > 0 && left < f.minimum_length) mask |= 1;
    if (f.maximum_length >= 0 && left > f.maximum_length) mask |= 2;
    if (f.max_n >= 0.0) {
        int n_count = 0;
        for (int j = 0; j < left; ++j) n_count += (ch(start + j) | 0x20) == 'n';
        const bool too_many = f.max_n < 1.0 ? (left > 0 && (double)n_count / (double)left > f.max_n)
                                            : (double)n_count > f.max_n;
        if (too_many) mask |= 4;
    }
    if (f.max_ee >= 0.0 || f.max_aer > 0.0) {
        // expected_errors(qualities) with its default base 33, once for both filters
        const double ee = expected_errors_core(buf + rec.qual_start + start, left, 33, phred, f.zero_cap);
        if (ee < 0.0) v.bad_quality = true;
        else {
            if (f.max_ee >= 0.0 && ee > f.max_ee) mask |= 8;
            if (f.max_aer > 0.0 && left > 0 && ee / (double)left > f.max_aer) mask |= 128;
        }
    }
    if (f.discard_casava && fq_casava_filtered(buf + rec.hdr_start, rec.hdr_len)) mask |= 16;
    if (matched) mask |= 32; else mask |= 64;          // masked by the enabled filters in the finish step
    v.start = start; v.stop = stop; v.k0 = k0; v.k1 = k1; v.mask = mask; v.last_adapter = last_adapter;
    v.matched = matched;
    return v;
}

// The verdict on a read (pair == false) or a pair: the first enabled filter, in chain order, that fires (its bit
// number), or -1.  Chain order (cli.py:700-830): bits 0, 1, 2, 3, 7, 4, 5, 6.
// PairedEndFilter (steps.py:105-180): a filter given for one mate only tests that mate; otherwise mode 0 "any",
// 1 "both", 2 "first" (mode_untrimmed: cli.py:859-893 overrides the mode of --discard-untrimmed to "both" when only one
// mate has adapters).
CG_HD int fq_finish_core(int m1, int m2, bool pair, int enabled1, int enabled2, int mode, int mode_untrimmed)
{
    for (int i = 0; i < 8; ++i) {
        const int k = i < 4 ? i : (i == 4 ? 7 : i - 1);
        const int bit = 1 << k;
        const bool e1 = (enabled1 & bit) != 0, e2 = pair && (enabled2 & bit) != 0;
        if (!e1 && !e2) continue;
        const bool f1 = (m1 & bit) != 0, f2 = (m2 & bit) != 0;
        const int md = k == 6 ? mode_untrimmed : mode;
        bool hit;
        if (!e2) hit = f1;
        else if (!e1) hit = f2;
        else hit = md == 0 ? (f1 || f2) : md == 1 ? (f1 && f2) : f1;
        if (hit) return k;
    }
    return -1;
}

// PairedReverseComplementer's decision (modifiers.py:311-400) for one pair: the score of a pairing is the sum of the
// scores of every record with adapter >= 0 (all rounds, both parts of a linked match).  m11 / m22: cutter1 on r1 and
// cutter2 on r2 (per1 / per2 records each); m12 / m21: cutter1 on r2 and cutter2 on r1.  A missing cutter passes
// nullptr for its two arrays and scores 0.  The swapped pairing wins only if its score is strictly greater.
CG_HD long long fq_match_score(const cg_match_rec *m, int per)
{
    long long s = 0;
    if (m)
        for (int k = 0; k < per; ++k)
            if (m[k].adapter >= 0) s += m[k].score;
    return s;
}
CG_HD bool fq_pair_swap_core(const cg_match_rec *m11, const cg_match_rec *m22, const cg_match_rec *m12,
                             const cg_match_rec *m21, int per1, int per2)
{
    return fq_match_score(m12, per1) + fq_match_score(m21, per2) > fq_match_score(m11, per1) + fq_match_score(m22, per2);
}

// Do two headers (without '@' / '>') name the two mates of one pair?  The rule of dnaio's paired readers
// (doc/reference.rst:925-950): compare the IDs, each header up to its first space or tab; a final '1', '2' or '3' of the
// IDs is ignored, so "read1/1 some text" matches "read1/2 other text", but "my_read/1;1" does not match "my_read/2;1".
// This is the strict reading: the last character is dropped only when it is 1, 2 or 3 in BOTH IDs ("r1" and "r"
// differ).  No stored answer of the reference pins that case.
#define CG_FQ_ERR_PAIR 8      // interleaved input: the two records of a pair are not mates
CG_HD bool fq_mates_match(const uint8_t *h1, int len1, const uint8_t *h2, int len2)
{
    int i1 = 0, i2 = 0;
    while (i1 < len1 && h1[i1] != ' ' && h1[i1] != '\t') ++i1;
    while (i2 < len2 && h2[i2] != ' ' && h2[i2] != '\t') ++i2;
    if (i1 > 0 && i2 > 0 && (uint8_t)(h1[i1 - 1] - '1') < 3 && (uint8_t)(h2[i2 - 1] - '1') < 3) { --i1; --i2; }
    if (i1 != i2) return false;
    for (int j = 0; j < i1; ++j)
        if (h1[j] != h2[j]) return false;
    return true;
}

// Filter outputs (cg_fastq_collect_split): where a read or pair goes once fq_finish_core named the filter that fired
// (-1: none).  0 the main output, 1 --too-short-output, 2 --too-long-output, 3 --untrimmed-output, -1 dropped.  A
// filter with an output writes what it removes (SingleEndFilter / PairedEndFilter with a writer, steps.py:70-180),
// every other filter drops it.  redirect: CG_REDIRECT_* bits (1 too-short, 2 too-long, 4 untrimmed).
// fq_route_enabled: the enabled filters of a mate given to fq_finish_core -- an untrimmed output is the IsUntrimmed
// filter with a writer, so it switches that filter (bit 6) on.
CG_HD int fq_route_enabled(int enabled, int redirect) { return enabled | ((redirect & 4) ? 64 : 0); }
CG_HD int fq_route_core(int fired, int redirect)
{
    if (fired < 0) return 0;
    if (fired == 0 && (redirect & 1)) return 1;
    if (fired == 1 && (redirect & 2)) return 2;
    if (fired == 6 && (redirect & 4)) return 3;
    return -1;
}
