// cg_names_core.cuh -- the read-name modifiers of the FASTQ path (cg_fastq.cu: the name stage), host + device.
//
// The reference runs them last in its modifier chain (cli.py:937-991, modifiers_applying_to_both_ends_if_paired at
// cli.py:1136-1146): after the adapters, PolyATrimmer, Shortener and NEndTrimmer come
//   LengthTagModifier (--length-tag), one SuffixRemover per --strip-suffix, PrefixSuffixAdder (-x / -y), ZeroCapper
//   (qualities only) and, last, Renamer / PairedEndRenamer (--rename; modifiers.py:529-760).
// The name the chain starts from already carries the " rc" of --revcomp.  The stage evaluates a compiled program
// (CgNameProg) once per record in two steps: the "pre" name (tag, suffixes, prefix / suffix), then, with --rename, the
// template over that name.  Every function here walks the bytes of a name once with a sink, so that the same code
// counts the bytes (sizes, then a scan) and writes them.  tests/hostsim compiles this header for the host tests.
#pragma once
#include "cg_fastq_core.cuh"

// template tokens (tokenize_braces of the --rename template; -x / -y split at "{name}")
#define CG_NT_LITERAL 0
#define CG_NT_HEADER 1
#define CG_NT_ID 2
#define CG_NT_COMMENT 3
#define CG_NT_CUT_PREFIX 4
#define CG_NT_CUT_SUFFIX 5
#define CG_NT_ADAPTER_NAME 6      // also {name} of -x / -y
#define CG_NT_RC 7
#define CG_NT_MATCH_SEQUENCE 8
#define CG_NT_RN 9
#define CG_NT_KINDS 10

struct CgNameToken {          // 16 bytes
    int32_t kind;             // CG_NT_*
    int32_t mate;             // 0: the record's own value, 1: R1's ({r1.x}), 2: R2's ({r2.x})
    int32_t off, len;         // CG_NT_LITERAL: the text, blob bytes [off, off + len)
};

// The blob of a names handle: this header, then everything its offsets point at (offsets from the blob's start).
struct CgNameProg {
    int32_t tag_off, tag_len;           // --length-tag TAG; tag_len 0 = off
    int32_t n_strip, strip_off;         // --strip-suffix values: int32 (off, len)[n_strip], in the order given
    int32_t n_prefix, prefix_off;       // -x as CgNameToken[n_prefix] (LITERAL / ADAPTER_NAME)
    int32_t n_suffix, suffix_off;       // -y as CgNameToken[n_suffix]
    int32_t n_rename, rename_off;       // --rename as CgNameToken[n_rename]; n_rename < 0: no renamer
    int32_t n_names[2], names_off[2];   // per mate: int32 offsets[n_names + 1] (blob offsets) of the adapter names
    int32_t linked_off[2];              // per mate: uint8 linked[n_names] (the adapter is a part of a linked adapter)
    int32_t cut_last[2][2];             // per mate: the last -u value of the 5' end, of the 3' end (bases, >= 0)
    int32_t total;                      // blob bytes
};

// A run of name bytes; rc: the reverse complement of [p, p + len) (a part of a read that --revcomp turned around)
struct CgSpan {
    const uint8_t *p;
    int len;
    int rc;
};
CG_HD CgSpan cg_span(const uint8_t *p, int len) { CgSpan s; s.p = p; s.len = len; s.rc = 0; return s; }
CG_HD uint8_t cg_span_at(const CgSpan &s, int j) { return s.rc ? fq_complement(s.p[s.len - 1 - j]) : s.p[j]; }

// Python's str.split() whitespace on ASCII (dnaio decodes names as ASCII): \t \n \v \f \r, \x1c-\x1f and ' '
CG_HD bool cg_name_space(uint8_t c) { return (c >= 9 && c <= 13) || (c >= 0x1c && c <= 0x20); }
// \b of Python's re: a word character is [A-Za-z0-9_] on ASCII
CG_HD bool cg_name_word(uint8_t c)
{
    return (uint8_t)((c | 0x20) - 'a') < 26 || (uint8_t)(c - '0') < 10 || c == '_';
}

// Sinks: the count of the bytes, or the bytes themselves (one thread)
struct CgNameCount {
    long long n = 0;
    CG_HD void ch(uint8_t) { ++n; }
    CG_HD void span(const CgSpan &s) { n += s.len; }
};
struct CgNameWrite {
    uint8_t *p;
    long long n = 0;
    CG_HD void ch(uint8_t c) { p[n++] = c; }
    CG_HD void span(const CgSpan &s)
    {
        for (int j = 0; j < s.len; ++j) p[n++] = cg_span_at(s, j);
    }
};

// Python's seq[a:b] for a sequence of length len: (start, count)
CG_HD void cg_py_slice(int a, int b, int len, int *start, int *count)
{
    if (a < 0) { a += len; if (a < 0) a = 0; } else if (a > len) a = len;
    if (b < 0) { b += len; if (b < 0) b = 0; } else if (b > len) b = len;
    *start = a;
    *count = b > a ? b - a : 0;
}

// ---- step 1: the name LengthTagModifier, the SuffixRemovers and PrefixSuffixAdder leave ----
// The start name: the header, then " rc" when --revcomp turned the read and appends its suffix
struct CgNameStart {
    const uint8_t *h;
    int hl, n;                // n = hl or hl + 3
    CG_HD uint8_t at(int i) const { return i < hl ? h[i] : (uint8_t)(" rc"[i - hl]); }
};

// LengthTagModifier (modifiers.py:529-547): re.sub(r"\b" + TAG + r"[0-9]*\b", TAG + str(len)), TAG a literal.  Does
// TAG match at i?  Returns where the match ends, or -1.  The digit run is the longest one followed by a word boundary.
CG_HD int cg_tag_match(const CgNameStart &s, const uint8_t *tag, int tl, int i)
{
    if (i + tl > s.n) return -1;
    const bool before = i > 0 && cg_name_word(s.at(i - 1));
    if (before == cg_name_word(s.at(i))) return -1;
    for (int k = 0; k < tl; ++k)
        if (s.at(i + k) != tag[k]) return -1;
    int d = i + tl;
    while (d < s.n && (uint8_t)(s.at(d) - '0') < 10) ++d;
    for (int e = d; e >= i + tl; --e)
        if (cg_name_word(s.at(e - 1)) != (e < s.n && cg_name_word(s.at(e)))) return e;
    return -1;
}

// Every character of the tagged name in order: visit(position, character)
template <class Visit>
CG_HD void cg_tag_walk(const uint8_t *blob, const CgNameProg &pr, const CgNameStart &s, int written_len, Visit &visit)
{
    const uint8_t *tag = blob + pr.tag_off;
    uint8_t digits[12];
    int nd = 0;
    unsigned v = (unsigned)(written_len < 0 ? 0 : written_len);
    do { digits[nd++] = (uint8_t)('0' + v % 10u); v /= 10u; } while (v);
    int pos = 0;
    for (int i = 0; i < s.n;) {
        const int e = pr.tag_len > 0 ? cg_tag_match(s, tag, pr.tag_len, i) : -1;
        if (e < 0) { visit(pos++, s.at(i)); ++i; continue; }
        for (int k = 0; k < pr.tag_len; ++k) visit(pos++, tag[k]);
        for (int k = nd - 1; k >= 0; --k) visit(pos++, digits[k]);
        i = e;
    }
}

struct CgTagCount {
    int n = 0;
    CG_HD void operator()(int, uint8_t) { ++n; }
};
struct CgTagTail {             // do the characters [from, from + len) equal s?
    const uint8_t *s;
    int from, len;
    bool same = true;
    CG_HD void operator()(int pos, uint8_t c)
    {
        if (pos >= from && pos < from + len && c != s[pos - from]) same = false;
    }
};
template <class Sink>
struct CgTagEmit {             // the first `keep` characters to the sink
    Sink *out;
    int keep;
    CG_HD void operator()(int pos, uint8_t c) { if (pos < keep) out->ch(c); }
};

// -x / -y: the text with "{name}" replaced by the adapter name (PrefixSuffixAdder, modifiers.py:567-588)
template <class Sink>
CG_HD void cg_emit_affix(const uint8_t *blob, const CgNameToken *tok, int n_tok, const CgSpan &adapter, Sink &out)
{
    for (int t = 0; t < n_tok; ++t) {
        if (tok[t].kind == CG_NT_ADAPTER_NAME) out.span(adapter);
        else out.span(cg_span(blob + tok[t].off, tok[t].len));
    }
}

// The name after step 1 of one record: header (+ " rc"), written_len = the length of the sequence as written (what
// LengthTagModifier counts), adapter = the name of the adapter of the last match or "no_adapter"
template <class Sink>
CG_HD void cg_pre_name(const uint8_t *blob, const CgNameProg &pr, const uint8_t *h, int hl, bool rc_suffix,
                       int written_len, const CgSpan &adapter, Sink &out)
{
    CgNameStart s;
    s.h = h; s.hl = hl; s.n = hl + (rc_suffix ? 3 : 0);
    CgTagCount cnt;
    cg_tag_walk(blob, pr, s, written_len, cnt);
    int L = cnt.n;
    // SuffixRemover (modifiers.py:550-564): name[:-len(suffix)] if name.endswith(suffix); an empty suffix empties the
    // name (name[:-0] is name[:0])
    const int32_t *strips = (const int32_t *)(blob + pr.strip_off);
    for (int k = 0; k < pr.n_strip; ++k) {
        const int sl = strips[2 * k + 1];
        if (sl == 0) { L = 0; continue; }
        if (sl > L) continue;
        CgTagTail tail;
        tail.s = blob + strips[2 * k]; tail.from = L - sl; tail.len = sl;
        cg_tag_walk(blob, pr, s, written_len, tail);
        if (tail.same) L -= sl;
    }
    cg_emit_affix(blob, (const CgNameToken *)(blob + pr.prefix_off), pr.n_prefix, adapter, out);
    CgTagEmit<Sink> emit;
    emit.out = &out; emit.keep = L;
    cg_tag_walk(blob, pr, s, written_len, emit);
    cg_emit_affix(blob, (const CgNameToken *)(blob + pr.suffix_off), pr.n_suffix, adapter, out);
}

// ---- step 2: Renamer / PairedEndRenamer (modifiers.py:595-760) ----
// What a template can name about one record
struct CgNameVars {
    CgSpan header;              // the name after step 1
    CgSpan cut_prefix, cut_suffix;
    CgSpan adapter;             // adapter of the last match, or "no_adapter"
    CgSpan ms_front, ms_back;   // match_sequence: ms_front, or for a linked match ms_front + "," + ms_back
    int ms_linked;
    int is_rc;
};

// Renamer.parse_name: name.split(maxsplit=1); with fewer than two fields the id is the whole name, the comment ""
CG_HD void cg_name_split(const CgSpan &h, CgSpan *id, CgSpan *comment)
{
    int i = 0;
    while (i < h.len && cg_name_space(h.p[i])) ++i;
    const int a = i;
    while (i < h.len && !cg_name_space(h.p[i])) ++i;
    const int b = i;
    while (i < h.len && cg_name_space(h.p[i])) ++i;
    if (b == a || i == h.len) { *id = h; *comment = cg_span(h.p, 0); return; }
    *id = cg_span(h.p + a, b - a);
    *comment = cg_span(h.p + i, h.len - i);
}

// The template for a record: self = the record's own variables, r[0] / r[1] those of R1 / R2 (pairs), rn = 1 / 2
template <class Sink>
CG_HD void cg_rename(const uint8_t *blob, const CgNameProg &pr, const CgNameVars &self, const CgNameVars *r, int rn,
                     Sink &out)
{
    const CgNameToken *tok = (const CgNameToken *)(blob + pr.rename_off);
    for (int t = 0; t < pr.n_rename; ++t) {
        const CgNameVars &v = tok[t].mate == 0 ? self : r[tok[t].mate - 1];
        CgSpan id, comment;
        switch (tok[t].kind) {
        case CG_NT_LITERAL: out.span(cg_span(blob + tok[t].off, tok[t].len)); break;
        case CG_NT_HEADER: out.span(v.header); break;
        case CG_NT_ID: cg_name_split(v.header, &id, &comment); out.span(id); break;
        case CG_NT_COMMENT: cg_name_split(v.header, &id, &comment); out.span(comment); break;
        case CG_NT_CUT_PREFIX: out.span(v.cut_prefix); break;
        case CG_NT_CUT_SUFFIX: out.span(v.cut_suffix); break;
        case CG_NT_ADAPTER_NAME: out.span(v.adapter); break;
        case CG_NT_RC: if (v.is_rc) { out.ch('r'); out.ch('c'); } break;
        case CG_NT_MATCH_SEQUENCE:
            out.span(v.ms_front);
            if (v.ms_linked) { out.ch(','); out.span(v.ms_back); }
            break;
        case CG_NT_RN: out.ch((uint8_t)('0' + rn)); break;
        default: break;
        }
    }
}

// The adapter name of a mate's adapter a (-1 = no match): "no_adapter" without a match (modifiers.py:584, 671)
CG_HD CgSpan cg_adapter_name(const uint8_t *blob, const CgNameProg &pr, int mate, int a)
{
    const int32_t *off = (const int32_t *)(blob + pr.names_off[mate]);
    if (a < 0 || a >= pr.n_names[mate]) return cg_span((const uint8_t *)"no_adapter", 10);
    return cg_span(blob + off[a], off[a + 1] - off[a]);
}

// UnconditionalCutter's cut_prefix / cut_suffix (modifiers.py:80-95) of a read as it came, `full` bases at `read`
// (reverse-complemented in place when rc): the bases the LAST cutter of each end removed.  -u values of one end add up
// (cut_front / cut_back); last_front / last_back are the last values; the 5' cutters come first, as in fq_record_core.
CG_HD void cg_cut_spans(const uint8_t *read, int full, bool rc, int cut_front, int cut_back, int last_front,
                        int last_back, CgSpan *prefix, CgSpan *suffix)
{
    auto part = [&](int a, int b) {
        CgSpan s;
        s.len = b > a ? b - a : 0;
        s.rc = rc ? 1 : 0;
        s.p = rc ? read + (full - b) : read + a;
        if (s.len == 0) { s.p = read; s.rc = 0; }
        return s;
    };
    const int cf = cut_front < full ? cut_front : full;
    const int a = cut_front - last_front < full ? cut_front - last_front : full;
    *prefix = part(last_front > 0 ? a : cf, cf);
    const int left = full - cf;
    const int bb = cut_back < left ? cut_back : left;
    const int rest = cut_back - last_back < left ? cut_back - last_back : left;
    *suffix = part(full - bb, last_back > 0 ? full - rest : full - bb);
}

// The last match of a read (info.matches[-1]): its adapter and match_sequence() -- sequence[rstart:rstop] of the
// sequence its round searched (SingleMatch, adapters.py:419-420), for a linked match front + "," + back
// (adapters.py:1173-1178).  seq = the record's sequence; [ws, we) the part the first round searched.
CG_HD void cg_last_match(const uint8_t *blob, const CgNameProg &pr, int mate, const uint8_t *seq, int ws, int we,
                         const cg_match_rec *mr, int times, int slots, CgNameVars *v)
{
    v->adapter = cg_adapter_name(blob, pr, mate, -1);
    v->ms_front = v->ms_back = cg_span(seq, 0);
    v->ms_linked = 0;
    if (!mr) return;
    const uint8_t *linked = blob + pr.linked_off[mate];
    for (int t = 0; t < times; ++t) {
        bool hit = false;
        CgSpan part[2] = {cg_span(seq, 0), cg_span(seq, 0)};
        int last = -1, last_slot = 0;
        for (int k = 0; k < slots; ++k) {
            const cg_match_rec h = mr[t * slots + k];
            if (h.adapter < 0) continue;
            hit = true;
            const int cur = we - ws;
            int s, c;
            cg_py_slice(h.rstart, h.rstop, cur, &s, &c);
            if (k < 2) part[k] = cg_span(seq + ws + s, c);
            last = h.adapter; last_slot = k;
            if (h.info & 256) { cg_py_slice(0, h.rstart, cur, &s, &c); we = ws + c; }
            else { cg_py_slice(h.rstop, cur, cur, &s, &c); ws += s; }
        }
        if (!hit) break;
        v->adapter = cg_adapter_name(blob, pr, mate, last);
        v->ms_linked = last < pr.n_names[mate] && linked[last] != 0;
        if (v->ms_linked) { v->ms_front = part[0]; v->ms_back = part[1]; }
        else { v->ms_front = last_slot < 2 ? part[last_slot] : cg_span(seq, 0); v->ms_back = cg_span(seq, 0); }
    }
}

#if !defined(__CUDACC_RTC__)
#include <string.h>

#include <string>
#include <vector>

// ---- the blob of a names handle, built on the host (cg_names_create / cg_names_set_mate; the host tests) ----
struct CgNameSpec {
    struct Token {
        int kind, mate;
        std::string text;
    };
    std::string tag;
    std::vector<std::string> strips;
    std::vector<Token> prefix, suffix, rename;
    bool has_rename = false, paired = false;
    std::string names[2];                               // per mate: the adapter names back to back ...
    std::vector<int32_t> name_off[2] = {{0}, {0}};      // ... where each starts (n + 1 values)
    std::vector<uint8_t> linked[2];
    int32_t cut_last[2][2] = {{0, 0}, {0, 0}};
};

// -x / -y: the text split at every "{name}" (str.replace, left to right)
inline std::vector<CgNameSpec::Token> cg_names_affix(const char *text)
{
    std::vector<CgNameSpec::Token> t;
    const std::string x = text ? text : "";
    size_t at = 0;
    for (size_t k; (k = x.find("{name}", at)) != std::string::npos; at = k + 6) {
        if (k > at) t.push_back({CG_NT_LITERAL, 0, x.substr(at, k - at)});
        t.push_back({CG_NT_ADAPTER_NAME, 0, std::string()});
    }
    if (at < x.size()) t.push_back({CG_NT_LITERAL, 0, x.substr(at)});
    return t;
}

inline std::vector<uint8_t> cg_names_blob(const CgNameSpec &sp)
{
    std::vector<uint8_t> b(sizeof(CgNameProg), 0);
    auto align4 = [&]() { while (b.size() % 4) b.push_back(0); };
    auto put = [&](const void *p, size_t n) {
        const size_t at = b.size();
        if (n) b.insert(b.end(), (const uint8_t *)p, (const uint8_t *)p + n);
        return (int32_t)at;
    };
    CgNameProg pr;
    memset(&pr, 0, sizeof pr);
    pr.tag_off = put(sp.tag.data(), sp.tag.size());
    pr.tag_len = (int32_t)sp.tag.size();
    std::vector<int32_t> strips;
    for (const std::string &x : sp.strips) {
        strips.push_back(put(x.data(), x.size()));
        strips.push_back((int32_t)x.size());
    }
    auto tokens = [&](const std::vector<CgNameSpec::Token> &t, int32_t *off) {
        std::vector<CgNameToken> v(t.size());
        for (size_t i = 0; i < t.size(); ++i) {
            v[i].kind = t[i].kind;
            v[i].mate = t[i].mate;
            v[i].len = (int32_t)t[i].text.size();
            v[i].off = put(t[i].text.data(), t[i].text.size());
        }
        align4();
        *off = put(v.data(), v.size() * sizeof(CgNameToken));
        return (int32_t)v.size();
    };
    pr.n_prefix = tokens(sp.prefix, &pr.prefix_off);
    pr.n_suffix = tokens(sp.suffix, &pr.suffix_off);
    pr.n_rename = tokens(sp.rename, &pr.rename_off);
    if (!sp.has_rename) pr.n_rename = -1;
    pr.n_strip = (int32_t)sp.strips.size();
    align4();
    pr.strip_off = put(strips.data(), strips.size() * sizeof(int32_t));
    for (int m = 0; m < 2; ++m) {
        const int32_t text = put(sp.names[m].data(), sp.names[m].size());
        std::vector<int32_t> off(sp.name_off[m]);
        for (int32_t &o : off) o += text;
        align4();
        pr.names_off[m] = put(off.data(), off.size() * sizeof(int32_t));
        pr.n_names[m] = (int32_t)off.size() - 1;
        pr.linked_off[m] = put(sp.linked[m].data(), sp.linked[m].size());
        pr.cut_last[m][0] = sp.cut_last[m][0];
        pr.cut_last[m][1] = sp.cut_last[m][1];
    }
    align4();
    pr.total = (int32_t)b.size();
    memcpy(b.data(), &pr, sizeof pr);
    return b;
}
#endif
