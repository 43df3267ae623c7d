// tests/hostsim/hostsim_names.cpp -- TEST-ONLY host build of the read-name modifiers of the FASTQ path
// (cutadapt_b200/csrc/cg_names_core.cuh: the two steps of the name stage, the -u parts and the last match), linked into
// libhostsim.so so that tests/test_names_host.py can check them against the known answers and tests/names_oracle.py
// without a GPU.  Nothing in cutadapt_b200/ loads this library; it is not a fallback.
#include <string.h>

#include "../../cutadapt_b200/csrc/cg_names_core.cuh"

static int64_t hs_copy(const std::string &s, uint8_t *out, int64_t cap)
{
    if ((int64_t)s.size() <= cap) memcpy(out, s.data(), s.size());
    return (int64_t)s.size();
}

// step 1 of one name: tag (NULL = off), strip suffixes, -x / -y; the adapter name of the last match (or "no_adapter")
extern "C" int64_t hs_names_pre(const char *tag, const char *const *strips, int n_strips, const char *prefix,
                                const char *suffix, const uint8_t *hdr, int hl, int rc_suffix, int written,
                                const char *adapter, uint8_t *out, int64_t cap)
{
    CgNameSpec sp;
    if (tag) sp.tag = tag;
    for (int k = 0; k < n_strips; ++k) sp.strips.emplace_back(strips[k]);
    sp.prefix = cg_names_affix(prefix);
    sp.suffix = cg_names_affix(suffix);
    const std::vector<uint8_t> blob = cg_names_blob(sp);
    const CgNameProg &pr = *(const CgNameProg *)blob.data();
    CgNameCount c;
    const CgSpan a = cg_span((const uint8_t *)adapter, (int)strlen(adapter));
    cg_pre_name(blob.data(), pr, hdr, hl, rc_suffix != 0, written, a, c);
    std::string s((size_t)c.n, '\0');
    CgNameWrite w;
    w.p = (uint8_t *)&s[0];
    cg_pre_name(blob.data(), pr, hdr, hl, rc_suffix != 0, written, a, w);
    return hs_copy(s, out, cap);
}

// step 2: the template (kinds / mates / literal texts) over three sets of variables (the record's own, R1's, R2's):
// per set the strings header, cut_prefix, cut_suffix, adapter_name, match front, match back and the flags
// (linked match, is_rc)
extern "C" int64_t hs_names_rename(const int32_t *kinds, const int32_t *mates, const char *const *texts, int n_tokens,
                                   const char *const *vars, const int32_t *flags, int rn, uint8_t *out, int64_t cap)
{
    CgNameSpec sp;
    sp.has_rename = true;
    for (int t = 0; t < n_tokens; ++t) sp.rename.push_back({kinds[t], mates[t], kinds[t] == CG_NT_LITERAL ? texts[t] : ""});
    const std::vector<uint8_t> blob = cg_names_blob(sp);
    const CgNameProg &pr = *(const CgNameProg *)blob.data();
    CgNameVars v[3];
    for (int k = 0; k < 3; ++k) {
        auto span = [&](int i) { return cg_span((const uint8_t *)vars[6 * k + i], (int)strlen(vars[6 * k + i])); };
        v[k].header = span(0); v[k].cut_prefix = span(1); v[k].cut_suffix = span(2); v[k].adapter = span(3);
        v[k].ms_front = span(4); v[k].ms_back = span(5);
        v[k].ms_linked = flags[2 * k]; v[k].is_rc = flags[2 * k + 1];
    }
    CgNameCount c;
    cg_rename(blob.data(), pr, v[0], v + 1, rn, c);
    std::string s((size_t)c.n, '\0');
    CgNameWrite w;
    w.p = (uint8_t *)&s[0];
    cg_rename(blob.data(), pr, v[0], v + 1, rn, w);
    return hs_copy(s, out, cap);
}

// the -u parts of a read as it came (rc: reverse-complemented in place): out receives cut_prefix then cut_suffix,
// lens their lengths
extern "C" void hs_names_cut(const uint8_t *read, int full, int rc, int cut_front, int cut_back, int last_front,
                             int last_back, uint8_t *out, int32_t *lens)
{
    CgSpan a, b;
    cg_cut_spans(read, full, rc != 0, cut_front, cut_back, last_front, last_back, &a, &b);
    CgNameWrite w;
    w.p = out;
    w.span(a);
    w.span(b);
    lens[0] = a.len;
    lens[1] = b.len;
}

// Renamer.parse_name: (id start, id length, comment start, comment length)
extern "C" void hs_names_split(const uint8_t *h, int hl, int32_t *out4)
{
    CgSpan id, comment;
    cg_name_split(cg_span(h, hl), &id, &comment);
    out4[0] = (int32_t)(id.p - h); out4[1] = id.len;
    out4[2] = (int32_t)(comment.p - h); out4[3] = comment.len;
}
