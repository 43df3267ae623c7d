// tests/hostsim/hostsim.cpp -- TEST-ONLY host build of the per-read device functions.
//
// Compiles cutadapt_b200/csrc/cg_core.cuh (the exact code the CUDA kernels run, one lane per
// read) with g++ so that the selection logic, the packed-cell DP and the adapter composition
// can be fuzzed against the oracle on a box without a GPU.  Nothing in cutadapt_b200/ loads
// this library; it is not a fallback.
#include <string.h>

#include <string>
#include <vector>

#include "../../cutadapt_b200/csrc/cg_core.cuh"
#include "../../cutadapt_b200/csrc/cg_fastq_core.cuh"
#include "../../cutadapt_b200/csrc/cg_setbuild.h"
#include "../../cutadapt_b200/csrc/cg_jit.h"

static thread_local std::string g_err;

extern "C" const char *hs_last_error(void) { return g_err.c_str(); }

extern "C" int hs_process_batch_indexed(const cg_adapter_desc *adapters, int n_adapters,
                                        const cg_group_desc *groups, int n_groups,
                                        const cg_index_desc *indexes, int n_indexes, const uint8_t *seq,
                                        const uint8_t *qual, const int64_t *offsets, int64_t n_reads,
                                        const cg_params *params, cg_match *matches, int32_t *qtrim,
                                        int force_wide)
{
    CgBuiltSet set;
    int rc = cg_build_set(adapters, n_adapters, groups, n_groups, set, g_err, indexes, n_indexes);
    if (rc != CG_OK) return rc;
    if (force_wide & 4) {   // query only: bit 0 two-phase program available, 1 windowed, 2 exact shortcut, 3 myers
        const CgSetHeader *h = (const CgSetHeader *)set.blob.data();
        return (set.simple_ok ? 1 : 0) | (h->windowed ? 2 : 0) | (h->exact_ok ? 4 : 0) | (h->myers ? 8 : 0) |
               (h->plane_count > 0 ? 16 : 0) | ((h->plane_flags & 1) ? 32 : 0) | ((h->plane_flags & 2) ? 64 : 0);
    }
    if (force_wide & 1) {
        CgSetHeader *h = (CgSetHeader *)set.blob.data();
        CgAdapter *ad = (CgAdapter *)(set.blob.data() + h->adapters_off);
        for (int a = 0; a < n_adapters; ++a) ad[a].cell_mode = CG_CELL_WIDE;
    }
    uint8_t enc[768];
    cg_build_enc_tables(enc);
    // flags and packed base/cutoff as pre_trim_core expects them (cg_api.cu: launch_trim_single)
    const int tflags = (params->quality_trim ? 1 : 0) | (params->nextseq_trim ? 2 : 0);
    const int tbase = (params->quality_base & 255) | (int)((unsigned)params->nextseq_cutoff << 8);
    if (force_wide & 128) {
        // the multi-pass schedule of cg_api.cu (launch_trim): per-component passes + select_best
        CgMultiPlan plan;
        rc = cg_plan_passes(adapters, n_adapters, groups, n_groups, indexes, n_indexes, plan, g_err);
        if (rc != CG_OK) return rc;
        if (plan.passes.empty() || params->times > 1) return 100;     // schedule not applicable
        const CgSetHeader *H = (const CgSetHeader *)set.blob.data();
        CgSelectTables T;
        cg_fill_select_tables((const CgGroup *)(set.blob.data() + H->groups_off), n_groups, set.slots, plan.passes, T);
        const int np = (int)plan.passes.size();
        std::vector<SetView> views(np);
        int max_m = 0;
        for (int pi = 0; pi < np; ++pi) {
            CgBuiltSet &b = plan.passes[pi].set;
            views[pi] = make_set_view(b.blob.data(), b.masks64.data(), enc, b.index_blob.empty() ? nullptr : b.index_blob.data());
            if (b.max_m > max_m) max_m = b.max_m;
        }
        std::vector<uint32_t> colp((size_t)max_m + 2);
        std::vector<int> colw(3 * ((size_t)max_m + 2));
        PackedCol pc; pc.base = colp.data(); pc.stride = 1;
        WideCol wc; wc.base = colw.data(); wc.stride = 1;
        std::vector<uint8_t> padded((size_t)offsets[n_reads] + 64, 0);
        if (offsets[n_reads]) memcpy(padded.data() + 32, seq, (size_t)offsets[n_reads]);
        const uint8_t *pseq = padded.data() + 32;
        if (tflags && !qual) { g_err = "no qualities"; return CG_ENOQUAL; }
        std::vector<cg_match_rec> recs(np);
        for (int64_t r = 0; r < n_reads; ++r) {
            const int n = (int)(offsets[r + 1] - offsets[r]);
            const uint8_t *sq = pseq + offsets[r];
            for (int i = 0; i < n; ++i) if (sq[i] & 0x80) { g_err = "non-ASCII"; return CG_ENONASCII; }
            int bs = 0, be = n;
            if (tflags)
                pre_trim_core(sq, qual + offsets[r], n, tflags, params->cutoff_front, params->cutoff_back, tbase, &bs, &be);
            if (qtrim) { qtrim[2 * r] = bs; qtrim[2 * r + 1] = be; }
            for (int pi = 0; pi < np; ++pi) {
                const CgPassPlan &P = plan.passes[pi];
                int vs = bs, ve = be;
                if (P.role == 1) linked_view(recs[P.front_pass], vs, ve);
                const SetView &V = views[pi];
                if (V.h->simple_ok && V.ad[0].m <= 64)
                    process_read_planned(V, sq + vs, nullptr, ve - vs, 0, 0, 0, 33, &recs[pi], nullptr);
                else {
                    const int32_t view[2] = {vs, ve};
                    process_read<true>(V, sq, nullptr, n, 0, 0, 0, 33, 1, pc, wc, &recs[pi], nullptr, view);
                }
            }
            cg_match_rec b0, b1;
            select_best(T, plan.pass_map.data(), [&](int pass) { return recs[pass]; }, b0, b1);
            cg_match_rec *dst = (cg_match_rec *)(matches + (size_t)r * set.slots);
            dst[0] = b0;
            if (set.slots > 1) dst[1] = b1;
        }
        return CG_OK;
    }
    SetView S = make_set_view(set.blob.data(), set.masks64.data(), enc,
                              set.index_blob.empty() ? nullptr : set.index_blob.data());
    std::vector<uint32_t> colp((size_t)set.max_m + 2);
    std::vector<int> colw(3 * ((size_t)set.max_m + 2));
    PackedCol pc; pc.base = colp.data(); pc.stride = 1;
    WideCol wc; wc.base = colw.data(); wc.stride = 1;
    // word-granular character loads may touch up to 7 bytes before/after a read: work on a padded copy
    // (the bit-plane scan reads up to 32 * 8 + 3 bytes in front of a read's end; fill with non-letters)
    std::vector<uint8_t> padded((size_t)offsets[n_reads] + 640, 0x7f);
    if (offsets[n_reads]) memcpy(padded.data() + 320, seq, (size_t)offsets[n_reads]);
    seq = padded.data() + 320;
    const int times = params->times < 1 ? 1 : params->times;
    if (tflags && !qual) { g_err = "no qualities"; return CG_ENOQUAL; }
    for (int64_t r = 0; r < n_reads; ++r) {
        const int n = (int)(offsets[r + 1] - offsets[r]);
        const uint8_t *s = seq + offsets[r];
        for (int i = 0; i < n; ++i) if (s[i] & 0x80) { g_err = "non-ASCII"; return CG_ENONASCII; }
        if ((force_wide & 256) && S.h->simple_ok && times == 1 && S.ad[0].m <= 64)
            process_read_planes(S, s, qual ? qual + offsets[r] : nullptr, n, tflags,
                                params->cutoff_front, params->cutoff_back, tbase,
                                (cg_match_rec *)(matches + (size_t)r * set.slots), qtrim ? qtrim + 2 * r : nullptr);
        else if ((force_wide & 64) && S.h->simple_ok && times == 1 && S.ad[0].m <= 64)
            process_read_planned(S, s, qual ? qual + offsets[r] : nullptr, n, tflags,
                                 params->cutoff_front, params->cutoff_back, tbase,
                                 (cg_match_rec *)(matches + (size_t)r * set.slots), qtrim ? qtrim + 2 * r : nullptr);
        else if ((force_wide & 2) && S.h->simple_ok && times == 1)
            process_read_simple(S, s, qual ? qual + offsets[r] : nullptr, n, tflags,
                                params->cutoff_front, params->cutoff_back, tbase, pc,
                                (cg_match_rec *)(matches + (size_t)r * set.slots), qtrim ? qtrim + 2 * r : nullptr,
                                (force_wide & 32) ? 3 : ((force_wide & 16) ? 2 : ((force_wide & 8) ? 1 : 0)));
        else
        process_read<true>(S, s, qual ? qual + offsets[r] : nullptr, n, tflags,
                           params->cutoff_front, params->cutoff_back, tbase, times, pc,
                           wc, (cg_match_rec *)(matches + (size_t)r * times * set.slots),
                           qtrim ? qtrim + 2 * r : nullptr);
    }
    return CG_OK;
}

// class of every read in the bit-plane first stage (0 none, 1 exact, 2 exact path after a re-scan, 3 exact path
// from the planes' hits, 4 exact overlap at the end, 5 like 3 without an end window; -1: no plane program)
extern "C" int hs_plane_classify(const cg_adapter_desc *adapters, int n_adapters, const cg_group_desc *groups, int n_groups,
                                 const uint8_t *seq, const int64_t *offsets, int64_t n_reads, int32_t *cls)
{
    CgBuiltSet set;
    int rc = cg_build_set(adapters, n_adapters, groups, n_groups, set, g_err, nullptr, 0);
    if (rc != CG_OK) return rc;
    uint8_t enc[768];
    cg_build_enc_tables(enc);
    SetView S = make_set_view(set.blob.data(), set.masks64.data(), enc, nullptr);
    std::vector<uint8_t> padded((size_t)offsets[n_reads] + 640, 0x7f);
    if (offsets[n_reads]) memcpy(padded.data() + 320, seq, (size_t)offsets[n_reads]);
    seq = padded.data() + 320;
    for (int64_t r = 0; r < n_reads; ++r) {
        const int n = (int)(offsets[r + 1] - offsets[r]);
        cls[r] = -1;
        if (S.h->plane_count <= 0 || n < 1 || n > 256) continue;
        const CgAdapter &A = S.ad[0];
        const uint8_t *ref = S.pool + A.ref_off;
        const PlaneOut po = n <= 160
            ? plane_scan_core<5, RuntimePlaneProg>(plane_program(S), S.h->plane_count, S.h->plane_flags, A.m, ref, seq + offsets[r + 1], n, A.pf_count == 0)
            : plane_scan_core<8, RuntimePlaneProg>(plane_program(S), S.h->plane_count, S.h->plane_flags, A.m, ref, seq + offsets[r + 1], n, A.pf_count == 0);
        cls[r] = po.cls == CG_PLANE_OVERLAP ? 4 : ((po.cls == CG_PLANE_SLOW && window_is_plain(seq + offsets[r], n)) ? (po.no_end ? 5 : 3) : po.cls);
    }
    return CG_OK;
}

// The run-time specialisation of the first stage (cg_jit.cpp): generate the translation unit for this adapter set
// and compile it with NVRTC for sm_90a (no device needed).  Returns the cubin size, 0 if the set has no plane
// program, -1 if the compilation failed (log says why), -2 if libnvrtc is not there.
extern "C" long hs_jit_compile(const cg_adapter_desc *adapters, int n_adapters, const cg_group_desc *groups, int n_groups,
                               int plane_words, int has_qual, char *src, long src_cap, char *log, long log_cap)
{
    CgBuiltSet set;
    int rc = cg_build_set(adapters, n_adapters, groups, n_groups, set, g_err, nullptr, 0);
    if (rc != CG_OK) return rc;
    const std::string text = cg_jit_pscan_source(set, plane_words, has_qual != 0);
    if (src && src_cap > 0) { strncpy(src, text.c_str(), (size_t)src_cap - 1); src[src_cap - 1] = 0; }
    if (text.empty()) return 0;
    std::string l;
    const long n = cg_jit_compile_only(set, plane_words, has_qual != 0, l);
    if (log && log_cap > 0) { strncpy(log, l.c_str(), (size_t)log_cap - 1); log[log_cap - 1] = 0; }
    if (n < 0 && l.find("libnvrtc") != std::string::npos) return -2;
    return n;
}

// The statistics vector of a batch (stats_read_core, the function cg_stats_kernel runs per read), on the host.
extern "C" int hs_statistics(const uint8_t *seq, const int64_t *offsets, int64_t n_reads, const cg_match *matches,
                             const int32_t *qtrim, int times, int slots, int n_adapters, int max_len, int kmax,
                             int64_t *stats)
{
    StatsScalars sc; sc.bp = sc.with_adapters = sc.qtrim_bp = sc.adapter_bp = 0;
    int64_t *hist = stats + CG_STATS_SCALARS;
    for (int64_t r = 0; r < n_reads; ++r) {
        const int len = (int)(offsets[r + 1] - offsets[r]);
        stats_read_core(seq ? seq + offsets[r] : nullptr, len, qtrim != nullptr, qtrim ? qtrim[2 * r] : 0,
                        qtrim ? qtrim[2 * r + 1] : len, (const cg_match_rec *)matches + (size_t)r * times * slots, times,
                        slots, n_adapters, max_len, kmax, sc, [&](long long idx, unsigned int v) { hist[idx] += v; });
    }
    stats[0] += n_reads; stats[1] += (int64_t)sc.bp; stats[2] += (int64_t)sc.with_adapters;
    stats[3] += (int64_t)sc.qtrim_bp; stats[4] += (int64_t)sc.adapter_bp;
    return 0;
}

// The DP matrices of one read (locate_core with its debug outputs: what cg_locate_debug_kernel runs), on the host.
extern "C" int hs_locate_debug(const cg_adapter_desc *adapter, const uint8_t *query, int n, int32_t *cost, int32_t *score,
                               int32_t *result8)
{
    cg_adapter_desc d = *adapter;
    d.n_kmer_entries = 0; d.kmer_entries = nullptr; d.kmer_masks = nullptr; d.reverse_read = 0;
    cg_group_desc g;
    memset(&g, 0, sizeof g);
    g.type = CG_GROUP_SINGLE; g.a0 = 0; g.a1 = -1;
    CgBuiltSet set;
    int rc = cg_build_set(&d, 1, &g, 1, set, g_err);
    if (rc != CG_OK) return rc;
    uint8_t enc[768];
    cg_build_enc_tables(enc);
    SetView S = make_set_view(set.blob.data(), set.masks64.data(), enc, nullptr);
    const CgAdapter &A = S.ad[0];
    const int m = A.m;
    for (size_t i = 0; i < (size_t)(m + 1) * (n + 1); ++i) cost[i] = score[i] = CG_DEBUG_NONE;
    std::vector<int> colw(3 * ((size_t)m + 2));
    WideCol wc; wc.base = colw.data(); wc.stride = 1;
    ReadView rv; rv.p = query; rv.n = n; rv.rev = 0;
    int o[6] = {0, 0, 0, 0, 0, 0};
    const bool found = locate_core<WideCell, WideCol>(A, S.pool + A.ref_off, (const int32_t *)(S.pool + A.ncount_off),
                                                      (const int32_t *)(S.pool + A.maxcost_off), enc + 256 * A.query_enc, rv,
                                                      wc, o, 0xFFFFFFFFu, 0, cost, score);
    result8[0] = found ? 1 : 0;
    for (int i = 0; i < 6; ++i) result8[1 + i] = o[i];
    return 0;
}

extern "C" int hs_process_batch(const cg_adapter_desc *adapters, int n_adapters,
                                const cg_group_desc *groups, int n_groups, const uint8_t *seq,
                                const uint8_t *qual, const int64_t *offsets, int64_t n_reads,
                                const cg_params *params, cg_match *matches, int32_t *qtrim,
                                int force_wide)
{
    return hs_process_batch_indexed(adapters, n_adapters, groups, n_groups, nullptr, 0, seq, qual, offsets,
                                    n_reads, params, matches, qtrim, force_wide);
}

// the two stand-alone 3'-end scans (qualtrim.pyx:76-169) as the kernels run them
extern "C" int hs_nextseq_trim(const uint8_t *seq, const uint8_t *qual, int n, int cutoff, int base)
{
    return nextseq_trim_core(seq, qual, n, cutoff, base);
}
extern "C" int hs_poly_a_trim(const uint8_t *seq, int n, int revcomp) { return poly_a_trim_core(seq, n, revcomp); }
extern "C" double hs_expected_errors(const uint8_t *qual, int n, int base)
{
    double table[256];
    cg_build_phred_table(table);
    return expected_errors_core(qual, n, base, table);
}


// ---- FASTQ path: the per-record logic of cg_fastq.cu (cg_fastq_core.cuh) on the host ---------------------------
// rec4: hdr_start, hdr_len, seq_start, qual_start per record; iparams: minimum_length, maximum_length,
// discard_trimmed, discard_untrimmed, poly_a, shorten, trim_n, discard_casava, action; dparams: max_n, max_ee.
extern "C" int hs_fastq_evaluate(const uint8_t *buf, int64_t n_records, const uint32_t *rec4, const int32_t *seq_len,
                                 const cg_match *matches, int times, int slots, const int32_t *qtrim,
                                 const int32_t *iparams, const double *dparams, int32_t *interval, int32_t *keep,
                                 int32_t *mask, int32_t *last_adapter)
{
    CgFastqFilter f;
    f.minimum_length = iparams[0]; f.maximum_length = iparams[1]; f.discard_trimmed = iparams[2];
    f.discard_untrimmed = iparams[3]; f.poly_a = iparams[4]; f.shorten = iparams[5]; f.trim_n = iparams[6];
    f.discard_casava = iparams[7]; f.action = iparams[8];
    f.max_n = dparams[0]; f.max_ee = dparams[1];
    double phred[256];
    cg_build_phred_table(phred);
    int bad = 0;
    for (int64_t r = 0; r < n_records; ++r) {
        CgFastqRecord rec;
        rec.hdr_start = rec4[4 * r]; rec.hdr_len = (int32_t)rec4[4 * r + 1];
        rec.seq_start = rec4[4 * r + 2]; rec.qual_start = rec4[4 * r + 3];
        const int n = seq_len[r];
        const int qs = qtrim ? qtrim[2 * r] : 0, qe = qtrim ? qtrim[2 * r + 1] : n;
        const FqVerdict v = fq_evaluate_core(buf, rec, n, matches ? (const cg_match_rec *)matches + (size_t)r * times * slots : nullptr,
                                             times, slots, qtrim != nullptr, qs, qe, f, phred);
        interval[2 * r] = v.start; interval[2 * r + 1] = v.stop;
        keep[2 * r] = v.k0; keep[2 * r + 1] = v.k1;
        mask[r] = v.mask; last_adapter[r] = v.last_adapter;
        bad |= v.bad_quality ? 1 : 0;
    }
    return bad;
}

extern "C" void hs_fastq_finish(int64_t n_records, const int32_t *mask1, const int32_t *mask2, int enabled1, int enabled2,
                                int mode, int mode_untrimmed, int32_t *fired)
{
    for (int64_t r = 0; r < n_records; ++r)
        fired[r] = fq_finish_core(mask1[r], mask2 ? mask2[r] : 0, mask2 != nullptr, enabled1, enabled2, mode, mode_untrimmed);
}

// record table of a chunk (fq_record_core); nl_pos is computed here the plain way.  Returns the first error code
// (0 = none) and its record in *bad_record.
extern "C" int hs_fastq_records(const uint8_t *buf, int64_t n, int cut_front, int cut_back, int64_t n_records,
                                uint32_t *rec4, int32_t *seq_len, int64_t *bad_record)
{
    std::vector<uint32_t> nl;
    for (int64_t i = 0; i < n; ++i)
        if (buf[i] == '\n') nl.push_back((uint32_t)i);
    int first = 0;
    *bad_record = -1;
    for (int64_t r = 0; r < n_records; ++r) {
        CgFastqRecord rec;
        int len;
        const int bad = fq_record_core(buf, n, nl.data(), (long long)nl.size(), r, cut_front, cut_back, &rec, &len);
        if (bad && *bad_record < 0) { first = bad; *bad_record = r; }
        rec4[4 * r] = rec.hdr_start; rec4[4 * r + 1] = (uint32_t)rec.hdr_len;
        rec4[4 * r + 2] = rec.seq_start; rec4[4 * r + 3] = rec.qual_start;
        seq_len[r] = len;
    }
    return first;
}
