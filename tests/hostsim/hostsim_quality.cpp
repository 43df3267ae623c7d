// tests/hostsim/hostsim_quality.cpp -- TEST-ONLY host build of the quality filters of the FASTQ path: fq_evaluate_core
// (cutadapt_b200/csrc/cg_fastq_core.cuh) with --max-aer (TooHighAverageErrorRate) and -z (ZeroCapper), linked into
// libhostsim.so next to hostsim.cpp so that tests/test_quality_filters_host.py can check it against the oracle without a
// GPU.  Nothing in cutadapt_b200/ loads this library; it is not a fallback.
#include <string.h>

#include "../../cutadapt_b200/csrc/cg_core.cuh"
#include "../../cutadapt_b200/csrc/cg_fastq_core.cuh"
#include "../../cutadapt_b200/csrc/cg_setbuild.h"

// hs_fastq_evaluate (hostsim.cpp) with the two new fields: iparams = minimum_length, maximum_length, discard_trimmed,
// discard_untrimmed, poly_a, shorten, trim_n, discard_casava, action, zero_cap (the cap character, 0 = off);
// dparams = max_n, max_ee, max_aer (0 = off).  Returns 1 when a quality filter met a character outside [33, 126].
extern "C" int hs_fastq_evaluate_quality(const uint8_t *buf, int64_t n_records, const uint32_t *rec4, const int32_t *seq_len,
                                         const cg_match_rec *matches, int times, int slots, const int32_t *qtrim,
                                         const int32_t *iparams, const double *dparams, int32_t *interval, int32_t *mask)
{
    CgFastqFilter f;
    f.minimum_length = iparams[0]; f.maximum_length = iparams[1]; f.discard_trimmed = iparams[2];
    f.discard_untrimmed = iparams[3]; f.poly_a = iparams[4]; f.shorten = iparams[5]; f.trim_n = iparams[6];
    f.discard_casava = iparams[7]; f.action = iparams[8]; f.zero_cap = iparams[9];
    f.max_n = dparams[0]; f.max_ee = dparams[1]; f.max_aer = dparams[2];
    double phred[256];
    cg_build_phred_table(phred);
    int bad = 0;
    for (int64_t r = 0; r < n_records; ++r) {
        CgFastqRecord rec;
        rec.hdr_start = rec4[4 * r]; rec.hdr_len = (int32_t)rec4[4 * r + 1];
        rec.seq_start = rec4[4 * r + 2]; rec.qual_start = rec4[4 * r + 3];
        const int n = seq_len[r];
        const int qs = qtrim ? qtrim[2 * r] : 0, qe = qtrim ? qtrim[2 * r + 1] : n;
        const FqVerdict v = fq_evaluate_core(buf, rec, n, matches ? matches + (size_t)r * times * slots : nullptr,
                                             times, slots, qtrim != nullptr, qs, qe, f, phred);
        interval[2 * r] = v.start; interval[2 * r + 1] = v.stop;
        mask[r] = v.mask;
        bad |= v.bad_quality ? 1 : 0;
    }
    return bad;
}

// expected_errors_core with ZeroCapper's cap in front of it (0 = no cap)
extern "C" double hs_expected_errors_capped(const uint8_t *qual, int n, int cap)
{
    double table[256];
    cg_build_phred_table(table);
    return expected_errors_core(qual, n, 33, table, cap);
}
