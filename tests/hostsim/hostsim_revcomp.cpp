// tests/hostsim/hostsim_revcomp.cpp -- TEST-ONLY host build of the pair decision of --revcomp on pairs
// (fq_pair_swap_core in cutadapt_b200/csrc/cg_fastq_core.cuh), linked into libhostsim.so next to hostsim.cpp so that
// tests/test_paired_revcomp_host.py can check it against a restatement of the rule without a GPU.  Nothing in
// cutadapt_b200/ loads this library; it is not a fallback.
#include <string.h>

#include "../../cutadapt_b200/csrc/cg_core.cuh"
#include "../../cutadapt_b200/csrc/cg_fastq_core.cuh"

// out[p] = fq_pair_swap_core of pair p.  m11 / m12 hold per1 records per pair, m22 / m21 per2; a null pointer is a
// missing cutter.
extern "C" void hs_pair_swap(int64_t n_pairs, const cg_match_rec *m11, const cg_match_rec *m22, const cg_match_rec *m12,
                             const cg_match_rec *m21, int per1, int per2, int32_t *out)
{
    for (int64_t p = 0; p < n_pairs; ++p)
        out[p] = fq_pair_swap_core(m11 ? m11 + p * per1 : nullptr, m22 ? m22 + p * per2 : nullptr,
                                   m12 ? m12 + p * per1 : nullptr, m21 ? m21 + p * per2 : nullptr, per1, per2)
                     ? 1 : 0;
}
