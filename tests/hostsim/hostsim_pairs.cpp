// tests/hostsim/hostsim_pairs.cpp -- TEST-ONLY host build of the mate-name check of interleaved input (fq_mates_match in
// cutadapt_b200/csrc/cg_fastq_core.cuh), linked into libhostsim.so next to hostsim.cpp so that
// tests/test_interleaved_host.py can check it against a restatement of the rule without a GPU.  Nothing in
// cutadapt_b200/ loads this library; it is not a fallback.
#include <string.h>

#include "../../cutadapt_b200/csrc/cg_core.cuh"
#include "../../cutadapt_b200/csrc/cg_fastq_core.cuh"

// out[p] = 1 when headers 2p and 2p + 1 (back to back in `names`, header k = names[off[k] .. off[k + 1])) name mates
extern "C" void hs_mates_match(int64_t n_pairs, const uint8_t *names, const int64_t *off, int32_t *out)
{
    for (int64_t p = 0; p < n_pairs; ++p) {
        const int64_t a = off[2 * p], b = off[2 * p + 1], e = off[2 * p + 2];
        out[p] = fq_mates_match(names + a, (int)(b - a), names + b, (int)(e - b)) ? 1 : 0;
    }
}
