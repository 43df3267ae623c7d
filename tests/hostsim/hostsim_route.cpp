// tests/hostsim/hostsim_route.cpp -- TEST-ONLY host build of the filter-output routing of the FASTQ path
// (fq_finish_core, fq_route_enabled, fq_route_core in cutadapt_b200/csrc/cg_fastq_core.cuh), linked into libhostsim.so
// next to hostsim.cpp so that tests/test_filter_outputs_host.py can check it against a model of the reference's filter
// chain without a GPU.  Nothing in cutadapt_b200/ loads this library; it is not a fallback.
#include <string.h>

#include <vector>

#include "../../cutadapt_b200/csrc/cg_core.cuh"
#include "../../cutadapt_b200/csrc/cg_fastq_core.cuh"

// What fq_finish_kernel does per record with a route: the filter that fired (fired[r], -1 none) and the destination
// (dest[r]: 0 main, 1 too-short, 2 too-long, 3 untrimmed, -1 dropped).  mask2 == nullptr: single-end.
extern "C" void hs_fastq_route(int64_t n_records, const int32_t *mask1, const int32_t *mask2, int enabled1, int enabled2,
                               int mode, int mode_untrimmed, int redirect, int32_t *fired, int32_t *dest)
{
    const int e1 = fq_route_enabled(enabled1, redirect), e2 = fq_route_enabled(enabled2, redirect);
    for (int64_t r = 0; r < n_records; ++r) {
        const int k = fq_finish_core(mask1[r], mask2 ? mask2[r] : 0, mask2 != nullptr, e1, e2, mode, mode_untrimmed);
        fired[r] = k;
        dest[r] = fq_route_core(k, redirect);
    }
}
