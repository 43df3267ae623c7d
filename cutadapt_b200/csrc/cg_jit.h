// cg_jit.h -- per-adapter-set specialisation of the bit-plane first stage with NVRTC.
//
// The op list of the plane program (cg_types.h) is written out as a sequence of plane_chain_step /
// plane_emit calls with literal arguments; cg_pscan.cuh (embedded in the library at build time together with
// the headers it includes) is compiled around it for sm_90a.  The compiler then sees every plane, shift, window
// mask and flag as a constant: ~45 instructions per chain step of the interpreter become the 10 that do the work.
// libnvrtc and libcuda are opened at run time (dlopen); if either is missing or the compilation fails the
// precompiled interpreter kernel keeps running and cg_jit_last_error() says why.
#pragma once
#include <stdint.h>
#include <string>

#include "cg_setbuild.h"

struct CgJitKernel;   // a loaded module + entry point

// Compile the plane program of `set` for W plane words; stats: the variant that counts the trim statistics of the
// reads it settles (cg_pscan.cuh).  Returns nullptr on failure (err filled).
CgJitKernel *cg_jit_build_pscan(const CgBuiltSet &set, int W, bool has_qual, bool stats, std::string &err);
void cg_jit_destroy(CgJitKernel *k);
// the generated translation unit (for inspection and the tests)
std::string cg_jit_pscan_source(const CgBuiltSet &set, int W, bool has_qual, bool stats = false);
// resident CTAs per SM for the given launch shape; <= 0 on error
int cg_jit_occupancy(CgJitKernel *k, int block, size_t smem);
// launches kernel(const CgKernelArgs) -- `args` points at the argument block; returns 0 or a CUresult
int cg_jit_launch(CgJitKernel *k, int grid, int block, size_t smem, void *stream, const void *args);
// compile only (no device needed): PTX/cubin size or -1; used by the CPU tests to check that the generated
// source builds for sm_90a
long cg_jit_compile_only(const CgBuiltSet &set, int W, bool has_qual, std::string &log, bool stats = false);
