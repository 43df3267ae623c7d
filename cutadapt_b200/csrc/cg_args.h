// cg_args.h -- the argument block of the trimming kernels (shared by nvcc and NVRTC translation units).
#pragma once
#include "cg_core.cuh"

#ifndef CG_NT
#define CG_NT 128  // lanes (= reads) per CTA tile
#endif

struct CgKernelArgs {
    // adapter tables (HBM)
    const uint8_t *blob;
    uint32_t blob_bytes;
    const uint64_t *masks64;
    const uint8_t *enc;  // 768 bytes
    const uint8_t *index;  // CgIndexHeader[] | CgIndexEntry[] for INDEXED groups, or null
    // batch (HBM)
    const uint8_t *seq;
    const uint8_t *qual;
    const int64_t *offsets;
    long long n_reads;
    // parameters
    int quality_trim, cutoff_front, cutoff_back, qbase, times, slots;
    // outputs (HBM)
    cg_match_rec *out;
    int32_t *qtrim;
    const int32_t *view;  // optional per-read (start, stop): search read[start:stop] instead of the
                          // quality-trimmed read (per-adapter passes of the multi-pass schedule)
    int *err_flag;
    // fused-kernel geometry
    int tile_cap;  // bytes per staged tile (multiple of 16)
    int col_rows;  // max_m + 1
    // warp-autonomous kernel geometry
    int mini_cap;    // bytes per staged 32-read mini-tile (multiple of 16)
    int carry_slot;  // bytes per carried task (multiple of 16)
    // split pipeline (scan kernel -> task list in HBM -> DP kernel)
    int task_rec;                     // uint4 words per task of the plan stage's input list (2: scan kernel; cg_pscan_kernel:
                                      // 4 + 2 W + 1, header + the window bytes)
    uint4 *tasks;                     // task_rec x uint4 per task
    unsigned long long *task_count;   // number of tasks appended by the scan kernel
    unsigned long long *task_count_b; // cg_pscan_kernel: tasks WITHOUT locator hits are filed from the end of `tasks`
                                      // backwards and counted here, so that the warps of the plan stage work on reads
                                      // of one kind (null: one list)
    long long task_cap;
    uint4 *tasks2;                    // output list of the plan / run kernels: 4 x uint4 per record
    unsigned long long *task2_count;
    unsigned long long *task2_count_b; // plan stage: run records whose first run has no band (run_band_d) are filed from
                                      // the end of tasks2 backwards and counted here (null: one list)
    uint4 *tasks3;                    // plan stage only: reads of cg_pscan_kernel whose window holds other letters than
    unsigned long long *task3_count;  //   A/C/G/T go here (2 x uint4, CG_TASK_RESCAN) for a second, dense plan launch
    int no_band;                      // 1: the DP runs keep all rows (CUTADAPT_B200_NO_BAND=1, for A/B runs)
    // statistics fused into the first stage (cg_pscan.cuh): the reads it settles are counted here, the rest by
    // cg_stats_kernel over the task list once their records are final.  null = not fused (the variant of the first
    // stage without the statistics code runs).
    unsigned long long *stats;
    int stats_max_len, stats_kmax;
    // generic-kernel scratch
    uint32_t *scratch_p;
    int *scratch_w;
    long long scratch_stride;
};

