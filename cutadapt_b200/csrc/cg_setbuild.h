// cg_setbuild.h -- host-side compiler: cg_adapter_desc[] / cg_group_desc[] -> device blob.
// Pure C++ (no CUDA) so that tests/hostsim can link it as well.
#pragma once
#include <stdint.h>
#include <string>
#include <vector>

#include "../../include/cutadapt_b200.h"
#include "cg_types.h"

struct CgBuiltSet {
    std::vector<uint8_t> blob;       // CgSetHeader | adapters | groups | entries | pool
    std::vector<uint64_t> masks64;   // 128 words per prefilter entry
    std::vector<int32_t> effective_length;  // per adapter
    std::vector<uint8_t> index_blob; // CgIndexHeader[n_indexes] | CgIndexEntry tables (HBM), may be empty
    int slots = 1;
    int n_adapters = 0, n_groups = 0, max_m = 0, any_wide = 0, simple_ok = 0;
    int all_indexed = 0;             // every group is an index lookup (IndexedPrefixAdapters / IndexedSuffixAdapters)
    int max_k = 0;                   // most errors any adapter can report: max (int)(max_error_rate * length)
};

// 3 x 256 bytes: upper, acgt, iupac  (src/cutadapt/_match_tables.py:4-66)
void cg_build_enc_tables(uint8_t *out768);

// table[q] = 10^(-q/10) as double, q = 0..255 (the first 94 entries equal SCORE_TO_ERROR_RATE of
// expected_errors.h bit for bit; tests/golden pins that)
void cg_build_phred_table(double *out256);

// Returns CG_OK or a negative code and fills `err`.
int cg_build_set(const cg_adapter_desc *adapters, int n_adapters, const cg_group_desc *groups,
                 int n_groups, CgBuiltSet &out, std::string &err,
                 const cg_index_desc *indexes = nullptr, int n_indexes = 0);

// ---- multi-pass schedule (several groups, one round) ------------------------------------------
// One single-adapter (or single-index) sub-set per component of every group, so that every aligner
// adapter runs through the split pipeline (scan -> plan -> DP rounds) on its own; select_best()
// (cg_core.cuh) then combines the per-adapter records.  Only planned when every aligner component
// qualifies for that pipeline and there are at most CG_MAX_PASSES components.
struct CgPassPlan {
    CgBuiltSet set;
    int group = 0, role = 0;      // role 1: back adapter of a LINKED group
    int front_pass = -1;          // role 1: the pass of the front adapter
    int map_off = 0;              // first entry in pass_map (local -> global adapter numbers)
};
struct CgMultiPlan {
    std::vector<CgPassPlan> passes;   // empty: keep the one-kernel schedule
    std::vector<int32_t> pass_map;
};
int cg_plan_passes(const cg_adapter_desc *adapters, int n_adapters, const cg_group_desc *groups, int n_groups,
                   const cg_index_desc *indexes, int n_indexes, CgMultiPlan &plan, std::string &err);
void cg_fill_select_tables(const CgGroup *groups, int n_groups, int slots, const std::vector<CgPassPlan> &passes,
                           CgSelectTables &t);
