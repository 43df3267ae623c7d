// cg_kernels.cuh -- launch-side declarations shared by cg_kernels.cu and cg_api.cu
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cg_core.cuh"

#include "cg_args.h"

// SMs of the current device: the grid-stride launches are sized in blocks per SM
int cg_device_sm_count();
static inline long long cg_grid_cap(long long grid, int blocks_per_sm)
{
    const long long cap = (long long)blocks_per_sm * cg_device_sm_count();
    return grid > cap ? cap : grid;
}

// Multi-pass schedule (several adapters, one round): every component adapter runs as its own pass into a
// scratch array of records; cg_select_kernel then applies MultipleAdapters.match_to / LinkedAdapter.match_to
// to the per-adapter results.
struct CgSelectArgs {
    const cg_match_rec *tmp;      // [n_passes][stride] records of the passes
    long long stride;
    long long n_reads;
    cg_match_rec *out;            // n_reads * slots
    const int32_t *pass_map;      // local -> global adapter numbers of all passes, concatenated
    CgSelectTables t;
};
cudaError_t cg_launch_select(const CgSelectArgs &a, cudaStream_t st);
// view of the back adapter of a LinkedAdapter: the base view with the front match trimmed off
cudaError_t cg_launch_linked_view(const cg_match_rec *front, const int32_t *base_view, const int64_t *offsets,
                                  long long n_reads, int32_t *out_view, cudaStream_t st);

size_t cg_fast_smem_bytes(uint32_t blob_bytes, int tile_cap, int col_rows, bool has_qual);
cudaError_t cg_launch_fast(const CgKernelArgs &a, bool has_qual, bool simple, int grid, size_t smem, cudaStream_t st);
cudaError_t cg_fast_occupancy(bool has_qual, bool simple, size_t smem, int *blocks_per_sm);
size_t cg_warp_smem_bytes(uint32_t blob_bytes, int mini_cap, int carry_slot, bool has_qual);
cudaError_t cg_warp_occupancy(bool has_qual, size_t smem, int *blocks_per_sm);
cudaError_t cg_launch_warp(const CgKernelArgs &a, bool has_qual, int grid, size_t smem, cudaStream_t st);
size_t cg_scan_smem_bytes(uint32_t blob_bytes, int mini_cap, bool has_qual);
cudaError_t cg_scan_occupancy(bool has_qual, size_t smem, int *blocks_per_sm);
cudaError_t cg_launch_scan(const CgKernelArgs &a, bool has_qual, int grid, size_t smem, cudaStream_t st);
// sets of index lookups only (cg_trim_light_kernel): rows of the local-memory column for the rare re-alignment
#define CG_LIGHT_ROWS 68
cudaError_t cg_launch_light(const CgKernelArgs &a, int grid, cudaStream_t st);
// one round over index groups without views: cg_index_kernel + cg_trim_listed_kernel for the reads it lists in
// a.tasks (32-bit read numbers, counted in a.task_count, which must be zero)
cudaError_t cg_launch_index(const CgKernelArgs &a, int grid, cudaStream_t st);
size_t cg_pscan_smem_bytes(uint32_t blob_bytes, int mini_cap, bool has_qual, int stats_max_len = -1);   // >= 0: + fused statistics
// stats: the variant that counts the trim statistics of the reads it settles (without qualities only); cg_launch_pscan
// runs it when a.stats is set
cudaError_t cg_pscan_occupancy(bool has_qual, int w, bool stats, size_t smem, int *blocks_per_sm);
cudaError_t cg_launch_pscan(const CgKernelArgs &a, bool has_qual, int w, int grid, size_t smem, cudaStream_t st);
size_t cg_dp_smem_bytes(uint32_t blob_bytes, int slot_bytes);
// stats: the variant that lists the statistics of the reads it finishes (a.stat_ents); cg_launch_list runs it when a.stats
// is set
cudaError_t cg_list_occupancy(bool plan, int mr, bool stats, size_t smem, int *blocks_per_sm);
cudaError_t cg_launch_list(const CgKernelArgs &a, bool plan, int mr, int grid, size_t smem, cudaStream_t st);
cudaError_t cg_launch_generic(const CgKernelArgs &a, int grid, int block, cudaStream_t st);
cudaError_t cg_launch_locate_debug(const uint8_t *d_blob, const uint8_t *d_enc, const uint8_t *d_query, int n,
                                   int *d_scratch, int32_t *d_cost, int32_t *d_score, int32_t *d_result, cudaStream_t st);
cudaError_t cg_launch_kmers_present(const CgEntry *d_entries, int n_entries, const uint64_t *d_masks,
                                    const uint8_t *d_seq, const int64_t *d_offsets, long long n_reads,
                                    uint8_t *d_out, int *d_err, cudaStream_t st);
cudaError_t cg_launch_quality_trim(const uint8_t *d_qual, const int64_t *d_offsets, long long n_reads,
                                   int cutoff_front, int cutoff_back, int base, int32_t *d_out,
                                   cudaStream_t st);
cudaError_t cg_launch_max_len(const int64_t *d_offsets, long long n_reads, int *d_out, cudaStream_t st);
cudaError_t cg_launch_stats(const uint8_t *d_seq, const int64_t *d_offsets, long long n_reads, int quality_trim, int times,
                            int slots, const cg_match_rec *d_matches, const int32_t *d_qtrim,
                            int n_adapters, int max_len, int kmax, unsigned long long *d_stats,
                            cudaStream_t st,
                            int count_lengths = 1,     // 0: leave the read-length histogram alone
                            int upper = 0);            // adjacent bases of the upper-cased read (--action=lowercase)
// the statistics of the *d_count (at most cap) entries the plan and run kernels listed (one adapter); the launch needs
// cg_stats_entries_smem_bytes(max_len, kmax) <= 48 KiB of shared memory
size_t cg_stats_entries_smem_bytes(int max_len, int kmax);
cudaError_t cg_launch_stats_entries(const uint2 *d_ents, const unsigned long long *d_count, long long cap, int max_len,
                                    int kmax, unsigned long long *d_stats, cudaStream_t st);
cudaError_t cg_launch_nextseq_trim(const uint8_t *d_seq, const uint8_t *d_qual, const int64_t *d_offsets,
                                   long long n_reads, int cutoff, int base, int32_t *d_out, cudaStream_t st);
cudaError_t cg_launch_poly_a_trim(const uint8_t *d_seq, const int64_t *d_offsets, long long n_reads, int revcomp,
                                  int32_t *d_out, cudaStream_t st);
cudaError_t cg_launch_expected_errors(const uint8_t *d_qual, const int64_t *d_offsets, long long n_reads, int base,
                                      const double *d_table, double *d_out, cudaStream_t st);
cudaError_t cg_launch_fill_offsets(int64_t *d_out, long long base, long long len, long long count, cudaStream_t st);
// expansion of the compressed host-to-device stream (cg_hostpack.h): packed_bytes is a multiple of 16,
// d_out receives 3 * packed_bytes characters, then the n_exc exceptions (position << 8 | byte)
cudaError_t cg_launch_unpack3(const uint8_t *d_packed, long long packed_bytes, uint8_t *d_out,
                              const unsigned long long *d_exc, long long n_exc, cudaStream_t st);

// ---- FASTQ chunk parse / trimmed-record formatting (cg_fastq.cu) ---------------------------------------
#include "cg_fastq_core.cuh"   // CgFastqRecord, CgFastqFilter, CG_FQ_ACTION_*, the per-record logic
#define CG_FQ_COUNTERS 16    // written, bp_in, bp_out, with_adapters, too_short, too_long, quality_trimmed_bp,
                             // discarded (trimmed/untrimmed), too_many_n, too_many_expected_errors, casava_filtered,
                             // reverse_complemented, too_high_average_error_rate
long long cg_fastq_tiles(long long n_bytes);
long long cg_scan_tiles(long long n);
// phase 0: newline count per tile + exclusive scan (total -> *d_total); phase 1: positions of the newlines
cudaError_t cg_launch_fastq_index(const uint8_t *d_buf, long long n_bytes, uint32_t *d_tile_counts,
                                  unsigned long long *d_total, uint32_t *d_nl_pos, int phase, cudaStream_t st);
cudaError_t cg_launch_fastq_records(const uint8_t *d_buf, long long n_bytes, const uint32_t *d_nl_pos, long long n_newlines,
                                    long long n_records, int cut_front, int cut_back, CgFastqRecord *d_rec,
                                    int32_t *d_seq_len, int32_t *d_origin, unsigned long long *d_counters, int *d_err,
                                    cudaStream_t st);
// FASTA chunk -> normalised chunk + record table (fa_line_core / fa_record_core): classify every line (bytes it keeps,
// header flag, first header line: *d_first_hdr must start at INT_MAX); after exclusive scans of keep (line offsets in
// the normalised buffer) and is_hdr (record of each header) the scatter writes the normalised buffer, hdr_start /
// hdr_len of every record and the first bad line (d_err as one 64-bit word: line << 32 | code); then the records.
cudaError_t cg_launch_fasta_classify(const uint8_t *d_buf, long long n_bytes, const uint32_t *d_nl_pos, long long n_newlines,
                                     long long n_lines, int32_t *d_keep, int32_t *d_is_hdr, int *d_first_hdr, cudaStream_t st);
cudaError_t cg_launch_fasta_scatter(const uint8_t *d_buf, long long n_bytes, const uint32_t *d_nl_pos, long long n_newlines,
                                    long long n_lines, const int64_t *d_line_off, const int64_t *d_hdr_idx,
                                    const int *d_first_hdr, uint8_t *d_norm, CgFastqRecord *d_rec, int *d_err,
                                    cudaStream_t st);
cudaError_t cg_launch_fasta_records(CgFastqRecord *d_rec, long long n_records, long long n_norm, int cut_front, int cut_back,
                                    int32_t *d_seq_len, int32_t *d_origin, unsigned long long *d_counters, cudaStream_t st);
// exclusive scan int32 -> int64, n + 1 outputs; d_tile_scratch: cg_scan_tiles(n) words
cudaError_t cg_launch_scan_i32(const int32_t *d_in, long long n, unsigned long long *d_tile_scratch, int64_t *d_out,
                               cudaStream_t st);
cudaError_t cg_launch_fastq_gather(const uint8_t *d_buf, const CgFastqRecord *d_rec, const int64_t *d_offsets,
                                   long long n_records, uint8_t *d_seq, uint8_t *d_qual, int rc, cudaStream_t st);
// the quality-trimmed interval becomes the record (counters[6] += removed bases)
cudaError_t cg_launch_fastq_fold_qtrim(CgFastqRecord *d_rec, int32_t *d_seq_len, const int32_t *d_qtrim, long long n_records,
                                       int32_t *d_origin, unsigned long long *d_counters, cudaStream_t st);
// --revcomp: choose the orientation per record, rewrite the chosen reads in place (counters[11] += replaced)
cudaError_t cg_launch_fastq_revcomp_commit(uint8_t *d_buf, CgFastqRecord *d_rec, const int32_t *d_seq_len, int32_t *d_origin,
                                           long long n_records, cg_match_rec *d_matches, const cg_match_rec *d_matches_rc,
                                           int per_read, uint8_t *d_is_rc, unsigned long long *d_counters, cudaStream_t st,
                                           int has_qual = 1);
// --revcomp on pairs: decide every pair, swap the records and matches of the swapped ones between the two slots
// (counters[11] of both += swapped pairs)
cudaError_t cg_launch_fastq_pair_swap(long long n_pairs, CgFastqRecord *d_rec1, int32_t *d_len1, int32_t *d_origin1,
                                      cg_match_rec *d_m11, const cg_match_rec *d_m21, int per1, CgFastqRecord *d_rec2,
                                      int32_t *d_len2, int32_t *d_origin2, cg_match_rec *d_m22, const cg_match_rec *d_m12,
                                      int per2, uint32_t base1, uint32_t base2, uint8_t *d_is_rc1, uint8_t *d_is_rc2,
                                      unsigned long long *d_counters1, unsigned long long *d_counters2, cudaStream_t st);
cudaError_t cg_launch_fastq_pretrim(const uint8_t *d_buf, const CgFastqRecord *d_rec, const int32_t *d_seq_len,
                                    long long n_records, int flags, int cutoff_front, int cutoff_back, int qbase,
                                    int32_t *d_qtrim, cudaStream_t st);
// kept interval + one bit per filter the read fails (bit order: too short, too long, too many N, too many expected
// errors, casava, trimmed, untrimmed, too high average error rate; CG_FQ_MASK_RC from d_is_rc); per-read counters (with_adapters, quality_trimmed_bp)
cudaError_t cg_launch_fastq_evaluate(const uint8_t *d_buf, const CgFastqRecord *d_rec, const int32_t *d_seq_len,
                                     long long n_records, const cg_match_rec *d_matches, int times, int slots,
                                     const int32_t *d_qtrim, CgFastqFilter f, const double *d_phred, const uint8_t *d_is_rc,
                                     int32_t *d_interval, int32_t *d_keep_interval, int32_t *d_fail_mask,
                                     unsigned long long *d_counters, int *d_err, cudaStream_t st,
                                     int32_t *d_poly_a_len = nullptr);   // optional: bases PolyATrimmer removed, per read
// statistics of the FASTQ path beyond the match records (after the finish kernel): written lengths of the records with
// d_out_len != 0, the poly-A histogram (d_poly_a_len may be null), reverse_complemented per adapter (per match of the
// records with d_is_rc set; d_is_rc may be null); every histogram has max_len + 1 bins.  d_route (filter outputs, may
// be null): only records routed to the main output (0) count as written.
cudaError_t cg_launch_fastq_stats_tail(long long n_records, const int32_t *d_interval, const int32_t *d_out_len,
                                       const int32_t *d_poly_a_len, const cg_match_rec *d_matches, int times, int slots,
                                       const uint8_t *d_is_rc, int n_adapters, int max_len, unsigned long long *d_lengths,
                                       unsigned long long *d_poly_a, unsigned long long *d_rc, cudaStream_t st,
                                       const int32_t *d_route = nullptr);
// verdict per read (second mate = nullptr) or pair -> sizes of the output records, filter counters.  d_route (filter
// outputs, may be null): every record's destination (fq_route_core of `redirect`, -1 = dropped); a redirected record is
// sized in its destination's format (bit d of fasta_dests: destination d is FASTA; fasta_out is then unused).
cudaError_t cg_launch_fastq_finish(long long n_records, const CgFastqRecord *d_rec1, const int32_t *d_interval1,
                                   const int32_t *d_mask1, int enabled1, int32_t *d_out_len1,
                                   unsigned long long *d_counters1, const CgFastqRecord *d_rec2,
                                   const int32_t *d_interval2, const int32_t *d_mask2, int enabled2, int32_t *d_out_len2,
                                   unsigned long long *d_counters2, int mode, int mode_untrimmed, int rc_suffix,
                                   const int32_t *d_dest, const uint8_t *d_dest_keep, cudaStream_t st, int fasta_out = 0,
                                   int redirect = 0, int fasta_dests = 0, int32_t *d_route = nullptr);
// d_route (may be null): write only the records whose destination's bit in fasta_dests equals fasta_out; zero_cap:
// quality characters below it are written as it (ZeroCapper), 0 = off
cudaError_t cg_launch_fastq_write(const uint8_t *d_buf, const CgFastqRecord *d_rec, const int32_t *d_interval,
                                  const int64_t *d_out_off, const int32_t *d_out_len, long long n_records,
                                  uint8_t *d_out, int action, const int32_t *d_keep_interval, const int32_t *d_mask,
                                  int rc_suffix, cudaStream_t st, int fasta_out = 0, const int32_t *d_route = nullptr,
                                  int fasta_dests = 0, int zero_cap = 0);
// demultiplexing: cg_launch_fastq_dest gives every record its destination (adapter of the most recent match of R1, or
// of both mates: d1 * (n_named2 + 1) + d2; reads without a match: the last value of the dimension); phase 0 fills
// d_bytes[n_dest][tiles] (output bytes per destination and tile of 256 records); after an exclusive scan of that
// array (d_base), phase 1 writes every record's output offset.
long long cg_demux_tiles(long long n_records);
cudaError_t cg_launch_fastq_dest(const int32_t *d_mask1, const int32_t *d_mask2, long long n_records,
                                 const int32_t *d_adapter_dest1, int n_named1, const int32_t *d_adapter_dest2, int n_named2,
                                 int32_t *d_dest, cudaStream_t st);
cudaError_t cg_launch_fastq_demux(int phase, const int32_t *d_out_len, const int32_t *d_dest, long long n_records,
                                  int n_dest, int32_t *d_bytes, const int64_t *d_base, int64_t *d_out_off, cudaStream_t st);
// --info-file rows: phase 0 = bytes of every record's rows, phase 1 (after a scan) = the rows
// ---- read names (cg_names_core.cuh): the name stage of a collect ----
#include "cg_names_core.cuh"
// One mate of the stage: its chunk (the names go into an arena behind the chunk's bytes, in the same buffer, and the
// record table is repointed at them), its record table and verdict, its matches, and where -u took its bases.
struct CgNameMate {
    uint8_t *buf;
    CgFastqRecord *rec;
    const int32_t *interval;      // the read as written: LengthTagModifier's length
    int32_t *mask;                // fail_mask: last adapter, RC bit; the CasavaFiltered bit is redone on the new name
    const int32_t *origin;        // (bases in front of the record in the read as it came, length of that read)
    const int32_t *seq_len, *qtrim;
    const cg_match_rec *matches;
    int times, slots;
    int mate;                     // 0 = R1 / single-end, 1 = R2
    int rc_suffix;                // the writers' " rc": the start name gets it instead
    int swapped;                  // paired --revcomp: a turned pair's reads sit in the other mate's slot (no reversal)
    int cut_front, cut_back;      // -u totals of this mate
};
// phase 0: bytes of every record's name (d_len1 / d_len2); phase 1: the names at arena + d_off, records repointed.
// rename 0: step 1 (tag, suffixes, prefix / suffix) per record of m1; rename 1: the template over the step-1 names, one
// thread per record of m1 or pair (m2.buf != nullptr); a pair whose step-1 names (code 0) or new names (code 1) do not
// name mates sets *d_mismatch to min(pair << 1 | code).  casava: bit 0 / bit 1 = --discard-casava of m1 / m2 (step 1:
// bit 0 for m1), its bit is redone on the final names.
cudaError_t cg_launch_fastq_names(int phase, int rename, const uint8_t *d_blob, CgNameMate m1, CgNameMate m2,
                                  long long n_records, int32_t *d_len1, int32_t *d_len2, const int64_t *d_off1,
                                  const int64_t *d_off2, uint32_t arena1, uint32_t arena2, int casava,
                                  unsigned long long *d_mismatch, cudaStream_t st);
cudaError_t cg_launch_fastq_info(int phase, const uint8_t *d_buf, const CgFastqRecord *d_rec, const int32_t *d_origin,
                                 const int32_t *d_interval, const int32_t *d_mask, const cg_match_rec *d_matches, int times,
                                 int slots, const uint8_t *d_names, const int32_t *d_name_off, int revcomp, int rc_suffix,
                                 int upper_unmatched, long long n_records, int32_t *d_row_bytes, const int64_t *d_row_off,
                                 uint8_t *d_out, cudaStream_t st, int kind = 0, const int32_t *d_qtrim = nullptr,
                                 const int32_t *d_seq_len = nullptr,    // kind 1 / 2: --rest-file / --wildcard-file rows
                                 int has_qual = 1,                      // 0: FASTA input, empty quality columns
                                 int zero_cap = 0);                     // ZeroCapper on the rows of unmatched reads
// interleaved input: phase 0 = per record of the chunk its span (d_start, d_size), mate (d_dest = r & 1) and name
// (d_rec; FASTQ: from the line index d_nl_pos, format checked; FASTA, d_nl_pos == nullptr: d_rec is the normalised
// chunk's record table), then the mate-name check per pair; d_err: first problem, record << 32 | code.  After the
// demultiplexer's partition of d_size by d_dest (d_off), phase 1 copies every record into d_out1 / d_out2 (mate 2's
// offsets start at seg1; fasta: a '\n' is appended to every record).
cudaError_t cg_launch_interleaved_split(int phase, const uint8_t *d_buf, long long n_bytes, const uint32_t *d_nl_pos,
                                        long long n_newlines, long long n_records, CgFastqRecord *d_rec, int32_t *d_start,
                                        int32_t *d_size, int32_t *d_dest, unsigned long long *d_err, const int64_t *d_off,
                                        long long seg1, uint8_t *d_out1, uint8_t *d_out2, int fasta, cudaStream_t st);
// interleaved outputs (bit d of ilv: destination d of d_route): phase 0 folds the sizes of such pairs into mate 1
// (d_fold1 / d_fold2, what the partition runs on); phase 1, after the partitions, gives mate 2 of such a pair the offset
// off1 + len1 and moves every other record of mate 2 behind mate 1's region (*d_total1 bytes)
cudaError_t cg_launch_fastq_interleave(int phase, long long n_records, const int32_t *d_route, int ilv,
                                       const int32_t *d_len1, const int32_t *d_len2, int32_t *d_fold1, int32_t *d_fold2,
                                       const int64_t *d_off1, int64_t *d_off2, const int64_t *d_total1, cudaStream_t st);
// gzip outputs (cg_gzip.cu): a piece of at most GZ_MEMBER bytes of a destination, at d_src + src; gz = 1 compresses it
// into one member, gz = 0 copies it.  Piece k goes to d_slots + k * GZ_SLOT, its size to d_sizes[k]; the gather then
// packs the pieces to d_out + d_dst_off[k].
struct CgGzPiece {
    long long src;
    int32_t len;
    int32_t gz;
};
cudaError_t cg_launch_gzip_compress(const uint8_t *d_src, const CgGzPiece *d_pieces, int n_pieces, uint8_t *d_slots,
                                    int32_t *d_sizes, cudaStream_t st);
cudaError_t cg_launch_gzip_gather(const uint8_t *d_slots, const int32_t *d_sizes, const int64_t *d_dst_off, int n_pieces,
                                  uint8_t *d_out, cudaStream_t st);
// gzip input (cg_gunzip.cu, decisions in cg_gunzip_core.cuh): phase 0 counts the positions of 1f 8b 08 per tile of
// cg_gunzip_tiles, phase 1 (after an exclusive scan of the counts) writes them in order; parse every candidate (no
// output); the chain (one thread); inflate the chain's members into d_out + their offsets and check their CRC-32
// (*d_bad: the first bad member, start it at INT_MAX).  Record cut: flag the newlines of the line index (gu_flag); after
// an exclusive scan of the flags, the select writes the offset behind flagged newline number s to *d_cut.
#include "cg_gunzip_core.cuh"
long long cg_gunzip_tiles(long long n_bytes);
cudaError_t cg_launch_gunzip_candidates(int phase, const uint8_t *d_gz, long long n, int32_t *d_counts,
                                        const int64_t *d_offs, int32_t *d_cand, cudaStream_t st);
cudaError_t cg_launch_gunzip_parse(const uint8_t *d_gz, long long n, const int32_t *d_cand, int n_cand, long long budget,
                                   GuMember *d_res, cudaStream_t st);
cudaError_t cg_launch_gunzip_chain(const uint8_t *d_gz, long long n, const int32_t *d_cand, const GuMember *d_res,
                                   int n_cand, int after_member, int final, long long base, long long limit,
                                   int32_t *d_members, long long *d_moff, GuChain *d_chain, long long from, int split,
                                   cudaStream_t st);
// Block path of one member (split streams): the start search of chunks 1..K-1 (warp per chunk); the speculative decode
// of the listed chunks (d_list == nullptr: chunks 0..n_list-1) into d_sym + d_off[k] with d_room[k] symbols; the walk
// (one thread); the windows (d_win: (n_ok + 1) x GU_WIN bytes, the first one the member's window so far) and the
// resolve of the n_ok confirmed chunks into d_out (*d_bad: the first chunk with a marker in front of the member, start
// it at INT_MAX); the raw CRC-32 register *d_state advanced over d_plain[0, len) (d_part: len / cg_gunzip_crc_piece()).
cudaError_t cg_launch_gunzip_search(const uint8_t *d_gz, long long n, long long s0, long long stride, int K, GuChunk *d_ch,
                                    cudaStream_t st);
cudaError_t cg_launch_gunzip_spec(const uint8_t *d_gz, long long n, long long s0, long long stride, int K,
                                  const int32_t *d_list, int n_list, const long long *d_off, const long long *d_room,
                                  uint16_t *d_sym, GuChunk *d_ch, cudaStream_t st);
cudaError_t cg_launch_gunzip_walk(GuChunk *d_ch, int K, long long limit, int32_t *d_redo, GuWalk *d_walk, cudaStream_t st);
cudaError_t cg_launch_gunzip_resolve(const GuChunk *d_ch, int n_ok, long long max_n, const long long *d_off,
                                     const uint16_t *d_sym, uint8_t *d_win, long long mpos, uint8_t *d_out, int *d_bad,
                                     cudaStream_t st);
int cg_gunzip_crc_piece();
cudaError_t cg_launch_gunzip_crc(const uint8_t *d_plain, long long len, uint32_t *d_part, uint32_t *d_state,
                                 cudaStream_t st);
cudaError_t cg_launch_gunzip_place(const uint8_t *d_gz, long long n, const int32_t *d_cand, const int32_t *d_members,
                                   const long long *d_moff, const GuChain *d_chain, int n_members, const GuMember *d_res,
                                   uint8_t *d_out, int *d_bad, cudaStream_t st);
cudaError_t cg_launch_gunzip_flags(const uint8_t *d_buf, long long n, const uint32_t *d_nl, long long n_nl, int fasta,
                                   int32_t *d_flag, cudaStream_t st);
cudaError_t cg_launch_gunzip_select(const uint32_t *d_nl, long long n_nl, const int32_t *d_flag, const int64_t *d_offs,
                                    long long s, long long *d_cut, cudaStream_t st);
// unaligned BAM input (cg_bam.cu, decisions in cg_bam_core.cuh) on the records behind the header, d_buf[0, n): the
// bounds (bitmap d_bm of cg_bam_words(n) words, link words and entries per tile of cg_bam_tiles(n), the chain's end in
// *d_sum, record starts per bitmap word in d_cnt); after an exclusive scan of d_cnt (d_woff) the starts in order and
// their FASTQ sizes (cg_bam_max_records(n) entries, zero behind the last); after an exclusive scan of those (d_foff) the
// cut under `limit` FASTQ bytes; then the refusals of the chain's n_rec records (*d_err: record << 3 | BAM_R_*, start
// it at ~0) and the FASTQ text of the first n_cut of them into d_out.
#include "cg_bam_core.cuh"
long long cg_bam_words(long long n);
long long cg_bam_tiles(long long n);
long long cg_bam_max_records(long long n);
cudaError_t cg_launch_bam_bounds(const uint8_t *d_buf, long long n, uint32_t *d_bm, uint64_t *d_link, long long *d_entry,
                                 BamSum *d_sum, int32_t *d_cnt, cudaStream_t st);
cudaError_t cg_launch_bam_starts(const uint8_t *d_buf, long long n, const uint32_t *d_bm, const long long *d_entry,
                                 const BamSum *d_sum, const int64_t *d_woff, uint32_t *d_start, int32_t *d_fsize,
                                 cudaStream_t st);
cudaError_t cg_launch_bam_cut(const int64_t *d_woff, long long n, const uint32_t *d_start, const int64_t *d_foff,
                              long long limit, BamSum *d_sum, cudaStream_t st);
cudaError_t cg_launch_bam_emit(const uint8_t *d_buf, const uint32_t *d_start, const int64_t *d_foff, long long n_rec,
                               long long n_cut, uint8_t *d_out, unsigned long long *d_err, cudaStream_t st);
// --pair-adapters: fold the records of adapter pair `pair` into the best pair per read (modifiers.py:480-503)
cudaError_t cg_launch_fastq_pair_select(long long n_records, int pair, const cg_match_rec *d_cur1, int slots1,
                                        const cg_match_rec *d_cur2, int slots2, cg_match_rec *d_best1, cg_match_rec *d_best2,
                                        int slots, int32_t *d_best_key, cudaStream_t st);
