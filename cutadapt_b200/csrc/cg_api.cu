// cg_api.cu -- the C ABI (include/cutadapt_b200.h): contexts, adapter sets, batch dispatch.
//
// Host batches are processed as a 2-lane software pipeline: each lane owns a stream, device
// buffers and pinned bounce buffers; consecutive sub-batches alternate lanes so that the H2D
// copy of chunk i+1, the fused kernel of chunk i and the D2H copy of chunk i-1 overlap.
// Caller buffers that are already pinned are copied from/to directly.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <ctype.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/cutadapt_b200.h"
#include "cg_hostpack.h"
#include <array>

#include "cg_gzip_core.cuh"
#include "cg_kernels.cuh"
#include "cg_jit.h"
#include "cg_setbuild.h"

static_assert(sizeof(cg_match) == 32 && sizeof(cg_match_rec) == 32, "cg_match must be 32 bytes");
static_assert(sizeof(CgAdapter) == 80 && sizeof(CgEntry) == 32 && sizeof(CgGroup) == 32 &&
                  sizeof(CgSetHeader) == 80, "table layout");

static thread_local std::string g_err;

static int fail(int code, const std::string &msg)
{
    g_err = msg;
    return code;
}
static int cuda_fail(cudaError_t e, const char *what)
{
    char buf[256];
    snprintf(buf, sizeof buf, "CUDA error in %s: %s", what, cudaGetErrorString(e));
    g_err = buf;
    return e == cudaErrorMemoryAllocation ? CG_ENOMEM : CG_ECUDA;
}
#define CU(x)                                                  \
    do {                                                       \
        cudaError_t _e = (x);                                  \
        if (_e != cudaSuccess) return cuda_fail(_e, #x);       \
    } while (0)

extern "C" int cg_version(void) { return CG_ABI_VERSION; }
extern "C" const char *cg_last_error(void) { return g_err.c_str(); }

// ------------------------------------------------------------------------------------------
// A growing device (DevBuf) or pinned host (PinBuf) buffer.  It owns its memory: freed when the buffer is destroyed or
// assigned to, handed over by moves, never copied.
template <class T, bool Pinned> class GrowBuf {
  public:
    T *p = nullptr;
    size_t cap = 0;
    GrowBuf() = default;
    GrowBuf(const GrowBuf &) = delete;
    GrowBuf &operator=(const GrowBuf &) = delete;
    GrowBuf(GrowBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    GrowBuf &operator=(GrowBuf &&o) noexcept
    {
        if (this != &o) {
            release();
            p = o.p; cap = o.cap;
            o.p = nullptr; o.cap = 0;
        }
        return *this;
    }
    ~GrowBuf() { release(); }
    int ensure(size_t n)
    {
        if (n <= cap) return CG_OK;
        release();
        size_t want = n + n / 4 + 64;
        cudaError_t e = Pinned ? cudaMallocHost((void **)&p, want * sizeof(T)) : cudaMalloc((void **)&p, want * sizeof(T));
        if (e != cudaSuccess) return cuda_fail(e, Pinned ? "cudaMallocHost" : "cudaMalloc");
        cap = want;
        return CG_OK;
    }

  private:
    void release()
    {
        if (p) Pinned ? cudaFreeHost(p) : cudaFree(p);
        p = nullptr; cap = 0;
    }
};
template <class T> using DevBuf = GrowBuf<T, false>;
template <class T> using PinBuf = GrowBuf<T, true>;
static_assert(!std::is_copy_constructible<DevBuf<uint8_t>>::value && !std::is_copy_constructible<PinBuf<uint8_t>>::value,
              "buffers own their memory: move them");

#define CG_N_LANES 3
struct Lane {
    cudaStream_t stream = nullptr;
    DevBuf<uint8_t> d_seq, d_qual, d_pack;
    DevBuf<uint64_t> d_exc;
    PinBuf<uint8_t> h_pack;
    PinBuf<uint64_t> h_exc;
    DevBuf<int64_t> d_offs;
    DevBuf<cg_match_rec> d_out;
    DevBuf<int32_t> d_qtrim;
    PinBuf<uint8_t> h_seq, h_qual;
    PinBuf<int64_t> h_offs;
    PinBuf<cg_match_rec> h_out;
    PinBuf<int32_t> h_qtrim;
    // pending result copy-back (bounce -> caller memory) of the chunk in flight
    bool busy = false;
    cg_match_rec *dst_out = nullptr; size_t n_out = 0; bool out_bounced = false;
    int32_t *dst_qtrim = nullptr; size_t n_qtrim = 0; bool qtrim_bounced = false;
};

// The rows of one kind for a slot's records (cg_fastq_request_rows): the request with its text, the device copy of the
// text, the row sizes and offsets, and the rows (compressed into d_gz when asked), kept until the slot is submitted again
#define CG_ROWS_KINDS 3
struct FqRows {
    bool requested = false;
    bool gzip = false;
    int32_t n_entries = 0;
    std::vector<char> text;
    std::vector<int32_t> text_off;
    int64_t limit = -1;                         // cg_fastq_collect_info / _rows: the caller's row capacity, or -1
    DevBuf<uint8_t> d_text, d_out, d_gz;
    DevBuf<int32_t> d_textoff, d_row;
    DevBuf<int64_t> d_rowoff;
    int64_t bytes = 0, bytes_plain = 0;
};

// One FASTQ chunk in flight (cg_fastq_submit ... cg_fastq_collect)
#define CG_FQ_SLOTS 4
struct FastqSlot {
    cudaStream_t stream = nullptr;
    bool busy = false;
    int64_t n_bytes = 0;
    DevBuf<uint8_t> d_in, d_out, d_seq, d_qual;
    DevBuf<uint32_t> d_tiles, d_nl;
    DevBuf<CgFastqRecord> d_rec;
    DevBuf<int32_t> d_len, d_interval, d_keep, d_outlen, d_qtrim, d_mask, d_adest, d_dmbytes, d_dest, d_pairkey, d_origin;
    DevBuf<uint8_t> d_destkeep;
    FqRows rows[CG_ROWS_KINDS];                 // row requests and their rows
    bool rows_ready = false;                    // the last collect of the slot succeeded: its rows can be read
    DevBuf<int64_t> d_dmbase;
    DevBuf<int64_t> d_offs, d_outoff;
    DevBuf<unsigned long long> d_scan;
    DevBuf<cg_match_rec> d_matches, d_matches_rc;
    DevBuf<uint8_t> d_isrc;
    DevBuf<uint8_t> d_norm;                     // FASTA: the normalised chunk (swapped into d_in once built)
    DevBuf<int32_t> d_faline;                   // FASTA: bytes kept and header flag per line, first header line
    DevBuf<int64_t> d_faoff;                    // FASTA: their exclusive scans
    DevBuf<unsigned long long> d_fqstats;       // statistics on: the chunk's statistics vector (added on success)
    DevBuf<int32_t> d_polya;                    // statistics with --poly-a: bases PolyATrimmer removed, per record
    PinBuf<unsigned long long> h_fqstats;
    DevBuf<int32_t> d_namelen;                  // read names: bytes of every new name (both steps, both mates' counts) ...
    DevBuf<int64_t> d_nameoff;                  // ... their scans: step 1, then step 2
    DevBuf<unsigned long long> d_namemis;       // ... the first pair whose new names no longer name mates
    DevBuf<int32_t> d_fold;                     // interleaved outputs: the sizes the partition runs on
    DevBuf<unsigned long long> d_ilverr;        // interleaved input: first problem of the split, record << 32 | code
    DevBuf<CgGzPiece> d_gzpieces;               // gzip outputs: the pieces of the destinations ...
    DevBuf<uint8_t> d_gzslots, d_gzout;         // ... each compressed into its slot, then packed
    DevBuf<int32_t> d_gzsizes;
    DevBuf<int64_t> d_gzoff;
    // interleaved input (cg_fastq_submit_interleaved): 0 = a chunk of its own, 1 / 2 = mate 1 / 2 of the chunk uploaded to
    // mate 1's slot, split when the pair is collected; ilv_peer = the other mate's slot, ilv_format = input format
    int ilv = 0, ilv_peer = -1, ilv_format = 0;
    DevBuf<unsigned long long> d_counters;      // [0] newline total, [1..] CG_FQ_COUNTERS
    DevBuf<int> d_err;                          // [0] code, [1] record
    PinBuf<uint8_t> h_in, h_out;
    PinBuf<unsigned long long> h_counters;
};

// A gzip input stream (cg_gzin_create): the carry in d_plain[0, carry) and the scratch of the submissions
struct GzinStream {
    DevBuf<uint8_t> d_gz, d_plain;
    PinBuf<uint8_t> h_gz;
    DevBuf<int32_t> d_counts, d_cand, d_members, d_flag;
    DevBuf<int64_t> d_offs;
    DevBuf<GuMember> d_res;
    DevBuf<long long> d_moff;
    DevBuf<unsigned long long> d_scan, d_small;  // d_small: newline total, cut, first bad member, chain
    DevBuf<uint32_t> d_tiles, d_nl;
    cudaEvent_t done = nullptr;                  // the last submission's work on the stream's buffers
    long long carry = 0, consumed = 0, members = 0;
    // the submission in progress, committed once its slots are known: plain bytes behind the carry, bytes and members
    long long pend_plain = 0, pend_consumed = 0, pend_members = 0;
    // CG_GZIN_SPLIT_MEMBERS: a long member is inflated block-parallel and may be consumed in part.  Then the stream
    // keeps the bit offset into the next byte, the running CRC-32 register and plain length, the member's offset in the
    // file, whether only its trailer is left, and its last GU_WIN plain bytes (d_win); the p* copies are pending.
    bool split = false;
    long long stride = CG_GZIN_STRIDE;
    struct Member { int in = 0, bitoff = 0, trailer = 0; uint32_t crc = 0; long long len = 0, start = 0; } mem, pmem;
    long long pend_respec = 0;
    DevBuf<uint8_t> d_win, d_pwin, d_wins;
    DevBuf<GuChunk> d_ch;
    DevBuf<long long> d_coff, d_room;
    DevBuf<uint16_t> d_sym;
    DevBuf<int32_t> d_redo;
    DevBuf<uint32_t> d_part;
    // the format of the stream's first committed submission: -1 none yet, 0 FASTQ / FASTA, 1 CG_FORMAT_BAM
    int bam = -1;
    // CG_FORMAT_BAM: whether the header was read and dropped; the offset of d_plain[0] in the decompressed stream and the
    // records cut so far (for the messages); the tiles of the boundary walk and those walked again, over the stream's life
    bool bam_hdr = false;
    long long bam_base = 0, bam_records = 0, bam_tiles = 0, bam_rewalked = 0;
    DevBuf<uint32_t> d_bm, d_start;
    DevBuf<uint64_t> d_link;
    DevBuf<long long> d_entry;
    DevBuf<int32_t> d_wcnt, d_fsize;
    DevBuf<int64_t> d_woff, d_foff;
    DevBuf<BamSum> d_sum;
    DevBuf<unsigned long long> d_berr;
    DevBuf<uint8_t> d_rest;
    ~GzinStream() { if (done) cudaEventDestroy(done); }   // not copyable, as its buffers are not
};

// A statistics accumulator of the FASTQ path (cg_fastq_stats_create): the vector of cg_fastq_stats_read at
// (n_adapters, max_len, kmax); both sizes grow when a chunk needs more.
struct FqStatsAcc {
    int32_t n_adapters = 0, max_len = 0, kmax = 0;
    std::vector<int64_t> v;
};

// A names handle (cg_names_create): the parts of the program, and its blob (CgNameProg + pool) built from them once
// the mates' adapter names are set, on the host and on the device
struct NamesProg {
    CgNameSpec spec;
    std::vector<uint8_t> blob;
    DevBuf<uint8_t> d_blob;
    bool uploaded = false;
};

struct cg_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 148;
    size_t smem_optin = 0;
    Lane lanes[CG_N_LANES];
    int *d_err = nullptr;       // [0] non-ASCII flag, [1] max_len scratch
    uint8_t *d_enc = nullptr;   // 768 bytes
    double *d_phred = nullptr;  // 256 doubles: 10^(-q/10)
    DevBuf<uint32_t> scratch_p;
    DevBuf<int> scratch_w;
    DevBuf<unsigned long long> d_stats;  // cg_process_batch_stats: the statistics vector of the batch in flight
    DevBuf<uint4> tasks;                 // split pipeline: 2 x uint4 per read of a sub-batch
    DevBuf<uint4> tasks2, tasks3;        // run-record lists (ping-pong): 4 x uint4 per read of a sub-batch
    DevBuf<uint2> stat_ents;             // fused statistics: one entry per read the plan and run kernels finish
    unsigned long long *d_task_count = nullptr;
    DevBuf<cg_match_rec> pass_tmp;       // multi-pass schedule: records of every pass for one sub-batch
    DevBuf<int32_t> view_base, view_back;
    long long launches = 0;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> timing;   // fused-kernel event pairs
    std::vector<cudaEvent_t> event_pool;
    double timed_ms = 0.0;
    long long timed_n = 0;
    // per-stage event timing of the split pipeline (CUTADAPT_B200_STAGE_TIMES=1; cg_ctx_stage_times)
    std::vector<std::array<cudaEvent_t, 4>> stage_events;
    double stage_ms[3] = {0, 0, 0};
    // host side of cg_process_batch
    CgHostPool *pool = nullptr;
    std::vector<std::vector<uint64_t>> exc_scratch;
    long long h2d_bytes = 0, d2h_bytes = 0;
    double prof[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // cg_ctx_host_profile
    double pack_fraction = 0.6;                  // share of a chunk that travels compressed (adapted)
    // hill climbing on the measured chunk rate (cg_process_batch): the share that gave the best rate so far, that
    // rate, the direction of the next probe, and whether the reference rate has to be measured again
    double pack_ref_fraction = 0.6, pack_ref_rate = 0.0;
    int pack_dir = +1;
    bool pack_have_ref = false;
    int numa_node = -1;                          // node the worker pool was bound to, or -1
    // ordering of the trimming passes of different lanes over the shared scratch
    cudaEvent_t scratch_ev = nullptr;
    cudaStream_t scratch_stream = nullptr;
    bool scratch_busy = false;
    FastqSlot fq[CG_FQ_SLOTS];
    int fq_next = 0;
    std::map<int32_t, FqStatsAcc> fq_stats;      // cg_fastq_stats_* by handle
    int32_t fq_stats_next = 1;
    std::map<int32_t, GzinStream> gzin;          // cg_gzin_* by handle
    std::map<int32_t, NamesProg> names;          // cg_names_* by handle
    int32_t names_next = 1;
    int32_t gzin_next = 1;
};

struct cg_adapterset {
    cg_ctx *ctx = nullptr;
    CgBuiltSet host;
    uint8_t *d_blob = nullptr;
    uint64_t *d_masks = nullptr;
    CgEntry *d_entries = nullptr;   // device pointer into d_blob
    uint8_t *d_index = nullptr;     // anchored-adapter hash tables, or null
    // multi-pass schedule (several groups, times == 1): one sub-set per component adapter
    struct Pass {
        cg_adapterset *sub = nullptr;
        int group = 0, role = 0;    // role 1: back adapter of a LINKED group
        int front_pass = -1;        // role 1: the pass of the front adapter
        int map_off = 0;            // first entry in pass_map (local -> global adapter numbers)
    };
    std::vector<Pass> passes;
    std::vector<int32_t> pass_map;
    int32_t *d_pass_map = nullptr;
    CgSelectTables select_tables;
    // run-time specialisation of the bit-plane first stage (cg_jit.h): one kernel per (plane words, qualities,
    // statistics counted in the stage or not)
    mutable CgJitKernel *jit[2][2][2] = {};
    mutable int jit_state[2][2][2] = {};                // 0 not tried, 1 ready, -1 failed
    mutable long long plane_reads = 0;                  // reads that went through the plane stage so far
    mutable std::string jit_error;
};

// ------------------------------------------------------------------------------------------
extern "C" int cg_ctx_create(int device, void *stream, cg_ctx **out)
{
    if (!out) return fail(CG_EINVAL, "cg_ctx_create: out is NULL");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(CG_ECUDA, std::string("no usable CUDA device (") + cudaGetErrorString(e) +
                                  "); cutadapt_b200 has no CPU fallback");
    if (device < 0 || device >= count) return fail(CG_EINVAL, "cg_ctx_create: device ordinal out of range");
    CU(cudaSetDevice(device));
    // until it is complete, a failed step destroys what has been built
    std::unique_ptr<cg_ctx, decltype(&cg_ctx_destroy)> c(new cg_ctx(), cg_ctx_destroy);
    c->device = device;
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    c->sm_count = prop.multiProcessorCount;
    c->smem_optin = prop.sharedMemPerBlockOptin;
    if (stream) { c->stream = (cudaStream_t)stream; c->own_stream = false; }
    else { CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)); c->own_stream = true; }
    for (int i = 0; i < CG_N_LANES; ++i) CU(cudaStreamCreateWithFlags(&c->lanes[i].stream, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&c->scratch_ev, cudaEventDisableTiming));
    CU(cudaMalloc((void **)&c->d_err, 16 * sizeof(int)));
    CU(cudaMemset(c->d_err, 0, 16 * sizeof(int)));
    CU(cudaMalloc((void **)&c->d_task_count, 64));
    CU(cudaMemset(c->d_task_count, 0, 64));
    CU(cudaMalloc((void **)&c->d_enc, 768));
    uint8_t enc[768];
    cg_build_enc_tables(enc);
    CU(cudaMemcpy(c->d_enc, enc, 768, cudaMemcpyHostToDevice));
    {
        double phred[256];
        cg_build_phred_table(phred);
        CU(cudaMalloc((void **)&c->d_phred, sizeof phred));
        CU(cudaMemcpy(c->d_phred, phred, sizeof phred, cudaMemcpyHostToDevice));
    }
    *out = c.release();
    return CG_OK;
}

static void resolve_timing(cg_ctx *c)
{
    for (auto &pr : c->timing) {
        float ms = 0.f;
        if (cudaEventSynchronize(pr.second) == cudaSuccess && cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) {
            c->timed_ms += ms; c->timed_n += 1;
        }
        c->event_pool.push_back(pr.first);
        c->event_pool.push_back(pr.second);
    }
    c->timing.clear();
}

extern "C" int cg_ctx_destroy(cg_ctx *c)
{
    if (!c) return CG_OK;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    resolve_timing(c);
    for (auto ev : c->event_pool) cudaEventDestroy(ev);
    delete c->pool;
    c->pool = nullptr;
    for (Lane &l : c->lanes)
        if (l.stream) cudaStreamDestroy(l.stream);
    for (FastqSlot &f : c->fq)
        if (f.stream) cudaStreamDestroy(f.stream);
    if (c->scratch_ev) cudaEventDestroy(c->scratch_ev);
    if (c->d_task_count) cudaFree(c->d_task_count);
    if (c->d_err) cudaFree(c->d_err);
    if (c->d_enc) cudaFree(c->d_enc);
    if (c->d_phred) cudaFree(c->d_phred);
    if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
    delete c;                                   // the buffers and the gzip input streams free themselves
    return CG_OK;
}

extern "C" int cg_ctx_synchronize(cg_ctx *c)
{
    if (!c) return fail(CG_EINVAL, "ctx is NULL");
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));
    for (int i = 0; i < CG_N_LANES; ++i) CU(cudaStreamSynchronize(c->lanes[i].stream));
    return CG_OK;
}

extern "C" int64_t cg_ctx_launch_count(cg_ctx *c) { return c ? c->launches : 0; }

// Device time of the three stages of the split pipeline (first stage, plan, DP rounds) since the last reset, in ms;
// only recorded while CUTADAPT_B200_STAGE_TIMES is set in the environment (tools).
extern "C" int cg_ctx_stage_times(cg_ctx *c, double *out3, int reset)
{
    if (!c || !out3) return fail(CG_EINVAL, "cg_ctx_stage_times: NULL argument");
    CU(cudaSetDevice(c->device));
    for (auto &e : c->stage_events) {
        CU(cudaEventSynchronize(e[3]));
        for (int i = 0; i < 3; ++i) {
            float ms = 0;
            CU(cudaEventElapsedTime(&ms, e[i], e[i + 1]));
            c->stage_ms[i] += ms;
        }
        for (auto ev : e) cudaEventDestroy(ev);
    }
    c->stage_events.clear();
    for (int i = 0; i < 3; ++i) out3[i] = c->stage_ms[i];
    if (reset) c->stage_ms[0] = c->stage_ms[1] = c->stage_ms[2] = 0;
    return CG_OK;
}

extern "C" int cg_ctx_kernel_time(cg_ctx *c, double *total_ms, int64_t *launches, int reset)
{
    if (!c) return fail(CG_EINVAL, "ctx is NULL");
    CU(cudaSetDevice(c->device));
    resolve_timing(c);
    if (total_ms) *total_ms = c->timed_ms;
    if (launches) *launches = c->timed_n;
    if (reset) { c->timed_ms = 0.0; c->timed_n = 0; }
    return CG_OK;
}

// ------------------------------------------------------------------------------------------
static void destroy_passes(cg_adapterset *s)
{
    for (auto &p : s->passes) cg_adapterset_destroy(p.sub);
    s->passes.clear();
    s->pass_map.clear();
    if (s->d_pass_map) { cudaFree(s->d_pass_map); s->d_pass_map = nullptr; }
}

// Copies the compiled tables of s->host to the device.
static int upload_set(cg_ctx *c, cg_adapterset *s)
{
    s->ctx = c;
    cudaError_t e = cudaSetDevice(c->device);
    if (e == cudaSuccess) e = cudaMalloc((void **)&s->d_blob, s->host.blob.size());
    if (e == cudaSuccess) e = cudaMemcpy(s->d_blob, s->host.blob.data(), s->host.blob.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc((void **)&s->d_masks, s->host.masks64.size() * 8);
    if (e == cudaSuccess) e = cudaMemcpy(s->d_masks, s->host.masks64.data(), s->host.masks64.size() * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && !s->host.index_blob.empty()) {
        e = cudaMalloc((void **)&s->d_index, s->host.index_blob.size());
        if (e == cudaSuccess) e = cudaMemcpy(s->d_index, s->host.index_blob.data(), s->host.index_blob.size(), cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) {
        if (s->d_blob) cudaFree(s->d_blob);
        if (s->d_masks) cudaFree(s->d_masks);
        if (s->d_index) cudaFree(s->d_index);
        s->d_blob = nullptr; s->d_masks = nullptr; s->d_index = nullptr;
        return cuda_fail(e, "adapter set upload");
    }
    return CG_OK;
}

extern "C" int cg_adapterset_create_indexed(cg_ctx *c, const cg_adapter_desc *adapters, int32_t n_adapters,
                                            const cg_group_desc *groups, int32_t n_groups,
                                            const cg_index_desc *indexes, int32_t n_indexes, cg_adapterset **out)
{
    if (!c || !out) return fail(CG_EINVAL, "cg_adapterset_create: NULL argument");
    cg_adapterset *s = new cg_adapterset();
    std::string err;
    int rc = cg_build_set(adapters, n_adapters, groups, n_groups, s->host, err, indexes, n_indexes);
    if (rc != CG_OK) { delete s; return fail(rc, err); }
    rc = upload_set(c, s);
    if (rc != CG_OK) { delete s; return rc; }
    // multi-pass schedule (cg_setbuild.cpp: cg_plan_passes); an empty plan keeps the one-kernel schedule
    CgMultiPlan plan;
    if (cg_plan_passes(adapters, n_adapters, groups, n_groups, indexes, n_indexes, plan, err) == CG_OK &&
        !plan.passes.empty()) {
        bool ok = true;
        for (auto &pp : plan.passes) {
            cg_adapterset::Pass P;
            P.group = pp.group; P.role = pp.role; P.front_pass = pp.front_pass; P.map_off = pp.map_off;
            P.sub = new cg_adapterset();
            P.sub->host = std::move(pp.set);
            if (upload_set(c, P.sub) != CG_OK) { delete P.sub; ok = false; break; }
            s->passes.push_back(P);
        }
        if (ok) {
            const CgSetHeader *H = (const CgSetHeader *)s->host.blob.data();
            cg_fill_select_tables((const CgGroup *)(s->host.blob.data() + H->groups_off), s->host.n_groups,
                                  s->host.slots, plan.passes, s->select_tables);
            s->pass_map = plan.pass_map;
            cudaError_t e = cudaMalloc((void **)&s->d_pass_map, s->pass_map.size() * sizeof(int32_t));
            if (e == cudaSuccess)
                e = cudaMemcpy(s->d_pass_map, s->pass_map.data(), s->pass_map.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
            if (e != cudaSuccess) { cudaGetLastError(); ok = false; }
        }
        if (!ok) destroy_passes(s);
    }
    *out = s;
    return CG_OK;
}

extern "C" int cg_adapterset_create(cg_ctx *c, const cg_adapter_desc *adapters, int32_t n_adapters,
                                    const cg_group_desc *groups, int32_t n_groups, cg_adapterset **out)
{
    return cg_adapterset_create_indexed(c, adapters, n_adapters, groups, n_groups, nullptr, 0, out);
}

extern "C" int cg_adapterset_destroy(cg_adapterset *s)
{
    if (!s) return CG_OK;
    if (s->ctx) cudaSetDevice(s->ctx->device);
    if (s->d_blob) cudaFree(s->d_blob);
    if (s->d_masks) cudaFree(s->d_masks);
    if (s->d_index) cudaFree(s->d_index);
    for (int w = 0; w < 2; ++w)
        for (int q = 0; q < 2; ++q)
            for (int v = 0; v < 2; ++v) cg_jit_destroy(s->jit[w][q][v]);
    destroy_passes(s);
    delete s;
    return CG_OK;
}

// Run-time specialisation of the first stage (cg_jit.h): 1 = a specialised kernel is in use, 0 = not (yet),
// -1 = compilation failed (the precompiled kernel runs; cg_last_error() holds the reason after this call).
extern "C" int cg_adapterset_jit_status(const cg_adapterset *s)
{
    if (!s) return 0;
    const cg_adapterset *t = (!s->passes.empty() && s->passes[0].sub) ? s->passes[0].sub : s;
    int st = 0;
    for (int w = 0; w < 2; ++w)
        for (int q = 0; q < 2; ++q)
            for (int v = 0; v < 2; ++v) {
                if (t->jit_state[w][q][v] == 1) st = 1;
                else if (t->jit_state[w][q][v] == -1 && st == 0) st = -1;
            }
    if (st == -1) g_err = "first-stage specialisation failed: " + t->jit_error;
    return st;
}

// The translation unit cg_jit.cpp would compile for this set (plane_words 5 or 8; stats: the variant that counts the
// trim statistics); returns its length (0: the set has no plane program) and copies at most cap - 1 characters.
extern "C" int64_t cg_adapterset_jit_source(const cg_adapterset *s, int32_t plane_words, int32_t has_qual, int32_t stats,
                                            char *buf, int64_t cap)
{
    if (!s) return 0;
    const std::string src = cg_jit_pscan_source(s->host, plane_words, has_qual != 0, stats != 0);
    if (buf && cap > 0) {
        const size_t n = std::min<size_t>(src.size(), (size_t)cap - 1);
        memcpy(buf, src.data(), n);
        buf[n] = 0;
    }
    return (int64_t)src.size();
}

extern "C" int cg_adapterset_slots(const cg_adapterset *s) { return s ? s->host.slots : 0; }

extern "C" int cg_adapterset_effective_length(const cg_adapterset *s, int32_t adapter, int32_t *out)
{
    if (!s || !out || adapter < 0 || adapter >= s->host.n_adapters) return fail(CG_EINVAL, "bad adapter index");
    *out = s->host.effective_length[adapter];
    return CG_OK;
}

// ------------------------------------------------------------------------------------------
// Launch of the trimming pass on device-resident data
// ------------------------------------------------------------------------------------------
// The environment switches of the trimming pass (kernel choices of the parity tests, measured experiments), read when
// a TrimSwitches is made: once per launch_trim call, not per context, since tests change them between calls.
struct TrimSwitches {
    static bool is(const char *name, const char *value) { const char *e = getenv(name); return e && strcmp(e, value) == 0; }
    static long long at_least_1024(const char *e) { const long long v = e ? atoll(e) : 0; return v >= 1024 ? v : 0; }
    bool force_general = is("CUTADAPT_B200_KERNEL", "general");
    bool force_block = is("CUTADAPT_B200_KERNEL", "block");
    bool force_warp = is("CUTADAPT_B200_KERNEL", "warp");
    bool shiftand = is("CUTADAPT_B200_SCAN", "shiftand");
    bool no_band = getenv("CUTADAPT_B200_NO_BAND") != nullptr;
    bool no_light = getenv("CUTADAPT_B200_NO_LIGHT") != nullptr;
    bool no_index_kernel = getenv("CUTADAPT_B200_NO_INDEX_KERNEL") != nullptr;
    bool two_lists = getenv("CUTADAPT_B200_TWO_LISTS") != nullptr;
    bool task_bytes = getenv("CUTADAPT_B200_TASK_BYTES") != nullptr;
    bool no_band_lists = getenv("CUTADAPT_B200_NO_BAND_LISTS") != nullptr;
    bool stage_times = getenv("CUTADAPT_B200_STAGE_TIMES") != nullptr;
    bool jit_never = is("CUTADAPT_B200_JIT", "0"), jit_always = is("CUTADAPT_B200_JIT", "1");
    long long sub_reads = at_least_1024(getenv("CUTADAPT_B200_SUB_READS"));   // 0: the schedule's default
};

// Statistics wanted together with a trimming pass (cg_stats_*), added to d_stats.
struct StatsRequest { unsigned long long *d_stats; int max_len, kmax; };

enum class TrimKind { Index, Light, Split, Warp, Fast, Generic, MultiPass };

// What choose_schedule decided for one call, and what the launcher of that schedule needs.
struct TrimSchedule {
    TrimKind kind = TrimKind::Generic;
    int tile_cap = 0, mini_cap = 0, carry_slot = 0;   // CgKernelArgs geometry
    size_t smem = 0;                // the first kernel (fast, warp, or the split pipeline's first stage)
    int occ = 0;                    // and its CTAs per SM
    bool simple = false;            // fast: the SIMPLE variant
    size_t list_smem = 0;           // split: the plan and run kernels
    int plan_occ = 0, run_occ = 0;
    int plane_w = 0, plane_rec = 0; // split: plane words of the first stage (0: shift-and scan), uint4 words per task
    long long sub = 0;              // reads per sub-batch (index, split, multi-pass)
    CgJitKernel *jit = nullptr;     // split: the specialised first stage, or null
    int jit_occ = 0;
    bool fuse_stats = false;        // split: the pass counts the statistics of its reads
};

// Decides how one call trims.  has_view: the call is a pass of the multi-pass schedule.  Besides deciding, it counts
// the reads of the set's plane stage and builds the specialised first stage once.
static int choose_schedule(cg_ctx *c, const cg_adapterset *s, int64_t n_reads, int max_read_len, const cg_params *p,
                           bool has_view, const StatsRequest *stats, const TrimSwitches &sw, TrimSchedule &d)
{
    const CgBuiltSet &h = s->host;
    const int times = p->times < 1 ? 1 : p->times;
    const bool want_q = p->quality_trim != 0 || p->nextseq_trim != 0;
    // several groups, one round: per-adapter passes + selection (CUTADAPT_B200_KERNEL=general: the one-phase kernel)
    if (!s->passes.empty() && times == 1 && !sw.force_general) {
        d.kind = TrimKind::MultiPass;
        d.sub = sw.sub_reads ? sw.sub_reads : 32LL << 20;
        return CG_OK;
    }
    // sets of index lookups only (demultiplexing), no quality trimming: the light kernel -- nothing to stage; for one
    // round without views the lookups alone (cg_index_kernel), in sub-batches so that 32-bit read numbers and one list
    // suffice
    if (h.all_indexed && !want_q && !h.any_wide && h.max_m + 1 <= CG_LIGHT_ROWS && !sw.force_general && !sw.no_light) {
        d.kind = times == 1 && !has_view && h.slots == 1 && !sw.no_index_kernel ? TrimKind::Index : TrimKind::Light;
        d.sub = 64LL << 20;
        return CG_OK;
    }
    const uint32_t blob_bytes = (uint32_t)h.blob.size();
    const long long tile_cap = ((long long)CG_NT * max_read_len + 32 + 15) / 16 * 16;
    bool fast = !h.any_wide && max_read_len <= CG_PACKED_MAX_N && tile_cap < (1 << 24);
    if (fast) {
        d.tile_cap = (int)tile_cap;
        d.smem = cg_fast_smem_bytes(blob_bytes, d.tile_cap, h.max_m + 1, want_q);
        fast = d.smem <= c->smem_optin;
    }
    // two-phase schedule when the set is one aligner adapter and a single round is asked for;
    // CUTADAPT_B200_KERNEL=general forces the one-phase kernel (used by the parity tests)
    d.simple = fast && h.simple_ok && times == 1 && !sw.force_general;
    if (fast) {
        CU(cg_fast_occupancy(want_q, d.simple, d.smem, &d.occ));
        fast = d.occ >= 1;
    }
    d.kind = fast ? TrimKind::Fast : TrimKind::Generic;
    const long long mini = ((long long)32 * max_read_len + 32 + 15) / 16 * 16;
    // warp-autonomous fused kernel (kept selectable: CUTADAPT_B200_KERNEL=warp)
    if (d.simple && h.max_m <= 32 && sw.force_warp && mini < (1 << 20)) {
        d.mini_cap = (int)mini;
        d.carry_slot = (int)(((long long)max_read_len + 4 + 15) / 16 * 16 + 16);   // + 4: word-granular reads past the last group
        const size_t wsmem = cg_warp_smem_bytes(blob_bytes, d.mini_cap, d.carry_slot, want_q);
        int wocc = 0;
        if (wsmem <= c->smem_optin) CU(cg_warp_occupancy(want_q, wsmem, &wocc));
        if (wocc >= 1) { d.kind = TrimKind::Warp; d.smem = wsmem; d.occ = wocc; }
        return CG_OK;
    }
    // split pipeline (default for one aligner adapter with m <= 64): scan kernel -> task list -> DP kernel
    if (!d.simple || h.max_m > 64 || sw.force_block || sw.force_warp || mini >= (1 << 20)) return CG_OK;
    // bit-plane first stage (plane_scan_core) when the adapter has a plane program and the reads fit 8 plane
    // words; CUTADAPT_B200_SCAN=shiftand keeps the shift-and scan kernel (parity tests run both)
    const CgSetHeader *hdr = (const CgSetHeader *)h.blob.data();
    if (hdr->plane_count > 0 && max_read_len <= 256 && !sw.shiftand) d.plane_w = max_read_len <= 160 ? 5 : 8;
    const long long cslot = ((long long)max_read_len + 4 + 15) / 16 * 16 + 32;   // + 4: word-granular reads past the last group
    d.mini_cap = (int)mini;
    d.carry_slot = (int)(d.plane_w ? std::max<long long>(cslot, 16LL * (2 * d.plane_w + 1) + 16) : cslot);   // the window bytes a plane task carries
    size_t scan_smem = d.plane_w ? cg_pscan_smem_bytes(blob_bytes, d.mini_cap, want_q)
                                 : cg_scan_smem_bytes(blob_bytes, d.mini_cap, want_q);
    d.list_smem = cg_dp_smem_bytes(blob_bytes, d.carry_slot);
    if (scan_smem > c->smem_optin || d.list_smem > c->smem_optin) return CG_OK;
    int scan_occ = 0;
    if (d.plane_w) CU(cg_pscan_occupancy(want_q, d.plane_w, false, scan_smem, &scan_occ));
    else CU(cg_scan_occupancy(want_q, scan_smem, &scan_occ));
    CU(cg_list_occupancy(true, h.max_m, false, d.list_smem, &d.plan_occ));
    CU(cg_list_occupancy(false, h.max_m, false, d.list_smem, &d.run_occ));
    if (scan_occ < 1 || d.plan_occ < 1 || d.run_occ < 1) return CG_OK;
    // statistics counted inside the pass: one plain adapter, one round, the whole set in this call (not a pass of the
    // multi-pass schedule), no quality trimming, and the first stage keeps its CTAs per SM with the histogram in shared
    // memory.  The first stage counts the reads it settles (88 % on the benchmark's reads) while they are in shared
    // memory; the plan and run kernels list an entry for each of the others where they write its final record, and one
    // cg_stats_entries_kernel launch per sub-batch counts them (its histograms must fit 48 KiB of shared memory).
    // Otherwise launch_trim_with_stats runs cg_stats_kernel over all records after the pass.
    // Measured on an H100 (DESIGN.md section 4.1): with quality trimming (config 4) the first stage grew by more than
    // the statistics kernel costs, so quality-trimmed passes keep the kernel.
    if (d.plane_w && stats && !has_view && h.n_adapters == 1 && times == 1 && h.slots == 1 && !want_q && !sw.two_lists &&
        stats->max_len <= 4096 && cg_stats_entries_smem_bytes(stats->max_len, stats->kmax) <= 48 * 1024) {
        const size_t fsmem = cg_pscan_smem_bytes(blob_bytes, d.mini_cap, want_q, stats->max_len);
        int focc = 0;
        if (fsmem <= c->smem_optin) CU(cg_pscan_occupancy(want_q, d.plane_w, true, fsmem, &focc));
        // (the listing variants of the plan and run kernels: same shared memory, the attribute set for them too)
        int pocc = 0, rocc = 0;
        CU(cg_list_occupancy(true, h.max_m, true, d.list_smem, &pocc));
        CU(cg_list_occupancy(false, h.max_m, true, d.list_smem, &rocc));
        d.fuse_stats = focc >= 1 && focc >= scan_occ && pocc >= d.plan_occ && rocc >= d.run_occ;
        if (d.fuse_stats) { scan_smem = fsmem; scan_occ = focc; }
    }
    // Run-time specialisation of the first stage for this adapter set (cg_jit.h): compiled once the set has seen
    // enough reads to pay for the ~1 s of NVRTC (CUTADAPT_B200_JIT=1: at once, =0: never), one kernel per variant
    // (with or without the statistics); any failure keeps the precompiled interpreter kernel.
    if (d.plane_w) {
        const int wi = d.plane_w <= 5 ? 0 : 1, qi = want_q ? 1 : 0, vi = d.fuse_stats ? 1 : 0;
        s->plane_reads += n_reads;
        if (!sw.jit_never && s->jit_state[wi][qi][vi] == 0 && (sw.jit_always || s->plane_reads >= (4LL << 20))) {
            std::string err;
            s->jit[wi][qi][vi] = cg_jit_build_pscan(h, d.plane_w, want_q, d.fuse_stats, err);
            s->jit_state[wi][qi][vi] = s->jit[wi][qi][vi] ? 1 : -1;
            if (!s->jit[wi][qi][vi]) s->jit_error = err;
        }
        if (!sw.jit_never && s->jit_state[wi][qi][vi] == 1) {
            d.jit_occ = cg_jit_occupancy(s->jit[wi][qi][vi], CG_NT, scan_smem);
            if (d.jit_occ >= 1) d.jit = s->jit[wi][qi][vi];
        }
    }
    d.kind = TrimKind::Split;
    d.smem = scan_smem; d.occ = scan_occ;
    // reads per sub-batch: bounds the lists to 1 + 2 x 2 GiB at the default 32 Mi (measured: fewer,
    // larger sub-batches amortise the kernel tails and the small late DP rounds; 32 Mi vs 4 Mi = +15 % on the 100 M-read bench).
    // CUTADAPT_B200_SUB_READS overrides it for experiments.
    d.sub = sw.sub_reads ? sw.sub_reads : (d.plane_w && sw.task_bytes) ? (16LL << 20) : (32LL << 20);   // (tasks with bytes: 240 B each)
    d.sub = std::min<long long>(d.sub, 1LL << 31);     // tasks name their read with 32 bits
    // header (4 words) and, with CUTADAPT_B200_TASK_BYTES=1, the window bytes (cg_pscan.cuh).  Carrying the bytes
    // turns the plan stage's gather into a stream but was measured neutral (plan 2.55 -> 2.65 ms, first stage
    // 4.44 -> 4.64 ms per 100 M reads): the plan stage is bound by its dependent shared-memory chains, not by HBM.
    d.plane_rec = d.plane_w ? (sw.task_bytes ? 4 + 2 * d.plane_w + 1 : 4) : 2;
    return CG_OK;
}

// CTAs of a launch: `need`, at most blocks_per_sm per SM, at least one
static int trim_grid(const cg_ctx *c, int blocks_per_sm, long long need)
{
    return (int)std::max<long long>(1, std::min<long long>((long long)blocks_per_sm * c->sm_count, need));
}

static int launch_index(cg_ctx *c, const CgKernelArgs &a, const TrimSchedule &d, cudaStream_t st)
{
    int rc = c->tasks.ensure((size_t)((std::min<long long>(a.n_reads, d.sub) + 3) / 4));
    if (rc != CG_OK) return rc;
    for (long long r0 = 0; r0 < a.n_reads; r0 += d.sub) {
        const long long n_sub = std::min<long long>(d.sub, a.n_reads - r0);
        CgKernelArgs b = a;
        b.offsets = a.offsets + r0; b.n_reads = n_sub; b.out = a.out + (size_t)r0 * a.slots;
        b.tasks = c->tasks.p; b.task_count = c->d_task_count;
        CU(cudaMemsetAsync(c->d_task_count, 0, sizeof(unsigned long long), st));
        CU(cg_launch_index(b, trim_grid(c, 16, (n_sub + CG_NT - 1) / CG_NT), st));
        c->launches += 2;     // cg_index_kernel and cg_trim_listed_kernel
    }
    return CG_OK;
}

// scan -> plan -> up to four DP rounds (one run of every unfinished read per round), per sub-batch
static int launch_split(cg_ctx *c, const cg_adapterset *s, const CgKernelArgs &a, const TrimSchedule &d,
                        const TrimSwitches &sw, cudaStream_t st)
{
    const long long cap = std::min<long long>(a.n_reads, d.sub);
    int rc = c->tasks.ensure((size_t)cap * d.plane_rec);
    if (rc == CG_OK) rc = c->tasks2.ensure((size_t)cap * 4);
    if (rc == CG_OK) rc = c->tasks3.ensure((size_t)cap * 4);
    if (rc == CG_OK && d.fuse_stats) rc = c->stat_ents.ensure((size_t)cap);
    if (rc != CG_OK) return rc;
    unsigned long long *cnt = c->d_task_count;
    for (long long r0 = 0; r0 < a.n_reads; r0 += d.sub) {
        const long long n_sub = std::min<long long>(d.sub, a.n_reads - r0);
        CgKernelArgs b = a;
        b.offsets = a.offsets + r0;
        b.n_reads = n_sub;
        b.out = a.out + (size_t)r0 * a.times * a.slots;
        b.qtrim = a.qtrim ? a.qtrim + 2 * r0 : nullptr;
        b.view = a.view ? a.view + 2 * r0 : nullptr;
        b.task_cap = n_sub;
        CU(cudaMemsetAsync(cnt, 0, 8 * sizeof(unsigned long long), st));
        const long long need = ((n_sub + 31) / 32 + 3) / 4;
        std::array<cudaEvent_t, 4> sev = {nullptr, nullptr, nullptr, nullptr};
        if (sw.stage_times && c->stage_events.size() < 4096) {
            for (auto &e : sev) CU(cudaEventCreate(&e));
            CU(cudaEventRecord(sev[0], st));
        }
        b.tasks = c->tasks.p; b.task_count = cnt;
        b.task_rec = d.plane_rec;
        // (two input lists for the plan stage -- reads with / without locator hits -- were measured: the first
        //  stage got 2.3x slower and the plan stage no faster, it is bound by its memory traffic; kept as an
        //  experiment: CUTADAPT_B200_TWO_LISTS=1)
        b.task_count_b = (d.plane_w && sw.two_lists) ? cnt + 4 : nullptr;
        if (d.plane_w && d.jit) {
            const int rcj = cg_jit_launch(d.jit, trim_grid(c, d.jit_occ, need), CG_NT, d.smem, (void *)st, &b);
            if (rcj != 0) return fail(CG_ECUDA, "launch of the specialised first stage failed (CUresult " + std::to_string(rcj) + ")");
        }
        else if (d.plane_w) CU(cg_launch_pscan(b, a.quality_trim != 0, d.plane_w, trim_grid(c, d.occ, need), d.smem, st));
        else CU(cg_launch_scan(b, a.quality_trim != 0, trim_grid(c, d.occ, need), d.smem, st));
        if (sev[0]) CU(cudaEventRecord(sev[1], st));
        b.stat_ents = c->stat_ents.p; b.stat_count = cnt + 6;
        b.tasks2 = c->tasks2.p; b.task2_count = cnt + 1;
        b.tasks3 = c->tasks3.p; b.task3_count = cnt + 2;
        // run records of the plane path go to two lists (banded first runs / the others): cnt[5] counts the second
        // (only with the band compiled in, CG_RUN_BAND)
        b.task2_count_b = (CG_RUN_BAND && d.plane_w && !sw.no_band_lists) ? cnt + 5 : nullptr;
        CU(cg_launch_list(b, true, s->host.max_m, trim_grid(c, d.plan_occ, need), d.list_smem, st));
        c->launches += 2;
        if (d.plane_w) {
            // second plan launch: the reads the first one set aside (windows with other letters than A/C/G/T),
            // scanned exactly on dense warps; its run records continue the same list
            CgKernelArgs b2 = b;
            b2.tasks = c->tasks3.p; b2.task_count = cnt + 2; b2.task_rec = 2;
            b2.tasks3 = nullptr; b2.task3_count = cnt + 3; b2.task_count_b = nullptr;
            CU(cg_launch_list(b2, true, s->host.max_m, trim_grid(c, d.plan_occ, need), d.list_smem, st));
            CU(cudaMemsetAsync(cnt + 2, 0, sizeof(unsigned long long), st));
            c->launches += 1;
        }
        if (sev[0]) CU(cudaEventRecord(sev[2], st));
        uint4 *lists[2] = {c->tasks2.p, c->tasks3.p};
        for (int round = 0; round < 4; ++round) {
            const int in = round & 1, outl = in ^ 1;
            if (round > 0) CU(cudaMemsetAsync(cnt + 1 + outl, 0, sizeof(unsigned long long), st));
            b.tasks = lists[in]; b.task_count = cnt + 1 + in;
            b.task_count_b = round == 0 ? b.task2_count_b : nullptr;     // the plan stage's second list
            b.tasks2 = lists[outl]; b.task2_count = cnt + 1 + outl;
            if (round == 0) b.task2_count_b = nullptr;                   // later rounds: one list
            else b.task_count_b = nullptr;
            CU(cg_launch_list(b, false, s->host.max_m, trim_grid(c, d.run_occ, need), d.list_smem, st));
            c->launches += 1;
        }
        if (sev[0]) { CU(cudaEventRecord(sev[3], st)); c->stage_events.push_back(sev); }
        if (d.fuse_stats) {
            // the reads the first stage handed on, as the plan and run kernels listed them (the event pair of the
            // call brackets these launches too)
            CU(cg_launch_stats_entries(c->stat_ents.p, cnt + 6, n_sub, a.stats_max_len, a.stats_kmax, a.stats, st));
            c->launches += 1;
        }
    }
    return CG_OK;
}

// generic path: thread per read, columns in HBM scratch (16 bytes per cell)
static int launch_generic(cg_ctx *c, CgKernelArgs a, cudaStream_t st)
{
    const int block = 128;
    long long threads = (long long)c->sm_count * 8 * block;
    const long long per_thread = (long long)a.col_rows * 16;
    while (threads > 32 * block && threads * per_thread > (1LL << 30)) threads /= 2;
    if (threads > ((a.n_reads + block - 1) / block) * block) threads = ((a.n_reads + block - 1) / block) * block;
    int rc = c->scratch_p.ensure((size_t)threads * a.col_rows);
    if (rc != CG_OK) return rc;
    rc = c->scratch_w.ensure((size_t)threads * a.col_rows * 3);
    if (rc != CG_OK) return rc;
    a.scratch_p = c->scratch_p.p; a.scratch_w = c->scratch_w.p; a.scratch_stride = threads;
    CU(cg_launch_generic(a, (int)(threads / block), block, st));
    c->launches += 1;
    return CG_OK;
}

static int trim_pass(cg_ctx *c, const cg_adapterset *s, const uint8_t *d_seq, const uint8_t *d_qual,
                     const int64_t *d_offsets, int64_t n_reads, int max_read_len, const cg_params *p,
                     cg_match_rec *d_out, int32_t *d_qtrim, const int32_t *d_view, cudaStream_t st, bool timed,
                     const StatsRequest *stats, const TrimSwitches &sw, bool *stats_counted);

// Several groups, one round: per-adapter passes + selection (see plan_passes_for).  The passes see single-adapter
// sub-sets whose statistics are not the set's, so they count none (the caller counts them on the selected records).
static int launch_multi_pass(cg_ctx *c, const cg_adapterset *s, const CgKernelArgs &a, int max_read_len,
                             const cg_params *p, const TrimSchedule &d, const TrimSwitches &sw, cudaStream_t st)
{
    const bool want_q = a.quality_trim != 0;
    const int np = (int)s->passes.size();
    const long long cap = std::min<long long>(a.n_reads, d.sub);
    int rc = c->pass_tmp.ensure((size_t)cap * np);
    if (rc != CG_OK) return rc;
    bool any_linked = false;
    for (auto &P : s->passes) any_linked = any_linked || P.role == 1;
    if (any_linked) { rc = c->view_back.ensure((size_t)cap * 2); if (rc != CG_OK) return rc; }
    if (want_q && !a.qtrim) { rc = c->view_base.ensure((size_t)cap * 2); if (rc != CG_OK) return rc; }

    CgSelectArgs sel;
    memset(&sel, 0, sizeof sel);
    sel.tmp = c->pass_tmp.p; sel.stride = cap; sel.pass_map = s->d_pass_map;
    sel.t = s->select_tables;

    for (long long r0 = 0; r0 < a.n_reads; r0 += d.sub) {
        const long long n_sub = std::min<long long>(d.sub, a.n_reads - r0);
        const int64_t *offs = a.offsets + r0;
        int32_t *qt = want_q ? (a.qtrim ? a.qtrim + 2 * r0 : c->view_base.p) : nullptr;
        const int32_t *base_view = nullptr;
        for (int pi = 0; pi < np; ++pi) {
            const auto &P = s->passes[pi];
            cg_match_rec *tmp = c->pass_tmp.p + (size_t)pi * cap;
            cg_params pp = *p;
            pp.times = 1;
            const int32_t *view = base_view;
            if (P.role == 1) {
                CU(cg_launch_linked_view(c->pass_tmp.p + (size_t)P.front_pass * cap, base_view, offs, n_sub,
                                         c->view_back.p, st));
                c->launches += 1;
                view = c->view_back.p;
            }
            const bool trims = want_q && pi == 0;    // the first pass does the quality trimming (fused) for all
            if (!trims) { pp.quality_trim = 0; pp.nextseq_trim = 0; }
            rc = trim_pass(c, P.sub, a.seq, trims ? a.qual : nullptr, offs, n_sub, max_read_len, &pp, tmp,
                           trims ? qt : nullptr, trims ? nullptr : view, st, false, nullptr, sw, nullptr);
            if (rc != CG_OK) return rc;
            if (trims) base_view = qt;
        }
        sel.n_reads = n_sub;
        sel.out = a.out + (size_t)r0 * s->host.slots;
        CU(cg_launch_select(sel, st));
        c->launches += 1;
    }
    return CG_OK;
}

// One trimming pass as choose_schedule decides it.  *stats_counted (when not null): whether the pass added the
// statistics of its reads to stats->d_stats.
static int trim_pass(cg_ctx *c, const cg_adapterset *s, const uint8_t *d_seq, const uint8_t *d_qual,
                     const int64_t *d_offsets, int64_t n_reads, int max_read_len, const cg_params *p,
                     cg_match_rec *d_out, int32_t *d_qtrim, const int32_t *d_view, cudaStream_t st, bool timed,
                     const StatsRequest *stats, const TrimSwitches &sw, bool *stats_counted)
{
    const bool want_q = p->quality_trim != 0 || p->nextseq_trim != 0;
    if (want_q && !d_qual) return fail(CG_ENOQUAL, "Cannot do quality trimming when no qualities are available");
    TrimSchedule d;
    int rc = choose_schedule(c, s, n_reads, max_read_len, p, d_view != nullptr, stats, sw, d);
    if (rc != CG_OK) return rc;
    CgKernelArgs a;
    memset(&a, 0, sizeof a);
    a.blob = s->d_blob; a.blob_bytes = (uint32_t)s->host.blob.size();
    a.masks64 = s->d_masks; a.enc = c->d_enc; a.index = s->d_index;
    a.seq = d_seq; a.qual = want_q ? d_qual : nullptr; a.offsets = d_offsets; a.n_reads = n_reads;
    // flags and packed base/cutoff as pre_trim_core expects them
    a.quality_trim = (p->quality_trim ? 1 : 0) | (p->nextseq_trim ? 2 : 0);
    a.cutoff_front = p->cutoff_front; a.cutoff_back = p->cutoff_back;
    a.qbase = (p->quality_base & 255) | (int)((unsigned)p->nextseq_cutoff << 8);
    a.times = p->times < 1 ? 1 : p->times; a.slots = s->host.slots;
    a.out = d_out; a.qtrim = d_qtrim; a.view = d_view; a.err_flag = c->d_err;
    a.col_rows = s->host.max_m + 1; a.no_band = sw.no_band;
    a.tile_cap = d.tile_cap; a.mini_cap = d.mini_cap; a.carry_slot = d.carry_slot;
    if (d.fuse_stats) { a.stats = stats->d_stats; a.stats_max_len = stats->max_len; a.stats_kmax = stats->kmax; }
    // the event pair of a timed call (cg_ctx_kernel_time) brackets everything the call launches
    cudaEvent_t ev[2] = {nullptr, nullptr};
    if (timed && c->timing.size() < 8192) {
        for (cudaEvent_t &e : ev) {
            if (!c->event_pool.empty()) { e = c->event_pool.back(); c->event_pool.pop_back(); }
            else CU(cudaEventCreate(&e));
        }
        CU(cudaEventRecord(ev[0], st));
    }
    switch (d.kind) {
    case TrimKind::Index: rc = launch_index(c, a, d, st); break;
    case TrimKind::Light:
        CU(cg_launch_light(a, trim_grid(c, 16, (n_reads + CG_NT - 1) / CG_NT), st));
        c->launches += 1;
        break;
    case TrimKind::Split: rc = launch_split(c, s, a, d, sw, st); break;
    case TrimKind::Warp:
        CU(cg_launch_warp(a, want_q, trim_grid(c, d.occ, ((n_reads + 31) / 32 + 3) / 4), d.smem, st));
        c->launches += 1;
        break;
    case TrimKind::Fast:
        CU(cg_launch_fast(a, want_q, d.simple, trim_grid(c, d.occ, (n_reads + CG_NT - 1) / CG_NT), d.smem, st));
        c->launches += 1;
        break;
    case TrimKind::Generic: rc = launch_generic(c, a, st); break;
    case TrimKind::MultiPass: rc = launch_multi_pass(c, s, a, max_read_len, p, d, sw, st); break;
    }
    if (rc != CG_OK) return rc;
    if (ev[0]) {
        CU(cudaEventRecord(ev[1], st));
        c->timing.emplace_back(ev[0], ev[1]);
    }
    if (stats_counted) *stats_counted = d.fuse_stats;
    return CG_OK;
}

// Aligner.enable_debug() (_align.pyx:291-296): the DP matrices of ONE read against ONE aligner adapter, every cell
// the search computes (cost and score; CG_DEBUG_NONE where the band never went).  A triage aid: one thread, exact
// int32 cells, no prefilter.  cost / score: (m + 1) x (n + 1) int32, row-major; result8: found, then the six numbers
// of Aligner.locate().
extern "C" int cg_locate_debug(cg_ctx *c, const cg_adapter_desc *adapter, const uint8_t *query, int32_t n,
                               int32_t *cost, int32_t *score, int32_t *result8)
{
    if (!c || !adapter || !cost || !score || !result8 || n < 0 || (n && !query))
        return fail(CG_EINVAL, "cg_locate_debug: bad argument");
    if (adapter->kind != CG_KIND_ALIGNER) return fail(CG_EINVAL, "cg_locate_debug: only aligner adapters have a DP matrix");
    for (int32_t i = 0; i < n; ++i) if (query[i] & 0x80) return fail(CG_ENONASCII, "String must contain only ASCII characters");
    CU(cudaSetDevice(c->device));
    cg_adapter_desc d = *adapter;
    d.n_kmer_entries = 0; d.kmer_entries = nullptr; d.kmer_masks = nullptr; d.reverse_read = 0;
    cg_group_desc g;
    memset(&g, 0, sizeof g);
    g.type = CG_GROUP_SINGLE; g.a0 = 0; g.a1 = -1;
    CgBuiltSet set;
    std::string err;
    int rc = cg_build_set(&d, 1, &g, 1, set, err);
    if (rc != CG_OK) return fail(rc, err);
    const int m = set.max_m;
    const size_t cells = (size_t)(m + 1) * ((size_t)n + 1);
    DevBuf<uint8_t> d_blob, d_query;
    DevBuf<int> d_scratch;
    DevBuf<int32_t> d_mat, d_res;
    if ((rc = d_blob.ensure(set.blob.size())) != CG_OK || (rc = d_query.ensure((size_t)n + 16)) != CG_OK ||
        (rc = d_scratch.ensure(3 * ((size_t)m + 2))) != CG_OK || (rc = d_mat.ensure(2 * cells)) != CG_OK ||
        (rc = d_res.ensure(8)) != CG_OK)
        return rc;
    std::vector<int32_t> none(2 * cells, CG_DEBUG_NONE);
    CU(cudaMemcpy(d_blob.p, set.blob.data(), set.blob.size(), cudaMemcpyHostToDevice));
    if (n) CU(cudaMemcpy(d_query.p, query, (size_t)n, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_mat.p, none.data(), 2 * cells * sizeof(int32_t), cudaMemcpyHostToDevice));
    CU(cg_launch_locate_debug(d_blob.p, c->d_enc, d_query.p, n, d_scratch.p, d_mat.p, d_mat.p + cells, d_res.p, c->stream));
    c->launches += 1;
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaMemcpy(cost, d_mat.p, cells * sizeof(int32_t), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(score, d_mat.p + cells, cells * sizeof(int32_t), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(result8, d_res.p, 8 * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return CG_OK;
}

// The work lists, counters and per-pass scratch of a context are shared by all of its streams: the
// kernels of one trimming pass are ordered after those of the previous pass, whichever lane issued it.
// (They fill the GPU on their own; what overlaps across lanes are the copies.)
// stats: statistics wanted with the pass, or null; *stats_counted (when not null): whether the pass counted them.
static int launch_trim(cg_ctx *c, const cg_adapterset *s, const uint8_t *d_seq, const uint8_t *d_qual,
                       const int64_t *d_offsets, int64_t n_reads, int max_read_len, const cg_params *p,
                       cg_match_rec *d_out, int32_t *d_qtrim, cudaStream_t st, bool timed,
                       const StatsRequest *stats = nullptr, bool *stats_counted = nullptr)
{
    if (n_reads <= 0) return CG_OK;
    if (c->scratch_busy && c->scratch_stream != st) CU(cudaStreamWaitEvent(st, c->scratch_ev, 0));
    const int rc = trim_pass(c, s, d_seq, d_qual, d_offsets, n_reads, max_read_len, p, d_out, d_qtrim, nullptr, st, timed,
                             stats, TrimSwitches(), stats_counted);
    CU(cudaEventRecord(c->scratch_ev, st));
    c->scratch_busy = true;
    c->scratch_stream = st;
    return rc;
}

// A trimming pass plus the statistics of its reads (cg_stats_*) added to d_stats: counted inside the split pipeline
// where choose_schedule fuses them, otherwise by cg_stats_kernel over the records afterwards.
static int launch_trim_with_stats(cg_ctx *c, const cg_adapterset *s, const uint8_t *d_seq, const uint8_t *d_qual,
                                  const int64_t *d_offsets, int64_t n_reads, int max_read_len, const cg_params *p,
                                  cg_match_rec *d_out, int32_t *d_qtrim, cudaStream_t st, bool timed,
                                  unsigned long long *d_stats, int stats_max_len, int stats_kmax)
{
    if (n_reads <= 0) return CG_OK;
    const StatsRequest req = {d_stats, stats_max_len, stats_kmax};
    bool counted = false;
    const int rc = launch_trim(c, s, d_seq, d_qual, d_offsets, n_reads, max_read_len, p, d_out, d_qtrim, st, timed, &req,
                               &counted);
    if (rc != CG_OK || counted) return rc;
    const int times = p->times < 1 ? 1 : p->times;
    CU(cg_launch_stats(d_seq, d_offsets, n_reads, (p->quality_trim || p->nextseq_trim) && d_qtrim, times, s->host.slots,
                       d_out, d_qtrim, s->host.n_adapters, stats_max_len, stats_kmax, d_stats, st));
    c->launches += 1;
    return CG_OK;
}

static int check_err_flag(cg_ctx *c)
{
    int flags[2] = {0, 0};
    CU(cudaMemcpy(flags, c->d_err, sizeof flags, cudaMemcpyDeviceToHost));
    if (flags[0]) {
        cudaMemset(c->d_err, 0, sizeof(int));
        return fail(CG_ENONASCII, "String must contain only ASCII characters");
    }
    return CG_OK;
}

extern "C" int cg_process_batch_device(cg_ctx *c, const cg_adapterset *s, const uint8_t *d_seq,
                                       const uint8_t *d_qual, const int64_t *d_offsets, int64_t n_reads,
                                       int32_t max_read_len, const cg_params *p, cg_match *d_matches,
                                       int32_t *d_qtrim)
{
    if (!c || !s || !p || !d_seq || !d_offsets || !d_matches) return fail(CG_EINVAL, "cg_process_batch_device: NULL argument");
    if (s->ctx != c) return fail(CG_EINVAL, "adapter set belongs to another context");
    if (((uintptr_t)d_seq & 15) || (d_qual && ((uintptr_t)d_qual & 15)))
        return fail(CG_EINVAL, "device sequence/quality buffers must be 16-byte aligned");
    if (n_reads < 0) return fail(CG_EINVAL, "n_reads < 0");
    CU(cudaSetDevice(c->device));
    if (max_read_len <= 0) {
        CU(cudaMemsetAsync(c->d_err + 1, 0, sizeof(int), c->stream));
        CU(cg_launch_max_len(d_offsets, n_reads, c->d_err + 1, c->stream));
        c->launches += 1;
        CU(cudaMemcpyAsync(&max_read_len, c->d_err + 1, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    return launch_trim(c, s, d_seq, d_qual, d_offsets, n_reads, max_read_len, p, (cg_match_rec *)d_matches,
                       d_qtrim, c->stream, true);
}

extern "C" int cg_process_batch_device_stats(cg_ctx *c, const cg_adapterset *s, const uint8_t *d_seq,
                                             const uint8_t *d_qual, const int64_t *d_offsets, int64_t n_reads,
                                             int32_t max_read_len, const cg_params *p, cg_match *d_matches,
                                             int32_t *d_qtrim, int32_t stats_max_len, int32_t stats_kmax, int64_t *d_stats)
{
    if (!c || !s || !p || !d_seq || !d_offsets || !d_matches || !d_stats || stats_max_len < 0 || stats_kmax < 0)
        return fail(CG_EINVAL, "cg_process_batch_device_stats: bad argument");
    if (s->ctx != c) return fail(CG_EINVAL, "adapter set belongs to another context");
    if (((uintptr_t)d_seq & 15) || (d_qual && ((uintptr_t)d_qual & 15)))
        return fail(CG_EINVAL, "device sequence/quality buffers must be 16-byte aligned");
    if (n_reads < 0) return fail(CG_EINVAL, "n_reads < 0");
    if ((p->quality_trim || p->nextseq_trim) && !d_qtrim)
        return fail(CG_EINVAL, "cg_process_batch_device_stats: quality trimming needs d_qtrim (the statistics read it)");
    CU(cudaSetDevice(c->device));
    if (max_read_len <= 0) {
        CU(cudaMemsetAsync(c->d_err + 1, 0, sizeof(int), c->stream));
        CU(cg_launch_max_len(d_offsets, n_reads, c->d_err + 1, c->stream));
        c->launches += 1;
        CU(cudaMemcpyAsync(&max_read_len, c->d_err + 1, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    return launch_trim_with_stats(c, s, d_seq, d_qual, d_offsets, n_reads, max_read_len, p, (cg_match_rec *)d_matches,
                                  d_qtrim, c->stream, true, (unsigned long long *)d_stats, stats_max_len, stats_kmax);
}

// ------------------------------------------------------------------------------------------
// Host batches: 2-lane pipeline
// ------------------------------------------------------------------------------------------
static void parallel_copy(cg_ctx *c, void *dst, const void *src, size_t n);

static bool is_pinned(const void *p)
{
    if (!p) return false;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost;
}

static int lane_finish(cg_ctx *c, Lane &l)
{
    if (!l.busy) return CG_OK;
    CU(cudaStreamSynchronize(l.stream));
    if (l.out_bounced && l.n_out) memcpy(l.dst_out, l.h_out.p, l.n_out * sizeof(cg_match_rec));
    if (l.qtrim_bounced && l.n_qtrim) memcpy(l.dst_qtrim, l.h_qtrim.p, l.n_qtrim * sizeof(int32_t));
    l.busy = false;
    return CG_OK;
}

// Longest read / equal lengths / validity of offsets[r0 .. r1], on the worker pool for large chunks.
struct OffsetScan { int64_t max_len = 0; bool uniform = true, valid = true; };
static OffsetScan scan_offsets_part(const int64_t *offsets, int64_t len0, int64_t a, int64_t b)
{
    OffsetScan o;
    for (int64_t r = a; r < b; ++r) {
        const int64_t len = offsets[r + 1] - offsets[r];
        if (len < 0 || len > 2000000000LL) o.valid = false;
        if (len > o.max_len) o.max_len = len;
        o.uniform = o.uniform && len == len0;
    }
    return o;
}
static void scan_merge(OffsetScan &t, const OffsetScan &o)
{
    t.max_len = std::max(t.max_len, o.max_len);
    t.uniform = t.uniform && o.uniform;
    t.valid = t.valid && o.valid;
}
static const int64_t SCAN_JOB = 1 << 15;
static OffsetScan scan_offsets(cg_ctx *c, const int64_t *offsets, int64_t r0, int64_t r1)
{
    const int64_t len0 = offsets[r0 + 1] - offsets[r0];
    const int64_t nr = r1 - r0;
    if (!c->pool || nr < (1 << 16)) return scan_offsets_part(offsets, len0, r0, r1);
    const int64_t n_jobs = (nr + SCAN_JOB - 1) / SCAN_JOB;
    std::vector<OffsetScan> parts((size_t)c->pool->size());
    c->pool->run(n_jobs, [&](int64_t j, int w) {
        const int64_t a = r0 + j * SCAN_JOB, b = std::min(r1, a + SCAN_JOB);
        scan_merge(parts[(size_t)w], scan_offsets_part(offsets, len0, a, b));
    });
    OffsetScan t;
    for (const OffsetScan &o : parts) scan_merge(t, o);
    return t;
}

// CUTADAPT_B200_H2D_PACK: "0" = raw bytes only, "all" = everything compressed, "0.xx" = that share compressed (fixed,
// for sweeps), otherwise adaptive
static int h2d_pack_mode(double *fixed_share = nullptr)
{
    const char *e = getenv("CUTADAPT_B200_H2D_PACK");
    if (e && e[0] == '0' && e[1] == '.') {
        const double v = atof(e);
        if (v > 0.0 && v < 1.0) { if (fixed_share) *fixed_share = v; return 3; }
    }
    if (e && e[0] == '0') return 0;
    if (e && strcmp(e, "all") == 0) return 2;
    return 1;
}

static int process_batch_impl(cg_ctx *c, const cg_adapterset *s, const uint8_t *seq, const uint8_t *qual,
                              const int64_t *offsets, int64_t n_reads, const cg_params *p,
                              cg_match *matches, int32_t *qtrim, int stats_max_len, int stats_kmax, int64_t *stats);

extern "C" int cg_process_batch(cg_ctx *c, const cg_adapterset *s, const uint8_t *seq, const uint8_t *qual,
                                const int64_t *offsets, int64_t n_reads, const cg_params *p,
                                cg_match *matches, int32_t *qtrim)
{
    return process_batch_impl(c, s, seq, qual, offsets, n_reads, p, matches, qtrim, 0, 0, nullptr);
}

// cg_process_batch plus the statistics vector of the batch (layout of cg_stats_accumulate_device), reduced on the
// device chunk by chunk and ADDED to the caller's host vector at the end: the payload a worker hands to the
// end-of-run merge (Statistics.__iadd__, report.py:81-126) without a second pass over the records.
extern "C" int cg_process_batch_stats(cg_ctx *c, const cg_adapterset *s, const uint8_t *seq, const uint8_t *qual,
                                      const int64_t *offsets, int64_t n_reads, const cg_params *p,
                                      cg_match *matches, int32_t *qtrim, int32_t max_len, int32_t kmax, int64_t *stats)
{
    if (!stats || max_len < 0 || kmax < 0) return fail(CG_EINVAL, "cg_process_batch_stats: bad statistics arguments");
    return process_batch_impl(c, s, seq, qual, offsets, n_reads, p, matches, qtrim, max_len, kmax, stats);
}

static int process_batch_impl(cg_ctx *c, const cg_adapterset *s, const uint8_t *seq, const uint8_t *qual,
                              const int64_t *offsets, int64_t n_reads, const cg_params *p,
                              cg_match *matches, int32_t *qtrim, int stats_max_len, int stats_kmax, int64_t *stats)
{
    if (!c || !s || !p || !offsets || !matches) return fail(CG_EINVAL, "cg_process_batch: NULL argument");
    if (s->ctx != c) return fail(CG_EINVAL, "adapter set belongs to another context");
    if (n_reads < 0) return fail(CG_EINVAL, "n_reads < 0");
    if (n_reads == 0) return CG_OK;
    if (!seq) return fail(CG_EINVAL, "cg_process_batch: seq is NULL");
    const std::chrono::steady_clock::time_point t_enter = std::chrono::steady_clock::now();
    const bool want_q = p->quality_trim != 0 || p->nextseq_trim != 0;
    if (want_q && !qual) return fail(CG_ENOQUAL, "Cannot do quality trimming when no qualities are available");
    CU(cudaSetDevice(c->device));
    const int times = p->times < 1 ? 1 : p->times;
    const size_t rec_per_read = (size_t)times * s->host.slots;
    const bool seq_pinned = is_pinned(seq), qual_pinned = want_q && is_pinned(qual);
    const bool offs_pinned = is_pinned(offsets), out_pinned = is_pinned(matches);
    const bool qt_pinned = qtrim && is_pinned(qtrim);

    // Large batches travel compressed (three characters per byte, cg_hostpack.h): PCIe, not the
    // kernels, bounds this entry point.  Small ones are not worth waking the worker pool for.
    const size_t n_stats = stats ? (size_t)cg_stats_total(s->host.n_adapters, stats_max_len, stats_kmax) : 0;
    if (stats) {
        int rcs = c->d_stats.ensure(n_stats);
        if (rcs != CG_OK) return rcs;
        CU(cudaMemset(c->d_stats.p, 0, n_stats * sizeof(unsigned long long)));
    }
    double fixed_share = 0.0;
    const int pack_mode = h2d_pack_mode(&fixed_share);
    const bool pack = pack_mode != 0 && n_reads >= (1 << 16);
    if (pack_mode == 3) c->pack_fraction = fixed_share;
    if (pack && !c->pool) {
        c->pool = new CgHostPool(cg_host_threads_default());
        c->exc_scratch.resize((size_t)c->pool->size());
    }
    if (pack) c->numa_node = c->pool->follow_memory(seq);
    const int n_lanes = pack ? CG_N_LANES : 2;
    const int64_t CHUNK_READS = pack ? (1 << 20) : (1 << 18);
    const int64_t CHUNK_BYTES = pack ? (192LL << 20) : (48LL << 20);
    int64_t r0 = 0;
    int lane_idx = 0, n_chunk = 0;
    int rc = CG_OK;
    using clk = std::chrono::steady_clock;
    auto secs = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double>(b - a).count(); };
    const clk::time_point t_begin = clk::now();
    clk::time_point fb_t0 = t_begin;
    // CUTADAPT_B200_HOST_TRACE=1: where the host side of this call spent its time (stderr, one line per call)
    const bool trace = getenv("CUTADAPT_B200_HOST_TRACE") != nullptr;
    double tr_setup = secs(t_enter, t_begin), tr_alloc = 0, tr_h2d = 0, tr_launch = 0, tr_d2h = 0, tr_tail = 0;
    int64_t fb_reads = 0;
    int64_t ahead_r0 = -1, ahead_r1 = -1;
    OffsetScan ahead_sc;
    while (r0 < n_reads && rc == CG_OK) {
        // chunk [r0, r1): bounded by reads and bytes; also find the longest read
        int64_t r1 = std::min(n_reads, r0 + CHUNK_READS);
        const clk::time_point t_scan0 = clk::now();
        // (while a chunk is packed, the workers also scan the offsets of the next one)
        OffsetScan sc = (ahead_r0 == r0 && ahead_r1 == r1) ? ahead_sc : scan_offsets(c, offsets, r0, r1);
        c->prof[1] += secs(t_scan0, clk::now());
        c->prof[5] += 1;
        if (!sc.valid) return fail(CG_EINVAL, "offsets must be non-decreasing");
        const int64_t byte0 = offsets[r0];
        if (offsets[r1] - byte0 > CHUNK_BYTES && r1 - r0 > 1) {
            // offsets[r0 .. r1] is non-decreasing: the last read that still fits
            const int64_t *it = std::upper_bound(offsets + r0 + 1, offsets + r1 + 1, byte0 + CHUNK_BYTES);
            r1 = std::max<int64_t>(r0 + 1, (it - offsets) - 1);
            sc = scan_offsets(c, offsets, r0, r1);
        }
        const int64_t len0 = offsets[r0 + 1] - offsets[r0];
        const bool uniform = sc.uniform;      // all reads of the chunk equally long (typical for raw Illumina data)
        const int max_len = (int)sc.max_len;
        const int64_t nr = r1 - r0;
        const int64_t nbytes = offsets[r1] - byte0;
        const int pad = (int)(byte0 & 15);
        const int64_t a0 = byte0 - pad;       // the chunk's device buffer starts at this absolute position
        Lane &l = c->lanes[lane_idx];
        lane_idx = (lane_idx + 1) % n_lanes;
        double lane_wait_s = 0.0;
        {
            const clk::time_point t0 = clk::now();
            rc = lane_finish(c, l);
            lane_wait_s = secs(t0, clk::now());
            c->prof[3] += lane_wait_s;
            if (rc != CG_OK) break;
        }
        const clk::time_point t_alloc0 = clk::now();
        if (want_q && (rc = l.d_qual.ensure((size_t)nbytes + 64)) != CG_OK) break;
        if ((rc = l.d_offs.ensure((size_t)nr + 1)) != CG_OK) break;
        if ((rc = l.d_out.ensure((size_t)nr * rec_per_read)) != CG_OK) break;
        if ((qtrim || (stats && want_q)) && (rc = l.d_qtrim.ensure((size_t)nr * 2)) != CG_OK) break;
        const clk::time_point t_h2d0 = clk::now();
        tr_alloc += secs(t_alloc0, t_h2d0);
        // ---- H2D of the sequences ----
        // The first `packed_bytes` of the chunk's buffer travel as the compressed stream, the rest raw: packing
        // costs host time, raw bytes cost PCIe time, and the split (c->pack_fraction) follows whichever of the
        // two was the bottleneck for the previous chunks (see the feedback rule below).
        int64_t packed_bytes = 0;       // characters [a0, a0 + packed_bytes) arrive through the stream
        double pack_s = 0.0;
        if (pack && nbytes > 0) {
            const int64_t span = offsets[r1] - a0;
            const bool all = pack_mode == 2 || c->pack_fraction >= 0.999 || span < (1 << 20);
            int64_t n_stream = all ? ((span + 2) / 3 + 15) / 16 * 16
                                   : (int64_t)(c->pack_fraction * (double)span / 48.0) * 16;
            if (n_stream > 0) {
                if ((rc = l.h_pack.ensure((size_t)n_stream)) != CG_OK) break;
                const int64_t lo = std::max(a0, offsets[0]), hi = offsets[r1];
                for (auto &v : c->exc_scratch) v.clear();
                const int64_t JOB = 1 << 16;
                uint8_t *h_pack = l.h_pack.p;
                const clk::time_point t_pack0 = clk::now();
                // ... and, in the same job set, the offsets of the next chunk
                const int64_t nx0 = r1, nx1 = std::min(n_reads, r1 + CHUNK_READS);
                const int64_t n_pack_jobs = (n_stream + JOB - 1) / JOB;
                const int64_t n_scan_jobs = nx1 > nx0 ? (nx1 - nx0 + SCAN_JOB - 1) / SCAN_JOB : 0;
                const int64_t nx_len0 = nx1 > nx0 ? offsets[nx0 + 1] - offsets[nx0] : 0;
                std::vector<OffsetScan> parts((size_t)c->pool->size());
                c->pool->run(n_pack_jobs + n_scan_jobs, [&](int64_t j, int w) {
                    if (j < n_pack_jobs) {
                        cg_pack3_range(seq, a0, lo, hi, j * JOB, std::min(n_stream, (j + 1) * JOB), h_pack,
                                       c->exc_scratch[(size_t)w]);
                    } else {
                        const int64_t a = nx0 + (j - n_pack_jobs) * SCAN_JOB, b = std::min(nx1, a + SCAN_JOB);
                        scan_merge(parts[(size_t)w], scan_offsets_part(offsets, nx_len0, a, b));
                    }
                });
                if (n_scan_jobs) {
                    ahead_sc = OffsetScan();
                    for (const OffsetScan &o : parts) scan_merge(ahead_sc, o);
                    ahead_r0 = nx0; ahead_r1 = nx1;
                }
                pack_s = secs(t_pack0, clk::now());
                c->prof[2] += pack_s;
                size_t n_exc = 0;
                for (auto &v : c->exc_scratch) n_exc += v.size();
                if ((int64_t)n_exc * 16 <= 3 * n_stream) {   // mostly A/C/G/T/N: send the stream, else the raw bytes
                    if ((rc = l.d_pack.ensure((size_t)n_stream)) != CG_OK) break;
                    if ((rc = l.d_seq.ensure((size_t)std::max<int64_t>(n_stream * 3, span) + 64)) != CG_OK) break;
                    if (n_exc) {
                        if ((rc = l.h_exc.ensure(n_exc)) != CG_OK) break;
                        if ((rc = l.d_exc.ensure(n_exc)) != CG_OK) break;
                        size_t k = 0;
                        for (auto &v : c->exc_scratch) {
                            if (!v.empty()) memcpy(l.h_exc.p + k, v.data(), v.size() * sizeof(uint64_t));
                            k += v.size();
                        }
                        CU(cudaMemcpyAsync(l.d_exc.p, l.h_exc.p, n_exc * sizeof(uint64_t), cudaMemcpyHostToDevice, l.stream));
                    }
                    CU(cudaMemcpyAsync(l.d_pack.p, l.h_pack.p, (size_t)n_stream, cudaMemcpyHostToDevice, l.stream));
                    CU(cg_launch_unpack3(l.d_pack.p, n_stream, l.d_seq.p, (const unsigned long long *)l.d_exc.p,
                                         (long long)n_exc, l.stream));
                    c->launches += n_exc ? 2 : 1;
                    c->h2d_bytes += n_stream + (long long)(n_exc * sizeof(uint64_t));
                    c->prof[6] += (double)std::min<int64_t>(3 * n_stream, span);
                    packed_bytes = 3 * n_stream;
                }
            }
        }
        if (a0 + packed_bytes < offsets[r1]) {
            // raw bytes (bounced through pinned memory unless the caller's buffer already is)
            if ((rc = l.d_seq.ensure((size_t)(offsets[r1] - a0) + 64)) != CG_OK) break;
            const int64_t from = std::max(a0 + packed_bytes, byte0);     // absolute position of the first raw byte
            const int64_t n_raw = offsets[r1] - from;
            const uint8_t *src_seq = seq + from;
            if (!seq_pinned) {
                if ((rc = l.h_seq.ensure((size_t)n_raw + 16)) != CG_OK) break;
                parallel_copy(c, l.h_seq.p, src_seq, (size_t)n_raw);
                src_seq = l.h_seq.p;
            }
            CU(cudaMemcpyAsync(l.d_seq.p + (from - a0), src_seq, (size_t)n_raw, cudaMemcpyHostToDevice, l.stream));
            c->h2d_bytes += n_raw;
        }
        if (pack && pack_mode == 1) {
            // The share of a chunk that travels compressed is tuned on what matters, the rate at which chunks get
            // through: over windows of 8 chunks the reads per second are measured; a probe to a neighbouring share
            // is kept if it was faster, else the best share so far is restored and the next probe goes the other
            // way.  Raw transfer is share 0, so the compressed path can never settle below the raw rate (packing
            // pays when host threads are plentiful, not when 8 ranks share them).
            if (n_chunk >= n_lanes && (n_chunk - n_lanes) % 8 == 0) { fb_t0 = clk::now(); fb_reads = 0; }
            if (n_chunk >= n_lanes) fb_reads += nr;
            if (n_chunk >= n_lanes && (n_chunk - n_lanes) % 8 == 7) {
                const double rate = (double)fb_reads / std::max(1e-9, secs(fb_t0, clk::now()));
                const double step = 0.08;
                auto clamp01 = [](double x) { return x < 0.0 ? 0.0 : (x > 1.0 ? 1.0 : x); };
                if (!c->pack_have_ref) {
                    c->pack_ref_rate = rate; c->pack_ref_fraction = c->pack_fraction; c->pack_have_ref = true;
                    if (clamp01(c->pack_fraction + c->pack_dir * step) == c->pack_fraction) c->pack_dir = -c->pack_dir;
                    c->pack_fraction = clamp01(c->pack_fraction + c->pack_dir * step);
                } else if (rate > c->pack_ref_rate * 1.01) {
                    c->pack_ref_rate = rate; c->pack_ref_fraction = c->pack_fraction;
                    if (clamp01(c->pack_fraction + c->pack_dir * step) == c->pack_fraction) c->pack_dir = -c->pack_dir;
                    c->pack_fraction = clamp01(c->pack_fraction + c->pack_dir * step);
                } else {
                    c->pack_fraction = c->pack_ref_fraction;      // the probe did not pay: back, and look the other way
                    c->pack_dir = -c->pack_dir;
                    c->pack_have_ref = false;                     // (the reference rate is re-measured: conditions drift)
                }
            }
        }
        ++n_chunk;
        if (want_q) {
            const uint8_t *src_q = qual + byte0;
            if (!qual_pinned) {
                if ((rc = l.h_qual.ensure((size_t)nbytes + 16)) != CG_OK) break;
                memcpy(l.h_qual.p, src_q, (size_t)nbytes);
                src_q = l.h_qual.p;
            }
            if (nbytes) CU(cudaMemcpyAsync(l.d_qual.p + pad, src_q, (size_t)nbytes, cudaMemcpyHostToDevice, l.stream));
            c->h2d_bytes += nbytes;
        }
        if (uniform) {
            // offsets[r0 + i] = byte0 + i * len0: generated on the device, 8 bytes per read less over PCIe
            CU(cg_launch_fill_offsets(l.d_offs.p, byte0, len0, nr + 1, l.stream));
            c->launches += 1;
        } else {
            const int64_t *src_offs = offsets + r0;
            if (!offs_pinned) {
                if ((rc = l.h_offs.ensure((size_t)nr + 1)) != CG_OK) break;
                memcpy(l.h_offs.p, src_offs, (size_t)(nr + 1) * sizeof(int64_t));
                src_offs = l.h_offs.p;
            }
            CU(cudaMemcpyAsync(l.d_offs.p, src_offs, (size_t)(nr + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, l.stream));
            c->h2d_bytes += (nr + 1) * (long long)sizeof(int64_t);
        }
        // offsets stay absolute: hand the kernel a virtual base so that base + offsets[r] lands
        // in this chunk's buffer with the same 16-byte phase as in the caller's array
        const uint8_t *vseq = l.d_seq.p - a0;
        const uint8_t *vqual = want_q ? l.d_qual.p - a0 : nullptr;
        int32_t *d_qt = (qtrim || (stats && want_q)) ? l.d_qtrim.p : nullptr;
        const clk::time_point t_launch0 = clk::now();
        tr_h2d += secs(t_h2d0, t_launch0);
        if (stats)
            rc = launch_trim_with_stats(c, s, vseq, vqual, l.d_offs.p, nr, max_len, p, l.d_out.p, d_qt, l.stream, true,
                                        c->d_stats.p, stats_max_len, stats_kmax);
        else
            rc = launch_trim(c, s, vseq, vqual, l.d_offs.p, nr, max_len, p, l.d_out.p, d_qt, l.stream, true);
        if (rc != CG_OK) break;
        const clk::time_point t_d2h0 = clk::now();
        tr_launch += secs(t_launch0, t_d2h0);
        // D2H
        cg_match_rec *dst = (cg_match_rec *)matches + (size_t)r0 * rec_per_read;
        l.n_out = (size_t)nr * rec_per_read; l.dst_out = dst; l.out_bounced = !out_pinned;
        if (out_pinned) CU(cudaMemcpyAsync(dst, l.d_out.p, l.n_out * sizeof(cg_match_rec), cudaMemcpyDeviceToHost, l.stream));
        else {
            if ((rc = l.h_out.ensure(l.n_out)) != CG_OK) break;
            CU(cudaMemcpyAsync(l.h_out.p, l.d_out.p, l.n_out * sizeof(cg_match_rec), cudaMemcpyDeviceToHost, l.stream));
        }
        c->d2h_bytes += (long long)(l.n_out * sizeof(cg_match_rec));
        l.n_qtrim = 0; l.qtrim_bounced = false;
        if (qtrim) {
            int32_t *qdst = qtrim + 2 * r0;
            l.n_qtrim = (size_t)nr * 2; l.dst_qtrim = qdst; l.qtrim_bounced = !qt_pinned;
            if (qt_pinned) CU(cudaMemcpyAsync(qdst, l.d_qtrim.p, l.n_qtrim * 4, cudaMemcpyDeviceToHost, l.stream));
            else {
                if ((rc = l.h_qtrim.ensure(l.n_qtrim)) != CG_OK) break;
                CU(cudaMemcpyAsync(l.h_qtrim.p, l.d_qtrim.p, l.n_qtrim * 4, cudaMemcpyDeviceToHost, l.stream));
            }
            c->d2h_bytes += (long long)(l.n_qtrim * 4);
        }
        l.busy = true;
        r0 = r1;
        tr_d2h += secs(t_d2h0, clk::now());
    }
    const clk::time_point t_drain0 = clk::now();
    for (int i = 0; i < CG_N_LANES; ++i) {
        int rc2 = lane_finish(c, c->lanes[i]);
        if (rc == CG_OK) rc = rc2;
    }
    c->prof[4] += secs(t_drain0, clk::now());
    if (rc == CG_OK && stats) {
        std::vector<unsigned long long> h(n_stats);
        CU(cudaMemcpy(h.data(), c->d_stats.p, n_stats * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < n_stats; ++i) stats[i] += (int64_t)h[i];
        c->d2h_bytes += (long long)(n_stats * sizeof(unsigned long long));
    }
    c->prof[0] += secs(t_begin, clk::now());
    if (rc != CG_OK) return rc;
    const clk::time_point t_tail0 = clk::now();
    const int rce = check_err_flag(c);
    tr_tail = secs(t_tail0, clk::now());
    if (trace)
        fprintf(stderr, "[cutadapt_b200] process_batch %lld reads, %d chunks: total %.4f s = setup %.4f + alloc %.4f + h2d (incl. packing, "
                        "h2d also counts the pack feedback) %.4f + launch %.4f + d2h issue %.4f + drain/stats/tail %.4f; share %.2f\n",
                (long long)n_reads, n_chunk, secs(t_enter, clk::now()), tr_setup, tr_alloc, tr_h2d, tr_launch, tr_d2h,
                secs(t_drain0, clk::now()), c->pack_fraction);
    (void)tr_tail;
    return rce;
}

extern "C" int cg_host_cpus_available(void) { return cg_host_cpus(); }
extern "C" int cg_host_threads(void) { return cg_host_threads_default(); }
extern "C" int cg_ctx_numa_node(cg_ctx *c) { return c ? c->numa_node : -1; }

extern "C" int cg_ctx_host_profile(cg_ctx *c, double *out, int reset)
{
    if (!c || !out) return fail(CG_EINVAL, "cg_ctx_host_profile: NULL argument");
    for (int i = 0; i < 8; ++i) out[i] = c->prof[i];
    out[7] = c->pack_fraction;
    if (reset) for (int i = 0; i < 8; ++i) c->prof[i] = 0.0;
    return CG_OK;
}

extern "C" int cg_ctx_transfer_bytes(cg_ctx *c, int64_t *h2d, int64_t *d2h, int reset)
{
    if (!c) return fail(CG_EINVAL, "ctx is NULL");
    if (h2d) *h2d = c->h2d_bytes;
    if (d2h) *d2h = c->d2h_bytes;
    if (reset) { c->h2d_bytes = 0; c->d2h_bytes = 0; }
    return CG_OK;
}

/* Host-side packer of the compressed transfer, exposed for the CPU tests (no device needed). */
extern "C" int64_t cg_pack3_host(const uint8_t *seq, int64_t a0, int64_t lo, int64_t hi, int64_t n_stream,
                                 uint8_t *packed, uint64_t *exceptions, int64_t capacity, int32_t n_threads)
{
    if (!seq || !packed || n_stream < 0 || n_threads < 1) return fail(CG_EINVAL, "cg_pack3_host: bad argument");
    CgHostPool pool(n_threads);
    std::vector<std::vector<uint64_t>> exc((size_t)pool.size());
    const int64_t JOB = 4096;
    pool.run((n_stream + JOB - 1) / JOB, [&](int64_t j, int w) {
        cg_pack3_range(seq, a0, lo, hi, j * JOB, std::min(n_stream, (j + 1) * JOB), packed, exc[(size_t)w]);
    });
    int64_t n = 0;
    for (auto &v : exc)
        for (uint64_t e : v) {
            if (exceptions && n < capacity) exceptions[n] = e;
            ++n;
        }
    return n;
}

// ------------------------------------------------------------------------------------------
// Stand-alone batched natives (host pointers; lane 0)
// ------------------------------------------------------------------------------------------
static int upload_reads(cg_ctx *c, Lane &l, const uint8_t *bytes, const int64_t *offsets, int64_t n_reads,
                        bool as_qual)
{
    const int64_t total = offsets[n_reads];
    DevBuf<uint8_t> &d = as_qual ? l.d_qual : l.d_seq;
    int rc = d.ensure((size_t)total + 64);
    if (rc != CG_OK) return rc;
    if ((rc = l.d_offs.ensure((size_t)n_reads + 1)) != CG_OK) return rc;
    if (total) CU(cudaMemcpyAsync(d.p, bytes, (size_t)total, cudaMemcpyHostToDevice, l.stream));
    CU(cudaMemcpyAsync(l.d_offs.p, offsets, (size_t)(n_reads + 1) * 8, cudaMemcpyHostToDevice, l.stream));
    return CG_OK;
}

extern "C" int cg_kmers_present_batch(cg_ctx *c, const cg_kmer_entry *entries, const uint64_t *masks,
                                      int32_t n_entries, const uint8_t *seq, const int64_t *offsets,
                                      int64_t n_reads, uint8_t *out)
{
    if (!c || !offsets || !out || n_reads < 0 || n_entries < 0) return fail(CG_EINVAL, "cg_kmers_present_batch: bad argument");
    if (n_reads == 0) return CG_OK;
    if (offsets[0] != 0) return fail(CG_EINVAL, "offsets[0] must be 0");
    CU(cudaSetDevice(c->device));
    Lane &l = c->lanes[0];
    int rc = lane_finish(c, l);
    if (rc != CG_OK) return rc;
    std::vector<CgEntry> ents((size_t)std::max(n_entries, 1));
    memset(ents.data(), 0, ents.size() * sizeof(CgEntry));
    for (int e = 0; e < n_entries; ++e) {
        if (entries[e].search_start > 2000000000LL || entries[e].search_start < -2000000000LL ||
            entries[e].search_stop > 2000000000LL || entries[e].search_stop < -2000000000LL)
            return fail(CG_EINVAL, "k-mer window out of range");
        ents[e].start = (int32_t)entries[e].search_start; ents[e].stop = (int32_t)entries[e].search_stop;
        ents[e].mask_index = (uint32_t)e;
        ents[e].init_mask = entries[e].init_mask; ents[e].found_mask = entries[e].found_mask;
    }
    CgEntry *d_ents = nullptr;
    uint64_t *d_masks = nullptr;
    uint8_t *d_out = nullptr;
    const size_t mask_words = (size_t)std::max(n_entries, 1) * 128;
    cudaError_t e = cudaMalloc((void **)&d_ents, ents.size() * sizeof(CgEntry));
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_masks, mask_words * 8);
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_out, (size_t)n_reads);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_ents, ents.data(), ents.size() * sizeof(CgEntry), cudaMemcpyHostToDevice, l.stream);
    if (e == cudaSuccess && n_entries > 0) e = cudaMemcpyAsync(d_masks, masks, (size_t)n_entries * 128 * 8, cudaMemcpyHostToDevice, l.stream);
    if (e == cudaSuccess) {
        rc = upload_reads(c, l, seq, offsets, n_reads, false);
        if (rc == CG_OK) {
            e = cg_launch_kmers_present(d_ents, n_entries, d_masks, l.d_seq.p, l.d_offs.p, n_reads, d_out, c->d_err, l.stream);
            c->launches += 1;
            if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out, (size_t)n_reads, cudaMemcpyDeviceToHost, l.stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(l.stream);
        }
    }
    if (d_ents) cudaFree(d_ents);
    if (d_masks) cudaFree(d_masks);
    if (d_out) cudaFree(d_out);
    if (rc != CG_OK) return rc;
    if (e != cudaSuccess) return cuda_fail(e, "cg_kmers_present_batch");
    return check_err_flag(c);
}

extern "C" int cg_quality_trim_batch(cg_ctx *c, const uint8_t *qual, const int64_t *offsets, int64_t n_reads,
                                     int32_t cutoff_front, int32_t cutoff_back, int32_t base, int32_t *out)
{
    if (!c || !offsets || !out || n_reads < 0) return fail(CG_EINVAL, "cg_quality_trim_batch: bad argument");
    if (n_reads == 0) return CG_OK;
    if (!qual) return fail(CG_ENOQUAL, "Cannot do quality trimming when no qualities are available");
    if (offsets[0] != 0) return fail(CG_EINVAL, "offsets[0] must be 0");
    CU(cudaSetDevice(c->device));
    Lane &l = c->lanes[0];
    int rc = lane_finish(c, l);
    if (rc != CG_OK) return rc;
    if ((rc = upload_reads(c, l, qual, offsets, n_reads, true)) != CG_OK) return rc;
    if ((rc = l.d_qtrim.ensure((size_t)n_reads * 2)) != CG_OK) return rc;
    CU(cg_launch_quality_trim(l.d_qual.p, l.d_offs.p, n_reads, cutoff_front, cutoff_back, base, l.d_qtrim.p, l.stream));
    c->launches += 1;
    CU(cudaMemcpyAsync(out, l.d_qtrim.p, (size_t)n_reads * 8, cudaMemcpyDeviceToHost, l.stream));
    CU(cudaStreamSynchronize(l.stream));
    return CG_OK;
}

extern "C" int cg_nextseq_trim_batch(cg_ctx *c, const uint8_t *seq, const uint8_t *qual, const int64_t *offsets,
                                     int64_t n_reads, int32_t cutoff, int32_t base, int32_t *out)
{
    if (!c || !offsets || !out || n_reads < 0) return fail(CG_EINVAL, "cg_nextseq_trim_batch: bad argument");
    if (n_reads == 0) return CG_OK;
    if (!qual) return fail(CG_ENOQUAL, "Cannot do quality trimming when no qualities are available");
    if (!seq) return fail(CG_EINVAL, "cg_nextseq_trim_batch: seq is NULL");
    if (offsets[0] != 0) return fail(CG_EINVAL, "offsets[0] must be 0");
    CU(cudaSetDevice(c->device));
    Lane &l = c->lanes[0];
    int rc = lane_finish(c, l);
    if (rc != CG_OK) return rc;
    if ((rc = upload_reads(c, l, seq, offsets, n_reads, false)) != CG_OK) return rc;
    if ((rc = upload_reads(c, l, qual, offsets, n_reads, true)) != CG_OK) return rc;
    if ((rc = l.d_qtrim.ensure((size_t)n_reads * 2)) != CG_OK) return rc;
    CU(cg_launch_nextseq_trim(l.d_seq.p, l.d_qual.p, l.d_offs.p, n_reads, cutoff, base, l.d_qtrim.p, l.stream));
    c->launches += 1;
    CU(cudaMemcpyAsync(out, l.d_qtrim.p, (size_t)n_reads * 4, cudaMemcpyDeviceToHost, l.stream));
    CU(cudaStreamSynchronize(l.stream));
    return CG_OK;
}

extern "C" int cg_expected_errors_batch(cg_ctx *c, const uint8_t *qual, const int64_t *offsets, int64_t n_reads,
                                        int32_t base, double *out)
{
    if (!c || !offsets || !out || n_reads < 0 || base < 0 || base > 126)
        return fail(CG_EINVAL, "cg_expected_errors_batch: bad argument");
    if (n_reads == 0) return CG_OK;
    if (!qual) return fail(CG_ENOQUAL, "no qualities available");
    if (offsets[0] != 0) return fail(CG_EINVAL, "offsets[0] must be 0");
    CU(cudaSetDevice(c->device));
    Lane &l = c->lanes[0];
    int rc = lane_finish(c, l);
    if (rc != CG_OK) return rc;
    if ((rc = upload_reads(c, l, qual, offsets, n_reads, true)) != CG_OK) return rc;
    if ((rc = l.d_qtrim.ensure((size_t)n_reads * 2)) != CG_OK) return rc;       // n doubles
    CU(cg_launch_expected_errors(l.d_qual.p, l.d_offs.p, n_reads, base, c->d_phred, (double *)l.d_qtrim.p, l.stream));
    c->launches += 1;
    CU(cudaMemcpyAsync(out, l.d_qtrim.p, (size_t)n_reads * 8, cudaMemcpyDeviceToHost, l.stream));
    CU(cudaStreamSynchronize(l.stream));
    return CG_OK;
}

extern "C" int cg_poly_a_trim_batch(cg_ctx *c, const uint8_t *seq, const int64_t *offsets, int64_t n_reads,
                                    int32_t revcomp, int32_t *out)
{
    if (!c || !offsets || !out || n_reads < 0) return fail(CG_EINVAL, "cg_poly_a_trim_batch: bad argument");
    if (n_reads == 0) return CG_OK;
    if (!seq) return fail(CG_EINVAL, "cg_poly_a_trim_batch: seq is NULL");
    if (offsets[0] != 0) return fail(CG_EINVAL, "offsets[0] must be 0");
    CU(cudaSetDevice(c->device));
    Lane &l = c->lanes[0];
    int rc = lane_finish(c, l);
    if (rc != CG_OK) return rc;
    if ((rc = upload_reads(c, l, seq, offsets, n_reads, false)) != CG_OK) return rc;
    if ((rc = l.d_qtrim.ensure((size_t)n_reads * 2)) != CG_OK) return rc;
    CU(cg_launch_poly_a_trim(l.d_seq.p, l.d_offs.p, n_reads, revcomp ? 1 : 0, l.d_qtrim.p, l.stream));
    c->launches += 1;
    CU(cudaMemcpyAsync(out, l.d_qtrim.p, (size_t)n_reads * 4, cudaMemcpyDeviceToHost, l.stream));
    CU(cudaStreamSynchronize(l.stream));
    return CG_OK;
}

// ------------------------------------------------------------------------------------------
// Statistics
// ------------------------------------------------------------------------------------------
extern "C" int64_t cg_stats_size(int32_t n_adapters, int32_t max_len, int32_t kmax)
{
    if (n_adapters < 0 || max_len < 0 || kmax < 0) return -1;
    return cg_stats_total(n_adapters, max_len, kmax);
}

extern "C" int cg_stats_accumulate_device(cg_ctx *c, const cg_adapterset *s, const uint8_t *d_seq, const int64_t *d_offsets,
                                          int64_t n_reads, const cg_params *p, const cg_match *d_matches,
                                          const int32_t *d_qtrim, int32_t max_len, int32_t kmax,
                                          int64_t *d_stats)
{
    if (!c || !s || !p || !d_offsets || !d_matches || !d_stats || max_len < 0 || kmax < 0)
        return fail(CG_EINVAL, "cg_stats_accumulate_device: bad argument");
    if (n_reads <= 0) return CG_OK;
    CU(cudaSetDevice(c->device));
    const int times = p->times < 1 ? 1 : p->times;
    CU(cg_launch_stats(d_seq, d_offsets, n_reads, (p->quality_trim || p->nextseq_trim) && d_qtrim, times, s->host.slots,
                       (const cg_match_rec *)d_matches, d_qtrim, s->host.n_adapters, max_len, kmax,
                       (unsigned long long *)d_stats, c->stream));
    c->launches += 1;
    return CG_OK;
}

// ------------------------------------------------------------------------------------------
// FASTQ chunks in, trimmed FASTQ out (SURVEY.md section 8(f) N1): the per-chunk worker of the reference
// (WorkerProcess.run, runners.py:174-214: parse the chunk, run the modifiers and filters per read, format
// the surviving records) as a handful of kernels around the trimming pass.
// ------------------------------------------------------------------------------------------
static void parallel_copy(cg_ctx *c, void *dst, const void *src, size_t n)
{
    if (!c->pool || n < (8u << 20)) { memcpy(dst, src, n); return; }
    const size_t JOB = 4u << 20;
    c->pool->run((int64_t)((n + JOB - 1) / JOB), [&](int64_t j, int) {
        const size_t o = (size_t)j * JOB;
        memcpy((uint8_t *)dst + o, (const uint8_t *)src + o, std::min(JOB, n - o));
    });
}

// mate (FastqSlot::ilv): the record number of a mate of an interleaved chunk is given as the chunk's (2r or 2r + 1)
static int fastq_format_error(const int err[2], int mate = 0)
{
    if (err[0] == CG_FA_ERR_BEFORE_HEADER || err[0] == CG_FA_ERR_LATE_COMMENT)
        return fail(CG_EINVAL, std::string("FASTA format error in line ") + std::to_string((long long)(unsigned)err[1] + 1) +
                                   (err[0] == CG_FA_ERR_BEFORE_HEADER
                                        ? ": expected '>' at the beginning of a record"
                                        : ": a '#' comment line after the first record"));
    static const char *what[] = {"", "a record does not start with '@'", "the third line of a record does not start with '+'",
                                 "sequence and qualities differ in length", "invalid quality value",
                                 "sequence descriptions don't match (the second one must be empty or equal to the first)"};
    const long long r = mate ? 2LL * err[1] + (mate - 1) : (long long)err[1];
    return fail(CG_EINVAL, std::string("FASTQ format error in record ") + std::to_string(r) +
                               (mate ? " of the interleaved chunk: " : ": ") + what[err[0] & 7]);
}

// Streams, counters and error words of a slot, the host pool
static int fastq_slot_init(cg_ctx *c, FastqSlot &f)
{
    f.ilv = 0;
    f.rows_ready = false;                       // a new chunk: the rows of the last one are gone, no requests yet
    for (FqRows &q : f.rows) {
        q.requested = false;
        q.limit = -1;
        q.bytes = q.bytes_plain = 0;
    }
    if (!f.stream) CU(cudaStreamCreateWithFlags(&f.stream, cudaStreamNonBlocking));
    int rc;
    if ((rc = f.d_counters.ensure(1 + CG_FQ_COUNTERS)) != CG_OK || (rc = f.d_err.ensure(2)) != CG_OK) return rc;
    if (!c->pool) {
        c->pool = new CgHostPool(cg_host_threads_default());
        c->exc_scratch.resize((size_t)c->pool->size());
    }
    if ((rc = f.h_counters.ensure(1 + CG_FQ_COUNTERS)) != CG_OK) return rc;
    CU(cudaMemsetAsync(f.d_counters.p, 0, (1 + CG_FQ_COUNTERS) * sizeof(unsigned long long), f.stream));
    const int err_init[2] = {0, 0x7FFFFFFF};
    CU(cudaMemcpyAsync(f.d_err.p, err_init, sizeof err_init, cudaMemcpyHostToDevice, f.stream));
    return CG_OK;
}

// The newline count of the chunk in f.d_in[0, n_bytes)
static int fastq_slot_count(cg_ctx *c, FastqSlot &f, int64_t n_bytes)
{
    int rc;
    if ((rc = f.d_tiles.ensure((size_t)cg_fastq_tiles(n_bytes) + 1)) != CG_OK) return rc;
    f.n_bytes = n_bytes;
    if (n_bytes) {
        CU(cg_launch_fastq_index(f.d_in.p, n_bytes, f.d_tiles.p, f.d_counters.p, nullptr, 0, f.stream));
        c->launches += 2;
    }
    CU(cudaMemcpyAsync(f.h_counters.p, f.d_counters.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, f.stream));
    return CG_OK;
}

// init, the upload of the chunk and its newline count
static int fastq_slot_upload(cg_ctx *c, FastqSlot &f, const uint8_t *fastq, int64_t n_bytes)
{
    int rc;
    if ((rc = fastq_slot_init(c, f)) != CG_OK) return rc;
    if ((rc = f.d_in.ensure((size_t)n_bytes + 64)) != CG_OK) return rc;
    if (n_bytes) {
        const uint8_t *src = fastq;
        if (!is_pinned(fastq)) {
            if ((rc = f.h_in.ensure((size_t)n_bytes)) != CG_OK) return rc;
            parallel_copy(c, f.h_in.p, fastq, (size_t)n_bytes);
            src = f.h_in.p;
        }
        CU(cudaMemcpyAsync(f.d_in.p, src, (size_t)n_bytes, cudaMemcpyHostToDevice, f.stream));
        c->h2d_bytes += n_bytes;
    }
    return fastq_slot_count(c, f, n_bytes);
}

// The argument checks of a submit: `ok` holds the caller's own, then up to two byte buffers and the format; `what` names
// a buffer in the size message.
static int submit_check(const char *who, bool ok, int32_t format, const char *what, const uint8_t *p1, int64_t n1,
                        const uint8_t *p2 = nullptr, int64_t n2 = 0, int32_t max_format = CG_FORMAT_FASTQ_TO_FASTA)
{
    if (!ok || n1 < 0 || n2 < 0 || (n1 && !p1) || (n2 && !p2) || format < CG_FORMAT_FASTQ || format > max_format)
        return fail(CG_EINVAL, std::string(who) + ": bad argument");
    if (n1 >= (1LL << 31) || n2 >= (1LL << 31))
        return fail(CG_EINVAL, std::string(who) + ": a " + what + " must be smaller than 2 GiB");
    return CG_OK;
}

// The n (1 or 2) slots a submission gets, from fq_next on; *s1 the first.  `busy`: the message when one is in flight.
static int fq_find(cg_ctx *c, int n, const char *busy, int *s1)
{
    *s1 = c->fq_next;
    for (int i = 0; i < n; ++i)
        if (c->fq[(*s1 + i) % CG_FQ_SLOTS].busy) return fail(CG_EINVAL, busy);
    return CG_OK;
}

// Hand out the slots fq_find found: one (slot2 == nullptr) or two, busy until collected.  ilv_format >= 0: the two are
// the mates of one interleaved chunk in that input format (FastqSlot::ilv).
static void fq_take(cg_ctx *c, int s1, int32_t *slot1, int32_t *slot2 = nullptr, int ilv_format = -1)
{
    const int s2 = (s1 + 1) % CG_FQ_SLOTS;
    c->fq[s1].busy = true;
    *slot1 = s1;
    c->fq_next = s2;
    if (!slot2) return;
    c->fq[s2].busy = true;
    *slot2 = s2;
    c->fq_next = (s2 + 1) % CG_FQ_SLOTS;
    if (ilv_format < 0) return;
    FastqSlot &f1 = c->fq[s1], &f2 = c->fq[s2];
    f1.ilv = 1; f1.ilv_peer = s2;
    f2.ilv = 2; f2.ilv_peer = s1;
    f1.ilv_format = f2.ilv_format = ilv_format == CG_FORMAT_FASTA ? CG_FORMAT_FASTA : CG_FORMAT_FASTQ;
}

extern "C" int cg_fastq_submit(cg_ctx *c, const uint8_t *fastq, int64_t n_bytes, int32_t *slot_out)
{
    int rc = submit_check("cg_fastq_submit", c && slot_out, CG_FORMAT_FASTQ, "chunk", fastq, n_bytes);
    if (rc != CG_OK) return rc;
    CU(cudaSetDevice(c->device));
    int si;
    if ((rc = fq_find(c, 1, "cg_fastq_submit: all slots are in flight, collect one first", &si)) != CG_OK) return rc;
    if ((rc = fastq_slot_upload(c, c->fq[si], fastq, n_bytes)) != CG_OK) return rc;
    fq_take(c, si, slot_out);
    return CG_OK;
}

extern "C" int cg_fastq_submit_interleaved(cg_ctx *c, const uint8_t *chunk, int64_t n_bytes, int32_t format, int32_t *slot1,
                                           int32_t *slot2)
{
    int rc = submit_check("cg_fastq_submit_interleaved", c && slot1 && slot2, format, "chunk", chunk, n_bytes);
    if (rc != CG_OK) return rc;
    CU(cudaSetDevice(c->device));
    int s1;
    if ((rc = fq_find(c, 2, "cg_fastq_submit_interleaved: two free slots are needed, collect one first", &s1)) != CG_OK)
        return rc;
    if ((rc = fastq_slot_upload(c, c->fq[s1], chunk, n_bytes)) != CG_OK) return rc;
    // its chunk comes from the split
    if ((rc = fastq_slot_upload(c, c->fq[(s1 + 1) % CG_FQ_SLOTS], nullptr, 0)) != CG_OK) return rc;
    fq_take(c, s1, slot1, slot2, format);
    return CG_OK;
}

// ------------------------------------------------------------------------------------------
// gzip input (cg_fastq_submit_gzip*): the compressed bytes are uploaded, their members inflated on the device
// (cg_gunzip.cu) behind the stream's carry, and the longest prefix of whole records becomes a slot's chunk.  Small
// readbacks per file and submission size the buffers and decide: the candidate count, the chain, the first bad CRC, the
// newline count, the flagged-newline count and the cut.  Everything runs on the stream of the slot the submission
// reserved.
// ------------------------------------------------------------------------------------------
#define CG_GZIN_LIMIT (1LL << 31)        // plain bytes of one submission stay under the slot limit

extern "C" int cg_gzin_create_ex(cg_ctx *c, int32_t flags, int32_t *handle)
{
    if (!c || !handle || (flags & ~CG_GZIN_SPLIT_MEMBERS)) return fail(CG_EINVAL, "cg_gzin_create: bad argument");
    CU(cudaSetDevice(c->device));
    const int32_t h = c->gzin_next++;
    GzinStream &g = c->gzin[h];
    int rc;
    if ((rc = g.d_small.ensure(4 + (std::max(sizeof(GuChain), sizeof(GuWalk)) + 7) / 8)) != CG_OK) {
        c->gzin.erase(h);
        return rc;
    }
    if (flags & CG_GZIN_SPLIT_MEMBERS) {
        g.split = true;
        // CUTADAPT_B200_GZIN_STRIDE (cutadapt_b200.h): the stride sweep of tools/measure_fastq.py --gzip-input
        if (const char *e = getenv("CUTADAPT_B200_GZIN_STRIDE")) g.stride = std::max(32768LL, atoll(e));
        if ((rc = g.d_win.ensure(GU_WIN)) != CG_OK || (rc = g.d_pwin.ensure(GU_WIN)) != CG_OK) {
            c->gzin.erase(h);
            return rc;
        }
    }
    CU(cudaEventCreateWithFlags(&g.done, cudaEventDisableTiming));
    *handle = h;
    return CG_OK;
}

extern "C" int cg_gzin_create(cg_ctx *c, int32_t *handle) { return cg_gzin_create_ex(c, 0, handle); }

extern "C" int cg_gzin_destroy(cg_ctx *c, int32_t handle)
{
    if (!c) return fail(CG_EINVAL, "cg_gzin_destroy: bad argument");
    auto it = c->gzin.find(handle);
    if (it == c->gzin.end()) return fail(CG_EINVAL, "cg_gzin_destroy: unknown handle");
    CU(cudaSetDevice(c->device));
    if (it->second.done) CU(cudaEventSynchronize(it->second.done));
    c->gzin.erase(it);
    return CG_OK;
}

// d_plain holds at least `total` bytes (+ 64); its first `keep` bytes stay
static int gzin_plain_room(GzinStream &g, long long keep, long long total, cudaStream_t st)
{
    if ((size_t)total + 64 <= g.d_plain.cap) return CG_OK;
    DevBuf<uint8_t> nb;
    int rc;
    if ((rc = nb.ensure((size_t)total + 64)) != CG_OK) return rc;
    if (keep) CU(cudaMemcpyAsync(nb.p, g.d_plain.p, (size_t)keep, cudaMemcpyDeviceToDevice, st));
    CU(cudaStreamSynchronize(st));
    g.d_plain = std::move(nb);
    return CG_OK;
}

// The chain of whole members from byte `from` inflated behind d_plain[0, base) and their CRC-32 checked (*ch).  split:
// the chain may end at a member for the block path (ch->status GU_LONG).
static int gzin_members(cg_ctx *c, GzinStream &g, long long n, int n_cand, long long from, bool after_member, bool final,
                        long long base, bool split, cudaStream_t st, GuChain *out)
{
    int rc;
    GuChain *d_chain = reinterpret_cast<GuChain *>(g.d_small.p + 4);
    CU(cg_launch_gunzip_chain(g.d_gz.p, n, g.d_cand.p, g.d_res.p, n_cand, after_member, final, base, CG_GZIN_LIMIT,
                              g.d_members.p, g.d_moff.p, d_chain, from, split, st));
    c->launches += 1;
    GuChain &ch = *out;
    CU(cudaMemcpyAsync(&ch, d_chain, sizeof ch, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const long long at = g.consumed + ch.err_at;
    if (ch.status == GU_INVALID)
        return fail(CG_EINVAL, "gzip input: invalid or truncated gzip member at byte " + std::to_string(at) +
                                   " of the compressed file");
    if (ch.status == GU_UNSUPPORTED && !split)
        return fail(CG_EUNSUPPORTED, "gzip input: the member at byte " + std::to_string(at) +
                                         " inflates to more than one submission can hold (2 GiB); decompress this input "
                                         "on the host");
    // the carry stays where it is; a larger buffer gets a copy of it
    if ((rc = gzin_plain_room(g, base, base + ch.plain, st)) != CG_OK) return rc;
    if (ch.n_members) {
        int *d_bad = reinterpret_cast<int *>(g.d_small.p + 2);
        const int none = 0x7FFFFFFF;
        CU(cudaMemcpyAsync(d_bad, &none, sizeof none, cudaMemcpyHostToDevice, st));
        CU(cg_launch_gunzip_place(g.d_gz.p, n, g.d_cand.p, g.d_members.p, g.d_moff.p, d_chain, ch.n_members, g.d_res.p,
                                  g.d_plain.p, d_bad, st));
        c->launches += 2;
        int bad = none;
        CU(cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (bad != none) {
            int32_t k = 0, pos = 0;
            CU(cudaMemcpy(&k, g.d_members.p + bad, sizeof k, cudaMemcpyDeviceToHost));
            CU(cudaMemcpy(&pos, g.d_cand.p + k, sizeof pos, cudaMemcpyDeviceToHost));
            return fail(CG_EINVAL, "gzip input: CRC-32 mismatch in the gzip member at byte " +
                                       std::to_string(g.consumed + pos) + " of the compressed file");
        }
    }
    return CG_OK;
}

// The block path (cg_gunzip_core.cuh, gu_chunk / gu_walk): the member's deflate bits from bit s0 of the uploaded bytes,
// inflated behind d_plain[0, base).  The stream's pending member (g.pmem) says how far the member got before; its
// window is g.d_win.  *r: the walk's verdict (r->plain bytes placed, r->end the bit behind them); the pending window,
// CRC register and length advance.
static int gzin_blocks(cg_ctx *c, GzinStream &g, long long n, long long bound, long long s0, long long base,
                       cudaStream_t st, GuWalk *r,
                       long long *respec)
{
    int rc;
    const long long S = g.stride, limit = CG_GZIN_LIMIT - base;
    const int K = (int)std::max(1LL, (bound * 8 - s0 + S * 8 - 1) / (S * 8));     // chunks up to gu_member_bound
    if ((rc = g.d_ch.ensure((size_t)K)) != CG_OK || (rc = g.d_coff.ensure((size_t)K)) != CG_OK ||
        (rc = g.d_room.ensure((size_t)K)) != CG_OK || (rc = g.d_redo.ensure((size_t)K)) != CG_OK)
        return rc;
    // room for the symbols of a chunk: 8 per compressed byte of its stride, more for a chunk that overflows
    std::vector<long long> off(K), room(K, std::min(limit, 8 * S));
    long long arena = 0;
    for (int k = 0; k < K; ++k) { off[k] = arena; arena += room[k]; }
    if ((rc = g.d_sym.ensure((size_t)arena)) != CG_OK) return rc;
    CU(cudaMemcpyAsync(g.d_coff.p, off.data(), K * sizeof(long long), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(g.d_room.p, room.data(), K * sizeof(long long), cudaMemcpyHostToDevice, st));
    const GuChunk c0 = {s0, s0, 0, 0, GU_INVALID, 0};
    CU(cudaMemcpyAsync(g.d_ch.p, &c0, sizeof c0, cudaMemcpyHostToDevice, st));
    CU(cg_launch_gunzip_search(g.d_gz.p, n, s0, S, K, g.d_ch.p, st));
    CU(cg_launch_gunzip_spec(g.d_gz.p, n, s0, S, K, nullptr, K, g.d_coff.p, g.d_room.p, g.d_sym.p, g.d_ch.p, st));
    c->launches += 2;
    GuWalk *d_walk = reinterpret_cast<GuWalk *>(g.d_small.p + 4);      // the chain's place: no chain runs meanwhile
    std::vector<int32_t> redo;
    std::vector<GuChunk> ch;
    const long long max_rounds = gu_walk_rounds(K, room[0], limit);
    for (long long round = 0;; ++round) {
        CU(cg_launch_gunzip_walk(g.d_ch.p, K, limit, g.d_redo.p, d_walk, st));
        c->launches += 1;
        CU(cudaMemcpyAsync(r, d_walk, sizeof *r, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (r->status != GU_MORE) break;
        if (round >= max_rounds)                      // unreachable by gu_walk_rounds: a defect, not bad input
            return fail(CG_EUNSUPPORTED, "gzip input: internal error: the block walk did not settle within " +
                                             std::to_string(max_rounds) + " rounds");
        *respec += r->respec;
        redo.resize(r->n_redo);
        ch.resize(K);
        CU(cudaMemcpyAsync(redo.data(), g.d_redo.p, r->n_redo * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(ch.data(), g.d_ch.p, K * sizeof(GuChunk), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        long long grown = 0, old_arena = arena;
        for (int32_t k : redo) {
            if (ch[k].status != GU_OVER || (grown && grown >= limit)) continue;
            if (room[k] >= limit) {
                if (k != r->n_ok) continue;
                // the next chunk alone reaches the limit: the submission ends in front of it
                r->status = r->n_ok ? GU_OK : GU_UNSUPPORTED;
                break;
            }
            room[k] = std::min(limit, room[k] * 8);
            off[k] = arena;
            arena += room[k];
            grown += room[k];
        }
        if (r->status != GU_MORE) break;
        if (arena > old_arena) {
            DevBuf<uint16_t> nb;
            if ((rc = nb.ensure((size_t)arena)) != CG_OK) return rc;
            CU(cudaMemcpyAsync(nb.p, g.d_sym.p, (size_t)old_arena * sizeof(uint16_t), cudaMemcpyDeviceToDevice, st));
            CU(cudaStreamSynchronize(st));
            g.d_sym = std::move(nb);
            CU(cudaMemcpyAsync(g.d_coff.p, off.data(), K * sizeof(long long), cudaMemcpyHostToDevice, st));
            CU(cudaMemcpyAsync(g.d_room.p, room.data(), K * sizeof(long long), cudaMemcpyHostToDevice, st));
        }
        CU(cg_launch_gunzip_spec(g.d_gz.p, n, s0, S, K, g.d_redo.p, r->n_redo, g.d_coff.p, g.d_room.p, g.d_sym.p,
                                 g.d_ch.p, st));
        c->launches += 1;
    }
    if (r->status != GU_OK) return CG_OK;
    // the resolve grid is sized by the largest confirmed chunk
    ch.resize(K);
    CU(cudaMemcpyAsync(ch.data(), g.d_ch.p, r->n_ok * sizeof(GuChunk), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    long long max_n = 0;
    for (int k = 0; k < r->n_ok; ++k) max_n = std::max(max_n, ch[k].n);
    if ((rc = gzin_plain_room(g, base, base + r->plain, st)) != CG_OK) return rc;
    if ((rc = g.d_wins.ensure((size_t)(r->n_ok + 1) * GU_WIN)) != CG_OK) return rc;
    CU(cudaMemcpyAsync(g.d_wins.p, g.d_win.p, GU_WIN, cudaMemcpyDeviceToDevice, st));
    int *d_bad = reinterpret_cast<int *>(g.d_small.p + 2);
    uint32_t *d_state = reinterpret_cast<uint32_t *>(g.d_small.p + 3);
    const int none = 0x7FFFFFFF;
    CU(cudaMemcpyAsync(d_bad, &none, sizeof none, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_state, &g.pmem.crc, sizeof g.pmem.crc, cudaMemcpyHostToDevice, st));
    CU(cg_launch_gunzip_resolve(g.d_ch.p, r->n_ok, max_n, g.d_coff.p, g.d_sym.p, g.d_wins.p, g.pmem.len,
                                g.d_plain.p + base, d_bad, st));
    if ((rc = g.d_part.ensure((size_t)(r->plain / cg_gunzip_crc_piece()) + 1)) != CG_OK) return rc;
    CU(cg_launch_gunzip_crc(g.d_plain.p + base, r->plain, g.d_part.p, d_state, st));
    CU(cudaMemcpyAsync(g.d_pwin.p, g.d_wins.p + (long long)r->n_ok * GU_WIN, GU_WIN, cudaMemcpyDeviceToDevice, st));
    c->launches += 4;
    int bad = none;
    CU(cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(&g.pmem.crc, d_state, sizeof g.pmem.crc, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (bad != none) r->status = GU_INVALID;
    g.pmem.len += r->plain;
    return CG_OK;
}

static uint32_t gzin_le32(const uint8_t *p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }

// A split stream's submission: whole members through the chain, a long member (or the rest of one) through the block
// path, then the chain again behind it, until the bytes run out or a member stops inside.
static int gzin_inflate_split(cg_ctx *c, GzinStream &g, const uint8_t *gz, long long n, int n_cand, bool final,
                              cudaStream_t st, cg_gzin_result *res, bool *fin)
{
    int rc;
    GzinStream::Member &m = g.pmem;
    std::vector<int32_t> hcand;                  // the candidates and their parses, read back for gu_member_bound
    std::vector<GuMember> hres;
    const auto bound = [&](long long at, long long *b) {
        if (n_cand && hcand.empty()) {
            hcand.resize(n_cand);
            hres.resize(n_cand);
            CU(cudaMemcpyAsync(hcand.data(), g.d_cand.p, n_cand * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
            CU(cudaMemcpyAsync(hres.data(), g.d_res.p, n_cand * sizeof(GuMember), cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
        }
        *b = gu_member_bound(hcand.data(), hres.data(), n_cand, at, n);
        return CG_OK;
    };
    m = g.mem;
    long long p = 0, base = g.carry, members = 0, respec = 0;
    bool after = g.members > 0;
    const auto bad_member = [&]() {
        return fail(CG_EINVAL, "gzip input: invalid or truncated gzip member at byte " + std::to_string(m.start) +
                                   " of the compressed file");
    };
    for (;;) {
        if (m.in && m.trailer) {
            const long long t = p + (m.bitoff ? 1 : 0);
            if (t + 8 > n) {
                if (final) return bad_member();
                break;
            }
            if (gzin_le32(gz + t) != ~m.crc || gzin_le32(gz + t + 4) != (uint32_t)m.len)
                return fail(CG_EINVAL, "gzip input: CRC-32 mismatch in the gzip member at byte " + std::to_string(m.start) +
                                           " of the compressed file");
            p = t + 8;
            m = GzinStream::Member();
            members += 1;
            after = true;
            continue;
        }
        if (m.in) {
            GuWalk r;
            long long b;
            if ((rc = bound(p, &b)) != CG_OK) return rc;
            if ((rc = gzin_blocks(c, g, n, b, p * 8 + m.bitoff, base, st, &r, &respec)) != CG_OK) return rc;
            if (r.status == GU_INVALID) return bad_member();
            if (r.status == GU_UNSUPPORTED) {
                if (base == g.carry && p == 0 && !members)
                    return fail(CG_EUNSUPPORTED, "gzip input: a stretch of deflate blocks of the member at byte " +
                                                     std::to_string(m.start) +
                                                     " inflates to more than one submission can hold (2 GiB); "
                                                     "decompress this input on the host");
                break;
            }
            base += r.plain;
            p = r.end >> 3;
            m.bitoff = (int)(r.end & 7);
            if (r.last) {
                m.trailer = 1;
                continue;
            }
            if (r.more && final) return bad_member();
            break;
        }
        GuChain ch;
        if ((rc = gzin_members(c, g, n, n_cand, p, after, final, base, true, st, &ch)) != CG_OK) return rc;
        if (ch.status == GU_UNSUPPORTED) {
            if (base == g.carry && p == 0 && !members)
                return fail(CG_EUNSUPPORTED, "gzip input: the member at byte " + std::to_string(g.consumed + ch.err_at) +
                                                 " inflates to more than one submission can hold (2 GiB); decompress "
                                                 "this input on the host");
        }
        base += ch.plain;
        members += ch.n_members;
        after = after || ch.n_members > 0;
        p = ch.consumed;
        if (ch.status != GU_LONG) break;
        m.in = 1;
        m.crc = 0xffffffffu;
        m.start = g.consumed + ch.err_at;
        p = ch.err_at + gu_head(gz + ch.err_at, n - ch.err_at);
    }
    g.pend_plain = base - g.carry;
    g.pend_consumed = p;
    g.pend_members = members;
    g.pend_respec = respec;
    res->consumed = p;
    res->members = members;
    res->plain_bytes = base - g.carry;
    res->in_member = m.in;
    res->respeculated = respec;
    *fin = final && p == n && !m.in;
    return CG_OK;
}

// Upload gz[0, n), inflate the chain of whole members behind the carry (not committed yet).  *fin: final and every byte
// consumed.
static int gzin_inflate(cg_ctx *c, GzinStream &g, const uint8_t *gz, int64_t n, bool final, cudaStream_t st,
                        cg_gzin_result *res, bool *fin)
{
    int rc;
    CU(cudaStreamWaitEvent(st, g.done, 0));
    if ((rc = g.d_gz.ensure((size_t)n + 16)) != CG_OK) return rc;
    if (n) {
        if ((rc = g.h_gz.ensure((size_t)n)) != CG_OK) return rc;
        parallel_copy(c, g.h_gz.p, gz, (size_t)n);
        CU(cudaMemcpyAsync(g.d_gz.p, g.h_gz.p, (size_t)n, cudaMemcpyHostToDevice, st));
        c->h2d_bytes += n;
    }
    const long long tiles = cg_gunzip_tiles(n);
    if ((rc = g.d_counts.ensure((size_t)tiles + 1)) != CG_OK) return rc;
    if ((rc = g.d_offs.ensure((size_t)tiles + 1)) != CG_OK) return rc;
    if ((rc = g.d_scan.ensure((size_t)cg_scan_tiles(tiles) + 1)) != CG_OK) return rc;
    int64_t n_cand = 0;
    if (tiles) {
        CU(cg_launch_gunzip_candidates(0, g.d_gz.p, n, g.d_counts.p, nullptr, nullptr, st));
        CU(cg_launch_scan_i32(g.d_counts.p, tiles, g.d_scan.p, g.d_offs.p, st));
        CU(cudaMemcpyAsync(&n_cand, g.d_offs.p + tiles, sizeof n_cand, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        c->launches += 3;
    }
    if ((rc = g.d_cand.ensure((size_t)n_cand + 1)) != CG_OK) return rc;
    if ((rc = g.d_res.ensure((size_t)n_cand + 1)) != CG_OK) return rc;
    if ((rc = g.d_members.ensure((size_t)n_cand + 1)) != CG_OK) return rc;
    if ((rc = g.d_moff.ensure((size_t)n_cand + 1)) != CG_OK) return rc;
    if (n_cand) {
        CU(cg_launch_gunzip_candidates(1, g.d_gz.p, n, nullptr, g.d_offs.p, g.d_cand.p, st));
        CU(cg_launch_gunzip_parse(g.d_gz.p, n, g.d_cand.p, (int)n_cand, g.split ? CG_GZIN_LONG_MEMBER : 0, g.d_res.p, st));
        c->launches += 2;
    }
    if (g.split) return gzin_inflate_split(c, g, gz, n, (int)n_cand, final, st, res, fin);
    GuChain ch;
    if ((rc = gzin_members(c, g, n, (int)n_cand, 0, g.members > 0, final, g.carry, false, st, &ch)) != CG_OK) return rc;
    g.pend_plain = ch.plain;
    g.pend_consumed = ch.consumed;
    g.pend_members = ch.n_members;
    res->consumed = ch.consumed;
    res->members = ch.n_members;
    res->plain_bytes = ch.plain;
    *fin = final && ch.consumed == n;
    return CG_OK;
}

// The flagged newlines of the carry plus the new plain bytes (gu_flag): their number *F, whether the buffer starts
// with '>', whether it ends in a newline; the line index and the flags' scan stay in g for gzin_cut.
struct GzinCount {
    long long total = 0, n_nl = 0, F = 0;
    int b0 = 0, nl_end = 1, fasta = 0;
};

static int gzin_count(cg_ctx *c, GzinStream &g, int fasta, cudaStream_t st, GzinCount *k)
{
    k->total = g.carry + g.pend_plain;
    k->fasta = fasta;
    if (!k->total) return CG_OK;
    int rc;
    if ((rc = g.d_tiles.ensure((size_t)cg_fastq_tiles(k->total) + 1)) != CG_OK) return rc;
    CU(cg_launch_fastq_index(g.d_plain.p, k->total, g.d_tiles.p, g.d_small.p, nullptr, 0, st));
    uint8_t ends[2];
    CU(cudaMemcpyAsync(&k->n_nl, g.d_small.p, sizeof k->n_nl, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(&ends[0], g.d_plain.p, 1, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(&ends[1], g.d_plain.p + k->total - 1, 1, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches += 2;
    k->b0 = ends[0] == '>';
    k->nl_end = ends[1] == '\n';
    const long long L = k->n_nl;
    if (!L) return CG_OK;
    if ((rc = g.d_nl.ensure((size_t)L + 1)) != CG_OK) return rc;
    if ((rc = g.d_flag.ensure((size_t)L + 1)) != CG_OK) return rc;
    if ((rc = g.d_offs.ensure((size_t)L + 1)) != CG_OK) return rc;
    if ((rc = g.d_scan.ensure((size_t)cg_scan_tiles(L) + 1)) != CG_OK) return rc;
    CU(cg_launch_fastq_index(g.d_plain.p, k->total, g.d_tiles.p, nullptr, g.d_nl.p, 1, st));
    CU(cg_launch_gunzip_flags(g.d_plain.p, k->total, g.d_nl.p, L, fasta, g.d_flag.p, st));
    CU(cg_launch_scan_i32(g.d_flag.p, L, g.d_scan.p, g.d_offs.p, st));
    CU(cudaMemcpyAsync(&k->F, g.d_offs.p + L, sizeof k->F, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches += 4;
    return CG_OK;
}

// the offset behind flagged newline s (s < 0: 0); *n_records: the records in front of it
static int gzin_cut(cg_ctx *c, GzinStream &g, const GzinCount &k, long long s, cudaStream_t st, long long *cut,
                    long long *n_records)
{
    *cut = 0;
    *n_records = 0;
    if (s < 0) return CG_OK;
    long long *d_cut = reinterpret_cast<long long *>(g.d_small.p + 1);
    CU(cg_launch_gunzip_select(g.d_nl.p, k.n_nl, g.d_flag.p, g.d_offs.p, s, d_cut, st));
    CU(cudaMemcpyAsync(cut, d_cut, sizeof *cut, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches += 1;
    *n_records = k.fasta ? k.b0 + s : (s + 1) / 4;
    return CG_OK;
}

// final: the whole buffer is the chunk
static void gzin_all(const GzinCount &k, long long *cut, long long *n_records)
{
    *cut = k.total;
    *n_records = k.fasta ? k.b0 + k.F : (k.n_nl + (k.total && !k.nl_end ? 1 : 0)) / 4;
}

// Commit the submission: the chunk [0, cut) goes to slot f (f == nullptr: cut must be 0), the rest becomes the carry.
// The slot takes the stream's buffer; the rest is copied into the slot's old one, which the stream keeps.
static int gzin_commit(cg_ctx *c, GzinStream &g, FastqSlot *f, long long cut, long long n_records, cudaStream_t st,
                       cg_gzin_result *res)
{
    const long long total = g.carry + g.pend_plain;
    int rc;
    if (f && cut) {
        std::swap(g.d_plain, f->d_in);
        const long long rest = total - cut;
        if ((rc = g.d_plain.ensure((size_t)rest + 64)) != CG_OK) return rc;
        if (rest) CU(cudaMemcpyAsync(g.d_plain.p, f->d_in.p + cut, (size_t)rest, cudaMemcpyDeviceToDevice, st));
        if ((rc = fastq_slot_count(c, *f, cut)) != CG_OK) return rc;
        g.carry = rest;
    } else {
        g.carry = total;
    }
    g.consumed += g.pend_consumed;
    g.members += g.pend_members;
    g.pend_plain = g.pend_consumed = g.pend_members = 0;
    if (g.bam < 0) g.bam = 0;
    if (g.split) {
        g.mem = g.pmem;
        if (g.mem.in) std::swap(g.d_win, g.d_pwin);
    }
    CU(cudaEventRecord(g.done, st));
    res->chunk_bytes = f ? cut : 0;
    res->carry_bytes = g.carry;
    res->n_records = f ? n_records : 0;
    return CG_OK;
}

static GzinStream *gzin_lookup(cg_ctx *c, int32_t handle)
{
    auto it = c->gzin.find(handle);
    return it == c->gzin.end() ? nullptr : &it->second;
}

// A stream keeps the format class (BAM or not) of its first committed submission
static int gzin_format_check(const GzinStream &g, int32_t format, const char *who)
{
    const int bam = format == CG_FORMAT_BAM;
    if (g.bam >= 0 && g.bam != bam)
        return fail(CG_EINVAL, std::string(who) + ": the stream was " + (g.bam ? "BAM" : "FASTQ / FASTA") +
                                   " input; a stream takes one format for its whole life");
    return CG_OK;
}

// ------------------------------------------------------------------------------------------
// BAM input (CG_FORMAT_BAM, cg_bam.cu): the inflated bytes behind the carry are the BAM stream.  The header is parsed on
// the host from a readback of its bytes and dropped once whole; the record boundaries come from the tile walk, and the
// records of the cut are written as FASTQ text into the slot.  The BAM bytes behind the cut become the carry.
// ------------------------------------------------------------------------------------------
static int bam_fail(int code, long long record, long long at, const std::string &what)
{
    return fail(code, "BAM input: record " + std::to_string(record) + " (at byte " + std::to_string(at) +
                          " of the decompressed stream): " + what);
}

// The header of d_plain[0, total) on the host: *hdr its size once whole (0 while it is not and not final).
static int bam_header_read(GzinStream &g, long long total, bool final, cudaStream_t st, long long *hdr)
{
    *hdr = 0;
    std::vector<uint8_t> h;
    for (long long want = 65536;; want *= 2) {
        const long long m = std::min(want, total);
        h.resize((size_t)m);
        if (m) CU(cudaMemcpyAsync(h.data(), g.d_plain.p, (size_t)m, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        int why = 0;
        const int s = bam_header(h.data(), m, hdr, &why);
        if (s == BAM_BAD)
            return fail(CG_EINVAL, why == BAM_H_MAGIC ? "BAM input: not a BAM file (the decompressed stream does not "
                                                        "start with BAM\\1)"
                                                      : "BAM input: not a BAM file (a negative length in the header)");
        if (s == BAM_OK) return CG_OK;
        if (m == total) break;
    }
    *hdr = 0;
    if (final) return fail(CG_EINVAL, "BAM input: the file ends inside the BAM header");
    return CG_OK;
}

static const char *bam_what(int code)
{
    switch (code) {
    case BAM_R_FLAG: return "flag is not 4 (an unmapped single read); only unaligned single-end BAM is read";
    case BAM_R_NAME: return "a read name byte outside '!'..'~'";
    case BAM_R_NOQUAL: return "the record has no quality values (first quality byte 0xFF)";
    case BAM_R_QUAL: return "a quality value above 93";
    default: return "block_size, l_read_name, n_cigar_op and l_seq do not fit together, or the name lacks its NUL";
    }
}

// The BAM submission after gzin_inflate: cut, emit into slot f, commit.  *cut_bytes: the FASTQ bytes in the slot.
static int gzin_bam(cg_ctx *c, GzinStream &g, FastqSlot &f, bool fin, cudaStream_t st, cg_gzin_result *res,
                    long long *cut_bytes)
{
    int rc;
    *cut_bytes = 0;
    const long long total = g.carry + g.pend_plain;
    long long s0 = 0;                          // header bytes in front of the records
    if (!g.bam_hdr) {
        if ((rc = bam_header_read(g, total, fin, st, &s0)) != CG_OK) return rc;
        if (!s0) {                             // the header waits in the carry
            g.carry = total;
            g.consumed += g.pend_consumed;
            g.members += g.pend_members;
            g.pend_plain = g.pend_consumed = g.pend_members = 0;
            g.bam = 1;
            if (g.split) {
                g.mem = g.pmem;
                if (g.mem.in) std::swap(g.d_win, g.d_pwin);
            }
            CU(cudaEventRecord(g.done, st));
            res->carry_bytes = g.carry;
            return CG_OK;
        }
    }
    const uint8_t *b = g.d_plain.p + s0;
    const long long n = total - s0, T = cg_bam_tiles(n), W = cg_bam_words(n), R = cg_bam_max_records(n);
    if ((rc = g.d_bm.ensure((size_t)W + 1)) != CG_OK || (rc = g.d_link.ensure((size_t)T + 1)) != CG_OK ||
        (rc = g.d_entry.ensure((size_t)T + 1)) != CG_OK || (rc = g.d_wcnt.ensure((size_t)W + 1)) != CG_OK ||
        (rc = g.d_woff.ensure((size_t)W + 1)) != CG_OK || (rc = g.d_start.ensure((size_t)R)) != CG_OK ||
        (rc = g.d_fsize.ensure((size_t)R)) != CG_OK || (rc = g.d_foff.ensure((size_t)R + 1)) != CG_OK ||
        (rc = g.d_sum.ensure(1)) != CG_OK || (rc = g.d_berr.ensure(1)) != CG_OK ||
        (rc = g.d_scan.ensure((size_t)cg_scan_tiles(std::max(W, R)) + 1)) != CG_OK)
        return rc;
    CU(cg_launch_bam_bounds(b, n, g.d_bm.p, g.d_link.p, g.d_entry.p, g.d_sum.p, g.d_wcnt.p, st));
    CU(cg_launch_scan_i32(g.d_wcnt.p, W, g.d_scan.p, g.d_woff.p, st));
    CU(cg_launch_bam_starts(b, n, g.d_bm.p, g.d_entry.p, g.d_sum.p, g.d_woff.p, g.d_start.p, g.d_fsize.p, st));
    CU(cg_launch_scan_i32(g.d_fsize.p, R, g.d_scan.p, g.d_foff.p, st));
    CU(cg_launch_bam_cut(g.d_woff.p, n, g.d_start.p, g.d_foff.p, CG_GZIN_LIMIT - 1, g.d_sum.p, st));
    c->launches += 12;
    BamSum sum;
    CU(cudaMemcpyAsync(&sum, g.d_sum.p, sizeof sum, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    // the refusals of every record of the chain, the text of the cut's
    if ((rc = f.d_in.ensure((size_t)sum.fq_bytes + 64)) != CG_OK) return rc;
    const unsigned long long none = ~0ULL;
    CU(cudaMemcpyAsync(g.d_berr.p, &none, sizeof none, cudaMemcpyHostToDevice, st));
    CU(cg_launch_bam_emit(b, g.d_start.p, g.d_foff.p, sum.n_rec, sum.n_cut, f.d_in.p, g.d_berr.p, st));
    c->launches += 1;
    unsigned long long err = none;
    CU(cudaMemcpyAsync(&err, g.d_berr.p, sizeof err, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const long long at0 = g.bam_base + s0;
    if (err != none) {
        const long long i = (long long)(err >> 3);
        const int code = (int)(err & 7);
        uint32_t p = 0;
        CU(cudaMemcpy(&p, g.d_start.p + i, sizeof p, cudaMemcpyDeviceToHost));
        return bam_fail(code == BAM_R_FLAG || code == BAM_R_NOQUAL ? CG_EUNSUPPORTED : CG_EINVAL, g.bam_records + i,
                        at0 + p, bam_what(code));
    }
    if (sum.end_st == BAM_BAD)
        return bam_fail(CG_EINVAL, g.bam_records + sum.n_rec, at0 + sum.end, bam_what(BAM_R_STRUCT));
    if (sum.end_st == BAM_SHORT && fin)
        return fail(CG_EINVAL, "BAM input: BAM file ends inside record " + std::to_string(g.bam_records + sum.n_rec) +
                                   " (at byte " + std::to_string(at0 + sum.end) + " of the decompressed stream)");
    if (sum.n_cut == 0 && sum.n_rec > 0)
        return bam_fail(CG_EUNSUPPORTED, g.bam_records, at0,
                        "its FASTQ text alone reaches the 2 GiB limit of a chunk");
    // commit: the BAM bytes behind the cut become the carry
    const long long drop = s0 + sum.bam_cut, rest = total - drop;
    if (drop) {
        if ((rc = g.d_rest.ensure((size_t)rest + 64)) != CG_OK) return rc;
        if (rest) CU(cudaMemcpyAsync(g.d_rest.p, g.d_plain.p + drop, (size_t)rest, cudaMemcpyDeviceToDevice, st));
        std::swap(g.d_rest, g.d_plain);
    }
    if (sum.n_cut && (rc = fastq_slot_count(c, f, sum.fq_bytes)) != CG_OK) return rc;
    g.bam_hdr = true;
    g.bam_base += drop;
    g.bam_records += sum.n_cut;
    g.bam_tiles += T;
    g.bam_rewalked += sum.rewalked;
    g.carry = rest;
    g.consumed += g.pend_consumed;
    g.members += g.pend_members;
    g.pend_plain = g.pend_consumed = g.pend_members = 0;
    g.bam = 1;
    if (g.split) {
        g.mem = g.pmem;
        if (g.mem.in) std::swap(g.d_win, g.d_pwin);
    }
    CU(cudaEventRecord(g.done, st));
    res->chunk_bytes = sum.n_cut ? sum.fq_bytes : 0;
    res->carry_bytes = g.carry;
    res->n_records = sum.n_cut;
    *cut_bytes = res->chunk_bytes;
    return CG_OK;
}

extern "C" int cg_gzin_bam_tiles(cg_ctx *c, int32_t handle, int64_t *tiles, int64_t *rewalked)
{
    if (!c || !tiles || !rewalked) return fail(CG_EINVAL, "cg_gzin_bam_tiles: bad argument");
    GzinStream *g = gzin_lookup(c, handle);
    if (!g) return fail(CG_EINVAL, "cg_gzin_bam_tiles: unknown handle");
    *tiles = g->bam_tiles;
    *rewalked = g->bam_rewalked;
    return CG_OK;
}

extern "C" int cg_fastq_submit_gzip(cg_ctx *c, int32_t handle, const uint8_t *gz, int64_t n_bytes, int32_t format,
                                    int32_t final, int32_t *slot, cg_gzin_result *res)
{
    int rc = submit_check("cg_fastq_submit_gzip", c && slot && res, format, "submission", gz, n_bytes, nullptr, 0,
                          CG_FORMAT_BAM);
    if (rc != CG_OK) return rc;
    GzinStream *g = gzin_lookup(c, handle);
    if (!g) return fail(CG_EINVAL, "cg_fastq_submit_gzip: unknown handle");
    if ((rc = gzin_format_check(*g, format, "cg_fastq_submit_gzip")) != CG_OK) return rc;
    CU(cudaSetDevice(c->device));
    *slot = -1;
    memset(res, 0, sizeof *res);
    int si;
    if ((rc = fq_find(c, 1, "cg_fastq_submit_gzip: all slots are in flight, collect one first", &si)) != CG_OK) return rc;
    FastqSlot &f = c->fq[si];
    bool fin = false;
    if ((rc = fastq_slot_init(c, f)) != CG_OK) return rc;
    if ((rc = gzin_inflate(c, *g, gz, n_bytes, final != 0, f.stream, res, &fin)) != CG_OK) return rc;
    if (format == CG_FORMAT_BAM) {
        long long cut = 0;
        if ((rc = gzin_bam(c, *g, f, fin, f.stream, res, &cut)) != CG_OK) return rc;
        if (cut) fq_take(c, si, slot);
        return CG_OK;
    }
    GzinCount k;
    if ((rc = gzin_count(c, *g, format == CG_FORMAT_FASTA, f.stream, &k)) != CG_OK) return rc;
    long long cut, n_records;
    if (fin) gzin_all(k, &cut, &n_records);
    else if ((rc = gzin_cut(c, *g, k, gu_select_single(k.fasta, k.F, k.b0, 0), f.stream, &cut, &n_records)) != CG_OK)
        return rc;
    if ((rc = gzin_commit(c, *g, cut ? &f : nullptr, cut, n_records, f.stream, res)) != CG_OK) return rc;
    if (cut) fq_take(c, si, slot);
    return CG_OK;
}

extern "C" int cg_fastq_slot_read(cg_ctx *c, int32_t slot, uint8_t *dst, int64_t capacity, int64_t *n_bytes)
{
    if (!c || !n_bytes || slot < 0 || slot >= CG_FQ_SLOTS || capacity < 0 || (capacity && !dst))
        return fail(CG_EINVAL, "cg_fastq_slot_read: bad argument");
    FastqSlot &f = c->fq[slot];
    // the first slot of an interleaved chunk holds the whole chunk until the collect splits it; the second holds none
    if (!f.busy || f.ilv == 2) return fail(CG_EINVAL, "cg_fastq_slot_read: the slot holds no chunk of its own");
    CU(cudaSetDevice(c->device));
    *n_bytes = f.n_bytes;
    if (capacity < f.n_bytes) return fail(CG_EINVAL, "cg_fastq_slot_read: buffer too small");
    if (f.n_bytes) CU(cudaMemcpyAsync(dst, f.d_in.p, (size_t)f.n_bytes, cudaMemcpyDeviceToHost, f.stream));
    CU(cudaStreamSynchronize(f.stream));
    c->d2h_bytes += f.n_bytes;
    return CG_OK;
}

extern "C" int cg_fastq_submit_gzip_interleaved(cg_ctx *c, int32_t handle, const uint8_t *gz, int64_t n_bytes,
                                                int32_t format, int32_t final, int32_t *slot1, int32_t *slot2,
                                                cg_gzin_result *res)
{
    int rc = submit_check("cg_fastq_submit_gzip_interleaved", c && slot1 && slot2 && res, format, "submission", gz, n_bytes);
    if (rc != CG_OK) return rc;
    GzinStream *g = gzin_lookup(c, handle);
    if (!g) return fail(CG_EINVAL, "cg_fastq_submit_gzip_interleaved: unknown handle");
    if ((rc = gzin_format_check(*g, format, "cg_fastq_submit_gzip_interleaved")) != CG_OK) return rc;
    CU(cudaSetDevice(c->device));
    *slot1 = *slot2 = -1;
    memset(res, 0, sizeof *res);
    int s1;
    if ((rc = fq_find(c, 2, "cg_fastq_submit_gzip_interleaved: two free slots are needed, collect one first", &s1)) != CG_OK)
        return rc;
    FastqSlot &f1 = c->fq[s1], &f2 = c->fq[(s1 + 1) % CG_FQ_SLOTS];
    bool fin = false;
    if ((rc = fastq_slot_init(c, f1)) != CG_OK) return rc;
    if ((rc = gzin_inflate(c, *g, gz, n_bytes, final != 0, f1.stream, res, &fin)) != CG_OK) return rc;
    GzinCount k;
    if ((rc = gzin_count(c, *g, format == CG_FORMAT_FASTA, f1.stream, &k)) != CG_OK) return rc;
    long long cut, n_records;
    if (fin) gzin_all(k, &cut, &n_records);
    else if ((rc = gzin_cut(c, *g, k, gu_select_single(k.fasta, k.F, k.b0, 1), f1.stream, &cut, &n_records)) != CG_OK)
        return rc;
    if ((rc = gzin_commit(c, *g, cut ? &f1 : nullptr, cut, n_records, f1.stream, res)) != CG_OK) return rc;
    if (!cut) return CG_OK;
    if ((rc = fastq_slot_init(c, f2)) != CG_OK) return rc;          // its chunk comes from the split
    if ((rc = fastq_slot_count(c, f2, 0)) != CG_OK) return rc;
    fq_take(c, s1, slot1, slot2, format);
    return CG_OK;
}

extern "C" int cg_fastq_submit_gzip_paired(cg_ctx *c, int32_t handle1, int32_t handle2, const uint8_t *gz1,
                                           int64_t n_bytes1, const uint8_t *gz2, int64_t n_bytes2, int32_t format,
                                           int32_t final, int32_t *slot1, int32_t *slot2, cg_gzin_result *res1,
                                           cg_gzin_result *res2)
{
    int rc = submit_check("cg_fastq_submit_gzip_paired", c && slot1 && slot2 && res1 && res2 && handle1 != handle2, format,
                          "submission", gz1, n_bytes1, gz2, n_bytes2);
    if (rc != CG_OK) return rc;
    GzinStream *g1 = gzin_lookup(c, handle1), *g2 = gzin_lookup(c, handle2);
    if (!g1 || !g2) return fail(CG_EINVAL, "cg_fastq_submit_gzip_paired: unknown handle");
    if ((rc = gzin_format_check(*g1, format, "cg_fastq_submit_gzip_paired")) != CG_OK ||
        (rc = gzin_format_check(*g2, format, "cg_fastq_submit_gzip_paired")) != CG_OK)
        return rc;
    CU(cudaSetDevice(c->device));
    *slot1 = *slot2 = -1;
    memset(res1, 0, sizeof *res1);
    memset(res2, 0, sizeof *res2);
    int s1;
    if ((rc = fq_find(c, 2, "cg_fastq_submit_gzip_paired: two free slots are needed, collect one first", &s1)) != CG_OK)
        return rc;
    FastqSlot &f1 = c->fq[s1], &f2 = c->fq[(s1 + 1) % CG_FQ_SLOTS];
    bool fin1 = false, fin2 = false;
    if ((rc = fastq_slot_init(c, f1)) != CG_OK) return rc;
    if ((rc = fastq_slot_init(c, f2)) != CG_OK) return rc;
    if ((rc = gzin_inflate(c, *g1, gz1, n_bytes1, final != 0, f1.stream, res1, &fin1)) != CG_OK)
        return fail(rc, "mate 1 (first input): " + g_err);
    if ((rc = gzin_inflate(c, *g2, gz2, n_bytes2, final != 0, f2.stream, res2, &fin2)) != CG_OK)
        return fail(rc, "mate 2 (second input): " + g_err);
    const int fasta = format == CG_FORMAT_FASTA;
    GzinCount k1, k2;
    if ((rc = gzin_count(c, *g1, fasta, f1.stream, &k1)) != CG_OK) return rc;
    if ((rc = gzin_count(c, *g2, fasta, f2.stream, &k2)) != CG_OK) return rc;
    long long cut1, cut2, n1, n2;
    if (fin1 && fin2) {
        gzin_all(k1, &cut1, &n1);
        gzin_all(k2, &cut2, &n2);
    } else {
        const long long r = std::min(gu_records(fasta, k1.F, k1.b0), gu_records(fasta, k2.F, k2.b0));
        const long long sel1 = r > 0 ? gu_select_records(fasta, r, k1.b0) : -1;
        const long long sel2 = r > 0 ? gu_select_records(fasta, r, k2.b0) : -1;
        if ((rc = gzin_cut(c, *g1, k1, sel1, f1.stream, &cut1, &n1)) != CG_OK) return rc;
        if ((rc = gzin_cut(c, *g2, k2, sel2, f2.stream, &cut2, &n2)) != CG_OK) return rc;
    }
    const bool take = cut1 || cut2;
    if ((rc = gzin_commit(c, *g1, take ? &f1 : nullptr, cut1, n1, f1.stream, res1)) != CG_OK) return rc;
    if ((rc = gzin_commit(c, *g2, take ? &f2 : nullptr, cut2, n2, f2.stream, res2)) != CG_OK) return rc;
    if (!take) return CG_OK;
    // a mate without bytes (the other file's last records) gets an empty chunk
    if (!cut1 && (rc = fastq_slot_count(c, f1, 0)) != CG_OK) return rc;
    if (!cut2 && (rc = fastq_slot_count(c, f2, 0)) != CG_OK) return rc;
    fq_take(c, s1, slot1, slot2);
    return CG_OK;
}

// One mate of a chunk between submit and the verdict
struct FqStage {
    long long n = 0, n_nl = 0;
    int times = 1, slots = 1;
    int32_t *d_qtrim = nullptr;
    const cg_match_rec *d_matches = nullptr;
    int action = 0;
    bool want_q = false;                 // quality trimming still to be done by the trimming kernels
    int max_len = 0;                     // longest packed read
    const uint8_t *d_is_rc = nullptr;    // --revcomp: the record was replaced by its reverse complement
    int rc_suffix = 0;                   // ... and gets " rc" appended to its name
    int format = CG_FORMAT_FASTQ;        // cg_fastq_params.format
    bool packed = false;                 // d_offs / d_seq / max_len hold this mate's reads
    FqStatsAcc *acc = nullptr;           // statistics on: the accumulator of this mate ...
    int st_len = 0, st_kmax = 0;         // ... and the layout of the chunk's vector in d_fqstats
    bool st_poly_a = false;              // d_polya was filled
    int zero_cap = 0;                    // ZeroCapper: the quality base the written qualities are capped at, 0 = off
    bool has_qual() const { return format != CG_FORMAT_FASTA; }
    bool fasta_out() const { return format != CG_FORMAT_FASTQ; }
};

static int fastq_enabled_filters(const cg_fastq_params *fp)
{
    return (fp->minimum_length > 0 ? 1 : 0) | (fp->maximum_length >= 0 ? 2 : 0) | (fp->max_n >= 0.0 ? 4 : 0) |
           (fp->max_expected_errors >= 0.0 ? 8 : 0) | (fp->discard_casava ? 16 : 0) | (fp->discard_trimmed ? 32 : 0) |
           (fp->discard_untrimmed ? 64 : 0) | (fp->max_average_error_rate > 0.0 ? 128 : 0);
}

// FASTA chunk (format 1) -> normalised chunk in f.d_in + record table: line classes, two scans, scatter, records.
// Returns the number of records in *n_records; reports a format error naming the first bad line.
static int fasta_stage_normalise(cg_ctx *c, FastqSlot &f, const cg_fastq_params *fp, long long n_lines, cudaStream_t st,
                                 FqStage &g, long long *n_records)
{
    *n_records = 0;
    const int64_t n_bytes = f.n_bytes;
    int rc;
    if ((rc = f.d_nl.ensure((size_t)g.n_nl + 1)) != CG_OK) return rc;
    if ((rc = f.d_faline.ensure((size_t)n_lines * 2 + 1)) != CG_OK) return rc;
    if ((rc = f.d_faoff.ensure((size_t)n_lines * 2 + 2)) != CG_OK) return rc;
    if ((rc = f.d_scan.ensure((size_t)cg_scan_tiles(n_lines) + 1)) != CG_OK) return rc;
    int32_t *d_keep = f.d_faline.p, *d_hdr = f.d_faline.p + n_lines, *d_first = f.d_faline.p + 2 * n_lines;
    int64_t *d_off = f.d_faoff.p, *d_idx = f.d_faoff.p + n_lines + 1;
    const int first_init = 0x7FFFFFFF;
    CU(cudaMemcpyAsync(d_first, &first_init, sizeof first_init, cudaMemcpyHostToDevice, st));
    CU(cg_launch_fastq_index(f.d_in.p, n_bytes, f.d_tiles.p, nullptr, f.d_nl.p, 1, st));
    CU(cg_launch_fasta_classify(f.d_in.p, n_bytes, f.d_nl.p, g.n_nl, n_lines, d_keep, d_hdr, d_first, st));
    CU(cg_launch_scan_i32(d_keep, n_lines, f.d_scan.p, d_off, st));
    CU(cg_launch_scan_i32(d_hdr, n_lines, f.d_scan.p, d_idx, st));
    c->launches += 8;
    int64_t sizes[2];                           // bytes of the normalised chunk, records
    CU(cudaMemcpyAsync(&sizes[0], d_off + n_lines, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(&sizes[1], d_idx + n_lines, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const long long n_norm = sizes[0], n = sizes[1];
    if ((rc = f.d_norm.ensure((size_t)n_norm + 64)) != CG_OK) return rc;
    if ((rc = f.d_rec.ensure((size_t)n + 1)) != CG_OK) return rc;
    if ((rc = f.d_len.ensure((size_t)n + 1)) != CG_OK) return rc;
    if ((rc = f.d_origin.ensure((size_t)n * 2 + 2)) != CG_OK) return rc;
    CU(cg_launch_fasta_scatter(f.d_in.p, n_bytes, f.d_nl.p, g.n_nl, n_lines, d_off, d_idx, d_first, f.d_norm.p, f.d_rec.p,
                               f.d_err.p, st));
    CU(cg_launch_fasta_records(f.d_rec.p, n, n_norm, fp->cut_front, fp->cut_back, f.d_len.p, f.d_origin.p, f.d_counters.p + 1,
                               st));
    c->launches += 2;
    int fa_err[2];
    CU(cudaMemcpyAsync(fa_err, f.d_err.p, sizeof fa_err, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (fa_err[0]) return fastq_format_error(fa_err);
    std::swap(f.d_in, f.d_norm);                // every later kernel reads the normalised chunk
    f.n_bytes = n_norm;
    *n_records = n;
    return CG_OK;
}

// The demultiplexer's stable byte partition: record r has d_len[r] bytes (0: none) for destination d_dest[r].  f.d_outoff
// receives every record's offset; segments (host, n_dest + 1 values) where each destination starts and *total the sum,
// both once the stream has got there.
static int fastq_partition(cg_ctx *c, FastqSlot &f, long long n, int n_dest, const int32_t *d_len, const int32_t *d_dest,
                           int64_t *segments, long long *total, cudaStream_t st)
{
    const long long tiles = cg_demux_tiles(n), cells = tiles * n_dest;
    int rc;
    if ((rc = f.d_dmbytes.ensure((size_t)cells)) != CG_OK) return rc;
    if ((rc = f.d_dmbase.ensure((size_t)cells + 1)) != CG_OK) return rc;
    if ((rc = f.d_scan.ensure((size_t)cg_scan_tiles(cells) + 1)) != CG_OK) return rc;
    CU(cg_launch_fastq_demux(0, d_len, d_dest, n, n_dest, f.d_dmbytes.p, nullptr, nullptr, st));
    CU(cg_launch_scan_i32(f.d_dmbytes.p, cells, f.d_scan.p, f.d_dmbase.p, st));
    CU(cg_launch_fastq_demux(1, d_len, d_dest, n, n_dest, nullptr, f.d_dmbase.p, f.d_outoff.p, st));
    c->launches += 5;
    // segment d starts at base[d][tile 0]; the last entry is the total
    CU(cudaMemcpy2DAsync(segments, sizeof(int64_t), f.d_dmbase.p, (size_t)tiles * sizeof(int64_t), sizeof(int64_t),
                         (size_t)n_dest, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(segments + n_dest, f.d_dmbase.p + cells, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(total, f.d_dmbase.p + cells, sizeof *total, cudaMemcpyDeviceToHost, st));
    return CG_OK;
}

// Interleaved input (cg_fastq_submit_interleaved): the chunk uploaded to f1 becomes two mate chunks, f1 and f2, as if
// each had been submitted.  FASTQ: records are 4 lines of the line index; FASTA: the chunk is normalised first (format
// errors name lines of the chunk), its records are ">name\n" + sequence.  Per record its span, mate (r & 1) and name
// (ilv_records_kernel, which also checks the FASTQ format), the mate-name check per pair (ilv_pairs_kernel), the
// demultiplexer's partition of the record sizes by mate, one copy kernel into the two slots; then every slot's newline
// count, as cg_fastq_submit leaves it.  Runs on f1's stream; the scratch buffers are f1's per-record buffers, which the
// collect sizes anew.
static int fastq_split_interleaved(cg_ctx *c, FastqSlot &f1, FastqSlot &f2, cudaStream_t st)
{
    CU(cudaStreamSynchronize(f2.stream));
    CU(cudaStreamSynchronize(st));              // upload + newline count of the chunk
    const bool fasta = f1.ilv_format == CG_FORMAT_FASTA;
    FqStage g;
    g.n_nl = (long long)f1.h_counters.p[0];
    long long n_lines = g.n_nl;                 // the last line may come without its newline
    if (f1.n_bytes > 0) {
        uint8_t last = 0;
        CU(cudaMemcpyAsync(&last, f1.d_in.p + f1.n_bytes - 1, 1, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (last != '\n') n_lines += 1;
    }
    int rc;
    long long n = 0;
    if (!fasta) {
        if (n_lines % 4 != 0)
            return fail(CG_EINVAL, "FASTQ chunk does not consist of complete 4-line records (" + std::to_string(n_lines) +
                                       " lines)");
        n = n_lines / 4;
        if ((rc = f1.d_nl.ensure((size_t)g.n_nl + 1)) != CG_OK) return rc;
        CU(cg_launch_fastq_index(f1.d_in.p, f1.n_bytes, f1.d_tiles.p, nullptr, f1.d_nl.p, 1, st));
        c->launches += 1;
    } else if (n_lines > 0) {
        cg_fastq_params plain;
        memset(&plain, 0, sizeof plain);
        if ((rc = fasta_stage_normalise(c, f1, &plain, n_lines, st, g, &n)) != CG_OK) return rc;
    }
    if (n % 2 != 0)
        return fail(CG_EINVAL, "Interleaved input file incomplete: the chunk holds an odd number of records (" +
                                   std::to_string(n) + "), record " + std::to_string(n - 1) + " has no mate");
    int64_t seg[3] = {0, 0, 0};                 // mate 1 starts, mate 2 starts, end
    if (n > 0) {
        if ((rc = f1.d_rec.ensure((size_t)n + 1)) != CG_OK) return rc;
        if ((rc = f1.d_len.ensure((size_t)n)) != CG_OK) return rc;
        if ((rc = f1.d_outlen.ensure((size_t)n)) != CG_OK) return rc;
        if ((rc = f1.d_dest.ensure((size_t)n)) != CG_OK) return rc;
        if ((rc = f1.d_outoff.ensure((size_t)n + 1)) != CG_OK) return rc;
        if ((rc = f1.d_ilverr.ensure(1)) != CG_OK) return rc;
        const unsigned long long none = ~0ull;
        CU(cudaMemcpyAsync(f1.d_ilverr.p, &none, sizeof none, cudaMemcpyHostToDevice, st));
        // d_len: where each record starts, d_outlen: its size, d_dest: its mate
        CU(cg_launch_interleaved_split(0, f1.d_in.p, f1.n_bytes, fasta ? nullptr : f1.d_nl.p, g.n_nl, n, f1.d_rec.p,
                                       f1.d_len.p, f1.d_outlen.p, f1.d_dest.p, f1.d_ilverr.p, nullptr, 0, nullptr, nullptr,
                                       fasta ? 1 : 0, st));
        c->launches += 2;
        long long total = 0;
        if ((rc = fastq_partition(c, f1, n, 2, f1.d_outlen.p, f1.d_dest.p, seg, &total, st)) != CG_OK) return rc;
        unsigned long long bad = none;
        CU(cudaMemcpyAsync(&bad, f1.d_ilverr.p, sizeof bad, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (bad != none) {
            const long long r = (long long)(bad >> 32);
            const int code = (int)(bad & 0xFFFFFFFFu);
            if (code != CG_FQ_ERR_PAIR) {
                const int e[2] = {code, (int)r};
                return fastq_format_error(e);
            }
            CgFastqRecord h[2];
            CU(cudaMemcpy(h, f1.d_rec.p + r - 1, sizeof h, cudaMemcpyDeviceToHost));
            std::string names[2];
            for (int k = 0; k < 2; ++k) {
                names[k].resize((size_t)std::max(h[k].hdr_len, 0));
                if (h[k].hdr_len > 0)
                    CU(cudaMemcpy(&names[k][0], f1.d_in.p + h[k].hdr_start, (size_t)h[k].hdr_len, cudaMemcpyDeviceToHost));
            }
            return fail(CG_EINVAL, "Reads are improperly paired: records " + std::to_string(r - 1) + " and " +
                                       std::to_string(r) + " of the interleaved chunk, read name '" + names[0] +
                                       "' does not match '" + names[1] + "'");
        }
        std::swap(f1.d_in, f1.d_norm);          // the chunk becomes the source, d_in receives mate 1
        if ((rc = f1.d_in.ensure((size_t)seg[1] + 64)) != CG_OK) return rc;
        if ((rc = f2.d_in.ensure((size_t)(seg[2] - seg[1]) + 64)) != CG_OK) return rc;
        CU(cg_launch_interleaved_split(1, f1.d_norm.p, 0, nullptr, 0, n, nullptr, f1.d_len.p, f1.d_outlen.p, nullptr,
                                       nullptr, f1.d_outoff.p, seg[1], f1.d_in.p, f2.d_in.p, fasta ? 1 : 0, st));
        c->launches += 1;
    }
    f1.n_bytes = seg[1];
    f2.n_bytes = seg[2] - seg[1];
    const int err_init[2] = {0, 0x7FFFFFFF};
    for (FastqSlot *f : {&f1, &f2}) {
        if ((rc = f->d_tiles.ensure((size_t)cg_fastq_tiles(f->n_bytes) + 1)) != CG_OK) return rc;
        CU(cudaMemsetAsync(f->d_counters.p, 0, (1 + CG_FQ_COUNTERS) * sizeof(unsigned long long), st));
        CU(cudaMemcpyAsync(f->d_err.p, err_init, sizeof err_init, cudaMemcpyHostToDevice, st));
        if (f->n_bytes) {
            CU(cg_launch_fastq_index(f->d_in.p, f->n_bytes, f->d_tiles.p, f->d_counters.p, nullptr, 0, st));
            c->launches += 2;
        }
        CU(cudaMemcpyAsync(f->h_counters.p, f->d_counters.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    }
    CU(cudaStreamSynchronize(st));
    return CG_OK;
}

// index the chunk, build the record table, run the modifiers (trimming pass included), evaluate the filters
// Line table -> record table of one mate (format checks, -u, bases read); sizes every per-record buffer.
static int fastq_stage_records(cg_ctx *c, FastqSlot &f, const cg_fastq_params *fp, bool has_set, cudaStream_t st, FqStage &g)
{
    if (fp->format < CG_FORMAT_FASTQ || fp->format > CG_FORMAT_FASTQ_TO_FASTA)
        return fail(CG_EINVAL, "cg_fastq: format must be 0 (FASTQ), 1 (FASTA) or 2 (FASTQ in, FASTA out)");
    if (fp->format == CG_FORMAT_FASTA && (fp->trim.quality_trim || fp->trim.nextseq_trim || fp->max_expected_errors >= 0.0 ||
                                          fp->max_average_error_rate != 0.0 || fp->zero_cap))
        return fail(CG_EINVAL, "FASTA input has no qualities: quality trimming, --nextseq-trim, --max-ee, --max-aer and "
                               "--zero-cap need FASTQ");
    // TooHighAverageErrorRate rejects a rate outside (0, 1) (predicates.py:81-85); 0 here means off
    if (!(fp->max_average_error_rate >= 0.0 && fp->max_average_error_rate < 1.0))
        return fail(CG_EINVAL, "cg_fastq: max_average_error_rate must be between 0.0 and 1.0 (0 = off)");
    if (fp->zero_cap != 0 && fp->zero_cap != 1) return fail(CG_EINVAL, "cg_fastq: zero_cap must be 0 or 1");
    g.format = fp->format;
    g.zero_cap = fp->zero_cap ? (fp->trim.quality_base & 255) : 0;
    CU(cudaStreamSynchronize(f.stream));        // upload + newline count of this slot
    const int64_t n_bytes = f.n_bytes;
    g.n_nl = (long long)f.h_counters.p[0];
    long long n_lines = g.n_nl;                 // the last line may come without its newline
    if (n_bytes > 0) {
        uint8_t last = 0;
        CU(cudaMemcpyAsync(&last, f.d_in.p + n_bytes - 1, 1, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (last != '\n') n_lines += 1;
    }
    const bool fasta = fp->format == CG_FORMAT_FASTA;
    if (!fasta && n_lines % 4 != 0)
        return fail(CG_EINVAL, "FASTQ chunk does not consist of complete 4-line records (" + std::to_string(n_lines) +
                                   " lines)");
    long long n_fasta = 0;
    if (fasta && n_lines > 0) {
        int rc = fasta_stage_normalise(c, f, fp, n_lines, st, g, &n_fasta);
        if (rc != CG_OK) return rc;
    }
    const long long n = g.n = fasta ? n_fasta : n_lines / 4;
    if (n == 0) return CG_OK;
    const cg_params *p = &fp->trim;
    g.want_q = p->quality_trim != 0 || p->nextseq_trim != 0;
    g.times = p->times < 1 ? 1 : p->times;
    if (fp->cut_front < 0 || fp->cut_back < 0) return fail(CG_EINVAL, "cg_fastq: cut_front / cut_back must be >= 0");
    if (fp->action < CG_FQ_ACTION_TRIM || fp->action > CG_FQ_ACTION_CROP) return fail(CG_EINVAL, "cg_fastq: unknown action");
    if ((fp->action == CG_FQ_ACTION_RETAIN || fp->action == CG_FQ_ACTION_CROP) && g.times > 1)
        return fail(CG_EINVAL, "'retain' and 'crop' cannot be combined with times > 1");   // modifiers.py:117-118
    if (fp->revcomp < 0 || fp->revcomp > 2) return fail(CG_EINVAL, "cg_fastq: revcomp must be 0, 1 or 2");
    g.action = has_set ? fp->action : CG_FQ_ACTION_TRIM;
    int rc;
    if ((rc = f.d_nl.ensure((size_t)g.n_nl + 1)) != CG_OK) return rc;
    if ((rc = f.d_rec.ensure((size_t)n)) != CG_OK) return rc;
    if ((rc = f.d_len.ensure((size_t)n)) != CG_OK) return rc;
    if ((rc = f.d_origin.ensure((size_t)n * 2)) != CG_OK) return rc;
    if ((rc = f.d_interval.ensure((size_t)n * 2)) != CG_OK) return rc;
    if ((rc = f.d_mask.ensure((size_t)n)) != CG_OK) return rc;
    if ((rc = f.d_keep.ensure((size_t)n * 2)) != CG_OK) return rc;
    if ((rc = f.d_outlen.ensure((size_t)n)) != CG_OK) return rc;
    if ((rc = f.d_outoff.ensure((size_t)n + 1)) != CG_OK) return rc;
    if ((rc = f.d_scan.ensure((size_t)cg_scan_tiles(n) + 1)) != CG_OK) return rc;
    if (g.want_q && (rc = f.d_qtrim.ensure((size_t)n * 2)) != CG_OK) return rc;
    if (!fasta) {
        CU(cg_launch_fastq_index(f.d_in.p, n_bytes, f.d_tiles.p, nullptr, f.d_nl.p, 1, st));
        CU(cg_launch_fastq_records(f.d_in.p, n_bytes, f.d_nl.p, g.n_nl, n, fp->cut_front, fp->cut_back, f.d_rec.p, f.d_len.p,
                                   f.d_origin.p, f.d_counters.p + 1, f.d_err.p, st));
        c->launches += 2;
    }
    g.d_qtrim = g.want_q ? f.d_qtrim.p : nullptr;
    return CG_OK;
}

// NextseqQualityTrimmer + QualityTrimmer as a pass of their own on the chunk
static int fastq_stage_pretrim(cg_ctx *c, FastqSlot &f, const cg_params *p, cudaStream_t st, FqStage &g)
{
    CU(cg_launch_fastq_pretrim(f.d_in.p, f.d_rec.p, f.d_len.p, g.n, (p->quality_trim ? 1 : 0) | (p->nextseq_trim ? 2 : 0),
                               p->cutoff_front, p->cutoff_back,
                               (p->quality_base & 255) | (int)((unsigned)p->nextseq_cutoff << 8), g.d_qtrim, st));
    c->launches += 1;
    return CG_OK;
}

// ... after which the quality-trimmed read IS the record: what --revcomp and --pair-adapters work on
static int fastq_stage_fold_qtrim(cg_ctx *c, FastqSlot &f, const cg_params *p, cudaStream_t st, FqStage &g)
{
    if (!g.want_q) return CG_OK;
    int rc = fastq_stage_pretrim(c, f, p, st, g);
    if (rc != CG_OK) return rc;
    CU(cg_launch_fastq_fold_qtrim(f.d_rec.p, f.d_len.p, g.d_qtrim, g.n, f.d_origin.p, f.d_counters.p + 1, st));
    c->launches += 1;
    g.d_qtrim = nullptr;
    g.want_q = false;
    return CG_OK;
}

// Packed reads for the trimming kernels (d_offs, d_seq, d_qual) + the longest read; reports format errors.
static int fastq_stage_pack(cg_ctx *c, FastqSlot &f, cudaStream_t st, FqStage &g, bool reverse_complement)
{
    const long long n = g.n;
    int rc;
    if ((rc = f.d_offs.ensure((size_t)n + 1)) != CG_OK) return rc;
    if ((rc = f.d_seq.ensure((size_t)f.n_bytes + 64)) != CG_OK) return rc;
    if (g.want_q && (rc = f.d_qual.ensure((size_t)f.n_bytes + 64)) != CG_OK) return rc;
    if (!reverse_complement) {
        CU(cg_launch_scan_i32(f.d_len.p, n, f.d_scan.p, f.d_offs.p, st));
        c->launches += 3;
    }
    CU(cg_launch_fastq_gather(f.d_in.p, f.d_rec.p, f.d_offs.p, n, f.d_seq.p, g.want_q ? f.d_qual.p : nullptr,
                              reverse_complement ? 1 : 0, st));
    c->launches += 1;
    if (reverse_complement) return CG_OK;       // offsets, longest read and format are those of the forward pass
    g.packed = true;
    CU(cudaMemsetAsync(c->d_err + 1, 0, sizeof(int), st));
    CU(cg_launch_max_len(f.d_offs.p, n, c->d_err + 1, st));
    c->launches += 1;
    int fq_err[2];
    CU(cudaMemcpyAsync(&g.max_len, c->d_err + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(fq_err, f.d_err.p, sizeof fq_err, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (fq_err[0]) return fastq_format_error(fq_err, f.ilv);
    return CG_OK;
}

// What is left of every record and which filters it fails (fq_evaluate_core)
static int fastq_stage_verdict(cg_ctx *c, FastqSlot &f, const cg_fastq_params *fp, int poly_a_mode, cudaStream_t st,
                               FqStage &g)
{
    int32_t *d_poly_a = nullptr;                // statistics: PolyATrimmer.trimmed_bases per record
    if (g.acc && fp->poly_a) {
        int rc = f.d_polya.ensure((size_t)g.n);
        if (rc != CG_OK) return rc;
        d_poly_a = f.d_polya.p;
        g.st_poly_a = true;
    }
    CgFastqFilter flt;
    flt.minimum_length = fp->minimum_length;
    flt.maximum_length = fp->maximum_length;
    flt.discard_trimmed = fp->discard_trimmed;
    flt.discard_untrimmed = fp->discard_untrimmed;
    flt.max_n = fp->max_n;
    flt.max_ee = fp->max_expected_errors;
    flt.poly_a = fp->poly_a ? poly_a_mode : 0;
    flt.shorten = !fp->shorten ? 0 : (fp->shorten_length >= 0 ? fp->shorten_length + 1 : fp->shorten_length);
    flt.trim_n = fp->trim_n;
    flt.discard_casava = fp->discard_casava;
    flt.action = g.action;
    flt.max_aer = fp->max_average_error_rate;
    flt.zero_cap = g.zero_cap;
    CU(cg_launch_fastq_evaluate(f.d_in.p, f.d_rec.p, f.d_len.p, g.n, g.d_matches, g.times, g.slots, g.d_qtrim, flt,
                                c->d_phred, g.d_is_rc, f.d_interval.p, f.d_keep.p, f.d_mask.p, f.d_counters.p + 1, f.d_err.p,
                                st, d_poly_a));
    c->launches += 1;
    return CG_OK;
}

// ---- statistics of the FASTQ path (cg_fastq_stats_*) ----
// Vector: the cg_stats_* layout at (n_adapters, max_len, kmax), then reverse_complemented[n_adapters], then the
// poly-A histogram [max_len + 1].
static long long fqstats_total(int n_adapters, int max_len, int kmax)
{
    return cg_stats_total(n_adapters, max_len, kmax) + n_adapters + (max_len + 1);
}

// Lay the accumulator out at a larger (max_len, kmax); every count keeps its (length, errors) cell.
static void fqstats_grow(FqStatsAcc &a, int max_len, int kmax)
{
    max_len = std::max(max_len, a.max_len);
    kmax = std::max(kmax, a.kmax);
    if (max_len == a.max_len && kmax == a.kmax) return;
    const int n = a.n_adapters, L0 = a.max_len, K0 = a.kmax;
    std::vector<int64_t> v((size_t)fqstats_total(n, max_len, kmax), 0);
    for (int i = 0; i < CG_STATS_SCALARS; ++i) v[i] = a.v[i];
    for (int l = 0; l <= L0; ++l) v[CG_STATS_SCALARS + l] = a.v[CG_STATS_SCALARS + l];
    const long long e0 = cg_stats_end_size(L0, K0), e1 = cg_stats_end_size(max_len, kmax);
    const long long b0 = cg_stats_adapters_off(L0), b1 = cg_stats_adapters_off(max_len);
    for (long long e = 0; e < 2LL * n; ++e) {
        const int64_t *src = a.v.data() + b0 + e * e0;
        int64_t *dst = v.data() + b1 + e * e1;
        for (int j = 0; j < CG_STATS_ADJ; ++j) dst[j] = src[j];
        for (int l = 0; l <= L0; ++l)
            for (int k = 0; k <= K0; ++k)
                dst[CG_STATS_ADJ + (long long)l * (kmax + 1) + k] = src[CG_STATS_ADJ + (long long)l * (K0 + 1) + k];
    }
    const long long t0 = cg_stats_total(n, L0, K0), t1 = cg_stats_total(n, max_len, kmax);
    for (int i = 0; i < n; ++i) v[t1 + i] = a.v[t0 + i];
    for (int l = 0; l <= L0; ++l) v[t1 + n + l] = a.v[t0 + n + l];
    a.v.swap(v);
    a.max_len = max_len;
    a.kmax = kmax;
}

// The accumulator a collect adds to (*out = nullptr: statistics off); it must count as many adapters as the set has.
static int fqstats_lookup(cg_ctx *c, int32_t handle, int n_adapters, FqStatsAcc **out)
{
    *out = nullptr;
    if (handle == 0) return CG_OK;
    auto it = c->fq_stats.find(handle);
    if (it == c->fq_stats.end()) return fail(CG_EINVAL, "cg_fastq: unknown statistics handle " + std::to_string(handle));
    if (it->second.n_adapters != n_adapters)
        return fail(CG_EINVAL, "cg_fastq: the statistics accumulator was created for " +
                                   std::to_string(it->second.n_adapters) + " adapters, the adapter set has " +
                                   std::to_string(n_adapters));
    *out = &it->second;
    return CG_OK;
}

// Per-adapter statistics of a mate's reads from their final match records (cg_stats_kernel on the packed reads in the
// orientation that was kept; the read-length histogram is left to the written records) into the slot's vector, laid
// out at the accumulator's (max_len, kmax) grown to this chunk's longest read and the set's largest error count.
static int fastq_stage_stats(cg_ctx *c, FastqSlot &f, FqStage &g, int kmax, cudaStream_t st)
{
    if (!g.acc || g.n == 0) return CG_OK;
    int rc;
    if (!g.packed && (rc = fastq_stage_pack(c, f, st, g, false)) != CG_OK) return rc;   // the longest read
    FqStatsAcc &a = *g.acc;
    fqstats_grow(a, g.max_len, kmax);
    g.st_len = a.max_len;
    g.st_kmax = a.kmax;
    const size_t total = (size_t)fqstats_total(a.n_adapters, a.max_len, a.kmax);
    if ((rc = f.d_fqstats.ensure(total)) != CG_OK) return rc;
    if ((rc = f.h_fqstats.ensure(total)) != CG_OK) return rc;
    CU(cudaMemsetAsync(f.d_fqstats.p, 0, total * sizeof(unsigned long long), st));
    if (g.d_matches && a.n_adapters > 0) {
        CU(cg_launch_stats(f.d_seq.p, f.d_offs.p, g.n, g.d_qtrim != nullptr, g.times, g.slots, g.d_matches, g.d_qtrim,
                           a.n_adapters, a.max_len, a.kmax, f.d_fqstats.p, st, 0,
                           g.action == CG_FQ_ACTION_LOWERCASE ? 1 : 0));
        c->launches += 1;
    }
    return CG_OK;
}

// After the finish kernel: written lengths, poly-A lengths, reverse_complemented per adapter; then the vector goes to
// the host (the output stage waits for it).
static int fastq_stage_stats_tail(cg_ctx *c, FastqSlot &f, const FqStage &g, cudaStream_t st,
                                  const int32_t *d_route = nullptr)
{
    if (!g.acc || g.n == 0) return CG_OK;
    const int n_ad = g.acc->n_adapters;
    unsigned long long *v = f.d_fqstats.p;
    const long long tail = cg_stats_total(n_ad, g.st_len, g.st_kmax);
    CU(cg_launch_fastq_stats_tail(g.n, f.d_interval.p, f.d_outlen.p, g.st_poly_a ? f.d_polya.p : nullptr, g.d_matches,
                                  g.times, g.slots, g.d_is_rc, n_ad, g.st_len, v + CG_STATS_SCALARS, v + tail + n_ad,
                                  v + tail, st, d_route));
    c->launches += 1;
    const size_t total = (size_t)fqstats_total(n_ad, g.st_len, g.st_kmax);
    CU(cudaMemcpyAsync(f.h_fqstats.p, v, total * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    return CG_OK;
}

// The call succeeded: add the chunk's vector; the scalars are those of cg_fastq_result (Statistics.collect takes
// them from the pipeline and the filters, report.py:128-160), the removed adapter bases from the records.
static void fastq_stats_commit(const FastqSlot &f, const FqStage &g, const cg_fastq_params *fp, const cg_fastq_result &res)
{
    if (!g.acc || g.n == 0) return;
    FqStatsAcc &a = *g.acc;
    const unsigned long long *h = f.h_fqstats.p;
    for (size_t i = CG_STATS_SCALARS; i < a.v.size(); ++i) a.v[i] += (int64_t)h[i];
    int64_t *v = a.v.data();
    v[0] += res.n_records; v[1] += res.bp_in; v[2] += res.with_adapters; v[3] += res.quality_trimmed_bp;
    v[4] += (int64_t)h[4]; v[5] += res.reverse_complemented; v[6] += res.n_written; v[7] += res.bp_out;
    v[8] += res.too_short; v[9] += res.too_long; v[10] += res.too_many_n; v[11] += res.too_many_expected_errors;
    v[12] += res.casava_filtered; v[15] += res.too_high_average_error_rate;
    // --discard-trimmed and --discard-untrimmed exclude each other (cli.py:798-808)
    v[fp->discard_trimmed ? 13 : 14] += res.discarded;
}

static int fastq_stage_evaluate(cg_ctx *c, FastqSlot &f, const cg_adapterset *s, const cg_fastq_params *fp, int poly_a_mode,
                                cudaStream_t st, FqStage &g)
{
    int rc = fastq_stage_records(c, f, fp, s != nullptr, st, g);
    if (rc != CG_OK || g.n == 0) return rc;
    const long long n = g.n;
    const cg_params *p = &fp->trim;
    g.slots = s ? s->host.slots : 1;
    if (s && fp->revcomp) {
        // ReverseComplementer (modifiers.py:264-308): the adapter rounds on the read and on its reverse complement, both
        // AFTER the quality trimmers; fq_revcomp_commit_kernel keeps the better orientation in the chunk itself.
        if ((rc = fastq_stage_fold_qtrim(c, f, p, st, g)) != CG_OK) return rc;
        cg_params pt = *p;
        pt.quality_trim = 0;
        pt.nextseq_trim = 0;
        const size_t per_read = (size_t)g.times * g.slots;
        if ((rc = f.d_matches.ensure((size_t)n * per_read)) != CG_OK) return rc;
        if ((rc = f.d_matches_rc.ensure((size_t)n * per_read)) != CG_OK) return rc;
        if ((rc = f.d_isrc.ensure((size_t)n)) != CG_OK) return rc;
        if ((rc = fastq_stage_pack(c, f, st, g, false)) != CG_OK) return rc;
        rc = launch_trim(c, s, f.d_seq.p, nullptr, f.d_offs.p, n, g.max_len, &pt, f.d_matches.p, nullptr, st, true);
        if (rc != CG_OK) return rc;
        if ((rc = fastq_stage_pack(c, f, st, g, true)) != CG_OK) return rc;
        rc = launch_trim(c, s, f.d_seq.p, nullptr, f.d_offs.p, n, g.max_len, &pt, f.d_matches_rc.p, nullptr, st, true);
        if (rc != CG_OK) return rc;
        CU(cg_launch_fastq_revcomp_commit(f.d_in.p, f.d_rec.p, f.d_len.p, f.d_origin.p, n, f.d_matches.p, f.d_matches_rc.p, (int)per_read,
                                          f.d_isrc.p, f.d_counters.p + 1, st, g.has_qual() ? 1 : 0));
        c->launches += 1;
        g.d_matches = f.d_matches.p;
        g.d_is_rc = f.d_isrc.p;
        g.rc_suffix = fp->revcomp == 1;
        if (g.acc) {                            // the statistics see the reads in the orientation that was kept
            CU(cg_launch_fastq_gather(f.d_in.p, f.d_rec.p, f.d_offs.p, n, f.d_seq.p, nullptr, 0, st));
            c->launches += 1;
        }
    } else if (s) {
        if ((rc = f.d_matches.ensure((size_t)n * g.times * g.slots)) != CG_OK) return rc;
        if ((rc = fastq_stage_pack(c, f, st, g, false)) != CG_OK) return rc;
        rc = launch_trim(c, s, f.d_seq.p, g.want_q ? f.d_qual.p : nullptr, f.d_offs.p, n, g.max_len, p, f.d_matches.p,
                         g.d_qtrim, st, true);
        if (rc != CG_OK) return rc;
        g.d_matches = f.d_matches.p;
    } else if (g.want_q) {
        if ((rc = fastq_stage_pretrim(c, f, p, st, g)) != CG_OK) return rc;
    }
    if ((rc = fastq_stage_stats(c, f, g, s ? s->host.max_k : 0, st)) != CG_OK) return rc;
    return fastq_stage_verdict(c, f, fp, poly_a_mode, st, g);
}

// Optional routing of the records (demultiplexing): destinations are decided once per chunk (fastq_stage_route, on
// the first mate's slot), then every mate's output is partitioned by them.
struct FqDemux {
    const int32_t *adapter_dest1 = nullptr;  // host, one destination per adapter of R1, values in [0, n_named1)
    int n_adapters1 = 0, n_named1 = 0;
    const int32_t *adapter_dest2 = nullptr;  // combinatorial: the same for R2 (nullptr: route by R1 alone)
    int n_adapters2 = 0, n_named2 = 0;
    const uint8_t *dest_keep = nullptr;      // host, optional: destinations without a writer drop their records
    int n_dest() const { return (n_named1 + 1) * (adapter_dest2 ? n_named2 + 1 : 1); }
    const int32_t *d_dest = nullptr;         // device, filled by fastq_stage_route
    const uint8_t *d_dest_keep = nullptr;
};

static int fastq_stage_route(cg_ctx *c, FastqSlot &f1, FastqSlot *f2, long long n, FqDemux &dm, cudaStream_t st)
{
    int rc;
    if ((rc = f1.d_adest.ensure((size_t)dm.n_adapters1 + dm.n_adapters2 + 1)) != CG_OK) return rc;
    if ((rc = f1.d_dest.ensure((size_t)n)) != CG_OK) return rc;
    CU(cudaMemcpyAsync(f1.d_adest.p, dm.adapter_dest1, (size_t)dm.n_adapters1 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (dm.adapter_dest2)
        CU(cudaMemcpyAsync(f1.d_adest.p + dm.n_adapters1, dm.adapter_dest2, (size_t)dm.n_adapters2 * sizeof(int32_t),
                           cudaMemcpyHostToDevice, st));
    CU(cg_launch_fastq_dest(f1.d_mask.p, dm.adapter_dest2 ? f2->d_mask.p : nullptr, n, f1.d_adest.p, dm.n_named1,
                            f1.d_adest.p + dm.n_adapters1, dm.n_named2, f1.d_dest.p, st));
    c->launches += 1;
    dm.d_dest = f1.d_dest.p;
    if (dm.dest_keep) {
        if ((rc = f1.d_destkeep.ensure((size_t)dm.n_dest())) != CG_OK) return rc;
        CU(cudaMemcpyAsync(f1.d_destkeep.p, dm.dest_keep, (size_t)dm.n_dest(), cudaMemcpyHostToDevice, st));
        dm.d_dest_keep = f1.d_destkeep.p;
    }
    return CG_OK;
}

// Filter outputs (cg_fastq_collect_split*): a read or pair that the too-short, too-long or untrimmed filter removes goes
// to destination 1, 2 or 3 when `redirect` has that filter's CG_REDIRECT_* bit; the finish kernel fills d_route, the
// output is partitioned by it like a demultiplexed one and written in each destination's format.
struct FqSplit {
    int redirect = 0;                // CG_REDIRECT_* bits
    int fasta_dests = 0;             // bit d: destination d is written as FASTA
    int32_t *d_route = nullptr;      // device, per record: destination, -1 = dropped
    bool interleaved = false;        // cg_fastq_collect_paired_interleaved ...
    int ilv_dests = 0;               // ... bit d: destination d is written interleaved
    static constexpr int n_dest = 4;
};

// The checks of cg_fastq_collect_split(_paired) on the parameters of a mate
static int split_check(const FqSplit &sp, const cg_fastq_params *fp, const char *who)
{
    if (sp.redirect & ~7) return fail(CG_EINVAL, std::string(who) + ": redirect takes CG_REDIRECT_* bits only");
    if ((sp.fasta_dests >> 1) & ~7) return fail(CG_EINVAL, std::string(who) + ": fasta_outputs takes CG_REDIRECT_* bits only");
    if ((sp.redirect & CG_REDIRECT_UNTRIMMED) && fp->discard_trimmed)
        return fail(CG_EINVAL, std::string(who) + ": the untrimmed output cannot be combined with discard_trimmed");
    if (fp->format == CG_FORMAT_FASTA && (sp.redirect & ~(sp.fasta_dests >> 1)))
        return fail(CG_EINVAL, std::string(who) + ": FASTA input can only be written as FASTA (set every redirect bit in "
                                                   "fasta_outputs)");
    return CG_OK;
}

// The counters of a mate into its result, once the stream has got there; reports format errors.
static int fastq_stage_result(FastqSlot &f, const FqStage &g, cudaStream_t st, cg_fastq_result *res)
{
    int fq_err[2];
    CU(cudaMemcpyAsync(fq_err, f.d_err.p, sizeof fq_err, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(f.h_counters.p, f.d_counters.p, (1 + CG_FQ_COUNTERS) * sizeof(unsigned long long),
                       cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (fq_err[0]) return fastq_format_error(fq_err, f.ilv);
    const unsigned long long *k = f.h_counters.p + 1;
    res->n_records = g.n;
    res->n_written = (int64_t)k[0]; res->bp_in = (int64_t)k[1]; res->bp_out = (int64_t)k[2];
    res->with_adapters = (int64_t)k[3]; res->too_short = (int64_t)k[4]; res->too_long = (int64_t)k[5];
    res->quality_trimmed_bp = (int64_t)k[6]; res->discarded = (int64_t)k[7]; res->too_many_n = (int64_t)k[8];
    res->too_many_expected_errors = (int64_t)k[9];
    res->casava_filtered = (int64_t)k[10];
    res->reverse_complemented = (int64_t)k[11];
    res->too_high_average_error_rate = (int64_t)k[12];
    return CG_OK;
}

// The formatted records of a mate at f.d_outoff in d_out.  sp: one writer per format that has bytes to write (segments:
// the destinations, host), each skipping the other format's destinations.
static int fastq_write_records(cg_ctx *c, FastqSlot &f, const FqStage &g, uint8_t *d_out, const FqSplit *sp,
                               const int64_t *segments, cudaStream_t st)
{
    if (!sp) {
        CU(cg_launch_fastq_write(f.d_in.p, f.d_rec.p, f.d_interval.p, f.d_outoff.p, f.d_outlen.p, g.n, d_out, g.action,
                                 f.d_keep.p, f.d_mask.p, g.rc_suffix, st, g.fasta_out() ? 1 : 0, nullptr, 0, g.zero_cap));
        c->launches += 1;
        return CG_OK;
    }
    for (int fa = 0; fa < 2; ++fa) {
        bool present = false;
        for (int d = 0; d < FqSplit::n_dest; ++d)
            present |= ((sp->fasta_dests >> d) & 1) == fa && segments[d + 1] > segments[d];
        if (!present) continue;
        CU(cg_launch_fastq_write(f.d_in.p, f.d_rec.p, f.d_interval.p, f.d_outoff.p, f.d_outlen.p, g.n, d_out, g.action,
                                 f.d_keep.p, f.d_mask.p, g.rc_suffix, st, fa, sp->d_route, sp->fasta_dests, g.zero_cap));
        c->launches += 1;
    }
    return CG_OK;
}

// bytes of d_src to the caller's `out` (through the slot's pinned bounce buffer unless `out` is pinned)
static int fastq_copy_out(cg_ctx *c, FastqSlot &f, uint8_t *out, const uint8_t *d_src, long long bytes, cudaStream_t st)
{
    if (bytes <= 0) return CG_OK;
    if (is_pinned(out)) {
        CU(cudaMemcpyAsync(out, d_src, (size_t)bytes, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    } else {
        const int rc = f.h_out.ensure((size_t)bytes);
        if (rc != CG_OK) return rc;
        CU(cudaMemcpyAsync(f.h_out.p, d_src, (size_t)bytes, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        parallel_copy(c, out, f.h_out.p, (size_t)bytes);
    }
    c->d2h_bytes += bytes;
    return CG_OK;
}

// gzip outputs: the destinations of d_src at bounds[0 .. n_dest] (host), destination d compressed when gz[d], else copied.
// Every destination is cut into pieces of GZ_MEMBER bytes from its start; gz_compress_kernel turns each gzip piece into a
// member in its slot, the host places the pieces behind each other and gz_gather_kernel packs them into `packed`
// (f.d_gzout for the outputs).  bounds then hold where each destination lies there; *total is the packed size.
static int fastq_gzip(cg_ctx *c, FastqSlot &f, const uint8_t *d_src, std::vector<int64_t> &bounds, const std::vector<char> &gz,
                      DevBuf<uint8_t> &packed, long long *total, cudaStream_t st)
{
    const size_t n_dest = gz.size();
    std::vector<CgGzPiece> pieces;
    for (size_t d = 0; d < n_dest; ++d)
        for (int64_t o = bounds[d]; o < bounds[d + 1]; o += GZ_MEMBER)
            pieces.push_back(CgGzPiece{(long long)o, (int32_t)std::min<int64_t>(GZ_MEMBER, bounds[d + 1] - o), gz[d] ? 1 : 0});
    const size_t np = pieces.size();
    *total = 0;
    if (np == 0) return CG_OK;
    int rc;
    if ((rc = f.d_gzpieces.ensure(np)) != CG_OK || (rc = f.d_gzsizes.ensure(np)) != CG_OK ||
        (rc = f.d_gzoff.ensure(np)) != CG_OK || (rc = f.d_gzslots.ensure(np * GZ_SLOT)) != CG_OK)
        return rc;
    CU(cudaMemcpyAsync(f.d_gzpieces.p, pieces.data(), np * sizeof(CgGzPiece), cudaMemcpyHostToDevice, st));
    CU(cg_launch_gzip_compress(d_src, f.d_gzpieces.p, (int)np, f.d_gzslots.p, f.d_gzsizes.p, st));
    std::vector<int32_t> sizes(np);
    CU(cudaMemcpyAsync(sizes.data(), f.d_gzsizes.p, np * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    std::vector<int64_t> off(np);
    int64_t at = 0;
    size_t k = 0;
    for (size_t d = 0; d < n_dest; ++d) {
        const int64_t n_pieces = (bounds[d + 1] - bounds[d] + GZ_MEMBER - 1) / GZ_MEMBER;
        bounds[d] = at;
        for (int64_t i = 0; i < n_pieces; ++i, ++k) { off[k] = at; at += sizes[k]; }
    }
    bounds[n_dest] = at;
    if ((rc = packed.ensure((size_t)at + 64)) != CG_OK) return rc;
    CU(cudaMemcpyAsync(f.d_gzoff.p, off.data(), np * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    CU(cg_launch_gzip_gather(f.d_gzslots.p, f.d_gzsizes.p, f.d_gzoff.p, (int)np, packed.p, st));
    c->launches += 2;
    *total = at;
    return CG_OK;
}

// whether destination d of a collect is written as gzip: the main output (every output of a demultiplexing collect)
// under CG_GZIP_MAIN, filter output d under CG_REDIRECT_* bit d - 1
static bool gzip_dest(int gzip_outputs, bool demux, int d)
{
    return (demux || d == 0) ? (gzip_outputs & CG_GZIP_MAIN) != 0 : ((gzip_outputs >> (d - 1)) & 1) != 0;
}

static int gzip_check(const cg_fastq_params *fp, const char *who)
{
    if (fp->gzip_outputs & ~(CG_GZIP_MAIN | 7))
        return fail(CG_EINVAL, std::string(who) + ": gzip_outputs takes CG_GZIP_MAIN and CG_REDIRECT_* bits only");
    return CG_OK;
}

// A mate of a collect: its slot and stage, its parameters and the caller's output for it
struct FqMate {
    FastqSlot *f = nullptr;
    FqStage *g = nullptr;
    const cg_fastq_params *fp = nullptr;
    uint8_t *out = nullptr;
    int64_t capacity = 0;
    cg_fastq_result *res = nullptr;
    int64_t *segments = nullptr;          // host, or null: where each destination starts in out
};

// The formatted records of a collect to the callers' outputs.  write(d_out) fills the device buffer; bounds (host) are
// its destinations, the n_out (1 or 2) outputs m[i] take an equal share of them in order.  With gzip (the caller asked
// for gzip outputs) the records go through fastq_gzip, destination d compressed when gz[d], before the capacity checks;
// bounds, out_bytes and segments then describe the packed bytes.  Without, the checks come before the records are
// written.  The scratch and the bounce buffer are slot f's.
template <class Write>
static int fastq_emit(cg_ctx *c, FastqSlot &f, std::vector<int64_t> &bounds, const std::vector<char> &gz, bool gzip,
                      const FqMate *m, int n_out, const char *who, cudaStream_t st, Write write)
{
    const size_t per = (bounds.size() - 1) / (size_t)n_out;
    const bool pack = gzip && bounds.back() > 0;
    int rc;
    if (pack) {
        if ((rc = f.d_out.ensure((size_t)bounds.back() + 64)) != CG_OK) return rc;
        if ((rc = write(f.d_out.p)) != CG_OK) return rc;
        long long packed = 0;
        if ((rc = fastq_gzip(c, f, f.d_out.p, bounds, gz, f.d_gzout, &packed, st)) != CG_OK) return rc;
        for (int i = 0; i < n_out; ++i) m[i].res->out_bytes = bounds[(i + 1) * per] - bounds[i * per];
    }
    std::string need;
    bool small = false, null = false;
    for (int i = 0; i < n_out; ++i) {
        const int64_t bytes = bounds[(i + 1) * per] - bounds[i * per];
        need += (i ? " and " : "") + std::to_string(bytes);
        small |= bytes > m[i].capacity;
        null |= bytes && !m[i].out;
    }
    if (small) return fail(CG_EINVAL, std::string(who) + ": output buffer too small (" + need + " bytes needed)");
    if (null) return fail(CG_EINVAL, std::string(who) + ": out is NULL");
    if (pack) {
        for (int i = 0; i < n_out; ++i)
            if (m[i].segments)
                for (size_t d = 0; d <= per; ++d) m[i].segments[d] = bounds[i * per + d] - bounds[i * per];
    } else {
        if (bounds.back() == 0) return CG_OK;
        if ((rc = f.d_out.ensure((size_t)bounds.back() + 64)) != CG_OK) return rc;
        if ((rc = write(f.d_out.p)) != CG_OK) return rc;
    }
    const uint8_t *d_src = pack ? f.d_gzout.p : f.d_out.p;
    for (int i = 0; i < n_out; ++i)
        if ((rc = fastq_copy_out(c, f, m[i].out, d_src + bounds[i * per], bounds[(i + 1) * per] - bounds[i * per], st)) !=
            CG_OK)
            return rc;
    return CG_OK;
}

// sizes -> offsets -> formatted records -> host; counters.  m.segments (n_dest + 1 values): where each destination
// starts in m.out.
static int fastq_stage_output(cg_ctx *c, const FqMate &m, cudaStream_t st, const FqDemux *dm, const FqSplit *sp)
{
    FastqSlot &f = *m.f;
    const FqStage &g = *m.g;
    const long long n = g.n;
    int rc;
    long long total = 0;
    if (dm || sp) {
        rc = fastq_partition(c, f, n, dm ? dm->n_dest() : FqSplit::n_dest, f.d_outlen.p, dm ? dm->d_dest : sp->d_route,
                             m.segments, &total, st);
        if (rc != CG_OK) return rc;
    } else {
        CU(cg_launch_scan_i32(f.d_outlen.p, n, f.d_scan.p, f.d_outoff.p, st));
        c->launches += 3;
        CU(cudaMemcpyAsync(&total, f.d_outoff.p + n, sizeof total, cudaMemcpyDeviceToHost, st));
    }
    if ((rc = fastq_stage_result(f, g, st, m.res)) != CG_OK) return rc;
    m.res->out_bytes = m.res->out_bytes_plain = total;
    const int n_dest = dm ? dm->n_dest() : sp ? FqSplit::n_dest : 1;
    std::vector<int64_t> bounds{0, (int64_t)total};
    if (m.segments) bounds.assign(m.segments, m.segments + n_dest + 1);
    std::vector<char> gz((size_t)n_dest);
    for (int d = 0; d < n_dest; ++d) gz[(size_t)d] = gzip_dest(m.fp->gzip_outputs, dm != nullptr, d);
    return fastq_emit(c, f, bounds, gz, m.fp->gzip_outputs != 0, &m, 1, "cg_fastq_collect", st,
                      [&](uint8_t *d_out) { return fastq_write_records(c, f, g, d_out, sp, m.segments, st); });
}

// Interleaved outputs (cg_fastq_collect_paired_interleaved): bit d of sp.ilv_dests = destination d gets both mates in
// out1, R1 then R2 per pair.  The pair's sizes are folded into mate 1 for the partition, mate 2 then follows its mate 1
// (off1 + len1); both mates go through the writer into one device buffer, mate 1's region (total1 bytes) then mate 2's.
static int fastq_stage_output_interleaved(cg_ctx *c, const FqMate *m, const FqSplit &sp, cudaStream_t st)
{
    FastqSlot &f1 = *m[0].f, &f2 = *m[1].f;
    const FqStage &g1 = *m[0].g, &g2 = *m[1].g;
    int64_t *segments1 = m[0].segments, *segments2 = m[1].segments;
    const long long n = g1.n;
    int rc;
    if ((rc = f1.d_fold.ensure((size_t)n)) != CG_OK) return rc;
    if ((rc = f2.d_fold.ensure((size_t)n)) != CG_OK) return rc;
    CU(cg_launch_fastq_interleave(0, n, sp.d_route, sp.ilv_dests, f1.d_outlen.p, f2.d_outlen.p, f1.d_fold.p, f2.d_fold.p,
                                  nullptr, nullptr, nullptr, st));
    c->launches += 1;
    long long total1 = 0, total2 = 0;
    if ((rc = fastq_partition(c, f1, n, FqSplit::n_dest, f1.d_fold.p, sp.d_route, segments1, &total1, st)) != CG_OK) return rc;
    if ((rc = fastq_partition(c, f2, n, FqSplit::n_dest, f2.d_fold.p, sp.d_route, segments2, &total2, st)) != CG_OK) return rc;
    CU(cg_launch_fastq_interleave(1, n, sp.d_route, sp.ilv_dests, f1.d_outlen.p, f2.d_outlen.p, nullptr, nullptr,
                                  f1.d_outoff.p, f2.d_outoff.p, f1.d_dmbase.p + cg_demux_tiles(n) * FqSplit::n_dest, st));
    c->launches += 1;
    if ((rc = fastq_stage_result(f1, g1, st, m[0].res)) != CG_OK) return rc;
    if ((rc = fastq_stage_result(f2, g2, st, m[1].res)) != CG_OK) return rc;
    m[0].res->out_bytes = m[0].res->out_bytes_plain = total1;
    m[1].res->out_bytes = m[1].res->out_bytes_plain = total2;
    // out1's four destinations, then out2's, in the one buffer the writer fills
    std::vector<int64_t> bounds(2 * FqSplit::n_dest + 1);
    std::vector<char> gz(2 * FqSplit::n_dest);
    for (int d = 0; d < FqSplit::n_dest; ++d) {
        bounds[d] = segments1[d];
        bounds[FqSplit::n_dest + d] = total1 + segments2[d];
        gz[d] = gzip_dest(m[0].fp->gzip_outputs, false, d);
        gz[FqSplit::n_dest + d] = gzip_dest(m[1].fp->gzip_outputs, false, d);
    }
    bounds[2 * FqSplit::n_dest] = total1 + total2;
    return fastq_emit(c, f1, bounds, gz, m[0].fp->gzip_outputs || m[1].fp->gzip_outputs, m, 2,
                      "cg_fastq_collect_paired_interleaved", st, [&](uint8_t *d_out) {
                          // a pair has bytes in a destination for both mates or for neither: segments1 says which formats
                          // mate 2 needs too
                          int rc2 = fastq_write_records(c, f1, g1, d_out, &sp, segments1, st);
                          return rc2 != CG_OK ? rc2 : fastq_write_records(c, f2, g2, d_out, &sp, segments1, st);
                      });
}

// ---- rows of a slot's records (cg_fastq_request_rows) ----
static const char *const rows_kind_name[CG_ROWS_KINDS] = {"info", "rest", "wildcard"};

// The requests of a slot against the collect's set: n_entries adapters (pairs with --pair-adapters, 0 without a set).
// Checked before the collect does any work.
static int fastq_rows_check(const FastqSlot &f, int n_entries, const char *who)
{
    for (int k = 0; k < CG_ROWS_KINDS; ++k) {
        const FqRows &q = f.rows[k];
        if (q.requested && q.n_entries != n_entries)
            return fail(CG_EINVAL, std::string(who) + ": the " + rows_kind_name[k] + " rows were requested with " +
                                       std::to_string(q.n_entries) + " entries of text, the collect's adapter set has " +
                                       std::to_string(n_entries));
    }
    return CG_OK;
}

// Every requested kind of rows of a mate, after its matches are final and before the finish kernel:
// fq_info_count_kernel -> scan -> fq_info_write_kernel into the kind's own buffer, then, for gzip rows, fastq_gzip
// into the kind's own packed buffer (the output stage reuses the slot's d_out / d_gzout).  The walks cut the read as it
// came: the record table keeps where the record lies in it (d_origin), also after the quality trimmers were folded in.
static int fastq_stage_rows(cg_ctx *c, FastqSlot &f, const FqStage &g, const cg_fastq_params *fp, cudaStream_t st)
{
    const long long n = g.n;
    const int upper = g.action == CG_FQ_ACTION_LOWERCASE;
    int rc;
    for (int k = 0; k < CG_ROWS_KINDS; ++k) {
        FqRows &q = f.rows[k];
        if (!q.requested) continue;
        const size_t text_bytes = (size_t)q.text_off[(size_t)q.n_entries];
        if ((rc = q.d_text.ensure(text_bytes + 1)) != CG_OK) return rc;
        if ((rc = q.d_textoff.ensure((size_t)q.n_entries + 1)) != CG_OK) return rc;
        if ((rc = q.d_row.ensure((size_t)n)) != CG_OK) return rc;
        if ((rc = q.d_rowoff.ensure((size_t)n + 1)) != CG_OK) return rc;
        if ((rc = f.d_scan.ensure((size_t)cg_scan_tiles(n) + 1)) != CG_OK) return rc;
        if (text_bytes) CU(cudaMemcpyAsync(q.d_text.p, q.text.data(), text_bytes, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(q.d_textoff.p, q.text_off.data(), ((size_t)q.n_entries + 1) * sizeof(int32_t),
                           cudaMemcpyHostToDevice, st));
        CU(cg_launch_fastq_info(0, f.d_in.p, f.d_rec.p, f.d_origin.p, f.d_interval.p, f.d_mask.p, g.d_matches, g.times,
                                g.slots, q.d_text.p, q.d_textoff.p, fp->revcomp != 0, g.rc_suffix, upper, n, q.d_row.p,
                                nullptr, nullptr, st, k, g.d_qtrim, f.d_len.p, g.has_qual() ? 1 : 0, g.zero_cap));
        CU(cg_launch_scan_i32(q.d_row.p, n, f.d_scan.p, q.d_rowoff.p, st));
        long long total = 0;
        CU(cudaMemcpyAsync(&total, q.d_rowoff.p + n, sizeof total, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        c->launches += 4;
        q.bytes = q.bytes_plain = total;
        if (q.limit >= 0 && total > q.limit)
            return fail(CG_EINVAL, std::string(k == CG_ROWS_INFO ? "cg_fastq_collect_info: info" : "cg_fastq_collect_rows: rows") +
                                       " buffer too small (" + std::to_string(total) + " bytes needed)");
        if (total == 0) continue;
        if ((rc = q.d_out.ensure((size_t)total + 64)) != CG_OK) return rc;
        CU(cg_launch_fastq_info(1, f.d_in.p, f.d_rec.p, f.d_origin.p, f.d_interval.p, f.d_mask.p, g.d_matches, g.times,
                                g.slots, q.d_text.p, q.d_textoff.p, fp->revcomp != 0, g.rc_suffix, upper, n, nullptr,
                                q.d_rowoff.p, q.d_out.p, st, k, g.d_qtrim, f.d_len.p, g.has_qual() ? 1 : 0, g.zero_cap));
        c->launches += 1;
        if (q.gzip) {
            std::vector<int64_t> bounds{0, (int64_t)total};
            long long packed = 0;
            if ((rc = fastq_gzip(c, f, q.d_out.p, bounds, std::vector<char>{1}, q.d_gz, &packed, st)) != CG_OK) return rc;
            q.bytes = packed;
        }
    }
    return CG_OK;
}

// A collect that took slot f succeeded (rows_ready) or not: the rows can be read after the one only
static int fastq_rows_done(FastqSlot &f, int rc)
{
    f.rows_ready = rc == CG_OK;
    return rc;
}

extern "C" int cg_fastq_request_rows(cg_ctx *c, int32_t slot, int32_t kind, const char *adapter_text,
                                     const int32_t *text_offsets, int32_t n_entries, int32_t gzip)
{
    if (!c || slot < 0 || slot >= CG_FQ_SLOTS || n_entries < 0 || !text_offsets)
        return fail(CG_EINVAL, "cg_fastq_request_rows: bad argument");
    if (kind < 0 || kind >= CG_ROWS_KINDS)
        return fail(CG_EINVAL, "cg_fastq_request_rows: unknown kind " + std::to_string(kind) +
                                   " (CG_ROWS_INFO, CG_ROWS_REST or CG_ROWS_WILDCARD)");
    FastqSlot &f = c->fq[slot];
    if (!f.busy) return fail(CG_EINVAL, "cg_fastq_request_rows: nothing was submitted to this slot");
    FqRows &q = f.rows[kind];
    if (q.requested)
        return fail(CG_EINVAL, std::string("cg_fastq_request_rows: the ") + rows_kind_name[kind] +
                                   " rows of this slot were requested already");
    if (text_offsets[0] != 0) return fail(CG_EINVAL, "cg_fastq_request_rows: text_offsets must start at 0");
    for (int a = 0; a < n_entries; ++a)
        if (text_offsets[a + 1] < text_offsets[a])
            return fail(CG_EINVAL, "cg_fastq_request_rows: text_offsets must not decrease");
    if (text_offsets[n_entries] && !adapter_text) return fail(CG_EINVAL, "cg_fastq_request_rows: adapter_text is NULL");
    q.text.assign(adapter_text, adapter_text + text_offsets[n_entries]);
    q.text_off.assign(text_offsets, text_offsets + n_entries + 1);
    q.n_entries = n_entries;
    q.gzip = gzip != 0;
    q.limit = -1;
    q.bytes = q.bytes_plain = 0;
    q.requested = true;
    return CG_OK;
}

extern "C" int cg_fastq_read_rows(cg_ctx *c, int32_t slot, int32_t kind, uint8_t *dst, int64_t capacity, int64_t *n_bytes,
                                  int64_t *n_bytes_plain)
{
    if (!c || slot < 0 || slot >= CG_FQ_SLOTS || capacity < 0) return fail(CG_EINVAL, "cg_fastq_read_rows: bad argument");
    if (kind < 0 || kind >= CG_ROWS_KINDS)
        return fail(CG_EINVAL, "cg_fastq_read_rows: unknown kind " + std::to_string(kind) +
                                   " (CG_ROWS_INFO, CG_ROWS_REST or CG_ROWS_WILDCARD)");
    FastqSlot &f = c->fq[slot];
    const FqRows &q = f.rows[kind];
    if (!q.requested)
        return fail(CG_EINVAL, std::string("cg_fastq_read_rows: no ") + rows_kind_name[kind] +
                                   " rows were requested for this slot");
    if (f.busy || !f.rows_ready)
        return fail(CG_EINVAL, "cg_fastq_read_rows: the slot's collect has not run or has failed; there are no rows");
    if (n_bytes) *n_bytes = q.bytes;
    if (n_bytes_plain) *n_bytes_plain = q.bytes_plain;
    if (!dst) return CG_OK;
    if (capacity < q.bytes)
        return fail(CG_EINVAL, "cg_fastq_read_rows: buffer too small (" + std::to_string(q.bytes) + " bytes needed)");
    CU(cudaSetDevice(c->device));
    return fastq_copy_out(c, f, dst, q.gzip ? q.d_gz.p : q.d_out.p, q.bytes, f.stream);
}

// The part of a collect after the evaluation, for one mate (n_mates 1) or a pair, on stream st: the routes, the finish
// kernel, the statistics, the output, the error flag and the statistics commit.  Both mates share one route per pair,
// held by mate 1's slot.
static int fastq_collect_finish(cg_ctx *c, const FqMate *m, int n_mates, FqDemux *dm, FqSplit *sp, int pair_filter_mode,
                                int mode_untrimmed, cudaStream_t st)
{
    const long long n = m[0].g->n;
    FastqSlot *f[2] = {};
    const CgFastqRecord *rec[2] = {};
    const int32_t *interval[2] = {}, *mask[2] = {};
    int32_t *outlen[2] = {};
    unsigned long long *counters[2] = {};
    int enabled[2] = {};
    for (int i = 0; i < n_mates; ++i) {
        f[i] = m[i].f;
        rec[i] = f[i]->d_rec.p; interval[i] = f[i]->d_interval.p; mask[i] = f[i]->d_mask.p; outlen[i] = f[i]->d_outlen.p;
        counters[i] = f[i]->d_counters.p + 1;
        enabled[i] = fastq_enabled_filters(m[i].fp);
    }
    int rc;
    if (dm && (rc = fastq_stage_route(c, *f[0], f[1], n, *dm, st)) != CG_OK) return rc;
    if (sp) {
        if ((rc = f[0]->d_dest.ensure((size_t)n)) != CG_OK) return rc;
        sp->d_route = f[0]->d_dest.p;
        for (int i = 0; i < n_mates; ++i) enabled[i] = fq_route_enabled(enabled[i], sp->redirect);
    }
    CU(cg_launch_fastq_finish(n, rec[0], interval[0], mask[0], enabled[0], outlen[0], counters[0], rec[1], interval[1],
                              mask[1], enabled[1], outlen[1], counters[1], pair_filter_mode, mode_untrimmed,
                              m[0].g->rc_suffix, dm ? dm->d_dest : nullptr, dm ? dm->d_dest_keep : nullptr, st,
                              m[0].g->fasta_out() ? 1 : 0, sp ? sp->redirect : 0, sp ? sp->fasta_dests : 0,
                              sp ? sp->d_route : nullptr));
    c->launches += 1;
    for (int i = 0; i < n_mates; ++i)
        if ((rc = fastq_stage_stats_tail(c, *f[i], *m[i].g, st, sp ? sp->d_route : nullptr)) != CG_OK) return rc;
    if (sp && sp->interleaved) {
        if ((rc = fastq_stage_output_interleaved(c, m, *sp, st)) != CG_OK) return rc;
    } else {
        for (int i = 0; i < n_mates; ++i)
            if ((rc = fastq_stage_output(c, m[i], st, dm, sp)) != CG_OK) return rc;
    }
    if ((rc = check_err_flag(c)) != CG_OK) return rc;
    for (int i = 0; i < n_mates; ++i) fastq_stats_commit(*f[i], *m[i].g, m[i].fp, *m[i].res);
    return CG_OK;
}

// ---- read names (cg_names_*; the name stage, cg_names_core.cuh) ----
static void names_build(NamesProg &np)
{
    np.blob = cg_names_blob(np.spec);
    np.uploaded = false;
}

extern "C" int cg_names_create(cg_ctx *c, const cg_names_desc *d, int32_t *handle)
{
    if (!c || !d || !handle || d->n_strip_suffix < 0 || (d->n_strip_suffix && !d->strip_suffix) ||
        (d->n_rename > 0 && !d->rename))
        return fail(CG_EINVAL, "cg_names_create: bad argument");
    NamesProg np;
    if (d->length_tag) {
        np.spec.tag = d->length_tag;
        if (np.spec.tag.empty()) return fail(CG_EINVAL, "cg_names_create: the length tag is empty");
        for (char ch : np.spec.tag) {
            const bool ok = isalnum((unsigned char)ch) || strchr("_=:,;/-@#%!~", ch) != nullptr;
            if (!ok)
                return fail(CG_EINVAL, std::string("cg_names_create: the length tag may hold letters, digits and "
                                                   "_ = : , ; / - @ # % ! ~ only (the reference reads it as a regular "
                                                   "expression), not '") + ch + "'");
        }
    }
    for (int k = 0; k < d->n_strip_suffix; ++k) {
        if (!d->strip_suffix[k]) return fail(CG_EINVAL, "cg_names_create: a strip suffix is NULL");
        np.spec.strips.emplace_back(d->strip_suffix[k]);
    }
    np.spec.prefix = cg_names_affix(d->prefix);
    np.spec.suffix = cg_names_affix(d->suffix);
    np.spec.paired = d->paired != 0;
    np.spec.has_rename = d->n_rename >= 0;
    if (np.spec.has_rename && (!np.spec.prefix.empty() || !np.spec.suffix.empty()))
        return fail(CG_EINVAL, "Option --rename cannot be combined with --prefix (-x) or --suffix (-y)");
    for (int k = 0; k < d->n_rename; ++k) {
        const cg_name_token &t = d->rename[k];
        const bool mate_ok = t.mate == 0 || (np.spec.paired && (t.mate == 1 || t.mate == 2) && t.kind != CG_NT_ID &&
                                             t.kind != CG_NT_RN && t.kind != CG_NT_LITERAL);
        if (t.kind < 0 || t.kind >= CG_NT_KINDS || !mate_ok || (t.kind == CG_NT_RC && np.spec.paired) ||
            (t.kind == CG_NT_RN && !np.spec.paired) || (t.kind == CG_NT_LITERAL && (t.len < 0 || (t.len && !t.text))))
            return fail(CG_EINVAL, "cg_names_create: rename token " + std::to_string(k) + " is not a variable of " +
                                       (np.spec.paired ? "PairedEndRenamer" : "Renamer"));
        np.spec.rename.push_back({t.kind, t.mate, t.kind == CG_NT_LITERAL ? std::string(t.text, (size_t)t.len) : std::string()});
    }
    names_build(np);
    const int32_t h = c->names_next++;
    c->names.emplace(h, std::move(np));
    *handle = h;
    return CG_OK;
}

extern "C" int cg_names_set_mate(cg_ctx *c, int32_t handle, int32_t mate, const char *names, const int32_t *offsets,
                                 int32_t n_names, const uint8_t *linked, int32_t last_cut_front, int32_t last_cut_back)
{
    if (!c || mate < 0 || mate > 1 || n_names < 0 || (n_names && (!offsets || !linked)) || last_cut_front < 0 ||
        last_cut_back < 0)
        return fail(CG_EINVAL, "cg_names_set_mate: bad argument");
    auto it = c->names.find(handle);
    if (it == c->names.end()) return fail(CG_EINVAL, "cg_names_set_mate: unknown names handle");
    NamesProg &np = it->second;
    if (n_names) {
        if (offsets[0] != 0) return fail(CG_EINVAL, "cg_names_set_mate: offsets must start at 0");
        for (int a = 0; a < n_names; ++a)
            if (offsets[a + 1] < offsets[a]) return fail(CG_EINVAL, "cg_names_set_mate: offsets must not decrease");
        if (offsets[n_names] && !names) return fail(CG_EINVAL, "cg_names_set_mate: names is NULL");
    }
    np.spec.names[mate].assign(names ? names : "", n_names ? (size_t)offsets[n_names] : 0);
    np.spec.name_off[mate].assign(offsets ? offsets : nullptr, offsets ? offsets + n_names + 1 : nullptr);
    if (!n_names) np.spec.name_off[mate].assign(1, 0);
    np.spec.linked[mate].assign(linked ? linked : nullptr, linked ? linked + n_names : nullptr);
    np.spec.cut_last[mate][0] = last_cut_front;
    np.spec.cut_last[mate][1] = last_cut_back;
    names_build(np);
    return CG_OK;
}

extern "C" int cg_names_destroy(cg_ctx *c, int32_t handle)
{
    if (!c) return fail(CG_EINVAL, "cg_names_destroy: bad argument");
    if (!c->names.erase(handle)) return fail(CG_EINVAL, "cg_names_destroy: unknown names handle");
    return CG_OK;
}

// Slot f's chunk buffer with room for `need` bytes, its first `used` bytes kept (the spare d_norm takes them)
static int names_room(FastqSlot &f, size_t used, size_t need, cudaStream_t st)
{
    if (need >= (1ull << 32))
        return fail(CG_EINVAL, "cg_fastq: the chunk and its new read names exceed 4 GiB; use smaller chunks");
    if (need <= f.d_in.cap) return CG_OK;
    int rc = f.d_norm.ensure(need);
    if (rc != CG_OK) return rc;
    if (used) CU(cudaMemcpyAsync(f.d_norm.p, f.d_in.p, used, cudaMemcpyDeviceToDevice, st));
    std::swap(f.d_in, f.d_norm);
    return CG_OK;
}

static size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// The name stage of a collect (one mate, or both of a pair), once the matches and the written part of every read are
// final and before the rows and the finish kernel: step 1 per mate (count, scan, write into an arena behind the
// chunk), then with --rename step 2 over the step-1 names into a second arena.  The record tables point at the new
// names and the writers' " rc" is off, so that every consumer reads the name as it is.
static int fastq_stage_names(cg_ctx *c, FastqSlot *const *f, FqStage *const *g, const cg_fastq_params *const *fp,
                             int n_mates, cudaStream_t st)
{
    if (fp[0]->names == 0 && (n_mates == 1 || fp[1]->names == 0)) return CG_OK;
    if (n_mates == 2 && fp[0]->names != fp[1]->names)
        return fail(CG_EINVAL, "cg_fastq_collect_paired: both mates' params must name the same names handle");
    auto it = c->names.find(fp[0]->names);
    if (it == c->names.end()) return fail(CG_EINVAL, "cg_fastq: unknown names handle");
    NamesProg &np = it->second;
    if (np.spec.paired != (n_mates == 2) && np.spec.has_rename)
        return fail(CG_EINVAL, np.spec.paired ? "cg_fastq_collect: a paired --rename template needs a paired collect"
                                         : "cg_fastq_collect_paired: a single-end --rename template on a pair");
    int rc;
    if (!np.uploaded) {
        if ((rc = np.d_blob.ensure(np.blob.size())) != CG_OK) return rc;
        CU(cudaMemcpyAsync(np.d_blob.p, np.blob.data(), np.blob.size(), cudaMemcpyHostToDevice, st));
        CU(cudaStreamSynchronize(st));
        np.uploaded = true;
    }
    const long long n = g[0]->n;
    CgNameMate m[2];
    memset(m, 0, sizeof m);
    size_t arena1[2] = {0, 0}, arena2[2] = {0, 0};
    long long total[2] = {0, 0};
    auto mate_of = [&](int i) {
        CgNameMate a;
        a.buf = f[i]->d_in.p; a.rec = f[i]->d_rec.p; a.interval = f[i]->d_interval.p; a.mask = f[i]->d_mask.p;
        a.origin = f[i]->d_origin.p; a.seq_len = f[i]->d_len.p; a.qtrim = g[i]->d_qtrim; a.matches = g[i]->d_matches;
        a.times = g[i]->times; a.slots = g[i]->slots; a.mate = i; a.rc_suffix = g[i]->rc_suffix;
        a.swapped = n_mates == 2 && g[i]->d_is_rc != nullptr;
        a.cut_front = fp[i]->cut_front; a.cut_back = fp[i]->cut_back;
        return a;
    };
    for (int i = 0; i < n_mates; ++i) {
        FastqSlot &s = *f[i];
        if ((rc = s.d_namelen.ensure((size_t)n * 2)) != CG_OK || (rc = s.d_nameoff.ensure((size_t)n * 2 + 2)) != CG_OK ||
            (rc = s.d_scan.ensure((size_t)cg_scan_tiles(n) + 1)) != CG_OK)
            return rc;
        m[i] = mate_of(i);
        const int casava = !np.spec.has_rename && fp[i]->discard_casava;
        CU(cg_launch_fastq_names(0, 0, np.d_blob.p, m[i], m[i], n, s.d_namelen.p, nullptr, nullptr, nullptr, 0, 0, 0,
                                 nullptr, st));
        CU(cg_launch_scan_i32(s.d_namelen.p, n, s.d_scan.p, s.d_nameoff.p, st));
        CU(cudaMemcpyAsync(&total[i], s.d_nameoff.p + n, sizeof total[i], cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        arena1[i] = align16((size_t)s.n_bytes);
        if ((rc = names_room(s, (size_t)s.n_bytes, arena1[i] + (size_t)total[i] + 64, st)) != CG_OK) return rc;
        m[i].buf = s.d_in.p;
        CU(cg_launch_fastq_names(1, 0, np.d_blob.p, m[i], m[i], n, nullptr, nullptr, s.d_nameoff.p, nullptr,
                                 (uint32_t)arena1[i], 0, casava, nullptr, st));
        c->launches += 5;
        g[i]->rc_suffix = 0;
        m[i].rc_suffix = 0;
    }
    if (!np.spec.has_rename) return CG_OK;
    const bool pair = n_mates == 2;
    CgNameMate none;
    memset(&none, 0, sizeof none);
    CU(cg_launch_fastq_names(0, 1, np.d_blob.p, m[0], pair ? m[1] : none, n, f[0]->d_namelen.p + n,
                             pair ? f[1]->d_namelen.p + n : nullptr, nullptr, nullptr, 0, 0, 0, nullptr, st));
    c->launches += 1;
    for (int i = 0; i < n_mates; ++i) {
        FastqSlot &s = *f[i];
        CU(cg_launch_scan_i32(s.d_namelen.p + n, n, s.d_scan.p, s.d_nameoff.p + n + 1, st));
        long long t2 = 0;
        CU(cudaMemcpyAsync(&t2, s.d_nameoff.p + 2 * n + 1, sizeof t2, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        arena2[i] = align16(arena1[i] + (size_t)total[i]);
        if ((rc = names_room(s, arena1[i] + (size_t)total[i], arena2[i] + (size_t)t2 + 64, st)) != CG_OK) return rc;
        m[i].buf = s.d_in.p;
        c->launches += 3;
    }
    if (pair) {
        if ((rc = f[0]->d_namemis.ensure(1)) != CG_OK) return rc;
        const unsigned long long unset = ~0ull;
        CU(cudaMemcpyAsync(f[0]->d_namemis.p, &unset, sizeof unset, cudaMemcpyHostToDevice, st));
    }
    CU(cg_launch_fastq_names(1, 1, np.d_blob.p, m[0], pair ? m[1] : none, n, nullptr, nullptr, f[0]->d_nameoff.p + n + 1,
                             pair ? f[1]->d_nameoff.p + n + 1 : nullptr, (uint32_t)arena2[0],
                             pair ? (uint32_t)arena2[1] : 0, (fp[0]->discard_casava ? 1 : 0) |
                             (pair && fp[1]->discard_casava ? 2 : 0), pair ? f[0]->d_namemis.p : nullptr, st));
    c->launches += 1;
    if (!pair) return CG_OK;
    unsigned long long bad = 0;
    CU(cudaMemcpyAsync(&bad, f[0]->d_namemis.p, sizeof bad, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (bad == ~0ull) return CG_OK;
    // PairedEndRenamer's messages (modifiers.py:717-735), from R1's step-1 name and the new names of the pair
    const long long p = (long long)(bad >> 1);
    auto read_name = [&](const FastqSlot &s, CgFastqRecord r, std::string *out) {
        out->resize((size_t)std::max(r.hdr_len, 0));
        if (r.hdr_len > 0) CU(cudaMemcpy(&(*out)[0], s.d_in.p + r.hdr_start, (size_t)r.hdr_len, cudaMemcpyDeviceToHost));
        return CG_OK;
    };
    auto split = [](const std::string &x, bool comment) {
        CgSpan id, cm;
        cg_name_split(cg_span((const uint8_t *)x.data(), (int)x.size()), &id, &cm);
        const CgSpan &w = comment ? cm : id;
        return std::string((const char *)w.p, (size_t)w.len);
    };
    std::string before, after[2];
    {
        int64_t o[2];
        CU(cudaMemcpy(o, f[0]->d_nameoff.p + p, sizeof o, cudaMemcpyDeviceToHost));
        CgFastqRecord r;
        r.hdr_start = (uint32_t)(arena1[0] + (size_t)o[0]);
        r.hdr_len = (int32_t)(o[1] - o[0]);
        if ((rc = read_name(*f[0], r, &before)) != CG_OK) return rc;
    }
    if ((bad & 1) == 0)                         // the reference names R1's ID and R1's comment here
        return fail(CG_EINVAL, "Input read IDs not identical: '" + split(before, false) + "' != '" + split(before, true) +
                                   "'");
    for (int k = 0; k < 2; ++k) {
        CgFastqRecord r;
        CU(cudaMemcpy(&r, f[k]->d_rec.p + p, sizeof r, cudaMemcpyDeviceToHost));
        if ((rc = read_name(*f[k], r, &after[k])) != CG_OK) return rc;
    }
    return fail(CG_EINVAL, "After renaming R1 and R2, their IDs are no longer identical: '" + split(after[0], false) +
                               "' != '" + split(after[1], false) + "'. Original read ID: '" + split(before, false) + "'. ");
}

static int fastq_collect_one(cg_ctx *c, FastqSlot &f, const cg_adapterset *s, const cg_fastq_params *fp, uint8_t *out,
                             int64_t out_capacity, cg_fastq_result *res, FqDemux *dm, int64_t *segments, FqSplit *sp)
{
    memset(res, 0, sizeof *res);
    int rc;
    if (sp && (rc = split_check(*sp, fp, "cg_fastq_collect_split")) != CG_OK) return rc;
    if ((rc = gzip_check(fp, "cg_fastq_collect")) != CG_OK) return rc;
    if ((rc = fastq_rows_check(f, s ? s->host.n_adapters : 0, "cg_fastq_collect")) != CG_OK) return rc;
    FqStage g;
    rc = fqstats_lookup(c, fp->stats, s ? s->host.n_adapters : 0, &g.acc);
    if (rc != CG_OK) return rc;
    rc = fastq_stage_evaluate(c, f, s, fp, 1, f.stream, g);
    if (rc != CG_OK || g.n == 0) return rc;
    FastqSlot *fs[1] = {&f};
    FqStage *gs[1] = {&g};
    if ((rc = fastq_stage_names(c, fs, gs, &fp, 1, f.stream)) != CG_OK) return rc;
    if ((rc = fastq_stage_rows(c, f, g, fp, f.stream)) != CG_OK) return rc;
    FqMate m;
    m.f = &f; m.g = &g; m.fp = fp; m.out = out; m.capacity = out_capacity; m.res = res; m.segments = segments;
    return fastq_collect_finish(c, &m, 1, dm, sp, 0, 0, f.stream);
}

static int fastq_collect_impl(cg_ctx *c, int32_t slot, const cg_adapterset *s, const cg_fastq_params *fp,
                              uint8_t *out, int64_t out_capacity, cg_fastq_result *res, FqDemux *dm, int64_t *segments,
                              FqSplit *sp = nullptr)
{
    if (!c || !fp || !res || slot < 0 || slot >= CG_FQ_SLOTS) return fail(CG_EINVAL, "cg_fastq_collect: bad argument");
    if (s && s->ctx != c) return fail(CG_EINVAL, "adapter set belongs to another context");
    FastqSlot &f = c->fq[slot];
    if (!f.busy) return fail(CG_EINVAL, "cg_fastq_collect: nothing was submitted to this slot");
    if (f.ilv) return fail(CG_EINVAL, "cg_fastq_collect: the slot holds a mate of an interleaved chunk, collect it as a pair");
    CU(cudaSetDevice(c->device));
    f.busy = false;
    return fastq_rows_done(f, fastq_collect_one(c, f, s, fp, out, out_capacity, res, dm, segments, sp));
}

extern "C" int cg_fastq_collect(cg_ctx *c, int32_t slot, const cg_adapterset *s, const cg_fastq_params *fp,
                                uint8_t *out, int64_t out_capacity, cg_fastq_result *res)
{
    return fastq_collect_impl(c, slot, s, fp, out, out_capacity, res, nullptr, nullptr);
}

// bit d of the destinations written as FASTA: 0 the main output (params.format), 1-3 the bits of fasta_outputs
static int split_fasta_dests(const cg_fastq_params *fp, int32_t fasta_outputs)
{
    return (fp && fp->format != CG_FORMAT_FASTQ ? 1 : 0) | (fasta_outputs << 1);
}

extern "C" int cg_fastq_collect_split(cg_ctx *c, int32_t slot, const cg_adapterset *s, const cg_fastq_params *fp,
                                      int32_t redirect, int32_t fasta_outputs, uint8_t *out, int64_t out_capacity,
                                      cg_fastq_result *res, int64_t *segments)
{
    if (!segments) return fail(CG_EINVAL, "cg_fastq_collect_split: bad argument");
    for (int d = 0; d <= FqSplit::n_dest; ++d) segments[d] = 0;
    FqSplit sp;
    sp.redirect = redirect;
    sp.fasta_dests = split_fasta_dests(fp, fasta_outputs);
    return fastq_collect_impl(c, slot, s, fp, out, out_capacity, res, nullptr, segments, &sp);
}

// cg_fastq_collect_info / _rows: a request of `kind` limited to the caller's buffer, the plain collect, the rows
static int fastq_collect_rows_into(cg_ctx *c, int32_t slot, const cg_adapterset *s, const cg_fastq_params *fp, int32_t kind,
                                   const char *text, const int32_t *text_offsets, uint8_t *out, int64_t out_capacity,
                                   uint8_t *rows_out, int64_t rows_capacity, cg_fastq_result *res, int64_t *rows_bytes,
                                   const char *who)
{
    if (!c || !s || !text || !text_offsets || !rows_bytes || rows_capacity < 0 || (rows_capacity && !rows_out) || slot < 0 ||
        slot >= CG_FQ_SLOTS)
        return fail(CG_EINVAL, std::string(who) + ": bad argument");
    *rows_bytes = 0;
    for (int a = 0; a < s->host.n_adapters; ++a)
        if (text_offsets[a] < 0 || text_offsets[a + 1] < text_offsets[a])
            return fail(CG_EINVAL, std::string(who) + (kind == CG_ROWS_INFO ? ": name_offsets" : ": text_offsets") +
                                       " must not decrease");
    int rc = cg_fastq_request_rows(c, slot, kind, text, text_offsets, s->host.n_adapters, 0);
    if (rc != CG_OK) return rc;
    FqRows &q = c->fq[slot].rows[kind];
    q.limit = rows_capacity;
    rc = fastq_collect_impl(c, slot, s, fp, out, out_capacity, res, nullptr, nullptr);
    *rows_bytes = q.bytes_plain;
    if (rc != CG_OK) return rc;
    return cg_fastq_read_rows(c, slot, kind, rows_out, rows_capacity, nullptr, nullptr);
}

extern "C" int cg_fastq_collect_info(cg_ctx *c, int32_t slot, const cg_adapterset *s, const cg_fastq_params *fp,
                                     const char *adapter_names, const int32_t *name_offsets, uint8_t *out,
                                     int64_t out_capacity, uint8_t *info_out, int64_t info_capacity, cg_fastq_result *res,
                                     int64_t *info_bytes)
{
    return fastq_collect_rows_into(c, slot, s, fp, CG_ROWS_INFO, adapter_names, name_offsets, out, out_capacity, info_out,
                                   info_capacity, res, info_bytes, "cg_fastq_collect_info");
}

extern "C" int cg_fastq_collect_rows(cg_ctx *c, int32_t slot, const cg_adapterset *s, const cg_fastq_params *fp,
                                     int32_t kind, const char *adapter_text, const int32_t *text_offsets, uint8_t *out,
                                     int64_t out_capacity, uint8_t *rows_out, int64_t rows_capacity, cg_fastq_result *res,
                                     int64_t *rows_bytes)
{
    if (kind < 0 || kind > 2) return fail(CG_EINVAL, "cg_fastq_collect_rows: kind must be 0 (info), 1 (rest) or 2 (wildcard)");
    return fastq_collect_rows_into(c, slot, s, fp, kind, adapter_text, text_offsets, out, out_capacity, rows_out,
                                   rows_capacity, res, rows_bytes,
                                   kind == CG_ROWS_INFO ? "cg_fastq_collect_info" : "cg_fastq_collect_rows");
}

static int demux_check(const cg_adapterset *s, const int32_t *adapter_dest, int32_t n_named, const char *who)
{
    if (!s || !adapter_dest || n_named < 1 || n_named > 4096) return fail(CG_EINVAL, std::string(who) + ": bad argument");
    for (int a = 0; a < s->host.n_adapters; ++a)
        if (adapter_dest[a] < 0 || adapter_dest[a] >= n_named)
            return fail(CG_EINVAL, std::string(who) + ": adapter_dest out of range");
    return CG_OK;
}

extern "C" int cg_fastq_collect_demux(cg_ctx *c, int32_t slot, const cg_adapterset *s, const cg_fastq_params *fp,
                                      const int32_t *adapter_dest, int32_t n_named, uint8_t *out, int64_t out_capacity,
                                      cg_fastq_result *res, int64_t *segments)
{
    if (!segments) return fail(CG_EINVAL, "cg_fastq_collect_demux: bad argument");
    int rc = demux_check(s, adapter_dest, n_named, "cg_fastq_collect_demux");
    if (rc != CG_OK) return rc;
    for (int d = 0; d < n_named + 2; ++d) segments[d] = 0;
    FqDemux dm;
    dm.adapter_dest1 = adapter_dest; dm.n_adapters1 = s->host.n_adapters; dm.n_named1 = n_named;
    return fastq_collect_impl(c, slot, s, fp, out, out_capacity, res, &dm, segments);
}

// --pair-adapters: sets1[i] / sets2[i] hold adapter i of the -a / -A lists alone
struct FqPairAdapters {
    const cg_adapterset *const *sets1 = nullptr;
    const cg_adapterset *const *sets2 = nullptr;
    int n_pairs = 0;
};

// PairedAdapterCutter (modifiers.py:412-503) for a chunk of pairs: every adapter pair is matched alone against both
// mates (two trimming passes), fq_pair_select_kernel keeps the best pair that matches BOTH mates.  The records the
// verdict kernels then see name the pair in `adapter`.
static int fastq_stage_pair_adapters(cg_ctx *c, FastqSlot &f1, FastqSlot &f2, const FqPairAdapters &pa,
                                     const cg_fastq_params *fp1, const cg_fastq_params *fp2, cudaStream_t st, FqStage &g1,
                                     FqStage &g2)
{
    int rc;
    if ((rc = fastq_stage_records(c, f1, fp1, true, st, g1)) != CG_OK) return rc;
    if ((rc = fastq_stage_records(c, f2, fp2, true, st, g2)) != CG_OK) return rc;
    if (g1.n != g2.n || g1.n == 0) return CG_OK;       // the caller reports the mismatch
    for (const cg_fastq_params *fp : {fp1, fp2})
        if (fp->action == CG_FQ_ACTION_LOWERCASE || fp->action == CG_FQ_ACTION_CROP)
            return fail(CG_EINVAL, "--pair-adapters supports the actions trim, none, mask and retain");
    const long long n = g1.n;
    int slots = 1;
    for (int i = 0; i < pa.n_pairs; ++i) slots = std::max(slots, std::max(pa.sets1[i]->host.slots, pa.sets2[i]->host.slots));
    g1.times = g2.times = 1;
    g1.slots = g2.slots = slots;
    // the quality trimmers come before the cutter in the chain (cli.py:940-1000): fold them into the records
    if ((rc = fastq_stage_fold_qtrim(c, f1, &fp1->trim, st, g1)) != CG_OK) return rc;
    if ((rc = fastq_stage_fold_qtrim(c, f2, &fp2->trim, st, g2)) != CG_OK) return rc;
    if ((rc = fastq_stage_pack(c, f1, st, g1, false)) != CG_OK) return rc;
    if ((rc = fastq_stage_pack(c, f2, st, g2, false)) != CG_OK) return rc;
    for (FastqSlot *f : {&f1, &f2}) {
        if ((rc = f->d_matches.ensure((size_t)n * slots)) != CG_OK) return rc;
        if ((rc = f->d_matches_rc.ensure((size_t)n * slots)) != CG_OK) return rc;     // records of the pair being tried
    }
    if ((rc = f1.d_pairkey.ensure((size_t)n * 2)) != CG_OK) return rc;
    cg_params p1 = fp1->trim, p2 = fp2->trim;
    p1.quality_trim = p1.nextseq_trim = p2.quality_trim = p2.nextseq_trim = 0;
    p1.times = p2.times = 1;
    for (int i = 0; i < pa.n_pairs; ++i) {
        rc = launch_trim(c, pa.sets1[i], f1.d_seq.p, nullptr, f1.d_offs.p, n, g1.max_len, &p1, f1.d_matches_rc.p, nullptr, st,
                         true);
        if (rc != CG_OK) return rc;
        rc = launch_trim(c, pa.sets2[i], f2.d_seq.p, nullptr, f2.d_offs.p, n, g2.max_len, &p2, f2.d_matches_rc.p, nullptr, st,
                         true);
        if (rc != CG_OK) return rc;
        CU(cg_launch_fastq_pair_select(n, i, f1.d_matches_rc.p, pa.sets1[i]->host.slots, f2.d_matches_rc.p,
                                       pa.sets2[i]->host.slots, f1.d_matches.p, f2.d_matches.p, slots, f1.d_pairkey.p, st));
        c->launches += 1;
    }
    g1.d_matches = f1.d_matches.p;
    g2.d_matches = f2.d_matches.p;
    int kmax1 = 0, kmax2 = 0;
    for (int i = 0; i < pa.n_pairs; ++i) {
        kmax1 = std::max(kmax1, pa.sets1[i]->host.max_k);
        kmax2 = std::max(kmax2, pa.sets2[i]->host.max_k);
    }
    if ((rc = fastq_stage_stats(c, f1, g1, kmax1, st)) != CG_OK) return rc;
    if ((rc = fastq_stage_stats(c, f2, g2, kmax2, st)) != CG_OK) return rc;
    if ((rc = fastq_stage_verdict(c, f1, fp1, 1, st, g1)) != CG_OK) return rc;
    return fastq_stage_verdict(c, f2, fp2, 2, st, g2);
}

// PairedReverseComplementer (modifiers.py:311-400) for a chunk of pairs, at least one set given.  Each mate's own
// modifiers in front of the cutters (-u, --nextseq-trim, -q) are folded into its records; then up to four trimming
// passes: m11 = set1 on slot 1, m22 = set2 on slot 2, m12 = set1 on slot 2, m21 = set2 on slot 1 (a cross pass is laid
// out for its set, so a slot's matches keep its own set's layout after the swap).  Each slot's chunk gets the other
// slot's chunk appended, and fq_pair_swap_kernel moves the records of the swapped pairs across.  From there on the
// pair is written, filtered, routed and counted like any other.
static int fastq_stage_paired_revcomp(cg_ctx *c, FastqSlot &f1, FastqSlot &f2, const cg_adapterset *s1,
                                      const cg_adapterset *s2, const cg_fastq_params *fp1, const cg_fastq_params *fp2,
                                      cudaStream_t st, FqStage &g1, FqStage &g2)
{
    int rc;
    if ((rc = fastq_stage_records(c, f1, fp1, s1 != nullptr, st, g1)) != CG_OK) return rc;
    if ((rc = fastq_stage_records(c, f2, fp2, s2 != nullptr, st, g2)) != CG_OK) return rc;
    if (g1.n != g2.n || g1.n == 0) return CG_OK;       // the caller reports the mismatch
    const long long n = g1.n;
    const int64_t b1 = f1.n_bytes, b2 = f2.n_bytes;
    if (b1 + b2 > (int64_t)UINT32_MAX)
        return fail(CG_EINVAL, "--revcomp on pairs: the two chunks of a pair must hold less than 4 GiB together");
    g1.slots = s1 ? s1->host.slots : 1;
    g2.slots = s2 ? s2->host.slots : 1;
    const int per1 = g1.times * g1.slots, per2 = g2.times * g2.slots;
    if ((rc = fastq_stage_fold_qtrim(c, f1, &fp1->trim, st, g1)) != CG_OK) return rc;
    if ((rc = fastq_stage_fold_qtrim(c, f2, &fp2->trim, st, g2)) != CG_OK) return rc;
    if ((rc = fastq_stage_pack(c, f1, st, g1, false)) != CG_OK) return rc;
    if ((rc = fastq_stage_pack(c, f2, st, g2, false)) != CG_OK) return rc;
    cg_params p1 = fp1->trim, p2 = fp2->trim;
    p1.quality_trim = p1.nextseq_trim = p2.quality_trim = p2.nextseq_trim = 0;
    // slot 1: d_matches = m11, d_matches_rc = m21; slot 2: d_matches = m22, d_matches_rc = m12
    if (s1) {
        if ((rc = f1.d_matches.ensure((size_t)n * per1)) != CG_OK) return rc;
        if ((rc = f2.d_matches_rc.ensure((size_t)n * per1)) != CG_OK) return rc;
        if ((rc = launch_trim(c, s1, f1.d_seq.p, nullptr, f1.d_offs.p, n, g1.max_len, &p1, f1.d_matches.p, nullptr, st,
                              true)) != CG_OK)
            return rc;
        if ((rc = launch_trim(c, s1, f2.d_seq.p, nullptr, f2.d_offs.p, n, g2.max_len, &p1, f2.d_matches_rc.p, nullptr, st,
                              true)) != CG_OK)
            return rc;
    }
    if (s2) {
        if ((rc = f2.d_matches.ensure((size_t)n * per2)) != CG_OK) return rc;
        if ((rc = f1.d_matches_rc.ensure((size_t)n * per2)) != CG_OK) return rc;
        if ((rc = launch_trim(c, s2, f2.d_seq.p, nullptr, f2.d_offs.p, n, g2.max_len, &p2, f2.d_matches.p, nullptr, st,
                              true)) != CG_OK)
            return rc;
        if ((rc = launch_trim(c, s2, f1.d_seq.p, nullptr, f1.d_offs.p, n, g1.max_len, &p2, f1.d_matches_rc.p, nullptr, st,
                              true)) != CG_OK)
            return rc;
    }
    // slot 1's chunk becomes [chunk1 | chunk2], slot 2's [chunk2 | chunk1]: the writers, the rows and the statistics
    // then find a record that moved to the other slot in that slot's own chunk
    if ((rc = f1.d_norm.ensure((size_t)(b1 + b2) + 64)) != CG_OK) return rc;
    if ((rc = f2.d_norm.ensure((size_t)(b1 + b2) + 64)) != CG_OK) return rc;
    if (b1) {
        CU(cudaMemcpyAsync(f1.d_norm.p, f1.d_in.p, (size_t)b1, cudaMemcpyDeviceToDevice, st));
        CU(cudaMemcpyAsync(f2.d_norm.p + b2, f1.d_in.p, (size_t)b1, cudaMemcpyDeviceToDevice, st));
    }
    if (b2) {
        CU(cudaMemcpyAsync(f2.d_norm.p, f2.d_in.p, (size_t)b2, cudaMemcpyDeviceToDevice, st));
        CU(cudaMemcpyAsync(f1.d_norm.p + b1, f2.d_in.p, (size_t)b2, cudaMemcpyDeviceToDevice, st));
    }
    std::swap(f1.d_in, f1.d_norm);
    std::swap(f2.d_in, f2.d_norm);
    f1.n_bytes = f2.n_bytes = b1 + b2;               // what the packed reads of either slot can now need
    if ((rc = f1.d_isrc.ensure((size_t)n)) != CG_OK) return rc;
    if ((rc = f2.d_isrc.ensure((size_t)n)) != CG_OK) return rc;
    CU(cg_launch_fastq_pair_swap(n, f1.d_rec.p, f1.d_len.p, f1.d_origin.p, s1 ? f1.d_matches.p : nullptr,
                                 s2 ? f1.d_matches_rc.p : nullptr, per1, f2.d_rec.p, f2.d_len.p, f2.d_origin.p,
                                 s2 ? f2.d_matches.p : nullptr, s1 ? f2.d_matches_rc.p : nullptr, per2, (uint32_t)b1,
                                 (uint32_t)b2, f1.d_isrc.p, f2.d_isrc.p, f1.d_counters.p + 1, f2.d_counters.p + 1, st));
    c->launches += 1;
    for (FqStage *g : {&g1, &g2}) {
        g->d_is_rc = (g == &g1 ? f1 : f2).d_isrc.p;
        g->rc_suffix = fp1->revcomp == 1;
        g->packed = false;                           // the statistics pack the swapped reads again
    }
    g1.d_matches = s1 ? f1.d_matches.p : nullptr;
    g2.d_matches = s2 ? f2.d_matches.p : nullptr;
    if ((rc = fastq_stage_stats(c, f1, g1, s1 ? s1->host.max_k : 0, st)) != CG_OK) return rc;
    if ((rc = fastq_stage_stats(c, f2, g2, s2 ? s2->host.max_k : 0, st)) != CG_OK) return rc;
    if ((rc = fastq_stage_verdict(c, f1, fp1, 1, st, g1)) != CG_OK) return rc;
    return fastq_stage_verdict(c, f2, fp2, 2, st, g2);
}

static int fastq_collect_paired_run(cg_ctx *c, int32_t slot1, int32_t slot2, const cg_adapterset *s1,
                                    const cg_adapterset *s2, const FqPairAdapters *pa, const cg_fastq_params *fp1,
                                    const cg_fastq_params *fp2, int32_t pair_filter_mode, uint8_t *out1,
                                    int64_t out_capacity1, uint8_t *out2, int64_t out_capacity2, cg_fastq_result *res1,
                                    cg_fastq_result *res2, FqDemux *dm, int64_t *segments1, int64_t *segments2,
                                    FqSplit *sp)
{
    if (!c || !fp1 || !fp2 || !res1 || !res2 || slot1 < 0 || slot1 >= CG_FQ_SLOTS || slot2 < 0 || slot2 >= CG_FQ_SLOTS ||
        slot1 == slot2 || pair_filter_mode < 0 || pair_filter_mode > 2)
        return fail(CG_EINVAL, "cg_fastq_collect_paired: bad argument");
    if ((s1 && s1->ctx != c) || (s2 && s2->ctx != c)) return fail(CG_EINVAL, "adapter set belongs to another context");
    if (fp1->revcomp != fp2->revcomp)
        return fail(CG_EINVAL, "cg_fastq_collect_paired: --revcomp is one option for the pair, params1.revcomp and "
                               "params2.revcomp must be equal");
    if (pa && fp1->revcomp) return fail(CG_EINVAL, "Cannot use --revcomp with --pair-adapters");   // cli.py:1086-1087
    FastqSlot &f1 = c->fq[slot1], &f2 = c->fq[slot2];
    if (!f1.busy || !f2.busy) return fail(CG_EINVAL, "cg_fastq_collect_paired: nothing was submitted to a slot");
    if ((f1.ilv || f2.ilv) && (f1.ilv != 1 || f2.ilv != 2 || f1.ilv_peer != slot2 || f2.ilv_peer != slot1))
        return fail(CG_EINVAL, "cg_fastq_collect_paired: the two slots were not submitted together (an interleaved chunk's "
                               "slots go in the order cg_fastq_submit_interleaved gave them)");
    CU(cudaSetDevice(c->device));
    f1.busy = f2.busy = false;
    // The slots are free again: every exit waits until mate 2's upload, on its own stream, is done with the caller's
    // buffer and the slot's.  Everything after it runs on mate 1's stream.
    struct StreamWait {
        cudaStream_t s;
        ~StreamWait() { cudaStreamSynchronize(s); }
    } wait_mate2{f2.stream};
    if (fp1->format != fp2->format) return fail(CG_EINVAL, "cg_fastq_collect_paired: both mates must have the same format");
    memset(res1, 0, sizeof *res1);
    memset(res2, 0, sizeof *res2);
    cudaStream_t st = f1.stream;
    FqStage g1, g2;
    int rc;
    if (f1.ilv) {
        if ((fp1->format == CG_FORMAT_FASTA) != (f1.ilv_format == CG_FORMAT_FASTA))
            return fail(CG_EINVAL, "cg_fastq_collect_paired: the input format of the parameters is not the one the "
                                   "interleaved chunk was submitted with");
        if ((rc = fastq_split_interleaved(c, f1, f2, st)) != CG_OK) return rc;
    }
    // one statistics accumulator per mate, as the reference keeps per-mate statistics (report.py:162-208)
    if (fp1->stats != 0 && fp1->stats == fp2->stats)
        return fail(CG_EINVAL, "cg_fastq_collect_paired: the two mates need different statistics handles");
    if (sp && ((rc = split_check(*sp, fp1, "cg_fastq_collect_paired_split")) != CG_OK ||
               (rc = split_check(*sp, fp2, "cg_fastq_collect_paired_split")) != CG_OK))
        return rc;
    if ((rc = gzip_check(fp1, "cg_fastq_collect_paired")) != CG_OK || (rc = gzip_check(fp2, "cg_fastq_collect_paired")) != CG_OK)
        return rc;
    if (sp && sp->interleaved) {
        // an interleaved destination holds both mates: both must agree on compressing it
        const int ilv_bits = ((sp->ilv_dests & 1) ? CG_GZIP_MAIN : 0) | (sp->ilv_dests >> 1);
        if ((fp1->gzip_outputs ^ fp2->gzip_outputs) & ilv_bits)
            return fail(CG_EINVAL, "cg_fastq_collect_paired_interleaved: an interleaved output must have its gzip_outputs bit "
                                   "set alike in both mates' parameters");
    }
    const int n_entries1 = pa ? pa->n_pairs : (s1 ? s1->host.n_adapters : 0);
    const int n_entries2 = pa ? pa->n_pairs : (s2 ? s2->host.n_adapters : 0);
    if ((rc = fastq_rows_check(f1, n_entries1, "cg_fastq_collect_paired (mate 1)")) != CG_OK ||
        (rc = fastq_rows_check(f2, n_entries2, "cg_fastq_collect_paired (mate 2)")) != CG_OK)
        return rc;
    // the reference builds the info row of a swapped pair from R1's own input read with the coordinates of the match
    // on r2 (steps.py:233-247); that row is not produced here
    if (fp1->revcomp && (f1.rows[CG_ROWS_INFO].requested || f2.rows[CG_ROWS_INFO].requested))
        return fail(CG_EINVAL, "cg_fastq_collect_paired: info rows (--info-file) cannot be combined with --revcomp on "
                               "pairs; rest and wildcard rows can");
    if ((rc = fqstats_lookup(c, fp1->stats, n_entries1, &g1.acc)) != CG_OK ||
        (rc = fqstats_lookup(c, fp2->stats, n_entries2, &g2.acc)) != CG_OK)
        return rc;
    if (pa) {
        if ((rc = fastq_stage_pair_adapters(c, f1, f2, *pa, fp1, fp2, st, g1, g2)) != CG_OK) return rc;
    } else if (fp1->revcomp && (s1 || s2)) {        // without adapters --revcomp does nothing (cli.py:1103-1110)
        if ((rc = fastq_stage_paired_revcomp(c, f1, f2, s1, s2, fp1, fp2, st, g1, g2)) != CG_OK) return rc;
    } else {
        if ((rc = fastq_stage_evaluate(c, f1, s1, fp1, 1, st, g1)) != CG_OK) return rc;
        if ((rc = fastq_stage_evaluate(c, f2, s2, fp2, 2, st, g2)) != CG_OK) return rc;
    }
    if (g1.n != g2.n)
        return fail(CG_EINVAL, "paired FASTQ chunks differ in their number of records (" + std::to_string(g1.n) + " vs " +
                                   std::to_string(g2.n) + ")");
    if (g1.n == 0) return CG_OK;
    {
        FastqSlot *fs[2] = {&f1, &f2};
        FqStage *gs[2] = {&g1, &g2};
        const cg_fastq_params *fps[2] = {fp1, fp2};
        if ((rc = fastq_stage_names(c, fs, gs, fps, 2, st)) != CG_OK) return rc;
    }
    if ((rc = fastq_stage_rows(c, f1, g1, fp1, st)) != CG_OK || (rc = fastq_stage_rows(c, f2, g2, fp2, st)) != CG_OK)
        return rc;
    // --discard-untrimmed with adapters on one mate only tests "both" (cli.py:859-893)
    const int mode_untrimmed = (!pa && (!s1 || !s2)) ? 1 : pair_filter_mode;
    FqMate m[2];
    m[0].f = &f1; m[0].g = &g1; m[0].fp = fp1; m[0].out = out1; m[0].capacity = out_capacity1; m[0].res = res1;
    m[0].segments = segments1;
    m[1].f = &f2; m[1].g = &g2; m[1].fp = fp2; m[1].out = out2; m[1].capacity = out_capacity2; m[1].res = res2;
    m[1].segments = segments2;
    return fastq_collect_finish(c, m, 2, dm, sp, pair_filter_mode, mode_untrimmed, st);
}

static int fastq_collect_paired_impl(cg_ctx *c, int32_t slot1, int32_t slot2, const cg_adapterset *s1,
                                     const cg_adapterset *s2, const FqPairAdapters *pa, const cg_fastq_params *fp1,
                                     const cg_fastq_params *fp2, int32_t pair_filter_mode, uint8_t *out1,
                                     int64_t out_capacity1, uint8_t *out2, int64_t out_capacity2, cg_fastq_result *res1,
                                     cg_fastq_result *res2, FqDemux *dm, int64_t *segments1, int64_t *segments2,
                                     FqSplit *sp = nullptr)
{
    const int rc = fastq_collect_paired_run(c, slot1, slot2, s1, s2, pa, fp1, fp2, pair_filter_mode, out1, out_capacity1,
                                            out2, out_capacity2, res1, res2, dm, segments1, segments2, sp);
    if (c && slot1 >= 0 && slot1 < CG_FQ_SLOTS && slot2 >= 0 && slot2 < CG_FQ_SLOTS && slot1 != slot2) {
        fastq_rows_done(c->fq[slot1], rc);
        fastq_rows_done(c->fq[slot2], rc);
    }
    return rc;
}

extern "C" int cg_fastq_collect_paired(cg_ctx *c, int32_t slot1, int32_t slot2, const cg_adapterset *s1,
                                       const cg_adapterset *s2, const cg_fastq_params *fp1, const cg_fastq_params *fp2,
                                       int32_t pair_filter_mode, uint8_t *out1, int64_t out_capacity1, uint8_t *out2,
                                       int64_t out_capacity2, cg_fastq_result *res1, cg_fastq_result *res2)
{
    return fastq_collect_paired_impl(c, slot1, slot2, s1, s2, nullptr, fp1, fp2, pair_filter_mode, out1, out_capacity1, out2,
                                     out_capacity2, res1, res2, nullptr, nullptr, nullptr);
}

extern "C" int cg_fastq_collect_paired_split(cg_ctx *c, int32_t slot1, int32_t slot2, const cg_adapterset *s1,
                                             const cg_adapterset *s2, const cg_fastq_params *fp1, const cg_fastq_params *fp2,
                                             int32_t pair_filter_mode, int32_t redirect, int32_t fasta_outputs,
                                             uint8_t *out1, int64_t out_capacity1, uint8_t *out2, int64_t out_capacity2,
                                             cg_fastq_result *res1, cg_fastq_result *res2, int64_t *segments1,
                                             int64_t *segments2)
{
    if (!segments1 || !segments2) return fail(CG_EINVAL, "cg_fastq_collect_paired_split: bad argument");
    for (int d = 0; d <= FqSplit::n_dest; ++d) segments1[d] = segments2[d] = 0;
    FqSplit sp;
    sp.redirect = redirect;
    sp.fasta_dests = split_fasta_dests(fp1, fasta_outputs);
    return fastq_collect_paired_impl(c, slot1, slot2, s1, s2, nullptr, fp1, fp2, pair_filter_mode, out1, out_capacity1, out2,
                                     out_capacity2, res1, res2, nullptr, segments1, segments2, &sp);
}

extern "C" int cg_fastq_collect_paired_interleaved(cg_ctx *c, int32_t slot1, int32_t slot2, const cg_adapterset *s1,
                                                   const cg_adapterset *s2, const cg_fastq_params *fp1,
                                                   const cg_fastq_params *fp2, int32_t pair_filter_mode, int32_t redirect,
                                                   int32_t fasta_outputs, int32_t interleaved_outputs, uint8_t *out1,
                                                   int64_t out_capacity1, uint8_t *out2, int64_t out_capacity2,
                                                   cg_fastq_result *res1, cg_fastq_result *res2, int64_t *segments1,
                                                   int64_t *segments2)
{
    if (!segments1 || !segments2) return fail(CG_EINVAL, "cg_fastq_collect_paired_interleaved: bad argument");
    if (interleaved_outputs & ~(CG_INTERLEAVE_MAIN | 7))
        return fail(CG_EINVAL, "cg_fastq_collect_paired_interleaved: interleaved_outputs takes CG_INTERLEAVE_MAIN and "
                               "CG_REDIRECT_* bits only");
    for (int d = 0; d <= FqSplit::n_dest; ++d) segments1[d] = segments2[d] = 0;
    FqSplit sp;
    sp.redirect = redirect;
    sp.fasta_dests = split_fasta_dests(fp1, fasta_outputs);
    sp.interleaved = true;
    sp.ilv_dests = ((interleaved_outputs & CG_INTERLEAVE_MAIN) ? 1 : 0) | ((interleaved_outputs & 7) << 1);
    return fastq_collect_paired_impl(c, slot1, slot2, s1, s2, nullptr, fp1, fp2, pair_filter_mode, out1, out_capacity1, out2,
                                     out_capacity2, res1, res2, nullptr, segments1, segments2, &sp);
}

extern "C" int cg_fastq_collect_pair_adapters(cg_ctx *c, int32_t slot1, int32_t slot2, const cg_adapterset *const *sets1,
                                              const cg_adapterset *const *sets2, int32_t n_pairs,
                                              const cg_fastq_params *fp1, const cg_fastq_params *fp2,
                                              int32_t pair_filter_mode, uint8_t *out1, int64_t out_capacity1, uint8_t *out2,
                                              int64_t out_capacity2, cg_fastq_result *res1, cg_fastq_result *res2)
{
    if (!c || !sets1 || !sets2 || n_pairs < 1)
        return fail(CG_EINVAL, "cg_fastq_collect_pair_adapters: the adapter lists must have the same, non-zero length");
    for (int i = 0; i < n_pairs; ++i) {
        if (!sets1[i] || !sets2[i] || sets1[i]->ctx != c || sets2[i]->ctx != c)
            return fail(CG_EINVAL, "cg_fastq_collect_pair_adapters: bad adapter set");
        if (sets1[i]->host.n_groups != 1 || sets2[i]->host.n_groups != 1)
            return fail(CG_EINVAL, "cg_fastq_collect_pair_adapters: every set must hold exactly one adapter");
    }
    FqPairAdapters pa;
    pa.sets1 = sets1; pa.sets2 = sets2; pa.n_pairs = n_pairs;
    return fastq_collect_paired_impl(c, slot1, slot2, sets1[0], sets2[0], &pa, fp1, fp2, pair_filter_mode, out1, out_capacity1,
                                     out2, out_capacity2, res1, res2, nullptr, nullptr, nullptr);
}

extern "C" int cg_fastq_collect_paired_demux(cg_ctx *c, int32_t slot1, int32_t slot2, const cg_adapterset *s1,
                                             const cg_adapterset *s2, const cg_fastq_params *fp1, const cg_fastq_params *fp2,
                                             int32_t pair_filter_mode, const int32_t *adapter_dest1, int32_t n_named1,
                                             const int32_t *adapter_dest2, int32_t n_named2, const uint8_t *dest_keep,
                                             uint8_t *out1, int64_t out_capacity1, uint8_t *out2, int64_t out_capacity2,
                                             cg_fastq_result *res1, cg_fastq_result *res2, int64_t *segments1,
                                             int64_t *segments2)
{
    if (!segments1 || !segments2) return fail(CG_EINVAL, "cg_fastq_collect_paired_demux: bad argument");
    int rc = demux_check(s1, adapter_dest1, n_named1, "cg_fastq_collect_paired_demux");
    if (rc != CG_OK) return rc;
    if (adapter_dest2 && (rc = demux_check(s2, adapter_dest2, n_named2, "cg_fastq_collect_paired_demux")) != CG_OK) return rc;
    FqDemux dm;
    dm.adapter_dest1 = adapter_dest1; dm.n_adapters1 = s1->host.n_adapters; dm.n_named1 = n_named1;
    if (adapter_dest2) { dm.adapter_dest2 = adapter_dest2; dm.n_adapters2 = s2->host.n_adapters; dm.n_named2 = n_named2; }
    dm.dest_keep = dest_keep;
    if ((long long)dm.n_dest() > 8192) return fail(CG_EINVAL, "cg_fastq_collect_paired_demux: more than 8192 destinations");
    for (int d = 0; d < dm.n_dest() + 1; ++d) segments1[d] = segments2[d] = 0;
    return fastq_collect_paired_impl(c, slot1, slot2, s1, s2, nullptr, fp1, fp2, pair_filter_mode, out1, out_capacity1, out2,
                                     out_capacity2, res1, res2, &dm, segments1, segments2);
}

extern "C" int cg_fastq_trim_chunk(cg_ctx *c, const cg_adapterset *s, const uint8_t *fastq, int64_t n_bytes,
                                   const cg_fastq_params *fp, uint8_t *out, int64_t out_capacity, cg_fastq_result *res)
{
    int32_t slot = -1;
    int rc = cg_fastq_submit(c, fastq, n_bytes, &slot);
    if (rc != CG_OK) return rc;
    return cg_fastq_collect(c, slot, s, fp, out, out_capacity, res);
}

extern "C" int cg_fastq_stats_create(cg_ctx *c, int32_t n_adapters, int32_t *handle)
{
    if (!c || !handle || n_adapters < 0) return fail(CG_EINVAL, "cg_fastq_stats_create: bad argument");
    FqStatsAcc a;
    a.n_adapters = n_adapters;
    a.v.assign((size_t)fqstats_total(n_adapters, 0, 0), 0);
    const int32_t h = c->fq_stats_next++;
    c->fq_stats[h] = std::move(a);
    *handle = h;
    return CG_OK;
}

extern "C" int cg_fastq_stats_read(cg_ctx *c, int32_t handle, int32_t *max_len, int32_t *kmax, int64_t *out, int64_t capacity,
                                   int64_t *size, int reset)
{
    if (!c) return fail(CG_EINVAL, "cg_fastq_stats_read: ctx is NULL");
    auto it = c->fq_stats.find(handle);
    if (it == c->fq_stats.end()) return fail(CG_EINVAL, "cg_fastq_stats_read: unknown handle " + std::to_string(handle));
    FqStatsAcc &a = it->second;
    const int64_t n = (int64_t)a.v.size();
    if (max_len) *max_len = a.max_len;
    if (kmax) *kmax = a.kmax;
    if (size) *size = n;
    if (!out) return CG_OK;
    if (capacity < n)
        return fail(CG_EINVAL, "cg_fastq_stats_read: the vector has " + std::to_string(n) + " entries, capacity is " +
                                   std::to_string(capacity));
    memcpy(out, a.v.data(), (size_t)n * sizeof(int64_t));
    if (reset) std::fill(a.v.begin(), a.v.end(), 0);
    return CG_OK;
}

extern "C" int cg_fastq_stats_destroy(cg_ctx *c, int32_t handle)
{
    if (!c || !c->fq_stats.erase(handle)) return fail(CG_EINVAL, "cg_fastq_stats_destroy: unknown handle");
    return CG_OK;
}
