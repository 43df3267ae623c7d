// cg_bam_core.cuh -- every decision of the unaligned-BAM input path (cg_bam.cu), host + device: the header, the record
// check, the tile walk that finds the record boundaries in parallel and its resolve, the refusals, and the FASTQ text of
// a record.
//
// The plain stream (after BGZF inflation) is the BAM header -- "BAM\1", l_text, the text, n_ref, n_ref x (l_name, name,
// l_ref) -- followed by records: block_size (int32), then block_size bytes: the 32-byte fixed part (refID, pos,
// l_read_name, mapq, bin, n_cigar_op, flag, l_seq, next_refID, next_pos, tlen), the NUL-terminated name, 4 x n_cigar_op
// bytes of CIGAR, (l_seq + 1) / 2 bytes of 4-bit sequence, l_seq quality bytes, the aux tags.
//
// Record boundaries: the buffer is cut into tiles of `tile` bytes (a multiple of 32).  Each tile walks speculatively
// from its first offset where bam_candidate passes (tile 0 from 0), p -> p + 4 + block_size, and marks every offset it
// visits in a bitmap (one bit per byte; a tile's words belong to its walk alone).  Its exit is the first offset at or
// behind the tile's end, or the offset where a record is short or invalid.  The resolve follows the true chain from
// offset 0 tile by tile: an entry on the tile's walk takes the walk's exit; any other entry is walked again until it
// meets the walk's marks (then the walk's exit holds) or leaves the tile, and the tile's marks in front of that point
// are rewritten.  The true record starts are then the marked offsets from each tile's entry up to the chain's end.
#pragma once
#include "cg_types.h"

#define BAM_TILE 8192          // bytes per tile of the record-boundary walk (a multiple of 32)
#define BAM_FIXED 32           // the fixed part of a record behind block_size
#define BAM_MIN_RECORD 36      // block_size + fixed part: no record is shorter

// bam_check / link-word status
#define BAM_OK 0
#define BAM_SHORT 1            // the record runs past the bytes given
#define BAM_BAD 2              // structurally invalid (CG_EINVAL)
#define BAM_NONE 3             // link word of a tile without a speculative walk

// refusals of a structurally valid record, in the order they are tested (the smallest code of the first record wins)
#define BAM_R_FLAG 1           // flag != 4: dnaio reads unmapped single reads only (CG_EUNSUPPORTED)
#define BAM_R_NAME 2           // a name byte outside 0x21..0x7E (CG_EINVAL)
#define BAM_R_NOQUAL 3         // l_seq > 0 and the first quality byte 0xFF: no qualities (CG_EUNSUPPORTED)
#define BAM_R_QUAL 4           // a quality value above 93 (CG_EINVAL)
#define BAM_R_STRUCT 5         // bam_check BAM_BAD (CG_EINVAL)

// header: bam_header's *why
#define BAM_H_MAGIC 1
#define BAM_H_NEGATIVE 2

// What the resolve and the cut leave for the host (one readback)
struct BamSum {
    long long end;             // offset where the chain stops: behind the last whole record, or at a short / bad one
    int32_t end_st;            // BAM_OK (end == n), BAM_SHORT or BAM_BAD
    int32_t pad;
    long long rewalked;        // tiles whose entry was not on their speculative walk
    long long n_rec;           // records of the chain
    long long n_cut;           // records of the cut (their FASTQ text under the limit)
    long long fq_bytes;        // FASTQ bytes of the cut
    long long bam_cut;         // offset behind the cut's last record
};

CG_HD int32_t bam_i32(const uint8_t *b)
{
    return (int32_t)((uint32_t)b[0] | ((uint32_t)b[1] << 8) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 24));
}

CG_HD int bam_u16(const uint8_t *b) { return b[0] | (b[1] << 8); }

// The header of b[0, n): BAM_OK with *len its size, BAM_SHORT when more bytes are needed, BAM_BAD (*why BAM_H_*).
CG_HD int bam_header(const uint8_t *b, long long n, long long *len, int *why)
{
    const uint8_t magic[4] = {'B', 'A', 'M', 1};
    for (long long i = 0; i < 4 && i < n; ++i)
        if (b[i] != magic[i]) { *why = BAM_H_MAGIC; return BAM_BAD; }
    if (n < 12) return BAM_SHORT;
    const int32_t l_text = bam_i32(b + 4);
    if (l_text < 0) { *why = BAM_H_NEGATIVE; return BAM_BAD; }
    long long p = 8 + (long long)l_text;
    if (p + 4 > n) return BAM_SHORT;
    const int32_t n_ref = bam_i32(b + p);
    if (n_ref < 0) { *why = BAM_H_NEGATIVE; return BAM_BAD; }
    p += 4;
    for (int32_t i = 0; i < n_ref; ++i) {
        if (p + 4 > n) return BAM_SHORT;
        const int32_t l_name = bam_i32(b + p);
        if (l_name < 1) { *why = BAM_H_NEGATIVE; return BAM_BAD; }
        p += 4 + (long long)l_name + 4;
        if (p > n) return BAM_SHORT;
    }
    *len = p;
    return BAM_OK;
}

// The record at b[p] of b[0, n): BAM_OK (*next = p + 4 + block_size), BAM_SHORT or BAM_BAD.  Structurally valid:
// block_size >= 32, l_read_name >= 1, l_seq >= 0, 32 + l_read_name + 4 n_cigar_op + (l_seq + 1) / 2 + l_seq <= block_size,
// and the name's last byte is NUL.  The fixed part is judged as soon as it is there, the NUL once the record is whole.
CG_HD int bam_check(const uint8_t *b, long long n, long long p, long long *next)
{
    if (p + 4 > n) return BAM_SHORT;
    const int32_t bs = bam_i32(b + p);
    if (bs < BAM_FIXED) return BAM_BAD;
    if (p + BAM_MIN_RECORD > n) return BAM_SHORT;
    const uint8_t *r = b + p + 4;
    const int lrn = r[8];
    const long long ncig = bam_u16(r + 12);
    const int32_t lseq = bam_i32(r + 16);
    if (lrn < 1 || lseq < 0) return BAM_BAD;
    if (BAM_FIXED + lrn + 4 * ncig + ((long long)lseq + 1) / 2 + lseq > bs) return BAM_BAD;
    if (p + 4 + (long long)bs > n) return BAM_SHORT;
    if (r[BAM_FIXED + lrn - 1] != 0) return BAM_BAD;
    *next = p + 4 + bs;
    return BAM_OK;
}

// Where a tile's speculative walk may start: a record that passes bam_check, whose refID and next_refID are at least -1
// and whose successor is not structurally invalid.  Only the speed depends on this choice (a wrong start costs a walk
// again); the extra tests reject the offsets just in front of a true record, whose block_size bytes shift into a
// plausible fixed part.
CG_HD bool bam_candidate(const uint8_t *b, long long n, long long p)
{
    long long nx = 0, nx2 = 0;
    if (bam_check(b, n, p, &nx) != BAM_OK) return false;
    if (bam_i32(b + p + 4) < -1 || bam_i32(b + p + 4 + 20) < -1) return false;
    return nx >= n || bam_check(b, n, nx, &nx2) != BAM_BAD;
}

// FASTQ bytes of a record: '@' + l_read_name - 1 name bytes + '\n' + l_seq + "\n+\n" + l_seq + '\n'
CG_HD long long bam_fastq_size(const uint8_t *rec) { return rec[4 + 8] + 2LL * bam_i32(rec + 4 + 16) + 5; }

CG_HD char bam_base(int nibble) { return "=ACMGRSVTWYHKDBN"[nibble & 15]; }
CG_HD bool bam_name_ok(uint8_t c) { return c >= 0x21 && c <= 0x7E; }

// Offsets inside a structurally valid record at rec (its block_size first)
struct BamFields {
    int lrn, flag;
    long long lseq, name, seq, qual;      // offsets from rec
};

CG_HD BamFields bam_fields(const uint8_t *rec)
{
    const uint8_t *r = rec + 4;
    BamFields f;
    f.lrn = r[8];
    f.flag = bam_u16(r + 14);
    f.lseq = bam_i32(r + 16);
    f.name = 4 + BAM_FIXED;
    f.seq = f.name + f.lrn + 4LL * bam_u16(r + 12);
    f.qual = f.seq + (f.lseq + 1) / 2;
    return f;
}

// The first refusal of a structurally valid record (0: none), tested serially (the device tests the same per lane)
CG_HD int bam_refusal(const uint8_t *rec)
{
    const BamFields f = bam_fields(rec);
    if (f.flag != 4) return BAM_R_FLAG;
    for (int i = 0; i + 1 < f.lrn; ++i)
        if (!bam_name_ok(rec[f.name + i])) return BAM_R_NAME;
    if (f.lseq > 0 && rec[f.qual] == 0xFF) return BAM_R_NOQUAL;
    for (long long i = 0; i < f.lseq; ++i)
        if (rec[f.qual + i] > 93) return BAM_R_QUAL;
    return 0;
}

// The FASTQ text of a record into out (bam_fastq_size bytes), serially
CG_HD void bam_emit(const uint8_t *rec, uint8_t *out)
{
    const BamFields f = bam_fields(rec);
    long long o = 0;
    out[o++] = '@';
    for (int i = 0; i + 1 < f.lrn; ++i) out[o++] = rec[f.name + i];
    out[o++] = '\n';
    for (long long i = 0; i < f.lseq; ++i) out[o++] = bam_base(rec[f.seq + (i >> 1)] >> ((i & 1) ? 0 : 4));
    out[o++] = '\n';
    out[o++] = '+';
    out[o++] = '\n';
    for (long long i = 0; i < f.lseq; ++i) out[o++] = (uint8_t)(rec[f.qual + i] + 33);
    out[o++] = '\n';
}

// ---- the tile walk ----------------------------------------------------------------------------------------------------
CG_HD uint64_t bam_link(long long pos, int on_walk, int st) { return ((uint64_t)pos << 3) | ((uint64_t)on_walk << 2) | (uint64_t)st; }
CG_HD long long bam_link_pos(uint64_t w) { return (long long)(w >> 3); }
CG_HD int bam_link_on(uint64_t w) { return (int)((w >> 2) & 1); }
CG_HD int bam_link_st(uint64_t w) { return (int)(w & 3); }

CG_HD bool bam_bit(const uint32_t *bm, long long p) { return (bm[p >> 5] >> (p & 31)) & 1u; }
CG_HD void bam_bit_set(uint32_t *bm, long long p) { bm[p >> 5] |= 1u << (p & 31); }

// The speculative walk of the tile [lo, hi) from `start` (its first bam_candidate offset, or 0 for tile 0;
// start >= hi: no walk): marks its offsets in bm, returns its exit as a link word (on_walk 0; the resolve fills it in).
CG_HD uint64_t bam_spec_walk(const uint8_t *b, long long n, long long hi, long long start, uint32_t *bm)
{
    if (start >= hi) return bam_link(0, 0, BAM_NONE);
    long long p = start;
    for (;;) {
        bam_bit_set(bm, p);
        long long nx = 0;
        const int st = bam_check(b, n, p, &nx);
        if (st != BAM_OK) return bam_link(p, 0, st);
        p = nx;
        if (p >= hi) return bam_link(p, 0, BAM_OK);
    }
}

// The link word of a tile's exit with on_walk filled in: whether the exit lands on the speculative walk of the tile it
// enters (its mark is set).  An exit at or behind n ends the chain, so it counts as on the walk.
CG_HD uint64_t bam_link_resolve(uint64_t w, long long n, const uint32_t *bm)
{
    if (bam_link_st(w) != BAM_OK) return w;
    const long long p = bam_link_pos(w);
    return bam_link(p, p >= n || bam_bit(bm, p), BAM_OK);
}

// Clear the marks of [lo, e) (lo a multiple of 32)
CG_HD void bam_clear(uint32_t *bm, long long lo, long long e)
{
    for (long long w = lo >> 5; (w << 5) < e; ++w) {
        const long long b0 = w << 5, k = e - b0;
        bm[w] &= k >= 32 ? 0u : ~((1u << k) - 1u);
    }
}

// The true entry p of tile [lo, hi) is not on its speculative walk: walk from p until an offset on the walk (the
// walk's exit `spec` then holds) or the tile's end.  The tile's marks in front of that point are replaced by the true
// chain's.  Returns the exit's link word, on_walk filled in.
CG_HD uint64_t bam_rewalk(const uint8_t *b, long long n, long long lo, long long hi, long long p, uint64_t spec,
                          uint32_t *bm)
{
    // first pass: where the true chain meets the walk (or leaves the tile, or stops)
    long long q = p, meet = hi;
    uint64_t out = 0;
    for (;;) {
        if (bam_link_st(spec) != BAM_NONE && bam_bit(bm, q)) { meet = q; out = spec; break; }
        long long nx = 0;
        const int st = bam_check(b, n, q, &nx);
        if (st != BAM_OK) { out = bam_link(q, 0, st); break; }
        q = nx;
        if (q >= hi) { out = bam_link_resolve(bam_link(q, 0, BAM_OK), n, bm); break; }
    }
    // second pass: the marks of [lo, meet) become the true chain's
    bam_clear(bm, lo, meet < hi ? meet : hi);
    for (q = p; q < meet && q < hi;) {
        bam_bit_set(bm, q);
        long long nx = 0;
        if (bam_check(b, n, q, &nx) != BAM_OK) break;
        q = nx;
    }
    return out;
}

// One step of the resolve: the chain enters tile t = p / tile at p (on: p is on the tile's walk); spec: the tile's link
// word.  Returns the link word of the chain's exit from the tile; *rewalked counts the walks again.
CG_HD uint64_t bam_resolve_step(const uint8_t *b, long long n, long long tile, long long p, int on, uint64_t spec,
                                uint32_t *bm, long long *rewalked)
{
    if (on) return spec;
    const long long lo = p / tile * tile, hi = lo + tile < n ? lo + tile : n;
    *rewalked += 1;
    return bam_rewalk(b, n, lo, hi, p, spec, bm);
}

// Marks of word w that are record starts: from its tile's entry (entry < 0: no record starts in the tile) up to end
CG_HD uint32_t bam_word_starts(const uint32_t *bm, long long w, long long tile, const long long *entry, long long end)
{
    const long long e = entry[(w << 5) / tile];
    if (e < 0) return 0;
    const long long b0 = w << 5;
    uint32_t m = bm[w];
    if (e > b0) m &= e - b0 >= 32 ? 0u : ~((1u << (e - b0)) - 1u);
    if (end < b0 + 32) m &= end <= b0 ? 0u : ((1u << (end - b0)) - 1u);
    return m;
}
