// tests/hostsim/hostsim_fasta.cpp -- TEST-ONLY host build of the FASTA line / record logic of the FASTQ path
// (fa_line_core, fa_line_error, fa_record_core in cutadapt_b200/csrc/cg_fastq_core.cuh), linked into libhostsim.so
// next to hostsim.cpp so that tests/test_fasta_host.py can fuzz it against the oracle's FASTA reader without a GPU.
// Nothing in cutadapt_b200/ loads this library; it is not a fallback.
#include <string.h>

#include <vector>

#include "../../cutadapt_b200/csrc/cg_core.cuh"
#include "../../cutadapt_b200/csrc/cg_fastq_core.cuh"

// FASTA chunk -> normalised buffer + record table, the steps of fa_classify / fa_scatter / fa_records_kernel one
// after the other (fa_line_core, fa_line_error, fa_record_core).  norm: n + 1 bytes; rec4 / seq_len: one entry per
// header line.  Returns 0 or the CG_FA_ERR_* code of the first bad line (its 0-based number in *bad_line).
extern "C" int hs_fasta_records(const uint8_t *buf, int64_t n, int cut_front, int cut_back, uint8_t *norm, int64_t *n_norm,
                                uint32_t *rec4, int32_t *seq_len, int64_t *n_records, int64_t *bad_line)
{
    std::vector<uint32_t> nl;
    for (int64_t i = 0; i < n; ++i)
        if (buf[i] == '\n') nl.push_back((uint32_t)i);
    const long long n_nl = (long long)nl.size();
    const long long n_lines = n_nl + ((n > 0 && buf[n - 1] != '\n') ? 1 : 0);
    std::vector<int> keep((size_t)n_lines), kind((size_t)n_lines);
    long long first = 0x7FFFFFFF;
    for (long long k = 0; k < n_lines; ++k) {
        uint32_t s, e;
        kind[k] = fa_line_core(buf, nl.data(), n_nl, n, k, &s, &e, &keep[k]);
        if (kind[k] == CG_FA_LINE_HEADER && k < first) first = k;
    }
    int64_t o = 0, r = 0;
    int bad = 0;
    *bad_line = -1;
    std::vector<CgFastqRecord> rec;
    for (long long k = 0; k < n_lines; ++k) {
        uint32_t s, e;
        int kp;
        fa_line_core(buf, nl.data(), n_nl, n, k, &s, &e, &kp);
        const int err = fa_line_error(kind[k], k, first);
        if (err && !bad) { bad = err; *bad_line = k; }
        if (kind[k] == CG_FA_LINE_COMMENT) continue;
        memcpy(norm + o, buf + s, e - s);
        if (kind[k] == CG_FA_LINE_HEADER) {
            norm[o + (e - s)] = '\n';
            CgFastqRecord x;
            x.hdr_start = (uint32_t)o + 1u;
            x.hdr_len = (int32_t)(e - s) - 1;
            rec.push_back(x);
            ++r;
        }
        o += keep[k];
    }
    *n_norm = o;
    *n_records = r;
    for (int64_t i = 0; i < r; ++i) {
        const uint32_t seq_end = i + 1 < r ? rec[i + 1].hdr_start - 1u : (uint32_t)o;
        CgFastqRecord x;
        int len, full, cf;
        fa_record_core(rec[i].hdr_start, rec[i].hdr_len, seq_end, cut_front, cut_back, &x, &len, &full, &cf);
        rec4[4 * i] = x.hdr_start; rec4[4 * i + 1] = (uint32_t)x.hdr_len;
        rec4[4 * i + 2] = x.seq_start; rec4[4 * i + 3] = x.qual_start;
        seq_len[i] = len;
    }
    return bad;
}
