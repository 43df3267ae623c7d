// tests/hostsim/hostsim_gunzip.cpp -- TEST-ONLY host build of the gzip input path's decisions
// (cutadapt_b200/csrc/cg_gunzip_core.cuh), linked into libhostsim.so so that tests/test_gunzip_host.py can check them
// against Python's gzip module and the chunk readers of pipeline.py without a GPU.  The steps run in the order of
// cg_fastq_submit_gzip (cg_api.cu): every 1f 8b 08 parsed, the chain, the members inflated behind each other, the CRC-32
// of each.  Nothing in cutadapt_b200/ loads this library.
#include <string.h>

#include <vector>

#include "../../cutadapt_b200/csrc/cg_gunzip_core.cuh"
#include "../../cutadapt_b200/csrc/cg_gzip_core.cuh"

// gz[0, n) -> out (room for every plain byte).  Returns GU_OK / GU_INVALID / GU_UNSUPPORTED; *consumed, *plain (bytes
// written) and *err_at as in GuChain.  limit: the plain-size limit of the chain.
extern "C" int hs_gunzip(const uint8_t *gz, int64_t n, int final, int after_member, int64_t limit, uint8_t *out,
                         int64_t *consumed, int64_t *plain, int64_t *err_at)
{
    std::vector<int32_t> cand;
    for (int64_t p = 0; p + 3 <= n; ++p)
        if (gz[p] == 0x1f && gz[p + 1] == 0x8b && gz[p + 2] == 8) cand.push_back((int32_t)p);
    GuTables T;
    std::vector<GuMember> res(cand.size());
    for (size_t k = 0; k < cand.size(); ++k) res[k] = gu_member(gz + cand[k], n - cand[k], nullptr, T);
    std::vector<int32_t> members(cand.size() + 1);
    std::vector<long long> moff(cand.size() + 1);
    const GuChain c = gu_chain(gz, n, cand.data(), res.data(), (int)cand.size(), after_member != 0, final != 0, 0, limit,
                               members.data(), moff.data());
    *consumed = c.consumed;
    *plain = c.plain;
    *err_at = c.err_at;
    if (c.status != GU_OK) return c.status;
    uint32_t tab[256];
    for (int i = 0; i < 256; ++i) tab[i] = gz_crc_entry((uint32_t)i);
    for (int k = 0; k < c.n_members; ++k) {
        const int32_t at = cand[members[k]];
        uint8_t *o = out + moff[k];
        gu_member(gz + at, n - at, o, T);
        if (~gz_crc_raw(0xffffffffu, o, (int)res[members[k]].plain, tab) != res[members[k]].crc) {
            *err_at = at;
            return GU_INVALID;
        }
    }
    return GU_OK;
}

// flagged newlines of buf[0, n) (gu_flag): their positions into pos (room for n), their number, whether buf starts
// with '>'
static long long flags(const uint8_t *buf, int64_t n, int fasta, std::vector<long long> &pos, int *b0)
{
    pos.clear();
    for (int64_t i = 0; i < n; ++i)
        if (gu_flag(buf, n, i, fasta)) pos.push_back(i);
    *b0 = n > 0 && buf[0] == '>';
    return (long long)pos.size();
}

// whole records of buf (gu_records)
extern "C" int64_t hs_gu_records(const uint8_t *buf, int64_t n, int fasta)
{
    std::vector<long long> pos;
    int b0;
    const long long F = flags(buf, n, fasta, pos, &b0);
    return gu_records(fasta, F, b0);
}

// where buf is cut: rule 0 = one file, 1 = whole pairs of an interleaved buffer, 2 = in front of record r (two files)
extern "C" int64_t hs_gu_cut(const uint8_t *buf, int64_t n, int fasta, int rule, int64_t r)
{
    std::vector<long long> pos;
    int b0;
    const long long F = flags(buf, n, fasta, pos, &b0);
    const long long s = rule == 2 ? (r > 0 ? gu_select_records(fasta, r, b0) : -1) : gu_select_single(fasta, F, b0, rule);
    return s < 0 ? 0 : pos[(size_t)s] + 1;
}
