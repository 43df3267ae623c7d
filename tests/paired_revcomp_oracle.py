"""
--revcomp on pairs (PairedReverseComplementer, modifiers.py:311-400) on top of the FASTQ oracle (test infrastructure).

Each mate first goes through its own -u / --nextseq-trim / -q.  Then cutter1 (the -a list) and cutter2 (the -A list)
run on (r1, r2) and on (r2, r1); a pair whose swapped matches score strictly more is written swapped: R1's output gets
r2 trimmed by cutter1, R2's output r1 trimmed by cutter2, " rc" on both names unless revcomp == 2.  The pairs, in their
output positions, then run through oracle.oracle_fastq_trim_paired with the matches fixed (match_override) and with
no quality trimming left to do, so that a swapped record is never trimmed again with the other mate's cutoffs.  bp_in
and the quality-trimmed bases stay those of the input mate.
"""
import numpy as np

from oracle import oracle

_QUALITY_KEYS = ("cut", "quality_trim", "cutoff_front", "cutoff_back", "nextseq_cutoff")


def _score(m):
    return int(m["score"][m["adapter"] >= 0].sum()) if m is not None else 0


def pair_swapped(m11, m22, m12, m21):
    """The pair decision for every pair: (n,) bool.  Arguments: match arrays (n, times, slots) or None."""
    n = next(len(m) for m in (m11, m22, m12, m21) if m is not None)
    return np.array([_score(None if m12 is None else m12[i]) + _score(None if m21 is None else m21[i]) >
                     _score(None if m11 is None else m11[i]) + _score(None if m22 is None else m22[i])
                     for i in range(n)], dtype=bool)


def _prepared(data, options):
    """(records after the mate's own -u / --nextseq-trim / -q, bp_in, quality-trimmed bases)"""
    parsed = oracle.parse_fastq(data)
    records = oracle._apply_cuts(parsed, options.get("cut", ()))
    records, removed = oracle._quality_trimmed(records, options.get("quality_trim", False), options.get("cutoff_front", 0),
                                               options.get("cutoff_back", 0), options.get("quality_base", 33),
                                               options.get("nextseq_cutoff"))
    return records, sum(len(r[1]) for r in parsed), removed


def _matches(adapters, groups, records, times):
    if not adapters:
        return None
    return oracle.oracle_process(adapters, groups, [r[1] for r in records], None, False, 0, 0, 33, times, None)[0]


def _first_adapters(m):
    """The adapter each round of a read counts for in reverse_complemented: its first record (a linked match once)."""
    out = []
    for r in range(m.shape[0]):
        present = [int(x["adapter"]) for x in m[r] if x["adapter"] >= 0]
        if present:
            out.append(present[0])
    return out


def swapped_pairs(data1: bytes, data2: bytes, adapters1=None, groups1=None, adapters2=None, groups2=None, options1=None,
                  options2=None, revcomp=1, n_adapters=(0, 0)):
    """The pairs of a chunk in their output positions: (data1, data2, options1, options2, extra) to run through any of the
    paired oracles (oracle_fastq_trim_paired, the filter-output oracle, ...), then fix_counters(c1, c2, extra).  The
    options have the matches fixed and no -u / quality trimming left.  extra = {"swapped": (n,) bool, "adapter_rc":
    ([per adapter of R1's set], [of R2's]), ...} with n_adapters adapters per set."""
    options1, options2 = dict(options1 or {}), dict(options2 or {})
    if not adapters1 and not adapters2:                  # --revcomp without adapters does nothing (cli.py:1103-1110)
        n = len(oracle.parse_fastq(data1))
        return data1, data2, options1, options2, {"swapped": np.zeros(n, dtype=bool),
                                                  "adapter_rc": ([0] * n_adapters[0], [0] * n_adapters[1])}
    rec1, bp1, q1 = _prepared(data1, options1)
    rec2, bp2, q2 = _prepared(data2, options2)
    if len(rec1) != len(rec2):
        raise oracle.FastqFormatError("paired FASTQ chunks differ in their number of records")
    t1, t2 = options1.get("times", 1), options2.get("times", 1)
    m11, m12 = _matches(adapters1, groups1, rec1, t1), _matches(adapters1, groups1, rec2, t1)
    m22, m21 = _matches(adapters2, groups2, rec2, t2), _matches(adapters2, groups2, rec1, t2)
    swapped = pair_swapped(m11, m22, m12, m21)
    suffix = " rc" if revcomp == 1 else ""
    datas, overrides = [], []
    for own, other, m_own, m_cross in ((rec1, rec2, m11, m12), (rec2, rec1, m22, m21)):
        out = []
        for i, sw in enumerate(swapped):
            name, seq, qual = other[i] if sw else own[i]
            out.append(oracle._fastq_record(name + (suffix if sw else ""), seq, qual))
        datas.append(b"".join(out))
        if m_own is None:
            overrides.append(None)
        else:
            m = m_own.copy()
            m[swapped] = m_cross[swapped]
            overrides.append(m)
    opts = []
    for o, override in zip((options1, options2), overrides):
        o = {k: v for k, v in o.items() if k not in _QUALITY_KEYS}
        if override is not None:
            o["match_override"] = override
        opts.append(o)
    adapter_rc = ([0] * n_adapters[0], [0] * n_adapters[1])
    for k, m in enumerate(overrides):
        if m is None:
            continue
        for i in np.flatnonzero(swapped):
            for a in _first_adapters(m[i]):
                if a < n_adapters[k]:
                    adapter_rc[k][a] += 1
    return datas[0], datas[1], opts[0], opts[1], {"swapped": swapped, "adapter_rc": adapter_rc, "bp_in": (bp1, bp2),
                                                  "quality_trimmed_bp": (q1, q2)}


def fix_counters(c1, c2, extra):
    """bp_in and the quality-trimmed bases of the input mates, reverse_complemented = swapped pairs."""
    for k, c in enumerate((c1, c2)):
        if "bp_in" in extra:
            c.update(bp_in=extra["bp_in"][k], quality_trimmed_bp=extra["quality_trimmed_bp"][k])
        c["reverse_complemented"] = int(extra["swapped"].sum())


def paired_revcomp_trim(data1: bytes, data2: bytes, adapters1=None, groups1=None, adapters2=None, groups2=None,
                        options1=None, options2=None, pair_filter="any", revcomp=1, route=None, n_adapters=(0, 0)):
    """(out1, out2, counters1, counters2, extra) of one paired chunk with --revcomp (revcomp 1: " rc" suffixes, 2: none)
    through oracle_fastq_trim_paired (route: demultiplexing, as there).  "rest_rows" / "wildcard_rows" lists in the
    options receive the rows of each output position."""
    d1, d2, o1, o2, extra = swapped_pairs(data1, data2, adapters1, groups1, adapters2, groups2, options1, options2,
                                          revcomp, n_adapters)
    out1, out2, c1, c2 = oracle.oracle_fastq_trim_paired(d1, d2, adapters1, groups1, adapters2, groups2, o1, o2,
                                                         pair_filter, route=route)
    fix_counters(c1, c2, extra)
    return out1, out2, c1, c2, extra
