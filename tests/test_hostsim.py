"""
The per-read device functions (cutadapt_b200/csrc/cg_core.cuh) compiled for the host and checked
against the oracle and the golden vectors.  This exercises exactly the code the kernels run per
lane -- packed-cell DP, wide-cell DP, prefilter, comparers, quality trimming, linked / multiple
composition, rounds -- without a GPU.  The host build lives under tests/ and is never loaded by
the product.
"""
import os
import random

import numpy as np
import pytest

from cutadapt_b200 import _lib as L
from oracle import oracle
from util import golden, hostsim_process, build_adapters, match_desc, spec_of, random_reads


def _single(ref, rate, flags, wr, wq, ic, mo, kind=0):
    return L.AdapterSetSpec([dict(sequence=ref, max_error_rate=rate, flags=flags, wildcard_ref=wr,
                                  wildcard_query=wq, indel_cost=ic, min_overlap=mo, kind=kind)])


@pytest.mark.parametrize("force_wide", [0, 1, 2, 10, 18, 34, 64, 256])   # packed, wide, two-phase: smem column / registers+refine / registers+inline runs / split main+end passes / planned runs + exact shortcut
def test_locate_golden(force_wide):
    cases = golden("locate_kat.json.gz")
    for ref, q, rate, flags, wr, wq, ic, mo, expected in cases:
        rec, _ = hostsim_process(_single(ref, rate, flags, wr, wq, ic, mo), [q], force_wide=force_wide)
        r = rec[0, 0, 0]
        got = None if r["adapter"] < 0 else [int(r[f]) for f in ("astart", "astop", "rstart", "rstop", "score", "errors")]
        assert got == expected, (ref, q, rate, flags, wr, wq, ic, mo)


def test_dp_matrix_dump_golden():
    """Aligner.enable_debug(): the cells locate_core records print like the reference's DPMatrix (cost and score)."""
    import ctypes as C
    from cutadapt_b200._align import DPMatrix
    from util import hostsim_lib

    lib = hostsim_lib()
    for ref, q, rate, flags, wr, mo, expected, dp_text, score_text in golden("dp_debug_kat.json.gz"):
        spec = _single(ref, rate, flags, wr, False, 1, mo)
        arr, _, _, _ = spec.to_ctypes()
        m, n = len(ref), len(q)
        cost = np.empty((m + 1, n + 1), dtype=np.int32)
        score = np.empty((m + 1, n + 1), dtype=np.int32)
        res = np.zeros(8, dtype=np.int32)
        rc = lib.hs_locate_debug(arr, q.encode(), C.c_int(n), C.c_void_p(cost.ctypes.data), C.c_void_p(score.ctypes.data),
                                 C.c_void_p(res.ctypes.data))
        assert rc == 0
        assert (list(map(int, res[1:7])) if res[0] else None) == expected
        assert str(DPMatrix(ref, q, cost)) == dp_text, (ref, q, flags)
        assert str(DPMatrix(ref, q, score)) == score_text, (ref, q, flags)


def test_comparers_golden():
    for ref, q, rate, wr, wq, mo, p, s in golden("comparer_kat.json.gz"):
        for kind, expected in ((1, p), (2, s)):
            rec, _ = hostsim_process(_single(ref, rate, 0, wr, wq, 1, mo, kind), [q])
            r = rec[0, 0, 0]
            got = None if r["adapter"] < 0 else [int(r[f]) for f in ("astart", "astop", "rstart", "rstop", "score", "errors")]
            assert got == expected, (kind, ref, q)


def test_adapters_golden():
    import cutadapt_b200.adapters as PA

    for case in golden("adapters_kat.json.gz"):
        multi = build_adapters(PA, case["adapters"])
        spec = spec_of(multi)
        reads = [r for r, _ in case["reads"]]
        recs, _ = hostsim_process(spec, reads)
        for i, (read, expected) in enumerate(case["reads"]):
            assert match_desc(multi.matches_from_records(recs[i, 0], read)) == expected, (case["adapters"], read)


def test_indexed_adapters_golden():
    """IndexedPrefixAdapters / IndexedSuffixAdapters (adapters.py:1289-1571): index build + lookups."""
    import cutadapt_b200.adapters as PA

    hits = 0
    for case in golden("index_kat.json.gz"):
        multi = build_adapters(PA, case["adapters"])
        indexed = [a for a in multi if isinstance(a, PA._IndexedAdapters)][0]
        assert len(indexed._index._index) == case["n_keys"]
        assert list(indexed._index._lengths) == case["lengths"]
        assert indexed._index._ambiguous == case["ambiguous"]
        spec = spec_of(multi)
        reads = [r for r, _ in case["reads"]]
        recs, _ = hostsim_process(spec, reads)
        for i, (read, expected) in enumerate(case["reads"]):
            assert match_desc(multi.matches_from_records(recs[i, 0], read)) == expected, (case["adapters"], read)
            hits += expected is not None
    assert hits > 1000


def test_rounds_and_quality_trim_against_oracle():
    import cutadapt_b200.adapters as PA

    rng = random.Random(5)
    for _ in range(60):
        ads = ["".join(rng.choice("ACGT") for _ in range(rng.randint(5, 20))) for _ in range(rng.randint(1, 3))]
        objs = [rng.choice([PA.BackAdapter, PA.FrontAdapter, PA.AnywhereAdapter])(a, max_errors=0.15, name="a") for a in ads]
        multi = PA.MultipleAdapters(objs)
        spec = spec_of(multi)
        reads = random_reads(rng, ads, 40)
        quals = ["".join(chr(33 + rng.choice([2, 2, 15, 30, 38])) for _ in r) for r in reads]
        times = rng.choice([1, 2, 3])
        params = L.make_params(quality_trim=True, cutoff_front=rng.choice([0, 10]), cutoff_back=20, times=times)
        got, qt = hostsim_process(spec, reads, quals, params)
        exp, eqt = oracle.oracle_process(spec.adapters, spec.groups, reads, quals, True, params.cutoff_front, 20, 33, times)
        assert (qt == eqt).all()
        assert (got == exp).all()


def test_empty_and_ragged_reads():
    import cutadapt_b200.adapters as PA

    multi = PA.MultipleAdapters([PA.BackAdapter("AGATCGGAAGAGC", name="a")])
    spec = spec_of(multi)
    reads = ["", "A", "AGA", "AGATCGGAAGAGC", "T" * 300 + "AGATCGGAAGAGC", "", "ACGT" * 50]
    got, _ = hostsim_process(spec, reads)
    exp, _ = oracle.oracle_process(spec.adapters, spec.groups, reads)
    assert (got == exp).all()
    assert got["adapter"][3, 0, 0] == 0 and got["rstart"][3, 0, 0] == 0


def test_two_phase_path_equals_general_path():
    """
    The scan + windowed-DP schedule of the two-phase kernel (process_read_simple: fused 32-bit scan
    words, locator hits, restarted DP windows) must reproduce the one-phase path bit for bit --
    every adapter type, wildcards, short and long reads (both group sizes), several adapter copies
    per read, partial occurrences at both ends, with and without quality trimming.
    """
    import cutadapt_b200.adapters as PA

    rng = random.Random(2024)
    types = ["FrontAdapter", "RightmostFrontAdapter", "BackAdapter", "RightmostBackAdapter", "AnywhereAdapter",
             "NonInternalFrontAdapter", "NonInternalBackAdapter", "PrefixAdapter", "SuffixAdapter", "BackAdapter"]
    n_windowed = 0
    for trial in range(250):
        alpha = rng.choice(["ACGT", "ACGT", "ACGTN", "AC", "ACGTacgtn"])
        m = rng.choice([rng.randint(3, 12), rng.randint(10, 34), 13, rng.randint(30, 70)])
        seq = "".join(rng.choice(rng.choice(["ACGT", "ACGT", "ACGTN", "ACGTRYN"])) for _ in range(m))
        if set(seq) <= {"N"}:
            seq = "A" + seq
        kw = dict(max_errors=rng.choice([0, 0.05, 0.1, 0.1, 0.15, 0.2, 0.3]), min_overlap=rng.randint(1, 6),
                  read_wildcards=rng.random() < 0.15, adapter_wildcards=rng.random() < 0.7)
        ad = getattr(PA, rng.choice(types))(seq, name="x", **kw)
        spec = spec_of(ad)
        reads = random_reads(rng, [seq], 50, alpha, rng.choice([60, 150, 150, 300, 700]))
        quals = ["".join(chr(33 + rng.choice([2, 2, 20, 30, 38])) for _ in r) for r in reads]
        qt = rng.random() < 0.3
        params = L.make_params(quality_trim=qt, cutoff_front=5, cutoff_back=20)
        a, qa = hostsim_process(spec, reads, quals if qt else None, params, 0)
        for mode in (2, 10, 18, 34, 64, 256):
            b, qb = hostsim_process(spec, reads, quals if qt else None, params, mode)
            assert (a == b).all() and (qa == qb).all(), (mode, repr(ad))
        n_windowed += 1
    assert n_windowed == 250


def test_bitplane_first_stage_against_oracle():
    """
    plane_scan_core (the first stage of the split pipeline for plain A/C/G/T 3' adapters): reads it settles
    itself ("no match", exact occurrence) and reads it hands to the exact path must all come out as the
    oracle says -- adapters of 5..60 bases, error rates up to 0.3, reads of 0..400 characters with N, lower
    case and other letters, several copies, with and without quality trimming.
    """
    import cutadapt_b200.adapters as PA
    from util import hostsim_plane_classes

    rng = random.Random(4242)
    seen = np.zeros(7, dtype=np.int64)
    n_planes = 0
    for trial in range(160):
        m = rng.choice([rng.randint(5, 12), 13, rng.randint(14, 33), 33, rng.randint(34, 60)])
        seq = "".join(rng.choice("ACGT") for _ in range(m))
        if trial == 0:
            seq = "AGATCGGAAGAGC"
        kw = dict(max_errors=rng.choice([0, 0.05, 0.1, 0.1, 0.15, 0.2, 0.3]), min_overlap=rng.randint(1, 6))
        ad = PA.BackAdapter(seq, name="x", **kw)
        spec = spec_of(ad)
        alpha = rng.choice(["ACGT", "ACGT", "ACGTN", "ACGTNacgtn", "ACGTRYKMEUXacgt"])
        max_len = rng.choice([40, 150, 150, 158, 200, 256, 400])
        reads = random_reads(rng, [seq], 60, alpha, max_len)
        # reads made the way the benchmark makes them: insert + adapter + tail, cut to a fixed length
        for _ in range(40):
            L0 = rng.choice([100, 150, 160, 161, 250])
            ins = rng.randint(0, L0)
            r = ("".join(rng.choice(alpha) for _ in range(ins)) + seq + "".join(rng.choice("ACGT") for _ in range(L0)))[:L0]
            if rng.random() < 0.3:
                r = r.lower() if rng.random() < 0.5 else r[: ins // 2] + r[ins // 2:].lower()
            reads.append(r)
        quals = ["".join(chr(33 + rng.choice([2, 2, 20, 30, 38])) for _ in r) for r in reads]
        qt = rng.random() < 0.3
        params = L.make_params(quality_trim=qt, cutoff_front=5, cutoff_back=20)
        exp, eqt = oracle.oracle_process(spec.adapters, spec.groups, reads, quals if qt else None, qt, 5, 20, 33, 1)
        got, gqt = hostsim_process(spec, reads, quals if qt else None, params, 256)
        assert (gqt == eqt).all() and (got == exp).all(), repr(ad)
        cls = hostsim_plane_classes(spec, reads)
        if (cls >= 0).any():
            n_planes += 1
        seen += np.bincount(cls + 1, minlength=7)
    # the stage must actually decide reads: most adapters qualify, and all three classes occur
    # (classes: none, exact occurrence, re-scan, plan from the planes' hits; with the end analysis also: exact overlap
    # at the end, plan without end window -- test_bitplane_end_analysis_and_repetitive_adapters)
    assert n_planes > 80 and seen[1] > 1000 and seen[2] > 1000 and seen[3] > 50 and seen[4] > 300, (n_planes, seen)


def test_bitplane_end_analysis_and_repetitive_adapters(monkeypatch):
    """
    The end analysis of the bit-plane stage (guard pieces, exact overlaps at the end of the read, "no end window")
    and locator chunks that repeat inside the adapter: reads ending with adapter prefixes of every length with 0..2
    edits, adapter pieces elsewhere, repetitive adapters -- first-stage decisions + hand-off == the plain path.
    """
    import cutadapt_b200.adapters as PA
    from util import hostsim_plane_classes

    monkeypatch.setenv("CUTADAPT_B200_END_ANALYSIS", "1")       # (off by default: see cg_setbuild.cpp)
    rng = random.Random(2718)
    seen = np.zeros(7, dtype=np.int64)
    for trial in range(150):
        m = rng.choice([6, 8, 10, 13, 13, 16, 20, 25, 33, 40])
        seq = "".join(rng.choice("ACGT") for _ in range(m))
        if rng.random() < 0.25:
            seq = (seq[:rng.choice([1, 2, 3])] * 40)[:m]
        ad = PA.BackAdapter(seq, max_errors=rng.choice([0.05, 0.1, 0.1, 0.15, 0.2, 0.25]), min_overlap=rng.randint(1, 7), name="x")
        spec = spec_of(ad)
        reads = []
        for _ in range(120):
            n = rng.choice([60, 100, 150, 160])
            piece = list(seq[:rng.randint(0, m)])
            for _ in range(rng.choice([0, 0, 0, 1, 1, 2])):
                if piece:
                    p, r = rng.randrange(len(piece)), rng.random()
                    if r < 0.4:
                        piece[p] = rng.choice("ACGTN")
                    elif r < 0.7:
                        del piece[p]
                    else:
                        piece.insert(p, rng.choice("ACGT"))
            body = "".join(rng.choice("ACGT") for _ in range(n))
            if rng.random() < 0.3:
                q, j = rng.randrange(n), rng.randint(0, m - 1)
                body = body[:q] + seq[j:j + rng.randint(3, m)] + body[q:]
            read = (body + "".join(piece))[-n:]
            reads.append(read.lower() if rng.random() < 0.1 else read)
        a, _ = hostsim_process(spec, reads, force_wide=0)
        b, _ = hostsim_process(spec, reads, force_wide=256)
        assert (a == b).all(), repr(ad)
        seen += np.bincount(hostsim_plane_classes(spec, reads) + 1, minlength=7)
    assert seen[5] > 1000 and seen[6] > 200, seen


def test_two_phase_on_golden_single_adapters():
    import cutadapt_b200.adapters as PA

    n = 0
    for case in golden("adapters_kat.json.gz"):
        if len(case["adapters"]) != 1 or case["adapters"][0][0] == "Linked":
            continue
        multi = build_adapters(PA, case["adapters"])
        spec = spec_of(multi)
        reads = [r for r, _ in case["reads"]]
        for mode in (2, 10, 18, 34, 64, 256):
            recs, _ = hostsim_process(spec, reads, force_wide=mode)
            for i, (read, expected) in enumerate(case["reads"]):
                assert match_desc(multi.matches_from_records(recs[i, 0], read)) == expected, (mode, case["adapters"], read)
        n += 1
    assert n > 40


def _multipass(spec, reads, quals=None, params=None):
    """Mode 128 = the multi-pass schedule (per-component passes + select_best); None if not planned."""
    try:
        return hostsim_process(spec, reads, quals, params, force_wide=128)
    except RuntimeError as e:
        if e.args[0][0] == 100:
            return None
        raise


def test_multipass_schedule_golden():
    """Per-adapter passes + selection == MultipleAdapters / LinkedAdapter / AdapterIndex of the reference."""
    import cutadapt_b200.adapters as PA

    planned = 0
    for name in ("adapters_kat.json.gz", "index_kat.json.gz"):
        for case in golden(name):
            multi = build_adapters(PA, case["adapters"])
            spec = spec_of(multi)
            reads = [r for r, _ in case["reads"]]
            res = _multipass(spec, reads)
            if res is None:
                continue
            planned += 1
            for i, (read, expected) in enumerate(case["reads"]):
                assert match_desc(multi.matches_from_records(res[0][i, 0], read)) == expected, (case["adapters"], read)
    assert planned > 100


def test_multipass_schedule_with_quality_trim_against_oracle():
    import cutadapt_b200.adapters as PA

    rng = random.Random(77)
    planned = 0
    for _ in range(60):
        ads = ["".join(rng.choice("ACGT") for _ in range(rng.randint(5, 45))) for _ in range(rng.randint(2, 4))]
        objs = [rng.choice([PA.BackAdapter, PA.FrontAdapter, PA.AnywhereAdapter, PA.SuffixAdapter])(a, max_errors=0.15, name="a")
                for a in ads]
        if rng.random() < 0.5:
            objs.append(PA.LinkedAdapter(PA.PrefixAdapter(ads[0][:12], max_errors=0.2), PA.BackAdapter(ads[1], max_errors=0.1),
                                         rng.random() < 0.5, rng.random() < 0.5, "l"))
        multi = PA.MultipleAdapters(objs)
        spec = spec_of(multi)
        reads = random_reads(rng, ads, 40, max_len=120)
        quals = ["".join(chr(33 + rng.choice([2, 2, 15, 30, 38])) for _ in r) for r in reads]
        params = L.make_params(quality_trim=True, cutoff_front=rng.choice([0, 10]), cutoff_back=20)
        res = _multipass(spec, reads, quals, params)
        assert res is not None
        planned += 1
        exp, eqt = oracle.oracle_process(spec.adapters, spec.groups, reads, quals, True, params.cutoff_front, 20, 33, 1)
        assert (res[1] == eqt).all()
        assert (res[0] == exp).all()
    assert planned == 60


def test_trim_scan_device_functions_golden():
    """The device functions behind cg_nextseq_trim_batch / cg_poly_a_trim_batch, compiled for the host."""
    import ctypes as C
    from util import hostsim_lib

    lib = hostsim_lib()
    g = golden("trim_scans_kat.json.gz")
    for seq, qual, cutoff, base, expected in g["nextseq"]:
        assert lib.hs_nextseq_trim(seq.encode(), qual.encode(), len(qual), cutoff, base) == expected
    for seq, revcomp, expected in g["polya"]:
        assert lib.hs_poly_a_trim(seq.encode(), len(seq), int(revcomp)) == expected
    lib.hs_expected_errors.restype = C.c_double
    for qual, base, expected in g["expected_errors"]:
        assert float(lib.hs_expected_errors(qual.encode(), len(qual), base)).hex() == expected


def test_fused_nextseq_and_quality_trim_against_oracle():
    """NextseqQualityTrimmer -> QualityTrimmer -> AdapterCutter fused in one pass, all schedules."""
    import cutadapt_b200.adapters as PA

    rng = random.Random(91)
    for trial in range(40):
        ads = ["".join(rng.choice("ACGT") for _ in range(rng.randint(6, 30))) for _ in range(rng.randint(1, 3))]
        objs = [rng.choice([PA.BackAdapter, PA.FrontAdapter])(a, max_errors=0.1, name="a") for a in ads]
        multi = PA.MultipleAdapters(objs)
        spec = spec_of(multi)
        reads = [r + "G" * rng.choice([0, 0, 3, 10]) for r in random_reads(rng, ads, 40, max_len=100)]
        quals = ["".join(chr(33 + rng.choice([2, 2, 15, 30, 38])) for _ in r) for r in reads]
        qt = rng.random() < 0.6
        params = L.make_params(quality_trim=qt, cutoff_front=rng.choice([0, 10]), cutoff_back=20,
                               nextseq_cutoff=rng.choice([10, 20, 30]))
        exp, eqt = oracle.oracle_process(spec.adapters, spec.groups, reads, quals, qt, params.cutoff_front, 20, 33, 1,
                                         nextseq_cutoff=params.nextseq_cutoff)
        modes = [0, 128] if len(ads) > 1 else [0, 2, 10, 34, 64, 256]
        for mode in modes:
            try:
                got, gqt = hostsim_process(spec, reads, quals, params, force_wide=mode)
            except RuntimeError as e:
                if e.args[0][0] == 100:
                    continue
                raise
            assert (gqt == eqt).all(), mode
            assert (got == exp).all(), mode


def test_reference_fasta_goldens_through_the_device_functions():
    """
    The command-line known answers of the reference with anchored / non-internal / linked adapters, --no-indels, -N
    and --match-read-wildcards (tests/golden/fastq_kat.json.gz, "fasta_cases"): match records from the host build of
    the device functions + pipeline.kept_intervals must give the expected reads.
    """
    import numpy as np
    from oracle import oracle
    from util import golden, fastq_file, adapter_from_spec, hostsim_process, spec_of
    import cutadapt_b200.adapters as PA
    from cutadapt_b200.pipeline import kept_intervals

    done = 0
    for c in golden("fastq_kat.json.gz")["fasta_cases"]:
        o = c["options"]
        if not o["specs"] or any(k in o for k in ("trim_n", "poly_a", "max_n")):
            continue
        params = dict(max_errors=o.get("error_rate", 0.1), min_overlap=o.get("min_overlap", 3),
                      adapter_wildcards=not o.get("no_wildcards", False), read_wildcards=o.get("read_wildcards", False),
                      indels=not o.get("no_indels", False))
        ads = [adapter_from_spec(spec, kind, name=f"a{i}", **params) for i, (kind, spec) in enumerate(o["specs"])]
        spec = spec_of(PA.MultipleAdapters(ads))
        records = oracle.parse_fastq(fastq_file(f"fa_{c['name']}.in.fastq"))
        seqs = [r[1] for r in records]
        matches, _ = hostsim_process(spec, seqs)
        iv = kept_intervals(matches, None, np.array([len(x) for x in seqs]))
        got = []
        for (name, seq, q), (a, b) in zip(records, iv):
            a, b = int(a), int(b)
            if o.get("minimum_length") and b - a < o["minimum_length"]:
                continue
            if "maximum_length" in o and b - a > o["maximum_length"]:
                continue
            got.append(f"@{name}\n{seq[a:b]}\n+\n{q[a:b]}\n")
        assert "".join(got).encode() == fastq_file(f"fa_{c['name']}.out.fastq"), (c["name"], c["command"])
        done += 1
    assert done >= 22


# ---- FASTQ path: cg_fastq_core.cuh on the host --------------------------------------------------------------

def _fastq_table(data, cut=()):
    """Record table of a FASTQ chunk as fq_records_kernel builds it (positions in `data`, -u cuts applied)."""
    cut_front = sum(c for c in cut if c > 0)
    cut_back = sum(-c for c in cut if c < 0)
    rec, lens, pos = [], [], 0
    lines = data.split(b"\n")
    if lines[-1] == b"":
        lines.pop()
    starts = []
    for ln in lines:
        starts.append(pos)
        pos += len(ln) + 1
    for r in range(len(lines) // 4):
        h, s, q = lines[4 * r], lines[4 * r + 1], lines[4 * r + 3]
        strip = lambda x: x[:-1] if x.endswith(b"\r") else x
        h, s, q = strip(h), strip(s), strip(q)
        n = len(s)
        cf = min(cut_front, n)
        n -= cf
        n = n - cut_back if cut_back < n else 0
        rec.append((starts[4 * r] + 1, len(h) - 1, starts[4 * r + 1] + cf, starts[4 * r + 3] + cf))
        lens.append(n)
    return np.array(rec, dtype=np.uint32).reshape(-1, 4), np.array(lens, dtype=np.int32)


def _hostsim_fastq(data, ads, opts, second_mate=False):
    """(per-record names, evaluate outputs) of one mate through hostsim: trimming pass + fq_evaluate_core."""
    import ctypes as C
    from cutadapt_b200 import _lib as L
    from cutadapt_b200.pipeline import _fastq_params
    from util import hostsim_lib, hostsim_process, spec_of
    import cutadapt_b200.adapters as PA

    fp = _fastq_params(**opts)
    rec, lens = _fastq_table(data, opts.get("cut", ()))
    buf = np.frombuffer(data, dtype=np.uint8)
    seqs = [data[int(r[2]):int(r[2]) + int(n)].decode("latin-1") for r, n in zip(rec, lens)]
    quals = [data[int(r[3]):int(r[3]) + int(n)].decode("latin-1") for r, n in zip(rec, lens)]
    want_q = bool(fp.trim.quality_trim or fp.trim.nextseq_trim)
    matches = qtrim = None
    times, slots = max(1, fp.trim.times), 1
    if ads:
        spec = spec_of(PA.MultipleAdapters(ads))
        matches, qtrim = hostsim_process(spec, seqs, quals if want_q else None, fp.trim)
        slots = spec.slots
        if not want_q:
            qtrim = None
    elif want_q:
        from oracle import oracle
        qtrim = np.zeros((len(seqs), 2), dtype=np.int32)
        for i, (s_, q_) in enumerate(zip(seqs, quals)):
            e = oracle.nextseq_trim_index(s_, q_, fp.trim.nextseq_cutoff, fp.trim.quality_base) if fp.trim.nextseq_trim else len(s_)
            qtrim[i] = oracle.quality_trim_index(q_[:e], fp.trim.cutoff_front, fp.trim.cutoff_back, fp.trim.quality_base) \
                if fp.trim.quality_trim else (0, e)
    n = len(seqs)
    shorten = 0 if not fp.shorten else (fp.shorten_length + 1 if fp.shorten_length >= 0 else fp.shorten_length)
    ip = np.array([fp.minimum_length, fp.maximum_length, fp.discard_trimmed, fp.discard_untrimmed,
                   (2 if second_mate else 1) if fp.poly_a else 0, shorten, fp.trim_n, fp.discard_casava,
                   fp.action if ads else 0], dtype=np.int32)
    dp = np.array([fp.max_n, fp.max_expected_errors], dtype=np.float64)
    interval = np.zeros((n, 2), dtype=np.int32)
    keep = np.zeros((n, 2), dtype=np.int32)
    mask = np.zeros(n, dtype=np.int32)
    last = np.zeros(n, dtype=np.int32)
    lib = hostsim_lib()
    lib.hs_fastq_evaluate.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                      C.c_void_p] + [C.c_void_p] * 6
    bad = lib.hs_fastq_evaluate(buf.ctypes.data, n, rec.ctypes.data, lens.ctypes.data,
                                matches.ctypes.data if matches is not None else None, times, slots,
                                qtrim.ctypes.data if qtrim is not None else None, ip.ctypes.data, dp.ctypes.data,
                                interval.ctypes.data, keep.ctypes.data, mask.ctypes.data, last.ctypes.data)
    assert bad == 0
    enabled = (1 if fp.minimum_length > 0 else 0) | (2 if fp.maximum_length >= 0 else 0) | (4 if fp.max_n >= 0 else 0) | \
        (8 if fp.max_expected_errors >= 0 else 0) | (16 if fp.discard_casava else 0) | (32 if fp.discard_trimmed else 0) | \
        (64 if fp.discard_untrimmed else 0)
    return dict(data=data, rec=rec, interval=interval, keep=keep, mask=mask, enabled=enabled, action=int(ip[8]), last=last)


def _format_fastq(ev, fired):
    """fq_write_kernel in Python: the surviving records with the action's character transform."""
    out = []
    data = ev["data"]
    for r in range(len(ev["mask"])):
        if fired[r] >= 0:
            continue
        hs, hl, ss, qs = (int(x) for x in ev["rec"][r])
        a, b = (int(x) for x in ev["interval"][r])
        k0, k1 = (int(x) for x in ev["keep"][r])
        seq = bytearray(data[ss + a:ss + b])
        for j in range(a, b):
            inside = k0 <= j < k1
            c = seq[j - a]
            if ev["action"] == 2:
                seq[j - a] = c if inside else ord("N")
            elif ev["action"] == 3 and chr(c).isalpha():
                seq[j - a] = ord(chr(c).upper()) if inside else ord(chr(c).lower())
        out.append(b"@" + data[hs:hs + hl] + b"\n" + bytes(seq) + b"\n+\n" + data[qs + a:qs + b] + b"\n")
    return b"".join(out)


def _finish(ev1, ev2=None, mode=0, mode_untrimmed=0):
    import ctypes as C
    from util import hostsim_lib

    n = len(ev1["mask"])
    fired = np.zeros(n, dtype=np.int32)
    lib = hostsim_lib()
    lib.hs_fastq_finish.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.hs_fastq_finish(n, ev1["mask"].ctypes.data, ev2["mask"].ctypes.data if ev2 else None, ev1["enabled"],
                        ev2["enabled"] if ev2 else 0, mode, mode_untrimmed, fired.ctypes.data)
    return fired


def test_fastq_logic_of_the_device_functions_against_the_oracle():
    """fq_evaluate_core / fq_finish_core (the per-record logic of the FASTQ kernels, compiled for the host) + the
    host build of the trimming pass must write what oracle_fastq_trim(_paired) writes: every variant of
    tests/test_gpu_fastq.py's randomized test, the command-line goldens, and paired chunks in all three filter modes."""
    from oracle import oracle
    from test_gpu_fastq import synthetic_fastq, oracle_for, trimmer_kwargs
    from util import fastq_cases, fastq_case_adapters, fastq_paired_cases, oracle_paired

    variants = {
        "plain": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]], quality_cutoff=[5, 20]), {}),
        "filters": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]], quality_cutoff=[5, 20]),
                    dict(minimum_length=20, maximum_length=140, max_n=0.1, max_expected_errors=2.5, discard_untrimmed=True)),
        "quality_only": (dict(adapters=[], quality_cutoff=[0, 25], nextseq_cutoff=20), dict(minimum_length=1, max_n=3)),
        "modifiers": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]], quality_cutoff=[5, 20]),
                      dict(cut=[3, -2], poly_a=True, length=-90, trim_n=True, discard_casava=True, minimum_length=1)),
        "modifiers2": (dict(adapters=[["anywhere", "AGATCGGAAGAGC"]]),
                       dict(cut=[-4, -3, 2], poly_a=True, length=60, trim_n=True, max_n=0, discard_trimmed=True)),
        "mask": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]], quality_cutoff=[5, 20]),
                 dict(action="mask", times=2, trim_n=True, max_n=0.3, minimum_length=5)),
        "lowercase": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]]), dict(action="lowercase", times=2, poly_a=True)),
        "none": (dict(adapters=[["back", "AGATCGGAAGAGC"]]), dict(action="none", discard_untrimmed=True, length=100)),
        "retain": (dict(adapters=[["linked", "TTGACNNACG", "AGATCGGAAGAGC"], ["back", "CACGTCTGAACTC"], ["front", "ACGTACGTAC"]],
                        quality_cutoff=[0, 15]), dict(action="retain", minimum_length=1)),
        "crop": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"], ["anywhere", "CACGTCTGAA"]]),
                 dict(action="crop", discard_untrimmed=True, trim_n=True)),
    }
    for k, (name, (options, extra)) in enumerate(variants.items()):
        data = synthetic_fastq(1500, seed=40 + k, crlf=name == "filters")
        opts = dict(options)
        opts.update(extra)
        kw = trimmer_kwargs({x: y for x, y in opts.items() if x != "adapters"})
        ev = _hostsim_fastq(data, fastq_case_adapters(options), kw)
        got = _format_fastq(ev, _finish(ev))
        exp, _ = oracle_for(options, data, **extra)
        assert got == exp, name
    for c in fastq_cases():
        kw = trimmer_kwargs({x: y for x, y in c["options"].items() if x not in ("adapters", "error_rate", "min_overlap")})
        ev = _hostsim_fastq(c["input_bytes"], fastq_case_adapters(c["options"]), kw)
        assert _format_fastq(ev, _finish(ev)) == c["expected_bytes"], c["name"]
    for c in fastq_paired_cases():
        o = c["options"]
        evs = []
        for k, key in enumerate(("adapters1", "adapters2")):
            kw = trimmer_kwargs(o[f"options{k + 1}"])
            evs.append(_hostsim_fastq(c["input_bytes"][k], fastq_case_adapters(o, key), kw, second_mate=k == 1))
        mode = {"any": 0, "both": 1, "first": 2}[o.get("pair_filter", "any")]
        mode_untrimmed = 1 if (not o["adapters1"] or not o["adapters2"]) else mode
        fired = _finish(evs[0], evs[1], mode, mode_untrimmed)
        assert [_format_fastq(evs[0], fired), _format_fastq(evs[1], fired)] == c["expected_bytes"], c["name"]


def test_fastq_record_table_of_the_device_functions():
    """fq_record_core (record table + dnaio's format checks + -u cuts) on the host: against the Python table of this
    file for LF / CRLF / missing final newline, and the error codes for malformed records."""
    import ctypes as C
    from test_gpu_fastq import synthetic_fastq
    from util import hostsim_lib

    lib = hostsim_lib()
    lib.hs_fastq_records.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]

    def table(data, cut=(), n_records=None):
        buf = np.frombuffer(data, dtype=np.uint8)
        lines = data.count(b"\n") + (0 if data.endswith(b"\n") or not data else 1)
        n = lines // 4 if n_records is None else n_records
        rec = np.zeros((n, 4), dtype=np.uint32)
        lens = np.zeros(n, dtype=np.int32)
        bad = C.c_int64(-1)
        code = lib.hs_fastq_records(buf.ctypes.data, len(data), sum(c for c in cut if c > 0), sum(-c for c in cut if c < 0),
                                    n, rec.ctypes.data, lens.ctypes.data, C.byref(bad))
        return code, bad.value, rec, lens

    for k, (crlf, cut) in enumerate(((False, ()), (True, ()), (False, (3, -2)), (True, (-1, 200)))):
        data = synthetic_fastq(800, seed=60 + k, crlf=crlf)
        for tail in (data, data + b"@last\nACGT\n+\nIIII"):
            code, bad, rec, lens = table(tail, cut)
            want_rec, want_lens = _fastq_table(tail, cut)
            assert code == 0 and bad == -1
            assert (rec == want_rec).all() and (lens == want_lens).all()
    for text, want in ((b"r\nACGT\n+\nIIII\n", 1), (b"@r\nACGT\n-\nIIII\n", 2), (b"@r\nACGT\n+\nIII\n", 3),
                       (b"@a\nAC\n+\nII\n@b\nACGT\n\nIIII\n", 2), (b"@r 1\nACGT\n+r 2\nIIII\n", 5),
                       (b"@r 1\nACGT\n+r\nIIII\n", 5), (b"@a\nAC\n+a\nII\n@b x\nACGT\n+b y\nIIII\n", 5)):
        code, bad, _, _ = table(text)
        assert code == want and bad == text.count(b"@a")


def test_first_stage_specialisation_compiles_without_a_device():
    """cg_jit.cpp: the translation unit generated for an adapter set (straight-line plane_chain_step / plane_emit calls)
    goes through NVRTC for sm_90a here, for 5- and 8-word planes, with and without qualities; a set without a plane
    program (wildcards) yields no source."""
    import cutadapt_b200.adapters as PA
    from util import hostsim_jit_compile, spec_of

    for seq, words, qual in (("AGATCGGAAGAGC", 5, False), ("AGATCGGAAGAGCACACGTCTGAACTCCAGTCA", 8, True),
                             ("CTGTCTCTTATACACATCT", 5, True)):
        spec = spec_of(PA.MultipleAdapters([PA.BackAdapter(seq, max_errors=0.1, name="a")]))
        n, src, log = hostsim_jit_compile(spec, words, qual)
        if n == -2:
            pytest.skip("libnvrtc is not installed")
        assert n > 10000, log
        assert src.count("plane_chain_step") >= len(seq) and f"cg_pscan_body<{str(qual).lower()}, {words}, StaticPlaneProg>" in src
    spec = spec_of(PA.MultipleAdapters([PA.BackAdapter("AGATCNNNNGAGC", max_errors=0.1, name="a")]))
    n, src, _ = hostsim_jit_compile(spec)
    assert n == 0 and src == ""


def test_banded_dp_runs_on_crowded_reads():
    """run_band_d (cg_core.cuh): the DP runs of the bit-plane path skip the rows no alignment through the run's hits
    can touch.  Reads crowded with mutated adapter copies a few bases apart, overlapping copies, partial copies and
    repetitive adapters (tools/fuzz_band.py makes them) must still come out as the oracle says; a band cut two rows
    too deep is caught by this generator within a few hundred reads (checked when the band was introduced)."""
    import importlib.util
    import os
    import cutadapt_b200.adapters as PA

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec_ = importlib.util.spec_from_file_location("fuzz_band", os.path.join(root, "tools", "fuzz_band.py"))
    fb = importlib.util.module_from_spec(spec_)
    spec_.loader.exec_module(fb)
    total = 0
    for trial in range(40):
        rng = random.Random(777 + trial)
        m = rng.choice([rng.randint(6, 12), 13, 13, rng.randint(14, 33), 33, rng.randint(34, 60)])
        seq = "".join(rng.choice("ACGT") for _ in range(m))
        if trial % 4 == 0:
            unit = "".join(rng.choice("ACGT") for _ in range(rng.randint(1, 4)))
            seq = (unit * m)[:m]
        cls = rng.choice([PA.BackAdapter, PA.BackAdapter, PA.FrontAdapter, PA.AnywhereAdapter])
        ad = cls(seq, name="x", max_errors=rng.choice([0.1, 0.1, 0.15, 0.2, 0.3]), min_overlap=rng.randint(1, 6))
        spec = spec_of(ad)
        reads = [fb.make_read(rng, seq, rng.choice([60, 150, 150, 200, 256])) for _ in range(250)]
        exp, _ = oracle.oracle_process(spec.adapters, spec.groups, reads, None, False, 0, 0, 33, 1)
        got, _ = hostsim_process(spec, reads, None, L.make_params(quality_trim=False), 256)
        assert (got == exp).all(), repr(ad)
        total += int((exp["adapter"] >= 0).sum())
    assert total > 5000


def test_index_lookups_on_random_barcode_sets():
    """match_indexed (the affix is packed once, keys of shorter lengths are a mask / shift away): random barcode sets of
    equal and mixed lengths, 5' and 3', with and without indels, mutated barcodes with N, lower case and other letters,
    reads shorter than the keys -- the host build against the oracle's own index (tools/fuzz_index.py runs the same
    with more trials)."""
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "tools", "fuzz_index.py"), "5", "25"], capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0 and "ok, hits" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
    assert int(out.stdout.strip().split()[-1]) > 2000
