#!/usr/bin/env python3
"""
Generate tests/golden/reference_kat.json.gz: what the REFERENCE answers on the inputs of the tests that compare
with it (test_gpu_gate.py, test_gpu_parity.py, test_oracle.py, test_distributed_cpu.py, test_reference_suite.py).

Needs a checkout of the reference and Cython: the reference's hot path is compiled afresh into oracle/_ref
(oracle/build_ref.py), and the file records the SHA-256 of every source it was compiled from ("provenance").

    python tests/golden/make_reference_golden.py --reference DIR      (or $CUTADAPT_REFERENCE)

Large answer lists are stored as SHA-256 digests of chunks of 1000 answers (tests/util.py answer_digests); the
tests compute the same digests from the device's or the oracle's answers.  Before writing, every answer list is
checked against the C oracle on the same inputs, so a generator that drifted from its test fails here.  The inputs
come from seeded CPU generators; re-running reproduces the file byte for byte.
"""
import argparse
import gzip
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)

import numpy as np  # noqa: E402

from util import answer_digests, canonical, end_statistics_answer, index_test_reads, match_desc, random_locate_cases  # noqa: E402

N_GATE, N_REF = 1_000_000, 100_000      # test_gpu_gate.py
F6 = ("astart", "astop", "rstart", "rstop", "score", "errors")


def m6(m):
    return None if m is None else [m.astart, m.astop, m.rstart, m.rstop, m.score, m.errors]


def rec6(rec):
    return None if rec["adapter"] < 0 else [int(rec[f]) for f in F6]


def packed(t):
    host = np.ascontiguousarray(t.numpy()).reshape(-1)
    return host, np.arange(t.shape[0] + 1, dtype=np.int64) * t.shape[1]


def digests(name, ref_answers, oracle_answers, out):
    ref_answers = canonical(ref_answers)
    assert ref_answers == canonical(oracle_answers), f"{name}: the oracle differs from the reference"
    out[name] = answer_digests(ref_answers)
    print(f"{name}: {len(ref_answers)} answers")


def gate(out):
    import cutadapt.adapters as RA
    from cutadapt.qualtrim import quality_trim_index
    from cutadapt_b200.configs import (CONFIG3_BACK, CONFIG3_LINKED, CONFIG4_R1, CONFIG4_R2, config5_barcodes,
                                       config_adapters, make_config_batch, to_strings)
    from oracle import oracle

    def flat(multi):
        singles, groups, owners = multi._flatten()
        multi._device_set = (None, singles, owners)
        return [s.descriptor() for s in singles], groups

    # config 2
    multi, _ = config_adapters(2)
    descs, groups = flat(multi)
    seq = make_config_batch(2, N_GATE, device="cpu")["seq"][:N_REF]
    exp, _ = oracle.oracle_process_packed(descs, groups, *packed(seq))
    ra = RA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1, min_overlap=3, name="adapter")
    digests("gate_config2", [m6(ra.match_to(r)) for r in to_strings(seq)], [rec6(r) for r in exp[:, 0, 0]], out)
    # config 3
    multi, _ = config_adapters(3)
    descs, groups = flat(multi)
    seq = make_config_batch(3, N_GATE, device="cpu")["seq"][:N_REF]
    exp, _ = oracle.oracle_process_packed(descs, groups, *packed(seq))
    objs = [RA.BackAdapter(s, max_errors=0.15, min_overlap=3, name=f"a{i}") for i, s in enumerate(CONFIG3_BACK)]
    objs.append(RA.LinkedAdapter(RA.PrefixAdapter(CONFIG3_LINKED[0], max_errors=0.15, min_overlap=3, name="lf"),
                                 RA.BackAdapter(CONFIG3_LINKED[1], max_errors=0.15, min_overlap=3, name="lb"),
                                 True, False, "linked"))
    rmulti = RA.MultipleAdapters(objs)
    reads = to_strings(seq)
    digests("gate_config3", [match_desc(rmulti.match_to(r)) for r in reads],
            [match_desc(multi.matches_from_records(exp[i, 0], r)) for i, r in enumerate(reads)], out)
    # config 4: both mates, quality trimming in front
    m1, m2 = config_adapters(4)
    b = make_config_batch(4, N_GATE // 2, device="cpu")
    for multi, skey, qkey, adapter in ((m1, "seq", "qual", CONFIG4_R1), (m2, "seq2", "qual2", CONFIG4_R2)):
        descs, groups = flat(multi)
        seq, qual = b[skey][:N_REF // 2], b[qkey][:N_REF // 2]
        data, offsets = packed(seq)
        exp, eqt = oracle.oracle_process_packed(descs, groups, data, offsets, packed(qual)[0], True, 0, 20)
        ra = RA.BackAdapter(adapter, max_errors=0.1, min_overlap=3, name="x")
        want = []
        for read, q in zip(to_strings(seq), to_strings(qual)):
            s, e = quality_trim_index(q, 0, 20, 33)
            want.append([[s, e], m6(ra.match_to(read[s:e]))])
        digests(f"gate_config4_{skey}", want, [[list(eqt[i]), rec6(exp[i, 0, 0])] for i in range(len(want))], out)
    # config 5: the barcode index
    multi, _ = config_adapters(5)
    seq = make_config_batch(5, N_GATE, device="cpu")["seq"][:N_REF]
    singles, _, _ = multi._flatten()
    barcodes = config5_barcodes()
    exp = oracle.oracle_index_process(barcodes, 0.1, True, True, *packed(seq), [s.descriptor() for s in singles])
    idx = RA.IndexedPrefixAdapters([RA.PrefixAdapter(bc, max_errors=0.1, min_overlap=3, indels=True, name=f"bc{i}")
                                    for i, bc in enumerate(barcodes)])
    want = []
    for read in to_strings(seq):
        m = idx.match_to(read)
        want.append(None if m is None else [int(m.adapter.name[2:])] + m6(m))
    digests("gate_config5", want, [None if r["adapter"] < 0 else [int(r["adapter"])] + rec6(r) for r in exp], out)


def parity(out):
    import cutadapt.adapters as RA
    import cutadapt_b200.adapters as PA
    from cutadapt_b200.synth import make_reads
    from oracle import oracle

    reads, _ = make_reads(10000, config=1)
    reads = reads[:3000]
    exp, _ = oracle.oracle_process([PA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1, name="a").descriptor()], None, reads)
    ra = RA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1, name="a")
    digests("config1_single_adapter", [m6(ra.match_to(r)) for r in reads], [rec6(r) for r in exp[:, 0, 0]], out)


def oracle_tests(out):
    import cutadapt._align as ra
    import cutadapt.adapters as RA
    import cutadapt_b200.adapters as PA
    from cutadapt.qualtrim import quality_trim_index
    from cutadapt_b200.configs import config5_barcodes, to_strings
    from oracle import oracle

    want, have = [], []
    for args, queries, qs in random_locate_cases():
        al = ra.Aligner(*args)
        want.append([[al.locate(q) for q in queries], quality_trim_index(qs, 5, 20)])
        have.append([[oracle.locate(args[0], q, *args[1:]) for q in queries], oracle.quality_trim_index(qs, 5, 20)])
    digests("locate_random", want, have, out)
    bcs = config5_barcodes()
    seq = index_test_reads()
    for indels in (True, False):
        idx = RA.IndexedPrefixAdapters([RA.PrefixAdapter(b, max_errors=0.1, indels=indels, name=f"bc{i}")
                                        for i, b in enumerate(bcs)])
        lengths, index = oracle.index_build(bcs, 0.1, indels)
        digests(f"index_keys_indels{int(indels)}", [[sorted(idx._index._index), list(idx._index._lengths)]],
                [[sorted(index), list(lengths)]], out)
        descs = [PA.PrefixAdapter(b, max_errors=0.1, indels=indels, name=f"bc{i}").descriptor() for i, b in enumerate(bcs)]
        exp = oracle.oracle_index_process(bcs, 0.1, indels, True, *packed(seq), descs)
        want = []
        for r in to_strings(seq):
            m = idx.match_to(r)
            want.append(None if m is None else [int(m.adapter.name[2:])] + m6(m))
        digests(f"index_matches_indels{int(indels)}", want,
                [None if r["adapter"] < 0 else [int(r["adapter"])] + rec6(r) for r in exp], out)


def distributed(out):
    import _dist_worker
    import cutadapt.adapters as RA

    reads, _ = _dist_worker.workload()
    robjs = [RA.BackAdapter("AGATCGGAAGAGC", max_errors=0.1, name="a"), RA.FrontAdapter("ACGTTGCATTGAC", max_errors=0.1, name="f"),
             RA.AnywhereAdapter("CTGTCTCTTATACACATCT", max_errors=0.1, name="w"),
             RA.LinkedAdapter(RA.PrefixAdapter("GTTCAGAGTTCTACAGTCCGACGATC", max_errors=0.1, name="lf"),
                              RA.BackAdapter("TGGAATTCTCGGGTGCCAAGG", max_errors=0.1, name="lb"), False, False, "linked")]
    rmulti = RA.MultipleAdapters(robjs)
    rstats = {id(a): a.create_statistics() for a in robjs}
    for read in reads:
        m = rmulti.match_to(read)
        if m is not None:
            rstats[id(m.adapter)].add_match(m)
    out["distributed_end_statistics"] = [end_statistics_answer(rstats[id(a)]) for a in robjs]


def kmer_heuristic(out):
    """The k-mer search sets of the reference's kmer_heuristic on the inputs of its own tests and on real adapters."""
    from cutadapt import kmer_heuristic as K

    adapter = "ABCDEFGHIJ0123456789"
    chunks = [[s, c, sorted(K.kmer_chunks(s, c))] for s, c in (("ABC", 3), ("ABCD", 3), (adapter, 3), (adapter[:10], 2))]
    lists = [[("ABC", -33, None), ("ABC", -19, None)],
             [("ABC", -33, None), ("ABC", -19, None), ("ABC", 0, None)],
             [("ABC", 0, 10), ("ABC", 0, 20)],
             [("ABC", 0, 10), ("ABC", 0, 20), ("ABC", 0, None)],
             [("ABC", 0, 10), ("ABC", -19, None), ("ABC", 0, None)],
             [("ABC", 0, 10), ("ABC", -19, None)]]
    minimized = [[canonical(lst), sorted(canonical(K.minimize_kmer_search_list(lst)), key=repr)] for lst in lists]
    searchsets = [[adapter, 3, 0.1, sorted(([a, b, sorted(k)] for a, b, k in K.create_back_overlap_searchsets(adapter, 3, 0.1)), key=repr)]]
    positions = []
    for seq in (adapter, "AGATCGGAAGAGC", "CTGTCTCTTATACACATCT", "AGATCGGAAGAGCACACGTCTGAACTCCAGTCA"):
        for back, front, internal, mo in ((True, False, True, 3), (True, False, False, 3), (False, True, False, 3),
                                          (True, False, True, 20), (False, False, True, 3), (False, True, True, 1)):
            kw = dict(back_adapter=back, front_adapter=front, internal=internal, min_overlap=mo)
            res = K.create_positions_and_kmers(seq, error_rate=0.1, **kw)
            positions.append([seq, kw, sorted(([a, b, sorted(k)] for a, b, k in res), key=repr)])
    out["kmer_heuristic"] = {"chunks": chunks, "minimize": minimized, "searchsets": searchsets, "positions": positions}


def provenance(reference):
    """Which reference sources the answers come from: SHA-256 of every file oracle/_ref was compiled from."""
    import hashlib

    import Cython
    import cutadapt._align
    from oracle import build_ref

    assert os.path.dirname(os.path.abspath(cutadapt._align.__file__)) == build_ref.OUT, cutadapt._align.__file__
    src = os.path.join(reference, "src", "cutadapt")
    files = {}
    for mod in build_ref.PYX + build_ref.PY:
        name = mod + (".pyx" if mod in build_ref.PYX else ".py")
        with open(os.path.join(src, name), "rb") as f:
            files[name] = hashlib.sha256(f.read()).hexdigest()
    return {"reference_sources_sha256": files, "cython": Cython.__version__,
            "checked_against": "every answer set equals the C oracle's (oracle/cutadapt_oracle.c) on the same inputs"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("CUTADAPT_REFERENCE"),
                    help="checkout of the reference (default: $CUTADAPT_REFERENCE)")
    args = ap.parse_args()
    if not args.reference:
        ap.error("needs a checkout of the reference: --reference DIR or $CUTADAPT_REFERENCE")
    from oracle import build_ref

    # always rebuilt from the given checkout, so the answers below come from exactly the sources hashed here
    build_ref.build(args.reference, force=True)
    build_ref.import_ref()
    out = {"provenance": provenance(args.reference)}
    kmer_heuristic(out)
    distributed(out)
    oracle_tests(out)
    parity(out)
    gate(out)
    path = os.path.join(HERE, "reference_kat.json.gz")
    data = json.dumps(out, separators=(",", ":"), sort_keys=True).encode()
    with open(path, "wb") as raw:
        with gzip.GzipFile(fileobj=raw, mode="wb", mtime=0, filename="") as f:
            f.write(data)
    print(f"{path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
