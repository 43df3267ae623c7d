"""
The per-read row outputs (--info-file, --rest-file, --wildcard-file) of one mate or of a pair from the oracle (test
infrastructure): oracle/oracle.py's _fastq_evaluate formats the rows of every record while it trims, applying the info
coordinates to the read as it came; oracle_fastq_trim_paired hands each mate's options on to it, so the rows of R1 and
R2 come through as they are -- with pair_specs too, where the matches come from match_override and `adapter` is the
number of the pair.  Also the known answer of the reference's paired info files (tests/golden/paired_rows_kat.json.gz).
"""
import gzip
import json
import os

import fasta_oracle as FO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "paired_rows_kat.json.gz")
KINDS = ("info", "rest", "wildcard")


def paired_rows_kat():
    with gzip.open(GOLDEN, "rb") as f:
        return json.loads(f.read().decode())


def kat_bytes(kat, key) -> bytes:
    return kat["files"][key].encode("latin-1")


def strip_trailing(text: bytes) -> bytes:
    """A file compared as the reference's assert_files_equal(..., ignore_trailing_space=True) compares it."""
    return b"\n".join(line.rstrip() for line in text.split(b"\n"))


def row_options(adapters, kinds):
    """(options for _fastq_evaluate, {kind: list receiving the rows}) of a mate's adapters (cutadapt_b200 objects, one
    entry per adapter, no linked adapters: rest and wildcard rows are undefined for them)."""
    lists = {k: [] for k in kinds}
    names = [a.name for a in adapters or []]
    opts = {}
    if "info" in lists:
        opts.update(info_names=names, info_rows=lists["info"])
    if "rest" in lists:
        opts["rest_rows"] = lists["rest"]
    if "wildcard" in lists:
        opts.update(wildcard_rows=lists["wildcard"], adapter_sequences=[a.sequence for a in adapters or []])
    return opts, lists


def _text(lists):
    return {k: "".join(r + "\n" for r in v).encode("latin-1") for k, v in lists.items()}


def oracle_rows_single(oracle, data, adapters, kw, kinds=KINDS):
    """(output, counters, {kind: rows}) of a single-end chunk."""
    descs, groups = FO.descriptors(adapters)
    opts, lists = row_options(adapters, kinds)
    out, c = oracle.oracle_fastq_trim(data, descs, groups, **kw, **opts)
    return out, c, _text(lists)


def oracle_rows_paired(oracle, data1, data2, adapters1, adapters2, kw1, kw2, kinds1=KINDS, kinds2=("info",),
                       pair_filter="any", pair_adapters=False):
    """(out1, out2, counters1, counters2, {kind: rows of R1}, {kind: rows of R2}) of a chunk pair; pair_adapters:
    adapter i of each list forms pair i (--pair-adapters)."""
    o1, l1 = row_options(adapters1, kinds1)
    o2, l2 = row_options(adapters2, kinds2)
    kw1, kw2 = dict(kw1, **o1), dict(kw2, **o2)
    if pair_adapters:
        specs = [(FO.descriptors([a1]), FO.descriptors([a2])) for a1, a2 in zip(adapters1, adapters2)]
        out1, out2, c1, c2 = oracle.oracle_fastq_trim_paired(data1, data2, options1=kw1, options2=kw2,
                                                             pair_filter=pair_filter, pair_specs=specs)
    else:
        out1, out2, c1, c2 = oracle.oracle_fastq_trim_paired(data1, data2, *FO.descriptors(adapters1),
                                                             *FO.descriptors(adapters2), kw1, kw2, pair_filter)
    return out1, out2, c1, c2, _text(l1), _text(l2)
