"""
Interleaved paired-end data on top of the paired oracles (test infrastructure): an interleaved chunk is split into its
two mates, the existing paired oracle (oracle_fastq_trim_paired via fasta_oracle.fasta_trim_paired, or the redirect
oracle) trims them, and every output written interleaved gets R1 and R2 of each pair one after the other.  Also the
rule of dnaio's mate-name check (doc/reference.rst:925-950), restated in Python.
"""
import fasta_oracle as FO
import filter_outputs_oracle as RO


def _lines(data: bytes):
    out = [line + b"\n" for line in data.split(b"\n")]
    out[-1] = out[-1][:-1]
    return out if out[-1] else out[:-1]


def records(data: bytes, fmt: str):
    """The records of a chunk as their bytes: FASTQ 4 lines, FASTA from one header to the next."""
    lines = _lines(data)
    if fmt == "fastq":
        return [b"".join(lines[i:i + 4]) for i in range(0, len(lines), 4)]
    out = []
    for line in lines:
        if line.startswith(b">") or not out:
            out.append(line)
        else:
            out[-1] += line
    return out


def deinterleave(data: bytes, fmt: str):
    recs = records(data, fmt)
    assert len(recs) % 2 == 0
    return b"".join(recs[0::2]), b"".join(recs[1::2])


def interleave(a: bytes, b: bytes, fmt: str) -> bytes:
    ra, rb = records(a, fmt), records(b, fmt)
    assert len(ra) == len(rb)
    return b"".join(x + y for x, y in zip(ra, rb))


def mates_match(h1: bytes, h2: bytes) -> bool:
    """doc/reference.rst:925-950, the strict reading: the IDs (up to the first space or tab) must be equal after
    dropping a final 1, 2 or 3 -- from both IDs, and only when both end in one of them."""
    def ident(h):
        for k, c in enumerate(h):
            if c in b" \t":
                return h[:k]
        return h
    a, b = ident(h1), ident(h2)
    if a and b and a[-1:] in (b"1", b"2", b"3") and b[-1:] in (b"1", b"2", b"3"):
        a, b = a[:-1], b[:-1]
    return a == b


def interleaved_trim(data1: bytes, data2=None, adapters1=None, groups1=None, adapters2=None, groups2=None,
                     options1=None, options2=None, pair_filter="any", redirect=(), interleaved_outputs=(),
                     input_format="fastq", output_format=None, formats=None):
    """({output: (bytes1, bytes2)}, counters1, counters2) of one chunk pair, or of one interleaved chunk (data2 None);
    an output in interleaved_outputs is (R1 and R2 interleaved, b"")."""
    if data2 is None:
        data1, data2 = deinterleave(data1, input_format)
    if redirect:
        outs, c1, c2 = RO.redirect_trim_paired(data1, data2, adapters1, groups1, adapters2, groups2, options1, options2,
                                               pair_filter, redirect, formats, input_format, output_format)
    else:
        o1, o2, c1, c2 = FO.fasta_trim_paired(data1, data2, adapters1, groups1, adapters2, groups2, options1, options2,
                                              pair_filter, input_format=input_format, output_format=output_format)
        outs = {"output": (o1, o2)}
    fmts = RO._formats(redirect, formats, input_format, output_format)
    return {k: ((interleave(a, b, fmts[k]), b"") if k in interleaved_outputs else (a, b)) for k, (a, b) in outs.items()}, \
        c1, c2


# ---- the known-answer cases of tests/golden/interleaved_kat.json.gz (make_interleaved_golden.py) ---------------------

_KAT = None


def interleaved_kat():
    global _KAT
    if _KAT is None:
        from util import golden

        _KAT = golden("interleaved_kat.json.gz")
    return _KAT


def kat_file(key) -> bytes:
    return interleaved_kat()["files"][key].encode("latin-1")


def kat_trimmer_kwargs(options):
    """(options1, options2) of a case as PairedFastqTrimmer takes them"""
    def conv(o):
        o = dict(o)
        if "quality_cutoff" in o:
            o["quality_cutoff"] = tuple(o["quality_cutoff"])
        return o
    return conv(options.get("options1", {})), conv(options.get("options2", {}))


def kat_interleaved_outputs(case):
    """The outputs a case writes interleaved: those with one expected file."""
    return tuple(k for k, v in case["expected"].items() if len(v) == 1)
