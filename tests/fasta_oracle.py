"""
FASTA on top of the FASTQ oracle (test infrastructure): a FASTA reader with the rules of cg_fastq_params.format 1
(include/cutadapt_b200.h), written line by line and independently of the device's normalisation, and the FASTA writer.
A FASTA chunk runs through oracle.oracle_fastq_* as FASTQ with placeholder qualities; nothing that reads qualities is
allowed on FASTA input, so the placeholders never matter, and the outputs are turned back into FASTA (info-file rows
get their empty quality columns back).
"""
from oracle import oracle

PLACEHOLDER_QUALITY = "I"


class FastaFormatError(ValueError):
    pass


def parse_fasta(data: bytes):
    """[(name, sequence)] as str.  '>' starts a record, sequence lines are joined, '#' lines in front of the first
    record are skipped, "\\r\\n" is accepted; a '#' line after the first record or any other line in front of it raises
    FastaFormatError naming the line (1-based)."""
    if not data:
        return []
    lines = data.split(b"\n")
    if lines[-1] == b"":
        lines.pop()
    records = []
    for i, line in enumerate(lines, 1):
        if line.endswith(b"\r"):
            line = line[:-1]
        if line.startswith(b">"):
            records.append([line[1:].decode("latin-1"), []])
        elif line.startswith(b"#"):
            if records:
                raise FastaFormatError(f"line {i}: a '#' comment line after the first record")
        elif not records:
            raise FastaFormatError(f"line {i}: expected '>' at the beginning of a record")
        else:
            records[-1][1].append(line.decode("latin-1"))
    return [(name, "".join(seq)) for name, seq in records]


def fasta_record(name: str, sequence: str) -> bytes:
    return f">{name}\n{sequence}\n".encode("latin-1")


def as_fastq(data: bytes) -> bytes:
    """A FASTA chunk as FASTQ with placeholder qualities (what the FASTQ oracle takes)."""
    return b"".join(f"@{n}\n{s}\n+\n{PLACEHOLDER_QUALITY * len(s)}\n".encode("latin-1") for n, s in parse_fasta(data))


def fastq_as_fasta(data: bytes) -> bytes:
    """FASTQ output of the oracle written as FASTA instead."""
    return b"".join(fasta_record(n, s) for n, s, _ in oracle.parse_fastq(data))


def _no_qualities(options):
    for key in ("quality_trim", "nextseq_cutoff"):
        if options.get(key):
            raise ValueError(f"{key} needs qualities")
    if options.get("max_expected_errors", -1) >= 0:
        raise ValueError("max_expected_errors needs qualities")


def _input(data, input_format, options):
    if input_format == "fasta":
        _no_qualities(options)
        return as_fastq(data)
    return data


def _output(data, input_format, output_format):
    return fastq_as_fasta(data) if (output_format or input_format) == "fasta" else data


def info_rows_without_qualities(rows):
    """--info-file rows of FASTA input: the quality columns are empty (adapters.py:408-415, steps.py:250)."""
    out = []
    for row in rows:
        f = row.split("\t")
        if len(f) == 4 and f[1] == "-1":
            f[3] = ""
        else:
            f[8] = f[9] = f[10] = ""
        out.append("\t".join(f))
    return out


def fasta_trim(data: bytes, adapters=None, groups=None, input_format="fasta", output_format=None, **options):
    """oracle.oracle_fastq_trim for FASTA input and / or FASTA output: (output bytes, counters)."""
    rows = options.get("info_rows")
    out, c = oracle.oracle_fastq_trim(_input(data, input_format, options), adapters, groups, **options)
    if rows is not None and input_format == "fasta":
        rows[:] = info_rows_without_qualities(rows)
    return _output(out, input_format, output_format), c


def fasta_demux(data: bytes, adapters, groups, adapter_names, input_format="fasta", output_format=None, **options):
    got = oracle.oracle_fastq_demux(_input(data, input_format, options), adapters, groups, adapter_names, **options)
    return {k: _output(v, input_format, output_format) for k, v in got.items()}


def fasta_trim_paired(data1: bytes, data2: bytes, adapters1=None, groups1=None, adapters2=None, groups2=None,
                      options1=None, options2=None, pair_filter="any", route=None, input_format="fasta",
                      output_format=None):
    options1, options2 = dict(options1 or {}), dict(options2 or {})
    o1, o2, c1, c2 = oracle.oracle_fastq_trim_paired(
        _input(data1, input_format, options1), _input(data2, input_format, options2), adapters1, groups1, adapters2,
        groups2, options1, options2, pair_filter, route=route)
    if route:
        return ({k: _output(v, input_format, output_format) for k, v in o1.items()},
                {k: _output(v, input_format, output_format) for k, v in o2.items()}, c1, c2)
    return _output(o1, input_format, output_format), _output(o2, input_format, output_format), c1, c2


# ---- the known-answer cases of tests/golden/fasta_kat.json.gz (tests/golden/make_fasta_golden.py) -------------------

_KAT = None


def fasta_kat():
    global _KAT
    if _KAT is None:
        from util import golden

        _KAT = golden("fasta_kat.json.gz")
    return _KAT


def kat_file(key) -> bytes:
    return fasta_kat()["files"][key].encode("latin-1")


def kat_adapters(options, key="specs"):
    """The adapters of a case as its command line builds them (-e, -O, -N, --no-indels, --match-read-wildcards)."""
    from util import adapter_from_spec

    params = dict(max_errors=options.get("error_rate", 0.1), min_overlap=options.get("min_overlap", 3),
                  adapter_wildcards=not options.get("no_wildcards", False),
                  read_wildcards=options.get("read_wildcards", False), indels=not options.get("no_indels", False))
    return [adapter_from_spec(spec, kind, name=None if "=" in spec else f"a{i}", **params)
            for i, (kind, spec) in enumerate(options.get(key, []))]


KAT_OPTION_KEYS = ("times", "action", "minimum_length", "maximum_length", "discard_untrimmed", "discard_trimmed",
                   "trim_n", "poly_a", "max_n", "revcomp", "rc_suffix")


def kat_kwargs(options):
    """Keyword arguments shared by the oracle and pipeline.FastqTrimmer (formats excluded)."""
    return {k: options[k] for k in KAT_OPTION_KEYS if k in options}


def kat_formats(options):
    return dict(input_format=options.get("input_format", "fasta"), output_format=options.get("output_format"))


def descriptors(adapters):
    """(descriptors, groups) of a list of cutadapt_b200 adapters for the oracle, or (None, None)."""
    import cutadapt_b200.adapters as PA
    from util import spec_of

    if not adapters:
        return None, None
    spec = spec_of(PA.MultipleAdapters(adapters))
    return spec.adapters, spec.groups


def info_names(adapters):
    """Adapter names per flattened adapter, as the info file shows them."""
    import cutadapt_b200.adapters as PA

    singles, _, _ = PA.MultipleAdapters(adapters)._flatten()
    return [s.name for s in singles]

