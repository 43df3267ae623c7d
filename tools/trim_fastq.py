#!/usr/bin/env python3
"""
Trim FASTQ and FASTA files on the GPU: a minimal driver around cutadapt_b200.pipeline.FastqTrimmer / PairedFastqTrimmer
that understands the subset of cutadapt's options the device path implements.  Not a replacement for cutadapt's
command line (no reports): it shows the per-chunk worker of INTEGRATION.md section 3 running on real files.

  python tools/trim_fastq.py -a AGATCGGAAGAGC -q 20 -m 20 -o out.fastq in.fastq
  python tools/trim_fastq.py -a ADAPT1 -A ADAPT2 -q 20 -m 20 -o out.1.fastq -p out.2.fastq in.1.fastq in.2.fastq
  python tools/trim_fastq.py -g bc1=^ACGTACGTAC -g bc2=^TTGCATTGCA -o 'demux-{name}.fastq' in.fastq     (demultiplex)
  python tools/trim_fastq.py -a AGATCGGAAGAGC -m 20 -o out.fasta in.fasta           (FASTA; also FASTQ -> FASTA)
  python tools/trim_fastq.py -a AGATCGGAAGAGC -m 20 --too-short-output short.fastq --untrimmed-output untrimmed.fasta \
      -o out.fastq in.fastq                                                            (filter outputs)
  python tools/trim_fastq.py --interleaved -a ADAPT1 -A ADAPT2 -m 20:25 -o out.fastq in.interleaved.fastq
  python tools/trim_fastq.py -a AGATCGGAAGAGC -o out.fastq.gz in.fastq.gz                   (gzip)

The input format comes from the first byte of the (first) input, as cutadapt's files.detect_file_format does: '>' or
'#' is FASTA, anything else (an empty file included) FASTQ.  The output is FASTA when the input is, when -o ends in
.fasta / .fa, or with --fasta; every filter output (--too-short-output, --too-long-output, --untrimmed-output and the
paired forms) gets its format from its own name the same way.  --json FILE also writes what the report shows per adapter (removed length x errors,
bases preceding the adapter, reverse-complemented count), the poly-A and written-length histograms and the counters,
collected on the device (collect_statistics=True); the stderr line stays as it is.

--interleaved, as in the reference: one input is interleaved input (R1 and R2 of each pair one after the other, split
on the device), no -p means an interleaved main output, and a filter output without its --*-paired-output is written
interleaved.  -m / -M take LEN[:LEN2], a length for each mate; an empty side means no filter on that mate.

Compressed files: every output whose name ends in .gz (-o, -p, the filter outputs, a {name} template) is written as gzip,
compressed on the device in members of 65 280 bytes; the others are plain, each decided by its own name.  One
exception: with demultiplexing the device compresses all demultiplexed outputs alike, so --untrimmed-output (which
receives the "unknown" output) must end in .gz exactly when the -o template does; otherwise the tool stops with an
error.  A .gz output
that receives no read still gets one empty gzip member.  The device has one compression strategy, comparable in size to
zlib's level 1, so there is no --compression-level.  An input ending in .gz whose first gzip member ends within its
first MiB (BGZF, concatenated .gz files, this tool's own .gz outputs) is inflated on the device: the compressed bytes are
uploaded (read_gzip_device_chunks; for two paired inputs only when both qualify).  Any other .gz input is decompressed on
the host with Python's gzip module.  The outputs are the same either way; the stderr line's "in_bytes_gzip" (the
compressed bytes consumed) appears only when the device inflated the input.  The format is detected from the first
decompressed byte.
"""
import argparse
import gzip
import zlib
import json
import sys

sys.path.insert(0, __file__.rsplit("/", 2)[0])
import cutadapt_b200.adapters as PA  # noqa: E402
from cutadapt_b200.pipeline import (FastqTrimmer, PairedFastqTrimmer, read_fasta_chunks,  # noqa: E402
                                    read_fastq_chunks, read_gzip_device_chunks, read_gzip_device_interleaved_chunks,
                                    read_gzip_device_paired_chunks, read_interleaved_fasta_chunks,
                                    read_interleaved_fastq_chunks, read_paired_fasta_chunks, read_paired_fastq_chunks)


def open_input(path):
    """An input file for reading; a .gz one is decompressed on the host."""
    return gzip.open(path, "rb") if path.endswith(".gz") else open(path, "rb")


# A .gz input goes to the device (read_gzip_device_chunks) when its first member ends within this many compressed
# bytes: one GPU thread inflates a member, so only files of many members gain (DESIGN.md section 4.8 has the measurement).
DEVICE_GZIP_FIRST_MEMBER = 1 << 20


def gzip_on_device(path):
    """Whether a .gz input is inflated on the device: host zlib inflates its first member from a prefix of the file,
    and the member must end within the first DEVICE_GZIP_FIRST_MEMBER compressed bytes."""
    if not path.endswith(".gz"):
        return False
    with open(path, "rb") as f:
        head = f.read(DEVICE_GZIP_FIRST_MEMBER)
    d = zlib.decompressobj(31)
    try:
        while head and not d.eof:
            d.decompress(head, 1 << 20)           # bounded output: only where the member ends matters
            head = d.unconsumed_tail
    except zlib.error:
        return False                              # the host path reports the error as Python's gzip module does
    return d.eof


def detect_format(path):
    """"fasta" or "fastq" from the first (decompressed) byte (files.py:314-333)."""
    with open_input(path) as f:
        return "fasta" if f.read(1) in (b">", b"#") else "fastq"


# what zlib writes for no data: the device's member header, an empty final block, CRC and size 0
EMPTY_GZIP = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff\x03\x00" + bytes(8)


class OutputFile:
    """An output file.  A .gz one receives gzip members from the device; if it gets no byte at all, close() writes one
    empty member so that it stays a valid gzip file, as the reference does."""

    def __init__(self, path):
        self.gzip = path.endswith(".gz")
        self.f = open(path, "wb")
        self.written = 0

    def write(self, data):
        self.written += len(data)
        self.f.write(data)

    def close(self):
        if self.gzip and self.written == 0:
            self.f.write(EMPTY_GZIP)
        self.f.close()


def make_adapters(specs, kind, error_rate, overlap):
    """-a / -g / -b values: [name=]SEQUENCE with the anchoring characters ^ (5') and $ (3')."""
    out = []
    for i, spec in enumerate(specs or []):
        name, _, seq = spec.rpartition("=")
        name = name or f"{kind}{i + 1}"
        kw = dict(max_errors=error_rate, min_overlap=overlap, name=name)
        if kind == "front" and seq.startswith("^"):
            out.append(PA.PrefixAdapter(seq[1:], **kw))
        elif kind == "back" and seq.endswith("$"):
            out.append(PA.SuffixAdapter(seq[:-1], **kw))
        else:
            out.append({"back": PA.BackAdapter, "front": PA.FrontAdapter, "anywhere": PA.AnywhereAdapter}[kind](seq, **kw))
    return out


def _end(e):
    if e is None:
        return None
    return {"errors": {str(length): {str(k): n for k, n in sorted(row.items())} for length, row in sorted(e.errors.items())},
            "adjacent_bases": dict(e.adjacent_bases)}


def report_json(counters, adapter_statistics, poly_a, written):
    """One mate's statistics as --json writes them."""
    return {"counters": counters,
            "adapters": [{"name": st.name, "reverse_complemented": int(st.reverse_complemented),
                          "five_prime_end": _end(st.front), "three_prime_end": _end(st.back)}
                         for st in adapter_statistics],
            "poly_a_trimmed_lengths": {str(k): v for k, v in sorted(poly_a.items())},
            "written_lengths": {str(k): v for k, v in sorted(written.items())}}


def parse_lengths(s):
    """-m / -M: LEN or LEN1:LEN2 with one side possibly empty (cli.py:443-465, parse_lengths) -> tuple of int / None.
    ValueError names what is wrong."""
    fields = s.split(":")
    if len(fields) not in (1, 2):
        raise ValueError("Only at most one colon is allowed")
    try:
        values = tuple(int(f) if f != "" else None for f in fields)
    except ValueError as e:
        raise ValueError(f"Value not recognized: {e}")
    if len(values) == 2 and values[0] is None and values[1] is None:
        raise ValueError(f"Cannot parse '{s}': At least one length needs to be given")
    return values


def mate_lengths(ap, value, paired):
    """(length of R1, length of R2) of a -m / -M value (None: no filter on that mate)."""
    if value is None:
        return None, None
    try:
        lengths = parse_lengths(value)
    except ValueError as e:
        ap.error(str(e))
    if not paired and len(lengths) == 2:
        ap.error("Two minimum or maximum lengths given for single-end data")
    return (lengths[0], lengths[0]) if len(lengths) == 1 else lengths


FILTER_OUTPUTS = (("too_short", "too-short"), ("too_long", "too-long"), ("untrimmed", "untrimmed"))


def check_filter_outputs(ap, args, paired, demultiplex, interleaved=False):
    """The command-line errors of the reference around the filter outputs (cli.py:588-592, 600-622, 713-733, 798-808):
    ap.error() exits with status 2."""
    if not paired and args.untrimmed_paired_output:
        ap.error("Option --untrimmed-paired-output can only be used when trimming paired-end reads.")
    if paired and not interleaved:
        for dest, name in FILTER_OUTPUTS:
            if bool(getattr(args, dest + "_output")) != bool(getattr(args, dest + "_paired_output")):
                ap.error("When trimming paired-end data, you must use either none or both of the"
                         f" --{name}-output/--{name}-paired-output options.")
    for length, dest, name, flag, what in ((args.minimum_length, "too_short", "too-short", "-m/--minimum-length", "minimum"),
                                           (args.maximum_length, "too_long", "too-long", "-M/--maximum-length", "maximum")):
        if length is None and (getattr(args, dest + "_output") or getattr(args, dest + "_paired_output")):
            ap.error(f"When --{name}-output or --{name}-paired-output are used, a {what} length must be provided with "
                     f"{flag}")
        if not paired and getattr(args, dest + "_paired_output"):
            ap.error("--too-short/long-paired-output cannot be used with single-end data")
    if int(args.discard_trimmed) + int(args.discard_untrimmed) + int(bool(args.untrimmed_output)) > 1:
        ap.error("Only one of the --discard-trimmed, --discard-untrimmed and --untrimmed-output options can be used at "
                 "the same time.")
    if demultiplex and (args.too_short_output or args.too_long_output):
        ap.error("--too-short-output and --too-long-output cannot be combined with demultiplexing ({name} in -o)")


def file_format(path, input_format, fasta):
    """Format of an output file: FASTA for FASTA input, with --fasta, or for a .fasta / .fa name (.gz behind it)."""
    name = path[:-3] if path.endswith(".gz") else path
    return "fasta" if input_format == "fasta" or fasta or name.endswith((".fasta", ".fa")) else "fastq"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    for flag, dest in (("-a", "back"), ("-g", "front"), ("-b", "anywhere"), ("-A", "back2"), ("-G", "front2"),
                       ("-B", "anywhere2")):
        ap.add_argument(flag, dest=dest, action="append")
    ap.add_argument("-e", "--error-rate", type=float, default=0.1)
    ap.add_argument("-O", "--overlap", type=int, default=3)
    ap.add_argument("-n", "--times", type=int, default=1)
    ap.add_argument("-q", "--quality-cutoff", default=None, help="[5'CUTOFF,]3'CUTOFF")
    ap.add_argument("--quality-base", type=int, default=33)
    ap.add_argument("--nextseq-trim", type=int, default=None)
    ap.add_argument("-u", "--cut", type=int, action="append", default=[])
    ap.add_argument("-m", "--minimum-length", default=None, metavar="LEN[:LEN2]")
    ap.add_argument("-M", "--maximum-length", default=None, metavar="LEN[:LEN2]")
    ap.add_argument("--interleaved", action="store_true",
                    help="read and/or write interleaved paired-end reads (one input file, or no -p)")
    ap.add_argument("--max-n", type=float, default=None)
    ap.add_argument("--max-ee", type=float, default=None)
    ap.add_argument("--length", "-l", type=int, default=None)
    ap.add_argument("--poly-a", action="store_true")
    ap.add_argument("--trim-n", action="store_true")
    ap.add_argument("--discard-casava", action="store_true")
    ap.add_argument("--discard-trimmed", action="store_true")
    ap.add_argument("--discard-untrimmed", action="store_true")
    ap.add_argument("--action", default="trim", choices=["trim", "none", "mask", "lowercase", "retain", "crop"])
    ap.add_argument("--pair-filter", default="any", choices=["any", "both", "first"])
    ap.add_argument("--fasta", action="store_true", help="write FASTA even for FASTQ input")
    ap.add_argument("--buffer-size", type=int, default=64 << 20)
    ap.add_argument("-o", "--output", required=True, help="output FASTQ; with {name}: one file per adapter name")
    ap.add_argument("-p", "--paired-output")
    ap.add_argument("--json", default=None, metavar="FILE", help="write the report's statistics as JSON")
    for dest, name in FILTER_OUTPUTS:
        ap.add_argument(f"--{name}-output", dest=dest + "_output", metavar="FILE",
                        help=f"write the reads the {name} filter removes to FILE instead of dropping them")
        ap.add_argument(f"--{name}-paired-output", dest=dest + "_paired_output", metavar="FILE",
                        help=f"the second mates of the pairs --{name}-output gets")
    ap.add_argument("inputs", nargs="+")
    args = ap.parse_args()
    if args.interleaved and len(args.inputs) == 2 and args.paired_output:
        ap.error("--interleaved was given with two input files and two output files (-o and -p): use it for interleaved "
                 "input (one input file) or interleaved output (no -p)")
    if len(args.inputs) > 2:
        ap.error("at most two input files")
    paired = len(args.inputs) == 2 or args.interleaved
    min1, min2 = mate_lengths(ap, args.minimum_length, paired)
    max1, max2 = mate_lengths(ap, args.maximum_length, paired)
    check_filter_outputs(ap, args, paired, "{name}" in args.output, args.interleaved)
    input_format = detect_format(args.inputs[0])
    fasta_out = file_format(args.output, input_format, args.fasta) == "fasta"
    output_format = "fasta" if fasta_out and input_format == "fastq" else None
    if input_format == "fasta" and args.max_ee is not None:
        print("WARNING: Ignoring option --max-ee because input does not provide quality values", file=sys.stderr)
        args.max_ee = None
    host_reader = read_fasta_chunks if input_format == "fasta" else read_fastq_chunks
    # compressed bytes per submission of a device-inflated input: one thread inflates a member, so a submission must hold
    # many members; with --buffer-size 64 MiB, members of up to 1 MiB give 64 or more at once
    gz_buffer = args.buffer_size

    def single_input(t):
        """(file, chunks) of the single input for trimmer t."""
        if gzip_on_device(args.inputs[0]):
            f = open(args.inputs[0], "rb")
            return f, read_gzip_device_chunks(f, t, gz_buffer)
        f = open_input(args.inputs[0])
        return f, host_reader(f, args.buffer_size)
    paired_reader = read_paired_fasta_chunks if input_format == "fasta" else read_paired_fastq_chunks

    qc = None
    if args.quality_cutoff is not None:
        parts = [int(x) for x in args.quality_cutoff.split(",")]
        qc = (0, parts[0]) if len(parts) == 1 else (parts[0], parts[1])
    common = dict(times=args.times, quality_cutoff=qc, quality_base=args.quality_base, nextseq_cutoff=args.nextseq_trim,
                  minimum_length=min1, maximum_length=max1, max_n=args.max_n,
                  max_expected_errors=args.max_ee, discard_trimmed=args.discard_trimmed,
                  discard_untrimmed=args.discard_untrimmed, cut=args.cut, poly_a=args.poly_a, length=args.length,
                  trim_n=args.trim_n, discard_casava=args.discard_casava, action=args.action)
    formats = dict(input_format=input_format, output_format=output_format, collect_statistics=args.json is not None)
    # filter outputs (the untrimmed output of a demultiplexer is its "unknown" output)
    redirect = [d for d, _ in FILTER_OUTPUTS if getattr(args, d + "_output") and "{name}" not in args.output]
    split = dict(redirect=redirect,
                 redirect_formats={d: file_format(getattr(args, d + "_output"), input_format, args.fasta)
                                   for d in redirect}) if redirect else {}
    # the outputs compressed on the device: R1's files, R2's (an interleaved output's R2 goes to R1's file)
    paths1 = dict({d: getattr(args, d + "_output") for d in redirect}, output=args.output)
    paths2 = dict({d: getattr(args, d + "_paired_output") or paths1[d] for d in redirect},
                  output=args.paired_output or args.output)
    gzip1 = [d for d, p in paths1.items() if p.endswith(".gz")]
    gzip2 = [d for d, p in paths2.items() if p.endswith(".gz")]
    ads1 = (make_adapters(args.back, "back", args.error_rate, args.overlap)
            + make_adapters(args.front, "front", args.error_rate, args.overlap)
            + make_adapters(args.anywhere, "anywhere", args.error_rate, args.overlap))
    ads2 = (make_adapters(args.back2, "back", args.error_rate, args.overlap)
            + make_adapters(args.front2, "front", args.error_rate, args.overlap)
            + make_adapters(args.anywhere2, "anywhere", args.error_rate, args.overlap))

    if paired:
        if not args.paired_output and not args.interleaved:
            ap.error("paired-end input needs -p (or --interleaved for an interleaved output)")
        if len(args.inputs) == 2 and detect_format(args.inputs[1]) != input_format:
            ap.error("both inputs must have the same format")
        options2 = dict(common, minimum_length=min2, maximum_length=max2)
        # an output is interleaved when its paired path is missing (cli.py:650-661, 913-921)
        interleaved = [d for d in ["output"] + redirect
                       if not (args.paired_output if d == "output" else getattr(args, d + "_paired_output"))]
        t = PairedFastqTrimmer(ads1, ads2, common, options2, args.pair_filter, **formats, **split,
                               interleaved_outputs=interleaved, gzip_outputs=gzip1, gzip_outputs2=gzip2)
        if len(args.inputs) == 2 and all(map(gzip_on_device, args.inputs)):
            f1, f2 = open(args.inputs[0], "rb"), open(args.inputs[1], "rb")
            chunks = read_gzip_device_paired_chunks(f1, f2, t, gz_buffer)
        elif len(args.inputs) == 2:
            f1, f2 = open_input(args.inputs[0]), open_input(args.inputs[1])
            chunks = paired_reader(f1, f2, args.buffer_size)
        elif gzip_on_device(args.inputs[0]):
            f1 = f2 = open(args.inputs[0], "rb")
            chunks = read_gzip_device_interleaved_chunks(f1, t, gz_buffer)
        else:
            f1 = f2 = open_input(args.inputs[0])
            chunks = (read_interleaved_fasta_chunks if input_format == "fasta" else read_interleaved_fastq_chunks)(
                f1, args.buffer_size)
        paths = {d: (getattr(args, d + "_output"), getattr(args, d + "_paired_output")) for d in redirect}
        paths["output"] = (args.output, args.paired_output)
        files = {d: tuple(OutputFile(p) if p else None for p in ps) for d, ps in paths.items()}
        for parts in t.process_chunks_split(chunks):
            for name, (r1, r2) in parts.items():
                files[name][0].write(r1)
                if files[name][1] is not None:
                    files[name][1].write(r2)
        for fhs in files.values():
            for fh in fhs:
                if fh is not None:
                    fh.close()
        f1.close()
        f2.close()
        stats = {"read1": t.statistics[0], "read2": t.statistics[1]}
    elif "{name}" in args.output:
        # every demultiplexed output, "unknown" included, is compressed alike
        if args.untrimmed_output and args.untrimmed_output.endswith(".gz") != args.output.endswith(".gz"):
            ap.error("with demultiplexing, --untrimmed-output must be compressed (.gz) exactly when the -o template is")
        t = FastqTrimmer(ads1, **common, **formats, gzip_outputs=gzip1)
        files = {}
        f, chunks = single_input(t)
        with f:
            for chunk in chunks:
                for name, data in t.process_chunk_demux(chunk).items():
                    if name == "unknown" and args.discard_untrimmed:
                        continue
                    if name not in files:
                        # Demultiplexer(untrimmed_output=...): reads without a match go to --untrimmed-output
                        path = args.untrimmed_output if name == "unknown" and args.untrimmed_output else \
                            args.output.replace("{name}", name)
                        files[name] = OutputFile(path)
                    files[name].write(data)
        for fh in files.values():
            fh.close()
        stats = t.statistics
    elif redirect:
        t = FastqTrimmer(ads1, **common, **formats, **split, gzip_outputs=gzip1)
        f, chunks = single_input(t)
        with f:
            files = {d: OutputFile(getattr(args, d + "_output")) for d in redirect}
            files["output"] = OutputFile(args.output)
            for parts in t.process_chunks_split(chunks, copy=False):
                for name, data in parts.items():
                    files[name].write(data)
            for fh in files.values():
                fh.close()
        stats = t.statistics
    else:
        t = FastqTrimmer(ads1, **common, **formats, gzip_outputs=gzip1)
        o = OutputFile(args.output)
        f, chunks = single_input(t)
        with f:
            for out in t.process_chunks(chunks, copy=False):
                o.write(out.tobytes() if hasattr(out, "tobytes") else out)
        o.close()
        stats = t.statistics
    print(json.dumps(stats), file=sys.stderr)
    if args.json is not None:
        if paired:
            report = {f"read{k + 1}": report_json(t.statistics[k], t.adapter_statistics()[k], t.poly_a_trimmed_lengths[k],
                                                  t.written_lengths[k]) for k in (0, 1)}
        else:
            report = report_json(t.statistics, t.adapter_statistics(), t.poly_a_trimmed_lengths, t.written_lengths)
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
