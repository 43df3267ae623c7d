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
  python tools/trim_fastq.py -a AGATCGGAAGAGC -q 20 -m 20 -o out.fastq reads.bam             (unaligned BAM)
  python tools/trim_fastq.py --revcomp -g ^TTATTTGTCT -G ^TCCGCACTGG -o out.1.fastq -p out.2.fastq in.1.fastq in.2.fastq
  python tools/trim_fastq.py -a ADAPT1 -A ADAPT2 --info-file info1.txt.gz --info-file-paired info2.txt.gz \
      -o out.1.fastq -p out.2.fastq in.1.fastq in.2.fastq                               (per-read row files)

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
uploaded (read_gzip_device_chunks; for two paired inputs only when each qualifies under either rule).  Any other .gz
input of at least 16 MiB (DEVICE_GZIP_SPLIT_MIN; the single member that gzip and pigz write) is inflated on the device
block-parallel (split_members=True).  Smaller ones are decompressed on the host with Python's gzip module.  The outputs are the same either way; the stderr line's "in_bytes_gzip" (the
compressed bytes consumed) appears only when the device inflated the input.  The format is detected from the first
decompressed byte.

Unaligned BAM input (uBAM, as basecallers and GATK-style workflows write it) is detected by content, whatever the file
is called: a gzip file whose first member inflates to "BAM\\1".  It is read single-end only, as in the reference: its BGZF
members are inflated and its records decoded into FASTQ on the device (read_gzip_device_chunks), and the output is
FASTQ, or FASTA with --fasta or a .fasta / .fa name.  Two BAM inputs, or --interleaved with BAM, stop with an error.

--revcomp / --rc: the adapters are also searched on the reverse complement of each read and the better orientation
is written, " rc" appended to its name (ReverseComplementer).  On pairs the -a adapters also run on R2 and the -A
adapters on R1, and a pair that matches better that way is written with R1 and R2 swapped, " rc" on both names
(PairedReverseComplementer); --info-file is refused there.  --json counts them in "reverse_complemented".

Read names, as in the reference and in its order (after the adapters, --poly-a, --length and --trim-n; on pairs for
each mate): --length-tag TAG replaces TAG followed by digits with TAG and the length of the read as written (TAG may
hold letters, digits and _ = : , ; / - @ # % ! ~ only); --strip-suffix S (repeatable) removes S from the end of a name;
-x / -y add a prefix / suffix in which {name} is the adapter of the last match (no_adapter without one); --rename
TEMPLATE writes the name from the template's variables ({header}, {id}, {comment}, {cut_prefix}, {cut_suffix},
{adapter_name}, {rc}, {match_sequence}; on pairs also {rn} and {r1.x} / {r2.x}) and turns the " rc" of --revcomp off.
--rename cannot be combined with -x / -y.  Every output gets the new names, the row files included.  On pairs, -u
cuts R1 and -U R2, as in the reference ({cut_prefix} / {cut_suffix} show what each cut).

Row files: --info-file, -r/--rest-file and --wildcard-file get the rows of every read, filtered or not, formatted on the
device next to every kind of output above.  On pairs they get R1's rows, as in the reference (PairedSingleEndStep,
cli.py:675-696); --info-file-paired adds R2's info rows, and only together with --info-file; it also makes the run
paired (cli.py:537), so one input then needs --interleaved.  A row file whose name ends in .gz is compressed on the
device like the other outputs.  Row files cannot go to standard output.
"""
import argparse
import gzip
import zlib
import json
import os
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


# A .gz input that fails gzip_on_device (typically the one member written by gzip or pigz) still goes to the device when
# it holds at least this many compressed bytes: read_gzip_device_chunks(split_members=True) inflates the member
# block-parallel.  Measured by file size (DESIGN.md section 4.8): the device wins from 16 MiB on and loses at 8 MiB,
# where one submission holds too few deflate blocks to occupy the GPU.
DEVICE_GZIP_SPLIT_MIN = 16 << 20


def gzip_route(path):
    """How a .gz input is read: "members" (gzip_on_device), "split" (a long member of a file of at least
    DEVICE_GZIP_SPLIT_MIN compressed bytes, inflated block-parallel on the device) or None (Python's gzip module)."""
    if gzip_on_device(path):
        return "members"
    if path.endswith(".gz") and os.path.getsize(path) >= DEVICE_GZIP_SPLIT_MIN:
        return "split"
    return None


def is_bam(path):
    """Whether an input is BAM, by content as xopen plus detect_file_format see it: the file starts with 1f 8b and its
    first gzip member inflates to "BAM\\1" (any name; .bam is the usual one)."""
    with open(path, "rb") as f:
        head = f.read(DEVICE_GZIP_FIRST_MEMBER)
    if head[:2] != b"\x1f\x8b":
        return False
    try:
        return zlib.decompressobj(31).decompress(head, 4) == b"BAM\x01"
    except zlib.error:
        return False


def detect_format(path):
    """"bam", or "fasta" / "fastq" from the first (decompressed) byte (files.py:304-333)."""
    if is_bam(path):
        return "bam"
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
    ap.add_argument("-U", dest="cut2", type=int, action="append", default=[],
                    help="as -u, for R2 (-u then applies to R1 only)")
    ap.add_argument("-m", "--minimum-length", default=None, metavar="LEN[:LEN2]")
    ap.add_argument("-M", "--maximum-length", default=None, metavar="LEN[:LEN2]")
    ap.add_argument("--interleaved", action="store_true",
                    help="read and/or write interleaved paired-end reads (one input file, or no -p)")
    ap.add_argument("--max-n", type=float, default=None)
    ap.add_argument("--max-ee", type=float, default=None)
    ap.add_argument("--max-average-error-rate", "--max-aer", dest="max_aer", type=float, default=None,
                    help="remove reads whose expected errors per base exceed this rate (0 < rate < 1)")
    ap.add_argument("-z", "--zero-cap", action="store_true",
                    help="change negative quality values to zero (characters below --quality-base)")
    ap.add_argument("--length", "-l", type=int, default=None)
    ap.add_argument("--poly-a", action="store_true")
    ap.add_argument("--trim-n", action="store_true")
    ap.add_argument("--discard-casava", action="store_true")
    ap.add_argument("--discard-trimmed", action="store_true")
    ap.add_argument("--discard-untrimmed", action="store_true")
    ap.add_argument("--action", default="trim", choices=["trim", "none", "mask", "lowercase", "retain", "crop"])
    ap.add_argument("--revcomp", "--rc", action="store_true",
                    help="also search the adapters on the reverse complement (pairs: with R1 and R2 swapped)")
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
    ap.add_argument("--info-file", metavar="FILE", help="write one row per adapter match (or per read without one)")
    ap.add_argument("--info-file-paired", dest="info_file2", metavar="FILE",
                    help="the info rows of the second mates (with --info-file)")
    ap.add_argument("-r", "--rest-file", metavar="FILE", help="write what follows (3') / precedes (5') the last match")
    ap.add_argument("--wildcard-file", metavar="FILE", help="write the read characters under the adapters' N positions")
    ap.add_argument("--rename", metavar="TEMPLATE", default=None,
                    help="rename reads with a template such as '{id} {adapter_name} {comment}'")
    ap.add_argument("-x", "--prefix", default="", help="add this prefix to read names; {name}: the adapter name")
    ap.add_argument("-y", "--suffix", default="", help="add this suffix to read names; {name}: the adapter name")
    ap.add_argument("--strip-suffix", action="append", default=[], help="remove this suffix from read names")
    ap.add_argument("--length-tag", metavar="TAG", default=None, help="replace TAG followed by a number with TAG and the "
                                                                       "length of the trimmed read")
    ap.add_argument("inputs", nargs="+")
    args = ap.parse_args()
    if args.rename and (args.prefix or args.suffix):
        ap.error("Option --rename cannot be combined with --prefix (-x) or --suffix (-y)")     # cli.py:982-985
    if args.info_file2 and len(args.inputs) == 1 and not args.interleaved:
        # --info-file-paired enables paired-end mode (cli.py:525-538, 560-566)
        ap.error("You used an option that enables paired-end mode (such as -p, -A, -G, -B, -U), but only provided one "
                 "input file. Please either provide two input files or use use --interleaved as appropriate.")
    for path in (args.info_file, args.info_file2, args.rest_file, args.wildcard_file):
        if path == "-":
            ap.error("row files (--info-file, --info-file-paired, --rest-file, --wildcard-file) cannot be written to "
                     "standard output")
    if args.interleaved and len(args.inputs) == 2 and args.paired_output:
        ap.error("--interleaved was given with two input files and two output files (-o and -p): use it for interleaved "
                 "input (one input file) or interleaved output (no -p)")
    if len(args.inputs) > 2:
        ap.error("at most two input files")
    paired = len(args.inputs) == 2 or args.interleaved
    min1, min2 = mate_lengths(ap, args.minimum_length, paired)
    max1, max2 = mate_lengths(ap, args.maximum_length, paired)
    check_filter_outputs(ap, args, paired, "{name}" in args.output, args.interleaved)
    if paired and args.revcomp and (args.info_file or args.info_file2):
        ap.error("--info-file cannot be combined with --revcomp on paired-end data: the info rows of swapped pairs are "
                 "not produced")
    input_format = detect_format(args.inputs[0])
    if input_format == "bam" or (len(args.inputs) == 2 and detect_format(args.inputs[1]) == "bam"):
        if paired:
            ap.error("BAM input is read single-end only: one BAM input file, without --interleaved")
    fasta_out = file_format(args.output, input_format, args.fasta) == "fasta"
    output_format = "fasta" if fasta_out and input_format in ("fastq", "bam") else None
    if input_format == "fasta" and args.max_ee is not None:
        print("WARNING: Ignoring option --max-ee because input does not provide quality values", file=sys.stderr)
        args.max_ee = None
    if input_format == "fasta" and args.max_aer is not None:
        print("WARNING: Ignoring option --max-aer because input does not provide quality values", file=sys.stderr)
        args.max_aer = None
    if input_format == "fasta" and args.zero_cap:
        ap.error("-z/--zero-cap needs quality values; the input is FASTA")
    if args.max_aer is not None and not 0.0 < args.max_aer < 1.0:
        ap.error(f"max_error_rate must be between 0.0 and 1.0, got {args.max_aer}.")
    host_reader = read_fasta_chunks if input_format == "fasta" else read_fastq_chunks
    # compressed bytes per submission of a device-inflated input: one thread inflates a member, so a submission must hold
    # many members; with --buffer-size 64 MiB, members of up to 1 MiB give 64 or more at once
    gz_buffer = args.buffer_size

    def single_input(t):
        """(file, chunks) of the single input for trimmer t."""
        if input_format == "bam":              # BGZF: every member inflated on the device, the records decoded there
            f = open(args.inputs[0], "rb")
            return f, read_gzip_device_chunks(f, t, gz_buffer)
        route = gzip_route(args.inputs[0])
        if route:
            f = open(args.inputs[0], "rb")
            return f, read_gzip_device_chunks(f, t, gz_buffer, split_members=route == "split")
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
                  trim_n=args.trim_n, discard_casava=args.discard_casava, action=args.action,
                  max_average_error_rate=args.max_aer, zero_cap=args.zero_cap)
    formats = dict(input_format=input_format, output_format=output_format, collect_statistics=args.json is not None)
    # --rename turns the " rc" suffix of --revcomp off (cli.py:964)
    revcomp1 = {} if paired else dict(revcomp=args.revcomp, rc_suffix=not args.rename)
    names = dict(rename=args.rename or None, prefix=args.prefix, suffix=args.suffix, strip_suffix=args.strip_suffix,
                 length_tag=args.length_tag)
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
    # row files: R1's (of the single reads), and R2's info rows with --info-file-paired (PairedInfoFileWriter)
    row_paths1 = {k: p for k, p in (("info", args.info_file), ("rest", args.rest_file), ("wildcard", args.wildcard_file))
                  if p}
    row_paths2 = {"info": args.info_file2} if paired and args.info_file and args.info_file2 else {}
    row_files = ({k: OutputFile(p) for k, p in row_paths1.items()}, {k: OutputFile(p) for k, p in row_paths2.items()})
    rows = dict(rows=tuple(row_paths1), gzip_rows=[k for k, p in row_paths1.items() if p.endswith(".gz")])

    def write_rows(t):
        """The rows of the chunk t returned last into the row files."""
        for kind, data in t.last_rows.items():
            r1, r2 = data if paired else (data, b"")
            row_files[0][kind].write(r1)
            if kind in row_files[1]:
                row_files[1][kind].write(r2)

    if paired:
        if not args.paired_output and not args.interleaved:
            ap.error("paired-end input needs -p (or --interleaved for an interleaved output)")
        if len(args.inputs) == 2 and detect_format(args.inputs[1]) != input_format:
            ap.error("both inputs must have the same format")
        options2 = dict(common, minimum_length=min2, maximum_length=max2, cut=args.cut2)   # -u is R1's, -U R2's
        # an output is interleaved when its paired path is missing (cli.py:650-661, 913-921)
        interleaved = [d for d in ["output"] + redirect
                       if not (args.paired_output if d == "output" else getattr(args, d + "_paired_output"))]
        t = PairedFastqTrimmer(ads1, ads2, common, options2, args.pair_filter, **formats, **split, revcomp=args.revcomp,
                               rc_suffix=not args.rename, **names, interleaved_outputs=interleaved, gzip_outputs=gzip1, gzip_outputs2=gzip2, **rows,
                               rows2=tuple(row_paths2),
                               gzip_rows2=[k for k, p in row_paths2.items() if p.endswith(".gz")])
        routes = [gzip_route(p) for p in args.inputs]
        if len(args.inputs) == 2 and all(routes):
            f1, f2 = open(args.inputs[0], "rb"), open(args.inputs[1], "rb")
            chunks = read_gzip_device_paired_chunks(f1, f2, t, gz_buffer, split_members=tuple(r == "split" for r in routes))
        elif len(args.inputs) == 2:
            f1, f2 = open_input(args.inputs[0]), open_input(args.inputs[1])
            chunks = paired_reader(f1, f2, args.buffer_size)
        elif routes[0]:
            f1 = f2 = open(args.inputs[0], "rb")
            chunks = read_gzip_device_interleaved_chunks(f1, t, gz_buffer, split_members=routes[0] == "split")
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
            write_rows(t)
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
        t = FastqTrimmer(ads1, **common, **formats, **revcomp1, **names, gzip_outputs=gzip1, **rows)
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
                write_rows(t)
        for fh in files.values():
            fh.close()
        stats = t.statistics
    elif redirect:
        t = FastqTrimmer(ads1, **common, **formats, **revcomp1, **names, **split, gzip_outputs=gzip1, **rows)
        f, chunks = single_input(t)
        with f:
            files = {d: OutputFile(getattr(args, d + "_output")) for d in redirect}
            files["output"] = OutputFile(args.output)
            for parts in t.process_chunks_split(chunks, copy=False):
                for name, data in parts.items():
                    files[name].write(data)
                write_rows(t)
            for fh in files.values():
                fh.close()
        stats = t.statistics
    else:
        t = FastqTrimmer(ads1, **common, **formats, **revcomp1, **names, gzip_outputs=gzip1, **rows)
        o = OutputFile(args.output)
        f, chunks = single_input(t)
        with f:
            for out in t.process_chunks(chunks, copy=False):
                o.write(out.tobytes() if hasattr(out, "tobytes") else out)
                write_rows(t)
        o.close()
        stats = t.statistics
    for fh in list(row_files[0].values()) + list(row_files[1].values()):
        fh.close()
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
