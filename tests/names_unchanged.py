"""
Collects without name options, to show that the name stage leaves them as they were: seeded chunks through every
kind of collect, the sha256 of every output and the number of launches each collect made (cg_ctx_launch_count).
tests/golden/names_unchanged.json holds what the commit before the name stage gave:

    PYTHONPATH=<checkout of that commit> python tests/names_unchanged.py --write tests/golden/names_unchanged.json

and tests/test_gpu_names.py compares this tree's answers with it.
"""
import gzip
import hashlib
import json
import random
import sys


def _fastq(rng, n, adapters, mate, fasta=False):
    recs = []
    for i in range(n):
        seq = "".join(rng.choice("ACGT") for _ in range(rng.randint(0, 60)))
        for _ in range(rng.choice([0, 1, 1])):
            a = rng.choice(adapters)
            piece = a if rng.random() < 0.6 else a[: rng.randint(3, len(a))]
            at = rng.randint(0, len(seq))
            seq = seq[:at] + piece + seq[at:]
        name = f"r{i}{mate}" + rng.choice(["", " length=99 x", " a  b "])
        if fasta:
            recs.append(f">{name}\n{seq}\n")
        else:
            recs.append(f"@{name}\n{seq}\n+\n{''.join(chr(33 + rng.choice([2, 20, 40])) for _ in seq)}\n")
    return "".join(recs).encode()


def answers():
    from cutadapt_b200 import _lib
    import cutadapt_b200.adapters as PA
    from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer

    ads1 = lambda: [PA.BackAdapter("AGATCGGAAGAGC", name="ilmn"), PA.FrontAdapter("ACGGTCAT", name="front")]
    ads2 = lambda: [PA.BackAdapter("CAGTGGAGTA", name="r2a"), PA.FrontAdapter("TTGACCAG", name="r2front")]
    rng = random.Random(31)
    a = _fastq(rng, 600, [x.sequence for x in ads1()], "/1")
    b = _fastq(rng, 600, [x.sequence for x in ads2()], "/2")
    fa = _fastq(rng, 300, [x.sequence for x in ads1()], "/1", fasta=True)
    il = b"".join(b"".join(a.splitlines(True)[i:i + 4] + b.splitlines(True)[i:i + 4])
                  for i in range(0, len(a.splitlines()), 4))
    opts = dict(minimum_length=5, cut=(1, -1), quality_cutoff=(0, 10))
    out = {}

    def digest(x):
        if isinstance(x, dict):
            return {str(k): digest(v) for k, v in sorted(x.items(), key=lambda kv: str(kv[0]))}
        if isinstance(x, (tuple, list)):
            return [digest(v) for v in x]
        return hashlib.sha256(bytes(x)).hexdigest()

    def run(name, t, call):
        n0 = _lib.lib().cg_ctx_launch_count(t.ctx.handle)
        res = call(t)
        out[name] = {"outputs": digest(res), "rows": digest(getattr(t, "last_rows", {})),
                     "launches": int(_lib.lib().cg_ctx_launch_count(t.ctx.handle) - n0)}

    single = lambda **kw: FastqTrimmer(ads1(), **opts, rows=("info", "rest"), **kw)
    run("single", single(), lambda t: t.process_chunk(a))
    run("single_revcomp", single(revcomp=True), lambda t: t.process_chunk(a))
    run("single_split", single(redirect=("too_short", "untrimmed"), redirect_formats={"untrimmed": "fasta"}),
        lambda t: t.process_chunk_split(a))
    run("single_demux", single(), lambda t: t.process_chunk_demux(a))
    run("single_gzip", single(gzip_outputs=("output",)), lambda t: gzip.decompress(t.process_chunk(a)))
    run("fasta", FastqTrimmer(ads1(), minimum_length=5, input_format="fasta"), lambda t: t.process_chunk(fa))
    run("fastq_to_fasta", FastqTrimmer(ads1(), **opts, output_format="fasta"), lambda t: t.process_chunk(a))
    pair = lambda **kw: PairedFastqTrimmer(ads1(), ads2(), opts, opts, rows=("info",), rows2=("info",), **kw)
    run("paired", pair(), lambda t: t.process_chunk(a, b))
    run("paired_both", pair(pair_filter="both"), lambda t: t.process_chunk(a, b))
    run("paired_interleaved_input", pair(), lambda t: t.process_chunk(il))
    run("paired_interleaved_outputs", pair(redirect=("too_short",), interleaved_outputs=("output", "too_short")),
        lambda t: t.process_chunk_split(a, b))
    run("paired_demux", pair(), lambda t: t.process_chunk_demux(a, b, combinatorial=True))
    run("paired_revcomp", PairedFastqTrimmer(ads1(), ads2(), opts, opts, revcomp=True), lambda t: t.process_chunk(a, b))
    run("pair_adapters", PairedFastqTrimmer(ads1(), ads2(), dict(minimum_length=5), dict(minimum_length=5),
                                            pair_adapters=True), lambda t: t.process_chunk(a, b))
    return out


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--write":
        with open(sys.argv[2], "w") as f:
            json.dump(answers(), f, indent=1, sort_keys=True)
            f.write("\n")
    else:
        print(json.dumps(answers(), indent=1, sort_keys=True))
