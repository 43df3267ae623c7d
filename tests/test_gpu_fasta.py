"""
FASTA on the device (cg_fastq_params.format 1 / 2; -m gpu): the reference's FASTA known answers byte for byte through
every entry point they need, randomized FASTA chunks against the FASTA oracle (tests/fasta_oracle.py), FASTQ -> FASTA,
format errors, several chunks in flight and one large chunk.
"""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import fasta_oracle as FO  # noqa: E402
from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer  # noqa: E402
from test_fasta_host import N_KAT_CASES, oracle_case  # noqa: E402
from util import random_reads  # noqa: E402

COUNTERS = ("n_records", "n_written", "bp_in", "bp_out", "with_adapters", "too_short", "too_long", "too_many_n",
            "discarded", "reverse_complemented")


def device_case(c):
    """A fasta_kat case on the device: (outputs in the shape of "expected", rows or None, statistics)."""
    o = c["options"]
    fmt = FO.kat_formats(o)
    data = [FO.kat_file(k) for k in c["inputs"]]
    if c["kind"] == "paired":
        shared = FO.kat_kwargs(o)
        t = PairedFastqTrimmer(FO.kat_adapters(o, "specs1"), FO.kat_adapters(o, "specs2"),
                               {**shared, **o.get("options1", {})}, {**shared, **o.get("options2", {})}, **fmt)
        return list(t.process_chunk(data[0], data[1])), None, t.statistics[0]
    t = FastqTrimmer(FO.kat_adapters(o), **FO.kat_kwargs(o), **fmt)
    if c["kind"] == "demux":
        return t.process_chunk_demux(data[0]), None, t.statistics
    if c["kind"] == "rows":
        run = {0: t.process_chunk_info, 1: t.process_chunk_rest, 2: t.process_chunk_wildcards}[c["row_kind"]]
        out, rows = run(data[0])
        return [out], rows, t.statistics
    return [t.process_chunk(data[0])], None, t.statistics


def test_reference_fasta_goldens_on_the_device():
    """Every case of fasta_kat.json.gz byte for byte through collect, demux, rows or paired; counters = the oracle's."""
    cases = FO.fasta_kat()["cases"]
    assert len(cases) == N_KAT_CASES
    for c in cases:
        got, rows, stats = device_case(c)
        want, want_rows = oracle_case(c)
        if c["kind"] == "demux":
            assert got == {k: FO.kat_file(v) for k, v in c["expected"].items()} == want, c["name"]
            continue
        for g, e in zip(got, c["expected"]):
            if e is not None:
                assert g == FO.kat_file(e), (c["name"], c["command"])
        assert got == want, c["name"]
        if c["kind"] == "rows":
            assert rows == FO.kat_file(c["rows"]) == want_rows, (c["name"], c["command"])
        if c["kind"] == "trim" and c["inputs"][0].endswith(("fasta", "fa", "gz")):
            ads = FO.kat_adapters(c["options"])
            _, cnt = FO.fasta_trim(FO.kat_file(c["inputs"][0]), *FO.descriptors(ads), **FO.kat_formats(c["options"]),
                                   **FO.kat_kwargs(c["options"]))
            assert {k: stats[k] for k in COUNTERS if k in cnt} == {k: cnt[k] for k in COUNTERS if k in cnt}, c["name"]


ADAPTERS = ["AGATCGGAAGAGC", "TTGACNNACG", "CACGTCTGAA"]


def messy_fasta(seed, n=600, wrap=None):
    """Random reads with adapters as FASTA: wrapped at random widths, "\\r\\n" half the time, leading comments, some
    records without sequence."""
    rng = random.Random(seed)
    reads = random_reads(rng, ADAPTERS, n, alpha="ACGTN", max_len=120)
    nl = "\r\n" if seed % 2 else "\n"
    text = [f"# run {seed}{nl}"]
    for i, s in enumerate(reads):
        if i % 37 == 5:
            s = ""
        w = wrap or rng.randint(5, 80)
        text.append(f">r{i} d{seed}{nl}" + "".join(s[k:k + w] + nl for k in range(0, len(s), w)))
    return "".join(text).encode()


def _adapters(kind="mixed"):
    import cutadapt_b200.adapters as PA

    if kind == "demux":
        return [PA.BackAdapter(ADAPTERS[0], name="one"), PA.FrontAdapter(ADAPTERS[1], max_errors=0.2, name="two")]
    return [PA.BackAdapter(ADAPTERS[0], max_errors=0.1, name="a"), PA.FrontAdapter(ADAPTERS[1], max_errors=0.2, name="b"),
            PA.AnywhereAdapter(ADAPTERS[2], name="c")]


VARIANTS = {
    "plain": dict(),
    "filters": dict(minimum_length=20, maximum_length=100, max_n=0.1, discard_untrimmed=True),
    "cut_and_modifiers": dict(cut=[3, -2], poly_a=True, length=60, trim_n=True, times=2),
    "mask": dict(action="mask"),
    "lowercase": dict(action="lowercase", discard_trimmed=True),
    "retain": dict(action="retain"),
    "crop": dict(action="crop"),
    "revcomp": dict(revcomp=True),
    "revcomp_no_suffix": dict(revcomp=True, rc_suffix=False, minimum_length=5),
}


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_random_fasta_chunks_against_the_oracle(variant):
    kw = VARIANTS[variant]
    ads = _adapters()
    data = messy_fasta(sorted(VARIANTS).index(variant))
    t = FastqTrimmer(ads, input_format="fasta", **kw)
    got = t.process_chunk(data)
    want, cnt = FO.fasta_trim(data, *FO.descriptors(ads), **kw)
    assert got == want
    assert {k: t.statistics[k] for k in COUNTERS} == {k: cnt[k] for k in COUNTERS}


def test_random_fasta_demultiplexing_and_rows():
    ads = _adapters("demux")
    data = messy_fasta(21)
    t = FastqTrimmer(ads, input_format="fasta", minimum_length=10)
    assert t.process_chunk_demux(data) == FO.fasta_demux(data, *FO.descriptors(ads), FO.info_names(ads),
                                                         minimum_length=10)
    for kw in (dict(), dict(revcomp=True), dict(times=2, action="lowercase")):
        ads = _adapters()
        t = FastqTrimmer(ads, input_format="fasta", **kw)
        out, rows = t.process_chunk_info(data)
        want_rows = []
        want, _ = FO.fasta_trim(data, *FO.descriptors(ads), info_names=FO.info_names(ads), info_rows=want_rows, **kw)
        assert out == want, kw
        assert rows == "".join(r + "\n" for r in want_rows).encode(), kw
    ads = _adapters()
    out, rows = FastqTrimmer(ads, input_format="fasta").process_chunk_rest(data)
    want_rows = []
    assert out == FO.fasta_trim(data, *FO.descriptors(ads), rest_rows=want_rows)[0]
    assert rows == "".join(r + "\n" for r in want_rows).encode()


@pytest.mark.parametrize("mode", ["any", "both", "first"])
def test_paired_random_fasta_against_the_oracle(mode):
    ads1, ads2 = _adapters()[:2], _adapters()[2:]
    d1, d2 = messy_fasta(31, 500), messy_fasta(32, 500, wrap=60)
    o1 = dict(minimum_length=15, cut=[2])
    o2 = dict(minimum_length=15, poly_a=True)
    t = PairedFastqTrimmer(ads1, ads2, o1, o2, pair_filter=mode, input_format="fasta")
    got = t.process_chunk(d1, d2)
    w1, w2, c1, c2 = FO.fasta_trim_paired(d1, d2, *FO.descriptors(ads1), *FO.descriptors(ads2), o1, o2, mode)
    assert got == (w1, w2)
    assert t.statistics[0]["n_written"] == c1["n_written"] and t.statistics[1]["bp_out"] == c2["bp_out"]
    # --pair-adapters and paired demultiplexing take FASTA too
    pa = PairedFastqTrimmer(_adapters()[:1], _adapters()[1:2], pair_adapters=True, input_format="fasta")
    a1, a2 = pa.process_chunk(d1, d2)
    assert a1.startswith(b">r0 d31\n") and a1.count(b"\n>") + 1 == 500 == a2.count(b"\n>") + 1
    dm = PairedFastqTrimmer(_adapters("demux"), None, input_format="fasta").process_chunk_demux(d1, d2)
    assert sum(v[0].count(b">") for v in dm.values()) == 500


def test_fastq_to_fasta_equals_fasta_to_fasta():
    """The same reads as FASTQ (format 2) and as FASTA (format 1), without quality options: identical output."""
    rng = random.Random(5)
    reads = random_reads(rng, ADAPTERS, 3000, alpha="ACGTN", max_len=150)
    fastq = "".join(f"@q{i} x\n{s}\n+\n{'I' * len(s)}\n" for i, s in enumerate(reads)).encode()
    fasta = "".join(f">q{i} x\n{s}\n" for i, s in enumerate(reads)).encode()
    for kw in (dict(), dict(minimum_length=30, action="mask"), dict(revcomp=True, cut=[4])):
        a = FastqTrimmer(_adapters(), output_format="fasta", **kw).process_chunk(fastq)
        b = FastqTrimmer(_adapters(), input_format="fasta", **kw).process_chunk(fasta)
        assert a == b, kw
        assert a == FO.fasta_trim(fastq, *FO.descriptors(_adapters()), input_format="fastq", output_format="fasta",
                                  **kw)[0]
    # quality trimming on FASTQ input with FASTA output is fine
    q = FastqTrimmer(_adapters(), quality_cutoff=(0, 20), output_format="fasta").process_chunk(fastq)
    assert q.count(b">") == 3000


def test_format_errors_and_quality_options_on_fasta():
    from cutadapt_b200 import _lib

    t = FastqTrimmer(_adapters(), input_format="fasta")
    for bad, msg in ((b"ACGT\n>a\nAC\n", "line 1: expected '>'"), (b"#c\n\n>a\n", "line 2: expected '>'"),
                     (b">a\nAC\n#x\nGT\n", "line 3: a '#' comment line"), (b">a\r\nAC\r\n>b\r\n#\r\n", "line 4: a '#'")):
        with pytest.raises(ValueError, match=msg):
            t.process_chunk(bad)
    ok = b">a\nACGTACGTTTGACGGACGA\n>b\n"
    assert t.process_chunk(ok) == FO.fasta_trim(ok, *FO.descriptors(_adapters()))[0]     # the context stays usable
    for kw in (dict(quality_cutoff=(0, 20)), dict(nextseq_cutoff=20), dict(max_expected_errors=1.0)):
        with pytest.raises(Exception, match="FASTA input has no qualities"):
            FastqTrimmer(None, input_format="fasta", **kw).process_chunk(b">a\nACGT\n")
    # both mates must have the same format
    p = PairedFastqTrimmer(None, None, input_format="fasta")
    p.params2.format = _lib.CG_FORMAT_FASTQ
    with pytest.raises(Exception, match="same format"):
        p.process_chunk(b">a\nAC\n", b"@a\nAC\n+\nII\n")
    with pytest.raises(ValueError):
        FastqTrimmer(None, input_format="fasta", output_format="fastq")


def test_records_without_sequence_make_the_output_larger():
    """">a\\n>b\\n..." is written as ">a\\n\\n>b\\n\\n...": the output of a FASTA chunk can exceed the input."""
    data = b"".join(b">%d\n" % i for i in range(20000)) + b">last"
    t = FastqTrimmer(None, input_format="fasta")
    got = t.process_chunk(data)
    assert got == b"".join(b">%d\n\n" % i for i in range(20000)) + b">last\n\n"
    assert len(got) > len(data)
    tiny = b">\n" * 5000
    assert FastqTrimmer(None, input_format="fasta").process_chunk(tiny) == b">\n\n" * 5000


def test_many_fasta_chunks_in_flight():
    chunks = [messy_fasta(40 + i, n) for i, n in enumerate((1, 700, 3, 2500, 50))] + [b""]
    t = FastqTrimmer(_adapters(), input_format="fasta", minimum_length=10)
    got = list(t.process_chunks(chunks))
    assert got == [FO.fasta_trim(c, *FO.descriptors(_adapters()), minimum_length=10)[0] for c in chunks]


def test_large_fasta_chunk():
    """2 M records (60-column wrapped, 150 bp): size-independent properties and the oracle on a strided sample."""
    n, L = 2_000_000, 150
    rng = np.random.default_rng(9)
    seq = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), (n, L))
    ad = np.frombuffer(b"AGATCGGAAGAGC", dtype=np.uint8)
    seq[::2, 100:100 + ad.size] = ad
    lines = [seq[:, 0:60], seq[:, 60:120], seq[:, 120:150]]
    names = np.char.add(b">r", np.arange(n).astype("S8"))
    recs = [b"%s\n%s\n%s\n%s\n" % (names[i], lines[0][i].tobytes(), lines[1][i].tobytes(), lines[2][i].tobytes())
            for i in range(n)]
    data = b"".join(recs)
    ads = _adapters()[:1]
    t = FastqTrimmer(ads, input_format="fasta", minimum_length=20)
    got = t.process_chunk(data)
    st = t.statistics
    assert st["n_records"] == n and st["bp_in"] == n * L
    assert st["n_written"] + st["too_short"] == n
    out = got.split(b"\n")
    assert out[-1] == b"" and len(out) - 1 == 2 * st["n_written"]
    assert sum(len(x) for x in out[1::2]) == st["bp_out"]
    idx = list(range(0, n, 10007))
    sample = b"".join(recs[i] for i in idx)
    want = FO.fasta_trim(sample, *FO.descriptors(ads), minimum_length=20)[0].split(b"\n")
    by_name = {out[k]: out[k + 1] for k in range(0, len(out) - 1, 2)}
    for k in range(0, len(want) - 1, 2):
        assert by_name[want[k]] == want[k + 1]
