"""
The stored known answers with every output gzip-compressed on the device (-m gpu): fastq_kat, fasta_kat,
filter_outputs_kat and interleaved_kat, each output decompressed and compared with the stored answer byte for byte, and
each compressed output compared with the host build of the encoder (tests/hostsim).  Row outputs (--info-file and
friends) stay plain.
"""
import gzip

import pytest

pytestmark = pytest.mark.gpu

import cutadapt_b200.adapters as PA  # noqa: E402
import fasta_oracle as FO  # noqa: E402
import filter_outputs_oracle as RO  # noqa: E402
import interleaved_oracle as IO  # noqa: E402
from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer  # noqa: E402
from test_gpu_fasta import device_case  # noqa: E402
from test_gpu_fastq import trimmer_for, trimmer_kwargs  # noqa: E402
from test_gzip_host import hs_gzip  # noqa: E402
from util import fastq_case_adapters, fastq_cases, fastq_demux_case, fastq_paired_cases  # noqa: E402

ALL = ("output", "too_short", "too_long", "untrimmed")


def unzip(z: bytes) -> bytes:
    """The plain bytes of a device gzip output, which must be what the host build writes for them."""
    plain = gzip.decompress(z) if z else b""
    assert z == hs_gzip(plain)
    return plain


def test_fastq_kat_all_outputs_gzipped():
    for c in fastq_cases():
        t = trimmer_for(c["options"], gzip_outputs=ALL)
        got = t.process_chunk(c["input_bytes"])
        assert unzip(got) == c["expected_bytes"], c["name"]
        assert t.statistics["out_bytes_plain"] == len(c["expected_bytes"])
    for c in fastq_paired_cases():
        o = c["options"]
        t = PairedFastqTrimmer(fastq_case_adapters(o, "adapters1"), fastq_case_adapters(o, "adapters2"),
                               trimmer_kwargs(o["options1"]), trimmer_kwargs(o["options2"]), o.get("pair_filter", "any"),
                               gzip_outputs=ALL)
        got = t.process_chunk(*c["input_bytes"])
        assert [unzip(g) for g in got] == c["expected_bytes"], c["name"]
    c = fastq_demux_case()
    ads = [PA.BackAdapter(seq, max_errors=0.1, min_overlap=3, name=name) for name, seq in c["adapters"]]
    got = FastqTrimmer(ads, gzip_outputs=ALL).process_chunk_demux(c["input_bytes"])
    assert {k: unzip(v) for k, v in got.items()} == c["expected"]


def test_fasta_kat_all_outputs_gzipped(monkeypatch):
    # device_case builds its trimmers itself: give them every output gzipped
    for cls in (FastqTrimmer, PairedFastqTrimmer):
        init = cls.__init__

        def gz_init(self, *a, _init=init, **kw):
            _init(self, *a, **kw, gzip_outputs=ALL)

        monkeypatch.setattr(cls, "__init__", gz_init)
    for c in FO.fasta_kat()["cases"]:
        got, rows, _ = device_case(c)
        if c["kind"] == "demux":
            assert {k: unzip(v) for k, v in got.items()} == {k: FO.kat_file(v) for k, v in c["expected"].items()}, \
                c["name"]
            continue
        for g, e in zip(got, c["expected"]):
            if e is not None:
                assert unzip(g) == FO.kat_file(e), (c["name"], c["command"])
        if c["kind"] == "rows":
            assert rows == FO.kat_file(c["rows"]), c["name"]


def test_filter_outputs_kat_all_outputs_gzipped():
    for c in RO.filter_outputs_kat()["cases"]:
        o = c["options"]
        data = [RO.kat_file(k) for k in c["inputs"]]
        fmt = RO.input_format_of(data[0])
        kw = RO.kat_trimmer_kwargs(o)
        if c["kind"] == "paired":
            t = PairedFastqTrimmer(FO.kat_adapters(o, "specs1"), FO.kat_adapters(o, "specs2"), kw, kw,
                                   o.get("pair_filter", "any"), input_format=fmt, redirect=o.get("redirect", ()),
                                   gzip_outputs=ALL)
            got = t.process_chunk_split(*data)
            for name, exp in c["expected"].items():
                assert (unzip(got[name][0]), unzip(got[name][1])) == (RO.kat_file(exp[0]), RO.kat_file(exp[1])), \
                    (c["name"], name)
            continue
        t = FastqTrimmer(FO.kat_adapters(o), input_format=fmt, redirect=o.get("redirect", ()), **kw, gzip_outputs=ALL)
        got = t.process_chunk_split(data[0])
        for name, exp in c["expected"].items():
            assert unzip(got[name]) == RO.kat_file(exp), (c["name"], name)
        for k, v in c["counters"].items():
            assert t.statistics[k] == v, (c["name"], k)


def test_interleaved_kat_all_outputs_gzipped():
    for c in IO.interleaved_kat()["cases"]:
        o = c["options"]
        data = [IO.kat_file(k) for k in c["inputs"]]
        fmt = "fasta" if data[0][:1] in (b">", b"#") else "fastq"
        kw1, kw2 = IO.kat_trimmer_kwargs(o)
        t = PairedFastqTrimmer(FO.kat_adapters(o, "specs1"), FO.kat_adapters(o, "specs2"), kw1, kw2, input_format=fmt,
                               redirect=o.get("redirect", ()), interleaved_outputs=IO.kat_interleaved_outputs(c),
                               gzip_outputs=ALL)
        got = t.process_chunk_split(data[0], data[1] if len(data) == 2 else None)
        for name, files in c["expected"].items():
            want = tuple(IO.kat_file(k) for k in files) + ((b"",) if len(files) == 1 else ())
            assert tuple(unzip(g) for g in got[name]) == want, (c["name"], name)
