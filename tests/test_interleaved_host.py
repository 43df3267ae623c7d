"""
Interleaved paired-end data (--interleaved) without a GPU: the test-side interleave oracle (tests/interleaved_oracle.py)
against the reference's known answers (tests/golden/interleaved_kat.json.gz), the host build of the mate-name check
(fq_mates_match via tests/hostsim) against a restatement of the rule, the interleaved chunk readers, and the command-line
errors and LEN:LEN2 lengths of tools/trim_fastq.py.
"""
import ctypes as C
import io
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

import fasta_oracle as FO
import interleaved_oracle as IO
from util import fastq_case_kwargs, spec_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def descs_of(adapters):
    import cutadapt_b200.adapters as PA

    if not adapters:
        return None, None
    spec = spec_of(PA.MultipleAdapters(adapters))
    return spec.adapters, spec.groups


def oracle_case(c):
    """({output: (bytes1, bytes2)}, counters1, counters2) of a stored case through the interleave oracle."""
    o = c["options"]
    data = [IO.kat_file(k) for k in c["inputs"]]
    fmt = "fasta" if data[0][:1] in (b">", b"#") else "fastq"
    kw1, kw2 = (fastq_case_kwargs(x) for x in IO.kat_trimmer_kwargs(o))
    return IO.interleaved_trim(data[0], data[1] if len(data) == 2 else None, *descs_of(FO.kat_adapters(o, "specs1")),
                               *descs_of(FO.kat_adapters(o, "specs2")), kw1, kw2, "any", tuple(o.get("redirect", ())),
                               IO.kat_interleaved_outputs(c), input_format=fmt)


def test_the_golden_holds_the_reference_cases():
    kat = IO.interleaved_kat()
    names = [c["name"] for c in kat["cases"]]
    assert len(names) == 100 and sum(n.startswith("separate_minmaxlength[") for n in names) == 96
    assert {e["name"] for e in kat["errors"]} == {"interleaved_neither_nor", "separate_minlength_single"}


def test_the_interleave_oracle_reproduces_every_stored_case():
    for c in IO.interleaved_kat()["cases"]:
        outs, c1, c2 = oracle_case(c)
        for name, files in c["expected"].items():
            want = tuple(IO.kat_file(k) for k in files) + ((b"",) if len(files) == 1 else ())
            assert outs[name] == want, (c["name"], name)
        assert c1["n_written"] == c2["n_written"]
        if c["name"] == "interleaved_untrimmed_output":         # every pair is untrimmed
            pairs = len(IO.records(IO.kat_file(c["inputs"][0]), "fastq")) // 2
            assert outs["output"] == (b"", b"") and c1["discarded"] == c2["discarded"] == pairs


# ---- the mate-name check ---------------------------------------------------------------------------------------------

def hostsim_mates(pairs):
    from util import hostsim_lib

    lib = hostsim_lib()
    lib.hs_mates_match.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    names = [h for p in pairs for h in p]
    blob = np.frombuffer(b"".join(names) + b"\0", dtype=np.uint8)
    off = np.zeros(len(names) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(h) for h in names])
    out = np.zeros(len(pairs), dtype=np.int32)
    lib.hs_mates_match(len(pairs), blob.ctypes.data, off.ctypes.data, out.ctypes.data)
    return out.astype(bool).tolist()


def test_mate_names_exhaustively_on_short_headers():
    alphabet = [b"a", b"1", b"2", b"3", b" ", b"\t", b"/"]
    headers = [b"".join(t) for k in range(4) for t in itertools.product(alphabet, repeat=k)]
    pairs = list(itertools.product(headers, headers))
    got = hostsim_mates(pairs)
    want = [IO.mates_match(a, b) for a, b in pairs]
    assert got == want
    assert 0 < sum(want) < len(want)


def test_mate_names_on_the_documented_examples_and_the_stored_data():
    pairs = [(b"my_read/1 a comment", b"my_read/2 another comment"), (b"my_read/1;1", b"my_read/2;1"),
             (b"read1/1 some text", b"read1/2 other text"), (b"r1", b"r"), (b"r", b"r"), (b"a\tx", b"a y"),
             (b"", b""), (b"1", b"2"), (b"r1/1", b"r2/1")]
    want = [True, False, True, False, True, True, True, True, False]
    assert [IO.mates_match(a, b) for a, b in pairs] == want
    assert hostsim_mates(pairs) == want
    recs = IO.records(IO.kat_file("data/interleaved.fastq"), "fastq")
    names = [r.split(b"\n", 1)[0][1:] for r in recs]
    stored = list(zip(names[0::2], names[1::2]))
    assert hostsim_mates(stored) == [True] * len(stored)
    shifted = list(zip(names[1::2], names[2::2]))
    assert hostsim_mates(shifted) == [IO.mates_match(a, b) for a, b in shifted] == [False] * len(shifted)


# ---- the chunk readers -----------------------------------------------------------------------------------------------

def _fastq(n, crlf=False):
    nl = b"\r\n" if crlf else b"\n"
    return b"".join(b"@r%d/%d x%s%s%s+%s%s%s" % (i // 2, i % 2 + 1, nl, b"ACGT" * (i % 3), nl, nl, b"I" * 4 * (i % 3), nl)
                    for i in range(n))


def _fasta(n, crlf=False):
    nl = b"\r\n" if crlf else b"\n"
    return b"#c" + nl + b"".join(b">r%d/%d%s%s" % (i // 2, i % 2 + 1, nl, (b"ACG" + nl) * (i % 4)) for i in range(n))


@pytest.mark.parametrize("fmt", ["fastq", "fasta"])
@pytest.mark.parametrize("crlf", [False, True])
def test_interleaved_readers_keep_pairs_together(fmt, crlf):
    from cutadapt_b200.pipeline import read_interleaved_fasta_chunks, read_interleaved_fastq_chunks

    reader = read_interleaved_fastq_chunks if fmt == "fastq" else read_interleaved_fasta_chunks
    for n in (0, 1, 2, 6, 7):
        data = (_fastq if fmt == "fastq" else _fasta)(n, crlf)
        for bs in range(1, len(data) + 2):
            chunks = list(reader(io.BytesIO(data), bs))
            assert b"".join(chunks) == data, (n, bs)
            for k, ch in enumerate(chunks):
                recs = IO.records(ch.replace(b"\r\n", b"\n"), fmt)
                if fmt == "fasta" and k == 0:
                    recs = [r for r in recs if not r.startswith(b"#")]
                if k < len(chunks) - 1 or n % 2 == 0:
                    assert len(recs) % 2 == 0 and (recs or n == 0), (n, bs, k)
            if n % 2:
                last = IO.records(chunks[-1].replace(b"\r\n", b"\n"), fmt)
                assert len([r for r in last if not r.startswith(b"#")]) % 2 == 1


def test_interleaved_readers_leave_an_unterminated_last_record_in_the_last_chunk():
    from cutadapt_b200.pipeline import read_interleaved_fastq_chunks

    data = _fastq(4)[:-1]
    for bs in range(1, len(data) + 2):
        chunks = list(read_interleaved_fastq_chunks(io.BytesIO(data), bs))
        assert b"".join(chunks) == data and chunks[-1].count(b"\n") == 7


# ---- tools/trim_fastq.py ---------------------------------------------------------------------------------------------

def _tool(argv, tmp_path):
    files = IO.interleaved_kat()["files"]
    args = []
    for a in argv:
        if a in files:
            p = tmp_path / a.replace("/", "_")
            p.write_bytes(files[a].encode("latin-1"))
            a = str(p)
        args.append(a.format(out1=tmp_path / "o1.fastq", out2=tmp_path / "o2.fastq"))
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py")] + args, capture_output=True,
                          text=True, cwd=str(tmp_path))


@pytest.mark.parametrize("name", ["interleaved_neither_nor", "separate_minlength_single"])
def test_tool_refuses_the_stored_command_lines(name, tmp_path):
    case = next(e for e in IO.interleaved_kat()["errors"] if e["name"] == name)
    r = _tool(case["argv"], tmp_path)
    assert r.returncode == 2, r.stderr
    want = "--interleaved" if name == "interleaved_neither_nor" else "single-end data"
    assert want in r.stderr


def test_tool_parses_lengths():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import trim_fastq

    assert trim_fastq.parse_lengths("25") == (25,)
    assert trim_fastq.parse_lengths("17:25") == (17, 25)
    assert trim_fastq.parse_lengths("25:") == (25, None)
    assert trim_fastq.parse_lengths(":25") == (None, 25)
    for bad in (":", "1:2:3", "x", "5:y"):
        with pytest.raises(ValueError):
            trim_fastq.parse_lengths(bad)
