"""
FASTA input / output without a GPU: the FASTA oracle (tests/fasta_oracle.py) against the reference's FASTA known answers
(tests/golden/fasta_kat.json.gz), the FASTA chunk readers of cutadapt_b200.pipeline, and the host build of the device's
line / record logic (fa_line_core, fa_line_error, fa_record_core via tests/hostsim) against the oracle's reader.
"""
import ctypes as C
import io
import random

import numpy as np
import pytest

import fasta_oracle as FO

N_KAT_CASES = 47


def oracle_case(c):
    """What the FASTA oracle gives for a fasta_kat case, in the shape of the case's "expected" (and rows)."""
    o = c["options"]
    fmt = FO.kat_formats(o)
    data = [FO.kat_file(k) for k in c["inputs"]]
    if c["kind"] == "paired":
        sets = [FO.descriptors(FO.kat_adapters(o, key)) for key in ("specs1", "specs2")]
        shared = {k: v for k, v in FO.kat_kwargs(o).items()}
        o1, o2, _, _ = FO.fasta_trim_paired(data[0], data[1], *sets[0], *sets[1], {**shared, **o.get("options1", {})},
                                            {**shared, **o.get("options2", {})}, **fmt)
        return [o1, o2], None
    ads = FO.kat_adapters(o)
    descs, groups = FO.descriptors(ads)
    if c["kind"] == "demux":
        return FO.fasta_demux(data[0], descs, groups, FO.info_names(ads), **fmt, **FO.kat_kwargs(o)), None
    kw = FO.kat_kwargs(o)
    rows = None
    if c["kind"] == "rows":
        rows = []
        kind = c["row_kind"]
        if kind == 0:
            kw.update(info_names=FO.info_names(ads), info_rows=rows)
        elif kind == 1:
            kw.update(rest_rows=rows)
        else:
            kw.update(wildcard_rows=rows, adapter_sequences=[a.sequence for a in ads])
    out, _ = FO.fasta_trim(data[0], descs, groups, **fmt, **kw)
    return [out], (None if rows is None else "".join(r + "\n" for r in rows).encode("latin-1"))


def test_fasta_oracle_reproduces_the_reference_fasta_goldens():
    """Every case of fasta_kat.json.gz, byte for byte: trimmed output (or every demultiplexed output) and the rows of
    --rest-file / --wildcard-file / --info-file."""
    cases = FO.fasta_kat()["cases"]
    assert len(cases) == N_KAT_CASES
    assert {c["kind"] for c in cases} == {"trim", "demux", "rows", "paired"}
    for c in cases:
        got, rows = oracle_case(c)
        if c["kind"] == "demux":
            assert got == {k: FO.kat_file(v) for k, v in c["expected"].items()}, c["name"]
            continue
        for g, e in zip(got, c["expected"]):
            if e is not None:
                assert g == FO.kat_file(e), (c["name"], c["command"])
        if c["kind"] == "rows":
            assert rows == FO.kat_file(c["rows"]), (c["name"], c["command"])


def test_fasta_reader_rules():
    assert FO.parse_fasta(b"") == []
    assert FO.parse_fasta(b"# a\n#b\r\n") == []
    assert FO.parse_fasta(b"#c\n>a x\r\nAC\r\nGT\n>b\n>c\nT") == [("a x", "ACGT"), ("b", ""), ("c", "T")]
    for bad, line in ((b"ACGT\n>a\n", 1), (b"\n>a\nA\n", 1), (b">a\nAC\n#x\n", 3), (b"#x\n\n>a\n", 2)):
        with pytest.raises(FO.FastaFormatError, match=f"line {line}:"):
            FO.parse_fasta(bad)


def random_fasta(rng, n_records, crlf=False, comments=False, wrap=None, final_newline=True):
    """(FASTA bytes, [(name, sequence)]): sequences of random lengths (some empty), wrapped at random widths."""
    recs, text = [], []
    nl = "\r\n" if crlf else "\n"
    if comments:
        text += [f"# comment {i}{nl}" for i in range(rng.randint(1, 3))]
    for i in range(n_records):
        seq = "".join(rng.choice("ACGTN") for _ in range(rng.choice([0, rng.randint(1, 30), rng.randint(30, 200)])))
        name = f"r{i} extra{rng.randint(0, 9)}" if rng.random() < 0.5 else f"r{i}"
        recs.append((name, seq))
        w = wrap or rng.randint(1, 80)
        text.append(f">{name}{nl}" + "".join(seq[k:k + w] + nl for k in range(0, len(seq), w)))
    data = "".join(text).encode()
    if not final_newline and data.endswith(nl.encode()):
        data = data[:-len(nl)]
    return data, recs


def test_fasta_chunk_readers_split_at_records():
    """read_fasta_chunks at every buffer size: the chunks join back to the input, each (but a first one with comments)
    starts at a header and holds complete records; read_paired_fasta_chunks gives equal record counts per mate."""
    from cutadapt_b200.pipeline import read_fasta_chunks, read_paired_fasta_chunks

    rng = random.Random(3)
    data, recs = random_fasta(rng, 40, comments=True)
    data2, recs2 = random_fasta(rng, 40, crlf=True, final_newline=False)
    for size in list(range(1, 64)) + [100, 333, 1000, 1 << 16]:
        chunks = list(read_fasta_chunks(io.BytesIO(data), size))
        assert b"".join(chunks) == data, size
        assert all(c.startswith(b">") for c in chunks[1:]), size
        assert [r for c in chunks for r in FO.parse_fasta(c)] == recs, size
        pairs = list(read_paired_fasta_chunks(io.BytesIO(data), io.BytesIO(data2), size))
        assert b"".join(p[0] for p in pairs) == data and b"".join(p[1] for p in pairs) == data2, size
        for c1, c2 in pairs:
            assert len(FO.parse_fasta(c1)) == len(FO.parse_fasta(c2)), size
    assert list(read_fasta_chunks(io.BytesIO(b""))) == []


def hostsim_fasta(data, cut_front=0, cut_back=0):
    """(code, bad line, records as (name, sequence after -u)) from the host build of the device's FASTA steps."""
    from util import hostsim_lib

    lib = hostsim_lib()
    n = len(data)
    buf = np.frombuffer(data, dtype=np.uint8) if n else np.zeros(1, dtype=np.uint8)
    norm = np.zeros(n + 2, dtype=np.uint8)
    cap = data.count(b">") + 1
    rec4 = np.zeros(4 * cap, dtype=np.uint32)
    seq_len = np.zeros(cap, dtype=np.int32)
    n_norm, n_rec, bad_line = C.c_int64(0), C.c_int64(0), C.c_int64(0)
    code = lib.hs_fasta_records(C.c_void_p(buf.ctypes.data), C.c_int64(n), C.c_int(cut_front), C.c_int(cut_back),
                                C.c_void_p(norm.ctypes.data), C.byref(n_norm), C.c_void_p(rec4.ctypes.data),
                                C.c_void_p(seq_len.ctypes.data), C.byref(n_rec), C.byref(bad_line))
    nb = norm[:n_norm.value].tobytes()
    out = []
    for r in range(n_rec.value):
        hs, hl, ss = int(rec4[4 * r]), int(rec4[4 * r + 1]), int(rec4[4 * r + 2])
        assert int(rec4[4 * r + 3]) == ss                      # no qualities: an empty span at the sequence
        out.append((nb[hs:hs + hl].decode("latin-1"), nb[ss:ss + int(seq_len[r])].decode("latin-1")))
    return code, bad_line.value, out


def test_hostsim_fasta_records_match_the_oracle_reader():
    """Fuzzed chunks: line-wrapped sequences of random widths, "\\r\\n", leading comments, empty sequences, a missing
    final newline, -u cuts, and every rejected form (the first bad line is named)."""
    rng = random.Random(11)
    for trial in range(400):
        data, _ = random_fasta(rng, rng.randint(0, 12), crlf=rng.random() < 0.3, comments=rng.random() < 0.4,
                               final_newline=rng.random() < 0.7)
        if trial % 5 == 0 and data:
            lines = data.split(b"\n")
            k = rng.randrange(len(lines))
            lines.insert(k, rng.choice([b"#late", b"ACGT", b"", b"\r"]))
            data = b"\n".join(lines)
        cf, cb = rng.choice([(0, 0), (0, 0), (3, 0), (0, 4), (2, 7)])
        try:
            want = [(n, s[cf:]) for n, s in FO.parse_fasta(data)]
            want = [(n, s[:len(s) - cb] if cb < len(s) else "") for n, s in want]
            want_err = None
        except FO.FastaFormatError as e:
            want_err = int(str(e).split(":")[0].split()[1])
        code, bad_line, got = hostsim_fasta(data, cf, cb)
        if want_err is None:
            assert code == 0, (data, bad_line)
            assert got == want, data
        else:
            assert code in (6, 7) and bad_line + 1 == want_err, (data, code, bad_line, want_err)
    assert hostsim_fasta(b">a\n>b")[2] == [("a", ""), ("b", "")]
    assert hostsim_fasta(b"#x\n>a\nAC\n#y\n")[:2] == (7, 3)
    assert hostsim_fasta(b"AC\n>a\n")[:2] == (6, 0)


def test_output_bound_of_fasta_chunks():
    """The Python output buffers cover the worst FASTA case: records without sequence grow by their empty line."""
    from cutadapt_b200 import _lib
    from cutadapt_b200.pipeline import _output_capacity

    for data in (b">\n" * 1000, b">" + b"\n>" * 999, b">a\n>b\n"):
        n = len(FO.parse_fasta(data))
        written = sum(len(FO.fasta_record(nm, s)) for nm, s in FO.parse_fasta(data))
        assert n and written <= _output_capacity(len(data), _lib.CG_FORMAT_FASTA)
