"""
Read names on the device (--length-tag, --strip-suffix, -x / -y, --rename): every collect against tests/names_oracle.py.
The oracle is composed onto the same collect without name options: that collect's records and info rows give what the
reference's ModificationInfo holds for each read (the sequence as written, the last match's adapter name and matched
bases), and the oracle rewrites the names.  Also the output growing past the usual bound (host chunks, gzip device
chunks, pairs), the paired ID check, FASTA, the tool, and the refusals.
"""
import gzip
import io
import os
import random
import subprocess
import sys

import pytest

import names_oracle as no

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ads(which):
    import cutadapt_b200.adapters as PA

    if which == 1:
        return [PA.BackAdapter("AGATCGGAAGAGC", name="ilmn"), PA.FrontAdapter("ACGGTCAT", name="front")]
    return [PA.BackAdapter("CAGTGGAGTA", name="r2a"), PA.FrontAdapter("TTGACCAG", name="r2front")]


def _random_fastq(rng, n, adapters, mate="", fasta=False):
    recs = []
    for i in range(n):
        seq = "".join(rng.choice("ACGT") for _ in range(rng.randint(0, 60)))
        for _ in range(rng.choice([0, 1, 1])):
            a = rng.choice(adapters)
            piece = a if rng.random() < 0.6 else a[: rng.randint(3, len(a))]
            at = rng.randint(0, len(seq))
            seq = seq[:at] + piece + seq[at:]
        comment = rng.choice(["", " length=99 x", "\tc length=1ab", " a  b ", " /1"])
        name = f"r{i}{mate}{comment}"
        if fasta:
            recs.append(f">{name}\n{seq}\n")
        else:
            recs.append(f"@{name}\n{seq}\n+\n{''.join(chr(33 + rng.choice([2, 20, 40])) for _ in seq)}\n")
    return "".join(recs).encode()


def _data(seed, n=500, fasta=False):
    rng = random.Random(seed)
    return (_random_fastq(rng, n, [a.sequence for a in _ads(1)], "/1", fasta),
            _random_fastq(rng, n, [a.sequence for a in _ads(2)], "/2", fasta))


def _records(data: bytes):
    """[(name, sequence, rest)] of FASTQ or FASTA bytes"""
    lines = data.decode().split("\n")[:-1]
    step = 2 if lines and lines[0].startswith(">") else 4
    return [(lines[i][1:], lines[i + 1], lines[i + 2:i + step]) for i in range(0, len(lines), step)]


def _format(recs) -> bytes:
    out = []
    for name, seq, rest in recs:
        out.append(("@" if rest else ">") + name + "\n" + seq + "\n" + "".join(x + "\n" for x in rest))
    return "".join(out).encode()


def _info(rows: bytes) -> dict:
    """{name as written: (adapter name, matched bases)} from info rows (one adapter round)"""
    out = {}
    for line in rows.decode().split("\n")[:-1]:
        f = line.rsplit("\t", 3)                       # names may hold tabs: split from the right
        if f[1] == "-1":
            out[f[0]] = (None, "")
        else:
            f = line.rsplit("\t", 11)
            out[f[0]] = (f[7], f[5])
    return out


NAMES = {
    "rename": dict(rename="{id} {adapter_name} {match_sequence} {comment}"),
    "rename_tab": dict(rename="{id}\\t{header}"),
    "suffix_tag": dict(suffix=" {name}", length_tag="length=", strip_suffix=(" x", "/1")),
    "prefix": dict(prefix="{name}_", strip_suffix=("b ",)),
}


def _expect(plain: bytes, info: dict, names: dict, cuts=None) -> bytes:
    recs = []
    for name, seq, rest in _records(plain):
        adapter, ms = info.get(name, (None, ""))
        pre = no.pre_name(name, len(seq), adapter, names.get("length_tag"), names.get("strip_suffix", ()),
                          names.get("prefix", ""), names.get("suffix", ""))
        if names.get("rename") is not None:
            d = dict(adapter=adapter, match_sequence=ms, is_rc=name.endswith(" rc"))
            d.update((cuts or {}).get(name, {}))
            pre = no.rename(names["rename"], pre, d)
        recs.append((pre, seq, rest))
    return _format(recs)


def _single(names=None, rows=("info",), **kw):
    from cutadapt_b200.pipeline import FastqTrimmer

    kw.setdefault("minimum_length", 5)
    return FastqTrimmer(_ads(1), rows=rows, **kw, **(names or {}))


SINGLE = {
    "plain": lambda t, d: t.process_chunk(d),
    "split": lambda t, d: t.process_chunk_split(d)["output"] + t.process_chunk_split(d)["too_short"],
    "demux": lambda t, d: b"".join(v for _, v in sorted(t.process_chunk_demux(d).items())),
}


@pytest.mark.parametrize("names", sorted(NAMES))
@pytest.mark.parametrize("variant", sorted(SINGLE))
def test_single_end_against_the_oracle(names, variant):
    data, _ = _data(1)
    extra = dict(redirect=("too_short",)) if variant == "split" else {}
    plain_t = _single(**extra)
    plain = SINGLE[variant](plain_t, data)
    info = _info(plain_t.last_rows["info"])
    t = _single(NAMES[names], **extra)
    got = SINGLE[variant](t, data)
    if variant == "demux":               # every output is in input order: compare the outputs one by one
        pt, nt = _single(**extra), _single(NAMES[names], **extra)
        for k, v in pt.process_chunk_demux(data).items():
            assert nt.process_chunk_demux(data)[k] == _expect(v, info, NAMES[names]), k
        return
    assert got == _expect(plain, info, NAMES[names])
    # the counters are those of the same collect without names, but for the bytes written
    drop = lambda st: {k: v for k, v in st.items() if not k.startswith("out_bytes")}
    assert drop(t.statistics) == drop(plain_t.statistics)


@pytest.mark.parametrize("revcomp", [False, True])
def test_single_end_revcomp_and_rows(revcomp):
    data, _ = _data(2)
    names = dict(suffix=" {name}", length_tag="length=")
    plain_t = _single(rows=("info", "rest"), revcomp=revcomp)
    plain = plain_t.process_chunk(data)
    t = _single(names, rows=("info", "rest"), revcomp=revcomp)
    got = t.process_chunk(data)
    info = _info(plain_t.last_rows["info"])
    assert got == _expect(plain, info, names)
    # the rows print the new names: every row of the renamed collect is the plain row with its name replaced
    renamed = {}
    for (pn, _, _), (gn, _, _) in zip(_records(_single(rows=(), revcomp=revcomp, minimum_length=0).process_chunk(data)),
                                      _records(_single(names, rows=(), revcomp=revcomp, minimum_length=0)
                                               .process_chunk(data))):
        renamed[pn] = gn
    for kind, cut in (("info", lambda x: x.split("\t", 1)[0] if x.count("\t") < 4 else None), ("rest", None)):
        got_rows = t.last_rows[kind].decode().splitlines()
        plain_rows = plain_t.last_rows[kind].decode().splitlines()
        assert len(got_rows) == len(plain_rows)
        for line, plain_line in zip(got_rows, plain_rows):
            if kind == "rest":
                seq, name = plain_line.split(" ", 1)
                assert line == seq + " " + renamed[name]
            else:
                n_fields = 3 if plain_line.rsplit("\t", 3)[1] == "-1" else 11
                name, rest = plain_line.rsplit("\t", n_fields)[0], plain_line.rsplit("\t", n_fields)[1:]
                assert line.rsplit("\t", n_fields) == [renamed[name]] + rest


def test_rename_without_rc_suffix_keeps_rc_variable():
    data, _ = _data(3)
    plain_t = _single(revcomp=True)
    plain = plain_t.process_chunk(data)
    t = _single(dict(rename="{id} {rc}"), revcomp=True, rc_suffix=False)
    got = [r[0] for r in _records(t.process_chunk(data))]
    want = [no.rename("{id} {rc}", n[:-3] if n.endswith(" rc") else n, dict(is_rc=n.endswith(" rc")))
            for n, _, _ in _records(plain)]
    assert got == want


def test_cut_prefix_and_suffix():
    data, _ = _data(4)
    names = dict(rename="{cut_prefix}_{cut_suffix} {header}")
    plain = _single(cut=(2, 3, -2)).process_chunk(data)
    cuts = {n: no.cut_parts(s, (2, 3, -2)) for n, s, _ in _records(data)}
    got = _single(names, cut=(2, 3, -2)).process_chunk(data)
    want = _format([(no.rename(names["rename"], n, cuts[n]), s, r) for n, s, r in _records(plain)])
    assert got == want


def test_output_larger_than_the_input():
    from cutadapt_b200.pipeline import read_gzip_device_chunks

    data, _ = _data(5, 3000)
    names = dict(rename="{header}{header}{header}{header}{header} {match_sequence}")
    plain_t = _single()
    plain = plain_t.process_chunk(data)
    want = _expect(plain, _info(plain_t.last_rows["info"]), names)
    assert len(want) > len(data)
    t = _single(names)
    assert t.process_chunk(data) == want
    gz = b"".join(gzip.compress(data[i:i + 40000]) for i in range(0, len(data), 40000))
    outs = [t.process_chunk(c) for c in read_gzip_device_chunks(io.BytesIO(gz), t, 1 << 16)]
    assert len(outs) > 1 and b"".join(outs) == want
    g = _single(names, gzip_outputs=("output",))
    assert gzip.decompress(g.process_chunk(data)) == want


def test_fasta_and_fastq_to_fasta():
    names = dict(suffix=" {name}", length_tag="length=")
    fa, _ = _data(6, fasta=True)
    plain_t = _single(input_format="fasta")
    plain = plain_t.process_chunk(fa)
    assert _single(names, input_format="fasta").process_chunk(fa) == _expect(plain, _info(plain_t.last_rows["info"]), names)
    fq, _ = _data(6)
    plain_t = _single(output_format="fasta")
    plain = plain_t.process_chunk(fq)
    assert _single(names, output_format="fasta").process_chunk(fq) == _expect(plain, _info(plain_t.last_rows["info"]),
                                                                               names)


# ---- pairs ------------------------------------------------------------------------------------------------------------

def _paired(names=None, **kw):
    from cutadapt_b200.pipeline import PairedFastqTrimmer

    return PairedFastqTrimmer(_ads(1), _ads(2), dict(minimum_length=5), dict(minimum_length=5), rows=("info",),
                              rows2=("info",), **kw, **(names or {}))


def _interleave(a, b):
    la, lb = a.splitlines(True), b.splitlines(True)
    return b"".join(b"".join(la[i:i + 4] + lb[i:i + 4]) for i in range(0, len(la), 4))


def _expect_pair(p1, p2, info1, info2, names):
    if names.get("rename") is None:
        return _expect(p1, info1, names), _expect(p2, info2, names)
    r1, r2 = [], []
    for (n1, s1, x1), (n2, s2, x2) in zip(_records(p1), _records(p2)):
        i1, i2 = info1.get(n1, (None, "")), info2.get(n2, (None, ""))
        a, b = no.rename_pair(names["rename"], n1, n2, dict(adapter=i1[0], match_sequence=i1[1]),
                              dict(adapter=i2[0], match_sequence=i2[1]))
        r1.append((a, s1, x1))
        r2.append((b, s2, x2))
    return _format(r1), _format(r2)


PNAMES = {
    "rename": dict(rename="{id} {r1.adapter_name} {r2.adapter_name} {rn} {r2.match_sequence}"),
    "suffix_tag": dict(suffix=" {name}", length_tag="length=", strip_suffix=(" x",)),
}
PAIRED = {
    "any": (dict(), lambda t, a, b: t.process_chunk(a, b)),
    "both": (dict(pair_filter="both"), lambda t, a, b: t.process_chunk(a, b)),
    "first": (dict(pair_filter="first"), lambda t, a, b: t.process_chunk(a, b)),
    "interleaved_input": (dict(), lambda t, a, b: t.process_chunk(_interleave(a, b))),
    "gzip": (dict(gzip_outputs=("output",)), lambda t, a, b: tuple(gzip.decompress(x) for x in t.process_chunk(a, b))),
}


@pytest.mark.parametrize("names", sorted(PNAMES))
@pytest.mark.parametrize("variant", sorted(PAIRED))
def test_paired_against_the_oracle(names, variant):
    extra, run = PAIRED[variant]
    a, b = _data(7)
    plain_t = _paired(**extra)
    p1, p2 = run(plain_t, a, b)
    info1, info2 = (_info(x) for x in plain_t.last_rows["info"])
    t = _paired(PNAMES[names], **extra)
    assert run(t, a, b) == _expect_pair(p1, p2, info1, info2, PNAMES[names])


def test_paired_interleaved_outputs_and_demux():
    a, b = _data(8)
    names = PNAMES["suffix_tag"]
    plain_t = _paired()
    p1, p2 = plain_t.process_chunk(a, b)
    info1, info2 = (_info(x) for x in plain_t.last_rows["info"])
    w1, w2 = _expect_pair(p1, p2, info1, info2, names)
    t = _paired(names, interleaved_outputs=("output",))
    assert t.process_chunk(a, b)[0] == _interleave(w1, w2)
    pd, nd = _paired(), _paired(names)
    for comb in (False, True):
        for k, (x1, x2) in pd.process_chunk_demux(a, b, combinatorial=comb).items():
            assert nd.process_chunk_demux(a, b, combinatorial=comb)[k] == (_expect(x1, info1, names),
                                                                           _expect(x2, info2, names)), k


def test_paired_revcomp_and_pair_adapters():
    a, b = _data(9)
    names = dict(suffix=" {name}")
    for extra in (dict(revcomp=True), dict(pair_adapters=True)):
        from cutadapt_b200.pipeline import PairedFastqTrimmer

        mk = lambda n: PairedFastqTrimmer(_ads(1), _ads(2), {}, {}, rows=("rest",), **extra, **n)
        plain_t = mk({})
        p1, p2 = plain_t.process_chunk(a, b)
        t = mk(names)
        g1, g2 = t.process_chunk(a, b)
        # the adapter of each output record's last match, from the rows of that record's mate as written
        info = [{}, {}]
        for mate, out in enumerate((p1, p2)):
            for n, _, _ in _records(out):
                info[mate].setdefault(n, (None, ""))
        adapters = [{}, {}]
        names1 = [x.name for x in _ads(1)]
        names2 = [x.name for x in _ads(2)]
        for mate, out in enumerate((g1, g2)):
            for (pn, ps, pr), (gn, gs, gr) in zip(_records((p1, p2)[mate]), _records(out)):
                assert (gs, gr) == (ps, pr)
                assert gn[:len(pn) + 1] == pn + " "
                adapters[mate][pn] = gn[len(pn) + 1:]
                # R1's output always holds the -a set's matches, R2's the -A set's (also for a swapped pair)
                assert adapters[mate][pn] in (names1, names2)[mate] + ["no_adapter"]
        if "pair_adapters" in extra:            # a pair matches adapter pair i on both mates, or neither
            for (n1, _, _), (n2, _, _) in zip(_records(p1), _records(p2)):
                x, y = adapters[0][n1], adapters[1][n2]
                assert (x == "no_adapter") == (y == "no_adapter")
                if x != "no_adapter":
                    assert names1.index(x) == names2.index(y)
        # rest rows of R1: the plain row with the record's new name, exactly (no second " rc")
        for pl, gl in zip(plain_t.last_rows["rest"][0].decode().splitlines(), t.last_rows["rest"][0].decode().splitlines()):
            seq, name = pl.split(" ", 1)
            assert gl == f"{seq} {name} {adapters[0][name]}"


def test_paired_output_growth_and_id_mismatch():
    a, b = _data(10, 2000)
    big = dict(rename="{id} {header}{header}{header}{header}{header}")
    plain_t = _paired()
    p1, p2 = plain_t.process_chunk(a, b)
    info1, info2 = (_info(x) for x in plain_t.last_rows["info"])
    t = _paired(big)
    want = _expect_pair(p1, p2, info1, info2, big)
    assert len(want[0]) > len(a)
    assert t.process_chunk(a, b) == want
    bad = _paired(dict(rename="{id}{rn} {comment}"))
    first = _records(a)[0][0].split()[0]
    with pytest.raises(Exception) as e:
        bad.process_chunk(a, b)
    assert str(e.value) == (f"After renaming R1 and R2, their IDs are no longer identical: '{first}1' != "
                            f"'{first[:-1]}22'. Original read ID: '{first}'. ")
    # the context goes on working
    assert t.process_chunk(a, b) == want


def test_refusals():
    from cutadapt_b200.pipeline import FastqTrimmer

    with pytest.raises(ValueError, match="Option --rename cannot be combined"):
        FastqTrimmer(_ads(1), rename="{id}", prefix="x")
    with pytest.raises(ValueError, match="Variable 'r1.id' not recognized"):
        _paired(dict(rename="{r1.id}"))
    with pytest.raises(ValueError, match="'\\.'"):
        FastqTrimmer(_ads(1), length_tag="len.")


def test_trim_fastq_tool(tmp_path):
    data, _ = _data(11)
    (tmp_path / "in.fastq").write_bytes(data)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), "-a", "ilmn=AGATCGGAAGAGC", "-m",
                        "5", "-y", " {name}", "--length-tag", "length=", "--strip-suffix", " x", "-o", "out.fastq",
                        "in.fastq"], capture_output=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    from cutadapt_b200.pipeline import FastqTrimmer
    import cutadapt_b200.adapters as PA

    t = FastqTrimmer([PA.BackAdapter("AGATCGGAAGAGC", name="ilmn")], minimum_length=5, rows=("info",))
    plain = t.process_chunk(data)
    want = _expect(plain, _info(t.last_rows["info"]), dict(suffix=" {name}", length_tag="length=", strip_suffix=(" x",)))
    assert (tmp_path / "out.fastq").read_bytes() == want


# ---- the reference's known answers (tests/golden/names_kat.json.gz) ----------------------------------------------------

def _kat_cli():
    from util import golden

    return golden("names_kat.json.gz")["cli"]


def _trimmer_of(argv, paired, fasta):
    """FastqTrimmer / PairedFastqTrimmer built from a known answer's argument list, as tools/trim_fastq.py reads it."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import trim_fastq as T
    from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer

    a = {"-a": [], "-b": [], "-g": [], "-A": []}
    kw, cut, i = {}, [], 0
    e, times, rename = 0.1, 1, None
    while i < len(argv):
        x = argv[i]
        if x.startswith("--rename="):
            rename = x.split("=", 1)[1]; i += 1; continue
        if x.startswith("--cut="):
            cut.append(int(x.split("=", 1)[1])); i += 1; continue
        v = argv[i + 1]
        if x in a: a[x].append(v)
        elif x == "-e": e = float(v)
        elif x == "-n": times = int(v)
        elif x == "--rename": rename = v
        elif x == "--length-tag": kw["length_tag"] = v
        elif x == "--strip-suffix": kw.setdefault("strip_suffix", []).append(v)
        elif x == "-y": kw["suffix"] = v
        elif x == "--revcomp":
            kw["revcomp"] = True; i += 1; continue
        i += 2
    ads = lambda flag, kind: T.make_adapters(a[flag], kind, e, 3)
    fmt = dict(input_format="fasta") if fasta else {}
    if paired:
        return PairedFastqTrimmer(ads("-a", "back"), ads("-A", "back"), dict(cut=cut, times=times), dict(times=times),
                                  rename=rename, rc_suffix=not rename, **fmt, **kw)
    return FastqTrimmer(ads("-a", "back") + ads("-b", "anywhere") + ads("-g", "front"), times=times, cut=cut,
                        rename=rename, rc_suffix=not rename, **fmt, **kw)


@pytest.mark.parametrize("case", range(7))
def test_known_answers_through_the_trimmers(case):
    c = _kat_cli()[case]
    inputs = [c["inputs"][k].encode() for k in c["input_order"]]
    t = _trimmer_of(c["argv"], len(inputs) == 2, c["input_order"][0].endswith((".fa", ".fasta")))
    got = t.process_chunk(*inputs)
    got = list(got) if isinstance(got, tuple) else [got]
    if c["expected"] is None:                   # test_reverse_complement_no_rc_suffix asserts these
        recs = _records(got[0])
        assert len(recs) == c["n_reads"] and list(recs[1][:2]) == c["read1"]
        return
    assert [x.decode() for x in got] == c["expected"], c["name"]


@pytest.mark.parametrize("case", range(7))
def test_known_answers_through_the_tool(case, tmp_path):
    c = _kat_cli()[case]
    paths = []
    for k in c["input_order"]:
        (tmp_path / ("in_" + k)).write_bytes(c["inputs"][k].encode())
        paths.append("in_" + k)
    ext = os.path.splitext(c["input_order"][0])[1]
    outs = ["-o", "out1" + ext] + (["-p", "out2" + ext] if len(paths) == 2 else [])
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py")] + c["argv"] + outs + paths,
                       capture_output=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    got = [(tmp_path / ("out%d" % (i + 1) + ext)).read_bytes() for i in range(len(paths))]
    if c["expected"] is None:
        recs = _records(got[0])
        assert len(recs) == c["n_reads"] and list(recs[1][:2]) == c["read1"]
        return
    assert [x.decode() for x in got] == c["expected"], c["name"]


# ---- collects without names are those of the commit before the name stage --------------------------------------------

def test_collects_without_names_are_unchanged():
    import json
    import names_unchanged
    from util import golden  # noqa: F401

    with open(os.path.join(ROOT, "tests", "golden", "names_unchanged.json")) as f:
        want = json.load(f)
    assert names_unchanged.answers() == want


def test_name_stage_launches():
    """A collect with names launches the collect without them plus the name stage: 5 per mate for step 1, then with
    --rename 1 + 3 per mate + 1."""
    from cutadapt_b200 import _lib

    data, _ = _data(12)

    def launches(t):
        t.process_chunk(data)                   # buffers
        n0 = _lib.lib().cg_ctx_launch_count(t.ctx.handle)
        t.process_chunk(data)
        return _lib.lib().cg_ctx_launch_count(t.ctx.handle) - n0

    base = launches(_single(rows=()))
    assert launches(_single(dict(suffix=" {name}"), rows=())) == base + 5
    assert launches(_single(dict(rename="{id} {adapter_name}"), rows=())) == base + 5 + 5
    assert launches(_single(dict(rename="{header}"), rows=())) == base       # installs no renamer: no stage


# ---- more paths ----------------------------------------------------------------------------------------------------------

def test_bam_input():
    import bam_oracle as BO
    import cutadapt_b200.adapters as PA
    from cutadapt_b200.pipeline import FastqTrimmer, read_gzip_device_chunks

    rng = random.Random(13)
    recs = []
    for i in range(800):
        seq = "".join(rng.choice("ACGT") for _ in range(rng.randint(1, 60)))
        if rng.random() < 0.6:
            at = rng.randint(0, len(seq))
            seq = seq[:at] + "AGATCGGAAGAGC" + seq[at:]
        recs.append(BO.record(f"r{i}".encode(), seq, [rng.choice([2, 20, 40]) for _ in seq]))
    bam = BO.bam_file(recs, member=4000)
    plain_in = BO.fastq_of(bam)
    names = dict(rename="{id} {adapter_name} {match_sequence} {header}{header}{header}{header}")
    ads = [PA.BackAdapter("AGATCGGAAGAGC", name="ilmn")]
    plain_t = FastqTrimmer(ads, rows=("info",))
    plain = plain_t.process_chunk(plain_in)
    want = _expect(plain, _info(plain_t.last_rows["info"]), names)
    t = FastqTrimmer(ads, input_format="bam", **names)
    outs = [t.process_chunk(c) for c in read_gzip_device_chunks(io.BytesIO(bam), t, 1 << 14)]
    assert len(outs) > 1 and b"".join(outs) == want


def test_wildcard_rows_and_fasta_filter_outputs():
    import cutadapt_b200.adapters as PA
    from cutadapt_b200.pipeline import FastqTrimmer

    data, _ = _data(14)
    names = dict(suffix=" {name}", length_tag="length=")
    wild = [PA.BackAdapter("AGATCNNAAGAGC", name="w")]
    plain_t = FastqTrimmer(wild, rows=("info", "wildcard"), redirect=("untrimmed",),
                           redirect_formats={"untrimmed": "fasta"}, minimum_length=5)
    t = FastqTrimmer(wild, rows=("info", "wildcard"), redirect=("untrimmed",), redirect_formats={"untrimmed": "fasta"},
                     minimum_length=5, **names)
    p, g = plain_t.process_chunk_split(data), t.process_chunk_split(data)
    info = _info(plain_t.last_rows["info"])
    for k in p:
        assert g[k] == _expect(p[k], info, names), k
    renamed = {n: m for (n, _, _), (m, _, _) in zip(_records(p["output"] + p["untrimmed"]),
                                                    _records(g["output"] + g["untrimmed"]))}
    for pl, gl in zip(plain_t.last_rows["wildcard"].decode().splitlines(), t.last_rows["wildcard"].decode().splitlines()):
        w, name = pl.split(" ", 1)
        if name in renamed:
            assert gl == w + " " + renamed[name]


def test_paired_info_rows_of_both_mates():
    a, b = _data(15)
    names = PNAMES["rename"]
    plain_t, t = _paired(), _paired(names)
    p1, p2 = plain_t.process_chunk(a, b)
    g1, g2 = t.process_chunk(a, b)
    for k, (prows, grows) in enumerate(zip(plain_t.last_rows["info"], t.last_rows["info"])):
        renamed = {n: m for (n, _, _), (m, _, _) in zip(_records((p1, p2)[k]), _records((g1, g2)[k]))}
        for pl, gl in zip(prows.decode().splitlines(), grows.decode().splitlines()):
            n_fields = 3 if pl.rsplit("\t", 3)[1] == "-1" else 11
            name, rest = pl.rsplit("\t", n_fields)[0], pl.rsplit("\t", n_fields)[1:]
            if name in renamed:
                assert gl.rsplit("\t", n_fields) == [renamed[name]] + rest


def test_cut_parts_under_revcomp():
    """{cut_prefix} / {cut_suffix} are the bases of the read as it came, also when --revcomp turned the read (single
    reads: reversed in place) or swapped the pair (the read sits in the other mate's slot)."""
    from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer

    a, b = _data(16)
    cuts1 = {n.split()[0]: no.cut_parts(s, (3, -2)) for n, s, _ in _records(a)}
    cuts2 = {n.split()[0]: no.cut_parts(s, (2,)) for n, s, _ in _records(b)}
    t = FastqTrimmer(_ads(1), cut=(3, -2), revcomp=True, rc_suffix=False, rename="{id} {cut_prefix}:{cut_suffix} {rc}")
    n_rc = 0
    for n, _, _ in _records(t.process_chunk(a)):
        rid, parts, rc = (n.split(" ") + [""])[:3]
        n_rc += rc == "rc"
        assert parts == cuts1[rid].get("cut_prefix", "") + ":" + cuts1[rid].get("cut_suffix", "")
    assert n_rc > 0
    pt = PairedFastqTrimmer(_ads(1), _ads(2), dict(cut=(3, -2)), dict(cut=(2,)), revcomp=True, rc_suffix=False,
                            rename="{id} {r1.cut_prefix}:{r1.cut_suffix}:{r2.cut_prefix}")
    o1, o2 = pt.process_chunk(a, b)
    assert pt.statistics[0]["reverse_complemented"] > 0
    for (n1, _, _), (n2, _, _) in zip(_records(o1), _records(o2)):
        rid = n1.split(" ")[0]
        key = rid[:-1] + "1"
        want = "%s:%s:%s" % (cuts1[key].get("cut_prefix", ""), cuts1[key].get("cut_suffix", ""),
                             cuts2[key[:-1] + "2"].get("cut_prefix", ""))
        assert n1.split(" ")[1] == want and n2.split(" ")[1] == want


def test_interleaved_gzip_device_input_that_grows():
    from cutadapt_b200.pipeline import read_gzip_device_interleaved_chunks

    a, b = _data(17, 2000)
    big = dict(rename="{id} {header}{header}{header}{header}{header}")
    plain_t = _paired()
    p1, p2 = plain_t.process_chunk(a, b)
    info1, info2 = (_info(x) for x in plain_t.last_rows["info"])
    want = _expect_pair(p1, p2, info1, info2, big)
    t = _paired(big)
    il = _interleave(a, b)
    gz = b"".join(gzip.compress(il[i:i + 40000]) for i in range(0, len(il), 40000))      # members: several chunks
    outs = [t.process_chunk(c) for c in read_gzip_device_interleaved_chunks(io.BytesIO(gz), t, 1 << 16)]
    assert len(outs) > 1
    assert (b"".join(o[0] for o in outs), b"".join(o[1] for o in outs)) == want


def test_empty_rename_changes_nothing():
    data, _ = _data(18)
    assert _single(dict(rename=""), rows=()).process_chunk(data) == _single(rows=()).process_chunk(data)
