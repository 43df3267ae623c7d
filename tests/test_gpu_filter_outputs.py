"""
GPU tests (-m gpu) of the filter outputs of the device FASTQ/FASTA path (cg_fastq_collect_split,
cg_fastq_collect_paired_split; --too-short-output, --too-long-output, --untrimmed-output and their paired forms):
the reference's known answers (tests/golden/filter_outputs_kat.json.gz) through the Python API and through
tools/trim_fastq.py, randomized chunks against the redirect oracle (tests/filter_outputs_oracle.py), and on every
chunk the main output, the counters and the statistics vector against the plain collect.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import fasta_oracle as FO  # noqa: E402
import filter_outputs_oracle as RO  # noqa: E402
from cutadapt_b200 import _lib  # noqa: E402
from cutadapt_b200.pipeline import FastqTrimmer, PairedFastqTrimmer, _fastq_params  # noqa: E402
from test_gpu_fastq import flip_records, synthetic_fastq, trimmer_kwargs  # noqa: E402
from util import fastq_case_adapters, fastq_case_kwargs, spec_of  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = ("too_short", "too_long", "untrimmed")


def descs_of(adapters):
    import cutadapt_b200.adapters as PA

    if not adapters:
        return None, None
    spec = spec_of(PA.MultipleAdapters(adapters))
    return spec.adapters, spec.groups


def without_out_bytes(st):
    return {k: v for k, v in st.items() if k != "out_bytes"}


# ---- the reference's answers --------------------------------------------------------------------------------------

def kat_cases():
    return RO.filter_outputs_kat()["cases"]


def test_kat_cases_through_the_api():
    for c in kat_cases():
        o = c["options"]
        data = [RO.kat_file(k) for k in c["inputs"]]
        fmt = RO.input_format_of(data[0])
        kw = RO.kat_trimmer_kwargs(o)
        if c["kind"] == "paired":
            t = PairedFastqTrimmer(FO.kat_adapters(o, "specs1"), FO.kat_adapters(o, "specs2"), kw, kw,
                                   o.get("pair_filter", "any"), input_format=fmt, redirect=o.get("redirect", ()))
            got = t.process_chunk_split(*data)
            for name, exp in c["expected"].items():
                assert got[name] == (RO.kat_file(exp[0]), RO.kat_file(exp[1])), (c["name"], name)
            _, c1, c2 = RO.redirect_trim_paired(data[0], data[1], *descs_of(FO.kat_adapters(o, "specs1")),
                                                *descs_of(FO.kat_adapters(o, "specs2")), kw, kw,
                                                o.get("pair_filter", "any"), o.get("redirect", ()), input_format=fmt)
            for st, cc in zip(t.statistics, (c1, c2)):
                for k, v in cc.items():
                    assert st[k] == v, (c["name"], k)
            continue
        t = FastqTrimmer(FO.kat_adapters(o), input_format=fmt, redirect=o.get("redirect", ()), **kw)
        got = t.process_chunk_split(data[0])
        for name, exp in c["expected"].items():
            assert got[name] == RO.kat_file(exp), (c["name"], name)
        for k, v in c["counters"].items():
            assert t.statistics[k] == v, (c["name"], k)
        _, counters = RO.redirect_trim(data[0], *descs_of(FO.kat_adapters(o)), o.get("redirect", ()),
                                       input_format=fmt, **kw)
        for k, v in counters.items():
            assert t.statistics[k] == v, (c["name"], k)


def tool_args(c, tmp_path):
    """tools/trim_fastq.py's command line of a case; {output: path(s)} of what it writes."""
    o = c["options"]
    args, files = [], {}
    for key, flag in (("specs", "-a"), ("specs1", "-a"), ("specs2", "-A")):
        for kind, spec in o.get(key, []):
            assert kind == "back"
            args += [flag, spec]
    if "minimum_length" in o:
        args += ["-m", str(o["minimum_length"])]
    if "maximum_length" in o:
        args += ["-M", str(o["maximum_length"])]
    if "pair_filter" in o:
        args += ["--pair-filter", o["pair_filter"]]
    for name, exp in c["expected"].items():
        exps = exp if isinstance(exp, list) else [exp]
        paths = [str(tmp_path / f"{name}.{k + 1}.{e.rsplit('.', 1)[1]}") for k, e in enumerate(exps)]
        files[name] = paths
        if name == "output":
            args += ["-o", paths[0]] + (["-p", paths[1]] if len(paths) > 1 else [])
        else:
            flag = "--" + name.replace("_", "-")
            args += [flag + "-output", paths[0]] + ([flag + "-paired-output", paths[1]] if len(paths) > 1 else [])
    for k, key in enumerate(c["inputs"]):
        p = tmp_path / f"in.{k + 1}.{key.rsplit('.', 1)[1]}"
        p.write_bytes(RO.kat_file(key))
        args.append(str(p))
    return args, files


def test_kat_cases_through_trim_fastq(tmp_path):
    for c in kat_cases():
        if not c["expected"]:
            continue
        d = tmp_path / c["name"]
        d.mkdir()
        args, files = tool_args(c, d)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), *args], capture_output=True,
                           text=True)
        assert r.returncode == 0, r.stderr
        for name, exp in c["expected"].items():
            for path, key in zip(files[name], exp if isinstance(exp, list) else [exp]):
                assert open(path, "rb").read() == RO.kat_file(key), (c["name"], name, path)


def test_untrimmed_output_receives_unknown_when_demultiplexing(tmp_path):
    """-o '{name}.fastq' --untrimmed-output: the reads without a match go to the untrimmed output (Demultiplexer's
    untrimmed_output), the named outputs are those of plain demultiplexing."""
    data = synthetic_fastq(3000, seed=91)
    inp = tmp_path / "in.fastq"
    inp.write_bytes(data)
    tool = os.path.join(ROOT, "tools", "trim_fastq.py")
    base = ["-a", "first=AGATCGGAAGAGC", "-g", "second=TTGACNNACG", "-m", "10"]
    r = subprocess.run([sys.executable, tool, *base, "-o", str(tmp_path / "a-{name}.fastq"), str(inp)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([sys.executable, tool, *base, "--untrimmed-output", str(tmp_path / "untrimmed.fastq"), "-o",
                        str(tmp_path / "b-{name}.fastq"), str(inp)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    read = lambda name: (tmp_path / name).read_bytes()  # noqa: E731
    assert read("untrimmed.fastq") == read("a-unknown.fastq") != b""
    assert not (tmp_path / "b-unknown.fastq").exists()
    for name in ("first", "second"):
        assert read(f"b-{name}.fastq") == read(f"a-{name}.fastq")


# ---- randomized chunks against the redirect oracle and against the plain collect ------------------------------------

BASE = dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]], quality_cutoff=[5, 20])
SINGLE = {
    "all": (BASE, dict(minimum_length=40, maximum_length=140), ALL, {}, "fastq"),
    "filters_in_front": (BASE, dict(minimum_length=30, maximum_length=149, max_n=0.1, max_expected_errors=2.5,
                                    discard_casava=True), ALL, {}, "fastq"),
    "too_short_only": (BASE, dict(minimum_length=40, maximum_length=140, discard_untrimmed=True), ("too_short",), {},
                       "fastq"),
    "m0": (BASE, dict(minimum_length=0, maximum_length=100), ("too_short", "too_long"), {}, "fastq"),
    "mask": (BASE, dict(action="mask", times=2, trim_n=True, minimum_length=50), ALL, {}, "fastq"),
    "lowercase": (BASE, dict(action="lowercase", times=2, poly_a=True, minimum_length=20), ALL, {}, "fastq"),
    "none": (dict(adapters=[["back", "AGATCGGAAGAGC"]]), dict(action="none", length=100, minimum_length=120), ALL, {},
             "fastq"),
    "retain": (dict(adapters=[["linked", "TTGACNNACG", "AGATCGGAAGAGC"], ["back", "CACGTCTGAACTC"]],
                    quality_cutoff=[0, 15]), dict(action="retain", minimum_length=30), ALL, {}, "fastq"),
    "crop": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["anywhere", "CACGTCTGAA"]]),
             dict(action="crop", trim_n=True, maximum_length=20), ALL, {}, "fastq"),
    "modifiers": (BASE, dict(cut=[3, -2], poly_a=True, length=-90, trim_n=True, minimum_length=60), ALL, {}, "fastq"),
    "revcomp": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]]),
                dict(revcomp=True, minimum_length=60, trim_n=True), ALL, {}, "fastq"),
    "no_adapters": (dict(adapters=[], quality_cutoff=[0, 25]), dict(minimum_length=50), ALL, {}, "fastq"),
    "to_fasta": (BASE, dict(minimum_length=40, maximum_length=140), ALL, {}, "fastq_to_fasta"),
    "mixed_formats": (BASE, dict(minimum_length=40, maximum_length=140), ALL,
                      dict(too_short="fasta", untrimmed="fasta"), "fastq"),
    "mixed_formats_fasta_main": (BASE, dict(minimum_length=40, maximum_length=140), ALL,
                                 dict(too_long="fastq"), "fastq_to_fasta"),
    "fasta": (dict(adapters=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]]),
              dict(minimum_length=40, maximum_length=140, cut=[2], poly_a=True), ALL, {}, "fasta"),
    "fasta_revcomp": (dict(adapters=[["back", "AGATCGGAAGAGC"]]), dict(revcomp=True, minimum_length=50), ALL, {},
                      "fasta"),
}
FORMATS = {"fastq": ("fastq", None), "fastq_to_fasta": ("fastq", "fasta"), "fasta": ("fasta", None)}


def plain_equivalent(kw, redirect):
    """The options of the plain collect that removes what the split call redirects: the untrimmed output is the
    untrimmed filter with a writer, so the plain call discards the untrimmed reads."""
    return {**kw, "discard_untrimmed": True} if "untrimmed" in redirect else dict(kw)


def single_case(options, extra, redirect, formats, fmt, data):
    """(split trimmer, plain trimmer, oracle outputs, oracle counters); both trimmers collect statistics."""
    input_format, output_format = FORMATS[fmt]
    kw = {**trimmer_kwargs(options), **extra, "input_format": input_format, "output_format": output_format,
          "collect_statistics": True}
    ads = fastq_case_adapters(options)
    split = FastqTrimmer(ads, redirect=redirect, redirect_formats=formats, **kw)
    plain = FastqTrimmer(ads, **plain_equivalent(kw, redirect))
    okw = {**fastq_case_kwargs(options), **extra}
    exp, counters = RO.redirect_trim(data, *descs_of(ads), redirect, formats, input_format, output_format, **okw)
    return split, plain, exp, counters


def as_fasta(data: bytes) -> bytes:
    return b"".join(FO.fasta_record(n, s) for n, s, _ in _parse(data))


def _parse(data):
    from oracle import oracle

    return oracle.parse_fastq(data)


def check_against_plain(split, plain, got, chunk):
    """The main output, the counters and the statistics vector of the split call equal the plain collect's."""
    assert got["output"] == plain.process_chunk(chunk)
    assert without_out_bytes(split.statistics) == without_out_bytes(plain.statistics)
    v1, l1, k1 = split.statistics_vector()
    v2, l2, k2 = plain.statistics_vector()
    assert (l1, k1) == (l2, k2) and np.array_equal(v1, v2)


@pytest.mark.parametrize("variant", list(SINGLE))
def test_random_chunks_against_oracle_and_collect(variant):
    options, extra, redirect, formats, fmt = SINGLE[variant]
    data = synthetic_fastq(5000, seed=300 + list(SINGLE).index(variant))
    if "revcomp" in variant:
        data = flip_records(data, 7)
    if fmt == "fasta":
        data = as_fasta(data)
    split, plain, exp, counters = single_case(options, extra, redirect, formats, fmt, data)
    got = split.process_chunk_split(data)
    assert set(got) == {"output", *redirect}
    for name in got:
        assert got[name] == exp[name], name
    for k, v in counters.items():
        assert split.statistics[k] == v, k
    check_against_plain(split, plain, got, data)
    if variant == "m0":                      # -m 0: the filter exists but never fires
        assert got["too_short"] == b"" and got["too_long"] != b""
    split.close()
    plain.close()


def test_edge_chunks_and_several_in_flight():
    """Empty chunks, a chunk whose every read is filtered, and several chunks in flight (process_chunks_split)."""
    options, extra = BASE, dict(minimum_length=40, maximum_length=140)
    chunks = [synthetic_fastq(n, seed=400 + i) for i, n in enumerate((0, 1, 2500, 0, 17, 30000, 3))]
    # every read filtered: nothing reaches the main output
    chunks.append(b"".join(b"@s%d\nACGT\n+\nIIII\n" % i for i in range(100)))
    split, plain, _, _ = single_case(options, extra, ALL, {}, "fastq", b"")
    got = list(split.process_chunks_split(chunks))
    assert got[-1]["output"] == b"" and got[-1]["too_short"].count(b"\n") == 400
    assert got[0] == {"output": b"", "too_short": b"", "too_long": b"", "untrimmed": b""}
    for part, chunk in zip(got, chunks):
        exp, _ = RO.redirect_trim(chunk, *descs_of(fastq_case_adapters(options)), ALL,
                                  **{**fastq_case_kwargs(options), **extra})
        assert part == exp
    assert list(plain.process_chunks(chunks)) == [p["output"] for p in got]
    assert without_out_bytes(split.statistics) == without_out_bytes(plain.statistics)
    assert np.array_equal(split.statistics_vector()[0], plain.statistics_vector()[0])


def test_two_million_records():
    """One chunk of 2 M records: the main output and the counters equal the plain collect's, and every redirected record
    is where its filter says."""
    n, L = 2_000_000, 60
    rng = np.random.default_rng(5)
    lengths = np.where(rng.random(n) < 0.5, 60, 40)        # untrimmed reads of 60 bp are too long, of 40 bp untrimmed
    seq = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), (n, L))
    ad = np.frombuffer(b"AGATCGGAAGAGC", dtype=np.uint8)
    starts = rng.integers(5, L, n)
    has = rng.random(n) < 0.5
    for j in range(ad.size):
        pos = starts + j
        ok = has & (pos < L)
        seq[np.nonzero(ok)[0], pos[ok]] = ad[j]
    names = np.char.encode(np.char.add("r", np.arange(n).astype(str)), "latin-1")
    recs = [b"@%s\n%s\n+\n%s\n" % (names[i], seq[i, :lengths[i]].tobytes(), b"I" * int(lengths[i])) for i in range(n)]
    data = b"".join(recs)
    kw = dict(minimum_length=30, maximum_length=55, collect_statistics=True)
    ads = fastq_case_adapters(dict(adapters=[["back", "AGATCGGAAGAGC"]]))
    split = FastqTrimmer(ads, redirect=ALL, **kw)
    plain = FastqTrimmer(ads, **plain_equivalent(kw, ALL))
    got = split.process_chunk_split(data)
    check_against_plain(split, plain, got, data)
    st = split.statistics
    assert st["n_records"] == n
    assert got["too_short"].count(b"\n") == 4 * st["too_short"] > 0
    assert got["too_long"].count(b"\n") == 4 * st["too_long"] > 0
    assert got["untrimmed"].count(b"\n") == 4 * st["discarded"] > 0
    assert st["n_written"] + st["too_short"] + st["too_long"] + st["discarded"] == n
    lines = got["too_short"].split(b"\n")
    assert all(len(x) < 30 for x in lines[1::4])
    lines = got["too_long"].split(b"\n")
    assert all(len(x) > 55 for x in lines[1:-1:4])


# ---- paired-end ----------------------------------------------------------------------------------------------------

PAIRED = {
    "any": (dict(adapters1=[["back", "AGATCGGAAGAGC"]], adapters2=[["back", "AGATCGGAAGAGC"], ["front", "TTGACNNACG"]],
                 options1=dict(quality_cutoff=[0, 20], minimum_length=40, maximum_length=140, cut=[2], poly_a=True),
                 options2=dict(quality_cutoff=[3, 15], minimum_length=35, maximum_length=140, cut=[-3], poly_a=True,
                               trim_n=True)), "any", ALL, {}, "fastq"),
    "both": (dict(adapters1=[["back", "AGATCGGAAGAGC"]], adapters2=[["back", "AGATCGGAAGAGC"]],
                  options1=dict(minimum_length=40, maximum_length=140, max_n=2),
                  options2=dict(minimum_length=40, maximum_length=140, max_n=2)), "both", ALL, {}, "fastq"),
    "first": (dict(adapters1=[["back", "AGATCGGAAGAGC"]], adapters2=[["back", "AGATCGGAAGAGC"]],
                   options1=dict(minimum_length=40, action="mask"), options2=dict(minimum_length=40, action="mask")),
              "first", ALL, {}, "fastq"),
    "one_mate_adapters": (dict(adapters1=[["back", "AGATCGGAAGAGC"]], adapters2=[],
                               options1=dict(minimum_length=20), options2=dict(minimum_length=20)), "any",
                          ("untrimmed", "too_short"), {}, "fastq"),
    "mate2_only_filter": (dict(adapters1=[["back", "AGATCGGAAGAGC"]], adapters2=[["back", "AGATCGGAAGAGC"]],
                               options1=dict(), options2=dict(minimum_length=50)), "any", ALL, {}, "fastq"),
    "mixed_formats": (dict(adapters1=[["back", "AGATCGGAAGAGC"]], adapters2=[["back", "AGATCGGAAGAGC"]],
                           options1=dict(minimum_length=40, maximum_length=140),
                           options2=dict(minimum_length=40, maximum_length=140)), "any", ALL,
                      dict(too_long="fasta"), "fastq"),
    "fasta": (dict(adapters1=[["back", "AGATCGGAAGAGC"]], adapters2=[["back", "AGATCGGAAGAGC"]],
                   options1=dict(minimum_length=40, maximum_length=140), options2=dict(minimum_length=40)), "any", ALL,
              {}, "fasta"),
}


@pytest.mark.parametrize("variant", list(PAIRED))
def test_paired_random_chunks_against_oracle_and_collect(variant):
    options, mode, redirect, formats, fmt = PAIRED[variant]
    data1 = synthetic_fastq(4000, seed=500 + 2 * list(PAIRED).index(variant))
    data2 = synthetic_fastq(4000, seed=501 + 2 * list(PAIRED).index(variant))
    if fmt == "fasta":
        data1, data2 = as_fasta(data1), as_fasta(data2)
    input_format, output_format = FORMATS[fmt]
    ads1, ads2 = fastq_case_adapters(options, "adapters1"), fastq_case_adapters(options, "adapters2")
    kw1, kw2 = trimmer_kwargs(options["options1"]), trimmer_kwargs(options["options2"])
    common = dict(input_format=input_format, output_format=output_format, collect_statistics=True)
    split = PairedFastqTrimmer(ads1, ads2, kw1, kw2, mode, redirect=redirect, redirect_formats=formats, **common)
    plain = PairedFastqTrimmer(ads1, ads2, plain_equivalent(kw1, redirect), plain_equivalent(kw2, redirect), mode,
                               **common)
    got = split.process_chunk_split(data1, data2)
    exp, c1, c2 = RO.redirect_trim_paired(data1, data2, *descs_of(ads1), *descs_of(ads2),
                                          fastq_case_kwargs(options["options1"]), fastq_case_kwargs(options["options2"]),
                                          mode, redirect, formats, input_format, output_format)
    assert set(got) == {"output", *redirect}
    for name in got:
        assert got[name] == exp[name], name
    for st, cc in zip(split.statistics, (c1, c2)):
        for k, v in cc.items():
            assert st[k] == v, k
    assert got["output"] == plain.process_chunk(data1, data2)
    for a, b in zip(split.statistics, plain.statistics):
        assert without_out_bytes(a) == without_out_bytes(b)
    for (v1, l1, k1), (v2, l2, k2) in zip(split.statistics_vector(), plain.statistics_vector()):
        assert (l1, k1) == (l2, k2) and np.array_equal(v1, v2)
    # several pairs in flight
    results = list(split.process_chunks_split([(data1, data2), (b"", b""), (data1, data2)]))
    assert results[0] == got == results[2]
    assert results[1] == {k: (b"", b"") for k in got}


# ---- the C entry points --------------------------------------------------------------------------------------------

def submit(ctx, data):
    buf = np.frombuffer(data, dtype=np.uint8)
    slot = C.c_int32(-1)
    _lib.check(_lib.lib().cg_fastq_submit(ctx.handle, buf.ctypes.data if buf.size else None, buf.size, C.byref(slot)))
    return slot.value, buf


def collect_split(t, data, params, redirect, fasta_outputs, capacity=None):
    slot, buf = submit(t.ctx, data)
    out = np.zeros(capacity if capacity is not None else 2 * len(data) + 64, dtype=np.uint8)
    res = _lib.cg_fastq_result()
    seg = np.full(5, -1, dtype=np.int64)
    rc = _lib.lib().cg_fastq_collect_split(t.ctx.handle, slot, t._set.handle, C.byref(params), redirect, fasta_outputs,
                                           out.ctypes.data, out.size, C.byref(res), seg.ctypes.data)
    return rc, out, res, seg


def collect_plain(t, data, params):
    slot, buf = submit(t.ctx, data)
    out = np.zeros(2 * len(data) + 64, dtype=np.uint8)
    res = _lib.cg_fastq_result()
    _lib.check(_lib.lib().cg_fastq_collect(t.ctx.handle, slot, t._set.handle, C.byref(params), out.ctypes.data,
                                           out.size, C.byref(res)))
    return out, res


def test_redirect_zero_is_the_collect_and_launch_counts():
    data = synthetic_fastq(3000, seed=600)
    t = FastqTrimmer(fastq_case_adapters(BASE), quality_cutoff=(5, 20), minimum_length=40, maximum_length=140)
    ctx = t.ctx
    n0 = ctx.launch_count()
    out_p, res_p = collect_plain(t, data, t.params)
    n1 = ctx.launch_count()
    rc, out_s, res_s, seg = collect_split(t, data, t.params, 0, 0)
    n2 = ctx.launch_count()
    assert rc == 0
    assert bytes(res_p) == bytes(res_s)
    assert list(seg) == [0] + [res_p.out_bytes] * 4
    assert out_s[:res_s.out_bytes].tobytes() == out_p[:res_p.out_bytes].tobytes()
    # the partition replaces the plain offset scan (5 launches instead of 3); one writer per format present
    assert n2 - n1 == (n1 - n0) + 2
    rc, _, _, seg = collect_split(t, data, t.params, 7, 0b101)
    n3 = ctx.launch_count()
    assert rc == 0 and seg[2] > seg[1] and seg[3] > seg[2] and seg[4] > seg[3]
    assert n3 - n2 == (n1 - n0) + 3
    # the plain collect launches what it launched before
    collect_plain(t, data, t.params)
    assert ctx.launch_count() - n3 == n1 - n0


def test_invalid_arguments():
    data = synthetic_fastq(500, seed=601)
    t = FastqTrimmer(fastq_case_adapters(BASE), minimum_length=40)
    with pytest.raises(ValueError):
        FastqTrimmer(fastq_case_adapters(BASE), discard_trimmed=True, redirect=("untrimmed",))
    with pytest.raises(ValueError):
        FastqTrimmer(fastq_case_adapters(BASE), input_format="fasta", redirect=("too_short",),
                     redirect_formats=dict(too_short="fastq"))
    with pytest.raises(ValueError):
        FastqTrimmer(fastq_case_adapters(BASE), redirect=("untrimmed",)).process_chunk_demux(data)
    # CG_EINVAL from the library itself
    p = _fastq_params(discard_trimmed=True)
    assert collect_split(t, data, p, _lib.CG_REDIRECT_UNTRIMMED, 0)[0] == _lib.CG_EINVAL
    p = _fastq_params(minimum_length=40, input_format="fasta")
    fasta = as_fasta(data)
    assert collect_split(t, fasta, p, _lib.CG_REDIRECT_TOO_SHORT, 0)[0] == _lib.CG_EINVAL
    assert collect_split(t, fasta, p, _lib.CG_REDIRECT_TOO_SHORT, _lib.CG_REDIRECT_TOO_SHORT)[0] == 0
    assert collect_split(t, data, t.params, 8, 0)[0] == _lib.CG_EINVAL
    # too small a buffer: the call says how much it needs; with that much it succeeds
    rc, _, res, _ = collect_split(t, data, t.params, 7, 0, capacity=100)
    assert rc == _lib.CG_EINVAL and res.out_bytes > 100
    need = res.out_bytes
    rc, _, res, seg = collect_split(t, data, t.params, 7, 0, capacity=need)
    assert rc == 0 and res.out_bytes == need == seg[4]
    # the context stays usable
    assert FastqTrimmer(fastq_case_adapters(BASE), minimum_length=40, redirect=ALL).process_chunk_split(data)
