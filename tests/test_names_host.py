"""
The read-name modifiers of the FASTQ path on the host: the hostsim build of cutadapt_b200/csrc/cg_names_core.cuh (both
steps of the name stage, the -u parts, parse_name) against tests/names_oracle.py, which restates the reference's
modifiers; the template and tag refusals of the trimmers and the argument errors of tools/trim_fastq.py.
"""
import ctypes as C
import os
import random
import subprocess
import sys

import pytest

import names_oracle as no
from util import hostsim_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cutadapt_b200 import pipeline  # noqa: E402

KINDS = dict(header=1, id=2, comment=3, cut_prefix=4, cut_suffix=5, adapter_name=6, rc=7, match_sequence=8, rn=9)


def _lib():
    lib = hostsim_lib()
    lib.hs_names_pre.restype = C.c_int64
    lib.hs_names_rename.restype = C.c_int64
    return lib


def device_pre(name, length, adapter=None, tag=None, strips=(), prefix="", suffix="", rc=False):
    lib = _lib()
    arr = (C.c_char_p * max(len(strips), 1))(*[s.encode() for s in strips])
    out = C.create_string_buffer(4096)
    hdr = name.encode()
    n = lib.hs_names_pre(tag.encode() if tag is not None else None, arr, len(strips), prefix.encode(), suffix.encode(),
                         hdr, len(hdr), int(rc), length, (adapter if adapter is not None else "no_adapter").encode(),
                         out, C.c_int64(4096))
    return out.raw[:n].decode()


def device_rename(template, infos, names, rn=1, paired=False):
    """infos / names: the record's own, R1's, R2's"""
    lib = _lib()
    toks = pipeline.rename_tokens(template, paired)
    kinds = (C.c_int32 * len(toks))(*[t[0] for t in toks])
    mates = (C.c_int32 * len(toks))(*[t[1] for t in toks])
    texts = (C.c_char_p * len(toks))(*[t[2].encode() for t in toks])
    strs, flags = [], []
    for info, name in zip(infos, names):
        ms = info.get("match_sequence", "") if info.get("adapter") is not None else ""
        front, back, linked = (ms.split(",", 1) + [""])[:2] + [0]
        if "," in ms and info.get("linked"):
            linked = 1
        else:
            front, back = ms, ""
        strs += [name, info.get("cut_prefix", ""), info.get("cut_suffix", ""),
                 info.get("adapter") if info.get("adapter") is not None else "no_adapter", front, back]
        flags += [linked, int(bool(info.get("is_rc")))]
    vs = (C.c_char_p * 18)(*[x.encode() for x in strs])
    fl = (C.c_int32 * 6)(*flags)
    out = C.create_string_buffer(4096)
    n = lib.hs_names_rename(kinds, mates, texts, len(toks), vs, fl, rn, out, C.c_int64(4096))
    return out.raw[:n].decode()


WS = [" ", "\t", "\x0b", "\x0c", "\x1c", "\x1d", "\x1e", "\x1f", "\r"]


def random_name(rng):
    parts = []
    for _ in range(rng.randint(0, 5)):
        parts.append(rng.choice(["read", "length=", "length=12", "12ab", "x", "/1", "_", "=", "length=7x", ";", "a b",
                                 rng.choice(WS), "len", "length", "length=3.5"]))
    return "".join(parts)


@pytest.mark.parametrize("seed", range(4))
def test_pre_name_against_oracle(seed):
    rng = random.Random(seed)
    for _ in range(400):
        name = random_name(rng)
        tag = rng.choice([None, "length=", "length", "x", "=", "_1", "12"])
        strips = rng.sample(["/1", "", "x", "length=", " ", name], rng.randint(0, 2))
        prefix, suffix = rng.choice([("", ""), ("{name}_", ""), ("", " {name}"), ("p{name}{name}", "{nam}s")])
        adapter = rng.choice([None, "ad1", "linked"])
        length = rng.randint(0, 300)
        want = no.pre_name(name, length, adapter, tag, strips, prefix, suffix)
        assert device_pre(name, length, adapter, tag, strips, prefix, suffix) == want, (name, tag, strips)


def test_pre_name_edges():
    assert device_pre("r length=12ab", 150, tag="length=") == "r length=15012ab"
    assert device_pre("r length=12 length=3", 7, tag="length=") == "r length=7 length=7"
    assert device_pre("a=5", 9, tag="=") == "a=9"          # a non-word first character needs a word character before it
    assert device_pre("=5", 9, tag="=") == "=5"
    assert device_pre("read", 4, strips=["read"]) == ""     # a suffix equal to the whole name
    assert device_pre("read", 4, strips=[""]) == ""         # name[:-0]
    assert device_pre("r", 1, rc=True, suffix="_{name}") == "r rc_no_adapter"


@pytest.mark.parametrize("name", ["", " ", "a", "a ", " a", "a b", "a  b c ", "\ta\x1fb", "a\x0bb", "a\x1c", "x\r y"])
def test_parse_name(name):
    lib = _lib()
    out = (C.c_int32 * 4)()
    b = name.encode()
    lib.hs_names_split(b, len(b), out)
    assert (name[out[0]:out[0] + out[1]], name[out[2]:out[2] + out[3]]) == no.parse_name(name)


TEMPLATES = ["{header}", "{id} {comment}", "{id}\\t{adapter_name}", "{cut_prefix}_{cut_suffix} {id}", "{id} {rc}",
             "{match_sequence}-{id}", "{header}{header} {match_sequence}", "x"]


@pytest.mark.parametrize("template", TEMPLATES)
def test_rename_against_oracle(template):
    rng = random.Random(template)
    for _ in range(200):
        name = random_name(rng)
        info = dict(adapter=rng.choice([None, "a1"]), match_sequence=rng.choice(["", "ACGT"]),
                    cut_prefix=rng.choice(["", "NN"]), cut_suffix=rng.choice(["", "T"]), is_rc=rng.random() < 0.5)
        assert device_rename(template, [info] * 3, [name] * 3) == no.rename(template, name, info)


def test_rename_linked_match_sequence():
    info = dict(adapter="lk", match_sequence="AC,GT", linked=True)
    assert device_rename("{match_sequence}", [info] * 3, ["r"] * 3) == "AC,GT"
    info = dict(adapter="lk", match_sequence=",GT", linked=True)
    assert device_rename("{match_sequence}", [info] * 3, ["r"] * 3) == ",GT"


@pytest.mark.parametrize("template", ["{id} {r1.comment} {r2.comment} {rn}", "{r1.adapter_name}_{r2.cut_prefix} {id}",
                                      "{r2.header}\\t{rn}", "{id} {r1.match_sequence}"])
def test_paired_rename_against_oracle(template):
    rng = random.Random(template)
    for _ in range(100):
        n1, n2 = "read/1 " + random_name(rng), "read/2 " + random_name(rng)
        i1 = dict(adapter=rng.choice([None, "a1"]), match_sequence="AC", cut_prefix=rng.choice(["", "G"]))
        i2 = dict(adapter=rng.choice([None, "b"]), match_sequence="T")
        w1, w2 = no.rename_pair(template, n1, n2, i1, i2)
        assert device_rename(template, [i1, i1, i2], [n1, n1, n2], 1, True) == w1
        assert device_rename(template, [i2, i1, i2], [n2, n1, n2], 2, True) == w2


@pytest.mark.parametrize("cut", [(3,), (-2,), (2, 3), (-1, -2), (4, -3), (10,), (-10,), (2, -9), ()])
@pytest.mark.parametrize("rc", [False, True])
def test_cut_parts(cut, rc):
    lib = _lib()
    read = "ACGTTGCAAC"
    comp = str.maketrans("ACGT", "TGCA")
    stored = read.translate(comp)[::-1] if rc else read
    front = [c for c in cut if c > 0]
    back = [-c for c in cut if c < 0]
    out = C.create_string_buffer(64)
    lens = (C.c_int32 * 2)()
    lib.hs_names_cut(stored.encode(), len(read), int(rc), sum(front), sum(back), front[-1] if front else 0,
                     back[-1] if back else 0, out, lens)
    got = out.raw[:lens[0] + lens[1]].decode()
    want = no.cut_parts(read, cut)
    assert (got[:lens[0]], got[lens[0]:]) == (want.get("cut_prefix", ""), want.get("cut_suffix", ""))


@pytest.mark.parametrize("template,paired,message", [
    ("{id", False, "Error in template '{id': Unexpected '{' encountered"),
    ("id}", False, "Error in template 'id}': Unexpected '}' encountered"),
    ("{idx}", False, "Error in template: Variable 'idx' not recognized"),
    ("{rn}", False, "Error in template: Variable 'rn' not recognized"),
    ("{r1.id}", True, "Error in template: Variable 'r1.id' not recognized"),
    ("{rc}", True, "Error in template: Variable 'rc' not recognized"),
    ("a\\t{", False, "Error in template 'a\t{': Unexpected '{' encountered"),
    ("a\\t{", True, "Error in template 'a\\t{': Unexpected '{' encountered"),
])
def test_template_refusals(template, paired, message):
    with pytest.raises(ValueError) as e:
        pipeline.rename_tokens(template, paired)
    assert str(e.value) == message


@pytest.mark.parametrize("tag", ["", "len.", "a b", "x*", "(a)", "a\\d", "é"])
def test_length_tag_refusals(tag):
    with pytest.raises(ValueError):
        pipeline.check_length_tag(tag)


def test_length_tag_accepted():
    pipeline.check_length_tag("length=_:,;/-@#%!~Ab9")


def _tool(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py"), *args], capture_output=True,
                          text=True)


def test_tool_rename_with_prefix_is_refused(tmp_path):
    r = _tool("--rename", "{id}", "-x", "p", "-o", str(tmp_path / "o.fastq"), str(tmp_path / "in.fastq"))
    assert r.returncode == 2
    assert "Option --rename cannot be combined with --prefix (-x) or --suffix (-y)" in r.stderr


def test_tool_documents_name_flags():
    r = _tool("--help")
    for flag in ("--rename", "--prefix", "--suffix", "--strip-suffix", "--length-tag"):
        assert flag in r.stdout


# ---- the reference's known answers (tests/golden/names_kat.json.gz) ----------------------------------------------------

def _kat():
    from util import golden

    return golden("names_kat.json.gz")


def test_kat_length_tag():
    for name, tag, length, want in _kat()["edges"]["length_tag"]:
        assert device_pre(name, length, tag=tag) == want, (name, tag)


def test_kat_strip_suffix():
    for name, suffix, want in _kat()["edges"]["strip_suffix"]:
        assert device_pre(name, 0, strips=[suffix]) == want, (name, suffix)


def test_kat_prefix_suffix():
    for name, prefix, suffix, adapter, want in _kat()["edges"]["affix"]:
        assert device_pre(name, 0, adapter, prefix=prefix, suffix=suffix) == want, (name, prefix, suffix)


def test_kat_parse_name():
    lib = _lib()
    out = (C.c_int32 * 4)()
    for name, id_, comment in _kat()["edges"]["parse_name"]:
        b = name.encode()
        lib.hs_names_split(b, len(b), out)
        assert (name[out[0]:out[0] + out[1]], name[out[2]:out[2] + out[3]]) == (id_, comment), name


def _mates_match(a: str, b: str) -> bool:
    lib = hostsim_lib()
    blob = (a + b).encode()
    off = (C.c_int64 * 3)(0, len(a.encode()), len(blob))
    out = (C.c_int32 * 1)()
    lib.hs_mates_match(C.c_int64(1), blob, off, out)
    return bool(out[0])


def test_kat_renamer_cases():
    for case in _kat()["modifiers"]:
        reads = case["reads"]
        if not case["paired"]:
            (name, info), = reads
            assert device_rename(case["template"], [info] * 3, [name] * 3) == case["expected"][0], case
            continue
        (n1, i1), (n2, i2) = reads
        got = [device_rename(case["template"], [i1, i1, i2], [n1, n1, n2], 1, True),
               device_rename(case["template"], [i2, i1, i2], [n2, n1, n2], 2, True)]
        if case["expected"] is None:            # PairedEndRenamer refuses the pair: the new IDs are not mates
            assert not _mates_match(*got), case
        else:
            assert got == case["expected"], case
            assert _mates_match(*got)
