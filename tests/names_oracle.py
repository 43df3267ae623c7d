"""
The reference's read-name modifiers restated on plain strings (test infrastructure): LengthTagModifier, SuffixRemover,
PrefixSuffixAdder (modifiers.py:529-588), Renamer and PairedEndRenamer (modifiers.py:595-760) in the chain order of
cli.py:937-991 and 1136-1146.  names() composes them onto the records a collect without name options wrote, given what
the reference's ModificationInfo would hold for each read (its last match's adapter name and match sequence, the -u
parts, is_rc); tests/test_gpu_names.py takes those from the info rows of the same collect.
"""
import re


def length_tag(name: str, tag: str, length: int) -> str:
    if name.find(tag) >= 0:
        name = re.sub(r"\b" + tag + r"[0-9]*\b", tag + str(length), name)
    return name


def strip_suffix(name: str, suffix: str) -> str:
    return name[: -len(suffix)] if name.endswith(suffix) else name


def parse_name(name: str):
    fields = name.split(maxsplit=1)
    return (fields[0], fields[1]) if len(fields) == 2 else (name, "")


def pre_name(name: str, length: int, adapter=None, tag=None, strips=(), prefix="", suffix="") -> str:
    """The name after LengthTagModifier, the SuffixRemovers and PrefixSuffixAdder (adapter None: no match)."""
    if tag:
        name = length_tag(name, tag, length)
    for s in strips:
        name = strip_suffix(name, s)
    if prefix or suffix:
        a = adapter if adapter is not None else "no_adapter"
        name = prefix.replace("{name}", a) + name + suffix.replace("{name}", a)
    return name


def _values(name, info):
    return dict(header=name, comment=parse_name(name)[1], cut_prefix=info.get("cut_prefix", ""),
                cut_suffix=info.get("cut_suffix", ""),
                adapter_name=info.get("adapter") if info.get("adapter") is not None else "no_adapter",
                match_sequence=info.get("match_sequence", "") if info.get("adapter") is not None else "")


def rename(template: str, name: str, info: dict) -> str:
    """Renamer: info holds adapter (None: no match), match_sequence, cut_prefix, cut_suffix, is_rc."""
    template = template.replace(r"\t", "\t")
    v = _values(name, info)
    return template.format(id=parse_name(name)[0], rc="rc" if info.get("is_rc") else "", **v)


class _NS:
    def __init__(self, d):
        self.__dict__.update(d)


def rename_pair(template: str, name1: str, name2: str, info1: dict, info2: dict):
    """PairedEndRenamer: (new name 1, new name 2), or ValueError when the new IDs no longer name mates."""
    template = template.replace(r"\t", "\t")
    d1, d2 = _values(name1, info1), _values(name2, info2)
    n1 = template.format(id=parse_name(name1)[0], rn=1, **d1, r1=_NS(d1), r2=_NS(d2))
    n2 = template.format(id=parse_name(name2)[0], rn=2, **d2, r1=_NS(d1), r2=_NS(d2))
    if not mates_match(n1, n2):
        raise ValueError("After renaming R1 and R2, their IDs are no longer identical: "
                         f"'{parse_name(n1)[0]}' != '{parse_name(n2)[0]}'. Original read ID: '{parse_name(name1)[0]}'. ")
    return n1, n2


def mates_match(a: str, b: str) -> bool:
    """dnaio's record_names_match: IDs up to the first space or tab, a final 1 / 2 / 3 of both ignored."""
    i1 = re.split("[ \t]", a, maxsplit=1)[0]
    i2 = re.split("[ \t]", b, maxsplit=1)[0]
    if i1 and i2 and i1[-1] in "123" and i2[-1] in "123":
        i1, i2 = i1[:-1], i2[:-1]
    return i1 == i2


def cut_parts(read: str, cut) -> dict:
    """cut_prefix / cut_suffix of UnconditionalCutter, one per -u value, the 5' values first."""
    info = {}
    for c in [c for c in cut if c > 0] + [c for c in cut if c < 0]:
        if c > 0:
            info["cut_prefix"], read = read[:c], read[c:]
        else:
            info["cut_suffix"], read = read[c:], read[:c]
    return info
