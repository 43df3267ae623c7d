"""
The per-read row outputs of pairs without a GPU: the paired oracle reproduces the reference's paired info files
(tests/golden/paired_rows_kat.json.gz, test_info_file.py::test_paired_info_file) and its two outputs, its rows of each
mate are those of that mate trimmed alone (with --pair-adapters: named by the pair's adapter of that mate's list), the
Python options of the row outputs are checked, and tools/trim_fastq.py refuses the row-file command lines the reference
refuses.
"""
import os
import subprocess
import sys

import pytest

import fasta_oracle as FO
import rows_oracle as RW
from oracle import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case():
    kat = RW.paired_rows_kat()
    assert [c["name"] for c in kat["cases"]] == ["paired_info_file"]
    return kat, kat["cases"][0]


def test_the_paired_oracle_reproduces_the_paired_info_files():
    kat, c = _case()
    o = c["options"]
    data1, data2 = (RW.kat_bytes(kat, k) for k in c["inputs"])
    out1, out2, c1, c2, rows1, rows2 = RW.oracle_rows_paired(
        oracle, data1, data2, FO.kat_adapters(o, "specs1"), FO.kat_adapters(o, "specs2"), o["options1"], o["options2"],
        kinds1=("info",), kinds2=("info",))
    want_out = [RW.kat_bytes(kat, k) for k in c["expected"]["output"]]
    want_info = [RW.kat_bytes(kat, k) for k in c["expected"]["info"]]
    assert (out1, out2) == tuple(want_out)
    assert RW.strip_trailing(rows1["info"]) == RW.strip_trailing(want_info[0])
    assert RW.strip_trailing(rows2["info"]) == RW.strip_trailing(want_info[1])
    # rows of every read, filtered or not: the -m 14 filter removes pairs, their rows stay
    n_reads = data1.count(b"\n") // 4
    assert c1["n_written"] < n_reads
    assert {line.split(b"\t")[0].split(b"/")[0] for line in rows1["info"].splitlines()} == \
        {line[1:].split(b"/")[0].split(b" ")[0] for line in data1.splitlines()[0::4]}


def test_the_rows_of_a_mate_are_those_of_the_mate_alone():
    """oracle_fastq_trim_paired passes each mate's row options on unchanged: R1's rows (and R2's) equal those of the
    mate trimmed as single-end data with the same options."""
    kat, c = _case()
    o = c["options"]
    data1, data2 = (RW.kat_bytes(kat, k) for k in c["inputs"])
    ads1, ads2 = FO.kat_adapters(o, "specs1"), FO.kat_adapters(o, "specs2")
    kw = dict(quality_trim=True, cutoff_front=0, cutoff_back=20, cut=(2, -1), times=2)
    _, _, _, _, rows1, rows2 = RW.oracle_rows_paired(oracle, data1, data2, ads1, ads2, kw, kw, kinds1=RW.KINDS,
                                                     kinds2=RW.KINDS)
    assert rows1 == RW.oracle_rows_single(oracle, data1, ads1, kw)[2]
    _, _, single2 = RW.oracle_rows_single(oracle, data2, ads2, dict(kw, second_mate=True))
    assert rows2 == single2


def test_pair_adapter_rows_name_each_mates_own_adapter():
    """--pair-adapters: `adapter` of the match records is the pair number, so R1's rows name adapter i of -a and R2's
    adapter i of -A; a pair without a match on both mates gets the "-1" row on both."""
    import cutadapt_b200.adapters as PA

    kat, c = _case()
    data1, data2 = (RW.kat_bytes(kat, k) for k in c["inputs"])
    ads1 = [PA.BackAdapter("TTAGACATAT", name="r1adapt"), PA.BackAdapter("GGGGGGGGGG", name="r1other")]
    ads2 = [PA.BackAdapter("CAGTGGAGTA", name="r2adapt"), PA.BackAdapter("CCCCCCCCCC", name="r2other")]
    kw = dict(quality_trim=True, cutoff_front=0, cutoff_back=20, cut=(1,))
    _, _, _, _, rows1, rows2 = RW.oracle_rows_paired(oracle, data1, data2, ads1, ads2, kw, kw, kinds1=("info",),
                                                     kinds2=("info",), pair_adapters=True)
    lines1, lines2 = rows1["info"].splitlines(), rows2["info"].splitlines()
    assert len(lines1) == len(lines2) == data1.count(b"\n") // 4
    matched = 0
    for a, b in zip(lines1, lines2):
        fa, fb = a.split(b"\t"), b.split(b"\t")
        assert (fa[1] == b"-1") == (fb[1] == b"-1")
        if fa[1] != b"-1":
            matched += 1
            assert (fa[7], fb[7]) in ((b"r1adapt", b"r2adapt"), (b"r1other", b"r2other"))
    assert matched > 0


def test_row_options_are_checked():
    from cutadapt_b200 import pipeline as P

    assert P._row_kinds(("info", "rest", "info"), ("rest",)) == (("info", "rest"), ("rest",))
    with pytest.raises(ValueError, match="unknown row output"):
        P._row_kinds(("infos",), ())
    with pytest.raises(ValueError, match="not in rows"):
        P._row_kinds(("info",), ("rest",))
    blob, off = P._row_text(None, "info")
    assert blob == b"" and off.tolist() == [0]


def test_row_text_of_each_kind():
    import cutadapt_b200.adapters as PA
    from cutadapt_b200 import pipeline as P

    ads = PA.MultipleAdapters([PA.BackAdapter("ACGTNNAC", name="one"), PA.FrontAdapter("GGTTA", name="two")])
    assert P._row_text(ads, "info")[0] == b"onetwo"
    assert P._row_text(ads, "info")[1].tolist() == [0, 3, 6]
    assert P._row_text(ads, "rest")[1].tolist() == [0, 0, 0]
    assert P._row_text(ads, "wildcard")[0] == b"ACGTNNACGGTTA"
    pairs = [PA.BackAdapter("AAAAC", name="p1"), PA.BackAdapter("CCCCA", name="p2")]
    assert P._row_text(pairs, "info", pair_list=True)[0] == b"p1p2"


def _tool(args, tmp_path):
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "trim_fastq.py")] + args, capture_output=True,
                          text=True, cwd=str(tmp_path))


def test_tool_refuses_info_file_paired_with_one_input(tmp_path):
    """--info-file-paired enables paired-end mode (cli.py:525-538): one input without --interleaved is refused with
    the reference's message (cli.py:560-566)."""
    kat, _ = _case()
    inp = tmp_path / "in.fastq"
    inp.write_bytes(RW.kat_bytes(kat, "data/paired.1.fastq"))
    r = _tool(["-a", "TTAGACATAT", "--info-file", "i1.txt", "--info-file-paired", "i2.txt", "-o", "out.fastq",
               str(inp)], tmp_path)
    assert r.returncode == 2, r.stderr
    assert "enables paired-end mode" in r.stderr and "only provided one input file" in r.stderr


@pytest.mark.parametrize("flag", ["--info-file", "--rest-file", "--wildcard-file"])
def test_tool_refuses_row_files_on_standard_output(flag, tmp_path):
    kat, _ = _case()
    inp = tmp_path / "in.fastq"
    inp.write_bytes(RW.kat_bytes(kat, "data/paired.1.fastq"))
    r = _tool(["-a", "TTAGACATAT", flag, "-", "-o", "out.fastq", str(inp)], tmp_path)
    assert r.returncode == 2 and "standard output" in r.stderr
