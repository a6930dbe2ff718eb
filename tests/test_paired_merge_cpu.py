"""read_merger.pl's rules (tests/paired.py) against the script's recorded output on crafted mate files, and the
argument checks of `classify --paired`, which run before any device call."""
import os
import subprocess

import pytest

from krakenuniq_b200 import build
from tests import paired

FQ = paired.fastq_bytes
FA = paired.fasta_bytes


def _fq_pairs(ids1, ids2, seqs=(b"ACGTAC", b"GGTTAA", b"CATCAT", b"TTTGGG", b"AACCGG")):
    return FQ([(i, s) for i, s in zip(ids1, seqs)]), FQ([(i, s[::-1]) for i, s in zip(ids2, seqs)])


CASES = {
    # ids with /1 /2, _1 _2, .1 .2, none, and suffixes that are not stripped
    "fq_suffixes": (*_fq_pairs([b"a/1", b"b_1", b"c.1", b"d", b"e/3"], [b"a/2", b"b_2", b"c.2", b"d", b"e/3"]), False),
    "fq_extra_words": (*_fq_pairs([b"a/1 x y", b"b/1\tz", b"c"], [b"a/2 q", b"b/2", b"c w"]), True),
    "fa_multiline": (FA([(b"a/1", b"ACGTACGTACGTAC"), (b"b/1", b"GGG"), (b"c/1", b"T" * 23)], width=5),
                     FA([(b"a/2", b"TTTTT"), (b"b/2", b"CCCCCCCCCCCC"), (b"c/2", b"A")], width=4), True),
    "fq_crlf": (*[FQ(r, crlf=True) for r in ([(b"a/1", b"ACGT"), (b"b/1", b"GG")], [(b"a/2", b"TT"), (b"b/2", b"CCA")])], True),
    "fa_crlf": (*[FA(r, width=3, crlf=True) for r in ([(b"a/1", b"ACGTACG"), (b"b/1", b"GG")], [(b"a/2", b"TT"), (b"b/2", b"CCAAT")])], True),
    "empty_mate_seq": (FQ([(b"a/1", b""), (b"b/1", b"ACG")]), FQ([(b"a/2", b"TTT"), (b"b/2", b"")]), False),
    "fa_empty_mate_seq": (FA([(b"a", b""), (b"b", b"ACG")]), FA([(b"a", b"TTT"), (b"b", b"")]), False),
    # a blank line where a FASTQ header should be ends that file; what follows it is never read
    "fq_trailing_blank_line": (FQ([(b"a/1", b"ACGT"), (b"b/1", b"GGA")]) + b"\n" + FQ([(b"c/1", b"TT")]),
                               FQ([(b"a/2", b"TT"), (b"b/2", b"CC"), (b"c/2", b"AA")]) + b"\n", False),
    "file1_longer": (*_fq_pairs([b"a/1", b"b/1", b"c/1", b"d/1"], [b"a/2", b"b/2"]), True),
    "file2_longer": (FA([(b"a/1", b"ACGT")]), FA([(b"a/2", b"GG"), (b"b/2", b"TTA"), (b"c/2", b"C")], width=2), False),
    "check_names_pass": (*_fq_pairs([b"a/1", b"b_1", b"c.1"], [b"a/2", b"b_2", b"c.2"]), True),
    "check_names_fail": (*_fq_pairs([b"a/1", b"b/1", b"c/1", b"d/1"], [b"a/2", b"b/2", b"x/2", b"d/2"]), True),
    "check_names_off": (*_fq_pairs([b"a/1", b"b/1", b"c/1", b"d/1"], [b"a/2", b"b/2", b"x/2", b"d/2"]), False),
    "malformed_header_file1": (*_fq_pairs([b"a/1", b" b/1", b"c/1"], [b"a/2", b"b/2", b"c/2"]), False),
    "malformed_header_file2": (*_fq_pairs([b"a/1", b"b/1", b"c/1"], [b"a/2", b"b/2", b""]), False),
    "fa_malformed_header": (FA([(b"a", b"AC"), (b"b", b"GT")]), FA([(b"a", b"TT"), (b" b", b"CC")]), False),
    # quality lines are skipped unread, whatever their first character
    "quality_line_starts_with_at": (b"@a/1\nACGT\n+\n@III\n@b/1\nGG\n+\n@@\n", b"@a/2\nTTTT\n+\n@@@@\n@b/2\nCC\n+\nII\n", True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_merge_rules_match_read_merger(reference, tmp_path, case):
    data1, data2, check = CASES[case]
    (tmp_path / "m1").write_bytes(data1)
    (tmp_path / "m2").write_bytes(data2)
    paired.install_merger()
    r = reference.run_tool(paired.MERGER, (["--check-names"] if check else []) + ["m1", "m2"], cwd=tmp_path)
    want, err = (tmp_path / "merged.fa").read_bytes(), (tmp_path / "merged.err").read_text(errors="replace")
    got, warnings, error = paired.merge(data1, data2, check)
    assert got == want
    assert (error is not None) == (r.returncode != 0), (error, r.returncode, err)
    if error:
        assert error in err, (error, err)
    for w in warnings:
        assert f"mismatched sequence counts - {w}" in err
    assert ("mismatched sequence counts" in err) == bool(warnings)


def test_file1_longer_ends_with_an_empty_record():
    """the merger's loop falls through after the rest of file 1 and writes one record with an empty id and 'N'"""
    got, warnings, error = paired.merge(*CASES["file1_longer"][:2])
    assert got.endswith(b">d\nTTTGGG\n>\nN\n") and warnings == ["file 1 has more reads"] and error is None
    got, _, _ = paired.merge(*CASES["file2_longer"][:2])
    assert got.endswith(b">c\nC\n")


def _classify(args, tmp_path):
    exe = build.build_classify()
    return subprocess.run([exe, "-d", "db.kdb", "-i", "db.idx", "-a", "taxDB"] + args, cwd=tmp_path,
                          capture_output=True, text=True)


@pytest.mark.parametrize("files", [["a.fq"], ["a.fq", "b.fq", "c.fq"], []])
@pytest.mark.parametrize("tool", ["classify", "classifyExact"])
def test_paired_needs_two_files(tmp_path, files, tool):
    exe = os.path.join(os.path.dirname(build.build_classify()), tool)
    r = subprocess.run([exe, "-d", "db.kdb", "-i", "db.idx", "--paired"] + files, cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 64, r.stderr
    assert "--paired requires exactly two filenames" in r.stderr


def test_long_options_keep_the_short_ones(tmp_path):
    """--paired / --check-names are parsed next to the short options; --check-names alone is accepted and ignored, so
    the run gets as far as opening the (missing) database"""
    r = _classify(["--check-names", "-t", "1", "a.fq"], tmp_path)
    assert r.returncode == 71 and "unable to open db.kdb" in r.stderr, r.stderr     # EX_OSERR from the database
    r = _classify(["--paired", "--check-names", "-t", "1", "a.fq", "b.fq"], tmp_path)
    assert r.returncode == 71 and "unable to open db.kdb" in r.stderr, r.stderr
    r = _classify(["--pared", "a.fq", "b.fq"], tmp_path)
    assert r.returncode == 64 and "Usage" in r.stderr
