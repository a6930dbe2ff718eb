"""`classify --sample-sheet`: the checks of the sheet that run before any database is opened.  Every bad sheet exits with
EX_USAGE (64) or EX_NOINPUT (66) and writes nothing; a good one gets as far as opening the (missing) database, EX_OSERR
(71), so these run without a GPU."""
import os
import subprocess

import pytest

from krakenuniq_b200 import build

OUTS = ("a.kraken", "a.report", "b.kraken", "b.report", "a.C", "a.U")


def _run(tmp_path, sheet, extra=(), tool="classify"):
    (tmp_path / "r1.fa").write_bytes(b">r1\nACGTACGTAC\n")
    (tmp_path / "r2.fq").write_bytes(b"@r2\nACGTACGTAC\n+\nIIIIIIIIII\n")
    (tmp_path / "m1.fq").write_bytes(b"@p/1\nACGT\n+\nIIII\n")
    (tmp_path / "m2.fq").write_bytes(b"@p/2\nACGT\n+\nIIII\n")
    (tmp_path / "s.tsv").write_text(sheet)
    exe = os.path.join(os.path.dirname(build.build_classify()), tool)
    r = subprocess.run([exe, "-d", "db.kdb", "-i", "db.idx", "-a", "taxDB", "--sample-sheet", "s.tsv"] + list(extra),
                       cwd=tmp_path, capture_output=True, text=True)
    assert not any((tmp_path / o).exists() for o in OUTS), os.listdir(tmp_path)
    return r


GOOD = "input\toutput\treport\nr1.fa\ta.kraken\ta.report\nr2.fq,r1.fa\tb.kraken\tb.report\n"

BAD = {
    "no_header_input": ("output\treport\na.kraken\ta.report\n", [], 64, "no input column"),
    "unknown_column": ("input\toutput\tsample_id\nr1.fa\ta.kraken\tx\n", [], 64, "unknown column 'sample_id'"),
    "column_twice": ("input\toutput\tinput\nr1.fa\ta.kraken\tr2.fq\n", [], 64, "named twice"),
    "only_comments": ("# a sheet\n\n# nothing else\n", [], 64, "no header line"),
    "no_rows": ("input\toutput\n", [], 64, "no samples"),
    "too_many_cells": ("input\toutput\nr1.fa\ta.kraken\textra\n", [], 64, "more cells"),
    "empty_input": ("input\toutput\n\ta.kraken\n", [], 64, "has no input"),
    "empty_file_in_list": ("input\toutput\nr1.fa,,r2.fq\ta.kraken\n", [], 64, "empty input file name"),
    "paired_without_input2": ("input\toutput\nm1.fq\ta.kraken\n", ["--paired"], 64, "needs an input2 column"),
    "paired_empty_input2": ("input\tinput2\toutput\nm1.fq\t\ta.kraken\n", ["--paired"], 64, "each hold one file"),
    "paired_two_files": ("input\tinput2\toutput\nm1.fq,r2.fq\tm2.fq\ta.kraken\n", ["--paired"], 64, "each hold one file"),
    "input2_without_paired": ("input\tinput2\toutput\nm1.fq\tm2.fq\ta.kraken\n", [], 64, "needs --paired"),
    "unreadable_input": ("input\toutput\nr1.fa\ta.kraken\nmissing.fa\tb.kraken\n", [], 66, "can't read input missing.fa"),
    "directory_input": ("input\toutput\nr1.fa,.\ta.kraken\n", [], 66, "can't read input ."),
    "missing_mate": ("input\tinput2\toutput\nm1.fq\tnope.fq\ta.kraken\n", ["--paired"], 66, "can't read input nope.fq"),
    "duplicate_output": ("input\toutput\nr1.fa\ta.kraken\nr2.fq\ta.kraken\n", [], 64, "both write a.kraken"),
    "duplicate_across_columns": ("input\toutput\treport\nr1.fa\ta.kraken\ta.report\nr2.fq\tb.kraken\t./a.kraken\n", [], 64,
                                 "both write ./a.kraken"),
    "output_is_input": ("input\toutput\nr1.fa\ta.kraken\nr2.fq\t./r1.fa\n", [], 64, "writes to one of the inputs"),
    "report_is_sheet": ("input\treport\nr1.fa\ts.tsv\n", [], 64, "writes to one of the inputs"),
    "with_o": (GOOD, ["-o", "a.kraken"], 64, "-o, -r, -C and -U"),
    "with_r": (GOOD, ["-r", "a.report"], 64, "-o, -r, -C and -U"),
    "with_C": (GOOD, ["-C", "a.C"], 64, "-o, -r, -C and -U"),
    "with_U": (GOOD, ["-U", "a.U"], 64, "-o, -r, -C and -U"),
    "with_positional_input": (GOOD, ["r1.fa"], 64, "no input files on the command line"),
}


@pytest.mark.parametrize("tool", ["classify", "classifyExact"])
@pytest.mark.parametrize("case", list(BAD))
def test_bad_sheet_is_refused_before_the_database(tmp_path, case, tool):
    sheet, extra, status, message = BAD[case]
    r = _run(tmp_path, sheet, extra, tool)
    assert r.returncode == status and message in r.stderr, r.stderr
    assert "Database" not in r.stderr


def test_missing_sheet(tmp_path):
    exe = build.build_classify()
    r = subprocess.run([exe, "-d", "db.kdb", "-i", "db.idx", "--sample-sheet", "none.tsv"], cwd=tmp_path,
                       capture_output=True, text=True)
    assert r.returncode == 66 and "can't open the sample sheet none.tsv" in r.stderr


@pytest.mark.parametrize("sheet,extra", [
    (GOOD, []),
    ("# comment\n\ninput\tname\toutput\r\n\n# skipped\nr1.fa\tfirst\r\nr2.fq\n", []),     # CRLF, short rows, blank lines
    ("name\tinput2\tinput\tclassified_out\tunclassified_out\np1\tm2.fq\tm1.fq\ta.C\ta.U\n", ["--paired", "--check-names"]),
    (GOOD, ["-M", "-t", "1", "-u", "20000", "-q", "-m", "2", "-c", "-s", "-p", "12", "-x", "40K"]),
])
def test_good_sheet_reaches_the_database(tmp_path, sheet, extra):
    r = _run(tmp_path, sheet, extra)
    assert r.returncode == 71 and "unable to open db.kdb" in r.stderr, r.stderr
