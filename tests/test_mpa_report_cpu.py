"""krakenuniq-mpa-report's rules (tests/mpa_report.py) against the script's recorded output on a crafted taxonomy and
crafted Kraken lines, the golden mini run's recorded table, and the argument checks of `classify --mpa-report` /
`--translate-out`, which run before any database file is opened."""
import itertools
import os
import shutil
import subprocess

import pytest

from krakenuniq_b200 import build
from tests import mpa_report, util

# taxDB rows in file order: every rank code, `no rank`, `clade` and `domain`; names with spaces, '|' and '.'; taxid 20
# with two rows under different parents; a repeated row (9); a parent without a row (999); a chain 40..139 under the
# root with an order and a species at its end; 150 is also a read length of the lines below (the empty-id line)
_ROWS = ([(1, 1, "root", "no rank"), (2, 1, "Bacteria", "superkingdom"), (3, 2, "Terra|bacteria", "kingdom"),
          (4, 3, "Phylum one", "phylum"), (5, 4, "Class.A", "class"), (6, 5, "Order x", "order"), (7, 6, "Fam ily", "family"),
          (8, 7, "Genus g.", "genus"), (9, 8, "Genus g. species one", "species"), (10, 8, "Genus g. sp|two", "species"),
          (11, 1, "clade node", "clade"), (12, 11, "domain node", "domain"), (13, 12, "Other genus", "genus"),
          (14, 13, "Other species", "species"), (20, 7, "Dup genus", "genus"), (20, 11, "Dup genus moved", "genus"),
          (21, 20, "Dup child", "species"), (9, 8, "Genus g. species one", "species"), (30, 999, "orphan", "species"),
          (150, 8, "length species", "species")] +
         [(40 + i, 1 if i == 0 else 39 + i, f"deep {i}", "order" if i == 60 else "no rank") for i in range(99)] +
         [(139, 138, "deep species", "species")])
TAXDB = b"".join(b"%d\t%d\t%s\t%s\n" % (t, p, n.encode(), r.encode()) for t, p, n, r in _ROWS)


def _lines(rows):
    return b"".join(b"\t".join(f) + b"\n" for f in rows)


# U lines, root-called lines before and after other classified lines and several in a row, taxa without a row (4242),
# a walk that stops at a parent without a row (30), the duplicated taxon, an empty read id, P= columns, a sequence
# column and Q: hit lists
KRAKEN_A = _lines([
    (b"C", b"root_first", b"1", b"100", b"1:5 0:3"),
    (b"C", b"root_again", b"1", b"100", b"1:2"),
    (b"U", b"u1", b"0", b"90", b"0:60"),
    (b"C", b"sp1", b"9", b"150", b"9:10 8:2 0:5"),
    (b"C", b"root_after", b"1", b"120", b"1:3"),
    (b"C", b"root_after2", b"1", b"120", b"1:1"),
    (b"C", b"sp2", b"10", b"150", b"10:1 A:3"),
    (b"C", b"missing", b"4242", b"80", b"4242:2"),
    (b"C", b"missing_again", b"4242", b"80", b"4242:2"),
    (b"C", b"other", b"14", b"150", b"14:4"),
    (b"C", b"dup", b"21", b"150", b"21:3"),
    (b"C", b"orphan", b"30", b"100", b"30:1"),
    (b"C", b"deep", b"139", b"200", b"139:9"),
    (b"C", b"", b"9", b"150", b"9:1"),
    (b"C", b"filtered", b"13", b"150", b"P=0.600", b"13:3 0:2"),
    (b"C", b"with_seq", b"7", b"50", b"7:2", b"ACGTACGTAC"),
    (b"C", b"quick", b"8", b"150", b"Q:3"),
    (b"U", b"u2", b"0", b"40", b"0:10", b"ACGT"),
    (b"C", b"root_end", b"1", b"30", b"1:1"),
    (b"C", b"clade", b"11", b"40", b"11:2"),
    (b"C", b"domain", b"12", b"40", b"12:2"),
])
# the second file starts with root-called lines (the first file's lineages carry over in translate)
KRAKEN_B = _lines([
    (b"C", b"b_root", b"1", b"100", b"1:5"),
    (b"C", b"b_orphan_stop", b"999", b"100", b"999:1"),
    (b"C", b"b_sp", b"14", b"100", b"14:1"),
    (b"C", b"b_root2", b"1", b"100", b"1:5"),
    (b"U", b"b_u", b"0", b"100", b"0:5"),
    (b"C", b"b_deep", b"100", b"100", b"100:5"),
])
KRAKEN_C = _lines([(b"U", b"c_u%d" % i, b"0", b"100", b"0:5") for i in range(3)] +
                  [(b"C", b"c_root", b"1", b"80", b"1:5")])
FILES = {"a.kraken": KRAKEN_A, "b.kraken": KRAKEN_B, "c.kraken": KRAKEN_C}
FLAGS = ["--show-zeros", "--header-line", "--intermediate-ranks"]


def _setup(tmp_path):
    mpa_report.write_db(tmp_path, TAXDB)
    for n, d in FILES.items():
        (tmp_path / n).write_bytes(d)
    mpa_report.install_mpa_report()


@pytest.mark.parametrize("flags", [list(c) for n in range(4) for c in itertools.combinations(FLAGS, n)],
                         ids=lambda f: "+".join(x[2:] for x in f) or "plain")
def test_mpa_rules_match_krakenuniq_mpa_report(reference, tmp_path, flags):
    _setup(tmp_path)
    opts = dict(show_zeros="--show-zeros" in flags, header_line="--header-line" in flags,
                intermediate="--intermediate-ranks" in flags)
    for names in (["a.kraken"], ["a.kraken", "b.kraken", "c.kraken"]):
        r = reference.run_tool(mpa_report.MPA, ["--db", "."] + flags + names, cwd=tmp_path)
        assert r.returncode == 0, r.stderr
        want = mpa_report.mpa_table([FILES[n] for n in names], TAXDB, ids=names, **opts)
        assert want.decode() == r.stdout
        assert want


def test_golden_mini_recorded(reference, tmp_path):
    """the scripts over the golden mini run's Kraken output: the tables and lineages tests/test_mpa_translate_gpu.py
    holds classify's outputs to"""
    from tests import translate
    taxdb = open(os.path.join(util.GOLDEN, "taxDB"), "rb").read()
    mpa_report.write_db(tmp_path, taxdb)
    shutil.copyfile(os.path.join(util.GOLDEN, "preload.kraken"), tmp_path / "preload.kraken")
    kraken = (tmp_path / "preload.kraken").read_bytes()
    mpa_report.install_mpa_report()
    translate.install_translate()
    for flags in ([], FLAGS):
        r = reference.run_tool(mpa_report.MPA, ["--db", "."] + flags + ["preload.kraken"], cwd=tmp_path)
        assert r.returncode == 0, r.stderr
        assert r.stdout.encode() == mpa_report.mpa_table([kraken], taxdb, bool(flags), bool(flags), bool(flags),
                                                         ids=["preload.kraken"])
    for flags in ([], ["--mpa-format"]):
        r = reference.run_tool(translate.TRANSLATE, ["--db", "."] + flags + ["preload.kraken"], cwd=tmp_path)
        assert r.returncode == 0, r.stderr
        assert r.stdout.encode() == translate.translate(kraken, taxdb, bool(flags))


# ---- classify's argument checks: exit status 64 before any database file is opened (db.kdb does not exist) --------
def _classify(args, tmp_path, taxdb=TAXDB):
    (tmp_path / "taxDB").write_bytes(taxdb)
    (tmp_path / "reads.fa").write_bytes(b">r\nACGT\n")
    return subprocess.run([build.build_classify(), "-d", "db.kdb", "-i", "db.idx"] + args, cwd=tmp_path,
                          capture_output=True, text=True)


def _refused(r, what):
    assert r.returncode == 64, r.stderr
    assert what in r.stderr
    assert "unable to open" not in r.stderr


@pytest.mark.parametrize("flag", ["--mpa-show-zeros", "--mpa-header-line", "--mpa-intermediate-ranks"])
def test_mpa_modifier_needs_mpa_report(tmp_path, flag):
    _refused(_classify(["-a", "taxDB", flag, "reads.fa"], tmp_path), "need --mpa-report")


def test_translate_mpa_format_needs_a_translation(tmp_path):
    _refused(_classify(["-a", "taxDB", "--translate-mpa-format", "reads.fa"], tmp_path), "--translate-out")
    (tmp_path / "s.tsv").write_text("input\toutput\nreads.fa\tx.kraken\n")
    _refused(_classify(["-a", "taxDB", "--translate-mpa-format", "--sample-sheet", "s.tsv"], tmp_path), "translate_out column")


@pytest.mark.parametrize("opt", [["--mpa-report", "t.mpa"], ["--translate-out", "t.tr"]])
def test_features_need_the_taxdb(tmp_path, opt):
    _refused(_classify(opt + ["-o", "x.kraken", "reads.fa"], tmp_path), "give it with -a")


def test_translate_out_refused_with_a_sheet(tmp_path):
    (tmp_path / "s.tsv").write_text("input\toutput\nreads.fa\tx.kraken\n")
    _refused(_classify(["-a", "taxDB", "--translate-out", "t.tr", "--sample-sheet", "s.tsv"], tmp_path), "translate_out")


@pytest.mark.parametrize("args,what", [
    (["--mpa-report", "reads.fa", "-o", "x.kraken"], "one of the inputs"),
    (["--translate-out", "reads.fa", "-o", "x.kraken"], "one of the inputs"),
    (["--mpa-report", "x.kraken", "-o", "x.kraken"], "written twice"),
    (["--translate-out", "t", "--mpa-report", "t", "-o", "x.kraken"], "written twice"),
    (["--translate-out", "r.txt", "-r", "r.txt", "-o", "x.kraken"], "written twice"),
    (["--mpa-report", "-"], "standard output"),                       # the Kraken lines go to standard output
    (["--translate-out", "-", "--mpa-report", "-", "-o", "x.kraken"], "standard output"),
    (["--translate-out", "-", "-C", "-", "-o", "x.kraken"], "standard output"),
])
def test_outputs_that_collide(tmp_path, args, what):
    _refused(_classify(["-a", "taxDB"] + args + ["reads.fa"], tmp_path), what)


def test_sheet_outputs_that_collide(tmp_path):
    (tmp_path / "s.tsv").write_text("name\tinput\toutput\ttranslate_out\na\treads.fa\ta.kraken\tt.tr\nb\treads.fa\tb.kraken\tt.tr\n")
    _refused(_classify(["-a", "taxDB", "--sample-sheet", "s.tsv"], tmp_path), "both write t.tr")
    (tmp_path / "s.tsv").write_text("name\tinput\toutput\ttranslate_out\na\treads.fa\ta.kraken\t-\nb\treads.fa\tb.kraken\t-\n")
    _refused(_classify(["-a", "taxDB", "--sample-sheet", "s.tsv"], tmp_path), "standard output")
    (tmp_path / "s.tsv").write_text("name\tinput\toutput\na\treads.fa\ta.kraken\n")
    _refused(_classify(["-a", "taxDB", "--mpa-report", "a.kraken", "--sample-sheet", "s.tsv"], tmp_path), "written twice")
    _refused(_classify(["-a", "taxDB", "--mpa-report", "s.tsv", "--sample-sheet", "s.tsv"], tmp_path), "one of the inputs")


def test_child_list_cycle_reachable_from_the_root(tmp_path):
    cyc = TAXDB + b"700\t701\tc0\tgenus\n701\t700\tc1\tgenus\n"        # unreachable from 1: accepted
    r = _classify(["-a", "taxDB", "--mpa-report", "t.mpa", "-o", "x.kraken", "reads.fa"], tmp_path, cyc)
    assert r.returncode != 64 and "cycle" not in r.stderr
    reach = cyc + b"700\t9\tc0 again\tgenus\n"                        # 9 -> 700 -> 701 -> 700
    _refused(_classify(["-a", "taxDB", "--mpa-report", "t.mpa", "-o", "x.kraken", "reads.fa"], tmp_path, reach), "cycle")
    assert not (tmp_path / "t.mpa").exists()


def test_parent_cycle_refused_with_translate(tmp_path):
    cyc = TAXDB + b"700\t701\tc0\tgenus\n701\t700\tc1\tgenus\n"
    _refused(_classify(["-a", "taxDB", "--translate-out", "t.tr", "-o", "x.kraken", "reads.fa"], tmp_path, cyc), "cycle")
    r = _classify(["-a", "taxDB", "--translate-out", "t.tr", "-o", "x.kraken", "reads.fa"], tmp_path)
    assert r.returncode != 64 and "unable to open" in r.stderr
