"""krakenuniq-filter's rules (tests/kraken_filter.py) against the script's recorded output on crafted Kraken lines and
a crafted taxonomy, and the argument checks of `classify --threshold`, which run before any device call."""
import subprocess

import pytest

from krakenuniq_b200 import build
from tests import kraken_filter

# taxDB rows in file order: a deep chain 2..60 under the root, a parent without a row (999), a parent 0, a self-parent
# row that is not the root, a later self-parent row after a real one (500 keeps parent 1) and a later row that
# overwrites (600 ends under 100)
TAXDB = b"".join(b"%d\t%d\tn%d\trank\n" % r for r in
                 [(1, 1, 1)] + [(i, i - 1, i) for i in range(2, 61)] +
                 [(100, 1, 100), (101, 100, 101), (102, 101, 102), (200, 999, 200), (201, 200, 201), (300, 0, 300),
                  (301, 300, 301), (400, 400, 400), (401, 400, 401), (500, 1, 500), (500, 500, 500), (600, 1, 600),
                  (600, 100, 600), (601, 600, 601)])

KRAKEN = b"".join(b"\t".join(f) + b"\n" for f in [
    (b"C", b"deep", b"60", b"150", b"60:3 A:5 0:2 59:1 30:4 A:1 2:1"),
    (b"C", b"deep_misses", b"60", b"90", b"60:1 0:40"),             # climbs to the root: P is the child's fraction
    (b"C", b"three_of_ten", b"3", b"40", b"3:3 0:7"),                # 0.3 lands exactly on T = 0.3
    (b"C", b"half", b"101", b"40", b"101:1 102:0 0:1"),              # 0.5 against T - 1e-5 around 0.5
    (b"C", b"repeat_runs", b"102", b"60", b"102:2 0:1 102:3 101:2 A:4 100:1"),
    (b"C", b"missing_taxa", b"102", b"50", b"9999:4 102:1 0:2"),     # 9999 has no row
    (b"C", b"no_row_parent", b"201", b"40", b"201:1 0:9"),           # the walk ends at 999
    (b"C", b"parent_zero", b"301", b"40", b"301:1 0:9"),             # ends at parent 0: U with taxon 0
    (b"C", b"self_parent", b"401", b"40", b"401:2 400:1 0:5"),
    (b"C", b"later_self_row", b"500", b"30", b"500:1 0:3"),
    (b"C", b"overwritten", b"601", b"30", b"601:1 100:2 1:1 0:4"),
    (b"C", b"at_root", b"1", b"30", b"1:4 0:1"),
    (b"U", b"zero", b"0", b"20", b"0:0"),
    (b"U", b"ambiguous", b"0", b"40", b"A:10"),
    (b"U", b"misses", b"0", b"40", b"0:10"),
    (b"C", b"quick", b"45", b"100", b"Q:3"),
    (b"C", b"quick_root", b"1", b"100", b"Q:1"),
    (b"C", b"spread", b"45", b"200", b"45:2 44:2 20:6 10:1 60:5 101:3 0:11 A:2"),
])


@pytest.mark.parametrize("threshold", ["0", "1", "0.3", "0.2", "0.50001", "0.500011", "0.75"])
def test_filter_rules_match_krakenuniq_filter(reference, tmp_path, threshold):
    (tmp_path / "taxDB").write_bytes(TAXDB)
    (tmp_path / "database.kdb").write_bytes(b"")                   # the script only checks that they exist
    (tmp_path / "database.idx").write_bytes(b"")
    (tmp_path / "in.kraken").write_bytes(KRAKEN)
    kraken_filter.install_filter()
    r = reference.run_tool(kraken_filter.FILTER, ["--db", ".", "--threshold", threshold, "in.kraken"], cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    F = kraken_filter.parent_map(kraken_filter.taxdb_rows(TAXDB))
    assert kraken_filter.filter_lines(KRAKEN, F, float(threshold)).decode() == r.stdout


def test_out_of_range_threshold_exits_64(reference, tmp_path):
    (tmp_path / "taxDB").write_bytes(TAXDB)
    (tmp_path / "database.kdb").write_bytes(b"")
    (tmp_path / "database.idx").write_bytes(b"")
    (tmp_path / "in.kraken").write_bytes(KRAKEN)
    kraken_filter.install_filter()
    r = reference.run_tool(kraken_filter.FILTER, ["--db", ".", "--threshold", "1.5", "in.kraken"], cwd=tmp_path)
    assert r.returncode == 64 and "threshold must be in the interval [0,1]." in r.stderr and r.stdout == ""


def _classify(args, tmp_path):
    return subprocess.run([build.build_classify(), "-d", "db.kdb", "-i", "db.idx", "-a", "taxDB"] + args, cwd=tmp_path,
                          capture_output=True, text=True)


@pytest.mark.parametrize("value", ["1.5", "-0.1", "1.0001", "nan"])
def test_threshold_outside_the_interval(tmp_path, value):
    r = _classify(["--threshold", value, "-o", "out.kraken", "reads.fa"], tmp_path)
    assert r.returncode == 64 and "threshold must be in the interval [0,1]." in r.stderr
    assert not (tmp_path / "out.kraken").exists()


@pytest.mark.parametrize("value", ["", "abc", "0.5x", "0,5", "1_0"])
def test_malformed_threshold(tmp_path, value):
    r = _classify(["--threshold", value, "reads.fa"], tmp_path)
    assert r.returncode == 64 and "--threshold" in r.stderr


def test_threshold_refuses_the_sequence_column(tmp_path):
    r = _classify(["--threshold", "0.5", "-s", "reads.fa"], tmp_path)
    assert r.returncode == 64 and "-s" in r.stderr


def test_threshold_bounds_are_accepted(tmp_path):
    """0 and 1 pass the checks: the run goes on to open the (missing) database"""
    for value in ("0", "1", "1e-1"):
        r = _classify(["--threshold", value, "reads.fa"], tmp_path)
        assert "threshold" not in r.stderr and r.returncode != 64
