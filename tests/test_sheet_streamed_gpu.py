"""`classify --sample-sheet` on a streamed database: the rounds of reads cross the samples' boundaries, so that a sheet
makes as many passes over the database as its reads need together.  Every file a row writes must still be the bytes a
separate `classify` run of that row writes, and errors must take effect at their sample's turn."""
import os
import re
import socket

import numpy as np
import pytest

from tests import util
from tests.test_sample_sheet_gpu import G, _common, _files, _mate_files, _run, _separate, _setup, _sheet_vs_separate, _stats, \
    _write_sheet

pytestmark = pytest.mark.gpu
STREAM = ["-x", "40K"]
# a budget far below the card's free memory: the rounds, and the batches a round may hold past an end of a sample, are
# then set by the budget and not by what other work leaves free on the card
CHUNKS = {"KUQ_FORCE_CHUNKS": "1", "KUQ_HBM_BUDGET": str(64 << 20)}
TWO = {"KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"}
ROWS = [("fa", "reads.fa", None), ("fq", "reads_300.fq", None), ("crlf", "reads_crlf_60.fa", None),
        ("two", "reads_crlf_60.fa,prefix.fa", None)]


def _rounds(stderr):
    m = re.findall(r"classify: (\d+) samples streamed in (\d+) rounds", stderr)
    assert len(m) == 1, stderr[-2000:]
    return int(m[0][0]), int(m[0][1])


def _range_bytes(budget=40 << 10):
    """the two range buffers of the golden database cut at `budget` (plan_ranges and stage_streamed of classify)"""
    idx = np.fromfile(os.path.join(G, "database.idx"), dtype=np.uint8)
    off = idx[8:].view(np.uint64).astype(np.int64)
    n_bins, first, max_rec, max_bins = len(off) - 1, 0, 1, 1
    fits = lambda lo, end: (end - lo + 1) * 8 + (off[end] - off[lo]) * 12 + 8 <= budget
    while first < n_bins:
        end = first + 1
        while end < n_bins and fits(first, end + 1):
            end += 1
        if off[end] > off[first]:
            max_rec, max_bins = max(max_rec, off[end] - off[first]), max(max_bins, end - first)
        first = end
    return 2 * (int(max_rec) * 12 + (int(max_bins) + 1) * 8 + 4096)


def _order_of_stats(stderr, rows):
    stats, text = _stats(stderr), stderr.replace("\r", "\n")
    assert len(stats) == len(rows)
    for i, (name, _, _) in enumerate(rows):                            # each block after the line naming its sample
        at = text.index(f"classify: sample {name} ({i + 1} of {len(rows)})")
        nxt = text.index("classify: sample", at + 1) if i + 1 < len(rows) else len(text)
        assert at < text.index(stats[i] + " processed in", at) < nxt


@pytest.mark.parametrize("contexts", ["one", "two"])
def test_one_round(tmp_path, contexts):
    _setup(tmp_path)
    env = dict(CHUNKS, **(TWO if contexts == "two" else {}))
    r, _ = _sheet_vs_separate(tmp_path, "classify", ["database"], STREAM, env, ROWS, "o")
    assert r.returncode == 0, r.stderr[-2000:]
    assert _rounds(r.stderr) == (4, 1)
    assert r.stderr.count("(database chunk 1 of") == 1
    _order_of_stats(r.stderr, ROWS)
    if contexts == "two":
        assert "streamed over 2 GPUs" in r.stderr

    rng = np.random.default_rng(5)
    ids, seqs = util.read_fastq(os.path.join(G, "reads_300.fq"))
    _mate_files(tmp_path, "a", ids, seqs, rng)
    ids2, seqs2 = util.read_fasta(os.path.join(G, "reads.fa"))
    _mate_files(tmp_path, "b", ids2[:150], seqs2[:150], rng)
    rows = [("a", "a_1.fq.gz", "a_2.fq.gz"), ("b", "b_1.fq.gz", "b_2.fq.gz")]
    r, _ = _sheet_vs_separate(tmp_path, "classify", ["database"], STREAM + ["--paired", "--check-names"], env, rows, "p")
    assert r.returncode == 0, r.stderr[-2000:]
    assert _rounds(r.stderr) == (2, 1)


def test_two_contexts_with_samples_over_both_owners(tmp_path):
    """a round budget that cuts the larger samples into several batches: a sample's batches on both owners"""
    _setup(tmp_path)
    env = dict(CHUNKS, **TWO, KUQ_HBM_BUDGET=str(_range_bytes() + 600000), KUQ_TIMING="1")
    r, _ = _sheet_vs_separate(tmp_path, "classify", ["database"], STREAM, env, ROWS, "t")
    assert r.returncode == 0, r.stderr[-2000:]
    _order_of_stats(r.stderr, ROWS)
    per_round = re.findall(r"streamed round \d+: stream per GPU [\d.]+ s \((\d+) batches\), [\d.]+ s \((\d+) batches\)", r.stderr)
    assert sum(int(a) + int(b) for a, b in per_round) > len(ROWS) + 1     # reads.fa alone takes several batches


def test_several_rounds(tmp_path):
    """rounds of 200000 bytes: batches of 33333 bases, so that reads_300.fq (45000 bases) spans two rounds and the small
    samples share the rounds after it"""
    _setup(tmp_path)
    rows = [("fq", "reads_300.fq", None)] + [(f"c{i}", "reads_crlf_60.fa", None) for i in range(4)]
    env = dict(CHUNKS, KUQ_HBM_BUDGET=str(_range_bytes() + 200000))
    r, _ = _sheet_vs_separate(tmp_path, "classify", ["database"], STREAM, env, rows, "r")
    assert r.returncode == 0, r.stderr[-2000:]
    s, rounds = _rounds(r.stderr)
    assert s == 5 and 1 < rounds < 5, r.stderr[-2000:]
    assert r.stderr.count("(database chunk 1 of") == rounds
    _order_of_stats(r.stderr, rows)


@pytest.mark.parametrize("contexts", ["one", "two"])
def test_two_databases_streamed(tmp_path, contexts):
    _setup(tmp_path, ("database", "db2"))
    env = {"KUQ_HBM_BUDGET": "200000", **(TWO if contexts == "two" else {})}
    r, _ = _sheet_vs_separate(tmp_path, "classify", ["database", "db2"], ["-M"], env, ROWS, "d")
    assert r.returncode == 0, r.stderr[-2000:]
    s, rounds = _rounds(r.stderr)
    assert s == 4 and r.stderr.count("2 databases streamed: %d rounds" % rounds) == 1


@pytest.mark.parametrize("contexts", ["one", "two"])
def test_classify_exact(tmp_path, contexts):
    _setup(tmp_path)
    env = dict(CHUNKS, **(TWO if contexts == "two" else {}))
    r, _ = _sheet_vs_separate(tmp_path, "classifyExact", ["database"], STREAM, env, ROWS, "e")
    assert r.returncode == 0, r.stderr[-2000:]
    assert _rounds(r.stderr) == (4, 1)


def test_per_sample_outputs(tmp_path):
    """--threshold, --extract on some rows, --translate-out columns and one --mpa-report table over the sheet"""
    _setup(tmp_path)
    cols = ["name", "input", "output", "report", "classified_out", "unclassified_out", "extract_out", "translate_out"]
    rows = [("fa", "reads.fa", True, True), ("fq", "reads_300.fq", False, True), ("two", "reads_crlf_60.fa,prefix.fa", True, False)]
    flags = ["--threshold", "0.3", "--extract", "105,106"]

    def sheet(tag):
        lines = ["\t".join(cols)]
        for name, inp, x, t in rows:
            lines.append("\t".join([name, inp] + [f"{tag}.{name}.{v}" for v in ("kraken", "report", "C", "U")] +
                                   [f"{tag}.{name}.x" if x else "", f"{tag}.{name}.tr" if t else ""]))
        (tmp_path / f"{tag}.tsv").write_text("\n".join(lines) + "\n")
        return f"{tag}.tsv"

    r = _run(tmp_path, "classify", _common(["database"]) + STREAM + flags + ["--mpa-report", "s.mpa", "--sample-sheet", sheet("s")],
             CHUNKS)
    assert r.returncode == 0, r.stderr[-2000:]
    assert _rounds(r.stderr) == (3, 1)
    m = _run(tmp_path, "classify", _common(["database"]) + ["-M"] + flags + ["--mpa-report", "m.mpa", "--sample-sheet", sheet("m")], {})
    assert m.returncode == 0, m.stderr[-2000:]
    assert (tmp_path / "s.mpa").read_bytes() == (tmp_path / "m.mpa").read_bytes()
    for name, inp, x, t in rows:
        outs = ["-o", f"p.{name}.kraken", "-r", f"p.{name}.report", "-C", f"p.{name}.C", "-U", f"p.{name}.U"]
        outs += (["--extract-out", f"p.{name}.x"] if x else []) + (["--translate-out", f"p.{name}.tr"] if t else [])
        sep = _run(tmp_path, "classify", _common(["database"]) + STREAM + flags[:2] + (flags[2:] if x else []) + outs + inp.split(","),
                   CHUNKS)
        assert sep.returncode == 0, sep.stderr[-2000:]
        for v in ("kraken", "report", "C", "U", "x", "tr"):
            got, want = tmp_path / f"s.{name}.{v}", tmp_path / f"p.{name}.{v}"
            assert got.exists() == want.exists(), (name, v)
            if want.exists():
                assert got.read_bytes() == want.read_bytes(), (name, v)
        assert (tmp_path / f"s.{name}.kraken").read_bytes().count(b"P=") > 0


def test_malformed_record_ends_its_sample_only(tmp_path):
    _setup(tmp_path)
    data = (tmp_path / "reads_300.fq").read_bytes().split(b"\n")
    data[4 * 120 + 2] = b"-"                                           # record 121 loses its '+' line
    (tmp_path / "bad.fq").write_bytes(b"\n".join(data))
    rows = [("one", "reads.fa", None), ("bad", "bad.fq", None), ("three", "prefix.fa", None)]
    r, seps = _sheet_vs_separate(tmp_path, "classify", ["database"], STREAM, CHUNKS, rows, "m")
    assert r.returncode == 0 and seps[1].returncode == 0, r.stderr[-2000:]
    assert _rounds(r.stderr) == (3, 1)
    assert (tmp_path / "m.bad.kraken").read_bytes().count(b"\n") == 120
    text = r.stderr.replace("\r", "\n")                               # the message comes in sample bad's turn
    at = text.index("malformed fastq file - quality header")
    assert text.index("classify: sample bad") < at < text.index("classify: sample three")


def test_mate_name_mismatch_lets_later_samples_run(tmp_path):
    _setup(tmp_path)
    rng = np.random.default_rng(4)
    ids, seqs = util.read_fastq(os.path.join(G, "reads_300.fq"))
    _mate_files(tmp_path, "bad", ids, seqs, rng, mismatch_at=150)
    _mate_files(tmp_path, "good", ids[:100], seqs[:100], rng)
    rows = [("bad", "bad_1.fq", "bad_2.fq"), ("good", "good_1.fq", "good_2.fq")]
    flags = _common(["database"]) + STREAM + ["--paired", "--check-names"]
    r = _run(tmp_path, "classify", flags + ["--sample-sheet", _write_sheet(tmp_path, rows, "n")], CHUNKS)
    assert r.returncode == 65, r.stderr[-2000:]
    assert _rounds(r.stderr) == (2, 1)
    assert r.stderr.count("mismatched mate pair names") == 1
    assert "classify: sample bad: mismatched mate pair names" in r.stderr
    for i, row in enumerate(rows):
        s, want = _separate(tmp_path, "classify", flags, CHUNKS, row, f"sep{i}")
        assert s.returncode == (65 if i == 0 else 0)
        assert _files(tmp_path, f"n.{row[0]}") == want, row
    assert 0 < (tmp_path / "n.bad.kraken").read_bytes().count(b"\n") < 300


def test_uncreatable_output_stops_at_its_sample(tmp_path):
    _setup(tmp_path)
    sheet = "name\tinput\toutput\treport\none\treads.fa\tc.one.kraken\tc.one.report\n" \
            "two\treads_300.fq\tno_such_dir/c.two.kraken\tc.two.report\nthree\tprefix.fa\tc.three.kraken\t\n"
    (tmp_path / "c.tsv").write_text(sheet)
    r = _run(tmp_path, "classify", _common(["database"]) + STREAM + ["--sample-sheet", "c.tsv"], CHUNKS)
    assert r.returncode == 73, r.stderr[-2000:]
    assert "classify: sample two: can't open no_such_dir/c.two.kraken" in r.stderr
    s = _run(tmp_path, "classify", _common(["database"]) + STREAM + ["-o", "sep.kraken", "-r", "sep.report", "reads.fa"], CHUNKS)
    assert s.returncode == 0
    assert (tmp_path / "c.one.kraken").read_bytes() == (tmp_path / "sep.kraken").read_bytes()
    assert (tmp_path / "c.one.report").read_bytes() == (tmp_path / "sep.report").read_bytes()
    assert not (tmp_path / "c.two.report").exists() and not (tmp_path / "c.three.kraken").exists()


def test_input_that_cannot_be_opened_stops_at_its_sample(tmp_path, monkeypatch):
    """row 3's input passes the sheet's checks (a readable directory entry) but cannot be opened (a socket): the run
    exits EX_NOINPUT naming sample 3 after rows 1 and 2 are complete, as the loop of separate runs does"""
    _setup(tmp_path)
    monkeypatch.chdir(tmp_path)
    sock = socket.socket(socket.AF_UNIX)
    sock.bind("sock.fa")
    try:
        rows = [("one", "reads.fa", None), ("two", "reads_300.fq", None), ("three", "sock.fa", None)]
        r = _run(tmp_path, "classify", _common(["database"]) + STREAM + ["--sample-sheet", _write_sheet(tmp_path, rows, "i")], CHUNKS)
        assert r.returncode == 66, r.stderr[-2000:]
        assert "classify: sample three: can't open sock.fa" in r.stderr
        assert len(_stats(r.stderr)) == 2
        for i, row in enumerate(rows):
            s, want = _separate(tmp_path, "classify", _common(["database"]) + STREAM, CHUNKS, row, f"sep{i}")
            assert s.returncode == (66 if i == 2 else 0), s.stderr[-2000:]
            assert _files(tmp_path, f"i.{row[0]}") == want, row
    finally:
        sock.close()


def test_no_state_carried(tmp_path):
    _setup(tmp_path)
    rows = [(n, "reads.fa", None) for n in "abc"]
    r, _ = _sheet_vs_separate(tmp_path, "classify", ["database"], STREAM, CHUNKS, rows, "n")
    assert r.returncode == 0, r.stderr[-2000:]
    assert _rounds(r.stderr) == (3, 1)
    for v in ("kraken", "report", "C", "U"):
        assert len({(tmp_path / f"n.{n}.{v}").read_bytes() for n in "abc"}) == 1
