"""`classify --mpa-report` / `--translate-out`: the table and the lineages must be what krakenuniq-mpa-report and
krakenuniq-translate (restated in tests/mpa_report.py and tests/translate.py) print from the same run's Kraken lines,
and every other output (Kraken lines, report, -C, -U, stats) must be the bytes of the run without them, in every layout.
On the golden mini run they must be the scripts' recorded output."""
import gzip
import os
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import synth
from tests import mpa_report, paired, translate, util
from tests.test_threshold_gpu import LAYOUTS, _copy, _exe, _setup, _stats, synthetic  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
G = util.GOLDEN
OUTS = ("-o", "-r", "-C", "-U")
MFLAGS = [(), ("--mpa-show-zeros",), ("--mpa-header-line", "--translate-mpa-format"),
          ("--mpa-intermediate-ranks", "--mpa-header-line"),
          ("--mpa-show-zeros", "--mpa-header-line", "--mpa-intermediate-ranks", "--translate-mpa-format")]


def _run(tmp_path, tool, args, env=None):
    r = subprocess.run([_exe(tool)] + args, cwd=tmp_path, capture_output=True, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stderr[-2000:].decode(errors="replace")
    assert b"not usable" not in r.stderr
    return r


def _want(tmp_path, kraken, mflags, ids):
    taxdb = (tmp_path / "taxDB").read_bytes()
    mpa = mpa_report.mpa_table([kraken], taxdb, "--mpa-show-zeros" in mflags, "--mpa-header-line" in mflags,
                               "--mpa-intermediate-ranks" in mflags, ids=ids)
    return mpa, translate.translate(kraken, taxdb, "--translate-mpa-format" in mflags)


def _read(path):
    data = path.read_bytes()
    return gzip.decompress(data) if path.name.endswith(".gz") else data


def _compare(tmp_path, tool, dbs, flags, env, inputs, mflags=(), kraken_off=False, mpa="new.mpa", tr="new.tr"):
    """runs without and with the two outputs; checks them and the unchanged outputs.  Returns the base Kraken lines."""
    common = sum((["-d", f"{d}.kdb", "-i", f"{d}.idx"] for d in dbs), []) + ["-a", "taxDB"] + flags
    base = _run(tmp_path, tool, common + sum(([o, f"base{o}"] for o in OUTS), []) + inputs, env)
    outs = [o for o in OUTS if not (kraken_off and o == "-o")]
    new = _run(tmp_path, tool, common + sum(([o, f"new{o}"] for o in outs), []) + (["-o", "off"] if kraken_off else []) +
               ["--mpa-report", mpa, "--translate-out", tr] + list(mflags) + inputs, env)
    for o in outs:
        assert (tmp_path / f"new{o}").read_bytes() == (tmp_path / f"base{o}").read_bytes(), o
    assert _stats(new.stderr.decode()) == _stats(base.stderr.decode())
    kraken = (tmp_path / "base-o").read_bytes()
    assert kraken
    want_mpa, want_tr = _want(tmp_path, kraken, mflags, ["-" if kraken_off else "new-o"])
    assert _read(tmp_path / mpa) == want_mpa
    assert _read(tmp_path / tr) == want_tr
    return kraken


def test_golden_mini_equals_the_recorded_scripts(tmp_path):
    """the run's Kraken output is preload.kraken; the table and lineages are the scripts' recorded output over it,
    root-called reads with their inherited lineages included"""
    _setup(tmp_path)
    rec = mpa_report.recorded_stdout("test_mpa_report_cpu.py", "test_golden_mini_recorded")
    allf = ["--mpa-show-zeros", "--mpa-header-line", "--mpa-intermediate-ranks"]
    common = ["-d", "database.kdb", "-i", "database.idx", "-a", "taxDB", "-M", "-o", "preload.kraken"]
    for mflags, want_mpa, tflags, want_tr in (([], rec[0], [], rec[2]), (allf, rec[1], ["--translate-mpa-format"], rec[3])):
        _run(tmp_path, "classify", common + ["--mpa-report", "t.mpa", "--translate-out", "t.tr"] + mflags + tflags + ["reads.fa"])
        assert (tmp_path / "preload.kraken").read_bytes() == open(os.path.join(G, "preload.kraken"), "rb").read()
        assert (tmp_path / "t.mpa").read_bytes() == want_mpa
        assert (tmp_path / "t.tr").read_bytes() == want_tr
    roots = [l for l in rec[2].split(b"\n") if l and l.split(b"\t")[0] in
             {x.split(b"\t")[1] for x in (tmp_path / "preload.kraken").read_bytes().split(b"\n") if x.split(b"\t")[2:3] == [b"1"]}]
    assert any(l.split(b"\t")[1] for l in roots)                     # some root-called read inherits a lineage
    # standard output: the table alone (the Kraken lines go to the file)
    r = _run(tmp_path, "classify", common + ["--mpa-report", "-", "reads.fa"])
    assert r.stdout == rec[0]


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_layouts(tmp_path, layout):
    tool, dbs, flags, env = LAYOUTS[layout]
    _setup(tmp_path, dbs)
    mflags = MFLAGS[list(LAYOUTS).index(layout) % len(MFLAGS)]
    _compare(tmp_path, tool, dbs, flags, env, ["reads.fa", "reads_crlf_60.fa", "reads_300.fq"], mflags)


@pytest.mark.parametrize("extra,env", [(["--threshold", "0.4"], {}), (["--threshold", "0.7", "-c"], {"KUQ_SERIAL_INGEST": "1"}),
                                       (["-q", "-s"], {"KUQ_BATCH_READS": "50"})])
def test_filtered_and_other_lines(tmp_path, extra, env):
    _setup(tmp_path)
    _compare(tmp_path, "classify", ["database"], ["-M"] + extra, env, ["reads.fa", "reads_300.fq"], MFLAGS[2])


@pytest.mark.parametrize("env", [{}, {"KUQ_SERIAL_INGEST": "1"}])
def test_kraken_output_off_and_gzip(tmp_path, env):
    _setup(tmp_path)
    _compare(tmp_path, "classify", ["database"], ["-M", "-t", "4"], env, ["reads.fa", "reads_300.fq"], MFLAGS[4],
             kraken_off=True, mpa="new.mpa.gz", tr="new.tr.gz")


def test_paired(tmp_path):
    _setup(tmp_path)
    ids, seqs = util.read_fasta(os.path.join(G, "reads.fa"))
    pairs = paired.split_pairs(seqs, np.random.default_rng(5))
    (tmp_path / "m_1.fq").write_bytes(paired.fastq_bytes([(f"{i}/1".encode(), a) for i, (a, _) in zip(ids, pairs)]))
    (tmp_path / "m_2.fq").write_bytes(paired.fastq_bytes([(f"{i}/2".encode(), b) for i, (_, b) in zip(ids, pairs)]))
    for env in ({}, {"KUQ_SERIAL_INGEST": "1"}):
        _compare(tmp_path, "classify", ["database"], ["-M", "--paired"], env, ["m_1.fq", "m_2.fq"], MFLAGS[3])


def test_empty_ids_and_many_parts(tmp_path):
    """reads with an empty id (the scripts take the length as taxid) and small batches formatted in many parts, so the
    root-called lines take their lineage from earlier parts and batches"""
    _setup(tmp_path)
    recs = (tmp_path / "reads.fa").read_bytes().split(b"\n")
    blank = b"\n".join(b">" if i % 14 == 0 and l.startswith(b">") else l for i, l in enumerate(recs))
    (tmp_path / "blank.fa").write_bytes(blank)
    kraken = _compare(tmp_path, "classify", ["database"], ["-M", "-t", "8"], {"KUQ_BATCH_READS": "37"}, ["blank.fa", "reads.fa"],
                      MFLAGS[2])
    assert any(l.split(b"\t")[1] == b"" for l in kraken.split(b"\n") if l)


def test_synthetic_taxonomy(tmp_path, synthetic):
    """2400 species with every standard rank above them (a family under parent 0 and a genus whose parent has no row
    included), reads over more than 32 taxa"""
    _copy(synthetic[0], tmp_path)
    synth.Taxonomy(synth.add_upper_ranks(synthetic[1].rows)).write(tmp_path / "taxDB")
    for mflags in (MFLAGS[1], MFLAGS[4]):
        kraken = _compare(tmp_path, "classify", ["database"], ["-M"], {}, ["reads.fa"], mflags)
    assert len({l.split(b"\t")[2] for l in kraken.split(b"\n") if l}) > 32


def test_sample_sheet(tmp_path):
    """one table for the sheet, a column per row in sheet order; each translate_out is the file of a separate run"""
    _setup(tmp_path)
    sheet = tmp_path / "s.tsv"
    sheet.write_text("name\tinput\toutput\ttranslate_out\n"
                     "a\treads.fa\ta.kraken\ta.tr\n"
                     "b\treads_300.fq,reads_crlf_60.fa\tb.kraken\tb.tr.gz\n"
                     "c\treads_300.fq\t\tc.tr\n"
                     "d\treads_crlf_60.fa\td.kraken\t\n")
    common = ["-d", "database.kdb", "-i", "database.idx", "-a", "taxDB", "-M"]
    _run(tmp_path, "classify", common + ["--sample-sheet", "s.tsv", "--mpa-report", "s.mpa", "--mpa-header-line",
                                         "--translate-mpa-format"])
    krakens = []
    for row, inputs in (("a", ["reads.fa"]), ("b", ["reads_300.fq", "reads_crlf_60.fa"]), ("c", ["reads_300.fq"]),
                        ("d", ["reads_crlf_60.fa"])):
        _run(tmp_path, "classify", common + ["-o", f"sep.{row}.kraken", "--translate-out", f"sep.{row}.tr",
                                             "--translate-mpa-format"] + inputs)
        krakens.append((tmp_path / f"sep.{row}.kraken").read_bytes())
        if row != "c":
            assert (tmp_path / f"{row}.kraken").read_bytes() == krakens[-1]
        if row != "d":
            assert _read(tmp_path / (f"{row}.tr.gz" if row == "b" else f"{row}.tr")) == (tmp_path / f"sep.{row}.tr").read_bytes()
    assert not (tmp_path / "d.tr").exists()
    want = mpa_report.mpa_table(krakens, (tmp_path / "taxDB").read_bytes(), header_line=True,
                                ids=["a.kraken", "b.kraken", "c", "d.kraken"])
    assert (tmp_path / "s.mpa").read_bytes() == want
