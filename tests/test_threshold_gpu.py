"""`classify --threshold T`: the Kraken lines must be what krakenuniq-filter (restated in tests/kraken_filter.py) makes
of the same run's unfiltered lines, and every other output (report, -C, -U, stats) must be the unfiltered run's bytes,
in every layout.  The C ABI's filtered_call / filter_hits / filter_total are checked directly."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import binding, build, synth
from tests import kraken_filter, paired, util

pytestmark = pytest.mark.gpu
G, M = util.GOLDEN, os.path.join(os.path.dirname(util.GOLDEN), "multidb")
SHARD_ENV = {"KUQ_FORCE_SHARDS": "1", "KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"}


def _exe(tool="classify"):
    return os.path.join(os.path.dirname(build.build_classify()), tool)


def _setup(tmp_path, dbs=("database",)):
    for d in dbs:
        for ext in (".kdb", ".idx", ".kdb.counts"):
            shutil.copyfile(os.path.join(M if d == "db2" else G, d + ext), tmp_path / (d + ext))
    for f in ("taxDB", "reads.fa", "reads_300.fq", "reads_crlf_60.fa"):
        shutil.copyfile(os.path.join(G, f), tmp_path / f)


def _stats(stderr):
    """the stats lines, without their timings"""
    lines = stderr.replace("\r", "\n").splitlines()
    return [l.split(" processed in")[0] for l in lines if " sequences " in l]


def _compare(tmp_path, tool, dbs, flags, env, inputs, threshold, outs=("-o", "-r", "-C", "-U")):
    """runs without and with --threshold; checks the filtered lines and the unchanged outputs"""
    common = sum((["-d", f"{d}.kdb", "-i", f"{d}.idx"] for d in dbs), []) + ["-a", "taxDB"] + flags
    runs = {}
    for tag, extra in (("base", []), ("thr", ["--threshold", str(threshold)])):
        files = sum(([o, f"{tag}{o}"] for o in outs), [])
        r = subprocess.run([_exe(tool)] + common + extra + files + inputs, cwd=tmp_path, capture_output=True,
                           text=True, env=dict(os.environ, **env))
        assert r.returncode == 0, r.stderr[-2000:]
        assert "not usable" not in r.stderr
        runs[tag] = r
    F = kraken_filter.parent_map(kraken_filter.taxdb_rows((tmp_path / "taxDB").read_bytes()))
    base = (tmp_path / "base-o").read_bytes()
    assert base
    assert (tmp_path / "thr-o").read_bytes() == kraken_filter.filter_lines(base, F, float(threshold))
    for o in outs[1:]:
        assert (tmp_path / f"thr{o}").read_bytes() == (tmp_path / f"base{o}").read_bytes(), o
    assert _stats(runs["thr"].stderr) == _stats(runs["base"].stderr)
    return base


@pytest.mark.parametrize("threshold", ["0", "0.2", "0.5", "1"])
def test_resident_mini(tmp_path, threshold):
    _setup(tmp_path)
    base = _compare(tmp_path, "classify", ["database"], ["-M"], {}, ["reads.fa", "reads_300.fq"], threshold)
    if threshold == "0.5":          # the filter moves some calls: the test would pass vacuously otherwise
        F = kraken_filter.parent_map(kraken_filter.taxdb_rows((tmp_path / "taxDB").read_bytes()))
        moved = [a.split(b"\t")[2] != b.split(b"\t")[2] for a, b in
                 zip(base.splitlines(), kraken_filter.filter_lines(base, F, 0.5).splitlines())]
        assert any(moved)


LAYOUTS = {
    "q2": ("classify", ["database"], ["-M", "-q", "-m", "2"], {}),
    "c": ("classify", ["database"], ["-M", "-c", "-t", "4"], {}),
    "x40K": ("classify", ["database"], ["-x", "40K"], {}),
    "streamed": ("classify", ["database"], ["-x", "40K"], {"KUQ_FORCE_CHUNKS": "1"}),
    "two_db": ("classify", ["database", "db2"], ["-M"], {}),
    "two_db_streamed": ("classify", ["database", "db2"], ["-M"], {"KUQ_HBM_BUDGET": "200000"}),
    "exact": ("classifyExact", ["database"], ["-M"], {}),
    "replicas": ("classify", ["database"], ["-M"], {"KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"}),
    "shards": ("classify", ["database"], ["-M"], SHARD_ENV),
    "two_db_sharded": ("classify", ["database", "db2"], ["-M"], SHARD_ENV),
    "serial": ("classify", ["database"], ["-M", "-t", "1"], {"KUQ_SERIAL_INGEST": "1"}),
}


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_layouts(tmp_path, layout):
    tool, dbs, flags, env = LAYOUTS[layout]
    _setup(tmp_path, dbs)
    _compare(tmp_path, tool, dbs, flags, env, ["reads.fa", "reads_crlf_60.fa"], "0.3")


def test_paired(tmp_path):
    _setup(tmp_path)
    ids, seqs = util.read_fasta(os.path.join(G, "reads.fa"))
    pairs = paired.split_pairs(seqs, np.random.default_rng(5))
    (tmp_path / "m_1.fq").write_bytes(paired.fastq_bytes([(f"{i}/1".encode(), a) for i, (a, _) in zip(ids, pairs)]))
    (tmp_path / "m_2.fq").write_bytes(paired.fastq_bytes([(f"{i}/2".encode(), b) for i, (_, b) in zip(ids, pairs)]))
    _compare(tmp_path, "classify", ["database"], ["-M", "--paired"], {}, ["m_1.fq", "m_2.fq"], "0.4")


def test_sample_sheet(tmp_path):
    """the threshold applies to every row; each row's lines are the filter's of that row's unfiltered lines"""
    _setup(tmp_path)
    F = kraken_filter.parent_map(kraken_filter.taxdb_rows((tmp_path / "taxDB").read_bytes()))
    common = [_exe(), "-d", "database.kdb", "-i", "database.idx", "-a", "taxDB", "-M"]
    for tag, extra in (("base", []), ("thr", ["--threshold", "0.6"])):
        sheet = tmp_path / f"{tag}.tsv"
        sheet.write_text("name\tinput\toutput\treport\tclassified_out\n"
                         f"a\treads.fa\t{tag}.a.kraken\t{tag}.a.report\t{tag}.a.C\n"
                         f"b\treads_300.fq,reads_crlf_60.fa\t{tag}.b.kraken\t{tag}.b.report\t{tag}.b.C\n")
        r = subprocess.run(common + extra + ["--sample-sheet", sheet.name], cwd=tmp_path, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
    for row in "ab":
        base = (tmp_path / f"base.{row}.kraken").read_bytes()
        assert (tmp_path / f"thr.{row}.kraken").read_bytes() == kraken_filter.filter_lines(base, F, 0.6)
        for ext in ("report", "C"):
            assert (tmp_path / f"thr.{row}.{ext}").read_bytes() == (tmp_path / f"base.{row}.{ext}").read_bytes()


def _synthetic(tmp_path, rng):
    """a database of 2400 species under a few thousand taxa, with a family under parent 0 and a genus whose parent
    has no row; long reads stitched from 40 genomes each hit more than 32 distinct taxa (the overflow table)"""
    tax = synth.make_taxonomy(2400, 600, 60)
    rows = list(tax.rows)
    rows[1] = (rows[1][0], 0, rows[1][2], rows[1][3])                      # family 0 under parent 0
    rows[61] = (rows[61][0], 999999, rows[61][2], rows[61][3])             # genus 0's parent has no row
    tax = synth.Taxonomy(rows)
    tax.write(tmp_path / "taxDB")
    genomes = synth.random_genomes(rng, 2400, 400, 0.2)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, 31)
    kdb, idx = synth.build_db_images(km, tx, 31, 8, 2)
    kdb.tofile(tmp_path / "database.kdb")
    idx.tofile(tmp_path / "database.idx")
    recs = []
    bases, offs = synth.sample_reads(rng, genomes, 3000, 120, 0.02, 0.01, 0.1)
    for i in range(3000):
        recs.append((f"r{i}", bases[offs[i]:offs[i + 1]].tobytes()))
    for i in range(60):
        picks = rng.choice(len(genomes), 40, replace=False)
        seq = b"".join(synth.decode(genomes[g][:100]).tobytes() for g in picks)
        recs.append((f"long{i}", seq))
    (tmp_path / "reads.fa").write_bytes(b"".join(b">%s\n%s\n" % (n.encode(), s) for n, s in recs))
    return tax


@pytest.fixture(scope="module")
def synthetic(tmp_path_factory):
    d = tmp_path_factory.mktemp("synthetic")
    return d, _synthetic(d, np.random.default_rng(11))


def _copy(src, dst):
    for f in ("taxDB", "database.kdb", "database.idx", "reads.fa"):
        shutil.copyfile(src / f, dst / f)


@pytest.mark.parametrize("threshold", ["0", "0.35", "0.8", "1"])
def test_synthetic_taxonomy_and_overflow(tmp_path, synthetic, threshold):
    _copy(synthetic[0], tmp_path)
    base = _compare(tmp_path, "classify", ["database"], ["-M"], {}, ["reads.fa"], threshold)
    long_lines = [l for l in base.splitlines() if l.split(b"\t")[1].startswith(b"long")]
    assert max(len({h.split(b":")[0] for h in l.split(b"\t")[4].split()}) for l in long_lines) > 34


def _kraken_line(res, i, name):
    n = int(res["run_count"][i])
    if n == 0:
        hits = b"0:0"
    else:
        runs = res["runs"][res["run_start"][i]:res["run_start"][i] + n]
        hits = b" ".join((b"A" if c == util.AMBIG else b"%d" % c) + b":%d" % k for c, k in runs)
    call = int(res["call"][i])
    return b"%s\t%s\t%d\t%d\t%s" % (b"C" if call else b"U", name, call, int(res["n_windows"][i]) + 30, hits)


def test_c_abi_result_arrays(tmp_path, synthetic):
    """filtered_call and P = filter_hits / filter_total from kuq_classify_batch, against the restatement of the lines
    the same result gives; NULL arrays without a threshold"""
    _copy(synthetic[0], tmp_path)
    tax = synthetic[1]
    kdb = np.fromfile(tmp_path / "database.kdb", np.uint8)
    idx = np.fromfile(tmp_path / "database.idx", np.uint8)
    seqs = (tmp_path / "reads.fa").read_bytes().split(b"\n")[1::2]
    bases = np.frombuffer(b"".join(seqs), np.uint8)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.uint64)
    rows = np.array([(r[0], r[1]) for r in tax.rows], np.uint32)
    F = kraken_filter.parent_map([(int(a), int(b)) for a, b in rows])
    for threshold in (None, 0.45):
        c = binding.Classifier(device=0, max_reads=1 << 14, max_bases=4 << 20)
        c.stage_db(kdb, idx)
        c.set_taxonomy(*tax.parent_map())
        if threshold is not None:
            c.set_threshold(threshold, rows[:, 0], rows[:, 1])
        res = c.classify(bases, offs)
        if threshold is None:
            assert "filtered_call" not in res
            c.close()
            continue
        for i in range(len(seqs)):
            want = kraken_filter.filter_line(_kraken_line(res, i, b"r"), F, threshold).split(b"\t")
            assert int(want[2]) == int(res["filtered_call"][i]), i
            den = int(res["filter_total"][i])
            got_p = b"P=%.3f" % (int(res["filter_hits"][i]) / den if den else 0.0)
            assert want[4] == got_p, i
        c.close()


def test_c_abi_refuses_a_looping_parent_map():
    c = binding.Classifier(device=0, max_reads=1 << 10, max_bases=1 << 20)
    c.set_taxonomy(np.array([1, 2, 3], np.uint32), np.array([0, 1, 2], np.uint32))
    with pytest.raises(binding.KuqError) as e:
        c.set_threshold(0.5, np.array([1, 2, 3, 1], np.uint32), np.array([1, 1, 2, 3], np.uint32))
    assert e.value.code == -10
    with pytest.raises(binding.KuqError) as e:
        c.set_threshold(1.5, np.array([1], np.uint32), np.array([1], np.uint32))
    assert e.value.code == -1
    c.close()
