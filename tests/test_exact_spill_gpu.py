"""classifyExact's k-mer set spilled to host memory by k-mer part when the table cannot grow, and counted part by part
at the end (kuq_set_exact_spill, kuq_exact_settle).

KUQ_EXACT_MAX_SLOTS caps the table as if the device had no room for more, so a small workload spills many times on one
card.  Results are held against the oracle's exact counts (`run.set_exact()`) through the C ABI, and against the
unmodified reference's classifyExact report on the golden database through the executable, in every layout."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from krakenuniq_b200 import binding, build
from tests import util
from tests.test_exact_partition_gpu import _check_against_oracle, _classify, _context, _oracle, _workload, _write

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
G = util.GOLDEN
E_STATE, E_NOMEM = -6, -8
BUDGET = 1 << 34
BATCH = 100                              # reads per batch: at most 15,000 windows, which an empty table of 32768 slots takes


def _cap(union, parts):
    """a power of two near union / parts that an empty table can fill with one batch"""
    return max(1 << int(round(np.log2(union / parts))), 1 << 15)


def _spilling(tax, kdb, idx, budget=BUDGET):
    clf = _context(tax, kdb, idx, 1 << 10)
    clf.set_exact_spill(budget)
    return clf


def _union(tax, kdb, idx, seqs):
    clf = _context(tax, kdb, idx, 1 << 10)
    _classify(clf, seqs, BATCH)
    clf.finish()
    return clf.exact_info()["pairs"]


# ---- 1. one context --------------------------------------------------------------------------------------------------
def test_one_context_spills_and_settles(oracle, monkeypatch):
    """a table capped at about an eighth of the union spills at least three times; after settling, kuq_read_counts and
    kuq_clade_counts_tree of every taxon equal the oracle's exact counts"""
    tax, kdb, idx, seqs = _workload(51)
    calls, want, run = _oracle(oracle, tax, kdb, idx, seqs)
    union = _union(tax, kdb, idx, seqs)
    assert union == int(want["unique"].sum())
    monkeypatch.setenv("KUQ_EXACT_MAX_SLOTS", str(_cap(union, 8)))
    clf = _spilling(tax, kdb, idx)
    assert np.array_equal(_classify(clf, seqs, BATCH), calls)
    clf.finish()
    spills, on_host = clf.exact_spill_info()
    assert spills >= 3 and on_host > 0, (spills, on_host)
    binding.Classifier.exact_settle([clf])
    assert clf.exact_spill_info() == (spills, 0)
    _check_against_oracle(clf, want, run, tax)


# ---- 2. three contexts on one card -----------------------------------------------------------------------------------
def test_three_contexts_spill_and_settle(oracle, monkeypatch):
    """three contexts with overlapping shares of the reads, each spilling: their counters joined and their parts settled
    over all three give the oracle's counts and clades for all the reads.  Rounds of 3000 slots: every spill takes
    several rounds, and the settle step packs pieces of several rounds and parts into each of its rounds"""
    tax, kdb, idx, base = _workload(52, n_reads=7500)
    shares = [base[:3000], base[2000:5000], base[5000:]]
    _, want, run = _oracle(oracle, tax, kdb, idx, [s for sh in shares for s in sh])
    monkeypatch.setenv("KUQ_EXACT_MAX_SLOTS", str(_cap(int(want["unique"].sum()), 8)))
    monkeypatch.setenv("KUQ_EXACT_MERGE_SLOTS", "3000")
    ctxs = [_spilling(tax, kdb, idx) for _ in shares]
    for c, sh in zip(ctxs, shares):
        _classify(c, sh, BATCH)
        c.finish()
        assert c.exact_spill_info()[0] >= 1
    for c in ctxs[1:]:
        ctxs[0].merge_counters_from(c)
    binding.Classifier.exact_settle(ctxs)
    assert all(c.exact_spill_info()[1] == 0 for c in ctxs)
    _check_against_oracle(ctxs[0], want, run, tax)


# ---- 3. states -------------------------------------------------------------------------------------------------------
def _state_error(fn):
    with pytest.raises(binding.KuqError) as e:
        fn()
    assert e.value.code == E_STATE, str(e.value)
    assert "kuq_exact_settle" in str(e.value)


def test_partial_readouts_refused_until_settled_and_reset(oracle, monkeypatch):
    """between a spill and the settle step every readout of a partial set refuses with KUQ_E_STATE (the counters still
    join); kuq_reset_counts drops the host parts, and a second workload then equals the oracle"""
    tax, kdb, idx, seqs = _workload(53, n_reads=5000)
    union = _union(tax, kdb, idx, seqs)
    monkeypatch.setenv("KUQ_EXACT_MAX_SLOTS", str(_cap(union, 8)))
    clf, other = _spilling(tax, kdb, idx), _spilling(tax, kdb, idx)
    _classify(clf, seqs, BATCH)
    clf.finish()
    _classify(other, seqs[:50], BATCH)
    other.finish()
    assert clf.exact_spill_info()[0] >= 1 and other.exact_spill_info()[0] == 0
    taxid = int(tax.rows[-1][0])
    buf = torch.zeros((1 << 16, 2), dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    _state_error(clf.counts)
    _state_error(lambda: clf.clade([1, taxid]))
    _state_error(lambda: clf.clade_counts_tree(np.array([1, taxid], np.uint32)))
    _state_error(lambda: clf.exact_export())
    _state_error(lambda: clf.exact_export_partitioned(2))
    _state_error(lambda: clf.exact_export_partitioned(2, buf.data_ptr(), buf.shape[0]))
    _state_error(lambda: clf.exact_export_partitioned_alloc(2))
    _state_error(lambda: other.merge_from(clf))                 # the union into a context that did not spill
    _state_error(lambda: clf.merge_from(other))
    _state_error(lambda: binding.Classifier.exact_partition([other, clf]))
    other.merge_counters_from(clf)                              # the counters join all the same
    other.close()
    # a reset drops the host parts; the next run spills afresh and settles to the oracle
    clf.reset_counts()
    assert clf.exact_spill_info() == (0, 0)
    seqs2 = seqs[1000:4500]
    calls, want, run = _oracle(oracle, tax, kdb, idx, seqs2)
    assert np.array_equal(_classify(clf, seqs2, BATCH), calls)
    clf.finish()
    assert clf.exact_spill_info()[0] >= 1
    binding.Classifier.exact_settle([clf])
    _check_against_oracle(clf, want, run, tax)


def test_budget_below_the_spill_fails(monkeypatch):
    """a host budget below what the run has to spill fails with KUQ_E_NOMEM naming KUQ_EXACT_HOST_BUDGET; a budget of 0
    keeps the failure to grow"""
    tax, kdb, idx, seqs = _workload(54, n_reads=4000)
    union = _union(tax, kdb, idx, seqs)
    monkeypatch.setenv("KUQ_EXACT_MAX_SLOTS", str(_cap(union, 8)))
    clf = _spilling(tax, kdb, idx, budget=16 * union // 4)
    with pytest.raises(binding.KuqError) as e:
        _classify(clf, seqs, BATCH)
        clf.finish()
        binding.Classifier.exact_settle([clf])
    assert e.value.code == E_NOMEM and "KUQ_EXACT_HOST_BUDGET" in str(e.value), str(e.value)
    clf.close()
    off = _spilling(tax, kdb, idx, budget=0)
    with pytest.raises(binding.KuqError) as e:
        _classify(off, seqs, BATCH)
    assert e.value.code == E_NOMEM and "no room to grow" in str(e.value), str(e.value)


# ---- 4. the executable against the reference ---------------------------------------------------------------------------
def _exe():
    return os.path.join(os.path.dirname(build.build_classify()), "classifyExact")


def _report_rows(path):
    rows = {}
    for line in open(path):
        if line.startswith("#") or line.startswith("%"):
            continue
        f = line.rstrip("\n").split("\t")
        rows[f[6]] = f
    return rows


def _setup(tmp_path):
    for f in ("database.kdb", "database.idx", "database.kdb.counts", "taxDB", "reads.fa", "reads_300.fq"):
        shutil.copyfile(os.path.join(G, f), tmp_path / f)


def _run(tmp_path, args, env):
    r = subprocess.run([_exe(), "-d", "database.kdb", "-i", "database.idx", "-a", "taxDB", "-t", "1", "-u", "7500"] + args, cwd=tmp_path,
                       capture_output=True, text=True, env=dict(os.environ, **env))
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stderr


# the golden reads hold about 10^5 (k-mer, taxon) pairs: a table of 2^14 slots spills many times with batches of about 50
# reads (KUQ_BATCH_READS closes a batch at the first work-unit boundary after 50 reads; `-u 7500` puts one every ~50)
SPILL_ENV = {"KUQ_EXACT_MAX_SLOTS": "16384", "KUQ_BATCH_READS": "50", "KUQ_SPARSE_SLOTS": "1024",
             "KUQ_EXACT_HOST_BUDGET": str(1 << 30), "KUQ_TIMING": "1"}
# the streamed layouts cut batches to their HBM budget (up to ~250 reads, 37,050 windows here), which an empty table of
# 2^16 slots takes at a load of 0.6.  The sharded layout cuts its batches by KUQ_SHARD_BATCH_READS; its spills and settle
# step move pairs in rounds of 3000 slots.
WIDE = {"KUQ_EXACT_MAX_SLOTS": "65536", "KUQ_FORCE_CHUNKS": "1", "KUQ_HBM_BUDGET": "400000"}
LAYOUTS = {"one": ([], {"KUQ_DEVICE": "0"}),
           "replicas": ([], {"KUQ_DEVICES": "0,0"}),
           "shards": ([], {"KUQ_DEVICES": "0,0,0", "KUQ_FORCE_SHARDS": "1", "KUQ_SHARD_BATCH_READS": "50",
                           "KUQ_EXACT_MERGE_SLOTS": "3000"}),
           "x": (["-x", "40K"], dict(WIDE, KUQ_DEVICE="0", KUQ_HBM_BUDGET="200000")),   # one context's rounds: half the reads
           "streamed": (["-x", "40K"], dict(WIDE, KUQ_DEVICES="0,0"))}


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_cli_spilled_golden(tmp_path, layout):
    """classifyExact with a capped table and a host budget, in every layout: the reference's Kraken lines and
    classifyExact report, and stderr tells that the set spilled and was settled"""
    _setup(tmp_path)
    extra, env = LAYOUTS[layout]
    err = _run(tmp_path, ["-M"] * (not extra) + extra + ["-r", "o.report", "-o", "o.kraken", "reads.fa"],
               dict(SPILL_ENV, **env))
    assert "spilled to host memory" in err and "[timing] exact set settled" in err, err[-3000:]
    spills = int(err.split("spilled to host memory ")[1].split(" times")[0])
    assert spills >= 1, err[-3000:]
    if layout == "shards":
        assert "sharded over 3 GPUs" in err, err[:1500]
    assert (tmp_path / "o.kraken").read_text() == open(os.path.join(G, "preload.kraken")).read()
    assert _report_rows(tmp_path / "o.report") == _report_rows(os.path.join(G, "exact.report.tsv"))


def test_cli_spilled_sample_sheet(tmp_path):
    """a two-row sheet with a capped table: every row writes the bytes of that row's separate run"""
    _setup(tmp_path)
    (tmp_path / "s.tsv").write_text("name\tinput\toutput\treport\n"
                                    "fa\treads.fa\ts.fa.kraken\ts.fa.report\nfq\treads_300.fq\ts.fq.kraken\ts.fq.report\n")
    err = _run(tmp_path, ["-M", "--sample-sheet", "s.tsv"], SPILL_ENV)
    assert "spilled to host memory" in err, err[-3000:]
    for name, inp in (("fa", "reads.fa"), ("fq", "reads_300.fq")):
        _run(tmp_path, ["-M", "-r", f"sep.{name}.report", "-o", f"sep.{name}.kraken", inp], SPILL_ENV)
        for ext in ("kraken", "report"):
            assert (tmp_path / f"s.{name}.{ext}").read_bytes() == (tmp_path / f"sep.{name}.{ext}").read_bytes(), (name, ext)
    assert _report_rows(tmp_path / "s.fa.report") == _report_rows(os.path.join(G, "exact.report.tsv"))


# ---- 5. larger -------------------------------------------------------------------------------------------------------
def test_cli_spilled_beyond_one_table(tmp_path):
    """test_cli_union_beyond_one_table's workload on one context capped at a quarter of the union, with a host budget:
    the report has the bytes of the uncapped one-context run"""
    tax, kdb, idx, seqs = _workload(46, n_reads=3000, random_frac=0.9)
    paths, taxdb, reads = _write(tmp_path, tax, kdb, idx, seqs)
    base = {"KUQ_BATCH_READS": "50", "KUQ_SPARSE_SLOTS": "1024", "KUQ_TIMING": "1", "KUQ_DEVICE": "0"}
    unit = ["-u", "7500"]

    def cli(name, env):
        out, rep = str(tmp_path / f"{name}.kraken"), str(tmp_path / f"{name}.report")
        cmd = [_exe(), "-d", paths[0][0], "-i", paths[0][1], "-a", taxdb, "-t", "1", "-M"] + unit + ["-r", rep, "-o", out, reads]
        r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, **env))
        assert r.returncode == 0, r.stderr[-3000:]
        return r.stderr, open(out, "rb").read(), open(rep, "rb").read()

    err, one_out, one_rep = cli("one", base)
    union = int(err.split("exact set of context 0: ")[1].split(" slots, ")[1].split(" pairs")[0])
    cap = 1 << int(round(np.log2(union / 4)))
    err, out, rep = cli("capped", dict(base, KUQ_EXACT_MAX_SLOTS=str(cap), KUQ_EXACT_HOST_BUDGET=str(1 << 30)))
    assert "spilled to host memory" in err, err[-3000:]
    assert rep == one_rep and out == one_out
