"""classifyExact on several GPUs: the exact k-mer set (KUQ_HLL_EXACT) grows on the device before batches that could fill
it, and kuq_merge_into unites the sets of replica and shard contexts.  On one H100 the GPUs are several contexts on
device 0 (KUQ_DEVICES=0,0); every result is compared with the oracle, and the merged state with one context that
classified all reads."""
import os
import subprocess

import numpy as np
import pytest
import torch

from krakenuniq_b200 import binding, build, synth
from tests import util
from tests.test_multi_db_gpu import _cli, _oracle, _report_matches_oracle, _workload, _write_inputs

pytestmark = pytest.mark.gpu
G = util.GOLDEN
DEV = "cuda:0"
KEYS = ("taxid", "n_reads", "n_kmers", "unique")


def _exact_workload(seed, n_reads):
    rng = np.random.default_rng(seed)
    tax = synth.make_taxonomy(12)
    genomes = synth.random_genomes(rng, 12, 3000, shared_frac=0.25)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, 31)
    kdb, idx = synth.build_db_images(km, tx, 31, 6, 1)
    bases, offs = synth.sample_reads(rng, genomes, n_reads, 150, 0.02, 0.2, 0.2)
    seqs = [bases[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n_reads)]
    return tax, kdb, idx, seqs


def _oracle_exact(oracle, tax, kdb, idx, seqs):
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*tax.parent_map()), 500000, 0)
    run.set_exact()
    calls, _, _ = run.classify(*synth.pack_reads(seqs), want_codes=False)
    run.finish()
    return calls, run.counts(), run


def _context(tax, kdb, idx, slots):
    clf = binding.Classifier(device=0, hll_mode=binding.HLL_EXACT, sparse_set_slots=slots, max_reads=1 << 14, max_bases=4 << 20)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*tax.parent_map())
    return clf


def _classify_batches(clf, seqs, sizes):
    """batches of the given read counts, two in flight on slots 0 and 1; returns the calls in read order"""
    parts, a = [], 0
    for n in sizes:
        parts.append(seqs[a:a + n])
        a += n
    assert a == len(seqs)
    calls = []
    for j in range(0, len(parts), 2):
        inflight = []
        for s, part in enumerate(parts[j:j + 2]):
            bases, offs = synth.pack_reads(part)
            clf.submit(s, bases.ctypes.data, offs)
            inflight.append((s, offs, bases))
        for s, offs, _ in inflight:
            calls.append(clf.wait(s, offs, copy=True)["call"])
    return np.concatenate(calls)


def _same_state(clf, want, run, tax):
    got = clf.counts()
    for key in KEYS:
        assert np.array_equal(got[key], want[key]), (key, got[key], want[key])
    members = util.clade_members(tax.rows, want["taxid"])
    assert len(members) > 5
    for taxid, mem in members.items():
        assert clf.clade(mem) == run.clade(mem), taxid
    # the roll-up the report uses gives the same unions
    ids = np.array(sorted(members), np.uint32)
    _, _, uniq = clf.clade_counts_tree(ids)
    assert [int(u) for u in uniq] == [run.clade(members[int(t)])[0] for t in ids]


def _pairs(clf):
    """the (k-mer + 1, dense taxon + 1) pairs a context holds (kuq_exact_export), sorted"""
    n = clf.exact_export()
    t = torch.zeros((max(n, 1), 2), dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    m = clf.exact_export(t.data_ptr(), n)
    assert m == n
    rows = t[:m].cpu().numpy().view(np.uint64)
    return rows[np.lexsort((rows[:, 0], rows[:, 1]))]


def test_exact_set_grows_from_a_tiny_table(oracle):
    """1024 slots to start with: small batches make the table grow step by step, two batches in flight, and a last batch
    larger than the whole table forces a growth on its own.  Calls, per-taxon set sizes and every clade union equal
    the oracle's."""
    tax, kdb, idx, seqs = _exact_workload(31, 3000)
    calls, want, run = _oracle_exact(oracle, tax, kdb, idx, seqs)
    clf = _context(tax, kdb, idx, 1 << 10)
    first = [20, 20, 40, 40, 80, 80, 160, 160]
    got = _classify_batches(clf, seqs[:sum(first)], first)
    before = clf.exact_info()
    assert before["pairs"] * 10 <= before["slots"] * 8
    last = seqs[sum(first):]
    res = clf.classify(*synth.pack_reads(last))
    after = clf.exact_info()
    assert (before["pairs"] + sum(len(s) for s in last)) * 10 > before["slots"] * 8    # its windows could fill the table
    assert after["times_grown"] > before["times_grown"] and after["slots"] > before["slots"]
    assert np.array_equal(np.concatenate([got, res["call"]]), calls)
    clf.finish()
    info = clf.exact_info()
    assert info["times_grown"] >= 3, info
    assert info["pairs"] == int(want["unique"].sum()) and info["pairs"] * 10 <= info["slots"] * 8
    _same_state(clf, want, run, tax)


def test_merge_of_exact_sets(oracle, monkeypatch):
    """three contexts on one device: the destination classifies a few reads in a tiny table, a second context the rest,
    with some reads given to both (their pairs must not count twice), a third stays idle.  After kuq_merge_into, which
    moves the pairs in rounds of 4096 slots here, the destination equals the oracle over every read given and one
    context that classified them all."""
    tax, kdb, idx, base = _exact_workload(32, 2400)
    part_dst, part_src = base[:300], base[150:]                     # reads 150..299 go to both
    seqs = part_dst + part_src
    calls, want, run = _oracle_exact(oracle, tax, kdb, idx, seqs)

    one = _context(tax, kdb, idx, 1 << 16)
    assert np.array_equal(_classify_batches(one, seqs, [600, 600, 600, 750]), calls)
    one.finish()
    _same_state(one, want, run, tax)

    dst = _context(tax, kdb, idx, 1 << 10)
    src = _context(tax, kdb, idx, 1 << 12)
    idle = _context(tax, kdb, idx, 1 << 10)
    got = [dst.classify(*synth.pack_reads(part_dst))["call"], _classify_batches(src, part_src, [1000, 1000, 250])]
    assert np.array_equal(np.concatenate(got), calls)
    for c in (dst, src, idle):
        c.finish()
    assert idle.exact_info()["pairs"] == 0
    before = dst.exact_info()
    n_src = src.exact_info()["pairs"]
    assert n_src * 10 > before["slots"] * 8                        # the import has to grow the destination
    monkeypatch.setenv("KUQ_EXACT_MERGE_SLOTS", "4096")
    dst.merge_from(src)
    dst.merge_from(idle)
    after = dst.exact_info()
    assert after["times_grown"] > before["times_grown"]
    assert after["pairs"] == one.exact_info()["pairs"] < before["pairs"] + n_src
    _same_state(dst, want, run, tax)
    assert np.array_equal(_pairs(dst), _pairs(one))


def test_exact_import_counts_only_new_pairs(oracle):
    """kuq_exact_export / kuq_exact_import as callers use them: importing a context's pairs twice adds them once"""
    tax, kdb, idx, seqs = _exact_workload(33, 400)
    _, want, run = _oracle_exact(oracle, tax, kdb, idx, seqs)
    a = _context(tax, kdb, idx, 1 << 10)
    a.classify(*synth.pack_reads(seqs))
    a.finish()
    b = _context(tax, kdb, idx, 1 << 10)
    b.classify(*synth.pack_reads(seqs[:1]))
    b.reset_counts()
    pairs = torch.from_numpy(_pairs(a).view(np.int64).copy()).to(DEV)
    torch.cuda.synchronize()
    for _ in range(2):
        b.exact_import(pairs.data_ptr(), pairs.shape[0])
    assert b.exact_info()["pairs"] == a.exact_info()["pairs"] == int(want["unique"].sum())
    assert np.array_equal(_pairs(b), _pairs(a))


# ---- the classifyExact executable -------------------------------------------------------------------------------
def _exact_exe():
    return os.path.join(os.path.dirname(build.build_classify()), "classifyExact")


def _report_lines(path):
    rows = {}
    for line in open(path):
        if line.startswith("#") or line.startswith("%"):
            continue
        f = line.rstrip("\n").split("\t")
        rows[f[6]] = f
    return rows


@pytest.mark.parametrize("layout", ["replicas", "shards"])
@pytest.mark.parametrize("extra", [["-M"], ["-M", "-u", "20000"]], ids=["M", "M_u20000"])
def test_cli_exact_two_contexts_golden(tmp_path, layout, extra):
    """classifyExact with two contexts on one device, as replicas (batches round-robin) and as minimizer-range shards,
    from a 1024-slot exact set: the reference's Kraken output and classifyExact report"""
    out, rep = tmp_path / "o.kraken", tmp_path / "o.report.tsv"
    cmd = [_exact_exe(), "-d", os.path.join(G, "database.kdb"), "-i", os.path.join(G, "database.idx"), "-a", os.path.join(G, "taxDB"),
           "-t", "1", "-r", str(rep), "-o", str(out)] + extra + [os.path.join(G, "reads.fa")]
    env = dict(os.environ, KUQ_DEVICES="0,0", KUQ_BATCH_READS="200", KUQ_SPARSE_SLOTS="1024")
    if layout == "shards":
        env["KUQ_FORCE_SHARDS"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "not usable" not in r.stderr
    assert ("sharded over 2 GPUs" if layout == "shards" else "2 GPUs, database replicated") in r.stderr, r.stderr[:1500]
    assert "-x rule" not in r.stderr and "streams" not in r.stderr
    assert open(out).read() == open(os.path.join(G, "preload.kraken")).read()
    assert _report_lines(rep) == _report_lines(os.path.join(G, "exact.report.tsv"))


def test_cli_exact_several_databases_sharded(oracle, tmp_path):
    """the three synthetic databases of test_multi_db_gpu (nt 9 / 7 / 9, both index types, stored zeros), sharded over two
    contexts: the oracle's Kraken lines and report, and the bytes of the one-context resident run"""
    tax, dbs, seqs = _workload(21, 31, [(9, 2), (7, 1), (9, 2)], n_reads=20000)
    paths = _write_inputs(tmp_path, tax, dbs, seqs)
    ids, rseqs = util.read_fasta(str(tmp_path / "reads.fa"))
    unit = 30000
    calls, codes, code_off, cnt, _, run = _oracle(oracle, tax, dbs, rseqs, unit, exact=True)
    want = util.kraken_lines(ids, rseqs, calls, codes, code_off)
    got = {}
    for mode, env in (("resident", {"KUQ_DEVICE": "0"}),
                      ("sharded", {"KUQ_FORCE_SHARDS": "1", "KUQ_DEVICES": "0,0", "KUQ_SPARSE_SLOTS": "1024"})):
        out = tmp_path / mode
        out.mkdir()
        kraken, rows, err = _cli(_exact_exe(), paths, str(tmp_path / "taxDB"), str(tmp_path / "reads.fa"), str(out), ["-u", str(unit)], env)
        assert kraken == want, mode
        _report_matches_oracle(str(out / "o.report.tsv"), tax, cnt, run)
        got[mode] = (kraken, rows)
        if mode == "sharded":
            assert "3 databases sharded over 2 GPUs by minimizer range" in err, err[-2000:]
            assert "streams" not in err
        else:
            assert "3 databases resident on 1 GPU(s)" in err, err[-2000:]
    assert got["resident"] == got["sharded"]
