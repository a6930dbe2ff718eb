"""classifyExact's k-mer set partitioned by k-mer over contexts, and every report clade rolled up from one sort.

Exact distinct counts add up over any partition of the k-mer space, so the contexts of a run keep disjoint parts of
the (k-mer, taxon) pairs instead of uniting them on one card, and a clade's union is the sum of per-node books
(pairs − adjacent equal-k-mer pairs booked at their LCA) over its subtree.  On one H100 the GPUs are several contexts
on device 0; results are held against the oracle (`run.set_exact()`, `run.clade(members)`) and against pairs crafted
so that one k-mer sits under several taxa, which reads never produce (a window's taxon is a function of its k-mer)."""
import os
import subprocess

import numpy as np
import pytest
import torch

from krakenuniq_b200 import binding, build, dist, synth
from tests import util
from tests.local_group import run_ranks

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEYS = ("taxid", "n_reads", "n_kmers", "unique")
MISSING = 990001                        # a database taxon without a taxonomy row


# ---- a deep and wide taxonomy --------------------------------------------------------------------------------------
def _deep_wide_taxonomy():
    """root → 24 families → 4 genera → 4 species (wide), a chain of 36 ranks under the root with species at several
    depths (deep), and leaves that no genome feeds (taxa without k-mers).  → (Taxonomy, taxa that get a genome)"""
    rows = [(1, 1, "root", "no rank")]
    nid, fed = 100, []
    for f in range(24):
        fam = nid
        rows.append((fam, 1, f"family{f}", "family"))
        nid += 1
        for g in range(4):
            gen = nid
            rows.append((gen, fam, f"genus{f}_{g}", "genus"))
            nid += 1
            for s in range(4):
                rows.append((nid, gen, f"species{f}_{g}_{s}", "species"))
                if (f + g + s) % 3:                 # a third of the species get no genome
                    fed.append(nid)
                nid += 1
    parent = 1
    for d in range(36):
        rows.append((nid, parent, f"rank{d}", "no rank"))
        if d in (4, 11, 19, 27, 35):
            rows.append((nid + 1, nid, f"deep{d}", "species"))
            fed.append(nid + 1)
        parent = nid
        nid += 2
    return synth.Taxonomy(rows), fed


def _workload(seed, n_genomes=150, n_reads=6000, random_frac=0.2):
    rng = np.random.default_rng(seed)
    tax, fed = _deep_wide_taxonomy()
    taxa = [int(t) for t in rng.choice(fed, n_genomes - 1, replace=False)] + [MISSING]
    genomes = synth.random_genomes(rng, n_genomes, 1500, shared_frac=0.3)
    km, tx = synth.label_kmers(genomes, taxa, tax, 31)
    kdb, idx = synth.build_db_images(km, tx, 31, 7, 2)
    bases, offs = synth.sample_reads(rng, genomes, n_reads, 150, 0.02, 0.0, random_frac)
    seqs = [bases[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n_reads)]
    return tax, kdb, idx, seqs


def _oracle(oracle, tax, kdb, idx, seqs):
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*tax.parent_map()), 500000, 0)
    run.set_exact()
    calls, _, _ = run.classify(*synth.pack_reads(seqs), want_codes=False)
    run.finish()
    return calls, run.counts(), run


def _context(tax, kdb, idx, slots=1 << 16):
    clf = binding.Classifier(device=0, hll_mode=binding.HLL_EXACT, sparse_set_slots=slots, max_reads=1 << 14, max_bases=4 << 20)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*tax.parent_map())
    return clf


def _classify(clf, seqs, batch=2000):
    out = [clf.classify(*synth.pack_reads(seqs[a:a + batch]))["call"] for a in range(0, len(seqs), batch)]
    return np.concatenate(out) if out else np.zeros(0, np.uint32)


def _tree(clf, ids):
    _, _, u = clf.clade_counts_tree(np.array(ids, np.uint32))
    return [int(x) for x in u]


def _pairs(clf):
    """the pairs a context holds as rows (k-mer + 1, dense taxon + 1), uint64"""
    n = clf.exact_export()
    t = torch.zeros((max(n, 1), 2), dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    assert clf.exact_export(t.data_ptr(), n) == n
    return t[:n].cpu().numpy().view(np.uint64)


def _owner(kmers, n_parts):
    """kuq_exact_owner in numpy (kuq.h)"""
    with np.errstate(over="ignore"):
        x = np.asarray(kmers, np.uint64) ^ np.uint64(0x2545F4914F6CDD1D)
        x ^= x >> np.uint64(30)
        x *= np.uint64(0xbf58476d1ce4e5b9)
        x ^= x >> np.uint64(27)
        x *= np.uint64(0x94d049bb133111eb)
        x ^= x >> np.uint64(31)
    return (((x >> np.uint64(32)) * np.uint64(n_parts)) >> np.uint64(32)).astype(np.int64)


def _check_against_oracle(clf, want, run, tax):
    got = clf.counts()
    for key in KEYS:
        assert np.array_equal(got[key], want[key]), key
    members = util.clade_members(tax.rows, want["taxid"])
    ids = sorted(members)
    assert _tree(clf, ids) == [run.clade(members[t])[0] for t in ids]
    return members


# ---- crafted pairs: one k-mer under several taxa --------------------------------------------------------------------
def _crafted_pairs(clf, tax, rng, n_kmers=20000):
    """pairs (k-mer, dense taxon) with 1–4 taxa per k-mer, mostly close relatives, some under taxon 0 and the root"""
    dense = clf.dense_taxids()
    n_sketch = clf.state_ptrs().n_sketch
    parent = {t: p for t, p, _, _ in tax.rows}
    sketch = np.arange(n_sketch)
    by_parent = {}
    for d in sketch[2:]:
        by_parent.setdefault(parent.get(int(dense[d]), 0), []).append(int(d))
    groups = [g for g in by_parent.values()]
    kmers = rng.integers(0, 1 << 62, n_kmers, dtype=np.uint64)
    rows = []
    for i, k in enumerate(kmers):
        m = int(rng.integers(1, 5))
        if i % 3 == 0:                                      # siblings: LCA at their genus / rank
            g = groups[int(rng.integers(0, len(groups)))]
            taxa = rng.choice(g, min(m, len(g)), replace=False)
        else:
            taxa = rng.choice(sketch, m, replace=False)
        rows += [(int(k), int(t)) for t in taxa]
    rows = np.array(rows, np.uint64)
    return rows, dense


def _install_crafted(clf, rows):
    """the pairs into a context whose counters were reset, and one counted k-mer per taxon that holds some (so that
    the taxa count as members, as every pair's taxon does after a run)"""
    t = torch.from_numpy((rows + np.uint64(1)).view(np.int64).copy()).to(DEV)
    torch.cuda.synchronize()
    clf.exact_import(t.data_ptr(), t.shape[0])
    sp = clf.state_ptrs()
    nk = dist.device_view(sp.d_n_kmers, sp.n_sketch * 8, torch.int64, DEV)
    for d in np.unique(rows[:, 1]):
        nk[int(d)] += 1
    torch.cuda.synchronize()


def _crafted_expect(tax, rows, dense, counted):
    members = util.clade_members(tax.rows, counted)
    by_taxon = {}
    for k, d in rows:
        by_taxon.setdefault(int(dense[int(d)]), set()).add(int(k))
    return {c: len(set().union(*[by_taxon.get(t, set()) for t in mem])) for c, mem in members.items()}, members


def _check_crafted(clf, tax, rows, dense):
    counted = clf.counts()["taxid"]
    want, members = _crafted_expect(tax, rows, dense, counted)
    ids = sorted(want)
    assert _tree(clf, ids) == [want[c] for c in ids]
    assert sum(1 for c in ids if len(members[c]) > 1) > 80
    return want, members


# ---- 1. the roll-up on one context --------------------------------------------------------------------------------
def test_rollup_matches_oracle_and_member_unions(oracle, monkeypatch):
    """every clade of a deep and wide taxonomy (chains deeper than 30, taxa without k-mers, a database taxon missing
    from the tree) from kuq_clade_counts_tree equals the oracle and kuq_clade_counts of its member list; again with a
    sort budget that forces several k-mer passes; the table grew from 1024 slots"""
    tax, kdb, idx, seqs = _workload(41)
    calls, want, run = _oracle(oracle, tax, kdb, idx, seqs)
    clf = _context(tax, kdb, idx, 1 << 10)
    assert np.array_equal(_classify(clf, seqs, 500), calls)
    clf.finish()
    assert clf.exact_info()["times_grown"] > 0
    assert MISSING in set(int(t) for t in want["taxid"])
    members = _check_against_oracle(clf, want, run, tax)
    assert sum(1 for m in members.values() if len(m) > 1) > 100
    ids = sorted(members)
    for t in ids:
        assert clf.clade(members[t])[0] == run.clade(members[t])[0], t
    assert clf.exact_rollup_passes() == 1
    pairs = clf.exact_info()["pairs"]
    monkeypatch.setenv("KUQ_EXACT_ROLLUP_BUDGET", str(pairs * 48 // 5))
    assert _tree(clf, ids) == [run.clade(members[t])[0] for t in ids]
    assert clf.exact_rollup_passes() >= 5


def test_rollup_of_kmers_shared_by_several_taxa(oracle, monkeypatch):
    """pairs crafted so that one k-mer sits under up to four taxa (siblings, cousins, taxon 0, the root): every clade
    from the roll-up equals the union of its members' sets, counted in numpy and by kuq_clade_counts; in one pass and
    in seven"""
    tax, kdb, idx, seqs = _workload(42, n_reads=10)
    clf = _context(tax, kdb, idx, 1 << 10)
    clf.classify(*synth.pack_reads(seqs))
    clf.reset_counts()
    rows, dense = _crafted_pairs(clf, tax, np.random.default_rng(5))
    _install_crafted(clf, rows)
    want, members = _check_crafted(clf, tax, rows, dense)
    for c in sorted(want)[::7]:
        assert clf.clade(members[c])[0] == want[c], c
    monkeypatch.setenv("KUQ_EXACT_ROLLUP_BUDGET", str(len(rows) * 48 // 7))
    _check_crafted(clf, tax, rows, dense)
    assert clf.exact_rollup_passes() >= 7


# ---- 2. the partition through the C ABI -----------------------------------------------------------------------------
def _partition_by_hand(ctxs):
    """kuq_exact_export_partitioned on every context, the parts exchanged on the device, kuq_exact_replace, and the
    summaries summed onto the first context"""
    world = len(ctxs)
    parts = []
    for c in ctxs:
        counts = c.exact_export_partitioned(world)
        buf = torch.zeros((max(int(counts.sum()), 1), 2), dtype=torch.int64, device=DEV)
        torch.cuda.synchronize()
        assert np.array_equal(c.exact_export_partitioned(world, buf.data_ptr(), buf.shape[0]), counts)
        offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        parts.append([buf[offs[o]:offs[o + 1]] for o in range(world)])
    for o, c in enumerate(ctxs):
        recv = torch.cat([parts[g][o] for g in range(world)]).contiguous()
        torch.cuda.synchronize()
        c.exact_replace(recv.data_ptr() if recv.shape[0] else None, recv.shape[0])
    sp = ctxs[0].state_ptrs()
    count = torch.zeros(sp.n_sketch, dtype=torch.int64, device=DEV)
    books = torch.zeros(sp.n_taxa, dtype=torch.int64, device=DEV)
    for c in ctxs:
        cc = torch.zeros_like(count)
        bb = torch.zeros_like(books)
        torch.cuda.synchronize()
        c.exact_summary(cc.data_ptr(), bb.data_ptr())
        torch.cuda.synchronize()
        count += cc
        books += bb
    torch.cuda.synchronize()
    ctxs[0].set_exact_summary(count.data_ptr(), books.data_ptr())


def _check_parts(ctxs, union_pairs):
    """pairs summed over the contexts = the union; each pair on its owner, none on two contexts"""
    rows = [_pairs(c) for c in ctxs]
    assert sum(len(r) for r in rows) == union_pairs
    for o, r in enumerate(rows):
        if len(r):
            assert (_owner(r[:, 0] - np.uint64(1), len(ctxs)) == o).all()
            for k in r[:5, 0]:
                assert ctxs[0].exact_owner(int(k) - 1, len(ctxs)) == o
    allr = np.concatenate(rows)
    assert len(np.unique(allr, axis=0)) == len(allr)


def test_partition_through_the_c_abi(oracle):
    """three contexts: one idle, some reads given to the two others.  After counters merge, partitioned export,
    exchange, replace, summary and set-summary: per-taxon `unique` and every clade equal the oracle, the parts add
    up to the union, every pair sits on its owner, and unions over member lists are refused"""
    tax, kdb, idx, base = _workload(43, n_reads=4000)
    a_reads, b_reads = base[:2500], base[1500:]
    seqs = a_reads + b_reads
    _, want, run = _oracle(oracle, tax, kdb, idx, seqs)
    a, b, idle = _context(tax, kdb, idx, 1 << 10), _context(tax, kdb, idx, 1 << 12), _context(tax, kdb, idx, 1 << 10)
    _classify(a, a_reads, 700)
    _classify(b, b_reads, 900)
    for c in (a, b):
        c.finish()
    a.merge_counters_from(b)
    a.merge_counters_from(idle)
    _partition_by_hand([a, b, idle])
    _check_against_oracle(a, want, run, tax)
    _check_parts([a, b, idle], int(want["unique"].sum()))
    with pytest.raises(RuntimeError, match="partitioned"):
        a.clade([int(t) for t in want["taxid"][:3]])


def test_partition_of_shared_kmers_in_one_process(oracle):
    """crafted pairs spread over three contexts with overlaps (a pair held by two senders collapses at its owner):
    kuq_exact_partition leaves the same clades as one context holding all pairs"""
    tax, kdb, idx, seqs = _workload(44, n_reads=10)
    ctxs = [_context(tax, kdb, idx, 1 << 10) for _ in range(3)]
    for c in ctxs:
        c.classify(*synth.pack_reads(seqs))
        c.reset_counts()
    rows, dense = _crafted_pairs(ctxs[0], tax, np.random.default_rng(6))
    rng = np.random.default_rng(7)
    where = rng.integers(0, 3, len(rows))
    extra = rng.random(len(rows)) < 0.2                         # a fifth of the pairs go to a second context as well
    for g, c in enumerate(ctxs):
        _install_crafted(c, rows[(where == g) | (extra & (where == (g + 1) % 3))])
    for g in (1, 2):
        ctxs[0].merge_counters_from(ctxs[g])
    binding.Classifier.exact_partition(ctxs)
    _check_crafted(ctxs[0], tax, rows, dense)
    _check_parts(ctxs, len(rows))


# ---- 3. the classifyExact executable --------------------------------------------------------------------------------
def _exact_exe():
    return os.path.join(os.path.dirname(build.build_classify()), "classifyExact")


def _run_cli(paths, taxdb, reads, out_dir, env, extra=()):
    os.makedirs(out_dir, exist_ok=True)
    out, rep = os.path.join(out_dir, "o.kraken"), os.path.join(out_dir, "o.report.tsv")
    cmd = [_exact_exe()]
    for kdb, idx in paths:
        cmd += ["-d", kdb, "-i", idx]
    cmd += ["-a", taxdb, "-t", "1", "-M"] + list(extra) + ["-r", rep, "-o", out, reads]
    r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, **env))
    return r, out, rep


# three replica contexts do not fit one 80 GB card (each takes three batch slots of 288 MiB of bases); three shard
# contexts take two slots each
@pytest.mark.parametrize("layout,devices", [("replicas", "0,0"), ("shards", "0,0"), ("shards", "0,0,0")])
@pytest.mark.parametrize("batch_min", [None, "100000"], ids=["tree", "few_clades"])
def test_cli_golden_partitioned(tmp_path, layout, devices, batch_min):
    """classifyExact on two and three contexts of one device, replicas and shards, with the report's usual roll-up and
    with the small-report path (fewer clades than KUQ_REPORT_BATCH_MIN): the reference's Kraken output and report"""
    G = util.GOLDEN
    env = {"KUQ_DEVICES": devices, "KUQ_BATCH_READS": "200", "KUQ_SPARSE_SLOTS": "1024", "KUQ_TIMING": "1"}
    if layout == "shards":
        env["KUQ_FORCE_SHARDS"] = "1"
    if batch_min:
        env["KUQ_REPORT_BATCH_MIN"] = batch_min
    r, out, rep = _run_cli([(os.path.join(G, "database.kdb"), os.path.join(G, "database.idx"))], os.path.join(G, "taxDB"),
                           os.path.join(G, "reads.fa"), str(tmp_path), env)
    assert r.returncode == 0, r.stderr[-2000:]
    n = devices.count(",") + 1
    assert f"exact set of context {n - 1}" in r.stderr
    assert open(out).read() == open(os.path.join(G, "preload.kraken")).read()
    assert util.parse_report(rep) == util.parse_report(os.path.join(G, "exact.report.tsv"))


def _write(tmp_path, tax, kdb, idx, seqs):
    kp, ip = str(tmp_path / "db.kdb"), str(tmp_path / "db.idx")
    kdb.tofile(kp)
    idx.tofile(ip)
    tax.write(str(tmp_path / "taxDB"))
    with open(tmp_path / "reads.fa", "wb") as f:
        for i, s in enumerate(seqs):
            f.write(b">r%d\n%s\n" % (i, s))
    return [(kp, ip)], str(tmp_path / "taxDB"), str(tmp_path / "reads.fa")


def test_cli_deep_taxonomy_report_is_the_one_context_report(tmp_path):
    """on the deep and wide taxonomy, the partitioned runs write the bytes of the one-context run"""
    tax, kdb, idx, seqs = _workload(45, n_reads=8000)
    paths, taxdb, reads = _write(tmp_path, tax, kdb, idx, seqs)
    got = {}
    for name, env in (("one", {"KUQ_DEVICE": "0"}), ("two", {"KUQ_DEVICES": "0,0"}),
                      ("three_shards", {"KUQ_DEVICES": "0,0,0", "KUQ_FORCE_SHARDS": "1"})):
        env = dict(env, KUQ_BATCH_READS="1000", KUQ_SPARSE_SLOTS="1024")
        r, out, rep = _run_cli(paths, taxdb, reads, str(tmp_path / name), env)
        assert r.returncode == 0, r.stderr[-2000:]
        got[name] = (open(out).read(), open(rep).read())
    assert got["two"] == got["one"] and got["three_shards"] == got["one"]


# ---- 4. a union larger than one context's table ---------------------------------------------------------------------
def test_cli_union_beyond_one_table(tmp_path):
    """KUQ_EXACT_MAX_SLOTS below the union but above each part: two contexts complete with the one-context report; one
    context fails with KUQ_E_NOMEM naming the exact set"""
    tax, kdb, idx, seqs = _workload(46, n_reads=3000, random_frac=0.9)
    paths, taxdb, reads = _write(tmp_path, tax, kdb, idx, seqs)
    base = {"KUQ_BATCH_READS": "50", "KUQ_SPARSE_SLOTS": "1024", "KUQ_TIMING": "1"}
    unit = ["-u", "7500"]                                       # batches end at work-unit boundaries: ~50 reads each
    r, out, rep = _run_cli(paths, taxdb, reads, str(tmp_path / "probe"), extra=unit, env=dict(base, KUQ_DEVICE="0"))
    assert r.returncode == 0, r.stderr[-2000:]
    union = int(r.stderr.split("exact set of context 0: ")[1].split(" slots, ")[1].split(" pairs")[0])
    # about as many reads as put the union at a power of two P: one table must grow past P, a part of half fits
    cap = 1 << int(round(np.log2(union)))
    seqs = seqs[:int(len(seqs) * cap / union)]
    paths, taxdb, reads = _write(tmp_path, tax, kdb, idx, seqs)
    one, _, one_rep = _run_cli(paths, taxdb, reads, str(tmp_path / "one"), extra=unit, env=dict(base, KUQ_DEVICE="0"))
    assert one.returncode == 0, one.stderr[-2000:]
    union = int(one.stderr.split("exact set of context 0: ")[1].split(" slots, ")[1].split(" pairs")[0])
    assert 0.85 * cap < union < 1.15 * cap, (union, cap)
    env = dict(base, KUQ_EXACT_MAX_SLOTS=str(cap))
    two, _, two_rep = _run_cli(paths, taxdb, reads, str(tmp_path / "two"), extra=unit, env=dict(env, KUQ_DEVICES="0,0"))
    assert two.returncode == 0, two.stderr[-2000:]
    assert open(two_rep).read() == open(one_rep).read()
    capped, _, _ = _run_cli(paths, taxdb, reads, str(tmp_path / "capped"), extra=unit, env=dict(env, KUQ_DEVICE="0"))
    assert capped.returncode != 0
    assert "exact k-mer set" in capped.stderr and "no room" in capped.stderr, capped.stderr[-2000:]


# ---- 5. dist.merge_exact_partitioned --------------------------------------------------------------------------------
def test_dist_merge_exact_partitioned(oracle):
    """one thread per context, the collectives of tests/local_group: every rank reports the oracle's counts and
    clades, and the ranks hold disjoint parts that add up to the union"""
    tax, kdb, idx, base = _workload(47, n_reads=4500)
    shares = [base[:1800], base[1200:3000], base[3000:]]
    _, want, run = _oracle(oracle, tax, kdb, idx, [s for sh in shares for s in sh])
    ctxs = [_context(tax, kdb, idx, 1 << 10) for _ in shares]
    for c, sh in zip(ctxs, shares):
        _classify(c, sh, 800)
        c.finish()

    def rank(r, coll):
        dist.merge_exact_partitioned(ctxs[r], DEV, coll)
        return ctxs[r].counts()

    outs = run_ranks(len(ctxs), rank)
    for got in outs:
        for key in KEYS:
            assert np.array_equal(got[key], want[key]), key
    for c in ctxs:
        _check_against_oracle(c, want, run, tax)
    _check_parts(ctxs, int(want["unique"].sum()))
