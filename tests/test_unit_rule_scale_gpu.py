"""The per-work-unit HLL rule (classify -M) at batch scale, against the oracle.

A taxon's sketch turns dense when one of its (work unit, taxon) sketches reaches 1025 distinct codes, or 1024 when
the last insert repeats a code.  The GPU decides this once per batch for every candidate pair (>= 1025 inserts).
These cases put thousands of candidates into one batch, put pairs into both tiers of the per-batch bookkeeping
(the dense (unit, taxon) table and the hash map past it) and run several batches through two slots.  Every case
counts its own inserts and distinct codes per pair with numpy first, so that a generator change cannot quietly
shrink it below what it claims to test."""
import os
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import binding, build, synth
from tests import util

pytestmark = pytest.mark.gpu
K = 31
U = 3000              # work-unit size: 20 reads of 150 bases
READ = 150
MISS = -1             # a source of reads that hit nothing (inserts on taxon 0)
_U64 = np.uint64


def _fmix64(x):
    """the reference's fmix64 (the key is incremented first)"""
    x = np.asarray(x, np.uint64) + _U64(1)
    with np.errstate(over="ignore"):
        x ^= x >> _U64(33)
        x *= _U64(0xff51afd7ed558ccd)
        x ^= x >> _U64(33)
        x *= _U64(0xc4ceb9fe1a85ec53)
        x ^= x >> _U64(33)
    return x


def _codes(oracle, canon):
    """encode_hash32(fmix64(canon)) for an array, checked against the oracle's scalar functions"""
    h = _fmix64(canon)
    idx = ((h >> _U64(39)) << _U64(7)).astype(np.uint32)
    out = idx.copy()
    rare = np.nonzero((idx << np.uint32(12)) == 0)[0]          # the rank-carrying encoding: let the oracle do it
    for i in rare.tolist():
        out[i] = oracle.encode_hash32(int(h[i]))
    for i in np.linspace(0, len(canon) - 1, min(len(canon), 64)).astype(np.int64).tolist():
        assert int(h[i]) == oracle.fmix64(int(canon[i]))
        assert int(out[i]) == oracle.encode_hash32(int(h[i]))
    return out


def _pair_stats(oracle, db_kmers, db_taxa, bases, offs, unit_id):
    """Inserts and distinct codes per (unit, taxon) pair as the reference's per-unit sketches see them: every valid
    window is an insert on its stored taxon (0 on a miss).  Windows across a '\\r' are skipped, so the counts
    are lower bounds there.  Returns {(unit, taxid): (inserts, distinct)} as arrays (unit, taxid, n, d)."""
    codes = synth.encode(bases)
    km, ok = synth.forward_kmers(codes, K)
    offs = np.asarray(offs, np.int64)
    lens = np.diff(offs)
    nwin = np.maximum(lens - K + 1, 0)
    read_of = np.repeat(np.arange(len(lens)), nwin)
    starts = offs[:-1][read_of] + np.arange(len(read_of)) - (np.cumsum(nwin) - nwin)[read_of]
    keep = ok[starts]
    starts, read_of = starts[keep], read_of[keep]
    canon = synth.canonical(km[starts], K)
    pos = np.minimum(np.searchsorted(db_kmers, canon), len(db_kmers) - 1)
    taxa = np.where(db_kmers[pos] == canon, db_taxa[pos], 0).astype(np.uint64)
    units = np.asarray(unit_id, np.uint64)[read_of]
    code = _codes(oracle, canon).astype(np.uint64)
    pair = (units << _U64(32)) | taxa
    up, n = np.unique(pair, return_counts=True)
    ud = np.unique((np.searchsorted(up, pair).astype(np.uint64) << _U64(32)) | code)
    d = np.bincount((ud >> _U64(32)).astype(np.int64), minlength=len(up))
    return (up >> _U64(32)).astype(np.int64), (up & _U64(0xFFFFFFFF)).astype(np.int64), n, d


def _species(seed, n_species=8, glen=200_000):
    rng = np.random.default_rng(seed)
    tax = synth.make_taxonomy(n_species)
    sp = synth.species_ids(tax)
    genomes = [rng.integers(0, 4, glen, dtype=np.uint8) for _ in range(n_species)]
    km, tx = synth.label_kmers(genomes, sp, tax, K)
    return rng, tax, sp, genomes, km, tx


def _unit_reads(rng, genomes, plan, cr_every=0):
    """One work unit per plan entry (a, b): 10 reads of source a and 10 of source b (MISS = random reads),
    interleaved at random.  With cr_every, every cr_every-th unit has a read with a '\\r' inside."""
    comp = np.array([3, 2, 1, 0], np.uint8)
    seqs = []
    for j, pair in enumerate(plan):
        src = np.repeat(np.array(pair), 10)
        rng.shuffle(src)
        for i, s in enumerate(src.tolist()):
            if s == MISS:
                r = rng.integers(0, 4, READ, dtype=np.uint8)
            else:
                g = genomes[s]
                p = int(rng.integers(0, len(g) - READ + 1))
                r = g[p:p + READ]
                if rng.random() < 0.5:
                    r = comp[r[::-1]]
            b = synth.decode(r).tobytes()
            if cr_every and j % cr_every == 0 and i == 7:
                b = b[:70] + b"\r" + b[70:]
            seqs.append(b)
    return seqs


def _plan(rng, n_units, sources):
    """two different sources per unit, drawn at random"""
    out = []
    for _ in range(n_units):
        a, b = rng.choice(len(sources), 2, replace=False).tolist()
        out.append((sources[a], sources[b]))
    return out


def _classifier(**kw):
    kw.setdefault("max_reads", 1 << 18)
    kw.setdefault("max_bases", 16 << 20)
    kw.setdefault("work_unit_size", U)
    kw.setdefault("sparse_set_slots", 1 << 23)
    return binding.Classifier(hll_mode=binding.HLL_PRELOAD, **kw)


def _subtrees(tax):
    kids = {}
    for t, p, _, _ in tax.rows:
        if t != p:
            kids.setdefault(p, []).append(t)
    out = []
    for t, _, _, _ in tax.rows:
        members, todo = [], [t]
        while todo:
            x = todo.pop()
            members.append(x)
            todo += kids.get(x, [])
        out.append(members)
    return out


def _check(clf, run, tax, got_calls, want_calls, max_clade_leaves=None):
    """calls, counters, tiers, estimates, registers of every taxon and every clade (with max_clade_leaves: every
    clade with children, and that many one-taxon clades)"""
    assert np.array_equal(got_calls, want_calls)
    got = clf.counts()
    want = run.counts(want_regs=True)
    for key in ("taxid", "n_reads", "n_kmers", "sparse", "unique"):
        bad = np.nonzero(got[key] != want[key])[0][:8] if len(got[key]) == len(want[key]) else []
        assert np.array_equal(got[key], want[key]), (key, [(int(want["taxid"][i]), int(want["n_kmers"][i]),
                                                             int(got[key][i]), int(want[key][i])) for i in bad])
    for j, t in enumerate(want["taxid"]):
        assert np.array_equal(clf.registers(int(t)), want["regs"][j]), f"registers of taxon {t}"
    clades = _subtrees(tax)
    if max_clade_leaves is not None:
        clades = [m for m in clades if len(m) > 1] + [m for m in clades if len(m) == 1][:max_clade_leaves]
    for members in clades:
        assert clf.clade(members) == run.clade(members), members
    return got


def _oracle_run(oracle, km, tx, tax, bases, offs, quick=0):
    kdb, idx = synth.build_db_images(km, tx, K, 10, 2)
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*tax.parent_map()), U, 0)
    if quick:
        run.set_quick(quick)
    calls, _, _ = run.classify(bases, offs, want_codes=False)
    run.finish()
    return kdb, idx, run, calls


# ---- (a) many candidates in one batch ----------------------------------------------------------------------------
# "below": ~3000 candidates with >= 1025 distinct codes; "above": >= 8000 (about 12 Mbp), more than a distinct-code
# set of 4 Mi entries shared by the whole batch could hold at ~1025 entries per candidate
@pytest.mark.parametrize("size,quick", [("below", 0), ("above", 0), ("above", 200)])
def test_many_candidates_in_one_batch(oracle, size, quick):
    rng, tax, sp, genomes, km, tx = _species(41)
    n_units = 1500 if size == "below" else 4100
    plan = _plan(rng, n_units, list(range(8)) + [MISS])
    bases, offs = synth.pack_reads(_unit_reads(rng, genomes, plan, cr_every=7))
    unit_id, _, _ = synth.work_unit_ids(offs, U)
    assert unit_id[-1] == n_units - 1 and len(offs) - 1 == 20 * n_units

    units, taxa, n, d = _pair_stats(oracle, km, tx, bases, offs, unit_id)
    cand = (n >= 1025) & (d >= 1025)
    assert 0 in taxa[cand].tolist()                                 # misses make taxon 0 a candidate too
    if size == "below":
        assert 2500 <= cand.sum() <= 3500
    else:
        assert cand.sum() >= 8000 and int(offs[-1]) >= 12_000_000

    kdb, idx, run, calls = _oracle_run(oracle, km, tx, tax, bases, offs, quick)
    clf = _classifier()
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*tax.parent_map())
    if quick:
        clf.set_quick_mode(quick)                                    # reads never reach 200 hits: all windows count
    res = clf.classify(bases, offs)                                  # one batch, units cut by the library
    clf.finish()
    got = _check(clf, run, tax, res["call"], calls)
    assert not got["sparse"][np.isin(got["taxid"], sp)].any()       # every species converted


# ---- (c) the 1024 corner in both tiers of one batch --------------------------------------------------------------
@pytest.mark.parametrize("order", ["ascending", "descending"])
def test_threshold_corner_in_both_tiers(oracle, order):
    """Pairs with exactly 1024 distinct codes whose last insert repeats a code (convert) or is new (stay sparse), and
    pairs with >= 1025 inserts but only 600 distinct codes (stay sparse), each in a unit inside the dense table and
    in a unit past it.  Caller-supplied unit ids with a gap put the second half past the table's last row.  Each of
    these taxa has this one pair, and 600 units of two-species reads come first: more candidates than k_unit_decide
    has CTAs, so the corner pairs are decided late, by CTAs that decided other pairs before.  "descending" numbers the
    same units the other way round (the C ABI accepts any ids; every pair is then in the map)."""
    rng = np.random.default_rng(43)
    kinds = ["repeat", "new", "few"]
    n_fill, n_sp = 600, 2 * len(kinds)
    tax = synth.make_taxonomy(8 + n_sp)
    sp = synth.species_ids(tax)
    fill_genomes = [rng.integers(0, 4, 200_000, dtype=np.uint8) for _ in range(8)]
    genomes = [rng.integers(0, 4, 1024 + K - 1 if j % 3 != 2 else 600 + K - 1, dtype=np.uint8) for j in range(n_sp)]
    km, tx = synth.label_kmers(fill_genomes + genomes, sp, tax, K)
    seqs = _unit_reads(rng, fill_genomes, _plan(rng, n_fill, list(range(8)) + [MISS]))
    unit_id, expect = list(np.repeat(np.arange(n_fill), 20)), {}
    sp = sp[8:]
    gap = 2000
    max_bases = 4 << 20
    for j in range(n_sp):
        kind, tier = kinds[j % 3], j // 3
        w = synth.decode(genomes[j]).tobytes()
        if kind == "repeat":                                         # 1024 codes, then a read of old k-mers
            group = [w, w[400:460]]
        elif kind == "new":                                          # repeats first; the 1024th code is the last insert
            group = [w[:200], w[:-1], w[-K:]]
        else:                                                        # 600 codes read twice: 1200 inserts
            group = [w, w]
        fill = U - sum(len(s) for s in group)                        # misses first, so that the unit ends with
        group = [synth.decode(rng.integers(0, 4, fill, dtype=np.uint8)).tobytes()] + group    # the group's last read
        seqs += group
        unit_id += [n_fill + j + gap * tier] * len(group)
        expect[sp[j]] = (kind, tier)
    unit_id = np.array(unit_id, np.int64)
    if order == "descending":
        unit_id = unit_id.max() - unit_id
    bases, offs = synth.pack_reads(seqs)
    ref_units, _, _ = synth.work_unit_ids(offs, U)
    assert np.array_equal(np.unique(ref_units, return_inverse=True)[1], np.unique(-unit_id, return_inverse=True)[1]
                          if order == "descending" else np.unique(unit_id, return_inverse=True)[1])

    units, taxa, n, d = _pair_stats(oracle, km, tx, bases, offs, unit_id)
    cand = (n >= 1025) & (d >= 1025)
    assert cand.sum() > 4 * 132                                      # more candidates than CTAs (4 per SM)
    stats = {int(t): (int(a), int(b), int(u)) for u, t, a, b in zip(units, taxa, n, d) if t in expect}
    for t, (kind, tier) in expect.items():
        ins, dist, unit = stats[t]
        assert ins >= 1025
        assert dist == (600 if kind == "few" else 1024), (t, kind, dist)

    kdb, idx, run, calls = _oracle_run(oracle, km, tx, tax, bases, offs)
    clf = _classifier(max_bases=max_bases)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*tax.parent_map())
    rows = clf.unit_table_rows()
    if order == "ascending":                                         # first tier inside the table, second past it
        for t, (kind, tier) in expect.items():
            assert (stats[t][2] >= rows) == (tier == 1)
    res = clf.classify(bases, offs, unit_id=unit_id.astype(np.uint32))
    clf.finish()
    got = _check(clf, run, tax, res["call"], calls)
    sparse = dict(zip(got["taxid"].tolist(), got["sparse"].tolist()))
    for t, (kind, tier) in expect.items():                           # both outcomes, in both tiers
        assert sparse[t] == (0 if kind == "repeat" else 1), (t, kind, tier)


# ---- (d) across batches and slots --------------------------------------------------------------------------------
def test_candidates_across_batches_and_slots(oracle):
    """Case (a)'s workload in 3 batches cut at unit boundaries, two in flight on two slots, counts read between
    batches.  Species 0 turns dense in batch 1 and has candidate pairs again later; species 7 only appears in
    batch 3."""
    rng, tax, sp, genomes, km, tx = _species(47)
    per = 500
    plan = _plan(rng, 2 * per, list(range(7)) + [MISS]) + _plan(rng, per, list(range(8)) + [MISS])
    plan = [(0, 1)] + plan[1:]
    plan[-1] = (7, MISS)
    bases, offs = synth.pack_reads(_unit_reads(rng, genomes, plan, cr_every=11))
    unit_id, _, _ = synth.work_unit_ids(offs, U)
    cuts = [0, 20 * per, 40 * per, 60 * per]
    assert np.all(unit_id[np.array(cuts[1:-1])] != unit_id[np.array(cuts[1:-1]) - 1])   # unit boundaries

    units, taxa, n, d = _pair_stats(oracle, km, tx, bases, offs, unit_id)
    cand = (n >= 1025) & (d >= 1025)
    batch = np.searchsorted(np.array([per, 2 * per]), units, side="right")
    assert cand[(taxa == sp[0]) & (batch == 0)].any() and cand[(taxa == sp[0]) & (batch == 2)].any()
    assert not (taxa == sp[7])[batch < 2].any() and cand[(taxa == sp[7]) & (batch == 2)].any()

    kdb, idx, run, calls = _oracle_run(oracle, km, tx, tax, bases, offs)
    clf = _classifier(n_slots=2)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*tax.parent_map())
    parts = [np.ascontiguousarray(offs[cuts[j]:cuts[j + 1] + 1]) for j in range(3)]
    got_calls = []
    clf.submit(0, bases.ctypes.data, parts[0])                       # batches 1 and 2 in flight together
    clf.submit(1, bases.ctypes.data, parts[1])
    got_calls.append(clf.wait(0, parts[0], copy=True)["call"])
    got_calls.append(clf.wait(1, parts[1], copy=True)["call"])
    mid = clf.counts()                                               # readout between batches
    assert not mid["sparse"][mid["taxid"] == sp[0]].any()
    assert sp[7] not in mid["taxid"].tolist() or mid["sparse"][mid["taxid"] == sp[7]].all()
    clf.submit(0, bases.ctypes.data, parts[2])
    got_calls.append(clf.wait(0, parts[2], copy=True)["call"])
    clf.finish()
    got = _check(clf, run, tax, np.concatenate(got_calls), calls)
    assert not got["sparse"][got["taxid"] == sp[7]].any()           # first a candidate in batch 3, and converted


# ---- (b) past the dense table ------------------------------------------------------------------------------------
def _decoy_taxonomy(tax, n_decoys):
    rows = list(tax.rows)
    genus = max(r[0] for r in rows) + 1
    ids = np.arange(genus + 1, genus + 1 + n_decoys, dtype=np.uint32)
    rows.append((genus, 1, "decoys", "genus"))
    rows += [(int(t), genus, f"decoy{i}", "species") for i, t in enumerate(ids.tolist())]
    return synth.Taxonomy(rows), ids


def test_pairs_past_the_dense_table(oracle):
    """50,000 decoy taxa with two k-mers each shrink the dense (unit, taxon) table to fewer rows than half the batch's
    units.  Every other unit is one 6 kb contig made of 187 decoys (> 32 taxa: resolve_overflow books it), so the
    units past the table put more than 100 k pairs into the hash map, next to the candidates of the two-species
    units in between."""
    rng, tax, sp, genomes, km, tx = _species(53)
    n_decoys, per_contig, n_units = 50_000, 187, 3000
    tax, decoy_ids = _decoy_taxonomy(tax, n_decoys)
    dseq = rng.integers(0, 4, (n_decoys, 32), dtype=np.uint8)
    dk = np.concatenate([synth.canonical(synth.forward_kmers(dseq[:, j:j + K].reshape(-1), K)[0][::K], K)
                         for j in range(2)])
    dt = np.concatenate([decoy_ids, decoy_ids])
    allk, first = np.unique(np.concatenate([km, dk]), return_index=True)
    km, tx = allk, np.concatenate([tx, dt])[first]
    two = _unit_reads(rng, genomes, _plan(rng, n_units // 2, list(range(8)) + [MISS]), cr_every=13)
    seqs = []
    for j in range(n_units // 2):
        seqs += two[20 * j:20 * j + 20]
        pick = (j * per_contig + np.arange(per_contig)) % n_decoys
        seqs.append(synth.decode(dseq[pick].reshape(-1)).tobytes())
    bases, offs = synth.pack_reads(seqs)
    unit_id, _, _ = synth.work_unit_ids(offs, U)
    assert unit_id[-1] == n_units - 1

    kdb, idx, run, calls = _oracle_run(oracle, km, tx, tax, bases, offs)
    # 1500 contigs take 1500 hit tables of 16 Ki entries: a slot for 128 MiB of bases has a large enough pool for them
    clf = _classifier(max_bases=128 << 20, n_slots=1)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*tax.parent_map())
    rows = clf.unit_table_rows()
    assert rows < n_units // 2                                       # at least half of the units past the table
    units, taxa, n, d = _pair_stats(oracle, km, tx, bases, offs, unit_id)
    cand = (n >= 1025) & (d >= 1025)
    in_map = int((units >= rows).sum() + (cand & (units < rows)).sum())
    assert 100_000 <= in_map < (1 << 21) // 2, in_map               # many pairs in the map, below half its capacity
    assert (np.bincount(units[taxa > 0])[1::2] >= 2 * 32).all()     # the contigs' units hit far more than 32 taxa
    res = clf.classify(bases, offs)
    clf.finish()
    _check(clf, run, tax, res["call"], calls, max_clade_leaves=200)


# ---- (e) the executable ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch_reads", [None, 20_000])
def test_classify_executable_at_scale(oracle, tmp_path, batch_reads):
    """`classify -M -u 3000` on a FASTQ of case (a)'s above-bound workload: in one batch, and cut into several with
    KUQ_BATCH_READS.  Every report row's reads / kmers equal the oracle's clade, and the Kraken lines its calls and hit
    lists."""
    rng, tax, sp, genomes, km, tx = _species(41)
    plan = _plan(rng, 4100, list(range(8)) + [MISS])
    seqs = _unit_reads(rng, genomes, plan)
    bases, offs = synth.pack_reads(seqs)
    ids = [f"r{i}" for i in range(len(seqs))]
    fq = tmp_path / "reads.fq"
    with open(fq, "wb") as f:
        for rid, s in zip(ids, seqs):
            f.write(b"@" + rid.encode() + b"\n" + s + b"\n+\n" + b"I" * len(s) + b"\n")
    kdb, idx = synth.build_db_images(km, tx, K, 10, 2)
    kdb.tofile(tmp_path / "database.kdb")
    idx.tofile(tmp_path / "database.idx")
    tax.write(str(tmp_path / "taxDB"))
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*tax.parent_map()), U, 0)
    calls, codes, code_off = run.classify(bases, offs)
    run.finish()
    want = run.counts()

    env = dict(os.environ)
    if batch_reads:
        env["KUQ_BATCH_READS"] = str(batch_reads)
    out, rep = tmp_path / "out.kraken", tmp_path / "out.report"
    r = subprocess.run([build.build_classify(), "-d", str(tmp_path / "database.kdb"), "-i", str(tmp_path / "database.idx"),
                        "-a", str(tmp_path / "taxDB"), "-M", "-u", str(U), "-t", "1", "-o", str(out), "-r", str(rep),
                        str(fq)], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    assert open(out).read() == util.kraken_lines(ids, seqs, calls, codes, code_off)
    rows = util.parse_report(rep)
    members = util.clade_members(tax.rows, want["taxid"][(want["n_reads"] > 0) | (want["n_kmers"] > 0)])
    assert set(sp) | {0} <= set(rows) <= set(members)
    for t, row in rows.items():
        u, nr, _ = run.clade(members[t])
        assert (row["reads"], row["kmers"]) == (nr, u), t
    assert all(rows[t]["kmers"] > 1024 for t in sp)                  # every species' clade is dense
