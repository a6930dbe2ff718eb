"""The record tier of the sparse HLL tier: a harvest marks the records whose (taxon, code) key is in the tier
(KEPT_BIT) instead of inserting the keys into the set.  Two records of one taxon can share a code (the code keeps
about the top 25 bits of the k-mer's hash); only one of them, the primary, may hold the key.  These tests place
such collisions in a database on purpose — k-mers chosen on the CPU whose hashes share `fmix64 >> 39` — and compare
every per-taxon and per-clade number with the oracle."""
import numpy as np
import pytest

from krakenuniq_b200 import binding, synth

pytestmark = pytest.mark.gpu
K = 31
TAX = synth.Taxonomy([(1, 1, "root", "no rank"), (10, 1, "g", "genus"), (11, 10, "a", "species"),
                      (12, 10, "b", "species"), (20, 1, "h", "genus"), (21, 20, "c", "species")])


def _fmix64(x):
    with np.errstate(over="ignore"):
        x = x + np.uint64(1)
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xff51afd7ed558ccd)
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xc4ceb9fe1a85ec53)
        x ^= x >> np.uint64(33)
    return x


def _kmer_pool(seed=5, n=400_000):
    """(pairs, singles): pairs of canonical k-mers with equal codes, and k-mers whose codes no other k-mer shares.
    Codes whose low 13 index bits are zero also carry a rank (encodeHashIn32Bit); those k-mers are left out."""
    rng = np.random.default_rng(seed)
    km = np.unique(synth.canonical(rng.integers(0, 1 << 62, n, dtype=np.uint64), K))
    top = _fmix64(km) >> np.uint64(39)
    km, top = km[(top & np.uint64(0x1FFF)) != 0], top[(top & np.uint64(0x1FFF)) != 0]
    order = np.argsort(top, kind="stable")
    km, top = km[order], top[order]
    _, first, count = np.unique(top, return_index=True, return_counts=True)
    pairs = [(km[f], km[f + 1]) for f, c in zip(first, count) if c == 2]
    singles = km[first[count == 1]]
    return pairs, singles


PAIRS, SINGLES = _kmer_pool()


def _read(kmer):
    codes = (int(kmer) >> (2 * (K - 1 - np.arange(K)))) & 3
    return synth.decode(codes.astype(np.uint8)).tobytes()


def _db(by_taxon):
    km = np.concatenate([np.asarray(v, np.uint64) for v in by_taxon.values()])
    tx = np.concatenate([np.full(len(v), t, np.uint32) for t, v in by_taxon.items()])
    assert len(np.unique(km)) == len(km)
    order = np.argsort(km)
    return synth.build_db_images(km[order], tx[order], K, 8, 2)


def _compare(oracle, kdb, idx, batches, mode=binding.HLL_PRELOAD, readout_between=False, clades=()):
    """classify `batches` (lists of k-mers, one read each) in one context and in the oracle; per-taxon and clade
    numbers must be equal.  readout_between: a readout (= a harvest) after every batch."""
    db = oracle.open_db(kdb, idx)
    run = oracle.run(db, oracle.parent_map(*TAX.parent_map()), 500000, 0 if mode == binding.HLL_PRELOAD else 1)
    clf = binding.Classifier(max_reads=1 << 12, max_bases=1 << 20, hll_mode=mode, sparse_set_slots=1 << 12)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*TAX.parent_map())
    for b in batches:
        bases, offs = synth.pack_reads([_read(x) for x in b])
        run.classify(bases, offs, want_codes=False)
        clf.classify(bases, offs)
        if readout_between:
            clf.counts()
    run.finish()
    clf.finish()
    _assert_same(clf, run, clades)
    return clf, run


def _assert_same(clf, run, clades=()):
    got, want = clf.counts(), run.counts()
    for key in ("taxid", "n_reads", "n_kmers", "sparse", "unique"):
        assert np.array_equal(got[key], want[key]), (key, got[key], want[key])
    for mem in clades:
        assert clf.clade(mem) == run.clade(mem), mem


def _species_a(n_pairs, n_single):
    pairs = PAIRS[:n_pairs]
    return pairs, SINGLES[:n_single]


@pytest.mark.parametrize("hits", ["first", "second", "both", "both_split"])
def test_colliding_records_of_one_taxon(oracle, hits):
    """only one member of each colliding pair is hit (whichever is the secondary), or both — in one harvest or in
    two.  Without the collision table a taxon would count the shared code twice."""
    pairs, single = _species_a(6, 40)
    kdb, idx = _db({11: np.concatenate([np.array(pairs).ravel(), single[:30]]), 12: single[30:]})
    first, second = [p[0] for p in pairs], [p[1] for p in pairs]
    rest = list(single)
    if hits == "first":
        batches = [first + rest]
    elif hits == "second":
        batches = [second + rest]
    elif hits == "both":
        batches = [first + rest + second]
    else:
        batches = [first + rest[:20], second + rest[20:]]
    _compare(oracle, kdb, idx, batches, readout_between=hits == "both_split")


def test_reset_then_the_same_run_again(oracle):
    pairs, single = _species_a(4, 20)
    kdb, idx = _db({11: np.concatenate([np.array(pairs).ravel(), single[:10]]), 12: single[10:]})
    batch = [p[1] for p in pairs] + list(single) + [p[0] for p in pairs[:2]]
    clf, run = _compare(oracle, kdb, idx, [batch])
    clf.reset_counts()
    bases, offs = synth.pack_reads([_read(x) for x in batch])
    clf.classify(bases, offs)
    clf.finish()
    _assert_same(clf, run)


@pytest.mark.parametrize("n_single,n_pairs", [(1023, 1), (1024, 1)])
def test_chunked_rule_at_the_boundary_with_collisions(oracle, n_single, n_pairs):
    """chunked rule: a taxon converts iff its sketch holds >= 1025 distinct codes.  1023 + one colliding pair =
    1025 k-mers but 1024 codes: the taxon stays sparse; one more k-mer and it converts."""
    pairs, single = _species_a(n_pairs, n_single + 10)
    kdb, idx = _db({11: np.concatenate([np.array(pairs).ravel(), single[:n_single]]), 12: single[n_single:]})
    batch = [x for p in pairs for x in p] + list(single)
    clf, run = _compare(oracle, kdb, idx, [batch], mode=binding.HLL_CHUNKED)
    sparse_of_11 = dict(zip(run.counts()["taxid"].tolist(), run.counts()["sparse"].tolist()))[11]
    assert sparse_of_11 == (n_single + n_pairs < 1025)


def test_merge_of_two_contexts(oracle):
    """kuq_merge_into: the destination's kept records move into its set before the source's keys are imported"""
    pairs, single = _species_a(5, 30)
    kdb, idx = _db({11: np.concatenate([np.array(pairs).ravel(), single[:20]]), 12: single[20:]})
    part_dst = [x for p in pairs for x in p] + list(single[:15])
    part_src = [p[0] for p in pairs] + list(single[15:])
    db = oracle.open_db(kdb, idx)
    run = oracle.run(db, oracle.parent_map(*TAX.parent_map()), 500000, 0)
    ctx = []
    for part in (part_dst, part_src):
        bases, offs = synth.pack_reads([_read(x) for x in part])
        run.classify(bases, offs, want_codes=False)
        c = binding.Classifier(max_reads=1 << 12, max_bases=1 << 20, hll_mode=binding.HLL_PRELOAD, sparse_set_slots=1 << 12)
        c.stage_db(kdb, idx)
        c.set_taxonomy(*TAX.parent_map())
        c.classify(bases, offs)
        c.finish()
        ctx.append(c)
    run.finish()
    ctx[0].merge_from(ctx[1])
    _assert_same(ctx[0], run)


def test_clade_union_over_colliding_members(oracle):
    """a code shared inside taxon 11 and the same code in its sibling 12: the clade of genus 10 counts it once"""
    pairs, single = _species_a(6, 30)
    a_pairs, cross = pairs[:4], pairs[4:]
    kdb, idx = _db({11: np.concatenate([np.array(a_pairs).ravel(), [c[0] for c in cross], single[:10]]),
                    12: np.concatenate([[c[1] for c in cross], single[10:20]]), 21: single[20:]})
    batch = [x for p in pairs for x in p] + list(single)
    clf, run = _compare(oracle, kdb, idx, [batch], clades=[[11], [11, 12], [11, 12, 21]])
    r, k, u = clf.clade_counts_tree([10, 1])
    for i, mem in enumerate([[10, 11, 12], [1, 10, 11, 12, 20, 21]]):
        assert (int(u[i]), int(r[i]), int(k[i])) == run.clade(mem), mem
