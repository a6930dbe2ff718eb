"""Keep mode: under the preload rule the fused lookup makes a record kept (KEPT_BIT) at its first sighting and the
resolve counts its code, so the end-of-run harvest only settles the collision groups (a kept secondary hands its flag
to its primary).  Every run here goes through both paths of one build — keep mode, and the flag-and-harvest path that
KUQ_KEEP_AT_HARVEST=1 forces — and the oracle: per-taxon counts, registers, the record flags and the kept-key count
must agree.  The databases hold crafted collision groups: 2-4 records of one taxon whose k-mers share their sparse
code (hashes chosen with the inverted fmix64 of tests/crafted.py)."""
import contextlib
import os

import numpy as np
import pytest
import torch

from krakenuniq_b200 import binding, synth
from tests import crafted

pytestmark = pytest.mark.gpu
K, NT = 31, 8
SEEN, KEPT = 0x80000000, 0x40000000
TAX = synth.Taxonomy([(1, 1, "root", "no rank"), (10, 1, "g", "genus"), (11, 10, "a", "species"),
                      (12, 10, "b", "species"), (20, 1, "h", "genus"), (21, 20, "c", "species")])
HDR = len(binding.kdb_header(K, 0))


@contextlib.contextmanager
def _path(old):
    prev = os.environ.pop("KUQ_KEEP_AT_HARVEST", None)
    if old:
        os.environ["KUQ_KEEP_AT_HARVEST"] = "1"
    try:
        yield
    finally:
        os.environ.pop("KUQ_KEEP_AT_HARVEST", None)
        if prev is not None:
            os.environ["KUQ_KEEP_AT_HARVEST"] = prev


def _groups(rng, sizes):
    """k-mer groups, one shared sparse code per group (codes whose low 13 index bits are zero carry a rank: avoided)"""
    out = []
    for n in sizes:
        top = int(rng.integers(1, 1 << 25))
        top |= 1 if not top & 0x1FFF else 0
        out.append([int(x) for x in crafted.kmers_with_hash(0xFFFFFF8000000000, top << 39, K, n, rng)])
    return out


def _singles(rng, n, taken):
    km = np.unique(synth.canonical(rng.integers(0, 1 << 62, 4 * n, dtype=np.uint64), K))
    km = km[~np.isin(km, np.asarray(sorted(taken), np.uint64))]
    return [int(x) for x in rng.permutation(km)[:n]]


def _db(by_taxon):
    km = np.concatenate([np.asarray(v, np.uint64) for v in by_taxon.values()])
    tx = np.concatenate([np.full(len(v), t, np.uint32) for t, v in by_taxon.items()])
    assert len(np.unique(km)) == len(km)
    return synth.build_db_images(km, tx, K, NT, 2)


class Arm:
    """one context on its own device copy of the records (so that its flags can be read back); old = forced
    flag-and-harvest path"""

    def __init__(self, kdb, idx, old, n_slots=3):
        self.old = old
        n = (kdb.size - HDR) // 12
        self.rec = torch.from_numpy(kdb[HDR:HDR + 12 * n].copy()).cuda()
        self.off = torch.from_numpy(idx[8:].copy().view(np.int64)).cuda()
        self.clf = binding.Classifier(n_slots=n_slots, max_reads=1 << 12, max_bases=1 << 20,
                                      hll_mode=binding.HLL_PRELOAD, sparse_set_slots=1 << 12)
        self.clf.attach_db_device(self.rec.data_ptr(), n, self.off.data_ptr(), K, NT, 2)
        self.clf.set_taxonomy(*TAX.parent_map())

    def call(self, fn, *a, **kw):
        with _path(self.old):
            return getattr(self.clf, fn)(*a, **kw)

    def words(self):
        torch.cuda.synchronize()
        return self.rec.cpu().numpy().view(np.uint32).reshape(-1, 3)


def _reads(kmers):
    return synth.pack_reads([crafted.kmer_read(x, K, rc=bool(i % 3 == 1)) for i, x in enumerate(kmers)])


def _run(arm, batches, readout_between=False, n_slots=3):
    """batches in flight on n_slots slots at once (host path: the library cuts the work units like the oracle)"""
    held, busy = [], set()
    for i, b in enumerate(batches):
        slot = i % n_slots
        if slot in busy:
            arm.clf.wait(slot)
        bases, offs = _reads(b)
        held.append((bases, offs))                           # host buffers of batches in flight stay alive
        arm.call("submit", slot, bases.ctypes.data, offs)
        busy.add(slot)
        if readout_between:
            arm.clf.counts()                                 # a harvest while other slots may still hold batches
    for s in sorted(busy):
        arm.clf.wait(s)
    arm.call("finish")


def _oracle_counts(oracle, kdb, idx, batches):
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*TAX.parent_map()), 500000, 0)
    for b in batches:
        bases, offs = _reads(b)
        run.classify(bases, offs, want_codes=False)
    run.finish()
    return run.counts()


def _assert_paths_agree(new, old, want):
    a, b = new.clf.counts(), old.clf.counts()
    for key in ("taxid", "n_reads", "n_kmers", "sparse", "unique"):
        assert np.array_equal(a[key], want[key]), (key, a[key], want[key])
        assert np.array_equal(b[key], want[key]), (key, b[key], want[key])
    for t in a["taxid"].tolist():
        assert np.array_equal(new.clf.registers(t), old.clf.registers(t)), t
    wn, wo = new.words(), old.words()
    assert not (wn[:, 1] & SEEN).any() and not (wo[:, 1] & SEEN).any()
    sparse_taxa = set(a["taxid"][a["sparse"] != 0].tolist())
    sparse_ids = [d for d, t in enumerate(np.asarray(new.clf.dense_taxids()).tolist()) if t in sparse_taxa]
    sel = np.isin(wn[:, 2], np.asarray(sparse_ids, np.uint32))
    assert sel.any()
    assert np.array_equal(wn[sel, 1] & KEPT, wo[sel, 1] & KEPT)
    if len(sparse_taxa) == len(a["taxid"]):                 # every taxon sparse: the kept keys are the same too
        assert new.clf.sparse_tier_info()["keys"] == old.clf.sparse_tier_info()["keys"]


def _pair(kdb, idx, batches, readout_between=False, n_slots=3):
    new, old = Arm(kdb, idx, False, n_slots), Arm(kdb, idx, True, n_slots)
    for arm in (new, old):
        _run(arm, batches, readout_between, n_slots)
    return new, old


@pytest.mark.parametrize("hits", ["secondary", "primary", "both", "both_split"])
def test_collision_groups(oracle, hits):
    """groups of 2-4 records of taxon 11 sharing a code; reads hit one member, the other, or all of them — in one
    batch or spread over batches with readouts between.  Which member is the primary is the library's choice: hitting
    the first or the last k-mer of each group reaches both roles across the groups."""
    rng = np.random.default_rng(31)
    groups = _groups(rng, [2, 3, 4, 2, 3, 4, 2])
    flat = [x for g in groups for x in g]
    single = _singles(rng, 60, flat)
    kdb, idx = _db({11: flat + single[:30], 12: single[30:50], 21: single[50:]})
    first, last = [g[0] for g in groups], [g[-1] for g in groups]
    if hits == "secondary":
        batches = [first + single[:20], first + single[20:]]
    elif hits == "primary":
        batches = [last + single, last]
    elif hits == "both":
        batches = [flat + single, flat, first]
    else:
        batches = [first + single[:25], single[25:], flat, last + single[:5], first]
    want = _oracle_counts(oracle, kdb, idx, batches)
    new, old = _pair(kdb, idx, batches, readout_between=hits == "both_split")
    _assert_paths_agree(new, old, want)


def test_duplicate_reads_in_flight_and_reset(oracle):
    """the same reads in three slots at once (one record sighted by many windows in one step and across slots),
    then reset_counts and a second run: exact again, no stale flags"""
    rng = np.random.default_rng(32)
    groups = _groups(rng, [3, 2, 4])
    flat = [x for g in groups for x in g]
    single = _singles(rng, 200, flat)
    kdb, idx = _db({11: flat + single[:100], 12: single[100:160], 21: single[160:]})
    batch = flat + single + flat + single[:50]
    batches = [batch] * 6
    want = _oracle_counts(oracle, kdb, idx, batches)
    new, old = _pair(kdb, idx, batches)
    _assert_paths_agree(new, old, want)
    for arm in (new, old):
        arm.clf.reset_counts()
        _run(arm, batches[:3])
    _assert_paths_agree(new, old, _oracle_counts(oracle, kdb, idx, batches[:3]))


def test_taxon_turns_dense_mid_run(oracle):
    """1100 distinct codes of taxon 12 in one work unit: its sketch converts during the first batch.  The records of
    sparse taxa carry the same flags on both paths (a record of a taxon that later converts may be kept at sighting)."""
    rng = np.random.default_rng(33)
    groups = _groups(rng, [2, 3])
    flat = [x for g in groups for x in g]
    single = _singles(rng, 1200, flat)
    kdb, idx = _db({11: flat + single[:40], 12: single[40:1150], 21: single[1150:]})
    batches = [single[40:1150] + flat, single[:40] + single[1150:], flat + single[:10]]
    want = _oracle_counts(oracle, kdb, idx, batches)
    assert not dict(zip(want["taxid"].tolist(), want["sparse"].tolist()))[12]
    new, old = _pair(kdb, idx, batches)
    _assert_paths_agree(new, old, want)


def test_transitions(oracle):
    """flags of the harvest path pending, then keep mode (which waits for the next harvest); a resolve-half call after
    keep-mode calls (the kept records move into the set); and kuq_merge_into of two keep-mode contexts"""
    rng = np.random.default_rng(34)
    groups = _groups(rng, [2, 3, 4])
    flat = [x for g in groups for x in g]
    single = _singles(rng, 80, flat)
    kdb, idx = _db({11: flat + single[:40], 12: single[40:60], 21: single[60:]})
    b1, b2, b3 = [g[0] for g in groups] + single[:30], flat + single[30:60], [g[-1] for g in groups] + single[60:]
    want = _oracle_counts(oracle, kdb, idx, [b1, b2, b3, b1])
    arm = Arm(kdb, idx, False)
    with _path(True):
        arm.clf.classify(*_reads(b1))                        # flags pending
    arm.clf.classify(*_reads(b2))                            # still the flag path: nothing may be kept beside flags
    arm.clf.counts()
    arm.clf.classify(*_reads(b3))                            # keep mode
    bases, offs = _reads(b1)
    codes, _ = arm.clf.lookup(bases, offs)
    arm.clf.resolve(bases, offs, codes)                      # resolve half: the set becomes the store
    arm.clf.finish()
    got = arm.clf.counts()
    for key in ("taxid", "n_reads", "n_kmers", "sparse", "unique"):
        assert np.array_equal(got[key], want[key]), key
    assert not (arm.words()[:, 1] & (SEEN | KEPT)).any()
    # merge: both sides classified in keep mode
    want = _oracle_counts(oracle, kdb, idx, [b2, b3])
    dst, src = Arm(kdb, idx, False), Arm(kdb, idx, False)
    dst.clf.classify(*_reads(b2))
    src.clf.classify(*_reads(b3))
    dst.clf.merge_from(src.clf)
    got = dst.clf.counts()
    for key in ("taxid", "n_reads", "n_kmers", "sparse", "unique"):
        assert np.array_equal(got[key], want[key]), key
