"""The multi-GPU merges and shard protocols with N classification contexts on ONE device.

Each rank is a thread that drives its own `binding.Classifier` on device 0 and calls the unchanged functions of
krakenuniq_b200.dist (`merge_classifier_state`, `merge_classifier_state_partitioned`, `clade_counts_distributed`)
through tests.local_group, the in-process stand-in for torch.distributed.  Contexts on one device exercise the same
library calls as one process per GPU: peer copies and peer stores work within a device, and device flags between
contexts are ordinary device memory.

Every merged state is compared exactly with one context that classified all reads, which is itself compared with
the oracle; the sparse-tier key sets are compared with a host computation from the oracle's per-window taxa."""
import functools

import numpy as np
import pytest
import torch

from krakenuniq_b200 import binding, synth
from krakenuniq_b200 import dist as kdist
from tests import util
from tests.local_group import run_ranks
from tests.test_record_tier_gpu import PAIRS, SINGLES, TAX as RT_TAX, _db as rt_db, _read as rt_read

pytestmark = pytest.mark.gpu
K = 31
DEV = "cuda:0"
KEYS = ("taxid", "n_reads", "n_kmers", "sparse", "unique")
FLAG_TIMEOUT_MS = 5000
M64 = (1 << 64) - 1


def _classifier(unit=500000, mode=binding.HLL_PRELOAD):
    # small contexts; a small sparse set so that it has to grow
    return binding.Classifier(device=0, max_reads=1 << 14, max_bases=4 << 20, work_unit_size=unit, hll_mode=mode,
                              sparse_set_slots=1 << 12)


def _mix64(x):
    """the table hash of the device sets (kuq_kernels.cu mix64); the partitioned merge sends a key to part
    (mix64(code) >> 33) % n_parts"""
    x = int(x)
    x ^= x >> 31
    x = (x * 0x7fb5d329728ea185) & M64
    x ^= x >> 27
    x = (x * 0x81dadef4bc2dd44d) & M64
    x ^= x >> 33
    return x


def _part(key, n):
    return (_mix64(int(key) & 0xFFFFFFFF) >> 33) % n


def _export(clf):
    """the sparse-tier keys a context holds (kuq_sparse_export), sorted"""
    n = clf.sparse_export()
    t = torch.zeros(max(n, 1), dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    m = clf.sparse_export(t.data_ptr(), t.numel())
    return np.sort(t[:m].cpu().numpy())


def _keys_of(oracle, dense_ids, sparse_taxa, taxa, kmers):
    """sparse-tier keys (dense id + 1) << 32 | encodeHashIn32Bit(fmix64(canonical k-mer)) of the (taxon, k-mer)
    pairs whose taxon ends sparse"""
    row = {int(t): i for i, t in enumerate(dense_ids)}
    pairs = np.unique(np.stack([np.asarray(taxa, np.uint64), np.asarray(kmers, np.uint64)], 1), axis=0)
    code = {}
    keys = set()
    for t, km in pairs.tolist():
        if t not in sparse_taxa:
            continue
        if km not in code:
            code[km] = oracle.encode_hash32(oracle.fmix64(oracle.canonical(km, K)))
        keys.add(((row[t] + 1) << 32) | code[km])
    return np.array(sorted(keys), np.int64)


def _check_state(clf, ref, label):
    got = clf.counts()
    for key in KEYS:
        assert np.array_equal(got[key], ref["want"][key]), (label, key, got[key], ref["want"][key])
    for t, regs in ref["regs"].items():
        assert np.array_equal(clf.registers(t), regs), (label, "registers", t)


def _check_partitioned_keys(exports, expected):
    """after a partitioned merge: context j holds exactly the keys of part j, and the parts cover the expected set"""
    n = len(exports)
    for j, e in enumerate(exports):
        assert all(_part(k, n) == j for k in e.tolist()), ("a key outside its part", j)
    allk = np.concatenate(exports) if exports else np.zeros(0, np.int64)
    assert len(np.unique(allk)) == len(allk), "a key lives in two parts"
    assert np.array_equal(np.sort(allk), expected)


# ---- workloads and their single-context / oracle reference ------------------------------------------------------
def _mixed():
    """4 abundant species (dense), 23 rare ones (sparse), and one species whose reads crowd the first work unit (dense
    there) and are sprinkled over the rest (sparse on every context that does not hold the first unit)"""
    rng = np.random.default_rng(17)
    tax = synth.make_taxonomy(28)
    genomes = synth.random_genomes(rng, 28, 2000, 0.2)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, K)
    kdb, idx = synth.build_db_images(km, tx, K, 9, 2)
    ab = synth.sample_reads(rng, genomes[:4], 2400, 150, 0.01, 0.1, 0.2)[0].reshape(-1, 150)
    md = synth.sample_reads(rng, genomes[4:5], 160, 150, 0.01, 0.1, 0.0)[0].reshape(-1, 150)
    ra = synth.sample_reads(rng, genomes[5:], 280, 150, 0.01, 0.1, 0.0)[0].reshape(-1, 150)
    other = np.concatenate([ab, ra])[rng.permutation(len(ab) + len(ra))]
    head = np.concatenate([other[:70], md[:130]])[rng.permutation(200)]        # = work unit 0 (200 reads of 150)
    tail = other[70:]
    at = np.sort(rng.integers(0, len(tail) + 1, len(md) - 130))
    reads = np.concatenate([head, np.insert(tail, at, md[130:], axis=0)])
    offs = np.arange(len(reads) + 1, dtype=np.uint64) * np.uint64(150)
    return dict(tax=tax, kdb=kdb, idx=idx, bases=reads.reshape(-1).copy(), offs=offs, unit=30000,
                medium=synth.species_ids(tax)[4])


def _collisions():
    """~10^5 codes per taxon: sibling taxa hold equal codes, so clade unions are smaller than the sums of their
    members (the "collisions" case of test_gpu_parity); every taxon stays sparse"""
    rng = np.random.default_rng(91)
    tax = synth.make_taxonomy(4, 2, 1)
    genomes = synth.random_genomes(rng, 4, 150000, shared_frac=0.02)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, K)
    kdb, idx = synth.build_db_images(km, tx, K, 8, 2)
    bases, offs = synth.sample_reads(rng, genomes, 5000, 150, 0.001, 0.1, 0.02)
    return dict(tax=tax, kdb=kdb, idx=idx, bases=bases, offs=offs, unit=1200, medium=None)


@functools.lru_cache(maxsize=None)
def _reference(name):
    from oracle.oracle_py import Oracle
    oracle = Oracle()
    w = {"mixed": _mixed, "collisions": _collisions}[name]()
    bases, offs, unit, tax = w["bases"], w["offs"], w["unit"], w["tax"]
    units, _, _ = synth.work_unit_ids(offs, unit)
    single = _classifier(unit)
    single.stage_db(w["kdb"], w["idx"])
    single.set_taxonomy(*tax.parent_map())
    res = single.classify(bases, offs, unit_id=units)
    single.finish()
    want = single.counts()
    # the oracle cuts the same work units itself
    run = oracle.run(oracle.open_db(w["kdb"], w["idx"]), oracle.parent_map(*tax.parent_map()), unit, 0)
    calls, codes, code_off = run.classify(bases, offs)
    run.finish()
    oc = run.counts()
    assert np.array_equal(calls, res["call"])
    for key in KEYS:
        assert np.array_equal(oc[key], want[key]), ("single context vs oracle", key)
    members = util.clade_members(tax.rows, want["taxid"])
    clades = [members[t] for t in sorted(members)]
    want_clades = [single.clade(c) for c in clades]
    for c, g in zip(clades, want_clades):
        assert g == run.clade(c), ("single context clade vs oracle", c)
    # the (taxon, k-mer) of every unambiguous window, from the oracle's scan and per-window taxa
    taxa, kmers = [], []
    for i in range(len(offs) - 1):
        km, amb = oracle.scan(bases[int(offs[i]):int(offs[i + 1])].tobytes(), K)
        wt = codes[int(code_off[i]):int(code_off[i + 1])]
        assert len(wt) == len(km)
        taxa.append(wt[amb == 0])
        kmers.append(km[amb == 0])
    dense_ids = single.dense_taxids()
    sparse_taxa = {int(t) for t, s in zip(want["taxid"], want["sparse"]) if s}
    expected = _keys_of(oracle, dense_ids, sparse_taxa, np.concatenate(taxa), np.concatenate(kmers))
    db_taxids, _ = single.db_taxids()
    ref = dict(w, units=units, want=want, calls=res["call"], clades=clades, want_clades=want_clades, expected=expected,
               regs={int(t): single.registers(t) for t in want["taxid"]}, db_taxids=db_taxids)
    single.close()
    if name == "mixed":
        assert 5 < int(want["sparse"].sum()) < len(want["taxid"]) - 2, "the case must mix sparse and dense taxa"
        assert not dict(zip(want["taxid"].tolist(), want["sparse"].tolist()))[w["medium"]]
    else:
        assert want["sparse"].all()
    return ref


def _unit_cut(units, a):
    n = len(units)
    while 0 < a < n and units[a] == units[a - 1]:
        a += 1
    return a


def _shares(units, lo, hi, world, idle):
    """contiguous shares of reads [lo, hi) cut at work-unit boundaries; rank `idle` receives none"""
    active = [r for r in range(world) if r != idle]
    out = [None] * world
    for j, r in enumerate(active):
        a, b = kdist.partition(hi - lo, len(active), j)
        out[r] = (_unit_cut(units, lo + a), _unit_cut(units, lo + b))
    if idle is not None:
        at = out[idle - 1][1] if idle > 0 else lo
        out[idle] = (at, at)
    return out


def _range_cuts(idx, world):
    """minimizer ranges cut by record count (prepare_chunking), the first range small"""
    idx_off = np.frombuffer(idx[8:].tobytes(), np.uint64)
    n_bins = len(idx_off) - 1
    wts = np.array([1] + [4] * (world - 1), np.float64)
    frac = np.concatenate([[0], np.cumsum(wts) / wts.sum()])
    cuts = [int(np.searchsorted(idx_off, np.uint64(int(idx_off[-1] * f)), side="left")) for f in frac]
    cuts[0], cuts[-1] = 0, n_bins
    assert all(a < b for a, b in zip(cuts, cuts[1:])), cuts
    return cuts


CASES = [(1, "mixed", None), (2, "mixed", None), (3, "mixed", 1), (8, "mixed", None),
         (2, "collisions", 1), (3, "collisions", None), (8, "collisions", 5)]


def _is_dense_here(clf, taxid):
    sp = clf.state_ptrs()
    flag = kdist.device_view(sp.d_dense_flag, sp.n_sketch, torch.uint8, DEV).cpu().numpy()
    return bool(flag[list(clf.dense_taxids()).index(taxid)])


def _merge_and_check(ctxs, ref, merge, label, buffers_of=None):
    """merge the contexts' states with `merge` (one thread per context) and check every context against the
    reference; returns the contexts' sparse-tier keys after the merge"""
    world = len(ctxs)

    def rank(r, coll):
        clf = ctxs[r]
        if merge == "gather":
            kdist.merge_classifier_state(clf, DEV, coll)
        else:
            kdist.merge_classifier_state_partitioned(clf, DEV, coll, buffers=buffers_of(r) if buffers_of else None)
        _check_state(clf, ref, (label, merge, r))
        if merge == "gather":
            for c, want in zip(ref["clades"], ref["want_clades"]):
                assert clf.clade(c) == want, (label, r, c)
        else:
            got = kdist.clade_counts_distributed(clf, ref["clades"], DEV, coll)
            for c, g, want in zip(ref["clades"], got, ref["want_clades"]):
                assert g == want, (label, r, c, g, want)
        return _export(clf)

    exports = run_ranks(world, rank)
    if merge == "gather":
        for e in exports:
            assert np.array_equal(e, ref["expected"])
    else:
        _check_partitioned_keys(exports, ref["expected"])
    return exports


# ---- the key computation itself, on one context ------------------------------------------------------------------
@pytest.mark.parametrize("workload", ["mixed", "collisions"])
def test_single_context_export_equals_the_oracle_keys(workload):
    """anchor: one context's sparse_export equals the host key set while records are flagged, kept, and both"""
    ref = _reference(workload)
    n = len(ref["offs"]) - 1
    h = _unit_cut(ref["units"], n // 2)
    for state in ("flagged", "kept", "both"):
        clf = _classifier(ref["unit"])
        clf.stage_db(ref["kdb"], ref["idx"])
        clf.set_taxonomy(*ref["tax"].parent_map())
        if state == "both":
            clf.classify(ref["bases"], np.ascontiguousarray(ref["offs"][:h + 1]), unit_id=ref["units"][:h])
            clf.counts()                                  # a harvest: these records become kept
            clf.classify(ref["bases"], np.ascontiguousarray(ref["offs"][h:]), unit_id=ref["units"][h:])
        else:
            clf.classify(ref["bases"], ref["offs"], unit_id=ref["units"])
            if state == "kept":
                clf.finish()
        assert np.array_equal(_export(clf), ref["expected"]), state
        _check_state(clf, ref, state)


# ---- replicas: every context stages the whole database and classifies a contiguous share of the reads ------------
@pytest.mark.parametrize("merge", ["gather", "partitioned", "partitioned_buffers"])
@pytest.mark.parametrize("world,workload,idle", CASES)
def test_replicas_merge_to_the_single_context_state(world, workload, idle, merge):
    ref = _reference(workload)
    n = len(ref["offs"]) - 1
    shares = _shares(ref["units"], 0, n, world, idle)
    ctxs = []
    for lo, hi in shares:
        c = _classifier(ref["unit"])
        c.stage_db(ref["kdb"], ref["idx"])
        c.set_taxonomy(*ref["tax"].parent_map())
        if hi > lo:
            res = c.classify(ref["bases"], np.ascontiguousarray(ref["offs"][lo:hi + 1]), unit_id=ref["units"][lo:hi])
            assert np.array_equal(res["call"], ref["calls"][lo:hi])
            c.finish()
        ctxs.append(c)
    if workload == "mixed" and world > 1:
        # the medium species is dense on the context of the first work unit and sparse on the others
        med = ref["medium"]
        assert _is_dense_here(ctxs[0], med)
        assert any(not _is_dense_here(c, med) for c, (lo, hi) in zip(ctxs[1:], shares[1:]) if hi > lo)
    buffers_of = None
    if merge == "partitioned_buffers":
        def buffers_of(r):
            # rank 0 (mod 3): export buffer too small (the export fails, consumes nothing, the library allocates);
            # rank 1: receive buffer too small; rank 2: both large enough
            need = int(ctxs[r].sparse_export_partitioned(world).sum())
            big = torch.zeros(need + 1024, dtype=torch.int64, device=DEV)
            small = torch.zeros(1, dtype=torch.int64, device=DEV)
            return [(small, big), (big, small), (big, torch.zeros(1 << 20, dtype=torch.int64, device=DEV))][r % 3]
    _merge_and_check(ctxs, ref, "gather" if merge == "gather" else "partitioned", ("replicas", world, workload),
                     buffers_of)
    for c in ctxs:
        c.close()


# ---- shards: context j stages minimizer range j --------------------------------------------------------------------
def _shard_contexts(ref, cuts, counting):
    ctxs = []
    for j in range(len(cuts) - 1):
        c = _classifier(ref["unit"])
        c.set_db_taxid_universe(ref["db_taxids"])
        c.stage_db(ref["kdb"], ref["idx"], cuts[j], cuts[j + 1])
        c.set_taxonomy(*ref["tax"].parent_map())
        if counting:
            c.set_shard_counting(True)
        c.state_ptrs()                                    # numbers the taxa now, not in the middle of a flag protocol
        ctxs.append(c)
    return ctxs


def _device_reads(ref):
    bases, offs = ref["bases"], ref["offs"]
    d_bases = torch.from_numpy(np.concatenate([bases, np.full(64, ord("N"), np.uint8)])).to(DEV)
    d_offs = torch.from_numpy(np.concatenate([offs, offs[-1:]]).astype(np.int64)).to(DEV)
    d_units = torch.from_numpy(ref["units"].astype(np.int32)).to(DEV)
    return d_bases, d_offs, d_units


@pytest.mark.parametrize("variant", ["reduce_ids", "peers", "flags"])
@pytest.mark.parametrize("world,workload,idle", CASES)
def test_shards_merge_to_the_single_context_state(world, workload, idle, variant):
    ref = _reference(workload)
    offs = ref["offs"]
    n, total = len(offs) - 1, int(offs[-1])
    cuts = _range_cuts(ref["idx"], world)
    ctxs = _shard_contexts(ref, cuts, counting=variant != "reduce_ids")
    d_bases, d_offs, d_units = _device_reads(ref)
    keep = []                                             # device slices the library reads asynchronously

    def sub(t, a, b):
        s = t[a:b].contiguous()
        keep.append(s)
        return s.data_ptr()

    if variant in ("reduce_ids", "peers"):
        shares = _shares(ref["units"], 0, n, world, idle)
        if variant == "reduce_ids":
            # (a) every range looks the whole batch up into ONE buffer (a key hits in at most one range) ...
            ids = [torch.zeros(total + 64, dtype=torch.int32, device=DEV)] * world
            torch.cuda.synchronize()
            for c in ctxs:
                c.lookup_device(0, d_bases.data_ptr(), d_offs.data_ptr(), n, total, ids[0].data_ptr(), only_hits=1)
        else:
            # (b) ... or scatters its hits into the buffer of the context that owns the read; the finder counts
            ids = [torch.zeros(total + 64, dtype=torch.int32, device=DEV) for _ in range(world)]
            bounds = np.array([int(offs[a]) for a, _ in shares] + [total], np.uint64)
            bounds[0] = 0
            torch.cuda.synchronize()
            for c in ctxs:
                c.lookup_device_peers(0, d_bases.data_ptr(), d_offs.data_ptr(), n, total, [t.data_ptr() for t in ids],
                                      bounds)
        for c in ctxs:
            c.sync(0)
        # ... then every owner resolves its share
        ptrs = [(sub(d_offs, a, b + 2), sub(d_units, a, b)) for a, b in shares]
        torch.cuda.synchronize()
        for j, (c, (a, b)) in enumerate(zip(ctxs, shares)):
            assert ptrs[j][0] % 16 == 0
            if b > a:
                c.resolve_device(0, d_bases.data_ptr(), ptrs[j][0], b - a, total, ids[j].data_ptr(), ptrs[j][1])
        for c in ctxs:
            c.sync(0)
            c.finish()
        merge = "gather" if variant == "reduce_ids" else "partitioned"
    else:
        _flag_steps(ctxs, ref, d_bases, d_offs, d_units, idle, sub)
        merge = "partitioned"                             # no finish(): the merge meets flagged records
    _merge_and_check(ctxs, ref, merge, ("shards", variant, world, workload))
    for c in ctxs:
        c.close()


def _flag_steps(ctxs, ref, d_bases, d_offs, d_units, idle, sub, n_steps=3):
    """(c) bench.py's and shard_loop's protocol: device flags instead of host barriers, double-buffered id buffers,
    several steps.  Every context's phase is queued before the host waits for any of them, in shard_loop's order."""
    world = len(ctxs)
    offs, units = ref["offs"], ref["units"]
    n, total = len(offs) - 1, int(offs[-1])
    nbytes = (total + 64) * 4
    steps = [(_unit_cut(units, a), _unit_cut(units, b)) for a, b in (kdist.partition(n, n_steps, i) for i in range(n_steps))]
    bufs = [[c.device_alloc(nbytes) for _ in range(2)] for c in ctxs]
    flg = [c.device_alloc(256) for c in ctxs]        # [0:64) "hits delivered" counters, [128:192) "buffer clean"
    for c, f, bb in zip(ctxs, flg, bufs):
        ft = kdist.device_view(f, 256, torch.int64, DEV)
        ft.zero_()
        ft[16:24] = 2                                # both id buffers are clean for steps 0 and 1
        for b_ in bb:
            c.device_memset(0, b_, 0, nbytes)
        c.sync(0)
    # every device slice of the loop exists before the first flag wait: a host synchronisation inside the loop would
    # wait for contexts whose peers have not been queued yet
    plan = []
    for sa, sb in steps:
        owners = _shares(units, sa, sb, world, idle)
        bnd = np.array([int(offs[a]) for a, _ in owners] + [int(offs[sb])], np.uint64)
        bnd[0] = int(offs[sa])
        plan.append((sa, sb, owners, bnd, sub(d_offs, sa, sb + 2),
                     [(sub(d_offs, a, b + 2), sub(d_units, a, b)) for a, b in owners]))
    torch.cuda.synchronize()
    try:
        for i, (sa, sb, owners, bnd, step_offs, own) in enumerate(plan):
            par = i & 1
            for j, c in enumerate(ctxs):
                c.wait_flags(0, flg[j] + 128, world, i + 1, timeout_ms=FLAG_TIMEOUT_MS)
                if sb > sa:
                    c.lookup_device_peers(0, d_bases.data_ptr(), step_offs, sb - sa, total, [b[par] for b in bufs], bnd)
                c.signal_peers(0, flg, j, i + 1)
            for j, c in enumerate(ctxs):
                c.wait_flags(0, flg[j], world, i + 1, timeout_ms=FLAG_TIMEOUT_MS)
                a, b = owners[j]
                if b > a:
                    assert own[j][0] % 16 == 0
                    c.resolve_device(0, d_bases.data_ptr(), own[j][0], b - a, total, bufs[j][par], own[j][1])
                c.device_memset(0, bufs[j][par], 0, nbytes)
                c.signal_peers(0, [f + 128 for f in flg], j, i + 3)
            for c in ctxs:
                c.sync(0)                            # a flag wait that timed out fails here with KUQ_E_STATE
    finally:
        for c in ctxs:
            try:
                c.sync(0)
            except binding.KuqError:
                pass
        for c, bb, f in zip(ctxs, bufs, flg):
            for b_ in bb:
                c.device_free(b_)
            c.device_free(f)


# ---- record-tier states at merge time ------------------------------------------------------------------------------
def _record_tier_case(oracle, shards):
    """a database with colliding pairs (two k-mers of taxon 11 with one code).  Context 0 sees the first member of
    half of the pairs and the second member of the other half, context 1 the opposite, so the primary of a pair is
    hit on one context and its secondary on the other; some singles are hit on both."""
    pairs, single, cut = PAIRS[:8], SINGLES[:60], None
    if shards:
        # pairs whose two records lie in different minimizer ranges, and pairs whose records share a range
        cand = np.array(PAIRS[:400], np.uint64)
        bins = synth.bin_key(cand.ravel(), K, 8, 2).reshape(-1, 2)
        cut = int(np.median(bins))                        # minimizer bins are far from uniform: cut at the median
        lower = bins < cut
        split = [tuple(p) for p, lw in zip(cand, lower) if lw[0] != lw[1]][:5]
        same = [tuple(p) for p, lw in zip(cand, lower) if lw[0] == lw[1]][:3]
        assert len(split) == 5 and len(same) == 3
        pairs = split + same
    flat = np.array(pairs, np.uint64).ravel()
    by_taxon = {11: np.concatenate([flat, single[:30]]), 12: single[30:50], 21: single[50:60]}
    kdb, idx = rt_db(by_taxon)
    a = [p[0] for p in pairs[:4]] + [p[1] for p in pairs[4:]]
    b = [p[1] for p in pairs[:4]] + [p[0] for p in pairs[4:]]
    batches = [[a + list(single[:20]), list(single[20:40])],      # context 0: a harvest between its two batches
               [b + list(single[30:60])]]                          # context 1: one batch, records only flagged
    mode = binding.HLL_CHUNKED if shards else binding.HLL_PRELOAD
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*RT_TAX.parent_map()), 500000,
                     1 if shards else 0)
    everything = [x for ctx in batches for bt in ctx for x in bt]
    run.classify(*synth.pack_reads([rt_read(x) for x in everything]), want_codes=False)
    run.finish()
    taxon_of = {int(k): t for t, ks in by_taxon.items() for k in np.asarray(ks, np.uint64).tolist()}
    return dict(kdb=kdb, idx=idx, batches=batches, mode=mode, run=run, reads=everything, taxon_of=taxon_of, cut=cut)


def _rt_context(kdb, idx, mode, bins=(0, 0), universe=None):
    c = binding.Classifier(max_reads=1 << 12, max_bases=1 << 20, hll_mode=mode, sparse_set_slots=1 << 12)
    if universe is not None:
        c.set_db_taxid_universe(universe)
    c.stage_db(kdb, idx, *bins)
    c.set_taxonomy(*RT_TAX.parent_map())
    return c


def _rt_check(oracle, ctxs, run, case, merge, label):
    want = run.counts()
    clades = [[11], [11, 12], [11, 12, 21], [12, 21]]
    sparse_taxa = {int(t) for t, s in zip(want["taxid"], want["sparse"]) if s}
    # every read is one k-mer of the database: its window's taxon is the record's
    kms = np.array(case["reads"], np.uint64)
    taxa = np.array([case["taxon_of"][int(k)] for k in kms.tolist()], np.uint64)
    expected = _keys_of(oracle, ctxs[0].dense_taxids(), sparse_taxa, taxa, kms)

    def rank(r, coll):
        clf = ctxs[r]
        if merge == "gather":
            kdist.merge_classifier_state(clf, DEV, coll)
        else:
            kdist.merge_classifier_state_partitioned(clf, DEV, coll)
        got = clf.counts()
        for key in KEYS:
            assert np.array_equal(got[key], want[key]), (label, r, key, got[key], want[key])
        if merge == "gather":
            for c in clades:
                assert clf.clade(c) == run.clade(c), (label, r, c)
        else:
            for c, g in zip(clades, kdist.clade_counts_distributed(clf, clades, DEV, coll)):
                assert g == run.clade(c), (label, r, c, g, run.clade(c))
        return _export(clf)

    exports = run_ranks(len(ctxs), rank)
    if merge == "gather":
        for e in exports:
            assert np.array_equal(e, expected), label
    else:
        _check_partitioned_keys(exports, expected)


@pytest.mark.parametrize("merge", ["gather", "partitioned"])
def test_record_tier_replicas(oracle, merge):
    case = _record_tier_case(oracle, shards=False)
    kdb, idx, batches, mode, run = (case[k] for k in ("kdb", "idx", "batches", "mode", "run"))
    ctxs = []
    for j, bl in enumerate(batches):
        c = _rt_context(kdb, idx, mode)
        for i, bt in enumerate(bl):
            c.classify(*synth.pack_reads([rt_read(x) for x in bt]))
            if j == 0 and i == 0:
                c.counts()                               # records of the first batch become KEPT
        ctxs.append(c)
    _rt_check(oracle, ctxs, run, case, merge, ("record tier replicas", merge))


def test_record_tier_shards(oracle):
    """the two records of a colliding pair in different minimizer ranges: each range keeps its record, the
    partitioned merge meets both keys on the code's owner and counts the code once"""
    case = _record_tier_case(oracle, shards=True)
    kdb, idx, batches, mode, run = (case[k] for k in ("kdb", "idx", "batches", "mode", "run"))
    universe = np.array(sorted({11, 12, 21}), np.uint32)
    ctxs = [_rt_context(kdb, idx, mode, r, universe) for r in ((0, case["cut"]), (case["cut"], 1 << 16))]
    for c in ctxs:
        c.set_shard_counting(True)
    # context j owns (resolves) the reads of batches[j]; step i looks up the i-th batch of each context
    steps = [batches[0][0] + batches[1][0], batches[0][1]]
    owners = [(len(batches[0][0]), len(batches[1][0])), (len(batches[0][1]), 0)]
    for i, (reads, (n0, n1)) in enumerate(zip(steps, owners)):
        bases, offs = synth.pack_reads([rt_read(x) for x in reads])
        total, n = int(offs[-1]), len(reads)
        d_bases = torch.from_numpy(np.concatenate([bases, np.full(64, ord("N"), np.uint8)])).to(DEV)
        d_offs = torch.from_numpy(np.concatenate([offs, offs[-1:]]).astype(np.int64)).to(DEV)
        ids = [torch.zeros(total + 64, dtype=torch.int32, device=DEV) for _ in ctxs]
        bounds = np.array([0, int(offs[n0]), total], np.uint64)
        share = [(0, n0), (n0, n0 + n1)]
        so = [d_offs[a:b + 2].contiguous() for a, b in share]
        torch.cuda.synchronize()
        for c in ctxs:
            c.lookup_device_peers(0, d_bases.data_ptr(), d_offs.data_ptr(), n, total, [t.data_ptr() for t in ids], bounds)
        for c in ctxs:
            c.sync(0)
        for j, c in enumerate(ctxs):
            a, b = share[j]
            if b > a:
                c.resolve_device(0, d_bases.data_ptr(), so[j].data_ptr(), b - a, total, ids[j].data_ptr())
            c.sync(0)
        if i == 0:
            ctxs[0].counts()                             # context 0's records of step 0 become KEPT
    _rt_check(oracle, ctxs, run, case, "partitioned", ("record tier shards",))


# ---- contract of the partitioned merge --------------------------------------------------------------------------
def test_partitioned_merge_contract():
    ref = _reference("mixed")
    n, world = len(ref["offs"]) - 1, 2
    shares = _shares(ref["units"], 0, n, world, None)
    ctxs = []
    for lo, hi in shares:
        c = _classifier(ref["unit"])
        c.stage_db(ref["kdb"], ref["idx"])
        c.set_taxonomy(*ref["tax"].parent_map())
        ctxs.append(c)

    def classify_all():
        for c, (lo, hi) in zip(ctxs, shares):
            c.classify(ref["bases"], np.ascontiguousarray(ref["offs"][lo:hi + 1]), unit_id=ref["units"][lo:hi])
            c.finish()

    classify_all()
    for bad in (0, 9):
        with pytest.raises(binding.KuqError) as e:
            ctxs[0].sparse_export_partitioned(bad)
        assert e.value.code == -1
        with pytest.raises(binding.KuqError) as e:
            ctxs[0].sparse_export_partitioned_alloc(bad)
        assert e.value.code == -1
    first = _merge_and_check(ctxs, ref, "partitioned", "first merge")

    # a second partitioned merge right away moves no key and changes no sketch; only the counters add up once more
    # (the merge sums them: it is meant to run once per run)
    def second(r, coll):
        kdist.merge_classifier_state_partitioned(ctxs[r], DEV, coll)
        got, want = ctxs[r].counts(), ref["want"]
        for key in ("taxid", "sparse", "unique"):
            assert np.array_equal(got[key], want[key]), ("second merge", r, key)
        for key in ("n_reads", "n_kmers"):
            assert np.array_equal(got[key], want[key] * world), ("second merge", r, key)
        for t, regs in ref["regs"].items():
            assert np.array_equal(ctxs[r].registers(t), regs), ("second merge", r, t)
        got_cl = kdist.clade_counts_distributed(ctxs[r], ref["clades"], DEV, coll)
        assert [g[0] for g in got_cl] == [w[0] for w in ref["want_clades"]]
        return _export(ctxs[r])

    for a, b in zip(first, run_ranks(world, second)):
        assert np.array_equal(a, b)
    # reset_counts clears the merged state and the kept records: the same run gives the same state again
    for c in ctxs:
        c.reset_counts()
    classify_all()
    _merge_and_check(ctxs, ref, "partitioned", "after reset")
    for c in ctxs:
        c.close()
