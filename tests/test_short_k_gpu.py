"""Databases with k <= 28: their records are key_len + 4 = 8..11 bytes in the file and are widened to the 12-byte layout
as they are staged (k_widen_records).  The C ABI against the oracle for every record size and HLL rule, the record tier,
ranged and streamed staging in several landing-zone pieces, the exported values, the refusals, and the drop-in
executables against the unmodified reference's recorded outputs (tests/ref_replay.py) for k = 21 databases.  The oracle
is held against the reference for these k by tests/test_oracle_short_k.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import binding, build, synth
from tests.test_gpu_parity import _check_against_oracle, _classifier, _runs_to_codes
from tests.test_record_tier_gpu import _fmix64

pytestmark = pytest.mark.gpu


def _workload(seed, k, nt, idx_type=2, n_sp=6, glen=2500, n_reads=700):
    rng = np.random.default_rng(seed)
    tax = synth.make_taxonomy(n_sp)
    genomes = synth.random_genomes(rng, n_sp, glen, shared_frac=0.25)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, k)
    kdb, idx = synth.build_db_images(km, tx, k, nt, idx_type)
    bases, offs = synth.sample_reads(rng, genomes, n_reads, 150, 0.01, 0.2, 0.2)
    g0 = synth.decode(genomes[0]).tobytes()
    extra = [b"", g0[:k - 1], g0[:k], g0[:k + 1], g0[7:7 + k] + b"N" + g0[300:300 + k], g0[50:50 + 2 * k].lower(),
             g0[900:1000].lower() + g0[1000:1100]]
    seqs = [bases[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)] + extra
    bases, offs = synth.pack_reads(seqs)
    return tax, genomes, kdb, idx, bases, offs


@pytest.fixture
def landing(monkeypatch):
    """a small landing zone, so that the small test databases arrive in many pieces"""
    def set_bytes(n):
        monkeypatch.setenv("KUQ_LANDING_BYTES", str(n))
    return set_bytes


# ---- C ABI parity, one case per record size --------------------------------------------------------------------
@pytest.mark.parametrize("k,nt,idx_type,mode,unit", [
    (15, 8, 2, binding.HLL_PRELOAD, 20000),        # 8-byte records
    (19, 10, 1, binding.HLL_CHUNKED, 500000),      # 9
    (21, 12, 2, binding.HLL_PRELOAD, 500000),      # 10, the reference's own smoke shape
    (25, 11, 2, binding.HLL_DENSE_ONLY, 3000),     # 11
    (28, 9, 2, binding.HLL_EXACT, 500000),         # 11
])
def test_short_k_matches_oracle(oracle, landing, k, nt, idx_type, mode, unit):
    tax, genomes, kdb, idx, bases, offs = _workload(2000 + k, k, nt, idx_type)
    landing(4096)
    if mode != binding.HLL_EXACT:
        _check_against_oracle(oracle, kdb, idx, tax, bases, offs, hll_mode=mode, unit=unit,
                              oracle_mode=1 if mode == binding.HLL_CHUNKED else 0)
        return
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*tax.parent_map()), unit, 0)
    run.set_exact()
    calls, codes, code_off = run.classify(bases, offs)
    run.finish()
    want = run.counts()
    clf = _classifier(hll_mode=mode, work_unit_size=unit)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*tax.parent_map())
    res = clf.classify(bases, offs, flags=binding.F_WANT_CODES)
    clf.finish()
    assert np.array_equal(res["call"], calls)
    for i in range(len(offs) - 1):
        assert np.array_equal(_runs_to_codes(res, i), codes[int(code_off[i]):int(code_off[i + 1])]), f"read {i}"
    got = clf.counts()
    for key in ("taxid", "n_reads", "n_kmers", "unique"):
        assert np.array_equal(got[key], want[key]), key


# ---- record tier (KEPT_BIT and the collision table) at k = 21 --------------------------------------------------
K = 21
TAX = synth.Taxonomy([(1, 1, "root", "no rank"), (10, 1, "g", "genus"), (11, 10, "a", "species"),
                      (12, 10, "b", "species"), (20, 1, "h", "genus"), (21, 20, "c", "species")])


def _kmer_pool(seed=21, n=400_000):
    """pairs of canonical 21-mers whose codes (fmix64 >> 39) are equal, and 21-mers with a code of their own"""
    rng = np.random.default_rng(seed)
    km = np.unique(synth.canonical(rng.integers(0, 1 << (2 * K), n, dtype=np.uint64), K))
    top = _fmix64(km) >> np.uint64(39)
    keep = (top & np.uint64(0x1FFF)) != 0
    km, top = km[keep], top[keep]
    order = np.argsort(top, kind="stable")
    km, top = km[order], top[order]
    _, first, count = np.unique(top, return_index=True, return_counts=True)
    return [(km[f], km[f + 1]) for f, c in zip(first, count) if c == 2], km[first[count == 1]]


def _read(kmer):
    codes = (int(kmer) >> (2 * (K - 1 - np.arange(K)))) & 3
    return synth.decode(codes.astype(np.uint8)).tobytes()


def _tier_db():
    pairs, singles = _kmer_pool()
    pairs = pairs[:8]
    by_taxon = {11: np.concatenate([np.array(pairs, np.uint64).ravel(), singles[:30]]), 12: singles[30:60], 21: singles[60:80]}
    km = np.concatenate(list(by_taxon.values()))
    tx = np.concatenate([np.full(len(v), t, np.uint32) for t, v in by_taxon.items()])
    kdb, idx = synth.build_db_images(km, tx, K, 8, 2)
    first, second = [p[0] for p in pairs], [p[1] for p in pairs]
    return kdb, idx, [first + list(singles[:40]), second + list(singles[40:80]), first[:3] + second[5:]]


def _oracle_run(oracle, kdb, idx, batches):
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*TAX.parent_map()), 500000, 0)
    for b in batches:
        run.classify(*synth.pack_reads([_read(x) for x in b]), want_codes=False)
    run.finish()
    return run


def _tier_clf(kdb, idx, batches, readout_between=True):
    clf = binding.Classifier(max_reads=1 << 12, max_bases=1 << 20, hll_mode=binding.HLL_PRELOAD, sparse_set_slots=1 << 12)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*TAX.parent_map())
    for b in batches:
        clf.classify(*synth.pack_reads([_read(x) for x in b]))
        if readout_between:
            clf.counts()                        # a readout = a harvest of the flagged records
    clf.finish()
    return clf


def _assert_same(clf, run):
    got, want = clf.counts(), run.counts()
    for key in ("taxid", "n_reads", "n_kmers", "sparse", "unique"):
        assert np.array_equal(got[key], want[key]), (key, got[key], want[key])
    for mem in ([11], [11, 12], [11, 12, 21]):
        assert clf.clade(mem) == run.clade(mem), mem


def test_record_tier_k21_harvest_reset_and_merge(oracle):
    kdb, idx, batches = _tier_db()
    run = _oracle_run(oracle, kdb, idx, batches)
    clf = _tier_clf(kdb, idx, batches)
    _assert_same(clf, run)
    # reset_counts, then the same run again
    clf.reset_counts()
    for b in batches:
        clf.classify(*synth.pack_reads([_read(x) for x in b]))
    clf.finish()
    _assert_same(clf, run)
    # two contexts, each with part of the batches, merged into one
    a = _tier_clf(kdb, idx, batches[:1], readout_between=False)
    b = _tier_clf(kdb, idx, batches[1:])
    a.merge_from(b)
    _assert_same(a, run)


# ---- ranged staging and streaming: the file offset of a range and the landing-zone pieces ------------------------
def _cuts(idx, n_ranges):
    nt = int(idx[7])
    idx_off = np.frombuffer(idx[8:].tobytes(), np.uint64)
    cuts = [int(np.searchsorted(idx_off, idx_off[-1] * r // n_ranges)) for r in range(n_ranges + 1)]
    cuts[0], cuts[-1] = 0, 1 << (2 * nt)
    return idx_off, cuts


def _chunked_oracle(oracle, tax, kdb, idx, bases, offs):
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*tax.parent_map()), 500000, 1)
    calls, codes, code_off = run.classify(bases, offs)
    run.finish()
    return calls, codes, code_off, run.counts()


@pytest.mark.parametrize("k,nt", [(21, 9), (25, 10)])
def test_ranged_stage_db(oracle, landing, k, nt):
    """kuq_stage_db of minimizer ranges [bin_lo, bin_hi) with bin_lo > 0: the range starts at rec_lo * (key_len + 4) in
    the file and arrives in many landing-zone pieces"""
    tax, genomes, kdb, idx, bases, offs = _workload(3000 + k, k, nt, n_reads=600)
    calls, codes, code_off, want = _chunked_oracle(oracle, tax, kdb, idx, bases, offs)
    landing(1000)                                      # ~90-100 records per piece
    idx_off, cuts = _cuts(idx, 3)
    clf = _classifier(hll_mode=binding.HLL_CHUNKED)
    clf.set_taxonomy(*tax.parent_map())
    _, _, taxa = synth.parse_kdb(kdb)
    clf.set_db_taxid_universe(np.unique(taxa))
    merged = np.zeros(int(offs[-1]), np.uint32)
    for r in range(3):
        assert cuts[r + 1] > cuts[r]
        clf.stage_db(kdb, idx, cuts[r], cuts[r + 1])
        assert sum(clf.db_taxids()[1]) == idx_off[cuts[r + 1]] - idx_off[cuts[r]]
        part, _ = clf.lookup(bases, offs)
        merged = np.where(part == binding.AMBIG, merged, np.maximum(merged, part))
    res = clf.resolve(bases, offs, merged, flags=binding.F_WANT_CODES)
    clf.finish()
    assert np.array_equal(res["call"], calls)
    for i in range(len(offs) - 1):
        assert np.array_equal(_runs_to_codes(res, i), codes[int(code_off[i]):int(code_off[i + 1])]), f"read {i}"
    got = clf.counts()
    for key in ("taxid", "n_reads", "n_kmers", "sparse", "unique"):
        assert np.array_equal(got[key], want[key]), key


@pytest.mark.parametrize("k,nt", [(21, 9), (25, 10)])
def test_streamed_ranges(oracle, landing, k, nt):
    """kuq_stream_open / kuq_stream_load: two ranges of file records (key_len + 4 bytes each) from pinned host memory,
    copied and widened in landing-zone pieces on the copy stream"""
    import torch
    from krakenuniq_b200 import dist as kdist
    tax, genomes, kdb, idx, bases, offs = _workload(4000 + k, k, nt, n_reads=600)
    calls, codes, code_off, want = _chunked_oracle(oracle, tax, kdb, idx, bases, offs)
    landing(1000)
    pair_sz = synth.key_len(k) + 4
    _, keys, taxa = synth.parse_kdb(kdb)
    header = kdb.size - pair_sz * len(keys)
    idx_off, cuts = _cuts(idx, 2)
    clf = _classifier(hll_mode=binding.HLL_CHUNKED, n_slots=2)
    clf.set_taxonomy(*tax.parent_map())
    clf.set_db_taxid_universe(np.unique(taxa))
    max_rec = max(int(idx_off[cuts[r + 1]] - idx_off[cuts[r]]) for r in range(2))
    clf.stream_open(k, nt, 2, max_rec, max(cuts[1] - cuts[0], cuts[2] - cuts[1]))
    L = clf.L
    rec_bytes = kdb[header:]
    h_rec = L.kuq_host_alloc(rec_bytes.size + 16)
    ctypes.memmove(h_rec, rec_bytes.ctypes.data, rec_bytes.size)
    h_off = L.kuq_host_alloc(idx_off.size * 8)
    ctypes.memmove(h_off, idx_off.ctypes.data, idx_off.size * 8)
    dev = "cuda:0"
    total = int(offs[-1])
    n = len(offs) - 1
    d_bases = torch.from_numpy(np.concatenate([bases, np.full(64, ord("N"), np.uint8)])).to(dev)
    d_offs = torch.from_numpy(np.concatenate([offs, offs[-1:]]).astype(np.int64)).to(dev)
    merged = torch.zeros(total + 64, dtype=torch.int32, device=dev)
    for r in range(2):
        a, b = int(idx_off[cuts[r]]), int(idx_off[cuts[r + 1]])
        clf.stream_load(r, h_rec + pair_sz * a, b - a, h_off + 8 * cuts[r], cuts[r], cuts[r + 1])
    for r in range(2):
        clf.stream_use(r)
        clf.lookup_device(0, d_bases.data_ptr(), d_offs.data_ptr(), n, total, merged.data_ptr(), only_hits=1)
    clf.sync(0)
    clf.stream_check()
    clf.resolve_device(0, d_bases.data_ptr(), d_offs.data_ptr(), n, total, merged.data_ptr(), None)
    clf.sync(0)
    call = kdist.device_view(clf.device_result(0).d_call, n * 4, torch.int32, dev).cpu().numpy().view(np.uint32)
    clf.finish()
    assert np.array_equal(call, calls)
    got = clf.counts()
    for key in ("taxid", "n_reads", "n_kmers", "sparse", "unique"):
        assert np.array_equal(got[key], want[key]), key
    L.kuq_host_free(h_rec); L.kuq_host_free(h_off)


# ---- exported values ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [15, 19, 21, 25, 28])
def test_export_db_values_and_set_lcas(oracle, landing, k):
    """after staging, the exported image equals the file (values at the file's stride); after kuq_set_lcas_batch it
    equals the oracle's set_lcas"""
    rng = np.random.default_rng(500 + k)
    tax = synth.make_taxonomy(6, 3, 2, first_id=100)
    sp = synth.species_ids(tax)
    genomes = synth.random_genomes(rng, 6, 2000, shared_frac=0.3)
    km, tx = synth.label_kmers(genomes, sp, tax, k)
    kdb, idx = synth.build_db_images(km, tx, k, 7, 2)
    landing(2048)
    clf = binding.Classifier(max_reads=1 << 16, max_bases=16 << 20)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*tax.parent_map())
    out = kdb.copy()
    _, _, vals = synth.parse_kdb(out)
    kl = synth.key_len(k)
    header = kdb.size - (kl + 4) * len(vals)
    out[header:].reshape(-1, kl + 4)[:, kl:] = 0
    clf.export_db_values(out)
    assert np.array_equal(out, kdb)
    # set_lcas on a database with zeroed values (db_sort -z), pieces of 400 bases overlapping by k - 1
    drop = rng.random(len(km)) < 0.05
    kdb0, idx0 = synth.build_db_images(km[~drop], np.zeros(int((~drop).sum()), np.uint32), k, 7, 2)
    seqs = [synth.decode(g).tobytes() for g in genomes]
    ids, parents = tax.parent_map()
    odb = oracle.open_db(kdb0.copy(), idx0)
    missing = sum(oracle.set_lcas_sequence(odb, oracle.parent_map(ids, parents), s, t) for s, t in zip(seqs, sp))
    pieces, taxids = [], []
    for s, t in zip(seqs, sp):
        for i in range(0, len(s), 400):
            pieces.append(s[i:i + 400 + k - 1])
            taxids.append(t)
    clf = binding.Classifier(max_reads=1 << 16, max_bases=16 << 20)
    clf.stage_db(kdb0, idx0)
    clf.set_taxonomy(ids, parents)
    assert clf.set_lcas(*synth.pack_reads(pieces), taxids) == missing
    out = kdb0.copy()
    clf.export_db_values(out)
    assert np.array_equal(out, odb.kdb)


# ---- refusals -------------------------------------------------------------------------------------------------
def test_refusals():
    clf = binding.Classifier(max_reads=1 << 10, max_bases=1 << 20)
    kdb, idx = synth.build_db_images(np.arange(1, 100, dtype=np.uint64) * 7919, np.full(99, 5, np.uint32), 21, 6, 2)
    k32 = kdb.copy()
    k32[8:16] = np.frombuffer(np.uint64(64).tobytes(), np.uint8)         # key_bits 64: k = 32
    with pytest.raises(binding.KuqError) as e:
        clf.stage_db(k32, idx)
    assert e.value.code == -5, str(e.value)            # KUQ_E_UNSUPPORTED_K
    # an index whose minimizer length exceeds k
    k6, _ = synth.build_db_images(np.arange(1, 50, dtype=np.uint64), np.full(49, 5, np.uint32), 6, 6, 2)
    idx7 = np.concatenate([np.frombuffer(b"KRAKIX2", np.uint8), np.array([7], np.uint8),
                           np.full(4 ** 7 + 1, 49, np.uint64).view(np.uint8)])
    idx7[8:16] = 0
    with pytest.raises(binding.KuqError) as e:
        clf.stage_db(k6, idx7)
    assert e.value.code == -4, str(e.value)            # KUQ_E_DB_FORMAT
    clf.stage_db(kdb, idx)                               # the context is still usable


# ---- the drop-in executables at k = 21 against the reference's outputs ------------------------------------------
def _k21_inputs(d):
    """k = 21 (10-byte records) from a seed: database (nt = 8) and a second database b (nt = 7, the first four genomes
    labelled with the next species plus a genome only b holds), taxonomy, reads.  The numpy builder is pinned against
    the reference's db_sort and set_lcas at k = 21 by tests/test_oracle_short_k.py."""
    rng = np.random.default_rng(21)
    tax = synth.make_taxonomy(6, 3, 2, first_id=100)
    sp = synth.species_ids(tax)
    genomes = synth.random_genomes(rng, 6, 1800, shared_frac=0.2)
    extra = rng.integers(0, 4, 1800, dtype=np.uint8)
    tax.write(str(d / "taxDB"))
    for name, gs, ts, nt in (("database", genomes, sp, 8), ("b", genomes[:4] + [extra], sp[1:5] + [sp[5]], 7)):
        kdb, idx = synth.build_db_images(*synth.label_kmers(gs, ts, tax, 21), 21, nt, 2)
        kdb.tofile(d / f"{name}.kdb")
        idx.tofile(d / f"{name}.idx")
    reads, offs = synth.sample_reads(rng, genomes + [extra], 400, 150, 0.01, 0.2, 0.2)
    g0, g3 = (synth.decode(g).tobytes() for g in (genomes[0], genomes[3]))
    seqs = [reads[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(400)]
    seqs += [b"", b"ACGT", g0[:20], g0[:21], g0[:22], b"N" * 150, g0[100:250].lower(), g0[10:45] + b"N" + g3[200:235]]
    with open(d / "reads.fa", "wb") as f:
        for i, s in enumerate(seqs):
            f.write(b">r%d\n" % i + s + b"\n")
    return tax, genomes


def _report_lines(path):
    rows = {}
    for line in open(path):
        if line.startswith("#") or line.startswith("%"):
            continue
        f = line.rstrip("\n").split("\t")
        rows[f[6]] = f
    return rows


REPLICAS = {"KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"}
SHARDS = {"KUQ_FORCE_SHARDS": "1", "KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"}
# tag: (tool, databases, the reference's flags, runs of ours: (our flags or None = the same, environment, stderr holds))
CLI = {
    "preload": ("classify", ["database"], ["-M"], [(None, {}, ""), (None, REPLICAS, "2 GPUs, database replicated")]),
    "preload_u20000": ("classify", ["database"], ["-M", "-u", "20000"],
                       [(None, {}, ""), (None, REPLICAS, "2 GPUs, database replicated")]),
    # -x: staged whole, streamed in ranges, sharded; and -M with an HBM budget between the file's size and the widened
    # size, which has to be processed in ranges (the -x rule), so counting file bytes fails here
    "chunked": ("classify", ["database"], ["-x", "16K"],
                [(None, {}, ""), (None, {"KUQ_FORCE_CHUNKS": "1"}, "Database split into"), (["-M"], SHARDS, "sharded over 2 GPUs"),
                 (["-M"], "budget", "processing it in ranges")]),
    "q2": ("classify", ["database"], ["-M", "-q", "-m", "2"], [(None, {}, "")]),
    "exact": ("classifyExact", ["database"], ["-M"], [(None, {}, "")]),
    "ab": ("classify", ["database", "b"], ["-M"], [(None, {}, "")]),
}


@pytest.mark.parametrize("tag", list(CLI))
def test_cli_k21_matches_reference(reference, tmp_path, tag):
    tool, dbs, flags, runs = CLI[tag]
    _k21_inputs(tmp_path)
    common = sum((["-d", f"{d}.kdb", "-i", f"{d}.idx"] for d in dbs), []) + ["-a", "taxDB", "-t", "1"]
    r = reference.run_tool(tool, common + ["-r", "ref.report", "-o", "ref.kraken"] + flags + ["reads.fa"], cwd=tmp_path)
    assert r.returncode == 0, r.stderr[-1500:]
    want_kraken, want_report = open(tmp_path / "ref.kraken").read(), _report_lines(tmp_path / "ref.report")
    build.build_classify()
    exe = os.path.join(os.path.dirname(build.CLASSIFY), tool)
    for ours, env, note in runs:
        if env == "budget":
            key_ct = int(np.fromfile(tmp_path / "database.kdb", np.uint64, count=7)[6])
            file_bytes = os.path.getsize(tmp_path / "database.kdb") + os.path.getsize(tmp_path / "database.idx")
            widened = key_ct * 12 + os.path.getsize(tmp_path / "database.idx")
            assert file_bytes < widened
            env = {"KUQ_HBM_BUDGET": str((file_bytes + widened) // 2)}
        cmd = [exe] + common + ["-r", "out.report", "-o", "out.kraken"] + (flags if ours is None else ours) + ["reads.fa"]
        r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True,
                           env=dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22), **env))
        assert r.returncode == 0, r.stderr[-2000:]
        assert note in r.stderr, (env, r.stderr[:1500])
        assert "split into 1 chunks" not in r.stderr
        assert open(tmp_path / "out.kraken").read() == want_kraken, env
        assert _report_lines(tmp_path / "out.report") == want_report, env


def test_cli_db_sort_and_set_lcas_k21(tmp_path, oracle):
    """the drop-in db_sort -z and set_lcas -x rebuild a k = 21 database byte for byte like the oracle's statements of the
    two tools (held against the reference's executables at k = 21 by tests/test_oracle_short_k.py)"""
    db_sort, set_lcas = build.build_dbtools()
    tax, genomes = _k21_inputs(tmp_path)
    seqs = [synth.decode(g).tobytes() for g in genomes]
    with open(tmp_path / "lib.fa", "wb") as f, open(tmp_path / "seqid2taxid.map", "w") as m:
        for i, (s, t) in enumerate(zip(seqs, synth.species_ids(tax))):
            f.write(b">seq%d\n" % i + b"\n".join(s[j:j + 70] for j in range(0, len(s), 70)) + b"\n")
            m.write(f"seq{i}\t{t}\n")
    allk = np.unique(np.concatenate([synth.canonical(km[ok], 21) for km, ok in (synth.forward_kmers(g, 21) for g in genomes)]))
    jdb = synth.unsorted_jdb_image(allk, 21)
    jdb.tofile(tmp_path / "database.jdb")
    r = subprocess.run([db_sort, "-z", "-n", "8", "-d", "database.jdb", "-o", "new.kdb", "-i", "new.idx"],
                       cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    want_kdb, want_idx = oracle.db_sort(jdb, 8, True)
    assert np.array_equal(np.fromfile(tmp_path / "new.idx", np.uint8), want_idx)
    assert np.array_equal(np.fromfile(tmp_path / "new.kdb", np.uint8), want_kdb)
    r = subprocess.run([set_lcas, "-x", "-d", "new.kdb", "-i", "new.idx", "-b", "taxDB", "-m", "seqid2taxid.map",
                        "-F", "lib.fa"], cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    odb = oracle.open_db(want_kdb.copy(), want_idx)
    pm = oracle.parent_map(*tax.parent_map())
    for s, t in zip(seqs, synth.species_ids(tax)):
        oracle.set_lcas_sequence(odb, pm, s, t)
    assert np.array_equal(np.fromfile(tmp_path / "new.kdb", np.uint8), odb.kdb)
    # and both equal the database the numpy builder makes from the labelled k-mers
    assert np.array_equal(odb.kdb, np.fromfile(tmp_path / "database.kdb", np.uint8))
