"""Several databases sharded over GPUs by minimizer range (`classify -d A -d B` when the databases fit the node's GPUs
only together): one lookup phase per run of databases with equal (nt, index type), every database of a run cut at the
same bins, hits stored into the id buffer of the GPU that resolves the read, device flags between the phases, the owners
doing the sketch work under the per-work-unit rule.  On one H100 the GPUs are several contexts on device 0
(KUQ_DEVICES=0,0 / 0,0,0).  Checked against the reference's golden runs, the oracle, and the resident and streamed
layouts of the same inputs, which must give the same bytes."""
import os
import re
import shutil

import numpy as np
import pytest
import torch

from krakenuniq_b200 import binding, build, synth
from krakenuniq_b200 import dist as kdist
from tests import util
from tests.test_multi_db_gpu import (M, _check_reads, _cli, _oracle, _report_matches_oracle, _report_rows, _runs_to_codes,
                                     _same_counts, _workload)

pytestmark = pytest.mark.gpu
G = util.GOLDEN
DEV = "cuda:0"
FLAG_TIMEOUT_MS = 5000


def _shards(n_ctx):
    return {"KUQ_FORCE_SHARDS": "1", "KUQ_DEVICES": ",".join(["0"] * n_ctx)}


def _sharded_line(err, n_db, n_ctx, phases):
    assert f"{n_db} databases sharded over {n_ctx} GPUs by minimizer range ({phases} lookup phases)" in err, err[-2000:]
    assert "not usable" not in err, err[-2000:]


def _idx_params(idx):
    idx = np.asarray(idx).view(np.uint8)
    return int(idx[7]), 1 if bytes(idx[:7]) == b"KRAKIDX" else 2, idx[8:].view(np.uint64)


def _plan(dbs, n_ctx):
    """the cuts classify makes: runs of equal (nt, index type), one cut per run by the run's summed record counts"""
    runs = []
    for i, (_, idx) in enumerate(dbs):
        nt, it, offs = _idx_params(idx)
        if runs and runs[-1]["nt"] == nt and runs[-1]["type"] == it:
            runs[-1]["dbs"].append(i)
            runs[-1]["sum"] = runs[-1]["sum"] + offs
        else:
            runs.append(dict(nt=nt, type=it, dbs=[i], sum=offs.copy()))
    for r in runs:
        n_bins = 1 << (2 * r["nt"])
        total = int(r["sum"][n_bins])
        cut = [0] + [int(np.searchsorted(r["sum"][:n_bins], total // n_ctx * g, "left")) for g in range(1, n_ctx)] + [n_bins]
        r["cut"] = list(np.maximum.accumulate(cut))
    return runs


# ---- the reference's golden two-database runs ---------------------------------------------------------------------
@pytest.mark.parametrize("n_ctx", [2, 3])
@pytest.mark.parametrize("tag", ["ab", "ba", "ab_q2", "ba_q1"])
def test_golden_two_databases_sharded(tmp_path, tag, n_ctx):
    """the mini database (nt 6, KRAKIX2) and db2 (nt 5, KRAKIDX): two lookup phases; missing .counts are regenerated"""
    for f in ("database.kdb", "database.idx"):
        shutil.copy(os.path.join(G, f), tmp_path / f)
    for f in ("db2.kdb", "db2.idx"):
        shutil.copy(os.path.join(M, f), tmp_path / f)
    a = (str(tmp_path / "database.kdb"), str(tmp_path / "database.idx"))
    b = (str(tmp_path / "db2.kdb"), str(tmp_path / "db2.idx"))
    quick = {"ab_q2": ["-q", "-m", "2"], "ba_q1": ["-q", "-m", "1"]}.get(tag, [])
    kraken, rows, err = _cli(build.build_classify(), [a, b] if tag.startswith("ab") else [b, a], os.path.join(G, "taxDB"),
                             os.path.join(G, "reads.fa"), str(tmp_path), ["-u", "20000"] + quick, _shards(n_ctx))
    _sharded_line(err, 2, n_ctx, 2)
    assert kraken == open(os.path.join(M, f"{tag}.kraken")).read()
    assert rows == _report_rows(os.path.join(M, f"{tag}.report.tsv"))
    assert open(tmp_path / "database.kdb.counts").read() == open(os.path.join(G, "database.kdb.counts")).read()
    assert open(tmp_path / "db2.kdb.counts").read() == open(os.path.join(M, "db2.kdb.counts.golden")).read()


# ---- synthetic databases: the oracle, and resident = streamed = sharded -------------------------------------------
def _converting_workload(seed, k=31):
    """two databases over 4 genomes of 12 kbp, 2500 reads of 150 bp and one whole genome as one read: with a small -u
    that read is a work unit whose (unit, taxon) pair sees thousands of distinct k-mers, so its sketch turns dense"""
    rng = np.random.default_rng(seed)
    tax = synth.make_taxonomy(4, 2)
    sp = synth.species_ids(tax)
    genomes = synth.random_genomes(rng, 4, 12000, 0.1)
    km, tx = synth.label_kmers(genomes, sp, tax, k)
    r = rng.random(len(km))
    dbs = [synth.build_db_images(km[r < 0.8], tx[r < 0.8], k, 9, 2), synth.build_db_images(km[r > 0.5], tx[r > 0.5], k, 7, 1)]
    bases, offs = synth.sample_reads(rng, genomes, 2500, 150, 0.01, 0.1, 0.2)
    seqs = [bases[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)]
    seqs.insert(1200, synth.decode(genomes[0]).tobytes())
    return tax, dbs, seqs


def _write_dbs(d, dbs):
    paths = []
    for i, (kdb, idx) in enumerate(dbs):
        kp, ip = str(d / f"db{i}.kdb"), str(d / f"db{i}.idx")
        kdb.tofile(kp)
        idx.tofile(ip)
        paths.append((kp, ip))
    return paths


def _write_reads(d, tax, seqs, crlf_every=7):
    """taxDB and a multi-line FASTA, some records with CRLF line ends"""
    tax.write(str(d / "taxDB"))
    with open(d / "reads.fa", "wb") as f:
        for i, s in enumerate(seqs):
            nl = b"\r\n" if i % crlf_every == 0 else b"\n"
            f.write(b">r%d x\n" % i + nl.join(s[j:j + 60] for j in range(0, len(s), 60)) + nl)


def _layouts(tmp_path, dbs, tax, extra, n_ctx, phases, layouts=("resident", "streamed", "sharded")):
    """the CLI in each layout, each with its own copy of the databases (so that each writes the .counts files); returns
    {layout: (kraken, report text, [counts texts])}"""
    hbm = [kdb.size + idx.size for kdb, idx in dbs]
    env = {"resident": {}, "streamed": {"KUQ_HBM_BUDGET": str(int(max(hbm) * 0.9))}, "sharded": _shards(n_ctx)}
    got = {}
    for mode in layouts:
        d = tmp_path / mode
        d.mkdir()
        paths = _write_dbs(d, dbs)
        kraken, _, err = _cli(build.build_classify(), paths, str(tmp_path / "taxDB"), str(tmp_path / "reads.fa"), str(d), extra,
                              env[mode])
        if mode == "sharded":
            _sharded_line(err, len(dbs), n_ctx, phases)
        elif mode == "resident":
            assert re.search(rf"{len(dbs)} databases resident on \d+ GPU", err), err[-2000:]
        else:
            assert re.search(r"databases streamed: \d+ rounds", err), err[-2000:]
        got[mode] = (kraken, open(d / "o.report.tsv").read(), [open(kp + ".counts").read() for kp, _ in paths])
    return got


CASES = {
    # name: (workload seed, k, shapes or None for the converting workload, -u, -q -m, contexts, lookup phases)
    "three_runs": (21, 31, [(9, 2), (7, 1), (9, 2)], 30000, 0, 3, 3),
    "one_run": (22, 31, [(8, 2)] * 3, 30000, 0, 2, 1),
    "empty_database_in_run": (23, 31, [(8, 2), (-8, 2), (8, 2)], 30000, 0, 3, 1),
    "k21": (24, 21, [(9, 2), (7, 2), (9, 1)], 30000, 0, 2, 3),
    "quick_m2": (25, 31, [(9, 2), (7, 1), (9, 2)], 30000, 2, 2, 3),
    "small_unit_converting_taxon": (26, 31, None, 2000, 0, 3, 2),
}


@pytest.mark.parametrize("case", list(CASES))
def test_cli_sharded_matches_oracle_and_other_layouts(oracle, tmp_path, case):
    seed, k, shapes, unit, quick, n_ctx, phases = CASES[case]
    tax, dbs, seqs = _converting_workload(seed, k) if shapes is None else _workload(seed, k, shapes, n_reads=20000)
    _write_reads(tmp_path, tax, seqs)
    ids, rseqs = util.read_fasta(str(tmp_path / "reads.fa"))
    calls, codes, code_off, cnt, _, run = _oracle(oracle, tax, dbs, rseqs, unit, quick=quick)
    extra = ["-u", str(unit)] + (["-q", "-m", str(quick)] if quick else [])
    got = _layouts(tmp_path, dbs, tax, extra, n_ctx, phases)
    kraken = got["sharded"][0]
    if quick:
        assert [int(l.split("\t")[2]) for l in kraken.splitlines()] == [int(c) for c in calls]
    else:
        assert kraken == util.kraken_lines(ids, rseqs, calls, codes, code_off)
    _report_matches_oracle(str(tmp_path / "sharded" / "o.report.tsv"), tax, cnt, run)
    assert got["sharded"] == got["resident"]
    assert got["streamed"] == got["resident"]


def _one_bin_db(km, tx, k, nt, it, bin_of_choice, limit=None):
    """a database holding only the k-mers of one minimizer bin (at most `limit` of them)"""
    bins = synth.bin_key(km, k, nt, it)
    keep = bins == bins[bin_of_choice]
    if limit is not None:
        keep &= np.cumsum(keep) <= limit
    return synth.build_db_images(km[keep], tx[keep], k, nt, it), int(bins[bin_of_choice])


def test_cut_edges(oracle, tmp_path):
    """a database of a run whose records all fall inside one context's range (the other contexts hold slices without
    records), and a run of one database with fewer non-empty bins than contexts (empty slices, the first one at bin 0):
    both give the resident run's bytes"""
    k = 31
    tax, dbs, seqs = _workload(31, k, [(8, 2)], n_reads=8000)
    rng = np.random.default_rng(5)
    sp = synth.species_ids(tax)
    genomes = synth.random_genomes(np.random.default_rng(31), 12, 2500, 0.25)
    km, tx = synth.label_kmers(genomes, sp, tax, k)
    one_bin, b = _one_bin_db(km, np.asarray(sp, np.uint32)[rng.integers(0, len(sp), len(km))], k, 8, 2, 17)
    single, _ = _one_bin_db(km, tx, k, 7, 1, 400, limit=2)
    all_dbs = [dbs[0], one_bin, single]
    plan = _plan(all_dbs, 3)
    assert len(plan) == 2 and plan[0]["dbs"] == [0, 1] and plan[1]["dbs"] == [2]
    cut = plan[0]["cut"]
    assert sum(cut[g] <= b < cut[g + 1] for g in range(3)) == 1
    _, _, single_offs = _idx_params(single[1])
    assert np.count_nonzero(np.diff(single_offs.astype(np.int64))) == 1 and plan[1]["cut"][:3] == [0, 0, 0]
    _write_reads(tmp_path, tax, seqs)
    got = _layouts(tmp_path, all_dbs, tax, ["-u", "30000"], 3, 2, layouts=("resident", "sharded"))
    assert got["sharded"] == got["resident"]
    ids, rseqs = util.read_fasta(str(tmp_path / "reads.fa"))
    calls, codes, code_off, _, _, _ = _oracle(oracle, tax, all_dbs, rseqs, 30000)
    assert got["sharded"][0] == util.kraken_lines(ids, rseqs, calls, codes, code_off)


# ---- the C ABI: contexts on device 0, device flags between the phases ---------------------------------------------
def _shard_contexts(tax, dbs, plan, n_ctx, unit):
    ctxs = []
    for g in range(n_ctx):
        c = binding.Classifier(device=0, max_reads=1 << 15, max_bases=8 << 20, work_unit_size=unit, sparse_set_slots=1 << 22,
                               hll_mode=binding.HLL_PRELOAD)
        for r in plan:
            lo, hi = r["cut"][g], r["cut"][g + 1]
            if lo == hi:
                lo = hi = 1 << (2 * r["nt"])                 # an empty slice
            for d in r["dbs"]:
                c.stage_db_append_range(*dbs[d], lo, hi)
        assert c.db_runs() == len(plan)
        ctxs.append(c)
    universe = sorted(set().union(*[set(c.db_taxids()[0].tolist()) for c in ctxs]))
    for c in ctxs:
        c.set_db_taxid_universe(universe)
        c.set_taxonomy(*tax.parent_map())
    return ctxs


def _unit_shares(units, n_ctx):
    n = len(units)
    first = [0]
    for g in range(1, n_ctx):
        x = max(first[-1], min(n, n * g // n_ctx))
        while 0 < x < n and units[x] == units[x - 1]:
            x += 1
        first.append(x)
    return first + [n]


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a).astype(dtype)).to(DEV)


def _run_phases(ctxs, n_phases, d_bases, d_offs, n, total, ids, bounds, flags=True):
    """every phase of every context, with device flags between them (queued before the host waits for anything), or
    phase by phase with host synchronisation; returns the probe counts [context][phase] in the second case"""
    world = len(ctxs)
    stats = [[0] * n_phases for _ in ctxs]
    if not flags:
        for r in range(n_phases):
            for g, c in enumerate(ctxs):
                c.lookup_device_peers_run(0, d_bases.data_ptr(), d_offs.data_ptr(), n, total, [t.data_ptr() for t in ids], bounds, r)
                stats[g][r] = c.slot_stats(0)[0]
        return stats, None
    flg = [c.device_alloc(256) for c in ctxs]            # [0:64) done counters, [128:192) ready counters
    for f in flg:
        ft = kdist.device_view(f, 256, torch.int64, DEV)
        ft.zero_()
        ft[16:24] = 1                                      # the buffers are clean for the one step
    torch.cuda.synchronize()
    for r in range(n_phases):
        for g, c in enumerate(ctxs):
            c.wait_flags(0, flg[g] + 128 if r == 0 else flg[g], world, 1 if r == 0 else r, timeout_ms=FLAG_TIMEOUT_MS)
            c.lookup_device_peers_run(0, d_bases.data_ptr(), d_offs.data_ptr(), n, total, [t.data_ptr() for t in ids], bounds, r)
            c.signal_peers(0, flg, g, r + 1)
    for g, c in enumerate(ctxs):
        c.wait_flags(0, flg[g], world, n_phases, timeout_ms=FLAG_TIMEOUT_MS)
    for c in ctxs:
        c.sync(0)                                          # a flag wait that timed out fails here with KUQ_E_STATE
    return stats, flg


def _abi_case(seed=41):
    return _workload(seed, 31, [(9, 2), (7, 1), (9, 2), (9, 2), (-6, 2)], n_reads=6000)


@pytest.mark.parametrize("n_ctx", [2, 3])
def test_cabi_sharded_matches_oracle(oracle, n_ctx):
    """calls, hit lists and merged counts of the owners' resolve halves, and the merged first-hit codes per window
    (KUQ_CODE_FOUND_ZERO included) against the oracle's in-order query"""
    unit = 30000
    tax, dbs, seqs = _abi_case()
    calls, codes, code_off, want, odbs, _ = _oracle(oracle, tax, dbs, seqs, unit)
    plan = _plan(dbs, n_ctx)
    assert len(plan) == 4
    ctxs = _shard_contexts(tax, dbs, plan, n_ctx, unit)
    bases, offs = synth.pack_reads(seqs)
    units = synth.work_unit_ids(offs, unit)[0]
    n, total = len(offs) - 1, int(offs[-1])
    first = _unit_shares(units, n_ctx)
    bounds = np.array([int(offs[a]) for a in first], np.uint64)
    bounds[0] = 0
    d_bases = _dev(np.concatenate([bases, np.full(64, ord("N"), np.uint8)]), np.uint8)
    d_offs = _dev(np.concatenate([offs, offs[-1:], offs[-1:]]), np.int64)
    ids = [torch.zeros(total + 64, dtype=torch.int32, device=DEV) for _ in ctxs]
    torch.cuda.synchronize()
    _, flg = _run_phases(ctxs, len(plan), d_bases, d_offs, n, total, ids, bounds)
    # merged first-hit codes: each position from its owner's buffer
    host = [t.cpu().numpy().view(np.uint32) for t in ids]
    merged = np.zeros(total, np.uint32)
    for g in range(n_ctx):
        merged[int(bounds[g]):int(offs[first[g + 1]])] = host[g][int(bounds[g]):int(offs[first[g + 1]])]
    raw = ctxs[0].dense_taxids()
    o = odbs[0].o
    for i, s in enumerate(seqs[:400]):
        kmers, amb = o.scan(s, 31)
        want_codes = []
        for km, a in zip(kmers.tolist(), amb.tolist()):
            v = 0
            if not a:
                c = o.canonical(km, 31)
                for d in odbs:
                    found, t = d.query(c)
                    if found:
                        v = t if t else binding.CODE_FOUND_ZERO
                        break
            want_codes.append(v)
        g_ = merged[int(offs[i]):int(offs[i]) + len(want_codes)]
        g_ = np.where((g_ == binding.CODE_FOUND_ZERO) | (g_ == 0), g_, raw[np.minimum(g_, len(raw) - 1)])
        assert np.array_equal(g_, np.array(want_codes, np.uint32)), f"read {i}"
    # the owners resolve their shares (whole work units) with work-unit ids
    got_calls, got_codes = [], []
    for g, c in enumerate(ctxs):
        a, b = first[g], first[g + 1]
        if b == a:
            continue
        d_own = _dev(np.concatenate([offs[a:b + 1], offs[b:b + 1], offs[b:b + 1]]), np.int64)
        d_units = _dev(units[a:b], np.int32)
        c.resolve_device(0, d_bases.data_ptr(), d_own.data_ptr(), b - a, total, ids[g].data_ptr(), d_units.data_ptr())
        res = c.collect_device(0)
        got_calls.append(res["call"])
        got_codes += [_runs_to_codes(res, i) for i in range(b - a)]
    for c in ctxs:
        c.finish()
    _check_reads(np.concatenate(got_calls), got_codes, calls, codes, code_off)
    for c in ctxs[1:]:
        ctxs[0].merge_from(c)
    _same_counts(ctxs[0].counts(), want)
    for c, f in zip(ctxs, flg):
        c.device_free(f)


def test_cabi_each_context_fetches_only_its_open_windows(oracle):
    """probe statistics: in phase r, context g fetches once per database it asks (in order, up to the first that holds
    the key) for exactly the non-ambiguous windows whose bin lies in its range of run r and that no earlier run
    answered on any context"""
    n_ctx, unit = 3, 30000
    tax, dbs, seqs = _abi_case(42)
    seqs = seqs[:1500]
    _, _, _, _, odbs, _ = _oracle(oracle, tax, dbs, seqs, unit)
    plan = _plan(dbs, n_ctx)
    ctxs = _shard_contexts(tax, dbs, plan, n_ctx, unit)
    for c in ctxs:
        c.set_stats(True)
    bases, offs = synth.pack_reads(seqs)
    n, total = len(offs) - 1, int(offs[-1])
    first = _unit_shares(synth.work_unit_ids(offs, unit)[0], n_ctx)
    bounds = np.array([int(offs[a]) for a in first], np.uint64)
    bounds[0] = 0
    d_bases = _dev(np.concatenate([bases, np.full(64, ord("N"), np.uint8)]), np.uint8)
    d_offs = _dev(np.concatenate([offs, offs[-1:], offs[-1:]]), np.int64)
    ids = [torch.zeros(total + 64, dtype=torch.int32, device=DEV) for _ in ctxs]
    torch.cuda.synchronize()
    stats, _ = _run_phases(ctxs, len(plan), d_bases, d_offs, n, total, ids, bounds, flags=False)
    # the model: canonical k-mers of the non-ambiguous windows, which databases hold them, their bins per run
    o = odbs[0].o
    canon = []
    for s in seqs:
        kmers, amb = o.scan(s, 31)
        canon += [o.canonical(km, 31) for km, a in zip(kmers.tolist(), amb.tolist()) if not a]
    canon = np.array(canon, np.uint64)
    held = np.array([[d.query(int(c))[0] for d in odbs] for c in canon.tolist()], bool).reshape(len(canon), len(odbs))
    answered = np.zeros(len(canon), bool)
    want = [[0] * len(plan) for _ in range(n_ctx)]
    for r, run in enumerate(plan):
        bins = synth.bin_key(canon, 31, run["nt"], run["type"]).astype(np.int64)
        h = held[:, run["dbs"]]
        asked = np.where(h.any(axis=1), h.argmax(axis=1) + 1, len(run["dbs"]))
        for g in range(n_ctx):
            mine = (bins >= run["cut"][g]) & (bins < run["cut"][g + 1]) & ~answered
            want[g][r] = int(asked[mine].sum())
        answered |= h.any(axis=1)
    assert stats == want


# ---- errors -------------------------------------------------------------------------------------------------------
def test_errors_leave_the_context_usable(oracle):
    tax, dbs, seqs = _workload(51, 31, [(8, 2), (7, 1)], n_reads=1500)
    _, dbs21, _ = _workload(52, 21, [(8, 2)], n_reads=10)
    c = binding.Classifier(device=0, max_reads=1 << 15, max_bases=8 << 20, work_unit_size=30000, sparse_set_slots=1 << 22)
    c.stage_db_append_range(*dbs[0], 0, 0)
    with pytest.raises(binding.KuqError) as e:
        c.stage_db_append_range(*dbs21[0], 0, 1 << 15)
    assert "differ in k" in str(e.value)
    for lo, hi in ((0, (1 << 14) + 1), (5, 3), (1 << 14, 1 << 16)):
        with pytest.raises(binding.KuqError) as e:
            c.stage_db_append_range(*dbs[1], lo, hi)
        assert e.value.code == -1 and "outside" in str(e.value), (lo, hi, str(e.value))
    c.stage_db_append_range(*dbs[1], 0, 1 << 13)          # the second database in two slices: one run
    c.stage_db_append_range(*dbs[1], 1 << 13, 1 << 14)
    assert c.db_runs() == 2
    c.set_taxonomy(*tax.parent_map())
    calls, codes, code_off, want, _, _ = _oracle(oracle, tax, dbs, seqs, 30000)
    res = c.classify(*synth.pack_reads(seqs))
    assert np.array_equal(res["call"], calls)
    # shard counting and the one-database peer lookup stay refused on several databases
    bases, offs = synth.pack_reads(seqs[:10])
    d_bases = _dev(np.concatenate([bases, np.full(64, ord("N"), np.uint8)]), np.uint8)
    d_offs = _dev(np.concatenate([offs, offs[-1:], offs[-1:]]), np.int64)
    ids = torch.zeros(int(offs[-1]) + 64, dtype=torch.int32, device=DEV)
    args = (0, d_bases.data_ptr(), d_offs.data_ptr(), len(offs) - 1, int(offs[-1]), [ids.data_ptr()], [0, int(offs[-1])])
    with pytest.raises(binding.KuqError) as e:
        c.lookup_device_peers(*args)
    assert e.value.code == -6
    c.set_shard_counting(True)
    with pytest.raises(binding.KuqError) as e:
        c.lookup_device_peers_run(*args, 0)
    assert e.value.code == -6
    c.set_shard_counting(False)
    with pytest.raises(binding.KuqError):
        c.lookup_device_peers_run(*args, 2)          # there are two runs
    c.lookup_device_peers_run(*args, 1)
    c.sync(0)
