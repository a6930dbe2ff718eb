"""Key search and HLL hash tails on crafted k-mers (tests/crafted.py), against the oracle.

Random databases reach three decisive paths with a probability no test comes near: two records of one scan window that
share the low 32-bit key word (the low-word compare of the bin search matches both and only the high word tells them
apart), hashes of rank 33..53 (the leading one in the low half of the hash, or none at all) and flagged sparse codes
(hash bits 51..39 zero) with large additional ranks or shared top-25 bits.  A wrong rank 30 against 31 moves the Ertl
estimate by 2^-31, so these tests compare the state itself — codes, registers, sparse keys, rank histograms — and not
only the estimates.  Each case first checks with numpy that its database and reads hold the shapes it claims."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from krakenuniq_b200 import binding, build, synth  # noqa: E402
from krakenuniq_b200 import dist as kdist  # noqa: E402
from tests import crafted, util  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_U = np.uint64
TAX = synth.Taxonomy([(1, 1, "root", "no rank"), (10, 1, "g", "genus"), (11, 10, "a", "species"),
                      (12, 10, "b", "species"), (20, 1, "h", "genus"), (21, 20, "c", "species"),
                      (22, 20, "d", "species")])
SPECIES = [11, 12, 21, 22]


def _runs_to_codes(res, i):
    out = []
    for code, cnt in binding.decode_runs(res, i):
        out += [code] * cnt
    return np.array(out, np.uint32)


def _db(keys, taxa, k, nt, idx_type):
    order = np.argsort(keys)
    keys, taxa = keys[order], taxa[order]
    assert len(np.unique(keys)) == len(keys)
    return synth.build_db_images(keys, taxa, k, nt, idx_type)


def _same_counts(got, want, dense_only=False):
    for key in ("taxid", "n_reads", "n_kmers") + (() if dense_only else ("sparse", "unique")):
        assert np.array_equal(got[key], want[key]), (key, got[key], want[key])


def _same_regs(clf, want):
    for j, t in enumerate(want["taxid"]):
        assert np.array_equal(clf.registers(int(t)), want["regs"][j]), f"registers of taxon {t}"


def _same_reads(res, calls, codes, code_off, offs):
    assert np.array_equal(res["call"], calls)
    assert np.array_equal(res["n_windows"], np.diff(code_off).astype(np.uint32))
    assert res["n_classified"] == int((calls != 0).sum())
    for i in range(len(offs) - 1):
        w = codes[int(code_off[i]):int(code_off[i + 1])]
        if "codes" in res:
            o = int(offs[i]) - int(offs[0])
            assert np.array_equal(res["codes"][o:o + len(w)], w), f"codes of read {i}"
        assert np.array_equal(_runs_to_codes(res, i), w), f"hit list of read {i}"


# ==== key search ===================================================================================================
def _pivots(n, levels=3):
    """record positions (inside the bin) of the pivots of the first `levels` 4-ary narrowing steps of k_lookup"""
    out, todo = [], [(0, n)]
    for _ in range(levels):
        nxt = []
        for lo, m in todo:
            if m <= 8:
                continue
            q = m >> 2
            out += [lo + q, lo + 2 * q, lo + 3 * q]
            nxt += [(lo, q), (lo + q, q), (lo + 2 * q, q), (lo + 3 * q, m - 3 * q)]
        todo = nxt
    return out


def _key_search_case(k, nt, idx_type, seed):
    """database: one giant bin (2^17 + 5 records), bins made only of keys sharing one low word (2..8 and 9..40
    records, where k leaves that many prefixes), bins of every size 0..40 side by side, and repeat k-mers, whose bins
    are the highest this case reaches.  Bin 4^nt - 1 is never one of them: its nt-mer is the complement of the xor mask,
    and no k-mer with more than one window (k > nt) has every window on that one canonical nt-mer.  Returns (kdb, idx,
    reads, keys, queries, taxa, facts)."""
    rng = np.random.default_rng(seed)
    bins = crafted.lowest_bins(nt, idx_type, 1 + 4 + 41)
    species = np.array(SPECIES, np.uint32)
    keys, queries, facts = [], [], {}

    giant = np.sort(crafted.kmers_in_bin(k, nt, idx_type, bins[0], (1 << 17) + 5, rng))
    keys.append(giant)
    pos = sorted(set([0, len(giant) - 1] + _pivots(len(giant)) + list(range(0, len(giant), 97))))
    queries.append(giant[pos])
    near = np.concatenate([giant[pos] - _U(1), giant[pos] + _U(1)])
    near = near[crafted.is_canonical(near, k) & (synth.bin_key(near, k, nt, idx_type) == _U(bins[0]))]
    near = np.setdiff1d(near, giant)
    queries.append(near)
    facts["giant"] = (bins[0], len(giant), len(near))

    facts["low_word"] = []
    for j, want in enumerate((2, 8, 9, 40)):
        lw, cand = crafted.kmers_sharing_low_word(k, nt, idx_type, bins[1 + j], rng)
        if len(cand) < 2:                                  # k = 16: the key is its low word
            keys.append(cand)
            queries.append(cand)
            facts["low_word"].append((bins[1 + j], 1, 0))
            continue
        size = min(want, len(cand) - 1)
        if len(cand) >= size + 2:                          # keep absent keys below and above the stored ones
            inner = cand[1:-1]
            stored = np.sort(inner[rng.choice(len(inner), size, replace=False)])
        else:
            stored = np.sort(cand[rng.choice(len(cand), size, replace=False)])
        absent = np.setdiff1d(cand, stored)
        keys.append(stored)
        queries += [stored, absent[rng.permutation(len(absent))[:60]], absent[absent < stored[0]][-3:],
                    absent[absent > stored[-1]][:3], absent[(absent > stored[0]) & (absent < stored[-1])][:6]]
        facts["low_word"].append((bins[1 + j], size, len(absent)))

    sizes = list(range(41))
    rng.shuffle(sizes)
    for b, s in zip(bins[5:], sizes):
        if s:
            km = crafted.kmers_in_bin(k, nt, idx_type, b, s, rng)
            keys.append(km)
            queries.append(km)
    facts["side_by_side"] = (bins[5], bins[-1])

    # the highest bins: repeats of 1..3 bases (their windows are all alike, so a high minimizer is possible)
    rep = []
    for period in (1, 2, 3):
        for u in range(4 ** period):
            motif = [(u >> (2 * (period - 1 - i))) & 3 for i in range(period)]
            x = 0
            for i in range(k):
                x = (x << 2) | motif[i % period]
            rep.append(x)
    rep = np.unique(synth.canonical(np.array(rep, np.uint64), k))
    rep = rep[~np.isin(synth.bin_key(rep, k, nt, idx_type), np.array(bins, np.uint64))]
    keys.append(rep)
    queries.append(rep)

    keys = np.concatenate(keys)
    taxa = species[rng.integers(0, len(species), len(keys))]
    queries = np.concatenate(queries)
    # reads: one to three queried k-mers each, either strand, joined (the windows between them mostly miss)
    reads, i = [], 0
    while i < len(queries):
        m = int(rng.integers(1, 4))
        reads.append(b"".join(crafted.kmer_read(x, k, bool(rng.integers(0, 2))) for x in queries[i:i + m]))
        i += m
    kdb, idx = _db(keys, taxa, k, nt, idx_type)
    return kdb, idx, reads, keys, queries, taxa, facts


def _assert_shapes(kdb, idx, k, nt, idx_type, keys, queries, facts):
    """the database and the reads hold what the case claims"""
    _, dbk, _ = synth.parse_kdb(kdb)
    off = np.frombuffer(idx, np.uint64, offset=8)         # a view: the nt = 15 index is 8.6 GB

    def size(b):
        return int(off[b + 1]) - int(off[b])

    b, n, n_near = facts["giant"]
    assert size(b) >= 1 << 17 and n_near > 100
    lo, hi = facts["side_by_side"]
    assert {size(x) for x in range(lo, hi + 1)} >= set(range(41))
    hits = np.isin(queries, dbk)
    for b, n, n_absent in facts["low_word"]:
        recs = dbk[int(off[b]):int(off[b + 1])]
        assert len(recs) == n and len(np.unique(recs & _U(0xFFFFFFFF))) == 1
        if k >= 19:
            assert n in (2, 8, 9, 40) and n_absent >= 3
        elif k == 17:
            assert n >= 2 and n_absent >= 1
    assert hits.sum() > 1000 and (~hits).sum() > 200
    if crafted.lowest_bins(nt, idx_type, 1)[0] == 0:     # bin 0, where a k-mer can fall into it
        assert size(0) > 0
    assert size((1 << (2 * nt)) - 1) == 0                  # unreachable (see _key_search_case)


KEY_CASES = [(31, 15, 2), (31, 6, 1), (21, 7, 2), (17, 5, 2), (16, 5, 1)]


@pytest.mark.parametrize("k,nt,idx_type", KEY_CASES)
def test_key_search_on_crafted_bins(oracle, k, nt, idx_type):
    kdb, idx, reads, keys, queries, taxa, facts = _key_search_case(k, nt, idx_type, 100 + k + nt)
    _assert_shapes(kdb, idx, k, nt, idx_type, keys, queries, facts)
    bases, offs = synth.pack_reads(reads)
    pm = TAX.parent_map()

    def oracle_run(mode, passes):
        run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*pm), 500000, mode)
        for _ in range(passes):
            calls, codes, code_off = run.classify(bases, offs)
        run.finish()
        return run, calls, codes, code_off

    run1, calls, codes, code_off = oracle_run(0, 1)
    want1 = run1.counts(want_regs=True)
    run2, _, _, _ = oracle_run(0, 2)
    want2 = run2.counts(want_regs=True)

    # the fused call; a readout between two runs (every hit record KEPT, SEEN set again), then reset and a third run
    clf = binding.Classifier(max_reads=1 << 16, max_bases=8 << 20, hll_mode=binding.HLL_PRELOAD, sparse_set_slots=1 << 16)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*pm)
    res = clf.classify(bases, offs, flags=binding.F_WANT_CODES)
    _same_reads(res, calls, codes, code_off, offs)
    clf.counts()                                           # readout: a harvest
    res = clf.classify(bases, offs, flags=binding.F_WANT_CODES)
    _same_reads(res, calls, codes, code_off, offs)
    clf.finish()
    _same_counts(clf.counts(), want2)
    _same_regs(clf, want2)
    clf.reset_counts()
    res = clf.classify(bases, offs, flags=binding.F_WANT_CODES)
    _same_reads(res, calls, codes, code_off, offs)
    clf.finish()
    _same_counts(clf.counts(), want1)
    clf.close()

    # the halves, the database staged in three ranges cut right before and right after the giant bin
    runc, calls, codes, code_off = oracle_run(1, 1)
    wantc = runc.counts(want_regs=True)
    g = facts["giant"][0]
    cuts = [(0, g), (g, g + 1), (g + 1, 1 << (2 * nt))]
    clf = binding.Classifier(max_reads=1 << 16, max_bases=8 << 20, hll_mode=binding.HLL_CHUNKED, sparse_set_slots=1 << 16)
    clf.set_taxonomy(*pm)
    universe = set()
    for lo, hi in cuts:
        if hi > lo:
            clf.stage_db(kdb, idx, lo, hi)
            universe |= set(clf.db_taxids()[0].tolist())
    clf.set_db_taxid_universe(np.array(sorted(universe), np.uint32))
    merged = np.zeros(int(offs[-1]), np.uint32)
    for lo, hi in cuts:
        if hi > lo:
            clf.stage_db(kdb, idx, lo, hi)
            part, _ = clf.lookup(bases, offs)
            merged = np.where(part == binding.AMBIG, merged, np.maximum(merged, part))
    res = clf.resolve(bases, offs, merged, flags=binding.F_WANT_CODES)
    clf.finish()
    _same_reads(res, calls, codes, code_off, offs)
    _same_counts(clf.counts(), wantc)
    _same_regs(clf, wantc)
    clf.close()

    # set_lcas: its own bin search (k_set_lcas), on the same database with zeroed values; every read is a library
    # sequence of one species, so found keys take LCAs and the absent ones count as not found
    kdb0, idx0 = _db(keys, np.zeros(len(keys), np.uint32), k, nt, idx_type)
    lib_taxa = np.array(SPECIES, np.uint32)[np.arange(len(reads)) % len(SPECIES)]
    odb = oracle.open_db(kdb0.copy(), idx0)
    opm = oracle.parent_map(*pm)
    missing = sum(oracle.set_lcas_sequence(odb, opm, s, int(t)) for s, t in zip(reads, lib_taxa))
    _, _, set_vals = synth.parse_kdb(odb.kdb)
    assert missing > 200 and (set_vals != 0).sum() > 1000
    clf = binding.Classifier(max_reads=1 << 16, max_bases=8 << 20)
    clf.stage_db(kdb0, idx0)
    clf.set_taxonomy(*pm)
    assert clf.set_lcas(bases, offs, lib_taxa) == missing
    out = kdb0.copy()
    clf.export_db_values(out)
    assert np.array_equal(out, odb.kdb)
    clf.close()
    if nt == 15:
        return      # the paths below would pin the whole 4^15-bin index in host memory once more

    # kuq_stream_*: two device buffers, the giant bin's range and the rest, loaded from pinned host records
    g1 = g + 1
    n_bins = 1 << (2 * nt)
    off = np.frombuffer(idx, np.uint64, offset=8)
    pair_sz = synth.key_len(k) + 4
    rec = kdb[kdb.size - pair_sz * len(keys):]
    clf = binding.Classifier(max_reads=1 << 16, max_bases=8 << 20, hll_mode=binding.HLL_CHUNKED, n_slots=2,
                             sparse_set_slots=1 << 16)
    clf.set_taxonomy(*pm)
    clf.set_db_taxid_universe(np.unique(taxa))
    ranges = [(0, g1), (g1, n_bins)]
    clf.stream_open(k, nt, idx_type, max(int(off[b] - off[a]) for a, b in ranges), max(b - a for a, b in ranges))
    L = clf.L
    h_rec = L.kuq_host_alloc(rec.size + 16)
    h_off = L.kuq_host_alloc(off.size * 8)
    try:
        ctypes.memmove(h_rec, rec.ctypes.data, rec.size)
        ctypes.memmove(h_off, off.ctypes.data, off.size * 8)
        n, total = len(offs) - 1, int(offs[-1])
        d_bases = torch.from_numpy(np.concatenate([bases, np.full(64, ord("N"), np.uint8)])).to(DEV)
        d_offs = torch.from_numpy(np.concatenate([offs, offs[-1:]]).astype(np.int64)).to(DEV)
        d_merged = torch.zeros(total + 64, dtype=torch.int32, device=DEV)
        for j, (a, b) in enumerate(ranges):
            lo, hi = int(off[a]), int(off[b])
            clf.stream_load(j, h_rec + pair_sz * lo, hi - lo, h_off + 8 * a, a, b)
        for j in range(len(ranges)):
            clf.stream_use(j)
            clf.lookup_device(0, d_bases.data_ptr(), d_offs.data_ptr(), n, total, d_merged.data_ptr(), only_hits=1)
        clf.sync(0)
        clf.stream_check()
        clf.resolve_device(0, d_bases.data_ptr(), d_offs.data_ptr(), n, total, d_merged.data_ptr(), None)
        clf.sync(0)
        call = kdist.device_view(clf.device_result(0).d_call, n * 4, torch.int32, DEV).cpu().numpy().view(np.uint32)
        clf.finish()
        assert np.array_equal(call, calls)
        _same_counts(clf.counts(), wantc)
        _same_regs(clf, wantc)
    finally:
        L.kuq_host_free(h_rec)
        L.kuq_host_free(h_off)
        clf.close()


@pytest.mark.parametrize("k,nt,idx_type", [c for c in KEY_CASES if c[1] < 15])
def test_chunked_classify_on_crafted_bins(oracle, tmp_path, k, nt, idx_type):
    """`classify -x` with KUQ_FORCE_CHUNKS and a chunk size that the giant bin's range only just fits (the giant is
    the lowest bin, and at most 40 records of other bins fit beside it): the planner must cut right after it"""
    kdb, idx, reads, keys, queries, taxa, facts = _key_search_case(k, nt, idx_type, 100 + k + nt)
    bases, offs = synth.pack_reads(reads)
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*TAX.parent_map()), 500000, 1)
    calls, codes, code_off = run.classify(bases, offs)
    run.finish()
    ids = [f"r{i}" for i in range(len(reads))]
    with open(tmp_path / "reads.fa", "wb") as f:
        for rid, s in zip(ids, reads):
            f.write(b">" + rid.encode() + b"\n" + s + b"\n")
    kdb.tofile(tmp_path / "database.kdb")
    idx.tofile(tmp_path / "database.idx")
    TAX.write(str(tmp_path / "taxDB"))
    g, n_giant = facts["giant"][0], facts["giant"][1]
    budget = 3 * 8 + n_giant * 12 + 8 + 40 * 12           # the giant bin's range (plan_ranges' formula) + 40 records
    r = subprocess.run([build.build_classify(), "-d", "database.kdb", "-i", "database.idx", "-a", "taxDB", "-t", "1",
                        "-x", str(budget), "-o", "out.kraken", "reads.fa"], cwd=tmp_path, capture_output=True, text=True,
                       env=dict(os.environ, KUQ_FORCE_CHUNKS="1", KUQ_SPARSE_SLOTS=str(1 << 20)))
    assert r.returncode == 0, r.stderr[-2000:]
    n_chunks = int(r.stderr.split("Database split into ")[1].split()[0])
    assert n_chunks >= 2, r.stderr[:1500]
    assert open(tmp_path / "out.kraken").read() == util.kraken_lines(ids, reads, calls, codes, code_off)


# ==== hash tails ===================================================================================================
K = 31
DENSE_RANKS = (1, 13, 32, 33, 40, 52, 53)
EDGE_IDX = (0, 1, 4094, 4095)
ADD_RANKS = (1, 27, 28, 32, 39, 40)
CONV_RANK = 33


def _with_rank(rng, idx, rank, n=1):
    """n k-mers of register idx and dense rank `rank`; for ranks 52 / 53 (one hash per register) the nearest register
    at or after idx that has one"""
    for j in range(4096):
        km = crafted.kmers_with_hash(*crafted.dense_rank_mask((idx + j) % 4096, rank), K, n, rng)
        if len(km) == n:
            return km
    raise AssertionError(rank)


def _flagged(rng, top12, a, n=1):
    for j in range(4096):
        km = crafted.kmers_with_hash(*crafted.flagged_mask((top12 + j) % 4096, a), K, n, rng)
        if len(km) == n:
            return km
    raise AssertionError(a)


def _code_pair(rng, a, b, top12):
    """two k-mers whose flagged codes share the top 25 hash bits (register top12, bits 51..39 zero), with additional
    ranks a and b: one code when a == b"""
    x = crafted.kmers_with_hash(*crafted.flagged_mask(top12, a), K, 1, rng)
    y = crafted.kmers_with_hash(*crafted.flagged_mask(top12, b), K, 2, rng)
    return int(x[0]), int(y[y != x[0]][0])


def _tails_case(seed=7):
    """k-mers per taxon (in read order) covering the rank tails; returns (by_taxon, facts)"""
    rng = np.random.default_rng(seed)
    used = set()

    def fresh(km):
        km = [int(x) for x in km if int(x) not in used]
        used.update(km)
        return km

    tails, flagged = {}, {}
    for t, first in ((11, 0), (12, 7), (21, 100), (22, 2000)):
        km = []
        for r in DENSE_RANKS:
            for i in EDGE_IDX:
                km += fresh(_with_rank(rng, (i + first) % 4096 if r >= 52 else i, r))
        flagged[t] = fresh(np.concatenate([_flagged(rng, 5 + first, a) for a in ADD_RANKS]))
        km += flagged[t]
        km += fresh(_code_pair(rng, 6, 6, 9 + first))      # equal top 25 bits, equal additional rank: one code
        km += fresh(_code_pair(rng, 6, 7, 11 + first))     # equal top 25 bits, different rank: two codes
        tails[t] = km
    # members of genus 10 share flagged codes: 12 gets other k-mers with the codes of 11's flagged k-mers
    for x in flagged[11]:
        h = int(crafted.fmix64(np.array([x], np.uint64))[0])
        a = int(crafted.add_rank(np.array([h], np.uint64))[0])
        if a < 39:                                         # ranks 39 / 40 have a single hash per register
            y = crafted.kmers_with_hash(*crafted.flagged_mask(h >> 52, a), K, 3, rng)
            tails[12] += fresh([z for z in y if int(z) != x][:1])
    # 21: 1024 plain codes, then a flagged 1025th code of additional rank 33 (its unit converts on it: the fold reads a
    # rank field above 31), then the tails
    plain = rng.integers(0, 1 << 62, 8000, dtype=np.uint64)
    plain = synth.canonical(plain, K)
    plain = plain[(crafted.encode_hash32(crafted.fmix64(plain)) & np.uint32(1)) == 0]
    codes = crafted.encode_hash32(crafted.fmix64(plain))
    _, first_of = np.unique(codes, return_index=True)
    plain = fresh(plain[np.sort(first_of)][:3200])
    by_taxon = {11: tails[11], 12: tails[12], 21: plain[:1024] + fresh(_flagged(rng, 77, CONV_RANK)) + tails[21],
                22: plain[1024:3200] + tails[22]}
    facts = {"conv_code": by_taxon[21][1024]}
    return by_taxon, facts


def _tails_reads(by_taxon, order=None):
    return [crafted.kmer_read(x, K) for t in (order or by_taxon) for x in by_taxon[t]]


def _check_tail_shapes(by_taxon, facts):
    allk = np.array([x for v in by_taxon.values() for x in v], np.uint64)
    assert len(np.unique(allk)) == len(allk)
    h = crafted.fmix64(allk)
    ranks, idx = crafted.dense_rank(h), crafted.reg_index(h)
    code = crafted.encode_hash32(h)
    assert set(DENSE_RANKS) <= set(ranks.tolist())
    for r in DENSE_RANKS:
        if r < 52:
            assert set(EDGE_IDX) <= set(idx[ranks == r].tolist()), r
    flagged = (code & 1) == 1
    assert set(ADD_RANKS) <= set(crafted.add_rank(h[flagged]).tolist())
    assert (crafted.encoded_rank(code[flagged]) == ranks[flagged]).all()
    for t in (11, 12):                                     # a shared code and a top-25 pair with two ranks per taxon
        ht = crafted.fmix64(np.array(by_taxon[t], np.uint64))
        ct = crafted.encode_hash32(ht)
        f = ct[(ct & 1) == 1]
        assert len(np.unique(f)) < len(f)
        top = (ht >> _U(39))[(ct & 1) == 1]
        assert any(len(np.unique(f[top == x])) >= 2 for x in np.unique(top))
    c11 = set(crafted.encode_hash32(crafted.fmix64(np.array(by_taxon[11], np.uint64))).tolist())
    c12 = crafted.encode_hash32(crafted.fmix64(np.array(by_taxon[12], np.uint64)))
    assert sum(1 for c in c12.tolist() if c & 1 and c in c11) >= 3
    c21 = crafted.encode_hash32(crafted.fmix64(np.array(by_taxon[21], np.uint64)))
    assert len(np.unique(c21[:1024])) == 1024 and c21[1024] & 1 and c21[1024] not in set(c21[:1024].tolist())


def _tail_db(by_taxon):
    keys = np.concatenate([np.array(v, np.uint64) for v in by_taxon.values()])
    taxa = np.concatenate([np.full(len(v), t, np.uint32) for t, v in by_taxon.items()])
    return _db(keys, taxa, K, 8, 2)


def _sparse_keys(clf):
    n = clf.sparse_export()
    d = torch.zeros(max(n, 1), dtype=torch.int64, device=DEV)
    m = clf.sparse_export(d.data_ptr(), n)
    assert m == n
    keys = d[:n].cpu().numpy().view(np.uint64)
    dense = clf.dense_taxids()
    return {(int(dense[int(x >> _U(32)) - 1]), int(x & _U(0xFFFFFFFF))) for x in keys}


CLADES = [[11], [12], [21], [22], [11, 12], [21, 22], [11, 21], [11, 12, 21, 22]]


@pytest.mark.parametrize("mode", [binding.HLL_PRELOAD, binding.HLL_CHUNKED, binding.HLL_DENSE_ONLY])
def test_hash_tails(oracle, mode):
    by_taxon, facts = _tails_case()
    _check_tail_shapes(by_taxon, facts)
    kdb, idx = _tail_db(by_taxon)
    reads = _tails_reads(by_taxon)
    bases, offs = synth.pack_reads(reads)
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*TAX.parent_map()), 500000,
                     1 if mode == binding.HLL_CHUNKED else 0)
    calls, codes, code_off = run.classify(bases, offs)
    run.finish()
    want = run.counts(want_regs=True)
    sparse = dict(zip(want["taxid"].tolist(), want["sparse"].tolist()))
    if mode == binding.HLL_PRELOAD:
        assert sparse[11] and sparse[12] and not sparse[21] and not sparse[22]

    clf = binding.Classifier(max_reads=1 << 14, max_bases=1 << 20, hll_mode=mode, sparse_set_slots=1 << 12)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*TAX.parent_map())
    res = clf.classify(bases, offs, flags=binding.F_WANT_CODES)
    clf.finish()
    _same_reads(res, calls, codes, code_off, offs)
    got = clf.counts()
    _same_counts(got, want, dense_only=mode == binding.HLL_DENSE_ONLY)
    _same_regs(clf, want)
    regs = {int(t): want["regs"][j] for j, t in enumerate(want["taxid"])}
    conv = crafted.fmix64(np.array([facts["conv_code"]], np.uint64))
    assert regs[21][crafted.reg_index(conv)[0]] == 13 + CONV_RANK     # the converting code decides its register
    if mode == binding.HLL_DENSE_ONLY:
        for j, t in enumerate(want["taxid"]):
            assert int(got["unique"][j]) == oracle.ertl_dense(regs[int(t)], int(want["n_kmers"][j]))
        return

    # the sparse tier's keys: the codes of every counted window of the taxa that stayed sparse
    code_of = {t: crafted.encode_hash32(crafted.fmix64(np.array(v, np.uint64))) for t, v in by_taxon.items()}
    want_keys = {(t, int(c)) for t, c_t in code_of.items() if sparse[t] for c in c_t.tolist()}
    assert _sparse_keys(clf) == want_keys

    for mem in CLADES:
        r, nk, is_dense, hist = clf.clade_partial(mem)
        assert clf.clade(mem) == run.clade(mem), mem
        if any(not sparse[t] for t in mem):
            assert is_dense
            union = np.max([regs[t] for t in mem], axis=0)
            assert np.array_equal(hist, np.bincount(union, minlength=64)), mem
        else:
            assert not is_dense
            union = np.unique(np.concatenate([code_of[t] for t in mem]))
            want_hist = np.bincount(crafted.encoded_rank(union), minlength=64)
            assert want_hist[41:].sum() > 0 and want_hist[0] == 0
            assert np.array_equal(hist, want_hist), mem          # hist[0] stays 0: C[0] is derived from |S|
    r, k, u = clf.clade_counts_tree([10, 20, 1])
    for i, mem in enumerate([[10, 11, 12], [20, 21, 22], [1, 10, 11, 12, 20, 21, 22]]):
        assert (int(u[i]), int(r[i]), int(k[i])) == run.clade(mem), mem
    clf.close()


def test_hash_tails_merge_of_two_contexts(oracle):
    """kuq_merge_into of two contexts that each classified half of the reads (21's conversion in the first half)"""
    by_taxon, facts = _tails_case()
    kdb, idx = _tail_db(by_taxon)
    halves = [_tails_reads({t: v[:len(v) // 2] for t, v in by_taxon.items() if t != 21}) + _tails_reads(by_taxon, (21,)),
              _tails_reads({t: v[len(v) // 2:] for t, v in by_taxon.items() if t != 21})]
    both = halves[0] + halves[1]
    bases, offs = synth.pack_reads(both)
    unit = sum(len(s) for s in halves[0])                 # one work unit per context
    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*TAX.parent_map()), unit, 0)
    run.classify(bases, offs, want_codes=False)
    run.finish()
    want = run.counts(want_regs=True)
    ctx = []
    for part in halves:
        b, o = synth.pack_reads(part)
        c = binding.Classifier(max_reads=1 << 14, max_bases=1 << 20, hll_mode=binding.HLL_PRELOAD, sparse_set_slots=1 << 12)
        c.stage_db(kdb, idx)
        c.set_taxonomy(*TAX.parent_map())
        c.classify(b, o)
        c.finish()
        ctx.append(c)
    ctx[0].merge_from(ctx[1])
    _same_counts(ctx[0].counts(), want)
    _same_regs(ctx[0], want)
    for mem in CLADES:
        assert ctx[0].clade(mem) == run.clade(mem), mem
