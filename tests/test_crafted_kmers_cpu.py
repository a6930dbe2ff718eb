"""The crafting helpers of tests/crafted.py, and the oracle at the tails they reach pinned to the unmodified reference
(its recorded answers, tests/ref_replay.py): the rank of every hash class 1..53, flagged codes of every additional rank
1..40, and the bin search over keys that share their low word, through the reference's stateful kmer_query."""
import numpy as np

from krakenuniq_b200 import synth
from tests import crafted

K = 31
_U = np.uint64


def test_fmix64_inverse_and_ranks(oracle):
    rng = np.random.default_rng(3)
    h = rng.integers(0, 1 << 64, 4000, dtype=np.uint64, endpoint=False)
    assert np.array_equal(crafted.fmix64(crafted.fmix64_inv(h)), h)
    x = crafted.fmix64_inv(h[:200])
    for xi, hi in zip(x.tolist(), h[:200].tolist()):
        assert oracle.fmix64(xi) == hi
    for r in (1, 13, 32, 33, 40, 52, 53):
        mask, bits = crafted.dense_rank_mask(4095, r)
        hh = (rng.integers(0, 1 << 64, 64, dtype=np.uint64, endpoint=False) & ~_U(mask)) | _U(bits)
        assert (crafted.dense_rank(hh) == r).all() and (crafted.reg_index(hh) == 4095).all()
    for a in (1, 27, 40):
        mask, bits = crafted.flagged_mask(0, a)
        hh = (rng.integers(0, 1 << 64, 64, dtype=np.uint64, endpoint=False) & ~_U(mask)) | _U(bits)
        code = crafted.encode_hash32(hh)
        assert (code & 1).all() and (crafted.add_rank(hh) == a).all()
        assert (crafted.encoded_rank(code) == 13 + a).all()


def test_crafted_bins_and_low_words():
    rng = np.random.default_rng(4)
    for k, nt, idx_type in ((31, 15, 2), (21, 7, 2), (17, 5, 2), (16, 5, 1)):
        bins = crafted.lowest_bins(nt, idx_type, 3)
        km = crafted.kmers_in_bin(k, nt, idx_type, bins[0], 500, rng)
        assert len(km) == 500
        lw, keys = crafted.kmers_sharing_low_word(k, nt, idx_type, bins[1], rng)
        assert len(keys) >= {31: 1000, 21: 500, 17: 3, 16: 1}[k]


def _rank_hashes(rng):
    """hashes covering every dense rank 1..53, register indexes 0 and 4095, every additional rank 1..40 (rest == 0
    included) and some random ones"""
    hs = []
    for r in range(1, 54):
        for idx in (0, 1, 4094, 4095):
            mask, bits = crafted.dense_rank_mask(idx, r)
            hs.append((rng.integers(0, 1 << 64, 3, dtype=np.uint64, endpoint=False) & ~_U(mask)) | _U(bits))
    hs.append(rng.integers(0, 1 << 64, 500, dtype=np.uint64, endpoint=False))
    return np.unique(np.concatenate(hs))


def test_encode_hash32_satisfies_the_reference_invariant(oracle, refshim):
    """hyperloglogplus.cpp:505-507 (the reference's debug check of the sparse encoding): the encoded code keeps the
    hash's register index and its rank, getEncodedRank(encode(h), 25, 12) == getRank(h, 12)"""
    h = _rank_hashes(np.random.default_rng(5))
    code = crafted.encode_hash32(h)
    ranks, flagged = crafted.dense_rank(h), (code & 1) == 1
    assert set(ranks.tolist()) == set(range(1, 54))
    assert set(crafted.add_rank(h[flagged]).tolist()) == set(range(1, 41))
    assert {0, 4095} <= set(crafted.reg_index(h).tolist())
    L = refshim.L
    for hi, c, r in zip(h.tolist(), code.tolist(), ranks.tolist()):
        assert oracle.encode_hash32(hi) == c
        assert L.kuref_get_rank64(hi, 12) == r
        assert L.kuref_get_encoded_rank(c, 25, 12) == r
        assert c >> 20 == hi >> 52
        if c & 1:
            assert L.kuref_get_rank64(hi, 25) == ((c >> 1) & 0x3F)


def test_query_on_shared_low_words_matches_reference(oracle, refshim):
    """the oracle's query against the reference's stateful kmer_query on a database of shared-low-word bins and a bin
    of about 20 k records; consecutive windows stay in one bin with misses between them (retry_on_failure,
    krakendb.cpp:304-319)"""
    rng = np.random.default_rng(6)
    nt, idx_type = 8, 2
    bins = crafted.lowest_bins(nt, idx_type, 5)
    big = np.sort(crafted.kmers_in_bin(K, nt, idx_type, bins[0], 20_000, rng))
    keys, probe = [big], [big[::37], big[::53] + _U(1)]
    for b, size in zip(bins[1:], (2, 8, 9, 40)):
        _, cand = crafted.kmers_sharing_low_word(K, nt, idx_type, b, rng)
        stored = np.sort(cand[1:-1][rng.choice(len(cand) - 2, size, replace=False)])
        keys.append(stored)
        probe += [stored, np.setdiff1d(cand, stored)[:40]]
    keys = np.concatenate(keys)
    taxa = rng.integers(1, 1000, len(keys)).astype(np.uint32)
    order = np.argsort(keys)
    kdb, idx = synth.build_db_images(keys[order], taxa[order], K, nt, idx_type)
    probe = np.concatenate(probe)
    # runs of one bin: hit, miss, hit ... (the retry path) and the same probes shuffled (bin changes)
    seq = np.concatenate([probe, probe[rng.permutation(len(probe))]])
    odb = oracle.open_db(kdb, idx)
    rdb = refshim.open_db(kdb, idx)
    want = np.array([odb.query(int(x))[1] for x in seq.tolist()], np.uint32)
    assert (want != 0).sum() > 1000 and (want == 0).sum() > 500
    assert np.array_equal(rdb.query_stateful(seq), want)
