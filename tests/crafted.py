"""Crafted k-mers: k-mers chosen on the CPU so that a test reaches, on purpose, what random genomes reach with a
probability no test comes near — hashes with a wanted rank, register index or sparse code, and minimizer bins made of
keys that share their low 32-bit key word.

fmix64 (the reference's murmurhash3_finalizer, hyperloglogplus.cpp:830-838) is a bijection of 64-bit words: the xor
shift by 33 is its own inverse and both multipliers are odd, so a k-mer with a wanted hash h is fmix64_inv(h) - 1,
usable when it is below 4^k and canonical.  Every helper checks its own output against the oracle (hashes, codes,
bins, canonicity), so that a change here cannot silently hand a test something else than it claims."""
from __future__ import annotations

import numpy as np

from krakenuniq_b200 import synth

_U = np.uint64
_M1, _M2 = 0xff51afd7ed558ccd, 0xc4ceb9fe1a85ec53
_INV1, _INV2 = pow(_M1, -1, 1 << 64), pow(_M2, -1, 1 << 64)
HLL_P, HLL_PPRIME = 12, 25
_ORACLE = None


def oracle():
    global _ORACLE
    if _ORACLE is None:
        from oracle.oracle_py import Oracle
        _ORACLE = Oracle()
    return _ORACLE


def _xs33(x):
    return x ^ (x >> _U(33))


def fmix64(x):
    """the reference's fmix64 over an array (the key is incremented first)"""
    x = np.asarray(x, np.uint64) + _U(1)
    with np.errstate(over="ignore"):
        x = _xs33(x) * _U(_M1)
        x = _xs33(x) * _U(_M2)
    return _xs33(x)


def fmix64_inv(h):
    """the k-mer x with fmix64(x) == h, for every 64-bit h"""
    h = np.asarray(h, np.uint64)
    with np.errstate(over="ignore"):
        x = _xs33(h) * _U(_INV2)
        x = _xs33(x) * _U(_INV1)
        return _xs33(x) - _U(1)


def clz64(x):
    """leading zeros of 64-bit words (64 for 0)"""
    x = np.asarray(x, np.uint64).copy()
    n = np.zeros(x.shape, np.int64)
    for s in (32, 16, 8, 4, 2, 1):
        top = (x >> _U(64 - s)) == 0
        n += np.where(top, s, 0)
        x = np.where(top, x << _U(s), x)
    return n + (x == 0)


def reg_index(h):
    """getIndex(hash, 12): the register of a hash"""
    return (np.asarray(h, np.uint64) >> _U(64 - HLL_P)).astype(np.int64)


def dense_rank(h):
    """getRank(hash, 12), hyperloglogplus.cpp:140-147: 1..53"""
    return np.minimum(clz64(np.asarray(h, np.uint64) << _U(HLL_P)), 64 - HLL_P) + 1


def add_rank(h):
    """getRank(hash, 25): the additional rank a flagged code carries, 1..40"""
    return np.minimum(clz64(np.asarray(h, np.uint64) << _U(HLL_PPRIME)), 64 - HLL_PPRIME) + 1


def encode_hash32(h):
    """encodeHashIn32Bit(hash, 25, 12) over an array (checked against the oracle's)"""
    h = np.asarray(h, np.uint64)
    idx = ((h >> _U(64 - HLL_PPRIME)) << _U(32 - HLL_PPRIME)).astype(np.uint32)
    flagged = (idx << np.uint32(HLL_P)) == 0
    out = np.where(flagged, idx | (add_rank(h).astype(np.uint32) << np.uint32(1)) | np.uint32(1), idx)
    for i in _sample(len(h)):
        assert int(out[i]) == oracle().encode_hash32(int(h[i]))
    return out


def encoded_rank(code):
    """getEncodedRank(code, 25, 12), hyperloglogplus.cpp:152-161"""
    code = np.asarray(code, np.uint32)
    plain = clz64(code.astype(np.uint64) << _U(32 + HLL_P)) + 1
    plain = np.minimum(plain, 32 - HLL_P + 1)
    return np.where(code & 1, (HLL_PPRIME - HLL_P) + ((code >> 1) & 0x3F), plain).astype(np.int64)


def _sample(n, m=256):
    return np.unique(np.linspace(0, n - 1, min(n, m)).astype(np.int64)) if n else np.zeros(0, np.int64)


def is_canonical(x, k):
    x = np.asarray(x, np.uint64)
    return x == synth.canonical(x, k)


def _check_kmers(km, k):
    o = oracle()
    km = np.asarray(km, np.uint64)
    assert len(np.unique(km)) == len(km)
    assert (km < _U(1 << (2 * k))).all() and is_canonical(km, k).all()
    for i in _sample(len(km)).tolist():
        assert o.canonical(int(km[i]), k) == int(km[i])
        assert o.fmix64(int(km[i])) == int(fmix64(km[i:i + 1])[0])


def _deposit(values, mask):
    """scatter the low bits of `values` into the set bits of `mask` (a software pdep)"""
    out = np.zeros(len(values), np.uint64)
    j = 0
    for b in range(64):
        if (mask >> b) & 1:
            out |= ((values >> _U(j)) & _U(1)) << _U(b)
            j += 1
    return out


def kmers_with_hash(fixed_mask, fixed_bits, k, n, rng):
    """n distinct canonical k-mers (< 4^k) whose hash h has h & fixed_mask == fixed_bits, in random order; fewer when
    fewer exist (all candidates are enumerated when at most 2^20 hashes qualify)."""
    fixed_mask, fixed_bits = int(fixed_mask), int(fixed_bits) & int(fixed_mask)
    free = ~fixed_mask & ((1 << 64) - 1)
    n_free = bin(free).count("1")
    out, tries = np.zeros(0, np.uint64), 0
    if n_free <= 20:
        h = _deposit(np.arange(1 << n_free, dtype=np.uint64), free) | _U(fixed_bits)
        x = fmix64_inv(h)
        x = x[(x < _U(1 << (2 * k))) & is_canonical(x, k)]
        out = x[rng.permutation(len(x))[:n]]
    else:
        while len(out) < n:
            tries += 1
            assert tries < 1000, "too few k-mers with this hash pattern"
            h = (rng.integers(0, 1 << 64, 8 * n + 64, dtype=np.uint64, endpoint=False) & _U(free)) | _U(fixed_bits)
            x = fmix64_inv(h)
            x = x[(x < _U(1 << (2 * k))) & is_canonical(x, k)]
            out = np.concatenate([out, x])
            out = out[np.sort(np.unique(out, return_index=True)[1])]
        out = out[:n]
    _check_kmers(out, k)
    h = fmix64(out)
    assert ((h & _U(fixed_mask)) == _U(fixed_bits)).all()
    return out


def dense_rank_mask(idx, rank):
    """(mask, bits) of the hashes in register idx with getRank(hash, 12) == rank"""
    mask, bits = ((1 << HLL_P) - 1) << (64 - HLL_P), idx << (64 - HLL_P)
    zeros = min(rank - 1, 64 - HLL_P)                      # bits 51 .. 52 - zeros are 0, the next one is 1
    mask |= ((1 << zeros) - 1) << (64 - HLL_P - zeros)
    if rank <= 64 - HLL_P:
        mask |= 1 << (63 - HLL_P - zeros)
        bits |= 1 << (63 - HLL_P - zeros)
    return mask, bits


def flagged_mask(top12, a):
    """(mask, bits) of the hashes in register top12 whose code is flagged (hash bits 51..39 zero) with additional rank
    a (getRank(hash, 25) == a)"""
    return dense_rank_mask(top12, HLL_PPRIME - HLL_P + a)


# ---- minimizer bins ------------------------------------------------------------------------------------------------
def xor_mask(nt, idx_type):
    return (0 if idx_type == 1 else synth.INDEX2_XOR_MASK) & ((1 << (2 * nt)) - 1)


def lowest_bins(nt, idx_type, count, start=0):
    """the `count` smallest bins >= start that a k-mer can fall into (bin ^ xor must be a canonical nt-mer)"""
    out, b = [], start
    x = xor_mask(nt, idx_type)
    while len(out) < count:
        v = np.array([b ^ x], np.uint64)
        if is_canonical(v, nt)[0]:
            out.append(b)
        b += 1
    return out


def kmers_in_bin(k, nt, idx_type, b, n, rng, at_least=None):
    """n distinct canonical k-mers of minimizer bin b: the nt-mer of the bin planted at a random position, the other
    bases random.  Works for low bins (no other window may fall below b).  Returns fewer than n only when fewer than
    `at_least` (default n) were found."""
    m = b ^ xor_mask(nt, idx_type)
    assert is_canonical(np.array([m], np.uint64), nt)[0], f"bin {b} holds no k-mer"
    out = np.zeros(0, np.uint64)
    for _ in range(200):
        c = 4 * n + 256
        x = rng.integers(0, 1 << (2 * k), c, dtype=np.uint64)
        pos = rng.integers(0, k - nt + 1, c).astype(np.uint64) * _U(2)
        x = (x & ~(_U((1 << (2 * nt)) - 1) << pos)) | (_U(m) << pos)
        x = synth.canonical(x, k)
        x = x[synth.bin_key(x, k, nt, idx_type) == _U(b)]
        out = np.concatenate([out, x])
        out = out[np.sort(np.unique(out, return_index=True)[1])]
        if len(out) >= n:
            break
    assert len(out) >= (n if at_least is None else at_least), (b, len(out))
    out = out[:n]
    _check_kmers(out, k)
    _check_bins(out, k, nt, idx_type, b)
    return out


def _check_bins(km, k, nt, idx_type, b):
    assert (synth.bin_key(km, k, nt, idx_type) == _U(b)).all()
    for i in _sample(len(km), 64).tolist():
        assert oracle().bin_key(int(km[i]), k, nt, idx_type) == b


def kmers_sharing_low_word(k, nt, idx_type, b, rng, n_suffix_tries=200):
    """(low word, keys): every canonical k-mer of bin b that ends in one fixed 16-base suffix — the low 32 bits of the
    key — sorted.  The suffix holds the bin's nt-mer (nt <= 16) and ends in A, so that a prefix not starting with T
    keeps the k-mer canonical; the prefix (k - 16 bases, all 4^(k-16) of them up to k = 23, a sample beyond) varies the
    high word.  The suffix with the most such keys among n_suffix_tries is taken."""
    assert 16 <= k and nt <= 15
    m = b ^ xor_mask(nt, idx_type)
    pk = k - 16
    n_pre = 1 << (2 * pk)
    prefixes = np.arange(n_pre, dtype=np.uint64) if pk <= 7 else \
        np.unique(rng.integers(0, 1 << (2 * pk), 1 << 14, dtype=np.uint64))
    best = (None, np.zeros(0, np.uint64))
    for _ in range(n_suffix_tries):
        s = int(rng.integers(0, 1 << 32))
        pos = 2 * int(rng.integers(1, 16 - nt + 1))            # not in the last base, which stays A
        s = (s & ~(((1 << (2 * nt)) - 1) << pos)) & ~3 | (m << pos)
        x = (prefixes << _U(32)) | _U(s)
        x = x[is_canonical(x, k) & (synth.bin_key(x, k, nt, idx_type) == _U(b))]
        if len(x) > len(best[1]):
            best = (s, np.sort(x))
    s, keys = best
    assert s is not None and len(keys) >= 1
    assert ((keys & _U(0xFFFFFFFF)) == _U(s)).all()
    _check_kmers(keys, k)
    _check_bins(keys, k, nt, idx_type, b)
    return s, keys


def kmer_read(x, k, rc=False):
    """the bases of one k-mer (its reverse complement with rc)"""
    codes = (int(x) >> (2 * (k - 1 - np.arange(k)))) & 3
    if rc:
        codes = 3 - codes[::-1]
    return synth.decode(codes.astype(np.uint8)).tobytes()
