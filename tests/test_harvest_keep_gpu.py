"""The record-tier harvest (kuq_finish on a resident range) on records with crafted flags, against a NumPy model of
the harvest: flagged secondaries hand their flag to their primaries, then every flagged record that is neither kept
nor of a dense taxon becomes kept and counts one distinct code of its taxon, and every flag is cleared.

The harvest streams the records in 16-byte-aligned groups of four and treats the records before the first aligned one
and after the last whole group one by one, so the ranges here start at every 4-byte offset and hold 1, 2, 3 and more
records.  Every byte of the buffer (records, and guard bytes on both sides) is compared, together with the per-taxon
counts and the number of records that became kept."""
import numpy as np
import pytest

from krakenuniq_b200 import binding

pytestmark = pytest.mark.gpu
SEEN, KEPT = np.uint32(0x80000000), np.uint32(0x40000000)
GUARD = 64


def model(words, sec, dense, distinct):
    """the harvest on a copy: (words, distinct, n_kept)"""
    w, d = words.copy(), distinct.copy()
    hi = w[:, 1]
    if len(sec):
        m = (hi[sec[:, 0]] & SEEN) != 0
        hi[sec[m, 0]] &= ~SEEN
        hi[sec[m, 1]] |= SEEN
    seen, kept = (hi & SEEN) != 0, (hi & KEPT) != 0
    new = seen & ~kept & (dense[w[:, 2]] == 0)
    hi[seen] &= ~SEEN
    hi[new] |= KEPT
    d += np.bincount(w[:, 2][new], minlength=len(d)).astype(np.uint32)
    return w, d, int(new.sum())


def records(rng, n, n_sketch):
    w = np.empty((n, 3), np.uint32)
    w[:, 0] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    w[:, 1] = rng.integers(0, 1 << 30, n, dtype=np.uint64).astype(np.uint32)     # key bits 32..61, no flags
    w[:, 2] = rng.integers(0, n_sketch, n, dtype=np.uint64).astype(np.uint32)
    return w


def run(words, sec, dense, distinct, offset, rng):
    """the library's harvest on a device copy of `words` placed `offset` bytes past a 16-byte boundary"""
    import torch
    n = len(words)
    guard = rng.integers(0, 256, GUARD + offset + 12 * n + GUARD, dtype=np.uint8)
    buf = guard.copy()
    buf[GUARD + offset:GUARD + offset + 12 * n] = words.view(np.uint8).ravel()
    d_buf = torch.from_numpy(buf).cuda()
    assert d_buf.data_ptr() % 16 == 0
    d_sec = torch.from_numpy(np.ascontiguousarray(sec, np.uint32).view(np.int32)).cuda() if len(sec) else None
    d_dense = torch.from_numpy(dense).cuda()
    d_distinct = torch.from_numpy(distinct.view(np.int32)).cuda()
    d_kept = torch.zeros(1, dtype=torch.int64, device="cuda")
    binding.harvest_keep_device(d_buf.data_ptr() + GUARD + offset, n, d_sec.data_ptr() if d_sec is not None else None,
                                len(sec), d_dense.data_ptr(), len(dense), d_distinct.data_ptr(), d_kept.data_ptr())
    out = d_buf.cpu().numpy()
    want_w, want_d, want_k = model(words, sec, dense, distinct)
    want = guard.copy()
    want[GUARD + offset:GUARD + offset + 12 * n] = want_w.view(np.uint8).ravel()
    assert np.array_equal(out, want), f"record bytes differ at {np.flatnonzero(out != want)[:8]}"
    assert np.array_equal(d_distinct.cpu().numpy().view(np.uint32), want_d)
    assert int(d_kept.item()) == want_k
    return want_k


def collision_list(rng, n, n_pairs):
    """(secondary, primary) pairs: disjoint sets of records, each secondary listed once"""
    idx = rng.permutation(n)[:2 * n_pairs].astype(np.uint32)
    return idx.reshape(n_pairs, 2)


@pytest.mark.parametrize("offset", [0, 4, 8, 12])
def test_every_record_flagged(offset):
    rng = np.random.default_rng(1 + offset)
    n, n_sketch = 200_003, 3000
    w = records(rng, n, n_sketch)
    w[:, 1] |= SEEN
    w[rng.random(n) < 0.3, 1] |= KEPT
    dense = (rng.random(n_sketch) < 0.2).astype(np.uint8)
    sec = collision_list(rng, n, 5000)
    distinct = rng.integers(0, 100, n_sketch, dtype=np.uint64).astype(np.uint32)
    assert run(w, sec, dense, distinct, offset, rng) > 0


@pytest.mark.parametrize("offset", [0, 4, 8, 12])
def test_no_record_flagged(offset):
    rng = np.random.default_rng(10 + offset)
    n, n_sketch = 100_001, 500
    w = records(rng, n, n_sketch)
    w[rng.random(n) < 0.5, 1] |= KEPT
    assert run(w, collision_list(rng, n, 1000), np.zeros(n_sketch, np.uint8), np.zeros(n_sketch, np.uint32), offset, rng) == 0


@pytest.mark.parametrize("offset", [0, 4, 8, 12])
def test_only_secondaries_flagged(offset):
    rng = np.random.default_rng(20 + offset)
    n, n_sketch = 150_002, 800
    w = records(rng, n, n_sketch)
    sec = collision_list(rng, n, 20_000)
    w[sec[:, 0], 1] |= SEEN
    w[sec[::3, 1], 1] |= KEPT                                  # a third of the primaries hold the key already
    dense = (rng.random(n_sketch) < 0.1).astype(np.uint8)
    assert run(w, sec, dense, np.zeros(n_sketch, np.uint32), offset, rng) > 0


@pytest.mark.parametrize("offset", [0, 4, 8, 12])
def test_only_dense_taxa_flagged(offset):
    rng = np.random.default_rng(30 + offset)
    n, n_sketch = 120_001, 1000
    w = records(rng, n, n_sketch)
    dense = (rng.random(n_sketch) < 0.3).astype(np.uint8)
    w[dense[w[:, 2]] != 0, 1] |= SEEN
    assert run(w, np.zeros((0, 2), np.uint32), dense, np.ones(n_sketch, np.uint32), offset, rng) == 0


@pytest.mark.parametrize("offset", [0, 4, 8, 12])
@pytest.mark.parametrize("n", [5, 8, 1001, 65_539])
def test_first_and_last_record(offset, n):
    rng = np.random.default_rng(40 + offset + n)
    n_sketch = 64
    w = records(rng, n, n_sketch)
    w[[0, n - 1], 1] |= SEEN
    assert run(w, np.zeros((0, 2), np.uint32), np.zeros(n_sketch, np.uint8), np.zeros(n_sketch, np.uint32), offset, rng) == 2


@pytest.mark.parametrize("offset", [0, 4, 8, 12])
@pytest.mark.parametrize("n", [1, 2, 3])
def test_tiny_databases(offset, n):
    rng = np.random.default_rng(50 + offset + n)
    n_sketch = 4
    for flags in range(1 << n):                              # every subset of flagged records, one of them kept
        w = records(rng, n, n_sketch)
        for r in range(n):
            if flags >> r & 1:
                w[r, 1] |= SEEN
        w[n - 1, 1] |= KEPT if flags == 1 << (n - 1) else 0
        sec = np.array([[0, n - 1]], np.uint32) if n > 1 else np.zeros((0, 2), np.uint32)
        run(w, sec, np.array([0, 1, 0, 0], np.uint8), np.zeros(n_sketch, np.uint32), offset, rng)


@pytest.mark.parametrize("n_sketch", [16_384, 50_000])
def test_many_taxa(n_sketch):
    """the largest taxonomy whose per-taxon counters fit a block's shared memory, and one past it (hashed table)"""
    rng = np.random.default_rng(60)
    n = 3_000_001
    w = records(rng, n, n_sketch)
    w[rng.random(n) < 0.6, 1] |= SEEN
    w[rng.random(n) < 0.1, 1] |= KEPT
    dense = (rng.random(n_sketch) < 0.05).astype(np.uint8)
    sec = collision_list(rng, n, 100_000)
    assert run(w, sec, dense, np.zeros(n_sketch, np.uint32), 4, rng) > 0
