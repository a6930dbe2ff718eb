"""world_size-2 gloo tests (CPU) of the multi-process host logic: read partitioning and the end-of-run merge of the
per-taxon state, checked against the oracle run over the whole input."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from krakenuniq_b200 import dist as kdist
from krakenuniq_b200 import synth

K = 31
MASK64 = (1 << 64) - 1


def _fmix64(x: np.ndarray) -> np.ndarray:
    x = x + np.uint64(1)
    x ^= x >> np.uint64(33); x *= np.uint64(0xff51afd7ed558ccd)
    x ^= x >> np.uint64(33); x *= np.uint64(0xc4ceb9fe1a85ec53)
    x ^= x >> np.uint64(33)
    return x


def _case():
    rng = np.random.default_rng(4)
    tax = synth.make_taxonomy(4)
    genomes = synth.random_genomes(rng, 4, 1500)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, K)
    kdb, idx = synth.build_db_images(km, tx, K, 7, 2)
    bases, offs = synth.sample_reads(rng, genomes, 400, 150, 0.01, 0.1, 0.2)
    return tax, kdb, idx, bases, offs


def _rank_state(oracle, tax, kdb, idx, bases, offs, lo, hi, taxa_all):
    """per-taxon state of reads [lo, hi) in the library's layout (rows = taxa_all): regs, n_kmers, n_reads, keys"""
    db = oracle.open_db(kdb, idx)
    pm = oracle.parent_map(*tax.parent_map())
    run = oracle.run(db, pm, 500000, 1)
    o = np.ascontiguousarray(offs[lo:hi + 1])
    calls, codes, code_off = run.classify(bases, o)
    run.finish()
    c = run.counts(want_regs=True)
    row = {int(t): i for i, t in enumerate(taxa_all)}
    regs = np.zeros((len(taxa_all), 4096), np.uint8)
    nk = np.zeros(len(taxa_all), np.int64)
    nr = np.zeros(len(taxa_all), np.int64)
    for j, t in enumerate(c["taxid"]):
        regs[row[int(t)]] = c["regs"][j]
        nk[row[int(t)]] = c["n_kmers"][j]
        nr[row[int(t)]] = c["n_reads"][j]
    # sparse keys (row+1) << 32 | encodeHashIn32Bit(fmix64(canon)) for every non-ambiguous window
    keys = set()
    for i in range(hi - lo):
        seq = bases[int(o[i]):int(o[i + 1])].tobytes()
        kmers, amb = oracle.scan(seq, K)
        w = codes[int(code_off[i]):int(code_off[i + 1])]
        for kmer, a, t in zip(kmers.tolist(), amb.tolist(), w.tolist()):
            if a:
                continue
            h = int(_fmix64(np.array([oracle.canonical(kmer, K)], np.uint64))[0])
            keys.add(((row[int(t)] + 1) << 32) | oracle.encode_hash32(h))
    return regs, nk, nr, np.array(sorted(keys), np.int64)


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle.oracle_py import Oracle
    oracle = Oracle()
    tax, kdb, idx, bases, offs = _case()
    taxa_all = sorted({0} | {r[0] for r in tax.rows})
    lo, hi = kdist.partition(len(offs) - 1, world, rank)
    regs, nk, nr, keys = _rank_state(oracle, tax, kdb, idx, bases, offs, lo, hi, taxa_all)
    t_regs, t_nk, t_nr = torch.from_numpy(regs.reshape(-1)), torch.from_numpy(nk), torch.from_numpy(nr)
    flag = torch.zeros(len(taxa_all), dtype=torch.uint8)
    flag[rank] = 1
    kdist.merge_state_tensors(t_regs, t_nk, t_nr, flag)
    others = kdist.gather_sparse_keys(torch.from_numpy(keys))
    union = np.union1d(keys, others.numpy())
    if rank == 0:
        q.put((t_regs.numpy().reshape(len(taxa_all), 4096).copy(), t_nk.numpy().copy(), t_nr.numpy().copy(),
               flag.numpy().copy(), union))
    dist.barrier()
    dist.destroy_process_group()


def test_partition_is_a_balanced_cover():
    for n in (0, 1, 7, 100, 1001):
        for world in (1, 2, 3, 8):
            parts = [kdist.partition(n, world, r) for r in range(world)]
            assert parts[0][0] == 0 and parts[-1][1] == n
            assert all(parts[i][1] == parts[i + 1][0] for i in range(world - 1))
            sizes = [b - a for a, b in parts]
            assert max(sizes) - min(sizes) <= 1


def test_two_rank_merge_equals_single_run(oracle):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    regs, nk, nr, flag, union = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    tax, kdb, idx, bases, offs = _case()
    taxa_all = sorted({0} | {r[0] for r in tax.rows})
    w_regs, w_nk, w_nr, w_keys = _rank_state(oracle, tax, kdb, idx, bases, offs, 0, len(offs) - 1, taxa_all)
    assert np.array_equal(regs, w_regs)
    assert np.array_equal(nk, w_nk) and np.array_equal(nr, w_nr)
    assert np.array_equal(union, w_keys)
    assert flag[:2].tolist() == [1, 1] and flag[2:].sum() == 0


def _exchange_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(100 + rank)
    # keys (taxon + 1) << 32 | code; the owner of a key is a function of its CODE only
    keys = ((rng.integers(1, 6, 5000, dtype=np.int64) << 32) | rng.integers(0, 3000, 5000, dtype=np.int64))
    keys = np.unique(keys)
    part = (keys & 0xFFFFFFFF) % world
    order = np.argsort(part, kind="stable")
    counts = np.bincount(part, minlength=world)
    got = kdist.exchange_partitioned_keys(torch.from_numpy(keys[order]), counts.tolist()).numpy()
    q.put((rank, keys, got))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 3, 8])
def test_in_process_group_runs_the_same_collectives(world):
    """tests.local_group (threads of one process) gives what the gloo ranks above give: reduced state, the other
    ranks' keys, and the all-to-all of code-partitioned keys"""
    from tests.local_group import run_ranks

    def rank(r, coll):
        rng = np.random.default_rng(200 + r)
        regs = torch.from_numpy(rng.integers(0, 40, 64, dtype=np.uint8))
        nk = torch.from_numpy(rng.integers(0, 1000, 8, dtype=np.int64))
        inputs = (regs.clone(), nk.clone())
        kdist.merge_state_tensors(regs, nk, nk.clone(), None, coll)
        keys = np.unique((rng.integers(1, 6, 300 + 50 * r, dtype=np.int64) << 32) | rng.integers(0, 3000, 300 + 50 * r))
        others = kdist.gather_sparse_keys(torch.from_numpy(keys), coll).numpy()
        part = (keys & 0xFFFFFFFF) % world
        order = np.argsort(part, kind="stable")
        got = kdist.exchange_partitioned_keys(torch.from_numpy(keys[order]), np.bincount(part, minlength=world).tolist(),
                                              coll).numpy()
        return inputs, regs, nk, keys, others, got

    res = run_ranks(world, rank)
    want_regs = torch.stack([x[0][0] for x in res]).max(0).values
    want_nk = torch.stack([x[0][1] for x in res]).sum(0)
    for r, (_, regs, nk, keys, others, got) in enumerate(res):
        assert torch.equal(regs, want_regs) and torch.equal(nk, want_nk)
        assert np.array_equal(np.sort(others), np.sort(np.concatenate([x[3] for j, x in enumerate(res) if j != r]
                                                                      + [np.zeros(0, np.int64)])))
        assert np.all((got & 0xFFFFFFFF) % world == r)
    assert np.array_equal(np.sort(np.concatenate([x[5] for x in res])), np.sort(np.concatenate([x[3] for x in res])))


def test_in_process_group_stops_every_rank_when_one_fails():
    from tests.local_group import run_ranks

    def rank(r, coll):
        if r == 1:
            raise ValueError("rank 1 failed")
        kdist.merge_state_tensors(torch.zeros(4, dtype=torch.uint8), torch.zeros(2, dtype=torch.int64),
                                  torch.zeros(2, dtype=torch.int64), None, coll)

    with pytest.raises(ValueError, match="rank 1 failed"):
        run_ranks(3, rank, timeout=60)


def test_partitioned_key_exchange_is_a_disjoint_cover():
    """the all-to-all of the code-partitioned sparse-tier keys: every key reaches exactly the rank that owns its code,
    so the union over ranks is the union of the inputs and no code lives on two ranks"""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    world = 2
    procs = [ctx.Process(target=_exchange_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in range(world)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    sent = np.unique(np.concatenate([r[1] for r in res]))
    for rank, _, got in res:
        assert np.all((got & 0xFFFFFFFF) % world == rank)
    assert np.array_equal(np.unique(np.concatenate([r[2] for r in res])), sent)
