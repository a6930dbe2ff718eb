"""The collectives of krakenuniq_b200.dist for N threads of one process: N classification contexts on one device
run the same end-of-run merges as N processes on N GPUs.

Every collective puts this rank's contribution (a host copy) into a shared slot table, meets the other ranks at a
barrier, computes its result from all slots and meets them again before the table is reused.  The barrier has a
timeout, and `run_ranks` aborts it as soon as one rank raises, so a failing rank never leaves the others waiting."""
import threading

import torch

from krakenuniq_b200 import dist as kdist


class LocalGroup:
    def __init__(self, world: int, timeout: float = 120.0):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=timeout)
        self.slots = [None] * world

    def rank(self, r: int) -> "LocalRank":
        return LocalRank(self, r)


class LocalRank(kdist.Collectives):
    def __init__(self, group: LocalGroup, r: int):
        super().__init__(None)
        self.g, self.r = group, r

    def rank(self):
        return self.r

    def world_size(self):
        return self.g.world

    def _exchange(self, value):
        """every rank's `value`, in rank order"""
        self.g.slots[self.r] = value
        self.g.barrier.wait()
        out = list(self.g.slots)
        self.g.barrier.wait()
        return out

    @staticmethod
    def _store(dst: torch.Tensor, src: torch.Tensor):
        dst.copy_(src.to(dst.device))
        if dst.is_cuda:
            torch.cuda.synchronize(dst.device)

    def all_reduce(self, t, op):
        vals = self._exchange(t.detach().cpu().clone())
        f = {"max": torch.maximum, "sum": torch.add}[op]
        acc = vals[0].clone()
        for v in vals[1:]:
            acc = f(acc, v)
        self._store(t, acc)

    def all_gather(self, out, t):
        vals = self._exchange(t.detach().cpu().clone())
        for o, v in zip(out, vals):
            self._store(o, v)

    def all_to_all_single(self, out, t, out_splits=None, in_splits=None):
        w = self.g.world
        if in_splits is None:
            in_splits = [t.numel() // w] * w
        chunks = list(torch.split(t.detach().cpu().clone(), [int(x) for x in in_splits]))
        vals = self._exchange(chunks)
        got = [vals[src][self.r] for src in range(w)]
        if out_splits is not None:
            assert [g.numel() for g in got] == [int(x) for x in out_splits], "split sizes disagree between ranks"
        self._store(out, torch.cat(got) if got else out.new_zeros(0).cpu())


def run_ranks(world: int, fn, timeout: float = 300.0):
    """fn(rank, collectives) on `world` threads; returns the list of results, re-raises the first rank's error"""
    g = LocalGroup(world)
    results, errors = [None] * world, [None] * world

    def body(r):
        try:
            results[r] = fn(r, g.rank(r))
        except BaseException as e:          # noqa: BLE001 - handed to the caller below
            errors[r] = e
            g.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout)
    if any(t.is_alive() for t in threads):
        g.barrier.abort()
        raise TimeoutError(f"a rank of {world} did not finish within {timeout} s")
    real = [e for e in errors if e is not None and not isinstance(e, threading.BrokenBarrierError)]
    if real:
        raise real[0]
    if any(e is not None for e in errors):
        raise next(e for e in errors if e is not None)
    return results
