"""Multi-process plumbing (one process per GPU, torch.distributed): how reads are partitioned over ranks and how the
per-taxon state is merged at the end of a run (SURVEY.md §8(e)).

The merge is the cross-process form of `taxon_counts[t] += my_taxon_counts[t]` (classify.cpp:542-544):
  counters add                         ReadCounts::operator+=     readcounts.hpp:76-88
  dense registers: element-wise max    HLL merge dense+dense       hyperloglogplus.cpp:614-620
  sparse tier: union of the code sets  HLL merge sparse+sparse     hyperloglogplus.cpp:600-603
  a taxon is dense if it is dense anywhere (sparse+dense → dense, :604-612)
Works on CPU tensors with gloo (tests) and on HBM tensors with NCCL over NVLink (bench / production).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist


class Collectives:
    """The collectives of this module, on a torch.distributed process group (`group`; None = the default group).
    Every function below takes `group=` and accepts either a torch.distributed group or an instance of a subclass of
    this class: a subclass can run the same merge over several contexts driven by threads of one process."""

    def __init__(self, group=None):
        self.group = group

    def rank(self) -> int:
        return dist.get_rank(self.group)

    def world_size(self) -> int:
        return dist.get_world_size(self.group)

    def all_reduce(self, t: torch.Tensor, op: str):
        """in place; op is 'max' or 'sum'"""
        dist.all_reduce(t, op={"max": dist.ReduceOp.MAX, "sum": dist.ReduceOp.SUM}[op], group=self.group)

    def all_gather(self, out: list, t: torch.Tensor):
        dist.all_gather(out, t, group=self.group)

    def all_to_all_single(self, out: torch.Tensor, t: torch.Tensor, out_splits=None, in_splits=None):
        dist.all_to_all_single(out, t, output_split_sizes=out_splits, input_split_sizes=in_splits, group=self.group)


def collectives(group=None) -> Collectives:
    return group if isinstance(group, Collectives) else Collectives(group)


def partition(n_items: int, world: int, rank: int):
    """contiguous, balanced [begin, end) of rank's share of n_items (reads of a file, bins of a database)"""
    base, rem = divmod(n_items, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def merge_state_tensors(regs: torch.Tensor, n_kmers: torch.Tensor, n_reads: torch.Tensor,
                        dense_flag: torch.Tensor | None = None, group=None):
    """in-place all-reduce of the per-taxon state"""
    c = collectives(group)
    c.all_reduce(regs, "max")
    c.all_reduce(n_kmers, "sum")
    c.all_reduce(n_reads, "sum")
    if dense_flag is not None:
        c.all_reduce(dense_flag, "max")


def gather_sparse_keys(keys: torch.Tensor, group=None) -> torch.Tensor:
    """all-gather variable-length int64 key arrays (0 = padding); returns the keys of all OTHER ranks"""
    c = collectives(group)
    world, rank = c.world_size(), c.rank()
    n = torch.tensor([keys.numel()], dtype=torch.int64, device=keys.device)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    c.all_gather(sizes, n)
    m = int(max(int(s.item()) for s in sizes))
    if m == 0:
        return keys.new_zeros(0)
    padded = keys.new_zeros(m)
    padded[:keys.numel()] = keys
    out = [keys.new_zeros(m) for _ in range(world)]
    c.all_gather(out, padded)
    return torch.cat([out[r][:int(sizes[r].item())] for r in range(world) if r != rank]) if world > 1 else keys.new_zeros(0)


def exchange_partitioned_keys(keys: torch.Tensor, counts, group=None, out: torch.Tensor | None = None) -> torch.Tensor:
    """One all-to-all of key segments: `keys` holds the segment for rank 0, 1, ... back to back (`counts[r]` keys for
    rank r); returns the keys every rank (this one included) sent to this rank.  O(keys / world) per rank."""
    c = collectives(group)
    world = c.world_size()
    send = torch.tensor([int(c) for c in counts], dtype=torch.int64, device=keys.device)
    recv = torch.empty_like(send)
    c.all_to_all_single(recv, send)
    recv_l = [int(x) for x in recv.tolist()]
    if out is not None and out.numel() >= sum(recv_l):
        out = out[:sum(recv_l)]
    else:
        out = keys.new_empty(sum(recv_l))
    c.all_to_all_single(out, keys[:int(send.sum())], recv_l, [int(x) for x in counts])
    assert len(recv_l) == world
    return out


def device_view(ptr: int, nbytes: int, dtype: torch.dtype, device):
    """torch view of library-owned device memory (for the collectives only)"""
    class _Holder:
        pass
    h = _Holder()
    itemsize = torch.empty(0, dtype=dtype).element_size()
    typestr = {torch.uint8: "|u1", torch.int64: "<i8", torch.int32: "<i4"}[dtype]
    h.__cuda_array_interface__ = {"shape": (int(nbytes // itemsize),), "typestr": typestr, "data": (int(ptr), False),
                                  "version": 3}
    return torch.as_tensor(h, device=device)


def merge_classifier_state(clf, device, group=None):
    """End-of-run merge of a `binding.Classifier`'s state across all ranks (replicas or database shards)."""
    sp = clf.state_ptrs()
    regs = device_view(sp.d_regs, sp.regs_bytes, torch.uint8, device)
    nk = device_view(sp.d_n_kmers, sp.n_sketch * 8, torch.int64, device)
    nr = device_view(sp.d_n_reads, sp.n_taxa * 8, torch.int64, device)
    flag = device_view(sp.d_dense_flag, sp.n_sketch, torch.uint8, device)
    merge_state_tensors(regs, nk, nr, flag, group)
    # the library works on its own streams: the reduced dense flags (which the export filters on) must have landed
    torch.cuda.synchronize()
    # sparse tier: union of the (taxon, code) sets of the taxa that are still sparse everywhere
    n = clf.sparse_export()
    keys = torch.zeros(max(n, 1), dtype=torch.int64, device=device)
    torch.cuda.synchronize()
    if n:
        n2 = clf.sparse_export(keys.data_ptr(), keys.numel())
        keys = keys[:n2]
    else:
        keys = keys[:0]
    others = gather_sparse_keys(keys, group)
    if others.numel():
        torch.cuda.synchronize()
        clf.sparse_import(others.data_ptr(), others.numel())
    torch.cuda.synchronize()


def merge_classifier_state_partitioned(clf, device, group=None, timings: dict | None = None, buffers=None):
    """End-of-run merge in O(state / world) per rank (replicas or database shards):
      1. all-reduce MAX of the dense flags FIRST, so that the harvest of the record flags skips taxa that are dense
         anywhere (their codes are never needed: sparse + dense → dense, hyperloglogplus.cpp:604-612);
      2. all-reduce MAX of the registers, SUM of the counters;
      3. sparse tier: keys (of the local set AND of the still-flagged records, which are not inserted locally first)
         grouped by the rank owning their code → one all-to-all → each rank dedups its slice
         (kuq_sparse_replace) → all-reduce SUM of the per-taxon rank histograms and distinct counts
         (kuq_set_sparse_summary).  Clade unions: `clade_counts_distributed`."""
    import time
    c = collectives(group)
    world = c.world_size()
    t0 = time.time()
    marks = []

    def mark(name):
        if timings is not None:
            torch.cuda.synchronize()
            marks.append((name, time.time()))

    sp = clf.state_ptrs()
    regs = device_view(sp.d_regs, sp.regs_bytes, torch.uint8, device)
    nk = device_view(sp.d_n_kmers, sp.n_sketch * 8, torch.int64, device)
    nr = device_view(sp.d_n_reads, sp.n_taxa * 8, torch.int64, device)
    flag = device_view(sp.d_dense_flag, sp.n_sketch, torch.uint8, device)
    c.all_reduce(flag, "max")
    torch.cuda.synchronize()
    merge_state_tensors(regs, nk, nr, None, c)
    mark("allreduce_state")
    # no local harvest: the keys of the flagged records go straight into the export buffer (kuq.h).
    # `buffers` = (export tensor, receive tensor), int64, allocated once by the caller: multi-GB cudaMallocs inside the
    # merge cost tens of ms and vary wildly when the card is nearly full
    kptr = None
    if buffers is not None:
        try:
            counts = clf.sparse_export_partitioned(world, buffers[0].data_ptr(), buffers[0].numel())
            keys = buffers[0]
        except Exception:                       # buffer too small: nothing was consumed yet, let the library allocate
            buffers = None
    if buffers is None:
        kptr, counts = clf.sparse_export_partitioned_alloc(world)
        keys = device_view(kptr, max(int(counts.sum()), 1) * 8, torch.int64, device)
    mark("export_partitioned")
    recv = exchange_partitioned_keys(keys, counts.tolist(), c, out=None if buffers is None else buffers[1])
    torch.cuda.synchronize()
    del keys
    if kptr is not None:
        clf.device_free(kptr)
    mark("all_to_all")
    clf.sparse_replace(recv.data_ptr() if recv.numel() else None, recv.numel())
    mark("replace_import")
    hist = torch.zeros(sp.n_sketch * 64, dtype=torch.int32, device=device)
    distinct = torch.zeros(sp.n_sketch, dtype=torch.int32, device=device)
    torch.cuda.synchronize()
    clf.sparse_summary(hist.data_ptr(), distinct.data_ptr())
    mark("summary")
    c.all_reduce(hist, "sum")
    c.all_reduce(distinct, "sum")
    torch.cuda.synchronize()
    clf.set_sparse_summary(hist.data_ptr(), distinct.data_ptr())
    mark("allreduce_summary")
    if timings is not None:
        timings["merge_wall_ms"] = (time.time() - t0) * 1e3
        timings["keys_exported"] = int(counts.sum())
        timings["keys_after_dedup"] = int(recv.numel())
        prev = t0
        for name, t in marks:
            timings[name + "_ms"] = (t - prev) * 1e3
            prev = t


def merge_exact_partitioned(clf, device, group=None):
    """End-of-run merge of exact k-mer sets (KUQ_HLL_EXACT) in O(pairs / world) per rank; no rank holds the union:
      1. all-reduce SUM of the counters;
      2. the (k-mer, taxon) pairs grouped by the rank owning their k-mer (kuq_exact_export_partitioned);
      3. one all-to-all of the pairs (two int64 words each);
      4. each rank rebuilds its table from what it received (kuq_exact_replace; duplicates collapse);
      5. all-reduce SUM of the per-taxon set sizes and roll-up books (kuq_exact_summary / kuq_set_exact_summary).
    Afterwards `counts()` and `clade_counts_tree()` report the union on every rank (until its next batch)."""
    c = collectives(group)
    world = c.world_size()
    sp = clf.state_ptrs()
    nk = device_view(sp.d_n_kmers, sp.n_sketch * 8, torch.int64, device)
    nr = device_view(sp.d_n_reads, sp.n_taxa * 8, torch.int64, device)
    c.all_reduce(nk, "sum")
    c.all_reduce(nr, "sum")
    torch.cuda.synchronize()
    ptr, counts = clf.exact_export_partitioned_alloc(world)
    n = int(counts.sum())
    pairs = device_view(ptr, max(n, 1) * 16, torch.int64, device)[:2 * n]
    recv = exchange_partitioned_keys(pairs, [2 * int(x) for x in counts], c)
    torch.cuda.synchronize()
    del pairs
    clf.device_free(ptr)
    recv = recv.contiguous()
    clf.exact_replace(recv.data_ptr() if recv.numel() else None, recv.numel() // 2)
    del recv
    count = torch.zeros(sp.n_sketch, dtype=torch.int64, device=device)
    books = torch.zeros(sp.n_taxa, dtype=torch.int64, device=device)
    torch.cuda.synchronize()
    clf.exact_summary(count.data_ptr(), books.data_ptr())
    c.all_reduce(count, "sum")
    c.all_reduce(books, "sum")
    torch.cuda.synchronize()
    clf.set_exact_summary(count.data_ptr(), books.data_ptr())


def clade_counts_distributed(clf, clades, device, group=None):
    """(unique, reads, kmers) per clade (list of taxid lists) after merge_classifier_state_partitioned: the union
    histograms of the code partitions add up; one all-reduce for all clades."""
    from . import binding
    coll = collectives(group)
    parts = [clf.clade_partial(c) for c in clades]
    hist = torch.tensor(np.stack([p[3] for p in parts]).astype(np.int64) if parts else np.zeros((0, 64), np.int64), device=device)
    dense = [p[2] for p in parts]
    # dense clades: every rank holds the all-reduced registers, so its histogram is already the global one
    for i, d in enumerate(dense):
        if d and coll.rank() != 0:
            hist[i] = 0
    coll.all_reduce(hist, "sum")
    h = hist.cpu().numpy().astype(np.uint32)
    out = []
    for i, (r, k, d, _) in enumerate(parts):
        u = 0
        if k:
            u = binding.ertl_dense_hist(h[i], k) if d else binding.ertl_sparse(h[i], k)
        out.append((u, r, k))
    return out
