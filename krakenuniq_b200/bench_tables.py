"""Times the end-of-run operations of the two device tables on one GPU, at about 10^8 keys and pairs:

  * export_replace: kuq_sparse_export_partitioned_alloc into 2 parts + kuq_sparse_replace with every key (the step a
    partitioned sparse-tier merge runs on each GPU; bench.py reaches it only with two or more GPUs);
  * sparse_grow / exact_grow: a table of 1024 slots that imports the items in 10 pieces, growing as it goes;
  * exact_partition: kuq_exact_partition over two contexts that hold half the pairs each.

Each figure is the time between CUDA events recorded around the call, with the device synchronised on both sides,
repeated --repeats times; the JSON line gives min / median / max in ms.  --lib times another build of
libkuq.so in this process, so that two builds can be compared in one session.

  python -m krakenuniq_b200.bench_tables [--n 100000000] [--repeats 5] [--lib path/to/libkuq.so]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from krakenuniq_b200 import binding, build, synth  # noqa: E402

DEV = "cuda:0"


def _db():
    rng = np.random.default_rng(0)
    tax = synth.make_taxonomy(16)
    genomes = synth.random_genomes(rng, 16, 2000)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, 31)
    kdb, idx = synth.build_db_images(km, tx, 31, 8, 2)
    return tax, kdb, idx


def _context(db, mode, slots):
    tax, kdb, idx = db
    clf = binding.Classifier(device=0, hll_mode=mode, sparse_set_slots=slots, max_reads=1 << 10, max_bases=1 << 16)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*tax.parent_map())
    clf.dense_taxids()                            # numbers the taxa and allocates the table
    return clf


def _timed(fn):
    """ms between two CUDA events recorded around the call, with the device synchronised before and after it (the
    library works on streams of its own and synchronises them before it returns)"""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    torch.cuda.synchronize()
    end.record()
    end.synchronize()
    return start.elapsed_time(end)


def _stats(ms):
    return {"min_ms": round(min(ms), 2), "median_ms": round(float(np.median(ms)), 2), "max_ms": round(max(ms), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000, help="keys of the sparse-tier set and pairs of the exact set")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--lib", default=None, help="the libkuq.so to time (default: the in-tree build)")
    a = ap.parse_args()
    if a.lib:
        build.LIB = os.path.abspath(a.lib)
    binding.load_library()
    db = _db()
    n_sketch = len(_context(db, binding.HLL_PRELOAD, 1 << 10).dense_taxids())
    g = torch.Generator(device=DEV).manual_seed(1)
    taxon = torch.randint(0, max(n_sketch // 2, 1), (a.n,), device=DEV, generator=g)       # sketch taxa have the low ids
    keys = ((taxon + 1) << 32) | torch.randint(1, 1 << 31, (a.n,), device=DEV, generator=g)
    pairs = torch.stack([torch.randint(1, 1 << 62, (a.n,), device=DEV, generator=g), taxon + 1], 1).contiguous()
    del taxon
    torch.cuda.synchronize()
    out = {"lib": build.LIB, "n": a.n, "gpu": torch.cuda.get_device_name(0)}

    big = _context(db, binding.HLL_PRELOAD, 1 << 10)
    big.sparse_import(keys.data_ptr(), a.n)
    n_keys = big.sparse_tier_info()["keys"]

    def export_replace():
        ptr, counts = big.sparse_export_partitioned_alloc(2)
        big.sparse_replace(ptr, int(counts.sum()))
        big.device_free(ptr)
    out["export_replace"] = _stats([_timed(export_replace) for _ in range(a.repeats)])
    assert big.sparse_tier_info()["keys"] == n_keys
    del big

    piece = a.n // 10
    for name, mode, items, imp in (("sparse_grow", binding.HLL_PRELOAD, keys, "sparse_import"),
                                   ("exact_grow", binding.HLL_EXACT, pairs, "exact_import")):
        ms = []
        for _ in range(a.repeats):
            c = _context(db, mode, 1 << 10)
            step = items.stride(0) * items.element_size()
            ms.append(_timed(lambda: [getattr(c, imp)(items.data_ptr() + i * piece * step, piece) for i in range(10)]))
            del c
        out[name] = _stats(ms)

    ms = []
    half = a.n // 2
    for _ in range(a.repeats):
        ctxs = [_context(db, binding.HLL_EXACT, 1 << 10) for _ in range(2)]
        for i, c in enumerate(ctxs):
            c.exact_import(pairs.data_ptr() + i * half * 16, half)
        ms.append(_timed(lambda: binding.Classifier.exact_partition(ctxs)))
        del ctxs
    out["exact_partition"] = _stats(ms)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
