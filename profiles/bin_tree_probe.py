#!/usr/bin/env python
"""Go / no-go measurement for laying out every minimizer bin as a two-level search tree (kuq_layout_experiment
variants 13-15), on the bench's configs[1] database and reads.

1. The split of the fused k_lookup: bench-shaped context (preload HLL rule, work units), stage times of batches with
   counting (HLL registers, record flags) and of batches with KUQ_F_NO_COUNTS, alternated.
2. The layout experiment on one batch's windows: every variant timed and checked window by window against the
   product's ids, with the windows_by_bin_size histogram.
usage: python profiles/bin_tree_probe.py [out.json]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from krakenuniq_b200 import binding, synth_gpu  # noqa: E402

B, L, RECORDS = 1_000_000, 150, 666_000_000
dev = "cuda:0"
out = {}
try:
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                capture_output=True, text=True, timeout=60).stdout.strip()
except Exception as e:  # noqa: BLE001
    out["gpu"] = f"{torch.cuda.get_device_name(0)} (nvidia-smi: {e})"
print("gpu:", out["gpu"], flush=True)

t0 = time.time()
db = synth_gpu.GpuDatabase(RECORDS, n_genomes=2000, k=31, nt=15, seed=2, device=dev, passes=1)
n_batches = 16
pool, _ = db.sample_reads(n_batches * B, L, seed=3)
torch.cuda.synchronize()
out["gen_s"] = round(time.time() - t0, 1)
torch.cuda.empty_cache()
d_off = torch.arange(B + 2, dtype=torch.int64, device=dev) * L


def batch(i):
    return pool.data_ptr() + (i % n_batches) * B * L


# ---- 1. fused k_lookup with and without counting, bench-shaped context ----------------------------------------------
per_unit = -(-500000 // L)
units_per_batch = -(-B // per_unit)
unit_local = (torch.arange(B, dtype=torch.int64, device=dev) // per_unit).to(torch.int32)
clf = binding.Classifier(device=0, n_slots=1, max_reads=B, max_bases=B * L + 4096, hll_mode=0, sparse_set_slots=1 << 31)
clf.attach_db_device(db.records.data_ptr(), db.key_ct, db.offsets.data_ptr(), 31, 15, 2)
clf.set_taxonomy(*db.parent_map())
keep = []
stages = {"counting": [], "no_counts": []}
for step in range(3 + 12):
    u = unit_local + step * units_per_batch
    keep.append(u)
    mode = "counting" if step < 3 or step % 2 else "no_counts"
    clf.classify_device(0, batch(step), d_off.data_ptr(), B, B * L, u.data_ptr(),
                        flags=binding.F_NO_COUNTS if mode == "no_counts" else 0)
    clf.sync(0)
    if step >= 3:
        stages[mode].append(clf.last_stage_ms(0))
clf.finish()
clf.close()
del clf, keep
torch.cuda.empty_cache()
out["fused_split_ms"] = {m: {"k_scan": float(np.mean([s[0] for s in v])), "k_lookup": float(np.mean([s[1] for s in v])),
                             "k_lookup_min": float(np.min([s[1] for s in v])), "k_lookup_max": float(np.max([s[1] for s in v])),
                             "k_resolve": float(np.mean([s[2] for s in v])), "batches": len(v)}
                         for m, v in stages.items()}
print(json.dumps(out["fused_split_ms"]), flush=True)

# ---- 2. layout experiment ---------------------------------------------------------------------------------------------
clf = binding.Classifier(device=0, n_slots=1, max_reads=B, max_bases=B * L + 4096, hll_mode=2)
clf.attach_db_device(db.records.data_ptr(), db.key_ct, db.offsets.data_ptr(), 31, 15, 2)
clf.set_taxonomy(*db.parent_map())
for s in range(2):                                          # batch 0 = warm-up, batch 1 = the measured windows
    clf.classify_device(0, batch(s), d_off.data_ptr(), B, B * L, None, flags=binding.F_NO_COUNTS)
    clf.sync(0)
res = clf.layout_experiment(0, B * L, reps=10)
clf.close()
out["layout"] = res
base = res["variants"][0]["best_ms"]
for v in res["variants"]:
    print(f"  {v['record_bytes']:2d} B records, {v['arity']:2d}-ary, scan <= {v['scan_window']:2d}, {v['shape']:46s}: "
          f"best {v['best_ms']:.3f} ms  mean {v['mean_ms']:.3f} ms  x{base / v['best_ms']:.2f}  mismatches {v['mismatches']}",
          flush=True)
print("windows_by_bin_size:", res["windows_by_bin_size"], " tree copy ms:", res["tree_ms"],
      " unordered bins:", res["tree_unordered_bins"], flush=True)
if len(sys.argv) > 1:
    os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
    with open(sys.argv[1], "w") as f:
        json.dump(out, f, indent=1)
