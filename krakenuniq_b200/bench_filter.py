"""Cost of the confidence filter (`classify --threshold T`, kuq_set_threshold): one JSON line per measurement.

1. `k_resolve` device time with and without a threshold, on the same batches: two contexts on one card, one of them
   filtering, fed the same batches in turn; kernel times from torch.profiler (CUDA activities), summed per context.
2. The CLI's wall time with and without `--threshold`, runs alternating, each writing its Kraken lines to a file.

The database is synthetic and built on the GPU (synth_gpu, `--records` records, k = 31, nt = 15, 2000 genomes under a
generated taxonomy); `--reads` reads of 150 bp are sampled from it (1 % substitutions, 20 % random reads).  The card's
name and power limit are read in the same run.  Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_filter.py [--records 1e8] [--reads 4000000] [--threshold 0.5]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import binding, build, synth, synth_gpu  # noqa: E402
from krakenuniq_b200.bench_multi_db import gpu_info  # noqa: E402


def resolve_times(tmp, threshold, batches, batch_reads):
    """k_resolve milliseconds of the same batches on a context without and one with a threshold"""
    kdb = np.fromfile(os.path.join(tmp, "db.kdb"), np.uint8)
    idx = np.fromfile(os.path.join(tmp, "db.idx"), np.uint8)
    tax = synth.Taxonomy.read(os.path.join(tmp, "taxDB"))
    rows = np.array([(r[0], r[1]) for r in tax.rows], np.uint32)
    ctxs = []
    for filt in (False, True):
        c = binding.Classifier(device=0, max_reads=batch_reads, max_bases=batch_reads * 160)
        c.stage_db(kdb, idx)
        c.set_taxonomy(*tax.parent_map())
        if filt:
            c.set_threshold(threshold, rows[:, 0], rows[:, 1])
        ctxs.append(c)
    offs = np.arange(batch_reads + 1, dtype=np.uint64) * 150
    for c in ctxs:                                               # warm-up: module loads, first-touch allocations
        c.classify(batches[0], offs)
    ms = [0.0, 0.0]
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for b in batches:
            for c in ctxs:
                c.classify(b, offs)
    for e in prof.events():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if "k_resolve<false, false>" in e.name or "k_resolveILb0ELb0E" in e.name:
            ms[0] += t / 1000.0
        elif "k_resolve<false, true>" in e.name or "k_resolveILb0ELb1E" in e.name:
            ms[1] += t / 1000.0
    for c in ctxs:
        c.close()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=float, default=1e8)
    ap.add_argument("--reads", type=int, default=4_000_000)
    ap.add_argument("--threshold", type=float, default=0.5)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--batch-reads", type=int, default=1 << 20)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    gpu = gpu_info()
    exe = build.build_classify()
    tmp = tempfile.mkdtemp(prefix="kuq_filter_")
    try:
        db = synth_gpu.GpuDatabase(int(a.records), n_genomes=2000, k=31, nt=15, idx_type=2, seed=a.seed, device="cuda:0")
        db.write_files(os.path.join(tmp, "db.kdb"), os.path.join(tmp, "db.idx"))
        db.write_taxdb(os.path.join(tmp, "taxDB"))
        key_ct = db.key_ct
        bases, _ = db.sample_reads(a.reads, read_len=150, seed=a.seed + 1)
        host = bases[:a.reads * 150].cpu().numpy()
        del bases, db
        torch.cuda.empty_cache()
        with open(os.path.join(tmp, "reads.fa"), "wb") as f:
            rows = host.reshape(-1, 150)
            for s in range(0, len(rows), 1 << 19):
                f.write(b"".join(b">r%d\n%s\n" % (s + i, r.tobytes()) for i, r in enumerate(rows[s:s + (1 << 19)])))
        n = a.batch_reads * 150
        batches = [np.ascontiguousarray(host[i * n:(i + 1) * n]) for i in range(min(a.batches, len(host) // n))]
        off, on = resolve_times(tmp, a.threshold, batches, a.batch_reads)
        print(json.dumps({"measure": "k_resolve device ms", "gpu": gpu, "records": key_ct,
                          "reads": len(batches) * a.batch_reads, "threshold": a.threshold,
                          "without": round(off, 3), "with": round(on, 3)}), flush=True)
        for rep in range(a.repeats):
            for tag, extra in (("without", []), ("with", ["--threshold", str(a.threshold)])):
                cmd = [exe, "-d", "db.kdb", "-i", "db.idx", "-a", "taxDB", "-M", "-t", str(a.threads), "-o",
                       f"{tag}.kraken", "-r", f"{tag}.report"] + extra + ["reads.fa"]
                t0 = time.time()
                r = subprocess.run(cmd, cwd=tmp, capture_output=True, text=True)
                wall = time.time() - t0
                if r.returncode:
                    print(json.dumps({"measure": "cli", "config": tag, "error": r.stderr[-1500:]}), flush=True)
                    continue
                line = [x for x in r.stderr.replace("\r", "\n").splitlines() if "processed in" in x][-1]
                secs = float(line.split("processed in ")[1].split("s")[0])
                print(json.dumps({"measure": "cli", "config": f"{tag} --threshold", "run": rep, "gpu": gpu,
                                  "records": key_ct, "reads": a.reads, "threads": a.threads, "wall_s": round(wall, 3),
                                  "processed_s": secs, "mreads_per_s": round(a.reads / 1e6 / secs, 3)}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
