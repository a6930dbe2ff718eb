"""Cost of spilling `classifyExact`'s exact k-mer set to host memory (KUQ_EXACT_HOST_BUDGET): one JSON line per run.

The workload is bench_exact.py's: a synthetic database of `--records` records (default 10^8, k = 31, nt = 15, built on
the GPU) and `--reads` reads of 150 bp (default 10^6).  One context on GPU 0 runs it:
  - uncapped: the table grows on the device as far as it needs;
  - with the table capped (KUQ_EXACT_MAX_SLOTS) so that the run spills about 2 and about 8 times, with a host budget.
    The caps are powers of two picked from the uncapped run's union of pairs, so the spill counts are approximate.
Each line reports the "processed in" time (the reads' pass, the spills and the settle step, without loading the
database; best of `--repeats`), the settle step's time, the spills, the bytes of pairs on the host when the run ended,
and the md5 of the Kraken output and of the report, which must be equal across the configurations.  The inputs are made
in a child process, so that this one holds no CUDA context while the executable runs.  Run from the repository root
after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_exact_spill.py [--records 1e8] [--reads 1000000] [--budget BYTES]
"""
import argparse
import hashlib
import json
import math
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import build  # noqa: E402
from krakenuniq_b200.bench_exact import parse  # noqa: E402
from krakenuniq_b200.bench_multi_db import gpu_info  # noqa: E402


def spill_stats(stderr):
    m = re.search(r"spilled to host memory (\d+) times \((\d+) pairs", stderr)
    s = re.search(r"\[timing\] exact set settled from host memory in ([\d.]+) s", stderr)
    return {"spills": int(m.group(1)) if m else 0, "host_bytes": int(m.group(2)) * 16 if m else 0,
            "settle_s": float(s.group(1)) if s else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=float, default=1e8)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=9)
    ap.add_argument("--genomes", type=int, default=2000)
    ap.add_argument("--budget", type=int, default=32 << 30, help="KUQ_EXACT_HOST_BUDGET of the capped runs (bytes)")
    a = ap.parse_args()
    exe = os.path.join(os.path.dirname(build.build_classify()), "classifyExact")
    gpu = gpu_info()
    tmp = tempfile.mkdtemp(prefix="kuq_exact_spill_")
    try:
        r = subprocess.run([sys.executable, os.path.join(ROOT, "krakenuniq_b200", "bench_exact.py"), "--make-inputs", tmp,
                            "--records", str(a.records), "--reads", str(a.reads), "--seed", str(a.seed), "--genomes", str(a.genomes)],
                           capture_output=True, text=True, check=True)
        key_ct, n_reads = json.loads(r.stdout.strip().splitlines()[-1])

        def run(name, env):
            best = None
            for _ in range(a.repeats):
                if os.path.exists(os.path.join(tmp, "out.report")):        # the executable appends to a report file
                    os.remove(os.path.join(tmp, "out.report"))
                cmd = [exe, "-d", "a.kdb", "-i", "a.idx", "-a", "taxDB", "-M", "-t", "8", "-o", "out.kraken", "-r", "out.report",
                       "reads.fq"]
                p = subprocess.run(cmd, cwd=tmp, capture_output=True, text=True, env=dict(os.environ, KUQ_TIMING="1", **env))
                if p.returncode:
                    print(json.dumps({"config": name, "gpu": gpu, "env": env, "error": p.stderr[-1500:]}), flush=True)
                    return None
                got = dict(parse(p.stderr), **spill_stats(p.stderr))
                if best is None or got["processed_s"] < best["processed_s"]:
                    best = got
            for f, key in (("out.kraken", "kraken_md5"), ("out.report", "report_md5")):
                with open(os.path.join(tmp, f), "rb") as fh:
                    best[key] = hashlib.md5(fh.read()).hexdigest()
            print(json.dumps(dict(config=name, gpu=gpu, reads=n_reads, records=key_ct, env=env,
                                  mreads_per_s=round(n_reads / 1e6 / best["processed_s"], 3), **best)), flush=True)
            return best

        base = run("uncapped", {"KUQ_DEVICE": "0"})
        if base is None or not base["exact_sets"]:
            return
        union = base["exact_sets"][0]["pairs"]
        # a spill empties a table at a load of about 0.8: s spills take a table of about union / (0.8 (s + 1)) pairs.
        # Batches of 2·10^4 reads, so that an empty capped table takes a batch's bound of one pair per window, and a
        # table of 2^20 slots to start (the default 2^26 would pass the smaller cap).
        for spills in (2, 8):
            cap = 1 << max(22, round(math.log2(union / (0.8 * (spills + 1)))))
            run(f"about {spills} spills: table capped at {cap} slots",
                {"KUQ_DEVICE": "0", "KUQ_EXACT_MAX_SLOTS": str(cap), "KUQ_BATCH_READS": "20000", "KUQ_SPARSE_SLOTS": str(1 << 20),
                 "KUQ_EXACT_HOST_BUDGET": str(a.budget)})
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
