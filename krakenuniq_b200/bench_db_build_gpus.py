"""Building a database over several GPUs: `db_sort` and `set_lcas` at a budget that cuts the database into `--ranges`
minimizer ranges, once for each `--devices` list (KUQ_DEVICES); one JSON line per tool and device list.

The inputs are bench_set_lcas.make_inputs' library (random genomes in mutated strains), its k-mer set from the drop-in
`kmer_set`, `db_sort -z -n 12` and build_db.sh's `set_lcas -x -T` line with `-c`.  Reported: wall seconds (best of
`--repeats`, the executable end to end), ranges, contexts (set_lcas) or devices (db_sort), whether set_lcas kept the
library's batches for a replay, the seconds set_lcas spent counting values for `.counts` on the devices, and the md5 of
every output file, which must be equal for every device list.  On a one-card machine `--devices 0,0` puts two workers on
one card: that measures what the layout costs, not what a second card gains.
Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_db_build_gpus.py --devices 0 --devices 0,0 [--devices 0,1] [--gbp 0.5]
"""
import argparse
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import build  # noqa: E402
from krakenuniq_b200.bench_set_lcas import gpu_info, make_inputs  # noqa: E402

NT = 12
RESERVE = 1 << 18          # kuq_dbbuild.cu: budget kept back from the plan of the per-range sorts
PASS_C_REC = 64            # kuq_dbbuild.cu: planned device bytes per record of a range besides its two copies
PLAN = re.compile(r"Database staged in (\d+) minimizer ranges over (\d+) contexts? \(batches kept: (yes|no)\)")


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--devices", action="append", default=[], help="a KUQ_DEVICES list; give it once per configuration")
    ap.add_argument("--ranges", type=int, default=2, help="minimizer ranges the budgets aim at")
    ap.add_argument("--gbp", type=float, default=0.5)
    ap.add_argument("--species", type=int, default=100)
    ap.add_argument("--strains", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    devices = a.devices or ["0", "0,0"]
    db_sort, set_lcas = build.build_dbtools()
    gpu = gpu_info()
    tmp = tempfile.mkdtemp(prefix="kuq_db_gpus_")
    try:
        n_bases, _ = make_inputs(tmp, a.gbp, a.species, a.strains, 0, a.seed)

        def run(cmd, env):
            best, r = None, None
            for _ in range(a.repeats):
                t = time.perf_counter()
                r = subprocess.run(cmd, cwd=tmp, capture_output=True, text=True, env={**os.environ, **env})
                if r.returncode:
                    raise RuntimeError(f"{cmd[0]} failed: {r.stderr[-2000:]}")
                dt = time.perf_counter() - t
                best = dt if best is None else min(best, dt)
            return best, r.stderr

        subprocess.run([build.KMER_SET, "count", "-m", "31", "-s", "1G", "-C", "-t", "8", "-o", "database", "lib.fa"],
                       cwd=tmp, check=True, capture_output=True)
        sort_cmd = [db_sort, "-z", "-M", "-n", str(NT), "-d", "database_0", "-o", "database0.kdb", "-i", "database.idx"]
        run(sort_cmd, {"KUQ_DEVICES": devices[0]})
        off = np.frombuffer(open(os.path.join(tmp, "database.idx"), "rb").read()[8:], np.uint64)
        n, n_bins, pair = int(off[-1]), len(off) - 1, 12
        idx_bytes = 8 * (n_bins + 1)
        sort_budget = max(idx_bytes + RESERVE + (64 << 20), RESERVE + (n * (2 * pair + PASS_C_REC) + 8 * n_bins) // a.ranges)
        lca_budget = (n * 12 + idx_bytes) // a.ranges + (1 << 20)
        for dl in devices:
            env = {"KUQ_DEVICES": dl, "KUQ_DB_SORT_BUDGET": str(sort_budget)}
            wall, err = run(sort_cmd, env)
            m = re.search(r"db_sort: (\d+) pass(?:es on (\d+) devices?)?", err)
            print(json.dumps({"metric": "db_sort", "devices": dl, "gpu": gpu, "records": n, "wall_s": round(wall, 2),
                              "passes": int(m.group(1)), "workers": int(m.group(2) or 1),
                              "md5": {f: md5(os.path.join(tmp, f)) for f in ("database0.kdb", "database.idx")},
                              "KUQ_DB_SORT_BUDGET": sort_budget}), flush=True)
        os.remove(os.path.join(tmp, "database_0"))
        shutil.copy(os.path.join(tmp, "database0.kdb"), os.path.join(tmp, "pristine.kdb"))
        lca_cmd = [set_lcas, "-x", "-d", "database0.kdb", "-o", "database.kdb", "-M", "-i", "database.idx", "-b", "taxDB",
                   "-t", "8", "-m", "seqid2taxid.map", "-c", "database.kdb.counts", "-F", "lib.fa", "-T"]
        for dl in devices:
            env = {"KUQ_DEVICES": dl, "KUQ_SET_LCAS_BUDGET": str(lca_budget), "KUQ_TIMING": "1"}
            wall, err = run(lca_cmd, env)
            m = PLAN.search(err)
            counts_s = re.search(r"\[timing\] value counts ([0-9.e-]+) s", err)
            print(json.dumps({"metric": "set_lcas", "devices": dl, "gpu": gpu, "records": n,
                              "gbp": round(n_bases / 1e9, 3), "wall_s": round(wall, 2),
                              "ranges": int(m.group(1)) if m else 1, "contexts": int(m.group(2)) if m else 1,
                              "batches_kept": m.group(3) if m else "no",
                              "counts_s": float(counts_s.group(1)) if counts_s else None,
                              "md5": {f: md5(os.path.join(tmp, f)) for f in ("database.kdb", "database.kdb.counts")},
                              "KUQ_SET_LCAS_BUDGET": lca_budget}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
