"""Cost of building a database in minimizer-range passes: `db_sort` and `set_lcas` at the default budget (one pass on
an H100 for this size) and at budgets that force 2 / 4 / 8 passes, on the same inputs; one JSON line per run.

The inputs are bench_set_lcas.make_inputs' library (random genomes in mutated strains), its k-mer set from the drop-in
`kmer_set`, `db_sort -z -n 12` and build_db.sh's `set_lcas -x -T` line.  Every run must write the bytes of the default
run.  Reported: wall seconds (best of `--repeats`, the executable end to end), passes, library Gbp per second, and the
bytes each run copies host→device and device→host, computed from the shapes:
  - db_sort in one pass: the records in, the records and the index out; in passes: the records in three times
    (histogram, grouping, per-range sort), out twice (grouping, per-range sort) and the index out once;
  - set_lcas: the records staged once (twice with more than one range: the first staging collects the taxids of every
    range), the library once per range, the 12-byte records out once.
Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_db_build_ranges.py [--gbp 0.5]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import build  # noqa: E402
from krakenuniq_b200.bench_set_lcas import gpu_info, make_inputs  # noqa: E402

NT = 12
RESERVE = 1 << 18          # kuq_dbbuild.cu: budget kept back from the plan of the per-range sorts
PASS_C_REC = 64            # kuq_dbbuild.cu: planned device bytes per record of a range besides its two copies


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbp", type=float, default=0.5)
    ap.add_argument("--species", type=int, default=100)
    ap.add_argument("--strains", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    db_sort, set_lcas = build.build_dbtools()
    gpu = gpu_info()
    tmp = tempfile.mkdtemp(prefix="kuq_db_ranges_")
    try:
        n_bases, _ = make_inputs(tmp, a.gbp, a.species, a.strains, 0, a.seed)
        lib_bytes = os.path.getsize(os.path.join(tmp, "lib.fa"))

        def run(cmd, env=None):
            best, r = None, None
            for _ in range(a.repeats):
                t = time.perf_counter()
                r = subprocess.run(cmd, cwd=tmp, capture_output=True, text=True, env={**os.environ, **(env or {})})
                if r.returncode:
                    raise RuntimeError(f"{cmd[0]} failed: {r.stderr[-2000:]}")
                dt = time.perf_counter() - t
                best = dt if best is None else min(best, dt)
            return best, r.stderr

        subprocess.run([build.KMER_SET, "count", "-m", "31", "-s", "1G", "-C", "-t", "8", "-o", "database", "lib.fa"],
                       cwd=tmp, check=True, capture_output=True)
        sort_cmd = [db_sort, "-z", "-M", "-n", str(NT), "-d", "database_0", "-o", "database0.kdb", "-i", "database.idx"]
        wall, _ = run(sort_cmd)
        ref_kdb = open(os.path.join(tmp, "database0.kdb"), "rb").read()
        ref_idx = open(os.path.join(tmp, "database.idx"), "rb").read()
        off = np.frombuffer(ref_idx[8:], np.uint64)
        n, n_bins, pair = int(off[-1]), len(off) - 1, 12
        idx_bytes = 8 * (n_bins + 1)
        for target in (0, 2, 4, 8):
            env = {}
            if target:
                env["KUQ_DB_SORT_BUDGET"] = str(max(idx_bytes + RESERVE + (64 << 20),
                                                    RESERVE + (n * (2 * pair + PASS_C_REC) + 8 * n_bins) // target))
            wall, err = run(sort_cmd, env)
            passes = int(err.split("db_sort: ")[-2].split(" pass")[0]) if " pass" in err else -1
            same = (open(os.path.join(tmp, "database0.kdb"), "rb").read() == ref_kdb and
                    open(os.path.join(tmp, "database.idx"), "rb").read() == ref_idx)
            h2d = n * pair * (1 if passes == 1 else 3)
            d2h = n * pair * (1 if passes == 1 else 2) + idx_bytes
            print(json.dumps({"metric": "db_sort", "target_passes": target or "default", "passes": passes, "gpu": gpu,
                              "records": n, "gbp": round(n_bases / 1e9, 3), "wall_s": round(wall, 2),
                              "gbp_per_s": round(n_bases / 1e9 / wall, 3), "h2d_gb": round(h2d / 1e9, 3),
                              "d2h_gb": round(d2h / 1e9, 3), "same_bytes": same, **env}), flush=True)
        os.remove(os.path.join(tmp, "database_0"))
        shutil.copy(os.path.join(tmp, "database0.kdb"), os.path.join(tmp, "pristine.kdb"))
        lca_cmd = [set_lcas, "-x", "-d", "database0.kdb", "-o", "database.kdb", "-M", "-i", "database.idx", "-b", "taxDB",
                   "-t", "8", "-m", "seqid2taxid.map", "-c", "database.kdb.counts", "-F", "lib.fa", "-T"]
        ref = None
        for target in (0, 2, 4, 8):
            env = {}
            if target:
                env["KUQ_SET_LCAS_BUDGET"] = str((n * 12 + idx_bytes) // target + (1 << 20))
            wall, err = run(lca_cmd, env)
            ranges = int(err.split(" minimizer ranges")[0].rsplit(" ", 1)[1]) if "minimizer ranges" in err else 1
            out = (open(os.path.join(tmp, "database.kdb"), "rb").read(), open(os.path.join(tmp, "database.kdb.counts")).read())
            ref = ref or out
            h2d = n * pair * (1 if ranges == 1 else 2) + idx_bytes + ranges * n_bases
            print(json.dumps({"metric": "set_lcas", "target_passes": target or "default", "passes": ranges, "gpu": gpu,
                              "records": n, "gbp": round(n_bases / 1e9, 3), "library_bytes": lib_bytes,
                              "wall_s": round(wall, 2), "gbp_per_s": round(n_bases / 1e9 / wall, 3),
                              "h2d_gb": round(h2d / 1e9, 3), "d2h_gb": round(n * 12 / 1e9, 3), "same_bytes": out == ref,
                              **env}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
