"""S samples against one database: S separate `classify` runs against one `classify --sample-sheet` run.  JSON lines.

A separate run stages the database (contexts, pinned staging sets, the database files to every card, the dense-id remap
and the collision table, the taxonomy) before it classifies; a sheet run stages once and then pays, per sample, the
reset of the per-taxon state (kuq_reset_counts), the merge across GPUs and the report.  This script measures:
  * each separate run's wall time, its "processed in" time (the reads' pass) and the difference, its staging;
  * the sheet run's wall time, and per sample the reset_counts / merge / print_report lines of KUQ_TIMING;
  * md5 sums of every sample's Kraken output and report, both ways (they must be equal).
With --hbm-budget BYTES (KUQ_HBM_BUDGET) below the database's size the database streams through the GPU in ranges;
the sheet run then shares each pass over it among the samples, and its line gives the passes ("rounds") it made.
The database is synthetic and built on the GPU (synth_gpu, `--records` records, k = 31, nt = 15); the samples are
`--samples` FASTQ files of `--reads` 150 bp reads sampled from its genome with different seeds.  Run from the
repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_samples.py [--records 1e9] [--samples 8] [--reads 1000000] [--hbm-budget BYTES]
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

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import build, synth_gpu  # noqa: E402
from krakenuniq_b200.bench_multi_db import gpu_info  # noqa: E402


def write_sample(path, db, n_reads, read_len, seed, chunk=1 << 19):
    qual = b"I" * read_len
    with open(path, "wb") as f:
        for a in range(0, n_reads, chunk):
            c = min(chunk, n_reads - a)
            bases, _ = db.sample_reads(c, read_len=read_len, seed=seed * 1000 + a // chunk)
            rows = bases[:c * read_len].view(c, read_len).cpu().numpy()
            f.write(b"".join(b"@s%dr%d\n%s\n+\n%s\n" % (seed, a + i, rows[i].tobytes(), qual) for i in range(c)))
            del bases


def md5(path):
    h = hashlib.md5()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    return h.hexdigest()


def timings(stderr, label):
    return [float(m) for m in re.findall(r"\[timing\] %s\s+([0-9.]+) s" % re.escape(label), stderr)]


def processed(stderr):
    return [float(x) for x in re.findall(r"processed in ([0-9.]+)s", stderr.replace("\r", "\n"))]


def passes(stderr):
    """passes over a streamed database: its first range is looked up once per round (one database)"""
    return stderr.count("(database chunk 1 of")


def round_mib(stderr):
    m = re.findall(r"\[timing\] streamed: \d+ database\(s\), (\d+) MiB per round", stderr)
    return int(m[0]) if m else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=float, default=1e9)
    ap.add_argument("--samples", type=int, default=8)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--read-len", type=int, default=150)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--seed", type=int, default=9)
    ap.add_argument("--classify", default=None, help="executable to time (default: this build's)")
    ap.add_argument("--hbm-budget", type=int, default=None, help="KUQ_HBM_BUDGET: below the database's size it streams")
    a = ap.parse_args()
    exe = os.path.abspath(a.classify or build.build_classify())
    gpu = gpu_info()
    tmp = tempfile.mkdtemp(prefix="kuq_samples_")
    try:
        db = synth_gpu.GpuDatabase(int(a.records), n_genomes=2000, k=31, nt=15, idx_type=2, seed=a.seed, device="cuda:0")
        db.write_files(os.path.join(tmp, "db.kdb"), os.path.join(tmp, "db.idx"))
        db.write_taxdb(os.path.join(tmp, "taxDB"))
        key_ct = db.key_ct
        names = [f"s{i}" for i in range(a.samples)]
        for i, n in enumerate(names):
            write_sample(os.path.join(tmp, n + ".fq"), db, a.reads, a.read_len, a.seed + 1 + i)
        del db
        torch.cuda.empty_cache()
        common = [exe, "-d", "db.kdb", "-i", "db.idx", "-a", "taxDB", "-M", "-t", str(a.threads)]
        budget = {"KUQ_HBM_BUDGET": str(a.hbm_budget)} if a.hbm_budget else {}
        env = dict(os.environ, KUQ_TIMING="1", **budget)
        # one run first, not timed: it writes db.kdb.counts (every later run reads it) and warms the page cache
        subprocess.run(common + ["-o", "off", "-r", "warm.report", names[0] + ".fq"], cwd=tmp, capture_output=True, check=True,
                       env=dict(os.environ, **budget))
        base = {"gpu": gpu, "records": key_ct, "samples": a.samples, "reads_per_sample": a.reads, "read_len": a.read_len,
                "threads": a.threads, "classify": exe, "hbm_budget": a.hbm_budget}

        sep = {"wall_s": [], "processed_s": [], "staging_s": [], "passes": [], "md5": []}
        t_all = time.perf_counter()
        for n in names:
            t0 = time.perf_counter()
            r = subprocess.run(common + ["-o", f"sep.{n}.kraken", "-r", f"sep.{n}.report", n + ".fq"], cwd=tmp,
                               capture_output=True, text=True, env=env)
            wall = time.perf_counter() - t0
            if r.returncode:
                print(json.dumps(dict(base, mode="separate", error=r.stderr[-1500:])), flush=True)
                return 1
            p = processed(r.stderr)[-1]
            sep["wall_s"].append(round(wall, 3))
            sep["processed_s"].append(p)
            sep["staging_s"].append(round(wall - p, 3))
            sep["passes"].append(passes(r.stderr))
            sep["md5"].append([md5(os.path.join(tmp, f"sep.{n}.kraken")), md5(os.path.join(tmp, f"sep.{n}.report"))])
        sep_total = time.perf_counter() - t_all
        print(json.dumps(dict(base, mode="separate runs", total_wall_s=round(sep_total, 3), **sep)), flush=True)

        with open(os.path.join(tmp, "sheet.tsv"), "w") as f:
            f.write("name\tinput\toutput\treport\n")
            for n in names:
                f.write(f"{n}\t{n}.fq\tsheet.{n}.kraken\tsheet.{n}.report\n")
        t0 = time.perf_counter()
        r = subprocess.run(common + ["--sample-sheet", "sheet.tsv"], cwd=tmp, capture_output=True, text=True, env=env)
        wall = time.perf_counter() - t0
        if r.returncode:
            print(json.dumps(dict(base, mode="sheet", error=r.stderr[-1500:])), flush=True)
            return 1
        md5s = [[md5(os.path.join(tmp, f"sheet.{n}.kraken")), md5(os.path.join(tmp, f"sheet.{n}.report"))] for n in names]
        reset, report, merge = timings(r.stderr, "reset_counts"), timings(r.stderr, "print_report"), timings(r.stderr, "merge")
        per_sample = [round(x + y, 4) for x, y in zip([0.0] + reset, report)]
        rounds = re.findall(r"samples streamed in (\d+) rounds", r.stderr)       # streamed only (this build)
        print(json.dumps(dict(base, mode="sample sheet", total_wall_s=round(wall, 3), processed_s=processed(r.stderr),
                              rounds=int(rounds[0]) if rounds else None, passes=passes(r.stderr), round_mib=round_mib(r.stderr),
                              reset_counts_s=reset, merge_s=merge, print_report_s=report,
                              fixed_per_sample_s=per_sample, md5=md5s, md5_equal=md5s == sep["md5"])), flush=True)
        return 0 if md5s == sep["md5"] else 2
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    sys.exit(main())
