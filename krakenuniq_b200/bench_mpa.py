"""Cost of writing the MetaPhlAn-style table and the read lineages while classifying (`classify --mpa-report`,
`--translate-out`): one JSON line per measurement.

1. The CLI's "processed in" time without the new options, with --mpa-report, with --translate-out (plain and with
   --translate-mpa-format) and with both, runs alternating.
2. An 8-sample --sample-sheet with one --mpa-report table against the same sheet without it: the sum of the samples'
   "processed in" times and the wall time of the whole process (which includes writing the table).

The database is synthetic and built on the GPU (synth_gpu, `--records` records, k = 31, nt = 15, 2000 genomes); its
taxonomy puts a superkingdom, a kingdom, phyla, classes and orders above the families (synth.add_upper_ranks), so that
every rank code of the table occurs.  `--reads` reads of 150 bp are sampled from it and run with -M -t 8.  The card's
name and power limit are read in the same run.  Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_mpa.py [--records 1e8] [--reads 4000000]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import build, synth, synth_gpu  # noqa: E402
from krakenuniq_b200.bench_multi_db import gpu_info  # noqa: E402


def fastq(rows, start):
    return b"".join(b"@r%d\n%s\n+\n%s\n" % (start + i, r.tobytes(), b"I" * len(r)) for i, r in enumerate(rows))


def processed(stderr):
    """the "processed in" seconds of every sample of a run"""
    return [float(x.split("processed in ")[1].split("s")[0]) for x in stderr.replace("\r", "\n").splitlines() if "processed in" in x]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=float, default=1e8)
    ap.add_argument("--reads", type=int, default=4_000_000)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--samples", type=int, default=8)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    gpu = gpu_info()
    exe = build.build_classify()
    tmp = tempfile.mkdtemp(prefix="kuq_mpa_")
    try:
        db = synth_gpu.GpuDatabase(int(a.records), n_genomes=2000, k=31, nt=15, idx_type=2, seed=a.seed, device="cuda:0")
        db.write_files(os.path.join(tmp, "db.kdb"), os.path.join(tmp, "db.idx"))
        db.rows = synth.add_upper_ranks(db.rows)
        db.write_taxdb(os.path.join(tmp, "taxDB"))
        key_ct = db.key_ct
        bases, _ = db.sample_reads(a.reads, read_len=150, seed=a.seed + 1)
        host = bases[:a.reads * 150].cpu().numpy()
        del bases, db
        torch.cuda.empty_cache()
        rows = host.reshape(-1, 150)
        per = len(rows) // a.samples
        with open(os.path.join(tmp, "reads.fq"), "wb") as f:
            for s in range(0, len(rows), 1 << 18):
                f.write(fastq(rows[s:s + (1 << 18)], s))
        sheet = "name\tinput\toutput\n"
        for k in range(a.samples):
            with open(os.path.join(tmp, f"s{k}.fq"), "wb") as f:
                f.write(fastq(rows[k * per:(k + 1) * per], k * per))
            sheet += f"s{k}\ts{k}.fq\ts{k}.kraken\n"
        with open(os.path.join(tmp, "sheet.tsv"), "w") as f:
            f.write(sheet)
        base = [exe, "-d", "db.kdb", "-i", "db.idx", "-a", "taxDB", "-M", "-t", str(a.threads)]
        configs = [("without", []), ("--mpa-report", ["--mpa-report", "t.mpa"]), ("--translate-out", ["--translate-out", "t.tr"]),
                   ("--translate-out --translate-mpa-format", ["--translate-out", "t.tr", "--translate-mpa-format"]),
                   ("both", ["--mpa-report", "t.mpa", "--translate-out", "t.tr"])]
        subprocess.run(base + ["-o", "out.kraken", "reads.fq"], cwd=tmp, check=True, capture_output=True)   # warm-up
        for rep in range(a.repeats):
            for tag, extra in configs:
                r = subprocess.run(base + ["-o", "out.kraken"] + extra + ["reads.fq"], cwd=tmp, capture_output=True, text=True)
                if r.returncode:
                    print(json.dumps({"measure": "cli", "config": tag, "error": r.stderr[-1500:]}), flush=True)
                    continue
                secs = processed(r.stderr)[-1]
                print(json.dumps({"measure": "cli", "config": tag, "run": rep, "gpu": gpu, "records": key_ct, "reads": len(rows),
                                  "threads": a.threads, "processed_s": secs, "mreads_per_s": round(len(rows) / 1e6 / secs, 3)}),
                      flush=True)
            for tag, extra in (("sheet without", []), ("sheet --mpa-report", ["--mpa-report", "s.mpa"])):
                t0 = time.time()
                r = subprocess.run(base + extra + ["--sample-sheet", "sheet.tsv"], cwd=tmp, capture_output=True, text=True)
                wall = time.time() - t0
                if r.returncode:
                    print(json.dumps({"measure": "sheet", "config": tag, "error": r.stderr[-1500:]}), flush=True)
                    continue
                print(json.dumps({"measure": "sheet", "config": tag, "run": rep, "gpu": gpu, "samples": a.samples,
                                  "reads": per * a.samples, "processed_s_sum": round(sum(processed(r.stderr)), 3),
                                  "wall_s": round(wall, 3)}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
