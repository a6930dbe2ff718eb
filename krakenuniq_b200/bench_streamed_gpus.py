"""Time of `classify` on a database streamed in minimizer ranges over 1, 2, ... GPUs: one JSON line per run.

The database is synthetic and built on the GPU (synth_gpu, as bench_multi_db.py builds its database A): `--records`
records (default 10^9, k = 31, nt = 15, about 20 GB in HBM with its index), and the input a FASTQ of `--reads` reads of
150 bp sampled from its genomes (1 % substitutions, 20 % random reads).  KUQ_HBM_BUDGET is set to half the database's
HBM bytes, so the run streams the database in ranges of an eighth of it (about 8 ranges).  The executable runs with
KUQ_DEVICES set to one device and then to every larger prefix of the visible devices; on a one-GPU machine the second
run is `0,0`, two contexts on one card, which measures what the layout costs (batches on every context, host barriers,
owners) and not a speed-up.  KUQ_HBM_BUDGET caps each context, so two contexts on one card also hold twice the reads per
round: fewer rounds, each a pass over the database, which the one-card comparison mixes into the layout's cost.  Per run: the "processed in" seconds (the reads' pass, without staging; best of
`--repeats`), the rounds, the ranges per GPU and the md5 sums of the Kraken output and of the report rows, which have to
be equal for every device count.
Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_streamed_gpus.py [--records 1e9] [--reads 2000000]
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

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import build, synth_gpu  # noqa: E402
from krakenuniq_b200.bench_multi_db import gpu_info, hbm_bytes, write_fastq  # noqa: E402


def make_inputs(d, records, n_reads, seed):
    db = synth_gpu.GpuDatabase(int(records), n_genomes=2000, k=31, nt=15, idx_type=2, seed=seed, device="cuda:0")
    db.write_files(os.path.join(d, "a.kdb"), os.path.join(d, "a.idx"))
    db.write_taxdb(os.path.join(d, "taxDB"))
    reads, _ = db.sample_reads(n_reads, seed=seed + 1)
    key_ct = db.key_ct
    del db
    n = write_fastq(os.path.join(d, "reads.fq"), [(reads, n_reads)])
    del reads
    torch.cuda.empty_cache()
    return key_ct, n


def report_md5(path):
    """md5 of the report's rows (its header names the date and the command line)"""
    with open(path, "rb") as f:
        rows = [line for line in f if not line.startswith(b"#")]
    return hashlib.md5(b"".join(rows)).hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=float, default=1e9)
    ap.add_argument("--reads", type=int, default=2_000_000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    ap.add_argument("--classify", default=None, help="executable to time (default: this build's)")
    a = ap.parse_args()
    exe = os.path.abspath(a.classify or build.build_classify())
    gpu = gpu_info()
    n_gpu = torch.cuda.device_count()
    if n_gpu < 1:
        raise SystemExit("no GPU visible")
    device_sets = [",".join(str(g) for g in range(n)) for n in range(1, n_gpu + 1)] if n_gpu > 1 else ["0", "0,0"]
    tmp = tempfile.mkdtemp(prefix="kuq_streamed_gpus_")
    try:
        key_ct, n_reads = make_inputs(tmp, a.records, a.reads, a.seed)
        hbm = hbm_bytes(tmp, "a")
        env = {"KUQ_HBM_BUDGET": str(hbm // 2)}
        for devices in device_sets:
            secs, out = [], {}
            for _ in range(a.repeats):
                for f in ("out.kraken", "out.report"):         # classify appends its report to an existing file
                    if os.path.exists(os.path.join(tmp, f)):
                        os.unlink(os.path.join(tmp, f))
                cmd = [exe, "-d", "a.kdb", "-i", "a.idx", "-a", "taxDB", "-M", "-t", "8", "-o", "out.kraken", "-r", "out.report",
                       "reads.fq"]
                r = subprocess.run(cmd, cwd=tmp, capture_output=True, text=True, env=dict(os.environ, KUQ_DEVICES=devices, **env))
                if r.returncode:
                    print(json.dumps({"devices": devices, "classify": exe, "error": r.stderr[-1500:]}), flush=True)
                    break
                err = r.stderr.replace("\r", "\n")
                secs.append(float(re.findall(r"processed in ([\d.]+)s", err)[-1]))
                chunks = int(re.search(r"Database split into (\d+) chunks", err).group(1))
                m = re.search(r"streamed over \d+ GPUs: ranges per GPU ([\d/]+)", err)
                with open(os.path.join(tmp, "out.kraken"), "rb") as f:
                    kraken_md5 = hashlib.md5(f.read()).hexdigest()
                out = {"chunks": chunks, "rounds": len(re.findall(r"\(database chunk 1 of \d+\)", err)),
                       "ranges_per_gpu": m.group(1) if m else str(chunks), "kraken_md5": kraken_md5,
                       "report_md5": report_md5(os.path.join(tmp, "out.report"))}
            if secs:
                label = "one GPU" if devices == "0" else (f"{devices.count(',') + 1} contexts on one GPU: cost of the layout, "
                                                          "not a speed-up" if n_gpu == 1 else f"{devices.count(',') + 1} GPUs")
                print(json.dumps({"devices": devices, "label": label, "gpu": gpu, "reads": n_reads, "records": key_ct,
                                  "hbm_bytes": hbm, "env": env, "processed_s": secs, "best_s": min(secs), **out}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
