"""Throughput of `classifyExact` (`krakenuniq --exact`) with an exact k-mer set that has to grow: one JSON line per run.

The database is synthetic and built on the GPU (synth_gpu): `--records` records (default 10^8, k = 31, nt = 15).  The
input is a FASTQ of `--reads` reads of 150 bp sampled from its genomes (1 % substitutions, 20 % random reads).  Nearly
every window of such reads adds a (k-mer, taxon) pair, so at the default million reads the set passes the 0.8 load of
its default 2^26 slots and grows during the run.  Each run is timed from the executable's "processed in" line (the
reads' pass and the end-of-run merge, without loading the database), best of `--repeats`; `report_s` is the driver's
"Report finished in" time (every clade of the taxonomy of `--genomes` species rolled up).  KUQ_TIMING=1 adds the merge
time and each context's exact set after the merge (slots, pairs, growths).  Configurations:
  - one context on GPU 0, from the default 2^26 slots;
  - one context on GPU 0 and two contexts on GPU 0 as replicas (KUQ_DEVICES=0,0), both from 2^20 slots: the cost of
    the layout and of the merge on one card, not a multi-GPU speed-up.  Two contexts take about 33 GB of batch slots
    each, so on an 80 GB card their sets start small and grow as they fill;
  - one and two contexts on GPU 0 with the table's growth capped at `--max-slots` (KUQ_EXACT_MAX_SLOTS): a union that
    does not fit one context's table, which one context refuses and two contexts hold as two k-mer parts;
  - every visible GPU as replicas, when there is more than one.
The inputs are made in a child process, so that this one holds no CUDA context while the executable runs.
md5 sums of the Kraken outputs show that the layouts write the same bytes.  Run from the repository root after
`python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_exact.py [--records 1e8] [--reads 1000000] [--genomes 2000] [--only REGEX]
        [--classify-exact path/to/classifyExact [--classify-exact path/to/other/classifyExact]]
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
from krakenuniq_b200.bench_multi_db import gpu_info, write_fastq  # noqa: E402


def make_inputs(d, records, n_reads, seed, genomes):
    db = synth_gpu.GpuDatabase(int(records), n_genomes=genomes, k=31, nt=15, idx_type=2, seed=seed, device="cuda:0")
    db.write_files(os.path.join(d, "a.kdb"), os.path.join(d, "a.idx"))
    db.write_taxdb(os.path.join(d, "taxDB"))
    reads, _ = db.sample_reads(n_reads, seed=seed + 1)
    key_ct = db.key_ct
    del db
    torch.cuda.empty_cache()
    n = write_fastq(os.path.join(d, "reads.fq"), [(reads, n_reads)])
    del reads
    torch.cuda.empty_cache()
    return key_ct, n


def parse(stderr):
    line = [x for x in stderr.splitlines() if "processed in" in x][-1]
    out = {"processed_s": float(line.split("processed in ")[1].split("s")[0])}
    m = re.search(r"\[timing\] merge\s+([\d.]+) s", stderr)
    out["merge_s"] = float(m.group(1)) if m else None
    out["exact_sets"] = [dict(context=int(a), slots=int(b), pairs=int(c), times_grown=int(e)) for a, b, c, e in
                         re.findall(r"exact set of context (\d+): (\d+) slots, (\d+) pairs, grown (\d+) times", stderr)]
    m = re.search(r"Report finished in ([\d.]+) seconds", stderr)
    out["report_s"] = float(m.group(1)) if m else None
    out["layout"] = [x.strip() for x in stderr.splitlines() if "GPUs, database replicated" in x or "sharded over" in x]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=float, default=1e8)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=9)
    ap.add_argument("--genomes", type=int, default=2000, help="genomes (species) of the synthetic taxonomy")
    ap.add_argument("--max-slots", type=int, default=1 << 27,
                    help="KUQ_EXACT_MAX_SLOTS of the capped configurations: below the union, above each of two parts")
    ap.add_argument("--classify-exact", action="append",
                    help="executable to time (default: this build's classifyExact); give it twice to alternate two builds")
    ap.add_argument("--only", help="run only the configurations whose name matches this regular expression")
    ap.add_argument("--make-inputs", help=argparse.SUPPRESS)          # the child process: inputs into this directory
    a = ap.parse_args()
    if a.make_inputs:
        print(json.dumps(make_inputs(a.make_inputs, a.records, a.reads, a.seed, a.genomes)))
        return
    exes = [os.path.abspath(e) for e in a.classify_exact or [os.path.join(os.path.dirname(build.build_classify()), "classifyExact")]]
    gpu = gpu_info()
    tmp = tempfile.mkdtemp(prefix="kuq_exact_")
    try:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--make-inputs", tmp, "--records", str(a.records), "--reads",
                            str(a.reads), "--seed", str(a.seed), "--genomes", str(a.genomes)], capture_output=True, text=True, check=True)
        key_ct, n_reads = json.loads(r.stdout.strip().splitlines()[-1])
        n_gpu = int(subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout.count("GPU "))
        small = str(1 << 20)
        runs = [("1 context on GPU 0", {"KUQ_DEVICE": "0"}),
                ("1 context on GPU 0, 2^20 slots to start", {"KUQ_DEVICE": "0", "KUQ_SPARSE_SLOTS": small}),
                ("2 contexts on GPU 0 (replicas), 2^20 slots to start", {"KUQ_DEVICES": "0,0", "KUQ_SPARSE_SLOTS": small})]
        # batches of 2·10^4 reads: the library reserves one pair per window before a batch, and a batch of 96 Mbp would
        # ask for more than a capped table on its own
        cap = {"KUQ_EXACT_MAX_SLOTS": str(a.max_slots), "KUQ_SPARSE_SLOTS": small, "KUQ_BATCH_READS": "20000"}
        runs += [(f"1 context on GPU 0, table capped at {a.max_slots} slots", dict(cap, KUQ_DEVICE="0")),
                 (f"2 contexts on GPU 0 (replicas), tables capped at {a.max_slots} slots", dict(cap, KUQ_DEVICES="0,0"))]
        if n_gpu > 1:
            runs.append((f"{n_gpu} GPUs (replicas)", {"KUQ_DEVICES": "all"}))
        if a.only:
            runs = [(name, env) for name, env in runs if re.fullmatch(a.only, name)]
        for name, env in runs:
            # several executables: each repeat runs them one after the other, so that they alternate on the card
            best, md5, rmd5, report_all, failed = {}, {}, {}, {e: [] for e in exes}, set()
            for _ in range(a.repeats):
                for exe in exes:
                    if exe in failed:
                        continue
                    cmd = [exe, "-d", "a.kdb", "-i", "a.idx", "-a", "taxDB", "-M", "-t", "8", "-o", "out.kraken", "-r", "out.report",
                           "reads.fq"]
                    if os.path.exists(os.path.join(tmp, "out.report")):    # the executable appends to a report file
                        os.remove(os.path.join(tmp, "out.report"))
                    r = subprocess.run(cmd, cwd=tmp, capture_output=True, text=True, env=dict(os.environ, KUQ_TIMING="1", **env))
                    if r.returncode:
                        print(json.dumps({"config": name, "classify_exact": exe, "gpu": gpu, "env": env, "error": r.stderr[-1500:]}), flush=True)
                        failed.add(exe)
                        continue
                    got = parse(r.stderr)
                    report_all[exe].append(got["report_s"])
                    if exe not in best or got["processed_s"] < best[exe]["processed_s"]:
                        best[exe] = got
                    with open(os.path.join(tmp, "out.kraken"), "rb") as f:
                        md5[exe] = hashlib.md5(f.read()).hexdigest()
                    with open(os.path.join(tmp, "out.report"), "rb") as f:
                        rmd5[exe] = hashlib.md5(f.read()).hexdigest()
            for exe in exes:
                if exe in best and exe not in failed:
                    print(json.dumps(dict(config=name, classify_exact=exe, gpu=gpu, reads=n_reads, records=key_ct, env=env,
                                          mreads_per_s=round(n_reads / 1e6 / best[exe]["processed_s"], 3), kraken_md5=md5[exe],
                                          report_md5=rmd5[exe], report_s_all=report_all[exe], **best[exe])), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
