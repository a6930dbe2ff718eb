"""Throughput of `classify` against several databases (`classify -d A -d B`, what `krakenuniq --db X --db Y` passes):
one JSON line per run.

The databases are synthetic and built on the GPU (synth_gpu): A of `--records-a` records (default 10^9, k = 31,
nt = 15, a reference-sized database) and B of `--records-b` records (k = 31, nt = 13, another genome under the same
taxonomy).  The input is a FASTQ of `--reads` reads of 150 bp, 80 % sampled from A's genome and 20 % from B's (1 %
substitutions, 20 % random reads).  Three runs of the executable, each timed from its own "processed in" line (the
reads' pass, without loading the databases), best of `--repeats`:
  - A alone;
  - A + B resident (their records fit the HBM budget together);
  - A + B streamed: KUQ_HBM_BUDGET set between A alone and A + B, so the databases stream through two range buffers;
  - A + B sharded: KUQ_FORCE_SHARDS=1 over the visible GPUs (KUQ_DEVICES), each GPU holding a minimizer range of both
    databases.  On a one-GPU machine the GPUs are two contexts on device 0 (KUQ_DEVICES=0,0): that measures what the
    lookup phases, the device flags and the owners' shares cost, not a multi-GPU speed-up.
The script drives only the command line, so `--classify` can time another build of the executable (for example the
parent commit's) on the same inputs; md5 sums of the Kraken outputs let the outputs of two builds be compared.
Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_multi_db.py [--records-a 1e9] [--reads 10000000] [--classify path/to/classify ...]
"""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import build, synth_gpu  # noqa: E402


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                       # the numbers still stand; say what is missing
        return f"unknown ({e})"


def write_fastq(path, parts, read_len=150, chunk=1 << 20):
    """parts: (bases uint8 on the GPU, n_reads) with reads of read_len back to back"""
    qual = b"I" * read_len
    n = 0
    with open(path, "wb") as f:
        for bases, n_reads in parts:
            for a in range(0, n_reads, chunk):
                c = min(chunk, n_reads - a)
                rows = bases[a * read_len:(a + c) * read_len].view(c, read_len).cpu().numpy()
                f.write(b"".join(b"@r%d\n%s\n+\n%s\n" % (n + i, rows[i].tobytes(), qual) for i in range(c)))
                n += c
    return n


def make_inputs(d, records_a, records_b, n_reads, seed):
    dev = "cuda:0"
    a = synth_gpu.GpuDatabase(int(records_a), n_genomes=2000, k=31, nt=15, idx_type=2, seed=seed, device=dev)
    a.write_files(os.path.join(d, "a.kdb"), os.path.join(d, "a.idx"))
    a.write_taxdb(os.path.join(d, "taxDB"))
    n_a = int(n_reads * 0.8)
    ra, _ = a.sample_reads(n_a, seed=seed + 1)
    parts = [(ra, n_a)]
    key_a = a.key_ct
    del a
    torch.cuda.empty_cache()
    b = synth_gpu.GpuDatabase(int(records_b), n_genomes=2000, k=31, nt=13, idx_type=2, seed=seed + 7, device=dev)
    b.write_files(os.path.join(d, "b.kdb"), os.path.join(d, "b.idx"))
    rb, _ = b.sample_reads(n_reads - n_a, seed=seed + 2)
    parts.append((rb, n_reads - n_a))
    key_b = b.key_ct
    del b
    torch.cuda.empty_cache()
    n = write_fastq(os.path.join(d, "reads.fq"), parts)
    del parts, ra, rb
    torch.cuda.empty_cache()
    return key_a, key_b, n


def hbm_bytes(d, name):
    return os.path.getsize(os.path.join(d, name + ".kdb")) - 72 - 2 * (4 + 8 * 62) + os.path.getsize(os.path.join(d, name + ".idx"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records-a", type=float, default=1e9)
    ap.add_argument("--records-b", type=float, default=1e8)
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    ap.add_argument("--classify", action="append", help="executables to time (default: this build's); repeatable")
    a = ap.parse_args()
    exes = [os.path.abspath(x) for x in (a.classify or [build.build_classify()])]
    gpu = gpu_info()
    tmp = tempfile.mkdtemp(prefix="kuq_multi_db_")
    try:
        key_a, key_b, n_reads = make_inputs(tmp, a.records_a, a.records_b, a.reads, a.seed)
        ha, hb = hbm_bytes(tmp, "a"), hbm_bytes(tmp, "b")
        n_gpu = torch.cuda.device_count()
        shard_devices = ",".join(str(g) for g in range(n_gpu)) if n_gpu > 1 else "0,0"
        shard_name = f"A+B sharded over {n_gpu} GPUs" if n_gpu > 1 else "A+B sharded (2 contexts on one GPU: phase and flag cost)"
        runs = [("A", ["a"], {}), ("A+B resident", ["a", "b"], {}),
                ("A+B streamed", ["a", "b"], {"KUQ_HBM_BUDGET": str(ha + hb // 2)}),
                (shard_name, ["a", "b"], {"KUQ_FORCE_SHARDS": "1", "KUQ_DEVICES": shard_devices})]
        for name, dbs, env in runs:
            for exe in exes:                         # builds alternate within a configuration
                secs, md5 = [], None
                for _ in range(a.repeats):
                    cmd = [exe]
                    for x in dbs:
                        cmd += ["-d", f"{x}.kdb", "-i", f"{x}.idx"]
                    cmd += ["-a", "taxDB", "-M", "-t", "8", "-o", "out.kraken", "-r", "out.report", "reads.fq"]
                    r = subprocess.run(cmd, cwd=tmp, capture_output=True, text=True, env=dict(os.environ, **env))
                    if r.returncode:
                        print(json.dumps({"config": name, "classify": exe, "error": r.stderr[-1500:]}), flush=True)
                        break
                    line = [x for x in r.stderr.splitlines() if "processed in" in x][-1]
                    secs.append(float(line.split("processed in ")[1].split("s")[0]))
                    with open(os.path.join(tmp, "out.kraken"), "rb") as f:
                        md5 = hashlib.md5(f.read()).hexdigest()
                    mode = [x.strip() for x in r.stderr.splitlines()
                            if "databases" in x and ("resident" in x or "streamed" in x or "sharded" in x)]
                if secs:
                    print(json.dumps({"config": name, "classify": exe, "gpu": gpu, "reads": n_reads, "records_a": key_a,
                                      "records_b": key_b, "hbm_bytes": [ha, hb], "env": env, "processed_s": secs,
                                      "mreads_per_s": round(n_reads / 1e6 / min(secs), 3), "kraken_md5": md5,
                                      "mode": mode[-1] if mode else ""}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
