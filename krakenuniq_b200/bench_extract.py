"""Cost of extracting reads while classifying (`classify --extract`, kuq_set_extract): one JSON line per measurement.

1. `k_extract_select` device time per 10^6 reads, from torch.profiler (CUDA activities) over a context with an
   extraction set, fed the same batches several times.
2. The CLI's "processed in" time without --extract and with it, at about 1 % and about 50 % of the reads selected and
   with --extract-invert, on plain and gzip FASTQ, single and paired (--paired), runs alternating.

The database is synthetic and built on the GPU (synth_gpu, `--records` records, k = 31, nt = 15, 2000 genomes under a
generated taxonomy); `--reads` reads of 150 bp are sampled from it.  The taxa of each selection are the most frequent
calls of a run without --extract, taken until they cover the wanted share of the reads.  The card's name and power
limit are read in the same run.  Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_extract.py [--records 1e8] [--reads 4000000]
"""
import argparse
import collections
import gzip
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from krakenuniq_b200 import binding, build, synth, synth_gpu  # noqa: E402
from krakenuniq_b200.bench_multi_db import gpu_info  # noqa: E402


def select_ms(tmp, taxa, batches, batch_reads):
    """k_extract_select milliseconds over the batches"""
    kdb = np.fromfile(os.path.join(tmp, "db.kdb"), np.uint8)
    idx = np.fromfile(os.path.join(tmp, "db.idx"), np.uint8)
    tax = synth.Taxonomy.read(os.path.join(tmp, "taxDB"))
    c = binding.Classifier(device=0, max_reads=batch_reads, max_bases=batch_reads * 160)
    c.stage_db(kdb, idx)
    c.set_taxonomy(*tax.parent_map())
    c.set_extract(taxa, 0)
    offs = np.arange(batch_reads + 1, dtype=np.uint64) * 150
    c.classify(batches[0], offs)                                  # warm-up
    ms = 0.0
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for b in batches:
            c.classify(b, offs)
    for e in prof.events():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if "k_extract_select" in e.name:
            ms += t / 1000.0
    c.close()
    return ms


def fastq(rows, start, suffix=b""):
    return b"".join(b"@r%d%s\n%s\n+\n%s\n" % (start + i, suffix, r.tobytes(), b"I" * len(r)) for i, r in enumerate(rows))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=float, default=1e8)
    ap.add_argument("--reads", type=int, default=4_000_000)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--batch-reads", type=int, default=1 << 20)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    gpu = gpu_info()
    exe = build.build_classify()
    tmp = tempfile.mkdtemp(prefix="kuq_extract_")
    try:
        db = synth_gpu.GpuDatabase(int(a.records), n_genomes=2000, k=31, nt=15, idx_type=2, seed=a.seed, device="cuda:0")
        db.write_files(os.path.join(tmp, "db.kdb"), os.path.join(tmp, "db.idx"))
        db.write_taxdb(os.path.join(tmp, "taxDB"))
        key_ct = db.key_ct
        bases, _ = db.sample_reads(a.reads, read_len=150, seed=a.seed + 1)
        host = bases[:a.reads * 150].cpu().numpy()
        del bases, db
        torch.cuda.empty_cache()
        rows = host.reshape(-1, 150)
        half = len(rows) // 2
        inputs = {"fastq": ["reads.fq"], "fastq.gz": ["reads.fq.gz"], "paired": ["m_1.fq", "m_2.fq"]}
        with open(os.path.join(tmp, "reads.fq"), "wb") as f, gzip.open(os.path.join(tmp, "reads.fq.gz"), "wb", 1) as g:
            for s in range(0, len(rows), 1 << 18):
                chunk = fastq(rows[s:s + (1 << 18)], s)
                f.write(chunk)
                g.write(chunk)
        for k, part in ((1, rows[:half]), (2, rows[half:2 * half])):
            with open(os.path.join(tmp, f"m_{k}.fq"), "wb") as f:
                for s in range(0, len(part), 1 << 18):
                    f.write(fastq(part[s:s + (1 << 18)], s, b"/%d" % k))
        base = [exe, "-d", "db.kdb", "-i", "db.idx", "-a", "taxDB", "-M", "-t", str(a.threads), "-o", "out.kraken"]
        subprocess.run(base + ["reads.fq"], cwd=tmp, check=True, capture_output=True)
        calls = collections.Counter(l.split(b"\t")[2] for l in open(os.path.join(tmp, "out.kraken"), "rb"))
        calls.pop(b"0", None)
        selections = {}
        for share in (0.01, 0.5):
            taxa, n = [], 0
            for t, c in sorted(calls.items(), key=lambda kv: kv[1]):          # rare taxa first: close to the share
                if n >= share * len(rows):
                    break
                taxa.append(t.decode())
                n += c
            selections[share] = (",".join(taxa), n / len(rows))
        n = a.batch_reads * 150
        batches = [np.ascontiguousarray(host[i * n:(i + 1) * n]) for i in range(min(a.batches, len(host) // n))]
        taxa50 = [int(t) for t in selections[0.5][0].split(",")]
        ms = select_ms(tmp, taxa50, batches, a.batch_reads)
        print(json.dumps({"measure": "k_extract_select device ms per 1e6 reads", "gpu": gpu, "taxa": len(taxa50),
                          "reads": len(batches) * a.batch_reads,
                          "ms_per_1e6_reads": round(ms / (len(batches) * a.batch_reads / 1e6), 4)}), flush=True)
        configs = [("without", [], None)]
        for share, (taxa, got) in selections.items():
            configs.append((f"{share:.0%} selected", ["--extract", taxa, "--extract-out", "x.fq"], got))
        configs.append(("1% list, --extract-invert", ["--extract", selections[0.01][0], "--extract-out", "x.fq",
                                                        "--extract-invert"], 1 - selections[0.01][1]))
        for layout, files in inputs.items():
            for rep in range(a.repeats):
                for tag, extra, share in configs:
                    cmd = base + (["--paired"] if layout == "paired" else []) + extra + files
                    r = subprocess.run(cmd, cwd=tmp, capture_output=True, text=True)
                    if r.returncode:
                        print(json.dumps({"measure": "cli", "config": tag, "error": r.stderr[-1500:]}), flush=True)
                        continue
                    line = [x for x in r.stderr.replace("\r", "\n").splitlines() if "processed in" in x][-1]
                    secs = float(line.split("processed in ")[1].split("s")[0])
                    reads = half if layout == "paired" else len(rows)
                    print(json.dumps({"measure": "cli", "input": layout, "config": tag, "selected_share": share,
                                      "run": rep, "gpu": gpu, "records": key_ct, "reads": reads, "threads": a.threads,
                                      "processed_s": secs, "mreads_per_s": round(reads / 1e6 / secs, 3)}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
