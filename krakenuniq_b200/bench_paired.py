"""Throughput of `classify --paired A B` against `classify merged.fa`: one JSON line per run.

`krakenuniq --paired` merges the mates with read_merger.pl into a temporary FASTA and classifies that file
(scripts/krakenuniq:230-237).  `classify --paired` merges them in its ingest.  This script times both classify stages on
the same pairs, without the Perl step: `merged.fa` is written here with the merger's layout (`>id` of mate 1, then
mate1 + "N" + mate2), so the second run is what the wrapper's classify stage costs after the merge.

The database is synthetic and built on the GPU (synth_gpu, `--records` records, k = 31, nt = 15).  `--pairs` pairs of
2 x `--mate-len` bp are sampled from its genome (1 % substitutions, 20 % random pairs) and written as two FASTQ mate
files, plain and gzip.  Each run is timed from the executable's own "processed in" line (the reads' pass, without
loading the database), best of `--repeats`; md5 sums of the Kraken outputs show that the runs classify the same
records.  Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_paired.py [--records 1e9] [--pairs 10000000] [--classify path/to/classify]
"""
import argparse
import gzip
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
from krakenuniq_b200.bench_multi_db import gpu_info  # noqa: E402

_COMP = torch.zeros(256, dtype=torch.uint8)
for a, b in zip(b"ACGTN", b"TGCAN"):
    _COMP[a] = b


def write_pairs(d, db, n_pairs, mate_len, seed, chunk=1 << 19):
    """m1.fq / m2.fq (mate 2 = reverse complement of the fragment's other end), merged.fa, and gzip copies of the mates"""
    frag = 2 * mate_len + 50
    bases, _ = db.sample_reads(n_pairs, read_len=frag, seed=seed)
    comp = _COMP.to(bases.device)
    qual = b"I" * mate_len
    with open(os.path.join(d, "m1.fq"), "wb") as f1, open(os.path.join(d, "m2.fq"), "wb") as f2, \
            open(os.path.join(d, "merged.fa"), "wb") as fm:
        for a in range(0, n_pairs, chunk):
            c = min(chunk, n_pairs - a)
            rows = bases[a * frag:(a + c) * frag].view(c, frag)
            m1 = rows[:, :mate_len].cpu().numpy()
            m2 = comp[rows[:, frag - mate_len:].flip(1).long()].cpu().numpy()
            f1.write(b"".join(b"@p%d/1\n%s\n+\n%s\n" % (a + i, m1[i].tobytes(), qual) for i in range(c)))
            f2.write(b"".join(b"@p%d/2\n%s\n+\n%s\n" % (a + i, m2[i].tobytes(), qual) for i in range(c)))
            fm.write(b"".join(b">p%d\n%sN%s\n" % (a + i, m1[i].tobytes(), m2[i].tobytes()) for i in range(c)))
    del bases
    torch.cuda.empty_cache()
    for m in ("m1.fq", "m2.fq"):
        with open(os.path.join(d, m), "rb") as src, gzip.open(os.path.join(d, m + ".gz"), "wb", compresslevel=1) as dst:
            shutil.copyfileobj(src, dst, 1 << 24)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=float, default=1e9)
    ap.add_argument("--pairs", type=int, default=10_000_000)
    ap.add_argument("--mate-len", type=int, default=150)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    ap.add_argument("--classify", action="append", help="executables to time (default: this build's); repeatable")
    a = ap.parse_args()
    exes = [os.path.abspath(x) for x in (a.classify or [build.build_classify()])]
    gpu = gpu_info()
    tmp = tempfile.mkdtemp(prefix="kuq_paired_")
    try:
        db = synth_gpu.GpuDatabase(int(a.records), n_genomes=2000, k=31, nt=15, idx_type=2, seed=a.seed, device="cuda:0")
        db.write_files(os.path.join(tmp, "db.kdb"), os.path.join(tmp, "db.idx"))
        db.write_taxdb(os.path.join(tmp, "taxDB"))
        key_ct = db.key_ct
        write_pairs(tmp, db, a.pairs, a.mate_len, a.seed + 1)
        del db
        torch.cuda.empty_cache()
        runs = [("merged.fa (the wrapper's classify stage)", ["merged.fa"], {}),
                ("--paired plain FASTQ", ["--paired", "m1.fq", "m2.fq"], {}),
                ("--paired plain FASTQ, serial ingest", ["--paired", "m1.fq", "m2.fq"], {"KUQ_SERIAL_INGEST": "1"}),
                ("--paired gzip FASTQ", ["--paired", "m1.fq.gz", "m2.fq.gz"], {})]
        for name, inputs, env in runs:
            for exe in exes:
                secs, md5 = [], None
                for _ in range(a.repeats):
                    cmd = [exe, "-d", "db.kdb", "-i", "db.idx", "-a", "taxDB", "-M", "-t", str(a.threads), "-o", "out.kraken",
                           "-r", "out.report"] + inputs
                    if os.path.exists(os.path.join(tmp, "out.report")):
                        os.unlink(os.path.join(tmp, "out.report"))
                    r = subprocess.run(cmd, cwd=tmp, capture_output=True, text=True, env=dict(os.environ, **env))
                    if r.returncode:
                        print(json.dumps({"config": name, "classify": exe, "error": r.stderr[-1500:]}), flush=True)
                        break
                    line = [x for x in r.stderr.replace("\r", "\n").splitlines() if "processed in" in x][-1]
                    secs.append(float(line.split("processed in ")[1].split("s")[0]))
                    with open(os.path.join(tmp, "out.kraken"), "rb") as f:
                        md5 = hashlib.md5(f.read()).hexdigest()
                if secs:
                    print(json.dumps({"config": name, "classify": exe, "gpu": gpu, "pairs": a.pairs, "mate_len": a.mate_len,
                                      "records": key_ct, "threads": a.threads, "env": env, "processed_s": secs,
                                      "mpairs_per_s": round(a.pairs / 1e6 / min(secs), 3), "kraken_md5": md5}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
