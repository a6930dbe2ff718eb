"""Throughput of `set_lcas` (step 6 of build_db.sh on the GPU) with and without -a -A (krakenuniq-build
--taxids-for-sequences --taxids-for-genomes), and of `classify` on the two databases; one JSON line per configuration.

The library: `--gbp` Gbp of `--species` random genomes, each in `--strains` mutated copies (0.1 % substitutions), every
strain an assembly of two records.  With -a -A every record becomes a sequence taxon under its strain's assembly
taxon, about 10^5 new taxa at 1 Gbp.  The k-mer set comes from the drop-in `kmer_set` and `db_sort -z`.
Measured:
  - set_lcas: build_db.sh's command line end to end (FASTA parsing, taxonomy, GPU lookups and LCAs, writing the
    database, the taxDB and the .counts), library Gbp / wall second, best of `--repeats`;
  - classify -M: reads sampled from the strains (1 % substitutions), Mreads / s from the executable's own
    "processed in" line (the reads' pass, without loading the database), best of `--repeats`.
Run from the repository root after `python -m krakenuniq_b200.build`:
    python krakenuniq_b200/bench_set_lcas.py [--gbp 1] [--reads 2000000]
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

WIDTH = 80
ACGT = np.frombuffer(b"ACGT", np.uint8)


def fasta_record(f, header, seq):
    f.write(b">" + header + b"\n")
    f.write(np.hstack([seq.reshape(-1, WIDTH), np.full((len(seq) // WIDTH, 1), ord("\n"), np.uint8)]).tobytes())


def make_inputs(d, gbp, species, strains, n_reads, seed):
    """lib.fa, seqid2taxid.map (with assembly names), taxDB, reads.fa; returns the library's size in bases"""
    rng = np.random.default_rng(seed)
    glen = int(gbp * 1e9) // (species * strains) // (2 * WIDTH) * (2 * WIDTH)      # two records per strain
    half = glen // 2
    rows = ["1\t1\troot\tno rank", "2\t1\tgenus\tgenus"] + [f"{100 + s}\t2\tspecies{s}\tspecies" for s in range(species)]
    with open(os.path.join(d, "taxDB"), "w") as f:
        f.write("".join(r + "\n" for r in rows))
    reads = []
    per_strain = max(1, n_reads // (species * strains))
    with open(os.path.join(d, "lib.fa"), "wb") as lib, open(os.path.join(d, "seqid2taxid.map"), "w") as m:
        for s in range(species):
            base = rng.integers(0, 4, glen, dtype=np.uint8)
            for j in range(strains):
                c = base.copy()
                pos = rng.integers(0, glen, glen // 1000)
                c[pos] = (c[pos] + rng.integers(1, 4, len(pos), dtype=np.uint8)) & 3
                a = ACGT[c]
                for r in range(2):
                    sid = f"s{s}_{j}_{r}"
                    fasta_record(lib, f"{sid}.1 species {s} strain {j} record {r}".encode(), a[r * half:(r + 1) * half])
                    m.write(f"{sid}\t{100 + s}\tspecies{s} strain{j}\n")
                rd = c[rng.integers(0, glen - 150, per_strain)[:, None] + np.arange(150)]
                e = rng.random(rd.shape) < 0.01
                rd[e] = (rd[e] + 1) & 3
                reads.append(ACGT[rd])
    reads = np.concatenate(reads)
    with open(os.path.join(d, "reads.fa"), "wb") as f:
        f.write(b"".join(b">r%d\n%s\n" % (i, r.tobytes()) for i, r in enumerate(reads)))
    return species * strains * glen, len(reads)


def set_lcas_args(taxdb, out, plus):
    return (["-M", "-x", "-d", "database0.kdb", "-o", out, "-i", "database.idx", "-v", "-b", taxdb]
            + (["-a", "-A"] if plus else []) + ["-t", "8", "-m", "seqid2taxid.map", "-c", out + ".counts", "-F", "lib.fa", "-T"])


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                       # the numbers still stand; say what is missing
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbp", type=float, default=1.0)
    ap.add_argument("--species", type=int, default=100)
    ap.add_argument("--strains", type=int, default=500)
    ap.add_argument("--reads", type=int, default=2_000_000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    db_sort, set_lcas = build.build_dbtools()
    classify = build.build_classify()
    gpu = gpu_info()
    tmp = tempfile.mkdtemp(prefix="kuq_set_lcas_")
    try:
        t = time.perf_counter()
        n_bases, n_reads = make_inputs(tmp, a.gbp, a.species, a.strains, a.reads, a.seed)
        gen_s = time.perf_counter() - t
        run = lambda cmd: subprocess.run(cmd, cwd=tmp, check=True, capture_output=True, text=True)   # noqa: E731
        run([build.KMER_SET, "count", "-m", "31", "-s", "1G", "-C", "-t", "8", "-o", "database", "lib.fa"])
        run([db_sort, "-z", "-M", "-n", "12", "-d", "database_0", "-o", "database0.kdb", "-i", "database.idx"])
        os.remove(os.path.join(tmp, "database_0"))
        key_ct = int(np.fromfile(os.path.join(tmp, "database0.kdb"), np.uint64, count=7)[6])
        for plus, name in ((False, "plain"), (True, "taxids")):
            times = []
            for _ in range(a.repeats):
                taxdb = f"taxDB.{name}"
                shutil.copy(os.path.join(tmp, "taxDB"), os.path.join(tmp, taxdb))
                t = time.perf_counter()
                r = run([set_lcas] + set_lcas_args(taxdb, f"{name}.kdb", plus))
                times.append(time.perf_counter() - t)
            n_taxa = sum(1 for _ in open(os.path.join(tmp, taxdb)))
            owners = sum(1 for _ in open(os.path.join(tmp, f"{name}.kdb.counts")))
            print(json.dumps({"metric": "set_lcas", "config": name, "flags": "-a -A" if plus else "", "gpu": gpu,
                              "gbp": round(n_bases / 1e9, 3), "distinct_kmers": key_ct, "wall_s": [round(x, 2) for x in times],
                              "gbp_per_s": round(n_bases / 1e9 / min(times), 3), "taxa": n_taxa,
                              "taxa_owning_kmers": owners, "stdout_lines": r.stdout.count("\n"),
                              "library_generation_s": round(gen_s, 1)}), flush=True)
        for name in ("plain", "taxids"):
            secs = []
            for _ in range(a.repeats):
                r = run([classify, "-d", f"{name}.kdb", "-i", "database.idx", "-a", f"taxDB.{name}", "-M", "-t", "8",
                         "-o", f"{name}.kraken", "-r", f"{name}.report", "reads.fa"])
                line = [x for x in r.stderr.splitlines() if "processed in" in x][-1]
                secs.append(float(line.split("processed in ")[1].split("s")[0]))
            with open(os.path.join(tmp, f"{name}.report")) as f:
                report_rows = sum(1 for x in f if x[:1].isdigit())
            print(json.dumps({"metric": "classify", "database": name, "gpu": gpu, "reads": n_reads,
                              "processed_s": secs, "mreads_per_s": round(n_reads / 1e6 / min(secs), 3),
                              "report_rows": report_rows}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
