"""`classify --paired A B` against the reference pipeline it replaces: `read_merger.pl A B > merged.fa`, then the
reference `classify merged.fa` (scripts/krakenuniq:230-237), both recorded (tests/ref_replay.py).  Kraken output, -C /
-U files and the stats lines byte for byte, report rows column by column, in every ingest path and database layout;
and equal to this project's own `classify merged.fa`."""
import bz2
import gzip
import os
import shutil
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import build, synth
from tests import paired, util

pytestmark = pytest.mark.gpu
G, M = util.GOLDEN, os.path.join(os.path.dirname(util.GOLDEN), "multidb")
DBS = {"database": G, "db2": M}


def _mates(tmp_path, kind):
    """mate files m1, m2 derived from the golden reads (seeded); kind picks format and the defects of the pair"""
    rng = np.random.default_rng(11)
    if kind.startswith("fq"):
        ids, seqs = util.read_fastq(os.path.join(G, "reads_300.fq"))
    else:
        ids, seqs = util.read_fasta(os.path.join(G, "reads.fa"))
    pairs = paired.split_pairs(seqs, rng)
    h1 = [f"{i}/1 mate one".encode() for i in ids]
    h2 = [f"{i}/2".encode() for i in ids]
    r1, r2 = list(zip(h1, [a for a, _ in pairs])), list(zip(h2, [b for _, b in pairs]))
    if kind.endswith("file1_longer"):
        r2 = r2[:-7]
    if kind.endswith("file2_longer"):
        r1 = r1[:-9]
    if kind.endswith("names_mismatch"):
        r2[150] = (b"other/2", r2[150][1])
    write = (lambda r: paired.fastq_bytes(r)) if kind.startswith("fq") else (lambda r: paired.fasta_bytes(r, width=60))
    d1, d2 = write(r1), write(r2)
    if kind.endswith("malformed"):
        at = d2.index(b"@" + h2[200])
        d2 = d2[:at] + b"@ " + d2[at + 1:]
    (tmp_path / "m1").write_bytes(d1)
    (tmp_path / "m2").write_bytes(d2)


T1 = (None, ["-t", "1"], {}, None)
T8 = (None, ["-t", "8"], {}, None)
SERIAL = (None, ["-t", "1"], {"KUQ_SERIAL_INGEST": "1"}, None)
GZ = (None, ["-t", "8"], {}, "gz+plain")
BZ2 = (None, ["-t", "1"], {}, "bz2")
REPLICAS = (None, ["-t", "8"], {"KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"}, None)
INGEST = [T1, T8, SERIAL, GZ, BZ2]
# tag: (mates, merger flags, tool, databases, the reference's flags, our runs: (flags instead of the reference's or None,
# ingest flags, environment, compression of the mates))
CASES = {
    "fq_M": ("fq", [], "classify", ["database"], ["-M"], INGEST + [REPLICAS]),
    "fq_M_s_c": ("fq", [], "classify", ["database"], ["-M", "-s", "-c"], [T8, SERIAL]),
    "fa_M_u20000": ("fa", [], "classify", ["database"], ["-M", "-u", "20000"], INGEST + [REPLICAS]),
    # -x: staged whole, streamed in ranges (BatchReader), and -M sharded over two contexts (the -x rule)
    "fq_x40K": ("fq", [], "classify", ["database"], ["-x", "40K"],
                [T1, (None, ["-t", "1"], {"KUQ_FORCE_CHUNKS": "1"}, None),
                 (["-M"], ["-t", "1"], {"KUQ_FORCE_SHARDS": "1", "KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"}, None)]),
    "fq_q2": ("fq", [], "classify", ["database"], ["-M", "-q", "-m", "2"], [T1, T8]),
    "fa_two_databases": ("fa", [], "classify", ["database", "db2"], ["-M"],
                         [T8, SERIAL, (None, ["-t", "1"], {"KUQ_HBM_BUDGET": "200000"}, None),
                          (None, ["-t", "1"], {"KUQ_FORCE_SHARDS": "1", "KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"}, None)]),
    "fq_exact": ("fq", [], "classifyExact", ["database"], ["-M"], [T1, T8, REPLICAS]),
    "fq_file1_longer": ("fq_file1_longer", [], "classify", ["database"], ["-M"], [T1, T8, SERIAL]),
    "fa_file2_longer": ("fa_file2_longer", [], "classify", ["database"], ["-M"], [T1, T8, SERIAL]),
    "fq_check_names_pass": ("fq", ["--check-names"], "classify", ["database"], ["-M"], [T8]),
    "fq_check_names_fail": ("fq_names_mismatch", ["--check-names"], "classify", ["database"], ["-M"], [T1, T8, SERIAL, GZ]),
    "fq_names_differ_unchecked": ("fq_names_mismatch", [], "classify", ["database"], ["-M"], [T8]),
    "fq_malformed": ("fq_malformed", [], "classify", ["database"], ["-M"], [T1, T8, SERIAL]),
}
OUTS = ("kraken", "C", "U")


def _stats(stderr):
    """the stats lines of classify.cpp:361-375 without their time-dependent numbers"""
    lines = stderr.replace("\r", "\n").splitlines()
    n = [l.split(" processed in")[0] for l in lines if " processed in " in l]
    return n + [l.strip() for l in lines if "sequences classified (" in l or "sequences unclassified (" in l]


def _report_lines(path):
    rows = {}
    for line in open(path):
        if line.startswith("#") or line.startswith("%"):
            continue
        f = line.rstrip("\n").split("\t")
        rows[f[6]] = f
    return rows


def _outputs(tmp_path, prefix):
    got = {o: (tmp_path / f"{prefix}.{o}").read_bytes() if (tmp_path / f"{prefix}.{o}").exists() else None for o in OUTS}
    rep = tmp_path / f"{prefix}.report"
    got["report"] = _report_lines(rep) if rep.exists() else None
    return got


def _run_ours(tmp_path, tool, args, env):
    exe = os.path.join(os.path.dirname(build.build_classify()), tool)
    for o in OUTS + ("report",):
        (tmp_path / f"o.{o}").unlink(missing_ok=True)
    r = subprocess.run([exe] + args, cwd=tmp_path, capture_output=True, text=True,
                       env=dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22), **env))
    return r, _outputs(tmp_path, "o")


@pytest.mark.parametrize("tag", list(CASES))
def test_paired_matches_reference_pipeline(reference, tmp_path, tag):
    kind, merger_flags, tool, dbs, flags, runs = CASES[tag]
    for d in dbs:
        for ext in (".kdb", ".idx", ".kdb.counts"):
            shutil.copyfile(os.path.join(DBS[d], d + ext), tmp_path / (d + ext))
    shutil.copyfile(os.path.join(G, "taxDB"), tmp_path / "taxDB")
    _mates(tmp_path, kind)
    paired.install_merger()
    merger = reference.run_tool(paired.MERGER, merger_flags + ["m1", "m2"], cwd=tmp_path)
    merger_err = (tmp_path / "merged.err").read_text(errors="replace")
    common = sum((["-d", f"{d}.kdb", "-i", f"{d}.idx"] for d in dbs), []) + ["-a", "taxDB"]
    outs = ["-C", "{p}.C", "-U", "{p}.U", "-r", "{p}.report", "-o", "{p}.kraken"]
    r = reference.run_tool(tool, common + ["-t", "1"] + [x.format(p="ref") for x in outs] + flags + ["merged.fa"], cwd=tmp_path)
    assert r.returncode == 0, r.stderr[-1500:]
    want, want_stats = _outputs(tmp_path, "ref"), _stats(r.stderr)
    assert want["kraken"] or "-c" in flags
    stopped = merger.returncode != 0
    assert stopped == (tag in ("fq_check_names_fail", "fq_malformed")), merger_err
    warned = "mismatched sequence counts" in merger_err

    # this project's classify on the merged file is the same run
    o, got = _run_ours(tmp_path, tool, common + ["-t", "1"] + [x.format(p="o") for x in outs] + flags + ["merged.fa"], {})
    assert o.returncode == 0, o.stderr[-2000:]
    assert got == want and _stats(o.stderr) == want_stats

    mates = {None: ["m1", "m2"]}
    mates["gz+plain"] = ["m1.gz", "m2"]
    mates["bz2"] = ["m1.bz2", "m2.bz2"]
    with open(tmp_path / "m1", "rb") as f:
        data1 = f.read()
    (tmp_path / "m1.gz").write_bytes(gzip.compress(data1, mtime=0))
    (tmp_path / "m1.bz2").write_bytes(bz2.compress(data1))
    (tmp_path / "m2.bz2").write_bytes(bz2.compress((tmp_path / "m2").read_bytes()))
    check = ["--check-names"] if merger_flags else []
    for ours, ingest, env, comp in runs:
        args = common + ingest + [x.format(p="o") for x in outs] + (flags if ours is None else ours) + ["--paired"] + check + mates[comp]
        o, got = _run_ours(tmp_path, tool, args, env)
        assert o.returncode == (65 if stopped else 0), (env, comp, o.stderr[-2000:])
        assert got == want, (ingest, env, comp)
        assert _stats(o.stderr) == want_stats, (ingest, env, comp)
        assert ("mismatched sequence counts" in o.stderr) == warned
        if stopped:
            assert ("mismatched mate pair names" if "check" in tag else "malformed fastq file") in o.stderr
        if env.get("KUQ_DEVICES"):
            assert "not usable" not in o.stderr and ("sharded over 2 GPUs" in o.stderr or "2 GPUs" in o.stderr), o.stderr[:1500]


def test_paired_large_crosses_batches_and_work_units(tmp_path):
    """200 k pairs of 2 x 150 bp from the synthetic generator: many work units and (with KUQ_BATCH_READS) batches, on the
    parallel and the serial ingest, against classify on the merged file tests/paired.py writes"""
    rng = np.random.default_rng(3)
    tax = synth.make_taxonomy(6)
    genomes = synth.random_genomes(rng, 6, 50000)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, 31)
    kdb, idx = synth.build_db_images(km, tx, 31, 8, 2)
    kdb.tofile(tmp_path / "db.kdb")
    idx.tofile(tmp_path / "db.idx")
    tax.write(tmp_path / "taxDB")
    n = 200_000
    bases, offs = synth.sample_reads(rng, genomes, n, 320, 0.01, 0.02, 0.2)
    seqs = [bases[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n)]
    pairs = paired.split_pairs(seqs, rng, mate_len=150)
    d1 = paired.fastq_bytes([(b"p%d/1" % i, a) for i, (a, _) in enumerate(pairs)])
    d2 = paired.fastq_bytes([(b"p%d/2" % i, b) for i, (_, b) in enumerate(pairs)])
    (tmp_path / "m1").write_bytes(d1)
    (tmp_path / "m2").write_bytes(d2)
    merged, warnings, error = paired.merge(d1, d2, check_names=True)
    assert not warnings and error is None
    (tmp_path / "merged.fa").write_bytes(merged)
    common = ["-d", "db.kdb", "-i", "db.idx", "-a", "taxDB", "-M", "-u", "100000", "-r", "{p}.report", "-o", "{p}.kraken"]
    exe = build.build_classify()
    r = subprocess.run([exe] + [x.format(p="ref") for x in common] + ["-t", "8", "merged.fa"], cwd=tmp_path,
                       capture_output=True, text=True, env=dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22)))
    assert r.returncode == 0, r.stderr[-2000:]
    want = _outputs(tmp_path, "ref")
    assert want["kraken"].count(b"\n") == n and want["kraken"].split(b"\n", 1)[0].split(b"\t")[1:4:2] == [b"p0", b"301"]
    for ingest, env in ((["-t", "8"], {}), (["-t", "3"], {"KUQ_BATCH_READS": "20000"}), (["-t", "1"], {"KUQ_SERIAL_INGEST": "1"})):
        o, got = _run_ours(tmp_path, "classify", [x.format(p="o") for x in common] + ingest + ["--paired", "--check-names", "m1", "m2"], env)
        assert o.returncode == 0, o.stderr[-2000:]
        assert got == want, (ingest, env)
        assert _stats(o.stderr) == _stats(r.stderr)
