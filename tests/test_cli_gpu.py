"""The drop-in `classify` executable (krakenuniq_b200/bin/classify) against the golden outputs of the unmodified
reference `classify`: Kraken output byte-identical, report rows identical column by column."""
import os
import subprocess

import pytest

from krakenuniq_b200 import build
from tests import util

pytestmark = pytest.mark.gpu
G = util.GOLDEN


def _run(tmp_path, tag, extra, reads, env_extra=None):
    exe = build.build_classify()
    out, rep = tmp_path / f"{tag}.kraken", tmp_path / f"{tag}.report.tsv"
    cmd = [exe, "-d", os.path.join(G, "database.kdb"), "-i", os.path.join(G, "database.idx"), "-a",
           os.path.join(G, "taxDB"), "-t", "1", "-r", str(rep), "-o", str(out)] + extra + [os.path.join(G, reads)]
    env = dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22))
    env.update(env_extra or {})
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    return out, rep, r


def _report_lines(path):
    rows = {}
    for line in open(path):
        if line.startswith("#") or line.startswith("%"):
            continue
        f = line.rstrip("\n").split("\t")
        rows[f[6]] = f
    return rows


@pytest.mark.parametrize("tag,extra,reads", [
    ("preload", ["-M"], "reads.fa"),
    ("preload_u20000", ["-M", "-u", "20000"], "reads.fa"),
    ("chunked", ["-x", "40K"], "reads.fa"),
    ("fastq", ["-M"], "reads_300.fq"),
    ("crlf", ["-M"], "reads_crlf_60.fa"),
])
def test_cli_matches_reference_outputs(tmp_path, tag, extra, reads):
    out, rep, r = _run(tmp_path, tag, extra, reads)
    assert open(out).read() == open(os.path.join(G, f"{tag}.kraken")).read()
    got, want = _report_lines(rep), _report_lines(os.path.join(G, f"{tag}.report.tsv"))
    assert got == want
    # the stats lines of classify.cpp:361-375 (time-dependent numbers masked)
    want_err = open(os.path.join(G, f"{tag}.stderr.txt")).read().split("\n")
    n_seq = want_err[0].split(" sequences")[0]
    assert f"{n_seq} sequences (" in r.stderr
    assert want_err[1].strip() in r.stderr and want_err[2].strip() in r.stderr


@pytest.mark.parametrize("tag,extra,env", [("preload", ["-M"], {}), ("preload_u20000", ["-M", "-u", "20000"], {}),
                                           ("chunked", ["-M"], {"KUQ_FORCE_SHARDS": "1"})])
def test_cli_one_device_as_several_gpus(tmp_path, tag, extra, env):
    """one device listed twice: the multi-GPU paths of one process, with a context per listed device — replicas
    (batches round-robin, kuq_merge_into at the end) and minimizer-range shards (shard_loop: peer stores, device
    flags between the contexts, kuq_merge_into over shard contexts; sketches follow the -x rule).  Each context of
    the executable reserves about 33 GB of batch slots (3 slots of 288 MiB bases), so an 80 GB card holds two."""
    # small batches so that every context gets work; a small sparse set so that it has to grow
    out, rep, r = _run(tmp_path, tag, extra, "reads.fa",
                       dict(env, KUQ_DEVICES="0,0", KUQ_BATCH_READS="200", KUQ_SPARSE_SLOTS=str(1 << 12)))
    assert "not usable" not in r.stderr, [l for l in r.stderr.splitlines() if "not usable" in l]
    assert ("sharded over 2 GPUs" if env else "2 GPUs, database replicated") in r.stderr, r.stderr[:1500]
    assert open(out).read() == open(os.path.join(G, f"{tag}.kraken")).read()
    assert _report_lines(rep) == _report_lines(os.path.join(G, f"{tag}.report.tsv"))


@pytest.mark.parametrize("threads,serial", [("8", False), ("3", False), ("1", True)])
@pytest.mark.parametrize("tag,extra,reads", [("preload_u20000", ["-M", "-u", "20000"], "reads.fa"),
                                              ("fastq", ["-M"], "reads_300.fq"), ("crlf", ["-M"], "reads_crlf_60.fa")])
def test_cli_ingest_paths(tmp_path, threads, serial, tag, extra, reads):
    """parallel mmap ingest (any -t) and the serial zlib reader give the reference's bytes"""
    exe = build.build_classify()
    out, rep = tmp_path / "o.kraken", tmp_path / "o.report.tsv"
    cmd = [exe, "-d", os.path.join(G, "database.kdb"), "-i", os.path.join(G, "database.idx"), "-a",
           os.path.join(G, "taxDB"), "-t", threads, "-r", str(rep), "-o", str(out)] + extra + [os.path.join(G, reads)]
    env = dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22), **({"KUQ_SERIAL_INGEST": "1"} if serial else {}))
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    assert open(out).read() == open(os.path.join(G, f"{tag}.kraken")).read()
    assert _report_lines(rep) == _report_lines(os.path.join(G, f"{tag}.report.tsv"))


def test_cli_bz2_input(tmp_path):
    """bzip2-compressed reads (seqreader.hpp:24,48: the reference reads them through bxzstr)"""
    import bz2
    bz = tmp_path / "reads.fa.bz2"
    bz.write_bytes(bz2.compress(open(os.path.join(G, "reads.fa"), "rb").read()))
    exe = build.build_classify()
    out = tmp_path / "o.kraken"
    cmd = [exe, "-d", os.path.join(G, "database.kdb"), "-i", os.path.join(G, "database.idx"), "-a",
           os.path.join(G, "taxDB"), "-M", "-o", str(out), str(bz)]
    r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22)))
    assert r.returncode == 0, r.stderr[-2000:]
    assert open(out).read() == open(os.path.join(G, "preload.kraken")).read()


def test_cli_gz_input(tmp_path):
    import gzip
    import shutil
    gz = tmp_path / "reads.fq.gz"
    with open(os.path.join(G, "reads_300.fq"), "rb") as fi, gzip.open(gz, "wb") as fo:
        shutil.copyfileobj(fi, fo)
    exe = build.build_classify()
    out = tmp_path / "o.kraken"
    cmd = [exe, "-d", os.path.join(G, "database.kdb"), "-i", os.path.join(G, "database.idx"), "-a",
           os.path.join(G, "taxDB"), "-M", "-o", str(out), str(gz)]
    r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22)))
    assert r.returncode == 0, r.stderr[-2000:]
    assert open(out).read() == open(os.path.join(G, "fastq.kraken")).read()


def test_cli_flags(tmp_path):
    exe = build.build_classify()
    base = [exe, "-d", os.path.join(G, "database.kdb"), "-i", os.path.join(G, "database.idx"), "-a",
            os.path.join(G, "taxDB")]
    env = dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22))
    reads = os.path.join(G, "reads_300.fq")
    # -c: only classified lines; -s: sequence column; stdout by default
    r = subprocess.run(base + ["-M", "-c", "-s", reads], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-1000:]
    want = [l for l in open(os.path.join(G, "fastq.kraken")) if l.startswith("C")]
    got = r.stdout.splitlines(keepends=True)
    assert len(got) == len(want)
    ids, seqs = util.read_fastq(reads)
    seq_of = dict(zip(ids, seqs))
    for g, w in zip(got, want):
        assert g.rstrip("\n").rsplit("\t", 1)[0] == w.rstrip("\n")
        assert g.rstrip("\n").rsplit("\t", 1)[1] == seq_of[w.split("\t")[1]].decode()
    # -C / -U echo the records; `-o -` prints nothing (classify.cpp:233-235); .gz output
    c, u, gz = tmp_path / "c.fq", tmp_path / "u.fq", tmp_path / "o.kraken.gz"
    r = subprocess.run(base + ["-M", "-C", str(c), "-U", str(u), "-o", "-", reads], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and r.stdout == ""
    n_c = sum(1 for l in open(os.path.join(G, "fastq.kraken")) if l.startswith("C"))
    assert open(c).read().count("\n+\n") == n_c and open(u).read().count("\n+\n") == len(ids) - n_c
    r = subprocess.run(base + ["-M", "-o", str(gz), reads], capture_output=True, text=True, env=env)
    import gzip
    assert gzip.open(gz, "rt").read() == open(os.path.join(G, "fastq.kraken")).read()
    # -M without input files is the page-cache warm-up idiom: a no-op that succeeds
    assert subprocess.run(base + ["-M"], capture_output=True, env=env).returncode == 0
    # unsupported modes fail loudly: -I (UID mapping) is outside the hot path (SURVEY.md §2)
    r = subprocess.run(base + ["-M", "-I", str(tmp_path / "uid.map"), reads], capture_output=True, text=True, env=env)
    assert r.returncode != 0 and "not supported" in r.stderr


@pytest.mark.parametrize("size", ["40K", "16K", "100K", pytest.param(None, id="shards")])
def test_cli_database_ranges(tmp_path, size):
    """-x with a database that must be split (process_file_with_db_chunk, classify.cpp:566-791): the database is
    staged range by range, every range looks the whole input up, the merged taxa are resolved in a final pass.
    Same Kraken output and report as the reference's `-x 40K` run, whatever the chunk size.  `shards`: the database
    sharded by minimizer range over two contexts on one device instead, whose ranges add up to the same .counts."""
    import shutil
    db = tmp_path / "db"
    db.mkdir()
    for f in ("database.kdb", "database.idx", "taxDB"):
        shutil.copy(os.path.join(G, f), db / f)                       # no database.kdb.counts: must be regenerated
    exe = build.build_classify()
    out, rep = tmp_path / "o.kraken", tmp_path / "o.report.tsv"
    cmd = [exe, "-d", str(db / "database.kdb"), "-i", str(db / "database.idx"), "-a", str(db / "taxDB"), "-t", "1",
           "-r", str(rep), "-o", str(out)] + (["-x", size] if size else ["-M"]) + [os.path.join(G, "reads.fa")]
    env = dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22),
               **({"KUQ_FORCE_CHUNKS": "1"} if size else {"KUQ_FORCE_SHARDS": "1", "KUQ_DEVICES": "0,0"}))
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    if size:
        assert "Database split into" in r.stderr and "split into 1 chunks" not in r.stderr
    else:
        assert "Database sharded over 2 GPUs by minimizer range" in r.stderr
    assert open(out).read() == open(os.path.join(G, "chunked.kraken")).read()
    assert _report_lines(rep) == _report_lines(os.path.join(G, "chunked.report.tsv"))
    assert open(db / "database.kdb.counts").read() == open(os.path.join(G, "database.kdb.counts")).read()


def test_cli_long_contigs_match_oracle(tmp_path, oracle):
    """multi-line FASTA contigs (hundreds of kb, > 32 distinct taxa): Kraken lines equal to the oracle's"""
    import numpy as np
    from krakenuniq_b200 import synth
    rng = np.random.default_rng(3)
    kdb = np.fromfile(os.path.join(G, "database.kdb"), np.uint8)
    idx = np.fromfile(os.path.join(G, "database.idx"), np.uint8)
    tax = synth.Taxonomy.read(os.path.join(G, "taxDB"))
    _, seqs = util.read_fasta(os.path.join(G, "reads.fa"))
    pool = [s for s in seqs if len(s) == 150 and b"N" not in s]
    contigs = [b"".join(pool[int(j)] for j in rng.integers(0, len(pool), n)) for n in (5, 400, 2500)]
    fa = tmp_path / "contigs.fa"
    with open(fa, "wb") as f:
        for i, c in enumerate(contigs):
            f.write(b">contig%d some description\n" % i)
            for a in range(0, len(c), 80):
                f.write(c[a:a + 80] + b"\n")
    db = oracle.open_db(kdb, idx)
    pm = oracle.parent_map(*tax.parent_map())
    run = oracle.run(db, pm, 500000, 0)
    bases, offs = synth.pack_reads(contigs)
    calls, codes, code_off = run.classify(bases, offs)
    want = util.kraken_lines([f"contig{i}" for i in range(3)], contigs, calls, codes, code_off)
    exe = build.build_classify()
    for threads in ("1", "6"):
        out = tmp_path / f"o{threads}.kraken"
        cmd = [exe, "-d", os.path.join(G, "database.kdb"), "-i", os.path.join(G, "database.idx"), "-a",
               os.path.join(G, "taxDB"), "-M", "-t", threads, "-o", str(out), str(fa)]
        r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22)))
        assert r.returncode == 0, r.stderr[-2000:]
        assert open(out).read() == want


@pytest.mark.parametrize("tag", ["ab", "ba", "ab_q2", "ba_q1"])
def test_cli_two_databases_first_hit(tmp_path, tag):
    """classify -d A -d B (both orders): the first database holding a k-mer decides, a stored taxon 0 included
    (classify.cpp:928-936); the report adds up the genome sizes of both .counts files (classify.cpp:262-285).
    `_q*`: the same with -q -m N (the read ends at its N-th hit, :943-944), golden files from the reference too."""
    M = os.path.join(util.ROOT, "tests", "golden", "multidb")
    a = ["-d", os.path.join(G, "database.kdb"), "-i", os.path.join(G, "database.idx")]
    b = ["-d", os.path.join(M, "db2.kdb"), "-i", os.path.join(M, "db2.idx")]
    exe = build.build_classify()
    out, rep = tmp_path / f"{tag}.kraken", tmp_path / f"{tag}.report.tsv"
    quick = {"ab_q2": ["-q", "-m", "2"], "ba_q1": ["-q", "-m", "1"]}.get(tag, [])     # quick mode over two databases
    cmd = [exe] + (a + b if tag.startswith("ab") else b + a) + ["-a", os.path.join(G, "taxDB"), "-t", "1", "-M", "-u", "20000"] + \
        quick + ["-r", str(rep), "-o", str(out), os.path.join(G, "reads.fa")]
    r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22)))
    assert r.returncode == 0, r.stderr[-2000:]
    assert open(out).read() == open(os.path.join(M, f"{tag}.kraken")).read()
    assert _report_lines(rep) == _report_lines(os.path.join(M, f"{tag}.report.tsv"))


@pytest.mark.parametrize("tag,extra,reads,env", [
    ("q1", ["-M", "-q"], "reads.fa", None),
    ("q3_u20000", ["-M", "-q", "-m", "3", "-u", "20000"], "reads.fa", None),
    ("q40", ["-M", "-q", "-m", "40"], "reads.fa", None),
    ("q2_crlf", ["-M", "-q", "-m", "2"], "reads_crlf_60.fa", None),
    ("q2_chunked", ["-x", "40K", "-q", "-m", "2"], "reads.fa", None),
    ("q2_chunked", ["-x", "40K", "-q", "-m", "2"], "reads.fa", {"KUQ_FORCE_CHUNKS": "1"}),
    # a database that has to be cut into ranges WITHOUT -x keeps the preloaded path's rule (reads end at the hit);
    # the sketches are global then, so only the Kraken lines are compared
    ("q3_u20000", ["-M", "-q", "-m", "3", "-u", "20000"], "reads.fa", {"KUQ_HBM_BUDGET": "40000"}),
])
def test_cli_quick_mode(tmp_path, tag, extra, reads, env):
    """classify -q [-m N] against the unmodified reference (tests/golden/quick, make_golden_quick.py):
    "Q:hits" lines, calls, and every report column — preloaded rule (classify.cpp:943-944,963-964) and -x rule
    (:701-702,705-721,737-738)."""
    Q = os.path.join(util.ROOT, "tests", "golden", "quick")
    out, rep, r = _run(tmp_path, tag, extra, reads, env)
    assert open(out).read() == open(os.path.join(Q, f"{tag}.kraken")).read()
    if not (env and "KUQ_HBM_BUDGET" in env):
        assert _report_lines(rep) == _report_lines(os.path.join(Q, f"{tag}.report.tsv"))
