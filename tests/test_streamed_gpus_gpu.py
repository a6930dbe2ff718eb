"""Databases streamed in minimizer ranges over several GPUs (`classify` when the databases fit neither one card nor the
cards together, or `-x` with KUQ_FORCE_CHUNKS): every GPU streams a contiguous group of each database's ranges and stores
its hits into the id buffer of the batch's owner; the owners resolve.  Several contexts on device 0 stand in for the GPUs
(KUQ_DEVICES=0,0 / 0,0,0); one case runs on two physical GPUs when there are two.  Every run must write what the golden
reference runs and the one-GPU streamed run write."""
import gzip
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from krakenuniq_b200 import binding, build, synth
from tests import paired, util

pytestmark = pytest.mark.gpu
G = util.GOLDEN
M = os.path.join(os.path.dirname(G), "multidb")
BASE_ENV = {"KUQ_SPARSE_SLOTS": str(1 << 22), "KUQ_TIMING": "1"}


def _devices(n):
    return ",".join(["0"] * n)


def _report_rows(path):
    rows = {}
    for line in open(path):
        if line.startswith("#") or line.startswith("%"):
            continue
        f = line.rstrip("\n").split("\t")
        rows[f[6]] = f
    return rows


def _setup(tmp_path, counts=True):
    for name, d in (("database", G), ("db2", M)):
        for ext in (".kdb", ".idx") + ((".kdb.counts",) if counts else ()):
            shutil.copyfile(os.path.join(d, name + ext), tmp_path / (name + ext))
    for f in ("taxDB", "reads.fa", "reads_300.fq"):
        shutil.copyfile(os.path.join(G, f), tmp_path / f)


def _run(tmp_path, args, env, tool="classify"):
    exe = os.path.join(os.path.dirname(build.build_classify()), tool)
    r = subprocess.run([exe] + args, cwd=tmp_path, capture_output=True, text=True, env=dict(os.environ, **BASE_ENV, **env))
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stderr


def _dbs(names):
    return sum((["-d", f"{d}.kdb", "-i", f"{d}.idx"] for d in names), []) + ["-a", "taxDB", "-t", "1"]


def _groups(stderr, n_gpu, n_db):
    """the ranges per GPU of every database, from the 'streamed over N GPUs' line"""
    what = "database" if n_db == 1 else f"{n_db} databases"
    m = re.search(rf"classify: {what} streamed over {n_gpu} GPUs: ranges per GPU ([\d/, ]+)\n", stderr)
    assert m, stderr[-2000:]
    groups = [[int(x) for x in part.split("/")] for part in m.group(1).split(", ")]
    assert len(groups) == n_db and all(len(g) == n_gpu for g in groups)
    return groups


def _owners(stderr):
    """batches owned per GPU in every round (KUQ_TIMING)"""
    return [[int(x) for x in re.findall(r"\((\d+) batches\)", line)]
            for line in stderr.splitlines() if line.startswith("[timing] streamed round")]


def _stats(stderr):
    lines = stderr.replace("\r", "\n").splitlines()
    return [l.split(" processed in")[0] for l in lines if " processed in " in l] + \
        [l for l in lines if l.startswith("  ") and "sequences" in l]


# ---- golden runs ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("budget", [None, "400000"])
@pytest.mark.parametrize("size", ["40K", "16K", "100K"])
@pytest.mark.parametrize("n_ctx", [2, 3])
def test_golden_chunked(tmp_path, n_ctx, size, budget):
    """-x with KUQ_FORCE_CHUNKS over 2 and 3 contexts: the reference's `-x 40K` Kraken lines and report, and a regenerated
    database.kdb.counts, whatever the chunk size.  Without a budget a round is one batch; KUQ_HBM_BUDGET=400000 makes
    rounds of several batches with several owners.  100K cuts the database into fewer ranges than 3 GPUs."""
    _setup(tmp_path, counts=False)
    env = {"KUQ_FORCE_CHUNKS": "1", "KUQ_DEVICES": _devices(n_ctx)}
    if budget:
        env["KUQ_HBM_BUDGET"] = budget
    err = _run(tmp_path, _dbs(["database"]) + ["-x", size, "-r", "o.report", "-o", "o.kraken", "reads.fa"], env)
    assert (tmp_path / "o.kraken").read_text() == open(os.path.join(G, "chunked.kraken")).read()
    assert _report_rows(tmp_path / "o.report") == _report_rows(os.path.join(G, "chunked.report.tsv"))
    assert (tmp_path / "database.kdb.counts").read_text() == open(os.path.join(G, "database.kdb.counts")).read()
    n = int(re.search(r"Database split into (\d+) chunks", err).group(1))
    groups = _groups(err, n_ctx, 1)[0]
    assert sum(groups) == n and n >= 2
    assert len(re.findall(r"database chunk \d+ of %d\n" % n, err.replace("\r", "\n"))) % n == 0
    if n < n_ctx:
        assert 0 in groups
    if budget:
        assert any(sum(1 for x in r if x) >= 2 for r in _owners(err)), _owners(err)
    one = tmp_path / "one"
    one.mkdir()
    _setup(one)
    err1 = _run(one, _dbs(["database"]) + ["-x", size, "-o", "o.kraken", "reads.fa"], {"KUQ_FORCE_CHUNKS": "1", "KUQ_DEVICES": "0"})
    assert f"Database split into {n} chunks" in err1 and "streamed over" not in err1


@pytest.mark.parametrize("tag", ["ab", "ba", "ab_q2", "ba_q1"])
@pytest.mark.parametrize("n_ctx", [2, 3])
def test_golden_two_databases(tmp_path, n_ctx, tag):
    """two databases that do not fit KUQ_HBM_BUDGET=200000 together, both orders, with -q -m: the reference's runs"""
    _setup(tmp_path)
    names = ["database", "db2"] if tag.startswith("ab") else ["db2", "database"]
    quick = {"ab_q2": ["-q", "-m", "2"], "ba_q1": ["-q", "-m", "1"]}.get(tag, [])
    err = _run(tmp_path, _dbs(names) + ["-M", "-u", "20000"] + quick + ["-r", "o.report", "-o", "o.kraken", "reads.fa"],
               {"KUQ_HBM_BUDGET": "200000", "KUQ_DEVICES": _devices(n_ctx)})
    assert (tmp_path / "o.kraken").read_text() == open(os.path.join(M, f"{tag}.kraken")).read()
    assert _report_rows(tmp_path / "o.report") == _report_rows(os.path.join(M, f"{tag}.report.tsv"))
    groups = _groups(err, n_ctx, 2)
    m = re.search(r"2 databases streamed: (\d+) rounds, ranges per database (\d+)/(\d+)", err)
    assert m and int(m.group(1)) >= 2
    assert [sum(g) for g in groups] == [int(m.group(2)), int(m.group(3))]


@pytest.mark.parametrize("tag", ["ab", "ba_q1"])
@pytest.mark.parametrize("n_ctx", [2, 3])
def test_two_databases_several_owners(tmp_path, n_ctx, tag):
    """-u 2000: rounds of several batches with different owners, so the second database's fill-empty lookups read words
    that other contexts stored.  The bytes of the one-context streamed run."""
    _setup(tmp_path)
    names = ["database", "db2"] if tag == "ab" else ["db2", "database"]
    args = _dbs(names) + ["-M", "-u", "2000"] + (["-q", "-m", "1"] if tag == "ba_q1" else [])
    out = {}
    for devices in ("0", _devices(n_ctx)):
        err = _run(tmp_path, args + ["-r", f"{devices}.report", "-o", f"{devices}.kraken", "reads.fa"],
                   {"KUQ_HBM_BUDGET": "300000", "KUQ_DEVICES": devices})
        out[devices] = ((tmp_path / f"{devices}.kraken").read_bytes(), (tmp_path / f"{devices}.report").read_bytes(), _stats(err))
        if devices != "0":
            owners = _owners(err)
            assert owners and any(sum(1 for x in r if x) >= 2 for r in owners), owners
    assert out["0"] == out[_devices(n_ctx)]


def test_classify_exact(tmp_path):
    """classifyExact -x streamed over 2 contexts: the report of the one-context streamed run and of the reference"""
    _setup(tmp_path)
    reports = {}
    for devices in ("0", "0,0"):
        _run(tmp_path, _dbs(["database"]) + ["-x", "40K", "-r", f"{devices}.report", "-o", f"{devices}.kraken", "reads.fa"],
             {"KUQ_FORCE_CHUNKS": "1", "KUQ_HBM_BUDGET": "400000", "KUQ_DEVICES": devices}, tool="classifyExact")
        reports[devices] = (tmp_path / f"{devices}.report").read_bytes()
        assert _report_rows(tmp_path / f"{devices}.report") == _report_rows(os.path.join(G, "exact.report.tsv"))
        assert (tmp_path / f"{devices}.kraken").read_text() == open(os.path.join(G, "preload.kraken")).read()
    assert reports["0"] == reports["0,0"]


# ---- features that live in the ingest or the resolve half --------------------------------------------------------------
LAYOUTS = {"x": (["database"], ["-x", "40K"], {"KUQ_FORCE_CHUNKS": "1", "KUQ_HBM_BUDGET": "400000"}),
           "two_db": (["database", "db2"], ["-M", "-u", "2000"], {"KUQ_HBM_BUDGET": "300000"})}


def _mates(tmp_path):
    ids, seqs = util.read_fastq(os.path.join(G, "reads_300.fq"))
    pairs = paired.split_pairs(seqs, np.random.default_rng(5))
    d1 = paired.fastq_bytes([(f"{i}/1".encode(), a) for i, (a, _) in zip(ids, pairs)])
    d2 = paired.fastq_bytes([(f"{i}/2".encode(), b) for i, (_, b) in zip(ids, pairs)])
    (tmp_path / "m1.fq").write_bytes(d1)
    (tmp_path / "m2.fq").write_bytes(d2)
    (tmp_path / "m1.fq.gz").write_bytes(gzip.compress(d1))
    (tmp_path / "m2.fq.gz").write_bytes(gzip.compress(d2))


FEATURES = {
    "paired": lambda p: ["-o", f"{p}.kraken", "-r", f"{p}.report", "--paired", "m1.fq", "m2.fq"],
    "paired_gzip": lambda p: ["-o", f"{p}.kraken", "-r", f"{p}.report", "--paired", "m1.fq.gz", "m2.fq.gz"],
    "threshold": lambda p: ["-o", f"{p}.kraken", "-r", f"{p}.report", "--threshold", "0.5", "reads.fa"],
    "extract": lambda p: ["-o", f"{p}.kraken", "-r", f"{p}.report", "--extract", "100,107", "--extract-subtree",
                          "--extract-out", f"{p}.extract", "reads_300.fq"],
    "classified_out": lambda p: ["-o", f"{p}.kraken", "-C", f"{p}.C", "-U", f"{p}.U", "reads.fa"],
    "sheet": lambda p: ["--sample-sheet", f"{p}.tsv"],
}


@pytest.mark.parametrize("feature", list(FEATURES))
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_features_through_the_layout(tmp_path, layout, feature):
    """every output file byte-identical to the same command on one context"""
    _setup(tmp_path)
    _mates(tmp_path)
    names, flags, env = LAYOUTS[layout]
    files = {}
    for devices in ("0", "0,0"):
        p = devices.replace(",", "_")
        if feature == "sheet":
            rows = [("fa", "reads.fa"), ("fq", "reads_300.fq")]
            (tmp_path / f"{p}.tsv").write_text("name\tinput\toutput\treport\n" + "".join(
                f"{n}\t{i}\t{p}.{n}.kraken\t{p}.{n}.report\n" for n, i in rows))
        err = _run(tmp_path, _dbs(names) + flags + FEATURES[feature](p), dict(env, KUQ_DEVICES=devices))
        if devices != "0":
            assert "streamed over 2 GPUs" in err
        files[devices] = {f.name[len(p) + 1:]: f.read_bytes() for f in tmp_path.iterdir()
                          if f.name.startswith(p + ".") and not f.name.endswith(".tsv")}
        files[devices]["stats"] = _stats(err)
    assert len(files["0"]) >= 2 and all(files["0"].values()), sorted(files["0"])
    assert files["0"] == files["0,0"]


# ---- two physical GPUs ------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_physical_gpus(tmp_path):
    """KUQ_DEVICES=0,1: the hits travel between the cards over the peer link (contexts on one card share its L2)"""
    _setup(tmp_path, counts=False)
    err = _run(tmp_path, _dbs(["database"]) + ["-x", "16K", "-r", "x.report", "-o", "x.kraken", "reads.fa"],
               {"KUQ_FORCE_CHUNKS": "1", "KUQ_HBM_BUDGET": "400000", "KUQ_DEVICES": "0,1"})
    _groups(err, 2, 1)
    assert (tmp_path / "x.kraken").read_text() == open(os.path.join(G, "chunked.kraken")).read()
    assert _report_rows(tmp_path / "x.report") == _report_rows(os.path.join(G, "chunked.report.tsv"))
    for tag, names in (("ab", ["database", "db2"]), ("ba", ["db2", "database"])):
        err = _run(tmp_path, _dbs(names) + ["-M", "-u", "20000", "-r", f"{tag}.report", "-o", f"{tag}.kraken", "reads.fa"],
                   {"KUQ_HBM_BUDGET": "200000", "KUQ_DEVICES": "0,1"})
        _groups(err, 2, 2)
        assert (tmp_path / f"{tag}.kraken").read_text() == open(os.path.join(M, f"{tag}.kraken")).read()
        assert _report_rows(tmp_path / f"{tag}.report") == _report_rows(os.path.join(M, f"{tag}.report.tsv"))


# ---- the C ABI recipe ---------------------------------------------------------------------------------------------------
def test_cabi_contexts_stream_into_one_owner(oracle):
    """kuq_stream_* on several contexts: each streams its half of every database's ranges and looks the batch up into
    the owner's id buffer (a pointer of another context); the first database stores hits, the second fills what is
    empty (KUQ_LOOKUP_FILL_EMPTY) after a host barrier; the owner resolves with the per-work-unit rule.  Calls, hit lists
    and counters equal the oracle's and those of one context streaming every range."""
    import ctypes
    from tests.test_multi_db_gpu import _check_reads, _oracle, _runs_to_codes, _same_counts, _workload
    k, unit = 31, 3000
    tax, dbs, seqs = _workload(77, k, [(9, 2), (9, 2)], n_reads=4000)
    calls, codes, code_off, want, _, _ = _oracle(oracle, tax, dbs, seqs, unit)
    bases, offs = synth.pack_reads(seqs)
    units = synth.work_unit_ids(offs, unit)[0].astype(np.uint32)
    universe = np.unique(np.concatenate([synth.parse_kdb(kdb)[2] for kdb, _ in dbs]))
    n, total = len(offs) - 1, int(offs[-1])
    dev = "cuda:0"
    d_bases = torch.from_numpy(np.concatenate([bases, np.full(64, ord("N"), np.uint8)])).to(dev)
    d_offs = torch.from_numpy(np.concatenate([offs, offs[-1:], offs[-1:]]).astype(np.int64)).to(dev)
    d_units = torch.from_numpy(units.view(np.int32)).to(dev)

    def run(n_ctx):
        ctxs = [binding.Classifier(device=0, n_slots=2, max_reads=1 << 15, max_bases=8 << 20, work_unit_size=unit,
                                   hll_mode=binding.HLL_PRELOAD, sparse_set_slots=1 << 22) for _ in range(n_ctx)]
        for c in ctxs:
            c.set_taxonomy(*tax.parent_map())
            c.set_db_taxid_universe(universe)
            c.mark_zero_hits(True)
        owner, L = ctxs[0], ctxs[0].L
        ids = owner.device_alloc((total + 64) * 4)
        owner.device_memset(0, ids, 0, (total + 64) * 4)
        owner.sync(0)
        pinned = []
        for d, (kdb, idx) in enumerate(dbs):
            _, keys, _ = synth.parse_kdb(kdb)
            nt, n_bins = int(idx[7]), 1 << (2 * int(idx[7]))
            idx_off = np.frombuffer(idx[8:].tobytes(), np.uint64)
            cuts = [int(np.searchsorted(idx_off, idx_off[-1] * r // 4)) for r in range(5)]
            cuts[0], cuts[-1] = 0, n_bins
            ranges = [(cuts[r], cuts[r + 1]) for r in range(4) if idx_off[cuts[r + 1]] > idx_off[cuts[r]]]
            rec = kdb[kdb.size - 12 * len(keys):]
            h_rec, h_off = L.kuq_host_alloc(rec.size + 16), L.kuq_host_alloc(idx_off.size * 8)
            ctypes.memmove(h_rec, rec.ctypes.data, rec.size)
            ctypes.memmove(h_off, idx_off.ctypes.data, idx_off.size * 8)
            pinned += [h_rec, h_off]
            max_rec = max(int(idx_off[b] - idx_off[a]) for a, b in ranges)
            max_bins = max(b - a for a, b in ranges)
            for g, c in enumerate(ctxs):
                mine = ranges[len(ranges) * g // n_ctx:len(ranges) * (g + 1) // n_ctx]
                c.stream_open(k, nt, 2, max_rec, max_bins)

                def load(buf, rg):
                    a, b = int(idx_off[rg[0]]), int(idx_off[rg[1]])
                    c.stream_load(buf, h_rec + 12 * a, b - a, h_off + 8 * rg[0], rg[0], rg[1])
                load(0, mine[0])
                for j, rg in enumerate(mine):
                    c.stream_use(j & 1)
                    if j + 1 < len(mine):
                        load((j + 1) & 1, mine[j + 1])
                    c.lookup_device(j & 1, d_bases.data_ptr(), d_offs.data_ptr(), n, total, ids,
                                    only_hits=1 if d == 0 else binding.LOOKUP_FILL_EMPTY)
            for c in ctxs:                                   # host barrier before the next database reads the buffer
                c.sync(0)
                c.sync(1)
                c.stream_check()
        owner.resolve_device(0, d_bases.data_ptr(), d_offs.data_ptr(), n, total, ids, d_units.data_ptr())
        res = owner.collect_device(0, offs)
        got = (res["call"].copy(), [_runs_to_codes(res, i) for i in range(n)])
        for c in ctxs:
            c.finish()
        counts = owner.counts()
        owner.device_free(ids)
        for p in pinned:
            L.kuq_host_free(p)
        for c in ctxs:
            c.close()
        return got, counts

    (one_calls, one_codes), one_counts = run(1)
    (two_calls, two_codes), two_counts = run(2)
    _check_reads(two_calls, two_codes, calls, codes, code_off)
    _same_counts(two_counts, want)
    _check_reads(one_calls, one_codes, calls, codes, code_off)
    _same_counts(one_counts, want)
