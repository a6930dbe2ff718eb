"""Several databases on the GPU (`classify -d A -d B`, classify.cpp:928-936): every k-mer takes the value of the first
database that holds it, a stored taxon 0 included.  Resident: all databases staged on every device
(kuq_stage_db_append), one in-order lookup per run of databases with equal (nt, index type).  Streamed: rounds of reads
in HBM, each database's minimizer ranges through two range buffers, later databases filling only unanswered windows.
Checked against the reference's golden runs and against the oracle."""
import os
import re
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import binding, build, synth
from tests import util

pytestmark = pytest.mark.gpu
G = util.GOLDEN
M = os.path.join(util.ROOT, "tests", "golden", "multidb")
ENV = dict(os.environ, KUQ_SPARSE_SLOTS=str(1 << 22))


def _report_rows(path):
    rows = {}
    for line in open(path):
        if line.startswith("#") or line.startswith("%"):
            continue
        f = line.rstrip("\n").split("\t")
        rows[f[6]] = f
    return rows


def _cli(exe, dbs, taxdb, reads, out_dir, extra=(), env=None):
    out, rep = os.path.join(out_dir, "o.kraken"), os.path.join(out_dir, "o.report.tsv")
    cmd = [exe]
    for kdb, idx in dbs:
        cmd += ["-d", kdb, "-i", idx]
    cmd += ["-a", taxdb, "-t", "1", "-M"] + list(extra) + ["-r", rep, "-o", out, reads]
    r = subprocess.run(cmd, capture_output=True, text=True, env=dict(ENV, **(env or {})))
    assert r.returncode == 0, r.stderr[-3000:]
    return open(out).read(), _report_rows(rep), r.stderr


def _streamed_shape(stderr):
    m = re.search(r"(\d+) databases streamed: (\d+) rounds, ranges per database ([\d/]+)", stderr)
    assert m, stderr[-2000:]
    return int(m.group(2)), [int(x) for x in m.group(3).split("/")]


# ---- the reference's golden runs, in every mode -------------------------------------------------------------------
MODES = {"resident": {}, "two_contexts": {"KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"},
         # A and B take ~150 kB each in HBM: ranges of at most 50 kB, and rounds of about one 20 kbp work unit
         "streamed": {"KUQ_HBM_BUDGET": "200000"}}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("tag", ["ab", "ba", "ab_q2", "ba_q1"])
def test_golden_two_databases(tmp_path, tag, mode):
    a = (os.path.join(G, "database.kdb"), os.path.join(G, "database.idx"))
    b = (os.path.join(M, "db2.kdb"), os.path.join(M, "db2.idx"))
    quick = {"ab_q2": ["-q", "-m", "2"], "ba_q1": ["-q", "-m", "1"]}.get(tag, [])
    kraken, rows, err = _cli(build.build_classify(), [a, b] if tag.startswith("ab") else [b, a], os.path.join(G, "taxDB"),
                             os.path.join(G, "reads.fa"), str(tmp_path), ["-u", "20000"] + quick, MODES[mode])
    assert kraken == open(os.path.join(M, f"{tag}.kraken")).read()
    assert rows == _report_rows(os.path.join(M, f"{tag}.report.tsv"))
    if mode == "streamed":
        rounds, ranges = _streamed_shape(err)
        assert rounds >= 2 and min(ranges) >= 2, (rounds, ranges)
    else:
        n_gpu = 2 if mode == "two_contexts" else 1
        assert f"2 databases resident on {n_gpu} GPU(s)" in err, err[-2000:]


# ---- synthetic databases against the oracle -----------------------------------------------------------------------
def _workload(seed, k, shapes, n_reads=20000):
    """len(shapes) databases over the k-mers of 12 genomes: each holds a random 60 % of them, a third of those under a
    conflicting species, a few with value 0.  shapes = [(nt, index type), ...]; a negative nt = a database without
    records (minimizer length -nt)."""
    rng = np.random.default_rng(seed)
    tax = synth.make_taxonomy(12, 3)
    sp = synth.species_ids(tax)
    genomes = synth.random_genomes(rng, 12, 2500, 0.25)
    km, tx = synth.label_kmers(genomes, sp, tax, k)
    dbs = []
    for nt, it in shapes:
        if nt < 0:
            dbs.append(synth.build_db_images(np.zeros(0, np.uint64), np.zeros(0, np.uint32), k, -nt, it))
            continue
        keep = rng.random(len(km)) < 0.6
        t = tx[keep].copy()
        r = rng.random(len(t))
        t[r < 0.33] = np.asarray(sp, np.uint32)[rng.integers(0, len(sp), int((r < 0.33).sum()))]
        t[r > 0.96] = 0
        dbs.append(synth.build_db_images(km[keep], t, k, nt, it))
    bases, offs = synth.sample_reads(rng, genomes, n_reads, 150, 0.01, 0.1, 0.2)
    g0 = synth.decode(genomes[0]).tobytes()
    extra = [b"", g0[:k - 1], g0[:k], g0[7:7 + k] + b"N" + g0[300:300 + k], g0[900:1000].lower() + g0[1000:1100]]
    seqs = [bases[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)] + extra
    return tax, dbs, seqs


def _oracle(oracle, tax, dbs, seqs, unit, quick=0, exact=False):
    odbs = [oracle.open_db(kdb, idx) for kdb, idx in dbs]
    run = oracle.run(odbs[0], oracle.parent_map(*tax.parent_map()), unit, 0)
    for d in odbs[1:]:
        run.add_db(d)
    if quick:
        run.set_quick(quick)
    if exact:
        run.set_exact()
    calls, codes, code_off = run.classify(*synth.pack_reads(seqs))
    run.finish()
    return calls, codes, code_off, run.counts(), odbs, run


def _classifier(tax, dbs, unit, **kw):
    clf = binding.Classifier(max_reads=1 << 15, max_bases=8 << 20, work_unit_size=unit, sparse_set_slots=1 << 22, **kw)
    clf.stage_db(*dbs[0])
    for d in dbs[1:]:
        clf.stage_db_append(*d)
    clf.set_taxonomy(*tax.parent_map())
    return clf


def _runs_to_codes(res, i):
    out = []
    for code, cnt in binding.decode_runs(res, i):
        out += [code] * cnt
    return np.array(out, np.uint32)


def _same_counts(got, want):
    for key in ("taxid", "n_reads", "n_kmers", "unique"):
        assert np.array_equal(got[key], want[key]), (key, got[key], want[key])


def _classify_two_slots(clf, seqs, batch=4000):
    """kuq_submit_batch on two slots, two batches in flight; returns calls and per-read hit codes"""
    calls, codes, keep = [], [], []
    parts = [seqs[a:a + batch] for a in range(0, len(seqs), batch)]
    for j in range(0, len(parts), 2):
        inflight = []
        for s, part in enumerate(parts[j:j + 2]):
            bases, offs = synth.pack_reads(part)
            bases = bases if bases.size else np.zeros(1, np.uint8)
            keep.append((bases, offs))
            clf.submit(s, bases.ctypes.data, offs)
            inflight.append((s, offs))
        for s, offs in inflight:
            res = clf.wait(s, offs, copy=True)
            calls.append(res["call"])
            codes += [_runs_to_codes(res, i) for i in range(len(offs) - 1)]
    return np.concatenate(calls), codes


def _check_reads(calls, codes, want_calls, want_codes, code_off):
    assert np.array_equal(calls, want_calls)
    for i in range(len(want_calls)):
        assert np.array_equal(codes[i], want_codes[int(code_off[i]):int(code_off[i + 1])]), f"read {i}"


def _first_hit_codes(clf, odbs, seqs, k, n_check=300):
    """kuq_lookup_batch codes of the first n_check reads against per-window queries of the oracle databases in order"""
    bases, offs = synth.pack_reads(seqs[:n_check])
    got, nwin = clf.lookup(bases, offs)
    raw = clf.dense_taxids()
    o = odbs[0].o
    for i, s in enumerate(seqs[:n_check]):
        kmers, amb = o.scan(s, k)
        want = []
        for km, a in zip(kmers.tolist(), amb.tolist()):
            if a:
                want.append(util.AMBIG)
                continue
            c = o.canonical(km, k)
            v = 0
            for d in odbs:
                found, t = d.query(c)
                if found:
                    v = t if t else binding.CODE_FOUND_ZERO
                    break
            want.append(v)
        g = got[int(offs[i]):int(offs[i]) + int(nwin[i])]
        g = np.where((g == util.AMBIG) | (g == binding.CODE_FOUND_ZERO) | (g == 0), g, raw[np.minimum(g, len(raw) - 1)])
        assert np.array_equal(g, np.array(want, np.uint32)), f"read {i}"


@pytest.mark.parametrize("k,shapes", [
    (31, [(10, 2), (8, 1), (10, 2), (6, 2)]),     # equal parameters not contiguous: 4 runs
    (21, [(9, 2), (7, 2), (9, 1)]),               # widened records
])
def test_cabi_matches_oracle(oracle, k, shapes):
    tax, dbs, seqs = _workload(100 + k, k, shapes)
    unit = 30000
    calls, codes, code_off, want, odbs, _ = _oracle(oracle, tax, dbs, seqs, unit)
    clf = _classifier(tax, dbs, unit, hll_mode=binding.HLL_PRELOAD)
    got_calls, got_codes = _classify_two_slots(clf, seqs)
    clf.finish()
    _check_reads(got_calls, got_codes, calls, codes, code_off)
    _same_counts(clf.counts(), want)
    _first_hit_codes(clf, odbs, seqs, k)


def _window_mask(offs, nwin, total):
    m = np.zeros(total, bool)
    for a, n in zip(offs[:-1].tolist(), nwin.tolist()):
        m[a:a + n] = True
    return m


def test_each_database_fetches_only_unanswered_windows(oracle):
    """probe statistics: database i fetches exactly the non-ambiguous windows no earlier database answered"""
    tax, dbs, seqs = _workload(7, 31, [(10, 2), (8, 1), (10, 2), (6, 2)], n_reads=3000)
    bases, offs = synth.pack_reads(seqs)
    fetched, open_windows = [], None
    for n in range(1, len(dbs) + 1):
        clf = _classifier(tax, dbs[:n], 500000, hll_mode=binding.HLL_PRELOAD)
        clf.set_stats(True)
        clf.mark_zero_hits(True)                    # one database: a stored zero also ends the search
        codes, nwin = clf.lookup(bases, offs)
        fetched.append(clf.slot_stats(0)[0])
        win = _window_mask(offs, nwin, len(codes))
        if open_windows is not None:
            assert fetched[-1] - (fetched[-2] if n > 1 else 0) == open_windows, n
        open_windows = int((win & (codes == 0)).sum())
        if n == 1:
            assert fetched[0] == int((win & (codes != util.AMBIG)).sum())
        clf.close()


def test_eleven_tiny_databases_with_an_empty_one(oracle):
    """11 databases of equal parameters, the sixth without records: one run of more than MAX_DBS databases, which
    takes two lookup launches after one k_scan, the second filling only the windows the first 8 databases left open"""
    shapes = [(7, 2)] * 5 + [(-7, 2)] + [(7, 2)] * 5
    tax, dbs, seqs = _workload(10, 31, shapes, n_reads=2000)
    calls, codes, code_off, want, odbs, _ = _oracle(oracle, tax, dbs, seqs, 20000)
    clf = _classifier(tax, dbs, 20000, hll_mode=binding.HLL_PRELOAD)
    got_calls, got_codes = _classify_two_slots(clf, seqs, batch=800)      # whole work units of 20 kbp per batch
    clf.finish()
    _check_reads(got_calls, got_codes, calls, codes, code_off)
    _same_counts(clf.counts(), want)
    _first_hit_codes(clf, odbs, seqs, 31, n_check=100)
    # kernels of one lookup call: k_scan + 2 lookup launches; fetches: every database asked until the first holds the key
    sub = seqs[:300]
    clf.set_stats(True)
    before = clf.launch_count()
    clf.lookup(*synth.pack_reads(sub))
    assert clf.launch_count() - before == 3
    o = odbs[0].o
    asked = 0
    for s in sub:
        kmers, amb = o.scan(s, 31)
        for km, a in zip(kmers.tolist(), amb.tolist()):
            if a:
                continue
            c = o.canonical(km, 31)
            n = len(odbs)
            for i, d in enumerate(odbs):
                if d.query(c)[0]:
                    n = i + 1
                    break
            asked += n
    assert clf.slot_stats(0)[0] == asked


def test_stage_db_after_appends_and_append_errors(oracle):
    tax, dbs, seqs = _workload(11, 31, [(8, 2), (8, 1)], n_reads=1500)
    calls, codes, code_off, want, _, _ = _oracle(oracle, tax, dbs[:1], seqs, 30000)
    clf = _classifier(tax, dbs, 30000, hll_mode=binding.HLL_PRELOAD)
    clf.stage_db(*dbs[0])                          # drops the appended database: one-database context again
    got_calls, got_codes = _classify_two_slots(clf, seqs, batch=600)      # whole work units of 30 kbp per batch
    clf.finish()
    _check_reads(got_calls, got_codes, calls, codes, code_off)
    _same_counts(clf.counts(), want)
    _, dbs21, _ = _workload(12, 21, [(8, 2)], n_reads=10)
    with pytest.raises(binding.KuqError) as e:
        clf.stage_db_append(*dbs21[0])
    assert "differ in k" in str(e.value)


def test_merge_of_two_multi_database_contexts(oracle):
    """kuq_merge_into of two contexts with the same databases equals one context over all reads"""
    tax, dbs, seqs = _workload(13, 31, [(9, 2), (7, 1), (9, 2)], n_reads=4000)
    unit = 30000
    calls, codes, code_off, want, _, _ = _oracle(oracle, tax, dbs, seqs, unit)
    cut = 2000                                      # at a work-unit boundary: 200 reads of 150 bp per unit
    ctxs = [_classifier(tax, dbs, unit, hll_mode=binding.HLL_PRELOAD) for _ in range(2)]
    units = synth.work_unit_ids(synth.pack_reads(seqs)[1], unit)[0]
    out_calls = []
    for c, part, u in ((ctxs[0], seqs[:cut], units[:cut]), (ctxs[1], seqs[cut:], units[cut:])):
        res = c.classify(*synth.pack_reads(part), unit_id=u)
        out_calls.append(res["call"])
        c.finish()
    ctxs[0].merge_from(ctxs[1])
    assert np.array_equal(np.concatenate(out_calls), calls)
    _same_counts(ctxs[0].counts(), want)


def _report_matches_oracle(path, tax, cnt, run):
    """every report row: the taxon's own reads, and the clade's reads and unique k-mers, equal the oracle's"""
    rep = util.parse_report(path)
    members = util.clade_members(tax.rows, cnt["taxid"])
    by_tax = {int(t): i for i, t in enumerate(cnt["taxid"])}
    assert rep
    for taxid, row in rep.items():
        i = by_tax.get(taxid)
        assert row["taxReads"] == (int(cnt["n_reads"][i]) if i is not None else 0), (taxid, row)
        u, r, _ = run.clade(members[taxid])
        assert (row["reads"], row["kmers"]) == (r, u), (taxid, row, r, u)


def _write_inputs(d, tax, dbs, seqs, crlf_every=7):
    """database files, taxDB and a multi-line FASTA, some records with CRLF line ends"""
    paths = []
    for i, (kdb, idx) in enumerate(dbs):
        kp, ip = str(d / f"db{i}.kdb"), str(d / f"db{i}.idx")
        kdb.tofile(kp)
        idx.tofile(ip)
        paths.append((kp, ip))
    tax.write(str(d / "taxDB"))
    with open(d / "reads.fa", "wb") as f:
        for i, s in enumerate(seqs):
            nl = b"\r\n" if i % crlf_every == 0 else b"\n"
            f.write(b">r%d x\n" % i + nl.join(s[j:j + 60] for j in range(0, len(s), 60)) + nl)
    return paths


@pytest.mark.parametrize("exe_name,quick", [("classify", 0), ("classify", 2), ("classifyExact", 0)])
def test_cli_resident_and_streamed_match_oracle(oracle, tmp_path, exe_name, quick):
    """3 databases (nt 9 / 7 / 9, both index types, stored zeros), CRLF multi-line FASTA: both modes give the oracle's
    Kraken lines and equal reports.  The streamed budget is below the first database alone (which the parent commit
    refused) but above the others."""
    tax, dbs, seqs = _workload(21, 31, [(9, 2), (7, 1), (9, 2)], n_reads=20000)
    paths = _write_inputs(tmp_path, tax, dbs, seqs)
    ids, rseqs = util.read_fasta(str(tmp_path / "reads.fa"))
    unit = 30000
    calls, codes, code_off, cnt, _, run = _oracle(oracle, tax, dbs, rseqs, unit, quick=quick, exact=exe_name == "classifyExact")
    want = util.kraken_lines(ids, rseqs, calls, codes, code_off)
    exe = os.path.join(os.path.dirname(build.build_classify()), exe_name)
    extra = ["-u", str(unit)] + (["-q", "-m", str(quick)] if quick else [])
    hbm = [kdb.size + idx.size for kdb, idx in dbs]
    budget = str(int(max(hbm) * 0.9))
    got = {}
    for mode, env in (("resident", {}), ("streamed", {"KUQ_HBM_BUDGET": budget})):
        out = tmp_path / mode
        out.mkdir()
        kraken, rows, err = _cli(exe, paths, str(tmp_path / "taxDB"), str(tmp_path / "reads.fa"), str(out), extra, env)
        if not quick:
            assert kraken == want, mode
        _report_matches_oracle(str(out / "o.report.tsv"), tax, cnt, run)
        got[mode] = (kraken, rows)
        if mode == "streamed":
            rounds, ranges = _streamed_shape(err)
            assert rounds >= 2 and max(ranges) >= 2, (rounds, ranges)
        else:
            assert "3 databases resident on" in err
    assert got["resident"] == got["streamed"]
    if quick:
        calls_cli = [int(l.split("\t")[2]) for l in got["resident"][0].splitlines()]
        assert calls_cli == [int(c) for c in calls]


def test_cli_counts_files_of_several_databases(tmp_path):
    """missing .counts files are written per database in both modes, equal to the reference's"""
    import shutil
    for mode, env in (("resident", {}), ("streamed", {"KUQ_HBM_BUDGET": "200000"})):
        d = tmp_path / mode
        d.mkdir()
        for f in ("database.kdb", "database.idx"):
            shutil.copy(os.path.join(G, f), d / f)
        for f in ("db2.kdb", "db2.idx"):
            shutil.copy(os.path.join(M, f), d / f)
        _cli(build.build_classify(), [(str(d / "database.kdb"), str(d / "database.idx")), (str(d / "db2.kdb"), str(d / "db2.idx"))],
             os.path.join(G, "taxDB"), os.path.join(G, "reads.fa"), str(d), ["-u", "20000"], env)
        assert open(d / "database.kdb.counts").read() == open(os.path.join(G, "database.kdb.counts")).read(), mode
        assert open(d / "db2.kdb.counts").read() == open(os.path.join(M, "db2.kdb.counts.golden")).read(), mode
