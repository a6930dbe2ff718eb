"""db_sort and set_lcas for databases larger than the device: both work in minimizer-range passes under a byte budget
(KUQ_DB_SORT_BUDGET, KUQ_SET_LCAS_BUDGET) and must write the bytes of the one-pass run.

- kuq_db_sort_budget at budgets forcing 2, several and the fewest-bytes passes, for 12-, 10- and 8-byte records, against
  the one-pass output and the oracle; the pass count against the planner; empty input, repeated keys, a budget below
  one bin.
- the set_lcas executable with at least 3 ranges against the same command at the default budget: the golden-style
  library (-x -c, then -TR and -T), the -a -A -T library, a pipe, the -f file map, k = 21, a missing k-mer without -x.
- the C ABI range by range: the whole-database image and missing count.
- kmer_set, db_sort and set_lcas, each in several passes, rebuild the golden database."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import binding, build, synth
from tests import taxid_cases, util
from tests import test_kmer_set_gpu as kmer_set_tests

pytestmark = pytest.mark.gpu

RESERVE = 1 << 18          # kuq_dbbuild.cu: budget kept back from the plan of the per-range sorts
PASS_C_REC = 64            # kuq_dbbuild.cu: planned device bytes per record of a range besides its two copies


def plan_ranges(offsets, budget, rec_bytes):
    """kuq_ranges.h restated: greedy ranges [lo, hi) of bins whose (hi - lo + 1) * 8 + records * rec_bytes + 8 bytes
    fit the budget; ranges without records left out; None when one bin does not fit"""
    offsets = [int(x) for x in offsets]
    n_bins, ranges, first = len(offsets) - 1, [], 0

    def fits(end):
        return (end - first + 1) * 8 + (offsets[end] - offsets[first]) * rec_bytes + 8 <= budget
    while first < n_bins:
        if not fits(first + 1):
            return None
        lo, hi = first + 1, n_bins
        while lo < hi:
            mid = lo + (hi - lo + 1) // 2
            lo, hi = (mid, hi) if fits(mid) else (lo, mid - 1)
        if offsets[lo] > offsets[first]:
            ranges.append((first, lo))
        first = lo
    return ranges


def _offsets(idx):
    return np.frombuffer(idx[8:].tobytes(), np.uint64)


@pytest.fixture(scope="module")
def tools():
    db_sort, set_lcas = build.build_dbtools()
    return build.KMER_SET, db_sort, set_lcas


# ---- 1. kuq_db_sort_budget -------------------------------------------------------------------------------------------
def _jdb(k, n, seed, repeats=0):
    rng = np.random.default_rng(seed)
    keys = np.unique(rng.integers(0, 1 << (2 * k), n, dtype=np.uint64))
    if repeats:
        keys = np.concatenate([keys, rng.choice(keys, repeats)])
    rng.shuffle(keys)
    vals = rng.integers(0, 1 << 20, len(keys)).astype(np.uint32)
    return np.concatenate([synth.kdb_header(k, len(keys)), synth.pack_records(keys, vals, k)])


def _budgets(idx, pair):
    """budgets for about 2 and 6 ranges and the smallest workable one (just above the largest bin), each at least
    the index plus the reserve that the histogram pass needs"""
    off = _offsets(idx)
    n, n_bins = int(off[-1]), len(off) - 1
    rec = 2 * pair + PASS_C_REC
    floor = 8 * (n_bins + 1) + RESERVE + 4096
    biggest = int(np.diff(off.astype(np.int64)).max())
    return {"two": max(floor, RESERVE + (n * rec + 8 * n_bins) // 2 + 64),
            "several": max(floor, RESERVE + (n * rec + 8 * n_bins) // 6 + 64),
            "smallest": max(floor, RESERVE + 16 + biggest * rec + 8)}


@pytest.mark.parametrize("k,nt,zero", [(31, 5, True), (31, 8, False), (31, 11, True), (21, 5, False), (21, 8, True),
                                       (21, 11, False), (15, 5, True), (15, 8, False), (15, 11, True)])
def test_db_sort_in_passes_matches_one_pass_and_oracle(oracle, k, nt, zero):
    # at nt = 11 the histogram pass holds the 32 MiB index whole: a million records keep the records the larger part
    jdb = _jdb(k, 1000000 if nt == 11 else 200000, 100 * k + nt)
    pair = (2 * k + 7) // 8 + 4
    one_kdb, one_idx, one_passes = binding.db_sort(jdb, nt, zero, with_passes=True)
    assert one_passes == 1
    want_kdb, want_idx = oracle.db_sort(jdb, nt, zero)
    assert np.array_equal(one_idx, want_idx) and np.array_equal(one_kdb, want_kdb[:one_kdb.size])
    seen = set()
    for name, budget in _budgets(one_idx, pair).items():
        plan = plan_ranges(_offsets(one_idx), budget - RESERVE, 2 * pair + PASS_C_REC)
        kdb, idx, passes = binding.db_sort(jdb, nt, zero, budget=budget, with_passes=True)
        assert passes == len(plan) and passes >= 2, (name, budget, passes, len(plan))
        assert np.array_equal(idx, one_idx), name
        assert np.array_equal(kdb, one_kdb), name
        seen.add(passes)
    assert max(seen) > 2


def test_db_sort_in_passes_keeps_repeated_keys_in_order():
    """keys that occur more than once come out in input order, as from the one-pass sort (stable by key, then bin)"""
    jdb = _jdb(31, 100000, 3, repeats=30000)
    one_kdb, one_idx = binding.db_sort(jdb, 6, False)
    for budget in _budgets(one_idx, 12).values():
        kdb, idx, passes = binding.db_sort(jdb, 6, False, budget=budget, with_passes=True)
        assert passes >= 2
        assert np.array_equal(idx, one_idx) and np.array_equal(kdb, one_kdb), budget


def test_db_sort_of_an_empty_database(oracle):
    jdb = synth.kdb_header(31, 0)
    want_kdb, want_idx = oracle.db_sort(jdb, 5, True)
    for budget in (0, 8 * (4 ** 5 + 1) + RESERVE + 4096):
        kdb, idx, passes = binding.db_sort(jdb, 5, True, budget=budget, with_passes=True)
        assert passes == 1 and np.array_equal(idx, want_idx) and np.array_equal(kdb, want_kdb[:kdb.size])


def test_db_sort_budget_below_one_bin(tools, tmp_path):
    jdb = _jdb(31, 200000, 9)
    budget = RESERVE + 8 * (4 ** 5 + 1) + 1000            # the histogram fits, no bin of about 200 records does
    with pytest.raises(binding.KuqError) as e:
        binding.db_sort(jdb, 5, True, budget=budget)
    assert e.value.code == -7 and "KUQ_DB_SORT_BUDGET" in str(e.value)
    jdb.tofile(tmp_path / "database.jdb")
    r = subprocess.run([tools[1], "-z", "-n", "5", "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"],
                       cwd=tmp_path, capture_output=True, text=True, env={**os.environ, "KUQ_DB_SORT_BUDGET": str(budget)})
    assert r.returncode != 0 and "KUQ_DB_SORT_BUDGET" in r.stderr
    assert not (tmp_path / "database0.kdb").exists() and not (tmp_path / "database.idx").exists()


def test_db_sort_executable_reports_passes(tools, tmp_path, oracle):
    jdb = _jdb(31, 200000, 4)
    jdb.tofile(tmp_path / "database.jdb")
    want_kdb, want_idx = oracle.db_sort(jdb, 8, True)
    budget = _budgets(want_idx, 12)["several"]
    plan = plan_ranges(_offsets(want_idx), budget - RESERVE, 12 * 2 + PASS_C_REC)
    for env, passes in (({}, 1), ({"KUQ_DB_SORT_BUDGET": str(budget)}, len(plan))):
        r = subprocess.run([tools[1], "-z", "-n", "8", "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"],
                           cwd=tmp_path, capture_output=True, text=True, env={**os.environ, **env})
        assert r.returncode == 0, r.stderr
        assert f"db_sort: {passes} pass{'' if passes == 1 else 'es'}" in r.stderr
        assert (tmp_path / "database.idx").read_bytes() == want_idx.tobytes()
        assert (tmp_path / "database0.kdb").read_bytes() == want_kdb.tobytes()


# ---- 2. the set_lcas executable over ranges -------------------------------------------------------------------------
def _lca_budget(d, n_ranges=4):
    """a KUQ_SET_LCAS_BUDGET that cuts the database in d into about n_ranges ranges"""
    off = _offsets(np.fromfile(d / "database.idx", np.uint8))
    need = 8 * len(off) + 12 * int(off[-1])
    budget = need // n_ranges + 8 * 16 + 12 * int(np.diff(off.astype(np.int64)).max())
    assert len(plan_ranges(off, budget, 12)) >= 3
    return budget


def _run_both(set_lcas, d, args, pipe=False):
    """the same set_lcas command in copies of d at the default budget and over >= 3 ranges: both results"""
    out = []
    budget = _lca_budget(d)
    for env in ({}, {"KUQ_SET_LCAS_BUDGET": str(budget)}):
        w = d.parent / f"{d.name}_{len(out)}"
        if w.exists():
            shutil.rmtree(w)
        shutil.copytree(d, w)
        cmd = " ".join([set_lcas] + args) if pipe else [set_lcas] + args
        r = subprocess.run(["bash", "-c", cmd] if pipe else cmd, cwd=w, capture_output=True, text=True,
                           env={**os.environ, **env})
        if env:
            assert "minimizer ranges" in r.stderr and int(r.stderr.split(" minimizer ranges")[0].rsplit(" ", 1)[1]) >= 3, r.stderr
        else:
            assert "minimizer ranges" not in r.stderr
        files = {f: (w / f).read_bytes() for f in sorted(os.listdir(w))}
        out.append((r.returncode, r.stdout, r.stderr.strip().split("\n")[-1], files))
    return out


def _golden_style(d, k=31, nt=6):
    """test_exact_dbbuild_gpu's library (an unknown taxid, a `.2` accession, an N) and its database0.kdb"""
    rng = np.random.default_rng(21)
    tax = synth.make_taxonomy(6, 3, 2, first_id=100)
    sp = synth.species_ids(tax)
    genomes = synth.random_genomes(rng, 6, 1500, shared_frac=0.3)
    ks = []
    for g in genomes:
        km, ok = synth.forward_kmers(g, k)
        ks.append(synth.canonical(km[ok], k))
    allk = np.unique(np.concatenate(ks))
    rng.shuffle(allk)
    names = [f"seq{i}" for i in range(6)] + ["unknown_tax", "novel.2"]
    extra = rng.integers(0, 4, 700, dtype=np.uint8)
    seqs = [synth.decode(g).tobytes() for g in genomes] + [synth.decode(genomes[0][:400]).tobytes(),
                                                           synth.decode(genomes[1][:300]).tobytes() + b"N" + synth.decode(extra).tobytes()]
    taxids = list(sp) + [4242, sp[3]]
    taxid_cases.write_fasta(d / "lib.fa", [(n + " some description", s) for n, s in zip(names, seqs)])
    with open(d / "seqid2taxid.map", "w") as f:
        for n, t in zip(names, taxids):
            f.write(f"{n[:-2] if n.endswith('.2') else n}\t{t}\n")
    tax.write(str(d / "taxDB"))
    jdb = synth.unsorted_jdb_image(allk, k)
    kdb, idx = binding.db_sort(jdb, nt, True)
    kdb.tofile(d / "database0.kdb")
    idx.tofile(d / "database.idx")
    return tax, names, seqs, taxids, kdb, idx


def _same(runs):
    (rc0, out0, last0, f0), (rc1, out1, last1, f1) = runs
    assert rc0 == rc1 == 0, last1
    assert out0 == out1
    assert f0.keys() == f1.keys()
    for f in f0:
        assert f0[f] == f1[f], f
    return f1


def test_set_lcas_ranges_on_the_golden_style_library(tools, tmp_path, oracle):
    d = tmp_path / "in"
    d.mkdir()
    tax, names, seqs, taxids, kdb0, idx = _golden_style(d)
    base = ["-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-m", "seqid2taxid.map", "-c", "database.kdb.counts"]
    files = _same(_run_both(tools[2], d, ["-x"] + base + ["-F", "lib.fa"]))
    ids, parents = tax.parent_map()
    pm = oracle.parent_map(ids, parents)
    odb = oracle.open_db(kdb0.copy(), idx)
    known = set(int(t) for t in ids)
    for s, t in zip(seqs, taxids):
        if t in known:
            oracle.set_lcas_sequence(odb, pm, s, t)
    assert files["database0.kdb"] == odb.kdb.tobytes()
    assert files["database.kdb.counts"].decode() == taxid_cases.counts_text(odb.kdb)
    # -TR then -T on a sub-library, each on the result of the step before
    (d / "database0.kdb").write_bytes(files["database0.kdb"])
    taxid_cases.write_fasta(d / "sub.fa", list(zip(names, seqs))[1:3])
    for fl, code in (("-TR", 3), ("-T", 1)):
        files = _same(_run_both(tools[2], d, ["-x"] + base + ["-F", "sub.fa", fl]))
        for s, t in list(zip(seqs, taxids))[1:3]:
            oracle.set_lcas_sequence(odb, pm, s, t, flags=code)
        assert files["database0.kdb"] == odb.kdb.tobytes(), fl
        (d / "database0.kdb").write_bytes(files["database0.kdb"])


def test_set_lcas_ranges_with_taxids_for_sequences_and_genomes(tools, tmp_path):
    """-a -A -T: stdout, the rewritten taxDB, database.kdb (-M -o) and .counts as at the default budget"""
    d = tmp_path / "in"
    d.mkdir()
    taxid_cases.write_inputs(d)
    kdb, idx = binding.db_sort(np.fromfile(d / "database.jdb", np.uint8), taxid_cases.NT, True)
    kdb.tofile(d / "database0.kdb")
    idx.tofile(d / "database.idx")
    runs = _run_both(tools[2], d, taxid_cases.command("aA_T"))
    files = _same(runs)
    assert runs[0][1].count("\n") > 5 and files["taxDB"] != (d / "taxDB").read_bytes()


def test_set_lcas_ranges_from_a_pipe_and_a_file_map(tools, tmp_path):
    d = tmp_path / "in"
    d.mkdir()
    _, names, seqs, taxids, _, _ = _golden_style(d)
    base = ["-x", "-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-c", "database.kdb.counts"]
    files = _same(_run_both(tools[2], d, base + ["-m", "seqid2taxid.map", "-F", "lib.fa"]))
    piped = _same(_run_both(tools[2], d, base + ["-m", "seqid2taxid.map", "-F", "<(cat lib.fa)"], pipe=True))
    assert piped == files
    with open(d / "files.map", "w") as f:
        for i, (n, s, t) in enumerate(zip(names, seqs, taxids)):
            taxid_cases.write_fasta(d / f"g{i}.fa", [(n, s)])
            f.write(f"g{i}.fa\t{t}\n")
    _same(_run_both(tools[2], d, base + ["-f", "files.map"]))


def test_set_lcas_ranges_at_k21(tools, tmp_path):
    d = tmp_path / "in"
    d.mkdir()
    _golden_style(d, k=21, nt=7)
    _same(_run_both(tools[2], d, ["-x", "-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-m",
                                  "seqid2taxid.map", "-F", "lib.fa", "-c", "database.kdb.counts"]))


def test_set_lcas_ranges_missing_kmer_without_x(tools, tmp_path):
    """a library k-mer that the database lacks: same status and message over ranges, and nothing written"""
    d = tmp_path / "in"
    d.mkdir()
    _golden_style(d)
    before = {f: (d / f).read_bytes() for f in os.listdir(d)}
    runs = _run_both(tools[2], d, ["-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-m", "seqid2taxid.map",
                                   "-F", "lib.fa", "-c", "database.kdb.counts"])
    assert runs[0][0] == runs[1][0] != 0
    for run in runs:
        assert run[2].endswith("set_lcas: kmer found in sequence that is not in database"), run[2]
    assert runs[0][3] == runs[1][3] == before


# ---- 3. the C ABI, range by range ----------------------------------------------------------------------------------
def test_set_lcas_range_by_range_through_the_c_abi(tmp_path, oracle):
    d = tmp_path
    tax, names, seqs, taxids, kdb0, idx = _golden_style(d)
    ids, parents = tax.parent_map()
    known = set(int(t) for t in ids)
    pieces, pt = [], []
    for s, t in zip(seqs, taxids):
        if t in known:
            for i in range(0, len(s), 400):
                pieces.append(s[i:i + 400 + 30])
                pt.append(t)
    bases, offs = synth.pack_reads(pieces)
    whole = kdb0.copy()
    clf = binding.Classifier(max_reads=1 << 16, max_bases=16 << 20)
    clf.stage_db(kdb0, idx)
    clf.set_taxonomy(ids, parents)
    want_missing = clf.set_lcas(bases, offs, pt, flags=1)
    clf.export_db_values(whole)
    clf.close()
    assert want_missing > 0
    off = _offsets(idx)
    ranges = plan_ranges(off, (8 * len(off) + 12 * int(off[-1])) // 4 + 4096, 12)
    assert len(ranges) >= 3
    ranges[0] = (0, ranges[0][1])
    ranges = [(a, ranges[i + 1][0] if i + 1 < len(ranges) else len(off) - 1) for i, (a, _) in enumerate(ranges)]
    out = kdb0.copy()
    clf = binding.Classifier(max_reads=1 << 16, max_bases=16 << 20)
    clf.set_db_taxid_universe([0])
    missing = 0
    for i, (lo, hi) in enumerate(ranges):
        clf.stage_db(kdb0, idx, lo, hi)
        if i == 0:
            clf.set_taxonomy(ids, parents)
        missing += clf.set_lcas(bases, offs, pt, flags=1)
        clf.export_db_values(out)
    clf.close()
    assert missing == want_missing
    assert np.array_equal(out, whole)


# ---- 4. the whole chain, each step in several passes ---------------------------------------------------------------
def test_golden_database_rebuilt_in_passes(tools, tmp_path, oracle):
    exe, db_sort, set_lcas = tools
    kmer_set_tests._golden_library(tmp_path)
    want = kmer_set_tests._expected([tmp_path / "lib.fa"], 31, oracle)
    bases, offs = kmer_set_tests._library(tmp_path / "lib.fa")
    ks_budget, ks_passes = kmer_set_tests._budget_for(bases, offs, 31, want, 3)
    img, err = kmer_set_tests._run(exe, 31, ["lib.fa"], tmp_path, {"KUQ_KMER_SET_BUDGET": str(ks_budget)}, pipe=True)
    assert kmer_set_tests._passes(err) == ks_passes >= 3
    img.tofile(tmp_path / "database.jdb")
    gold_idx = np.fromfile(os.path.join(util.GOLDEN, "database.idx"), np.uint8)
    ds_budget = _budgets(gold_idx, 12)["several"]
    r = subprocess.run([db_sort, "-z", "-n", "6", "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"],
                       cwd=tmp_path, capture_output=True, text=True, env={**os.environ, "KUQ_DB_SORT_BUDGET": str(ds_budget)})
    assert r.returncode == 0, r.stderr
    assert int(r.stderr.split(" passes")[0].rsplit(" ", 1)[1]) >= 3, r.stderr
    r = subprocess.run([set_lcas, "-x", "-d", "database0.kdb", "-o", "database.kdb", "-i", "database.idx", "-b", "taxDB",
                        "-m", "seqid2taxid.map", "-F", "lib.fa", "-c", "database.kdb.counts"],
                       cwd=tmp_path, capture_output=True, text=True,
                       env={**os.environ, "KUQ_SET_LCAS_BUDGET": str(_lca_budget(tmp_path))})
    assert r.returncode == 0, r.stderr
    assert "minimizer ranges" in r.stderr
    for f in ("database.kdb", "database.idx"):
        assert (tmp_path / f).read_bytes() == open(os.path.join(util.GOLDEN, f), "rb").read(), f
    gold = np.fromfile(os.path.join(util.GOLDEN, "database.kdb"), np.uint8)
    assert (tmp_path / "database.kdb.counts").read_text() == taxid_cases.counts_text(gold)
