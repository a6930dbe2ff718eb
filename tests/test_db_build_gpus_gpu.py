"""db_sort and set_lcas over several GPUs: the minimizer ranges of a database too large for one card are split over the
workers of KUQ_DEVICES (one card listed twice or three times here, two cards where there are two).  Every run must
write the bytes of the one-device run, and of the oracle where the case has one.

- kuq_db_sort_devices and the db_sort executable at budgets that give fewer, as many and more ranges than workers;
  repeated keys across the cut between two workers' slices; an empty database; a budget below one bin.
- the set_lcas executable: the golden-style library (-x -c, -TR, -T), -a -A -T, a pipe, the -f file map, k = 21, a
  missing k-mer without -x; the plan line says that one range per context keeps no batches.
- kuq_db_value_counts against a count of the exported image, value 0 and taxids above 10^9 included.
- kmer_set, db_sort and set_lcas rebuild the golden database on two workers."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from krakenuniq_b200 import binding, build, synth
from tests import taxid_cases, util
from tests import test_db_build_ranges_gpu as ranges_tests
from tests import test_kmer_set_gpu as kmer_set_tests

pytestmark = pytest.mark.gpu

RESERVE, PASS_C_REC = ranges_tests.RESERVE, ranges_tests.PASS_C_REC
two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")


@pytest.fixture(scope="module")
def tools():
    db_sort, set_lcas = build.build_dbtools()
    return build.KMER_SET, db_sort, set_lcas


def _offsets(idx):
    return ranges_tests._offsets(idx)


def _two_ranges_budget(idx, pair):
    """the smallest KUQ_DB_SORT_BUDGET whose plan has two ranges"""
    off, rec = _offsets(idx), 2 * pair + PASS_C_REC
    lo, hi = RESERVE + 8 * len(off), RESERVE + 8 * len(off) + rec * int(off[-1]) + 64
    while lo < hi:
        mid = (lo + hi) // 2
        plan = ranges_tests.plan_ranges(off, mid - RESERVE, rec)
        if plan is not None and len(plan) <= 2:
            hi = mid
        else:
            lo = mid + 1
    assert len(ranges_tests.plan_ranges(off, lo - RESERVE, rec)) == 2
    return lo


# ---- 1. db_sort ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,nt,zero", [(31, 5, True), (31, 8, False), (31, 11, True), (21, 5, False), (21, 8, True),
                                       (21, 11, False)])
def test_db_sort_devices_match_one_device_and_oracle(oracle, k, nt, zero):
    jdb = ranges_tests._jdb(k, 1000000 if nt == 11 else 200000, 100 * k + nt + 7)
    pair = (2 * k + 7) // 8 + 4
    one_kdb, one_idx = binding.db_sort(jdb, nt, zero)
    want_kdb, want_idx = oracle.db_sort(jdb, nt, zero)
    assert np.array_equal(one_idx, want_idx) and np.array_equal(one_kdb, want_kdb[:one_kdb.size])
    shapes = set()
    budgets = dict(ranges_tests._budgets(one_idx, pair), exactly_two=_two_ranges_budget(one_idx, pair))
    for name, budget in budgets.items():
        plan = ranges_tests.plan_ranges(_offsets(one_idx), budget - RESERVE, 2 * pair + PASS_C_REC)
        for devices in ([0, 0], [0, 0, 0]):
            kdb, idx, passes = binding.db_sort(jdb, nt, zero, budget=budget, with_passes=True, devices=devices)
            assert passes == len(plan) >= 2, (name, devices, passes, len(plan))
            assert np.array_equal(idx, one_idx), (name, devices)
            assert np.array_equal(kdb, one_kdb), (name, devices)
            shapes.add((passes > len(devices)) - (passes < len(devices)))
    assert shapes == {-1, 0, 1}, shapes                            # fewer, as many and more ranges than workers


@pytest.mark.parametrize("n_dev", [2, 3])
def test_db_sort_devices_keep_repeated_keys_across_slice_cuts(n_dev):
    """a key repeated on both sides of the cut between two workers' slices comes out in input order"""
    rng = np.random.default_rng(5)
    k, nt = 31, 6
    keys = np.unique(rng.integers(0, 1 << (2 * k), 120000, dtype=np.uint64))
    rng.shuffle(keys)
    n = len(keys)
    for w in range(1, n_dev):
        cut = n * w // n_dev
        keys[cut - 3:cut + 3] = keys[cut]                  # six records of one key, three in each slice
    keys[: n // 10] = rng.choice(keys, n // 10)            # and repeats everywhere else
    vals = np.arange(1, n + 1, dtype=np.uint32)            # distinct values show the order of equal keys
    jdb = np.concatenate([synth.kdb_header(k, n), synth.pack_records(keys, vals, k)])
    one_kdb, one_idx = binding.db_sort(jdb, nt, False)
    for budget in ranges_tests._budgets(one_idx, 12).values():
        kdb, idx, passes = binding.db_sort(jdb, nt, False, budget=budget, with_passes=True, devices=[0] * n_dev)
        assert passes >= 2
        assert np.array_equal(idx, one_idx) and np.array_equal(kdb, one_kdb), budget


def test_db_sort_devices_of_an_empty_database(oracle):
    jdb = synth.kdb_header(31, 0)
    want_kdb, want_idx = oracle.db_sort(jdb, 5, True)
    for budget in (0, 8 * (4 ** 5 + 1) + RESERVE + 4096):
        kdb, idx, passes = binding.db_sort(jdb, 5, True, budget=budget, with_passes=True, devices=[0, 0])
        assert passes == 1 and np.array_equal(idx, want_idx) and np.array_equal(kdb, want_kdb[:kdb.size])


def test_db_sort_devices_budget_below_one_bin(tools, tmp_path):
    jdb = ranges_tests._jdb(31, 200000, 9)
    budget = RESERVE + 8 * (4 ** 5 + 1) + 1000
    with pytest.raises(binding.KuqError) as one:
        binding.db_sort(jdb, 5, True, budget=budget)
    with pytest.raises(binding.KuqError) as two:
        binding.db_sort(jdb, 5, True, budget=budget, devices=[0, 0])
    assert two.value.code == one.value.code == -7 and str(two.value) == str(one.value)
    jdb.tofile(tmp_path / "database.jdb")
    errs = []
    for devices in ("0", "0,0"):
        r = subprocess.run([tools[1], "-z", "-n", "5", "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"],
                           cwd=tmp_path, capture_output=True, text=True,
                           env={**os.environ, "KUQ_DB_SORT_BUDGET": str(budget), "KUQ_DEVICES": devices})
        assert r.returncode != 0 and "KUQ_DB_SORT_BUDGET" in r.stderr
        errs.append((r.returncode, r.stderr.strip().split("\n")[-1]))
        assert not (tmp_path / "database0.kdb").exists() and not (tmp_path / "database.idx").exists()
    assert errs[0] == errs[1]


def _db_sort_executable(tools, tmp_path, oracle, devices):
    jdb = ranges_tests._jdb(31, 200000, 4)
    jdb.tofile(tmp_path / "database.jdb")
    want_kdb, want_idx = oracle.db_sort(jdb, 8, True)
    budget = ranges_tests._budgets(want_idx, 12)["several"]
    plan = ranges_tests.plan_ranges(_offsets(want_idx), budget - RESERVE, 12 * 2 + PASS_C_REC)
    r = subprocess.run([tools[1], "-z", "-n", "8", "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"],
                       cwd=tmp_path, capture_output=True, text=True,
                       env={**os.environ, "KUQ_DB_SORT_BUDGET": str(budget), "KUQ_DEVICES": devices})
    assert r.returncode == 0, r.stderr
    n_dev = len(devices.split(","))
    assert f"db_sort: {len(plan)} passes on {n_dev} devices" in r.stderr, r.stderr
    assert (tmp_path / "database.idx").read_bytes() == want_idx.tobytes()
    assert (tmp_path / "database0.kdb").read_bytes() == want_kdb.tobytes()


def test_db_sort_executable_on_two_workers(tools, tmp_path, oracle):
    _db_sort_executable(tools, tmp_path, oracle, "0,0")


@two_gpus
def test_db_sort_executable_on_two_gpus(tools, tmp_path, oracle):
    _db_sort_executable(tools, tmp_path, oracle, "0,1")


# ---- 2. set_lcas -----------------------------------------------------------------------------------------------------
def _lca_budget(d, n_ranges):
    """the smallest KUQ_SET_LCAS_BUDGET that cuts the database in d into at most n_ranges ranges, and their count"""
    off = _offsets(np.fromfile(d / "database.idx", np.uint8))
    lo, hi = 8 * 16 + 12 * int(np.diff(off.astype(np.int64)).max()), 8 * len(off) + 12 * int(off[-1]) + 64
    while lo < hi:
        mid = (lo + hi) // 2
        plan = ranges_tests.plan_ranges(off, mid, 12)
        if plan is not None and len(plan) <= n_ranges:
            hi = mid
        else:
            lo = mid + 1
    return lo, len(ranges_tests.plan_ranges(off, lo, 12))


PLAN = re.compile(r"Database staged in (\d+) minimizer ranges over (\d+) contexts? \(batches kept: (yes|no)\)")


def _run_devices(set_lcas, d, args, pipe=False, shapes=((2, "0,0"), (2, "0,0,0"), (5, "0,0"), (5, "0,0,0"))):
    """the same set_lcas command in copies of d: on one device at the default budget, then for each (ranges, devices)
    on one device and on those devices at a budget of about that many ranges.  Every run's (status, stdout, last stderr
    line, files) must equal the first one's; returns them and the plans of the several-device runs."""
    runs, plans = [], []
    envs = [{"KUQ_DEVICES": "0"}]
    for n_ranges, devices in shapes:
        budget, _ = _lca_budget(d, n_ranges)
        envs += [{"KUQ_DEVICES": "0", "KUQ_SET_LCAS_BUDGET": str(budget)},
                 {"KUQ_DEVICES": devices, "KUQ_SET_LCAS_BUDGET": str(budget)}]
    for i, env in enumerate(envs):
        w = d.parent / f"{d.name}_{i}"
        if w.exists():
            shutil.rmtree(w)
        shutil.copytree(d, w)
        cmd = " ".join([set_lcas] + args) if pipe else [set_lcas] + args
        r = subprocess.run(["bash", "-c", cmd] if pipe else cmd, cwd=w, capture_output=True, text=True,
                           env={**os.environ, **env})
        files = {f: (w / f).read_bytes() for f in sorted(os.listdir(w))}
        runs.append((r.returncode, r.stdout, r.stderr.strip().split("\n")[-1], files))
        m = PLAN.search(r.stderr)
        if "," in env["KUQ_DEVICES"]:
            assert m, r.stderr
            n_ranges, n_ctx, kept = int(m.group(1)), int(m.group(2)), m.group(3)
            n_dev = len(env["KUQ_DEVICES"].split(","))
            assert n_ctx == min(n_ranges, n_dev) if n_ranges <= n_dev else n_ctx <= n_dev
            assert kept == ("no" if n_ranges <= n_dev else "yes"), r.stderr
            plans.append((n_ranges, n_dev, kept))
        elif "KUQ_SET_LCAS_BUDGET" not in env:
            assert "minimizer ranges" not in r.stderr
    for run in runs[1:]:
        assert run[0] == runs[0][0] and run[1] == runs[0][1], run[2]
        assert run[3].keys() == runs[0][3].keys()
        for f in run[3]:
            assert run[3][f] == runs[0][3][f], f
    return runs, plans


def _shapes_covered(plans):
    """the several-device runs had fewer, as many and more ranges than contexts"""
    sides = {(r > g) - (r < g) for r, g, _ in plans}
    assert sides == {-1, 0, 1}, plans


def test_set_lcas_devices_on_the_golden_style_library(tools, tmp_path, oracle):
    d = tmp_path / "in"
    d.mkdir()
    tax, names, seqs, taxids, kdb0, idx = ranges_tests._golden_style(d)
    base = ["-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-m", "seqid2taxid.map", "-c", "database.kdb.counts"]
    runs, plans = _run_devices(tools[2], d, ["-x"] + base + ["-F", "lib.fa"])
    _shapes_covered(plans)
    assert runs[0][0] == 0, runs[0][2]
    files = runs[0][3]
    ids, parents = tax.parent_map()
    pm = oracle.parent_map(ids, parents)
    odb = oracle.open_db(kdb0.copy(), idx)
    known = set(int(t) for t in ids)
    for s, t in zip(seqs, taxids):
        if t in known:
            oracle.set_lcas_sequence(odb, pm, s, t)
    assert files["database0.kdb"] == odb.kdb.tobytes()
    assert files["database.kdb.counts"].decode() == taxid_cases.counts_text(odb.kdb)
    (d / "database0.kdb").write_bytes(files["database0.kdb"])
    taxid_cases.write_fasta(d / "sub.fa", list(zip(names, seqs))[1:3])
    for fl, code in (("-TR", 3), ("-T", 1)):
        runs, _ = _run_devices(tools[2], d, ["-x"] + base + ["-F", "sub.fa", fl])
        assert runs[0][0] == 0
        for s, t in list(zip(seqs, taxids))[1:3]:
            oracle.set_lcas_sequence(odb, pm, s, t, flags=code)
        assert runs[0][3]["database0.kdb"] == odb.kdb.tobytes(), fl
        (d / "database0.kdb").write_bytes(runs[0][3]["database0.kdb"])


def test_set_lcas_devices_with_taxids_for_sequences_and_genomes(tools, tmp_path):
    """-a -A -T: stdout, the rewritten taxDB, database.kdb (-M -o) and .counts as on one device"""
    d = tmp_path / "in"
    d.mkdir()
    taxid_cases.write_inputs(d)
    kdb, idx = binding.db_sort(np.fromfile(d / "database.jdb", np.uint8), taxid_cases.NT, True)
    kdb.tofile(d / "database0.kdb")
    idx.tofile(d / "database.idx")
    runs, _ = _run_devices(tools[2], d, taxid_cases.command("aA_T"), shapes=((2, "0,0"), (5, "0,0,0")))
    assert runs[0][0] == 0
    assert runs[0][1].count("\n") > 5 and runs[0][3]["taxDB"] != (d / "taxDB").read_bytes()


def test_set_lcas_devices_from_a_pipe_and_a_file_map(tools, tmp_path):
    """a library piped in is read once: with one range per context no batch is kept, and the bytes are the file's"""
    d = tmp_path / "in"
    d.mkdir()
    _, names, seqs, taxids, _, _ = ranges_tests._golden_style(d)
    base = ["-x", "-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-c", "database.kdb.counts"]
    shapes = ((2, "0,0"), (2, "0,0,0"), (5, "0,0"))
    files, _ = _run_devices(tools[2], d, base + ["-m", "seqid2taxid.map", "-F", "lib.fa"], shapes=shapes)
    piped, plans = _run_devices(tools[2], d, base + ["-m", "seqid2taxid.map", "-F", "<(cat lib.fa)"], pipe=True, shapes=shapes)
    assert any(kept == "no" for _, _, kept in plans)
    assert piped[0][3] == files[0][3]
    with open(d / "files.map", "w") as f:
        for i, (n, s, t) in enumerate(zip(names, seqs, taxids)):
            taxid_cases.write_fasta(d / f"g{i}.fa", [(n, s)])
            f.write(f"g{i}.fa\t{t}\n")
    runs, _ = _run_devices(tools[2], d, base + ["-f", "files.map"], shapes=shapes)
    assert runs[0][0] == 0


def test_set_lcas_devices_at_k21(tools, tmp_path):
    d = tmp_path / "in"
    d.mkdir()
    ranges_tests._golden_style(d, k=21, nt=7)
    runs, _ = _run_devices(tools[2], d, ["-x", "-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-m",
                                         "seqid2taxid.map", "-F", "lib.fa", "-c", "database.kdb.counts"])
    assert runs[0][0] == 0


def test_set_lcas_devices_missing_kmer_without_x(tools, tmp_path):
    """a library k-mer that the database lacks: the one-device status and message on every layout, nothing written"""
    d = tmp_path / "in"
    d.mkdir()
    ranges_tests._golden_style(d)
    before = {f: (d / f).read_bytes() for f in os.listdir(d)}
    runs, _ = _run_devices(tools[2], d, ["-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-m",
                                         "seqid2taxid.map", "-F", "lib.fa", "-c", "database.kdb.counts"])
    for run in runs:
        assert run[0] == runs[0][0] != 0
        assert run[2].endswith("set_lcas: kmer found in sequence that is not in database"), run[2]
        assert run[3] == before


@two_gpus
def test_set_lcas_on_two_gpus(tools, tmp_path):
    d = tmp_path / "in"
    d.mkdir()
    ranges_tests._golden_style(d)
    runs, plans = _run_devices(tools[2], d, ["-x", "-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-m",
                                             "seqid2taxid.map", "-F", "lib.fa", "-c", "database.kdb.counts"],
                               shapes=((2, "0,1"), (5, "0,1")))
    assert runs[0][0] == 0 and {kept for _, _, kept in plans} == {"yes", "no"}


# ---- 3. kuq_db_value_counts -------------------------------------------------------------------------------------------
def _value_counts(kdb):
    _, _, vals = synth.parse_kdb(kdb)
    t, c = np.unique(vals, return_counts=True)
    return t.astype(np.uint32), c.astype(np.uint64)


@pytest.mark.parametrize("extra_taxa", [0, 20000])
def test_db_value_counts_through_the_c_abi(tmp_path, extra_taxa):
    """the device count equals a count of the exported image: as staged, after LCAs, after -R zeroes some values, and
    with taxa above 10^9 (what -a / -A add); 20000 more taxa take the counters out of shared memory"""
    tax, names, seqs, taxids, kdb0, idx = ranges_tests._golden_style(tmp_path)
    sp = synth.species_ids(tax)
    big = [1000000001 + i for i in range(3)]
    rows = tax.rows + [(b, int(sp[i]), f"seq{i}", "sequence") for i, b in enumerate(big)]
    rows += [(2000000000 + i, 1, f"filler{i}", "no rank") for i in range(extra_taxa)]
    ids, parents = synth.Taxonomy(rows).parent_map()
    known = set(int(t) for t in ids)
    clf = binding.Classifier(max_reads=1 << 16, max_bases=16 << 20)
    clf.stage_db(kdb0, idx)
    t, c = clf.db_value_counts()
    want_t, want_c = _value_counts(kdb0)
    assert np.array_equal(t, want_t) and np.array_equal(c, want_c)
    clf.set_taxonomy(ids, parents)

    def batch(seq_taxa, flags):
        pieces, pt = [], []
        for s, tx in seq_taxa:
            for i in range(0, len(s), 400):
                pieces.append(s[i:i + 430])
                pt.append(tx)
        bases, offs = synth.pack_reads(pieces)
        clf.set_lcas(bases, offs, pt, flags=flags)
        out = kdb0.copy()
        clf.export_db_values(out)
        t, c = clf.db_value_counts()
        want_t, want_c = _value_counts(out)
        assert np.array_equal(t, want_t) and np.array_equal(c, want_c), flags
        return want_t
    batch([(s, tx) for s, tx in zip(seqs, taxids) if tx in known], 0)
    assert batch([(seqs[i], int(sp[i])) for i in range(3)], 2)[0] == 0          # -R: values 0
    assert batch([(seqs[i], big[i]) for i in range(3)], 0).max() > 10 ** 9     # lca(t, 0) = t: taxa above 10^9
    clf.close()


# ---- 4. the whole chain on two workers ---------------------------------------------------------------------------------
def test_golden_database_rebuilt_on_two_workers(tools, tmp_path, oracle):
    exe, db_sort, set_lcas = tools
    kmer_set_tests._golden_library(tmp_path)
    img, err = kmer_set_tests._run(exe, 31, ["lib.fa"], tmp_path, {}, pipe=True)
    img.tofile(tmp_path / "database.jdb")
    gold_idx = np.fromfile(os.path.join(util.GOLDEN, "database.idx"), np.uint8)
    ds_budget = ranges_tests._budgets(gold_idx, 12)["several"]
    env = {**os.environ, "KUQ_DEVICES": "0,0"}
    r = subprocess.run([db_sort, "-z", "-n", "6", "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"],
                       cwd=tmp_path, capture_output=True, text=True, env={**env, "KUQ_DB_SORT_BUDGET": str(ds_budget)})
    assert r.returncode == 0, r.stderr
    assert re.search(r"db_sort: \d+ passes on 2 devices", r.stderr), r.stderr
    budget, _ = _lca_budget(tmp_path, 4)
    r = subprocess.run([set_lcas, "-x", "-d", "database0.kdb", "-o", "database.kdb", "-i", "database.idx", "-b", "taxDB",
                        "-m", "seqid2taxid.map", "-F", "lib.fa", "-c", "database.kdb.counts"],
                       cwd=tmp_path, capture_output=True, text=True, env={**env, "KUQ_SET_LCAS_BUDGET": str(budget)})
    assert r.returncode == 0, r.stderr
    assert PLAN.search(r.stderr) and " over 2 contexts" in r.stderr, r.stderr
    for f in ("database.kdb", "database.idx"):
        assert (tmp_path / f).read_bytes() == open(os.path.join(util.GOLDEN, f), "rb").read(), f
    assert (tmp_path / "database.kdb.counts").read_bytes() == open(os.path.join(util.GOLDEN, "database.kdb.counts"), "rb").read()
