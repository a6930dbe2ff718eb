"""The drop-in set_lcas with -a / -A (krakenuniq-build --taxids-for-sequences / --taxids-for-genomes) against the
unmodified reference's recorded runs (tests/ref_replay.py), byte for byte: stdout, rewritten taxDB, database and
.counts.  Then `classify` on such a database against the reference's classify, and a library of a few species and
hundreds of strains, built by the drop-in tools and classified through the CLI, against the oracle."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import build, synth
from tests import ref_replay, taxid_cases as tc, util

pytestmark = pytest.mark.gpu


def _ours(tool, args, cwd):
    exe = dict(zip(("db_sort", "set_lcas"), build.build_dbtools())).get(tool) or os.path.join(os.path.dirname(build.CLASSIFY), tool)
    return subprocess.run([exe] + [str(a) for a in args], cwd=cwd, capture_output=True, text=True)


def _reference_case(tmp_path, case):
    """the recording of tests/test_oracle_taxids_for_genomes.py for this case, replayed"""
    tape = ref_replay.Tape(f"test_oracle_taxids_for_genomes.py::test_oracle_matches_reference[{case}]")
    ref, pristine, r = tc.run_reference(tape, tmp_path, case)
    tape.close()
    return ref, pristine, r


@pytest.mark.parametrize("case", list(tc.CASES))
def test_set_lcas_matches_reference(tmp_path, case):
    ref, pristine, r = _reference_case(tmp_path, case)
    ours = tmp_path / "ours"
    shutil.copytree(pristine, ours)
    g = _ours("set_lcas", tc.command(case), ours)
    assert g.returncode == 0, g.stderr[-2000:]
    assert g.stdout == r.stdout
    assert tc.outputs(ours) == tc.outputs(ref)
    assert open(ours / "database0.kdb", "rb").read() == open(pristine / "database0.kdb", "rb").read()
    assert "[starting new taxonomy IDs with 1000000001]" in g.stderr
    # the drop-in db_sort gives the reference's database0.kdb / database.idx too
    d = tmp_path / "sort"
    d.mkdir()
    shutil.copy(pristine / "database.jdb", d)
    g = _ours("db_sort", ["-z", "-M", "-n", tc.NT, "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"], d)
    assert g.returncode == 0, g.stderr
    for n in ("database0.kdb", "database.idx"):
        assert open(d / n, "rb").read() == open(pristine / n, "rb").read(), n


# variants of build_db.sh's command line: (arguments to add, arguments to drop)
VARIANTS = {"pretend": (["-p"], []), "no_ram": ([], ["-M"]), "reset": (["-R"], []), "threads": (["-t", "2"], ["-t"]),
            "files": (["-f", "files.map"], [])}


def _variant_args(tag):
    add, drop = VARIANTS[tag]
    args = tc.command("aA_T")
    for a in drop:
        i = args.index(a)
        del args[i:i + (2 if a == "-t" else 1)]
    return args + add


def _variant_inputs(d, tag):
    d.mkdir()
    tc.write_inputs(d)
    if tag == "files":                                 # process_files: the first record of each file, its line's taxid
        records = tc.read_fasta(d / "lib.fa")
        sp = synth.species_ids(synth.Taxonomy.read(str(d / "taxDB")))
        with open(d / "files.map", "w") as f:
            for i, t in ((0, sp[0]), (2, sp[1]), (9, sp[3]), (10, sp[4])):
                tc.write_fasta(d / f"g{i}.fa", records[i:i + 2])
                f.write(f"g{i}.fa\t{t}\n")


def test_set_lcas_option_variants(reference, tmp_path):
    """-p, -o without -M, -R, -t 2 and -f on build_db.sh's -a -A -T command line: the reference first (all of its
    runs), then ours on copies of the same inputs"""
    want = {}
    for tag in VARIANTS:
        d = tmp_path / ("ref_" + tag)
        _variant_inputs(d, tag)
        r = reference.run_tool("db_sort", ["-z", "-M", "-n", tc.NT, "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"], cwd=d)
        assert r.returncode == 0, r.stderr
        shutil.copytree(d, tmp_path / ("in_" + tag))
        r = reference.run_tool("set_lcas", _variant_args(tag), cwd=d)
        assert r.returncode == 0, r.stderr[-2000:]
        want[tag] = r
    for tag, r in want.items():
        ref, ours = tmp_path / ("ref_" + tag), tmp_path / ("ours_" + tag)
        shutil.copytree(tmp_path / ("in_" + tag), ours)
        g = _ours("set_lcas", _variant_args(tag), ours)
        assert g.returncode == 0, (tag, g.stderr[-2000:])
        assert g.stdout == r.stdout, tag
        assert sorted(os.listdir(ours)) == sorted(os.listdir(ref)), tag
        for n in sorted(os.listdir(ref)):
            assert open(ours / n, "rb").read() == open(ref / n, "rb").read(), (tag, n)
    assert want["pretend"].stdout and not os.path.exists(tmp_path / "ref_pretend" / "database.kdb")
    assert not want["files"].stdout


def test_taxdb_with_pseudo_ids(reference, tmp_path):
    """A second -a -A run on a taxDB that the first one rewrote: 200 consecutive new ids are in it, and where the next
    ones start depends on the order the reference's hash map visits them (set_lcas.cpp:219-224)"""
    rng = np.random.default_rng(11)
    tax = synth.make_taxonomy(4, 2, 1, first_id=100)
    sp = synth.species_ids(tax)
    genomes = synth.random_genomes(rng, 4, 6000, shared_frac=0.2)
    records, map_lines = [], []
    for i in range(150):
        g = genomes[i % 4]
        a = int(rng.integers(0, len(g) - 300))
        records.append((f"p{i} piece", synth.decode(g[a:a + 300]).tobytes()))
        map_lines.append(f"p{i}\t{sp[i % 4]}\tstrain{i // 3}")
    d = tmp_path / "ref"
    d.mkdir()
    tax.write(str(d / "taxDB"))
    with open(d / "seqid2taxid.map", "w") as f:
        f.write("".join(m + "\n" for m in map_lines))
    tc.write_fasta(d / "lib.fa", records)
    allk = np.unique(np.concatenate([synth.canonical(km[ok], tc.K) for km, ok in (synth.forward_kmers(g, tc.K) for g in genomes)]))
    rng.shuffle(allk)
    synth.unsorted_jdb_image(allk, tc.K).tofile(d / "database.jdb")
    r = reference.run_tool("db_sort", ["-z", "-M", "-n", tc.NT, "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"], cwd=d)
    assert r.returncode == 0, r.stderr
    shutil.copytree(d, tmp_path / "ours")
    runs = []
    for _ in range(2):
        r = reference.run_tool("set_lcas", tc.command("aA_T"), cwd=d)
        assert r.returncode == 0, r.stderr[-2000:]
        runs.append((r, tc.outputs(d)))
    ids = [int(line.split("\t")[0]) for line in runs[0][1][1].decode().splitlines()]
    assert sum(t > 1_000_000_000 for t in ids) == 200                 # 150 sequences, 50 strains
    assert "[starting new taxonomy IDs with 1000000001]" not in runs[1][0].stderr
    for r, want in runs:
        g = _ours("set_lcas", tc.command("aA_T"), tmp_path / "ours")
        assert g.returncode == 0, g.stderr[-2000:]
        assert g.stdout == r.stdout
        assert re.search(r"\[starting new taxonomy IDs with \d+\]", r.stderr).group(0) in g.stderr   # the same start
        assert tc.outputs(tmp_path / "ours") == want


def _report_rows(path):
    return {line.split("\t")[6]: line for line in open(path) if line[:1] not in ("#", "%")}


def test_classify_matches_reference(reference, tmp_path):
    """classify on the database build_db.sh's -a -A -T command line gives: the reference's Kraken lines and report,
    with assembly and sequence taxa, their ids >= 10^9 and the names the headers gave them"""
    ref, pristine, _ = _reference_case(tmp_path, "aA_T")
    d = tmp_path / "cls"
    d.mkdir()
    for n in ("database.kdb", "database.idx", "taxDB", "database.kdb.counts"):
        shutil.copy(ref / n, d)
    records = [s for _, s in tc.read_fasta(pristine / "lib.fa") if len(s) >= 300]
    rng = np.random.default_rng(5)
    bases, offs = synth.sample_reads(rng, [synth.encode(s) for s in records], 600, 120, 0.01, 0.1, 0.5)
    seqs = [bases[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)]
    seqs.append(b"".join(records))                                    # one read over the whole library
    tc.write_fasta(d / "reads.fa", [(f"r{i}", s) for i, s in enumerate(seqs)], width=1 << 20)
    args = ["-d", "database.kdb", "-i", "database.idx", "-a", "taxDB", "-t", "1", "-M"]
    r = reference.run_tool("classify", args + ["-r", "ref.report", "-o", "ref.kraken", "reads.fa"], cwd=d)
    assert r.returncode == 0, r.stderr[-1500:]
    g = _ours("classify", args + ["-r", "out.report", "-o", "out.kraken", "reads.fa"], d)
    assert g.returncode == 0, g.stderr[-2000:]
    assert open(d / "out.kraken").read() == open(d / "ref.kraken").read()
    got, want = _report_rows(d / "out.report"), _report_rows(d / "ref.report")
    assert got == want
    rows = util.parse_report(d / "ref.report")
    ranks = {v["rank"] for t, v in rows.items() if t > 1_000_000_000}
    assert {"assembly", "sequence"} <= ranks
    assert any(v["name"].strip() == "hs2 neanderthal" for v in rows.values())


# ---- a strain library at moderate scale, against the oracle ----------------------------------------------------
def test_strain_library_at_scale(oracle, tmp_path):
    """4 species x 250 strains, one record each, built with db_sort -z and set_lcas -a -A -T by the drop-in tools:
    2,000 new taxa.  The reads include contigs over 60 strains each (more than 32 distinct taxa per read)."""
    rng = np.random.default_rng(23)
    n_sp, n_strains, glen = 4, 250, 4000
    tax = synth.make_taxonomy(n_sp, 2, 1, first_id=100)
    sp = synth.species_ids(tax)
    base = [rng.integers(0, 4, glen, dtype=np.uint8) for _ in range(n_sp)]
    strains, records, map_lines = [], [], []
    for s in range(n_sp):
        for j in range(n_strains):
            g = base[s].copy()
            m = rng.random(glen) < 0.004
            g[m] = (g[m] + rng.integers(1, 4, int(m.sum()), dtype=np.uint8)) & 3
            strains.append(g)
            records.append((f"sp{s}_st{j}.1 strain {j} of species {s}", synth.decode(g).tobytes()))
            map_lines.append(f"sp{s}_st{j}\t{sp[s]}\tspecies{s} strain{j}")
    d = tmp_path / "db"
    d.mkdir()
    tax.write(str(d / "taxDB"))
    with open(d / "seqid2taxid.map", "w") as f:
        f.write("".join(m + "\n" for m in map_lines))
    tc.write_fasta(d / "lib.fa", records)
    allk = np.unique(np.concatenate([synth.canonical(km[ok], tc.K) for km, ok in (synth.forward_kmers(g, tc.K) for g in strains)]))
    rng.shuffle(allk)
    synth.unsorted_jdb_image(allk, tc.K).tofile(d / "database.jdb")
    g = _ours("db_sort", ["-z", "-M", "-n", 10, "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"], d)
    assert g.returncode == 0, g.stderr
    shutil.copytree(d, tmp_path / "in")
    g = _ours("set_lcas", tc.command("aA_T"), d)
    assert g.returncode == 0, g.stderr[-2000:]

    ext, kdb, counts = tc.expected(oracle, tmp_path / "in", True, True, True, 0)
    assert g.stdout == ext.stdout
    got_kdb, got_taxdb, got_counts = tc.outputs(d)
    assert got_taxdb.decode() == ext.taxdb_text()
    assert np.array_equal(np.frombuffer(got_kdb, np.uint8), kdb)
    assert got_counts.decode() == counts
    new = [r for r in ext.rows() if r[0] > 1_000_000_000]
    assert len(new) == 2 * n_sp * n_strains

    bases, offs = synth.sample_reads(rng, strains, 20000, 150, 0.01, 0.1, 0.5)
    seqs = [bases[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)]
    for c in range(40):
        pick = rng.choice(len(strains), 60, replace=False)
        seqs.append(b"".join(records[int(j)][1][a:a + 200] for j, a in zip(pick, rng.integers(0, glen - 200, 60))))
    ids = [f"r{i}" for i in range(len(seqs))]
    tc.write_fasta(d / "reads.fa", list(zip(ids, seqs)), width=80)
    bases, offs = synth.pack_reads(seqs)
    run = oracle.run(oracle.open_db(kdb, np.fromfile(d / "database.idx", np.uint8)), oracle.parent_map(*ext.parent_map()), 500000, 0)
    calls, codes, code_off = run.classify(bases, offs)
    run.finish()
    want = run.counts()
    many = [len(set(codes[int(code_off[i]):int(code_off[i + 1])].tolist()) - {0, util.AMBIG}) for i in range(20000, len(seqs))]
    assert min(many) > 32, many

    r = _ours("classify", ["-d", "database.kdb", "-i", "database.idx", "-a", "taxDB", "-M", "-t", "1", "-o", "out.kraken",
                           "-r", "out.report", "reads.fa"], d)
    assert r.returncode == 0, r.stderr[-2000:]
    assert open(d / "out.kraken").read() == util.kraken_lines(ids, seqs, calls, codes, code_off)
    rows = util.parse_report(d / "out.report")
    members = util.clade_members(ext.rows(), want["taxid"][(want["n_reads"] > 0) | (want["n_kmers"] > 0)])
    assert set(rows) <= set(members)
    for t, row in rows.items():
        u, nr, _ = run.clade(members[t])
        assert (row["reads"], row["kmers"]) == (nr, u), t
    names = {r[0]: (r[2], r[3]) for r in ext.rows()}
    assert sum(t > 1_000_000_000 for t in rows) > 1000                 # strain-level rows
    for t, row in rows.items():
        assert (row["name"].strip(), row["rank"]) == names[t], t
