"""`classify --sample-sheet`: many samples against one staging of the database.  Every file a row writes must be the
bytes a separate `classify` run of that row writes, in every database layout, and the golden reference outputs where
they exist.  The library side, kuq_reset_counts, must leave a context that answers like a freshly staged one."""
import gzip
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from krakenuniq_b200 import binding, build, synth
from tests import paired, util

pytestmark = pytest.mark.gpu
G, M = util.GOLDEN, os.path.join(os.path.dirname(util.GOLDEN), "multidb")
OUTS = {"output": "kraken", "report": "report", "classified_out": "C", "unclassified_out": "U"}
SEEN, KEPT = 0x80000000, 0x40000000


def _exe(tool="classify"):
    return os.path.join(os.path.dirname(build.build_classify()), tool)


def _setup(tmp_path, dbs=("database",)):
    for d in dbs:
        for ext in (".kdb", ".idx", ".kdb.counts"):
            shutil.copyfile(os.path.join(M if d == "db2" else G, d + ext), tmp_path / (d + ext))
    for f in ("taxDB", "reads.fa", "reads_300.fq", "reads_crlf_60.fa"):
        shutil.copyfile(os.path.join(G, f), tmp_path / f)
    data = open(os.path.join(G, "reads.fa"), "rb").read()
    at = [i for i in range(len(data)) if data.startswith(b"\n>", i)][99]
    (tmp_path / "prefix.fa").write_bytes(data[:at + 1])                # the first 100 records of reads.fa


def _common(dbs):
    return sum((["-d", f"{d}.kdb", "-i", f"{d}.idx"] for d in dbs), []) + ["-a", "taxDB"]


def _run(tmp_path, tool, args, env):
    return subprocess.run([_exe(tool)] + args, cwd=tmp_path, capture_output=True, text=True,
                          env=dict(os.environ, **env))


def _files(tmp_path, prefix, cols=OUTS):
    return {o: (tmp_path / f"{prefix}.{o}").read_bytes() if (tmp_path / f"{prefix}.{o}").exists() else None
            for o in cols.values()}


def _write_sheet(tmp_path, rows, tag, cols=OUTS):
    """rows: (name, input cell, input2 cell or None); every row writes <tag>.<name>.<kraken|report|C|U>"""
    paired_cols = rows[0][2] is not None
    head = ["name", "input"] + (["input2"] if paired_cols else []) + list(cols)
    lines = ["\t".join(head)]
    for name, inp, inp2 in rows:
        lines.append("\t".join([name, inp] + ([inp2] if paired_cols else []) + [f"{tag}.{name}.{v}" for v in cols.values()]))
    (tmp_path / f"{tag}.tsv").write_text("# sample sheet\n" + "\n".join(lines) + "\n")
    return f"{tag}.tsv"


def _separate(tmp_path, tool, flags, env, row, prefix, cols=OUTS):
    name, inp, inp2 = row
    opt = {"output": "-o", "report": "-r", "classified_out": "-C", "unclassified_out": "-U"}
    outs = sum(([opt[c], f"{prefix}.{v}"] for c, v in cols.items()), [])
    files = ["--paired", inp, inp2] if inp2 is not None else inp.split(",")
    r = _run(tmp_path, tool, flags + outs + files, env)
    return r, _files(tmp_path, prefix, cols)


def _stats(stderr):
    lines = stderr.replace("\r", "\n").splitlines()
    return [l.split(" processed in")[0] for l in lines if " processed in " in l]


def _sheet_vs_separate(tmp_path, tool, dbs, flags, env, rows, tag, cols=OUTS):
    """the sheet's files of every row, checked against a separate run of the row; returns both runs' results"""
    sheet = _write_sheet(tmp_path, rows, tag, cols)
    r = _run(tmp_path, tool, _common(dbs) + flags + ["--sample-sheet", sheet], env)
    seps = []
    for row in rows:
        s, want = _separate(tmp_path, tool, _common(dbs) + flags, env, row, f"{tag}.sep.{row[0]}", cols)
        assert s.returncode == 0, s.stderr[-2000:]
        assert _files(tmp_path, f"{tag}.{row[0]}", cols) == want, (tag, row)
        assert want["kraken"] or "-c" in flags
        seps.append(s)
    return r, seps


ROWS = [("fq", "reads_300.fq", None), ("fa", "reads.fa", None), ("prefix", "prefix.fa", None)]


def test_sheet_matches_reference_and_separate_runs(tmp_path):
    """4 samples, -M: the golden Kraken lines and report rows, the bytes of separate runs and one stats block per
    sample; then, without the database's .counts file, the sheet writes it once, as the first separate run does"""
    _setup(tmp_path)
    golden = {"fa": "preload", "fq": "fastq", "crlf": "crlf"}
    rows = [("fa", "reads.fa", None), ("fq", "reads_300.fq", None), ("crlf", "reads_crlf_60.fa", None),
            ("prefix", "prefix.fa", None)]
    r, _ = _sheet_vs_separate(tmp_path, "classify", ["database"], ["-M"], {}, rows, "s")
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout == ""
    for name, tag in golden.items():
        assert (tmp_path / f"s.{name}.kraken").read_bytes() == open(os.path.join(G, f"{tag}.kraken"), "rb").read(), name
        assert util.parse_report(tmp_path / f"s.{name}.report") == util.parse_report(os.path.join(G, f"{tag}.report.tsv"))
    stats, text = _stats(r.stderr), r.stderr.replace("\r", "\n")
    assert len(stats) == 4
    for i, (name, _, _) in enumerate(rows):                            # each block after the line naming its sample
        at = text.index(f"classify: sample {name} ({i + 1} of 4)")
        assert text.index(stats[i] + " processed in", at) < (text.index("classify: sample", at + 1) if i < 3 else len(text))

    (tmp_path / "database.kdb.counts").unlink()
    s, _ = _separate(tmp_path, "classify", _common(["database"]) + ["-M"], {}, rows[0], "first")
    assert s.returncode == 0, s.stderr[-2000:]
    counts = (tmp_path / "database.kdb.counts").read_bytes()
    (tmp_path / "database.kdb.counts").unlink()
    r = _run(tmp_path, "classify", _common(["database"]) + ["-M", "--sample-sheet", _write_sheet(tmp_path, rows[:2], "c")], {})
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stderr.count("Writing kmer counts") == 1
    assert (tmp_path / "database.kdb.counts").read_bytes() == counts


@pytest.mark.parametrize("order", ["reversed", "repeated"])
def test_no_state_carried_across_samples(tmp_path, order):
    _setup(tmp_path)
    rows = ROWS[::-1] if order == "reversed" else [("a", "reads.fa", None), ("b", "reads.fa", None), ("c", "reads.fa", None)]
    r, _ = _sheet_vs_separate(tmp_path, "classify", ["database"], ["-M"], {}, rows, order)
    assert r.returncode == 0, r.stderr[-2000:]
    if order == "repeated":
        assert len({(tmp_path / f"repeated.{n}.kraken").read_bytes() for n in "abc"}) == 1
        assert len({(tmp_path / f"repeated.{n}.report").read_bytes() for n in "abc"}) == 1


SHARD_ENV = {"KUQ_FORCE_SHARDS": "1", "KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"}
LAYOUTS = {
    "u20000": ("classify", ["database"], ["-M", "-u", "20000"], {}),
    "x40K": ("classify", ["database"], ["-x", "40K"], {}),
    "replicas": ("classify", ["database"], ["-M"], {"KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200",
                                                    "KUQ_SPARSE_SLOTS": str(1 << 12)}),
    "shards": ("classify", ["database"], ["-M"], SHARD_ENV),
    "streamed": ("classify", ["database"], ["-x", "40K"], {"KUQ_FORCE_CHUNKS": "1"}),
    "two_db_resident": ("classify", ["database", "db2"], ["-M"], {}),
    "two_db_sharded": ("classify", ["database", "db2"], ["-M"], SHARD_ENV),
    "two_db_streamed": ("classify", ["database", "db2"], ["-M"], {"KUQ_HBM_BUDGET": "200000"}),
    "q2": ("classify", ["database"], ["-M", "-q", "-m", "2"], {}),
    "exact": ("classifyExact", ["database"], ["-M"], {}),
    "exact_partitioned": ("classifyExact", ["database"], ["-M"], {"KUQ_DEVICES": "0,0", "KUQ_BATCH_READS": "200"}),
    "c_s": ("classify", ["database"], ["-M", "-c", "-s", "-t", "4"], {}),
    "serial": ("classify", ["database"], ["-M", "-t", "1"], {"KUQ_SERIAL_INGEST": "1"}),
}


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_every_layout_matches_separate_runs(tmp_path, layout):
    tool, dbs, flags, env = LAYOUTS[layout]
    _setup(tmp_path, dbs)
    rows = ROWS + [("two", "reads_crlf_60.fa,prefix.fa", None)]
    r, _ = _sheet_vs_separate(tmp_path, tool, dbs, flags, env, rows, layout)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "not usable" not in r.stderr
    if "KUQ_FORCE_SHARDS" in env:
        assert "sharded over 2 GPUs" in r.stderr
    if layout == "streamed":
        assert "Database split into" in r.stderr


def _mate_files(tmp_path, name, ids, seqs, rng, mismatch_at=None):
    pairs = paired.split_pairs(seqs, rng)
    r1 = [(f"{i}/1 mate one".encode(), a) for i, (a, _) in zip(ids, pairs)]
    r2 = [(f"{i}/2".encode(), b) for i, (_, b) in zip(ids, pairs)]
    if mismatch_at is not None:
        r2[mismatch_at] = (b"other/2", r2[mismatch_at][1])
    (tmp_path / f"{name}_1.fq").write_bytes(paired.fastq_bytes(r1))
    (tmp_path / f"{name}_2.fq").write_bytes(paired.fastq_bytes(r2))
    for k in (1, 2):
        with open(tmp_path / f"{name}_{k}.fq", "rb") as src, gzip.open(tmp_path / f"{name}_{k}.fq.gz", "wb") as dst:
            dst.write(src.read())


@pytest.mark.parametrize("gz", [False, True])
def test_paired_columns(tmp_path, gz):
    _setup(tmp_path)
    rng = np.random.default_rng(3)
    ids, seqs = util.read_fastq(os.path.join(G, "reads_300.fq"))
    _mate_files(tmp_path, "a", ids, seqs, rng)
    ids2, seqs2 = util.read_fasta(os.path.join(G, "reads.fa"))
    _mate_files(tmp_path, "b", ids2[:150], seqs2[:150], rng)
    x = ".gz" if gz else ""
    rows = [("a", f"a_1.fq{x}", f"a_2.fq{x}"), ("b", f"b_1.fq{x}", f"b_2.fq{x}")]
    r, _ = _sheet_vs_separate(tmp_path, "classify", ["database"], ["-M", "--paired", "--check-names"], {}, rows, "p")
    assert r.returncode == 0, r.stderr[-2000:]


def test_check_names_stop_lets_later_samples_run(tmp_path):
    _setup(tmp_path)
    rng = np.random.default_rng(4)
    ids, seqs = util.read_fastq(os.path.join(G, "reads_300.fq"))
    _mate_files(tmp_path, "bad", ids, seqs, rng, mismatch_at=150)
    _mate_files(tmp_path, "good", ids[:100], seqs[:100], rng)
    rows = [("bad", "bad_1.fq", "bad_2.fq"), ("good", "good_1.fq", "good_2.fq")]
    sheet = _write_sheet(tmp_path, rows, "n")
    flags = _common(["database"]) + ["-M", "--paired", "--check-names"]
    r = _run(tmp_path, "classify", flags + ["--sample-sheet", sheet], {})
    assert r.returncode == 65, r.stderr[-2000:]
    assert "classify: sample bad: mismatched mate pair names" in r.stderr
    for i, row in enumerate(rows):
        s, want = _separate(tmp_path, "classify", flags, {}, row, f"sep{i}")
        assert s.returncode == (65 if i == 0 else 0)
        assert _files(tmp_path, f"n.{row[0]}") == want, row
    assert 0 < (tmp_path / "n.bad.kraken").read_bytes().count(b"\n") < 300


def test_errors_stop_or_continue_like_separate_runs(tmp_path):
    """a malformed record in row 2 ends that sample's input as a separate run would (exit 0, the records before it), and
    row 3 still runs; an output that cannot be created in row 2 stops the run there with EX_CANTCREAT, after row 1's
    files are complete, and row 3 never starts"""
    _setup(tmp_path)
    data = (tmp_path / "reads_300.fq").read_bytes().split(b"\n")
    data[4 * 120 + 2] = b"-"                                           # record 121 loses its '+' line
    (tmp_path / "bad.fq").write_bytes(b"\n".join(data))
    rows = [("one", "reads.fa", None), ("bad", "bad.fq", None), ("three", "prefix.fa", None)]
    r, seps = _sheet_vs_separate(tmp_path, "classify", ["database"], ["-M"], {}, rows, "m")
    assert r.returncode == 0 and seps[1].returncode == 0, r.stderr[-2000:]
    assert (tmp_path / "m.bad.kraken").read_bytes().count(b"\n") == 120

    sheet = "name\tinput\toutput\treport\none\treads.fa\tc.one.kraken\tc.one.report\n" \
            "two\treads_300.fq\tno_such_dir/c.two.kraken\tc.two.report\nthree\tprefix.fa\tc.three.kraken\t\n"
    (tmp_path / "c.tsv").write_text(sheet)
    r = _run(tmp_path, "classify", _common(["database"]) + ["-M", "--sample-sheet", "c.tsv"], {})
    assert r.returncode == 73, r.stderr[-2000:]                       # EX_CANTCREAT, as a separate run of row 2
    assert "classify: sample two: can't open no_such_dir/c.two.kraken" in r.stderr
    s = _run(tmp_path, "classify", _common(["database"]) + ["-M", "-o", "sep.kraken", "-r", "sep.report", "reads.fa"], {})
    assert s.returncode == 0
    assert (tmp_path / "c.one.kraken").read_bytes() == (tmp_path / "sep.kraken").read_bytes()
    assert (tmp_path / "c.one.report").read_bytes() == (tmp_path / "sep.report").read_bytes()
    assert not (tmp_path / "c.three.kraken").exists()


# ---- the preloaded HLL rule across samples: sample 1 turns taxa dense and keeps records, sample 2 touches them lightly
def _synthetic(tmp_path):
    rng = np.random.default_rng(21)
    tax = synth.make_taxonomy(4, 2)
    genomes = synth.random_genomes(rng, 4, 30000)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, 31)
    kdb, idx = synth.build_db_images(km, tx, 31, 10, 2)
    kdb.tofile(tmp_path / "database.kdb")
    idx.tofile(tmp_path / "database.idx")
    tax.write(str(tmp_path / "taxDB"))
    for name, n, src in (("heavy", 3000, genomes[:3]), ("light", 6, genomes)):
        bases, offs = synth.sample_reads(rng, src, n, 150, 0.01, 0.0, 0.1)
        with open(tmp_path / f"{name}.fa", "wb") as f:
            for i in range(n):
                f.write(b">%s%d\n%s\n" % (name.encode(), i, bases[int(offs[i]):int(offs[i + 1])].tobytes()))
    return rng


@pytest.mark.parametrize("keep_at_harvest", [False, True])
def test_preload_rule_across_samples(tmp_path, keep_at_harvest):
    _synthetic(tmp_path)
    env = {"KUQ_KEEP_AT_HARVEST": "1"} if keep_at_harvest else {}
    rows = [("heavy", "heavy.fa", None), ("light", "light.fa", None)]
    r, _ = _sheet_vs_separate(tmp_path, "classify", ["database"], ["-M"], env, rows, "h")
    assert r.returncode == 0, r.stderr[-2000:]
    heavy, light = util.parse_report(tmp_path / "h.heavy.report"), util.parse_report(tmp_path / "h.light.report")
    assert any(row["kmers"] > 5000 for t, row in heavy.items() if t > 1)        # dense sketches in sample 1
    assert all(row["kmers"] < 1024 for row in light.values())                  # sparse ones in sample 2


# ---- kuq_reset_counts: a reset context is a fresh one ----------------------------------------------------------------
K, NT = 31, 10
HDR = len(binding.kdb_header(K, 0))


class Ctx:
    """a context on its own device copy of the records (kuq_attach_db_device), so their bytes can be read back"""

    def __init__(self, kdb, idx, tax, hll_mode=binding.HLL_PRELOAD):
        n = (kdb.size - HDR) // 12
        self.rec = torch.from_numpy(kdb[HDR:HDR + 12 * n].copy()).cuda()
        self.off = torch.from_numpy(idx[8:].copy().view(np.int64)).cuda()
        self.clf = binding.Classifier(n_slots=2, max_reads=1 << 14, max_bases=1 << 22, hll_mode=hll_mode,
                                      sparse_set_slots=1 << 12)
        self.clf.attach_db_device(self.rec.data_ptr(), n, self.off.data_ptr(), K, NT, 2)
        self.clf.set_taxonomy(*tax.parent_map())
        self.exact = hll_mode == binding.HLL_EXACT

    def words(self):
        torch.cuda.synchronize()
        return self.rec.cpu().numpy().view(np.uint32).reshape(-1, 3).copy()

    def run(self, bases, offs):
        self.clf.classify(bases, offs)
        self.clf.finish()

    def state(self, taxa=None):
        c = self.clf
        cn = c.counts()
        st = {k: v.tolist() for k, v in cn.items()}
        st["regs"] = [c.registers(t).tobytes() for t in cn["taxid"].tolist()]
        if taxa:
            st["clades"] = [x.tolist() for x in c.clade_counts_tree(taxa)]
        n = c.exact_export() if self.exact else c.sparse_export()
        buf = torch.zeros(2 * max(n, 1), dtype=torch.int64, device="cuda")
        if self.exact:
            c.exact_export(buf.data_ptr(), n)
            st["items"] = sorted(map(tuple, buf[:2 * n].view(-1, 2).tolist()))
        else:
            c.sparse_export(buf.data_ptr(), n)
            st["items"] = sorted(buf[:n].tolist())
        return st


def _reads(rng, genomes, n):
    return synth.sample_reads(rng, genomes, n, 150, 0.01, 0.0, 0.1)


def _lib_workload():
    rng = np.random.default_rng(8)
    tax = synth.make_taxonomy(4, 2)
    genomes = synth.random_genomes(rng, 4, 30000)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, K)
    kdb, idx = synth.build_db_images(km, tx, K, NT, 2)
    first = _reads(rng, genomes[:3], 3000)                             # dense taxa, many kept records
    second = _reads(rng, genomes, 60)                                  # light hits on the same taxa
    taxa = [t for t, *_ in tax.rows]
    return tax, kdb, idx, first, second, taxa


def _halves(bases, offs):
    n = len(offs) - 1
    a = offs[:n // 2 + 1]
    b = offs[n // 2:] - offs[n // 2]
    return (bases, a), (bases[int(offs[n // 2]):], b)


@pytest.mark.parametrize("case", ["keep", "flag_and_harvest", "merge_from", "exact_partition", "sparse_replace_summary"])
def test_reset_context_equals_fresh_context(monkeypatch, case):
    if case == "flag_and_harvest":
        monkeypatch.setenv("KUQ_KEEP_AT_HARVEST", "1")
    tax, kdb, idx, first, second, taxa = _lib_workload()
    mode = binding.HLL_EXACT if case == "exact_partition" else binding.HLL_PRELOAD
    world = 2 if case in ("merge_from", "exact_partition") else 1

    def one_run(ctxs, reads):
        parts = _halves(*reads) if world == 2 else [reads]
        for c, (b, o) in zip(ctxs, parts):
            c.run(b, o)
        if case == "merge_from":
            ctxs[0].clf.merge_from(ctxs[1].clf)
        elif case == "exact_partition":
            binding.Classifier.exact_partition([c.clf for c in ctxs])
        elif case == "sparse_replace_summary":
            c = ctxs[0].clf
            n_sketch = len(c.dense_taxids())
            hist = torch.zeros(n_sketch * 64, dtype=torch.int32, device="cuda")
            distinct = torch.zeros(n_sketch, dtype=torch.int32, device="cuda")
            c.sparse_summary(hist.data_ptr(), distinct.data_ptr())
            n = c.sparse_export()
            keys = torch.zeros(max(n, 1), dtype=torch.int64, device="cuda")
            c.sparse_export(keys.data_ptr(), n)
            c.sparse_replace(keys.data_ptr(), n)
            c.set_sparse_summary(hist.data_ptr(), distinct.data_ptr())
            torch.cuda.synchronize()

    used = [Ctx(kdb, idx, tax, mode) for _ in range(world)]
    staged = [c.words() for c in used]
    one_run(used, first)
    flagged = [c.words() for c in used]
    if case in ("keep", "merge_from"):
        assert any(((w[:, 1] & KEPT) != 0).any() for w in flagged)          # sample 1 left kept records behind
    for c in used:
        c.clf.reset_counts()
    for c, w, f in zip(used, staged, flagged):
        after = c.words()
        assert not (after[:, 1] & (SEEN | KEPT)).any()
        f[:, 1] &= ~np.uint32(SEEN | KEPT)
        assert np.array_equal(after, f)                                    # nothing else of the records changed
        assert np.array_equal(after[:, 0], w[:, 0]) and np.array_equal(after[:, 1] & 0x3FFFFFFF, w[:, 1] & 0x3FFFFFFF)
    one_run(used, second)
    fresh = [Ctx(kdb, idx, tax, mode) for _ in range(world)]
    one_run(fresh, second)
    # every context's counters, registers, keys or pairs; the first one's clades (the one that holds the summaries;
    # a partitioned sparse tier answers clades only summed over the GPUs)
    for i, (u, f) in enumerate(zip(used, fresh)):
        clades = taxa if i == 0 and case != "sparse_replace_summary" else None
        assert u.state(clades) == f.state(clades), (case, i)
    for c in used + fresh:
        c.clf.close()
