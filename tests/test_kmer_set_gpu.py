"""`kmer_set` / kuq_kmer_set_*: the k-mer set of a FASTA library on the GPU, step 1 of build_db.sh.

The golden database is rebuilt from its library through kmer_set + db_sort + set_lcas byte for byte; every record size
(k = 15 .. 31) is held against the oracle's KmerScanner over FastaReader records; the bytes do not depend on batch size,
number of passes, where the packed library lives, pipe or file input, or executable versus C ABI; the strict set_lcas
(without -x) accepts the result; empty input gives an empty set."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import binding, build, synth
from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tools():
    db_sort, set_lcas = build.build_dbtools()
    return build.KMER_SET, db_sort, set_lcas


def _write_fasta(path, names, seqs, width=None, crlf=False):
    nl = b"\r\n" if crlf else b"\n"
    with open(path, "wb") as f:
        for n, s in zip(names, seqs):
            f.write(b">" + n + nl)
            w = width or max(len(s), 1)
            for i in range(0, len(s), w):
                f.write(s[i:i + w] + nl)


def _expected(paths, k, oracle):
    """header + records of np.unique over the canonical non-ambiguous KmerScanner windows of every FastaReader record"""
    parts = []
    for p in paths:
        for s in util.read_fasta(p)[1]:
            km, amb = oracle.scan(s, k)
            parts.append(synth.canonical(km[amb == 0], k))
    keys, counts = np.unique(np.concatenate(parts) if parts else np.zeros(0, np.uint64), return_counts=True)
    return np.concatenate([synth.kdb_header(k, len(keys)), synth.pack_records(keys, counts.astype(np.uint32), k)])


def _run(exe, k, inputs, cwd, env=None, pipe=False, prefix="database"):
    files = " ".join(f"<(cat {i})" if pipe else str(i) for i in inputs)
    cmd = f"{exe} count -m {k} -s 1M -C -t 4 -o {prefix} {files}"
    r = subprocess.run(["bash", "-c", cmd], capture_output=True, text=True, cwd=cwd, env={**os.environ, **(env or {})})
    assert r.returncode == 0, r.stderr
    out = os.path.join(cwd, prefix + "_0")
    img = np.fromfile(out, np.uint8)
    os.remove(out)
    return img, r.stderr


def _passes(stderr):
    return int(stderr.split(" pass")[0].rsplit(" ", 1)[1])


def _library(path):
    ids, seqs = util.read_fasta(path)
    return synth.pack_reads([s for s in seqs])


def _budget_for(bases, offs, k, want_image, min_passes):
    """the first of a falling series of HBM budgets whose run takes >= min_passes passes (each run checked against
    want_image); the series ends just above the 512 KiB the key histogram takes"""
    for i in range(80):
        b = (1 << 19) + int((1 << 23) * 0.87 ** i)
        try:
            img, passes = binding.kmer_set(bases, offs, k, budget=b, batch=1 << 20)
        except binding.KuqError as e:
            assert e.code == -7 and "KUQ_KMER_SET_BUDGET" in str(e)
            break
        assert np.array_equal(img, want_image), b
        if passes >= min_passes:
            return b, passes
    pytest.fail(f"no budget gives {min_passes} passes")


# ---- 1. the golden database, rebuilt from its library ------------------------------------------------------------
def _golden_library(d):
    """lib.fa and seqid2taxid.map as tests/golden/make_golden.py writes them"""
    rng = np.random.default_rng(1)
    tax = synth.make_taxonomy(6, 3, 2, first_id=100)
    sp = synth.species_ids(tax)
    genomes = synth.random_genomes(rng, 6, 1800, shared_frac=0.2)
    orphan = rng.integers(0, 4, 900, dtype=np.uint8)
    names = [f"seq{i}".encode() for i in range(6)] + [b"orphan"]
    seqs = [synth.decode(g).tobytes() for g in genomes + [orphan]]
    _write_fasta(os.path.join(d, "lib.fa"), names, seqs, width=70)
    with open(os.path.join(d, "seqid2taxid.map"), "w") as f:
        for n, t in zip(names, sp + [900]):
            f.write(f"{n.decode()}\t{t}\n")
    shutil.copy(os.path.join(util.GOLDEN, "taxDB"), os.path.join(d, "taxDB"))
    return genomes + [orphan]


def test_golden_database_rebuilt_from_its_library(tools, tmp_path, oracle):
    exe, db_sort, set_lcas = tools
    genomes = _golden_library(tmp_path)
    # self-check: the library's canonical set is the golden database's key set
    ks = []
    for g in genomes:
        km, ok = synth.forward_kmers(g, 31)
        ks.append(synth.canonical(km[ok], 31))
    _, gold_keys, _ = synth.parse_kdb(np.fromfile(os.path.join(util.GOLDEN, "database.kdb"), np.uint8))
    assert np.array_equal(np.unique(np.concatenate(ks)), np.sort(gold_keys)) and len(gold_keys) == 9840
    want = _expected([tmp_path / "lib.fa"], 31, oracle)
    bases, offs = _library(tmp_path / "lib.fa")
    budget, passes = _budget_for(bases, offs, 31, want, 4)
    for env in ({}, {"KUQ_KMER_SET_BUDGET": str(budget)}):
        img, err = _run(exe, 31, ["lib.fa"], tmp_path, env, pipe=True)
        assert np.array_equal(img, want)
        assert _passes(err) == (passes if env else 1), err
        img.tofile(tmp_path / "database.jdb")
        for f in ("database0.kdb", "database.kdb", "database.idx"):
            if os.path.exists(tmp_path / f):
                os.remove(tmp_path / f)
        subprocess.run([db_sort, "-z", "-n", "6", "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"],
                       cwd=tmp_path, check=True, capture_output=True)
        subprocess.run([set_lcas, "-x", "-d", "database0.kdb", "-o", "database.kdb", "-i", "database.idx", "-b", "taxDB",
                        "-m", "seqid2taxid.map", "-F", "lib.fa"], cwd=tmp_path, check=True, capture_output=True)
        for f in ("database.kdb", "database.idx"):
            assert (tmp_path / f).read_bytes() == open(os.path.join(util.GOLDEN, f), "rb").read(), (f, env)


# ---- 2. every record size against the oracle --------------------------------------------------------------------
def _edge_library(d, seed):
    """two FASTA files with lowercase, N and IUPAC letters, records shorter than k, header-only records, a 100 kbp
    poly-A run, mixed line widths, CRLF line ends and descriptions after the id"""
    rng = np.random.default_rng(seed)
    g = [synth.decode(x).tobytes() for x in synth.random_genomes(rng, 5, 6000, shared_frac=0.3)]
    iupac = bytearray(g[1])
    for i, c in zip(rng.integers(0, len(iupac), 60), rng.choice(list(b"NRYKMSWBDHVn"), 60)):
        iupac[int(i)] = int(c)
    names1 = [b"lower some description", b"iupac\tmore", b"short", b"empty", b"polyA", b"mixed"]
    seqs1 = [g[0][:3000].lower() + g[0][3000:], bytes(iupac), g[2][:14], b"", b"A" * 100000 + g[2][100:400],
             g[3] + g[3][:500]]
    _write_fasta(os.path.join(d, "a.fa"), names1, seqs1, width=60)
    with open(os.path.join(d, "a.fa"), "ab") as f:               # mixed line widths inside one record
        f.write(b">ragged\n" + b"\n".join(g[4][i:i + w] for i, w in zip(range(0, 4000, 97), [97, 13, 1, 80] * 50)) + b"\n")
    names2 = [b"crlf with words", b"tiny", b"headeronly", b"last"]
    seqs2 = [g[4][:2500], b"ACG", b"", g[0][1000:2000] + b"N" + g[1][:700]]
    _write_fasta(os.path.join(d, "b.fa"), names2, seqs2, width=71, crlf=True)
    return [os.path.join(d, "a.fa"), os.path.join(d, "b.fa")]


@pytest.mark.parametrize("k", [15, 19, 21, 25, 31])
def test_every_record_size_matches_oracle(tools, tmp_path, oracle, k):
    exe = tools[0]
    inputs = _edge_library(tmp_path, 40 + k)
    want = _expected(inputs, k, oracle)
    assert int(np.frombuffer(want[48:56].tobytes(), np.uint64)[0]) > 1000
    img, err = _run(exe, k, inputs, tmp_path)
    assert np.array_equal(img, want), err
    # the C ABI on the FastaReader records, '\r' of the CRLF file included
    seqs = [s for p in inputs for s in util.read_fasta(p)[1]]
    assert any(b"\r" in s for s in seqs)
    img, _ = binding.kmer_set(*synth.pack_reads(seqs), k, batch=3000)
    assert np.array_equal(img, want)


# ---- 3. invariance ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [31, 21])
def test_bytes_do_not_depend_on_batches_passes_or_input(tools, tmp_path, oracle, k):
    exe = tools[0]
    rng = np.random.default_rng(7 + k)
    g = [synth.decode(x).tobytes() for x in synth.random_genomes(rng, 6, 20000, shared_frac=0.3)]
    g[0] = g[0][:5000] + b"N" + g[0][5000:]
    _write_fasta(tmp_path / "lib.fa", [f"s{i} d".encode() for i in range(len(g))] + [b"t"], g + [b"ACGTTGCA" * 9], width=80)
    want = _expected([tmp_path / "lib.fa"], k, oracle)
    base, err = _run(exe, k, ["lib.fa"], tmp_path)
    assert np.array_equal(base, want) and _passes(err) == 1
    # a batch of 7000 bases: every 20 kbp sequence spans >= 3 batches
    img, _ = _run(exe, k, ["lib.fa"], tmp_path, {"KUQ_KMER_SET_BATCH": "7000"})
    assert np.array_equal(img, base)
    # pipe input
    img, _ = _run(exe, k, ["lib.fa"], tmp_path, pipe=True)
    assert np.array_equal(img, base)
    # the C ABI
    bases, offs = _library(tmp_path / "lib.fa")
    img, passes = binding.kmer_set(bases, offs, k)
    assert np.array_equal(img, base) and passes == 1
    img, _ = binding.kmer_set(bases, offs, k, batch=7000)
    assert np.array_equal(img, base)
    # >= 8 passes with the packed library in pinned host memory, through the executable and the C ABI
    budget, passes = _budget_for(bases, offs, k, base, 8)
    ks = binding.KmerSet(k, budget)
    ks.add(bases, offs)
    buf = np.zeros(1000 * ks.rec, np.uint8)
    parts = []
    while True:
        n = ks.next(buf)
        if not n:
            break
        parts.append(buf[:n * ks.rec].copy())
    st = ks.stats()
    n_keys = sum(len(x) for x in parts) // ks.rec
    assert ks.info() == (n_keys, passes)
    assert not st["library_in_hbm"] and st["windows"] == int(synth.parse_kdb(base)[2].sum())
    ks.close()
    assert np.array_equal(np.concatenate([synth.kdb_header(k, n_keys)] + parts), base)
    img, err = _run(exe, k, ["lib.fa"], tmp_path, {"KUQ_KMER_SET_BUDGET": str(budget), "KUQ_KMER_SET_BATCH": str(1 << 20)},
                    pipe=True)
    assert np.array_equal(img, base) and _passes(err) >= 8


def test_budget_too_small_is_a_clean_error(tools, tmp_path):
    exe = tools[0]
    _write_fasta(tmp_path / "lib.fa", [b"polyA"], [b"A" * 50000])
    r = subprocess.run([exe, "count", "-m", "31", "-s", "1M", "-C", "-o", "database", "lib.fa"], capture_output=True,
                       text=True, cwd=tmp_path, env={**os.environ, "KUQ_KMER_SET_BUDGET": "100000"})
    assert r.returncode != 0 and "KUQ_KMER_SET_BUDGET" in r.stderr
    assert not list(tmp_path.glob("database*"))


# ---- 4. the strict set_lcas accepts the database -----------------------------------------------------------------
@pytest.mark.parametrize("k", [31, 21])
def test_strict_set_lcas_finds_every_kmer(tools, tmp_path, k):
    exe, db_sort, set_lcas = tools
    rng = np.random.default_rng(100 + k)
    tax = synth.make_taxonomy(5)
    sp = synth.species_ids(tax)
    g = [synth.decode(x).tobytes() for x in synth.random_genomes(rng, 5, 5000, shared_frac=0.3)]
    g[1] = g[1][:2000].lower() + b"NNRY" + g[1][2000:]
    names = [f"s{i}".encode() for i in range(5)]
    _write_fasta(tmp_path / "lib.fa", names, g, width=60)
    (tmp_path / "map").write_text("".join(f"s{i}\t{t}\n" for i, t in enumerate(sp)))
    tax.write(tmp_path / "taxDB")
    img, _ = _run(exe, k, ["lib.fa"], tmp_path, pipe=True)
    img.tofile(tmp_path / "database.jdb")
    subprocess.run([db_sort, "-z", "-n", "8", "-d", "database.jdb", "-o", "database.kdb", "-i", "database.idx"],
                   cwd=tmp_path, check=True, capture_output=True)
    r = subprocess.run([set_lcas, "-d", "database.kdb", "-i", "database.idx", "-b", "taxDB", "-m", "map", "-F", "lib.fa"],
                       cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


# ---- 5. empty input ----------------------------------------------------------------------------------------------
def test_empty_input_gives_an_empty_set(tools, tmp_path):
    exe, db_sort, _ = tools
    (tmp_path / "empty.fa").write_bytes(b"")
    img, err = _run(exe, 25, ["empty.fa"], tmp_path, pipe=True)
    assert np.array_equal(img, synth.kdb_header(25, 0)) and _passes(err) == 0
    img.tofile(tmp_path / "database.jdb")
    r = subprocess.run([db_sort, "-z", "-n", "5", "-d", "database.jdb", "-o", "database.kdb", "-i", "database.idx"],
                       cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert os.path.getsize(tmp_path / "database.kdb") == len(img)
