"""Databases with k <= 28, whose records are shorter than 12 bytes (key_len + 4 = 8..11 bytes): the oracle against the
UNMODIFIED reference `classify`, `db_sort` and `set_lcas` (their recorded outputs, tests/ref_replay.py), and the numpy
database builder against the reference's db_sort.  One case per record size; Kraken lines byte for byte, report rows
exactly."""
import zlib

import numpy as np
import pytest

from krakenuniq_b200 import synth
from tests import util
from tests.test_oracle_live_reference import _report_equals, _write_fasta

CASES = [
    # tag, k, nt, idx_type, n_species, genome length, reads, classify flags, oracle (unit, mode); record bytes in the name
    ("k15_nt8_8B", 15, 8, 2, 6, 2200, 900, ["-M"], (500000, 0)),
    ("k19_nt10_krakidx_9B", 19, 10, 1, 7, 2000, 900, ["-M"], (500000, 0)),
    ("k21_nt12_10B", 21, 12, 2, 8, 2400, 1000, ["-M"], (500000, 0)),
    ("k25_nt11_small_units_11B", 25, 11, 2, 5, 3000, 1200, ["-M", "-u", "3000"], (3000, 0)),
    ("k28_nt9_chunked_11B", 28, 9, 2, 5, 1800, 700, ["-x", "40K"], (500000, 1)),
]


@pytest.mark.parametrize("tag,k,nt,idx_type,n_sp,glen,n_reads,flags,omode", CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_reference_short_k(oracle, reference, tmp_path, tag, k, nt, idx_type, n_sp, glen, n_reads, flags, omode):
    rng = np.random.default_rng(zlib.crc32(tag.encode()))
    tax = synth.make_taxonomy(n_sp, max(2, n_sp // 2), 2)
    genomes = synth.random_genomes(rng, n_sp, glen, shared_frac=0.25)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, k)
    kdb, idx = synth.build_db_images(km, tx, k, nt, idx_type)
    assert len(kdb) == len(synth.kdb_header(k, 0)) + len(km) * (synth.key_len(k) + 4)
    kdb.tofile(tmp_path / "database.kdb")
    idx.tofile(tmp_path / "database.idx")
    tax.write(str(tmp_path / "taxDB"))
    bases, offs = synth.sample_reads(rng, genomes, n_reads, 150, 0.01, 0.15, 0.15)
    seqs = [bases[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n_reads)]
    g0 = synth.decode(genomes[0]).tobytes()
    seqs += [b"", b"ACG", g0[:k - 1], g0[:k], g0[5:5 + k] + b"N" + g0[400:400 + k + 3], b"N" * 90, g0[100:460],
             g0[600:700].lower()]
    ids = [f"r{i}" for i in range(len(seqs))]
    _write_fasta(tmp_path / "reads.fa", ids, seqs)
    r = reference.run_tool("classify", ["-d", "database.kdb", "-i", "database.idx", "-a", "taxDB", "-t", 1, "-r", "ref.report",
                                        "-o", "ref.kraken"] + flags + ["reads.fa"], cwd=tmp_path)
    assert r.returncode == 0, r.stderr[-1500:]

    run = oracle.run(oracle.open_db(kdb, idx), oracle.parent_map(*tax.parent_map()), *omode)
    b2, o2 = synth.pack_reads(seqs)
    calls, codes, code_off = run.classify(b2, o2)
    run.finish()
    assert (calls != 0).sum() > n_reads // 2
    assert util.kraken_lines(ids, seqs, calls, codes, code_off) == open(tmp_path / "ref.kraken").read()
    _report_equals(run, tax, tmp_path / "ref.report")


def _library_kmers(rng, genomes, k):
    ks = []
    for g in genomes:
        km, ok = synth.forward_kmers(g, k)
        ks.append(synth.canonical(km[ok], k))
    allk = np.unique(np.concatenate(ks))
    rng.shuffle(allk)
    return allk


@pytest.mark.parametrize("k,nt", [(21, 9), (25, 10)])
def test_numpy_builder_equals_reference_db_sort(reference, tmp_path, k, nt):
    """synth.build_db_images packs and orders records like the reference's db_sort for every record size"""
    rng = np.random.default_rng(300 + k)
    genomes = synth.random_genomes(rng, 5, 1500, shared_frac=0.3)
    allk = _library_kmers(rng, genomes, k)
    vals = rng.integers(1, 1 << 20, len(allk)).astype(np.uint32)
    jdb = np.concatenate([synth.kdb_header(k, len(allk)), synth.pack_records(allk, vals, k)])
    jdb.tofile(tmp_path / "in.jdb")
    r = reference.run_tool("db_sort", ["-n", nt, "-d", "in.jdb", "-o", "out.kdb", "-i", "out.idx"], cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    kdb, idx = synth.build_db_images(allk, vals, k, nt, 2)
    assert np.array_equal(np.fromfile(tmp_path / "out.kdb", np.uint8), kdb)
    assert np.array_equal(np.fromfile(tmp_path / "out.idx", np.uint8), idx)
    k2, keys, taxa = synth.parse_kdb(kdb)
    assert k2 == k and set(keys.tolist()) == set(allk.tolist())
    assert dict(zip(keys.tolist(), taxa.tolist())) == dict(zip(allk.tolist(), vals.tolist()))


def test_db_sort_and_set_lcas_k21_match_reference(oracle, reference, tmp_path):
    """db_sort -z and set_lcas -x at k = 21 (10-byte records): the oracle's tools equal the reference's byte for byte"""
    k = 21
    rng = np.random.default_rng(2121)
    tax = synth.make_taxonomy(6, 3, 2, first_id=100)
    sp = synth.species_ids(tax)
    genomes = synth.random_genomes(rng, 6, 1500, shared_frac=0.3)
    allk = _library_kmers(rng, genomes, k)
    extra = rng.integers(0, 4, 500, dtype=np.uint8)
    names = [f"seq{i}" for i in range(len(genomes))] + ["novel"]
    seqs = [synth.decode(g).tobytes() for g in genomes] + [synth.decode(genomes[2][:300]).tobytes() + b"N" + synth.decode(extra).tobytes()]
    taxids = list(sp) + [sp[4]]
    with open(tmp_path / "lib.fa", "wb") as f:
        for n, s in zip(names, seqs):
            f.write(b">" + n.encode() + b"\n")
            for i in range(0, len(s), 70):
                f.write(s[i:i + 70] + b"\n")
    with open(tmp_path / "seqid2taxid.map", "w") as f:
        for n, t in zip(names, taxids):
            f.write(f"{n}\t{t}\n")
    tax.write(str(tmp_path / "taxDB"))
    jdb = synth.unsorted_jdb_image(allk, k)
    jdb.tofile(tmp_path / "database.jdb")
    r = reference.run_tool("db_sort", ["-z", "-n", 8, "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"], cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    kdb0 = np.fromfile(tmp_path / "database0.kdb", np.uint8)
    idx = np.fromfile(tmp_path / "database.idx", np.uint8)
    okdb, oidx = oracle.db_sort(jdb, 8, True)
    assert np.array_equal(okdb, kdb0) and np.array_equal(oidx, idx)
    r = reference.run_tool("set_lcas", ["-x", "-d", "database0.kdb", "-i", "database.idx", "-b", "taxDB", "-m",
                                        "seqid2taxid.map", "-F", "lib.fa"], cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    want = np.fromfile(tmp_path / "database0.kdb", np.uint8)
    assert not np.array_equal(want, kdb0)
    ids, parents = tax.parent_map()
    pm = oracle.parent_map(ids, parents)
    db = oracle.open_db(kdb0.copy(), idx)
    missing = sum(oracle.set_lcas_sequence(db, pm, s, t) for s, t in zip(seqs, taxids))
    assert missing > 0
    assert np.array_equal(db.kdb, want)
    km, tx = synth.label_kmers(genomes + [genomes[2][:300]], list(sp) + [sp[4]], tax, k)
    _, keys, vals = synth.parse_kdb(db.kdb)
    got = dict(zip(keys.tolist(), vals.tolist()))
    assert all(got[a] == b for a, b in zip(km.tolist(), tx.tolist()))
