"""Inputs and expected outputs of the set_lcas -a / -A tests (tests/test_oracle_taxids_for_genomes.py against the
reference's recorded runs, tests/test_taxids_for_genomes_gpu.py for the drop-in on the same recordings).

One library holds the edge cases of the taxonomy extension: a `.N` suffix, two sequences of one assembly, an assembly
name with blanks, a repeated seq id in the map, human / mouse and a child of human, a contaminant (32630), a
`kraken:taxid|` header behind leading blanks, an assembly named like a later seq id, a parent missing from the taxDB,
a sequence shorter than -E, an empty record and an unmapped one."""
import os
import shutil

import numpy as np

from krakenuniq_b200 import synth
from oracle.taxids import Extension

K = 31
NT = 6
MIN_LEN = 100
# case → (-a, -A, -T, -E): the last one is build_db.sh's command line (build_db.sh:270-272)
CASES = {"a": (True, False, False, True), "A": (False, True, False, True), "aA": (True, True, False, True),
         "a_T": (True, False, True, False), "A_T": (False, True, True, False), "aA_T": (True, True, True, False)}


def command(case, threads=1):
    a, A, T, E = CASES[case]
    return (["-M", "-x", "-d", "database0.kdb", "-o", "database.kdb", "-i", "database.idx", "-v", "-b", "taxDB"]
            + (["-a"] if a else []) + (["-A"] if A else [])
            + ["-t", str(threads), "-m", "seqid2taxid.map", "-c", "database.kdb.counts", "-F", "lib.fa"]
            + (["-T"] if T else []) + (["-E", str(MIN_LEN)] if E else []))


def write_fasta(path, records, width=61):
    with open(path, "wb") as f:
        for header, seq in records:
            f.write(b">" + header.encode() + b"\n")
            for i in range(0, len(seq), width):
                f.write(seq[i:i + width] + b"\n")


def read_fasta(path):
    """(header line after '>', sequence) per record, as FastaReader reads them"""
    out = []
    for line in open(path, "rb").read().split(b"\n"):
        if line.startswith(b">"):
            out.append([line[1:].decode(), []])
        elif out:
            out[-1][1].append(line)
    return [(h, b"".join(s)) for h, s in out]


def library(seed=77):
    rng = np.random.default_rng(seed)
    tax = synth.make_taxonomy(6, 3, 2, first_id=100)
    sp = synth.species_ids(tax)
    rows = tax.rows + [(9605, 1, "Homo", "genus"), (9606, 9605, "Homo sapiens", "species"),
                       (63221, 9606, "Homo sapiens neanderthalensis", "subspecies"),
                       (10090, 1, "Mus musculus", "species"), (32630, 1, "synthetic construct", "species")]
    g = [synth.decode(x).tobytes() for x in synth.random_genomes(rng, 12, 1500, shared_frac=0.3)]
    novel = synth.decode(rng.integers(0, 4, 300, dtype=np.uint8)).tobytes()
    map_lines = [f"s0\t{sp[0]}\tasm0", f"s1\t{sp[0]}\tasm0", f"s2\t{sp[1]}\tasm1 strain X", f"s3\t{sp[2]}",
                 f"s2\t{sp[4]}\tasm_dup", "hs1\t9606\tGRCh38", "hs2\t63221\tneand", "mm1\t10090", "vec1\t32630",
                 f"s4\t{sp[3]}\ts5", f"s5\t{sp[4]}\tasm5", "s6\t4242\tasm6", f"short1\t{sp[5]}\tasm7", f"empty1\t{sp[5]}"]
    records = [("s0.1 chromosome one", g[0]), ("s1", g[1]), ("s2 some description", g[2]), ("s3", g[3]),
               ("hs1 human", g[4]), ("hs2 neanderthal", g[5]), ("mm1 mouse", g[6]),
               ("vec1 vector", g[2][200:500] + novel + g[0][900:1100]), ("s4", g[7]),
               (f"  kraken:taxid|{sp[3]}|x  extra words", g[11][300:1500]), ("s5", g[8]), ("s6", g[9]),
               ("short1", g[10][:80]), ("empty1", b""), ("unmapped1", g[11][:300])]
    return rng, rows, map_lines, records


def write_inputs(d, seed=77):
    """taxDB, seqid2taxid.map, lib.fa and an unsorted k-mer set (3 % of the library's k-mers left out: -x) in d"""
    rng, rows, map_lines, records = library(seed)
    synth.Taxonomy(rows).write(str(d / "taxDB"))
    with open(d / "seqid2taxid.map", "w") as f:
        f.write("".join(line + "\n" for line in map_lines))
    write_fasta(d / "lib.fa", records)
    ks = [np.zeros(0, np.uint64)]
    for _, s in records:
        if len(s) >= K:
            km, ok = synth.forward_kmers(synth.encode(s), K)
            ks.append(synth.canonical(km[ok], K))
    allk = np.unique(np.concatenate(ks))
    allk = allk[rng.random(len(allk)) >= 0.03]
    rng.shuffle(allk)
    synth.unsorted_jdb_image(allk, K).tofile(d / "database.jdb")


def run_reference(reference, d, case):
    """db_sort and set_lcas of the reference (recorded) in d/ref; d/in keeps the inputs of set_lcas"""
    ref, pristine = d / "ref", d / "in"
    ref.mkdir()
    write_inputs(ref)
    r = reference.run_tool("db_sort", ["-z", "-M", "-n", NT, "-d", "database.jdb", "-o", "database0.kdb", "-i", "database.idx"], cwd=ref)
    assert r.returncode == 0, r.stderr
    shutil.copytree(ref, pristine)
    r = reference.run_tool("set_lcas", command(case), cwd=ref)
    assert r.returncode == 0, r.stderr[-2000:]
    return ref, pristine, r


def counts_text(kdb):
    _, _, vals = synth.parse_kdb(kdb)
    t, c = np.unique(vals, return_counts=True)
    return "".join(f"{int(a)}\t{int(b)}\n" for a, b in zip(t, c))


def expected(oracle, d, add_sequences, add_assembly, contaminant, min_len):
    """the oracle's set_lcas on the inputs in d: (Extension, database image, .counts text)"""
    ext = Extension(synth.Taxonomy.read(str(d / "taxDB")).rows, open(d / "seqid2taxid.map").read().split("\n"),
                    add_sequences, add_assembly)
    records = read_fasta(d / "lib.fa")
    taxids = ext.assign(records, min_len)
    db = oracle.open_db(np.fromfile(d / "database0.kdb", np.uint8), np.fromfile(d / "database.idx", np.uint8))
    pm = oracle.parent_map(*ext.parent_map())
    for (_, s), t in zip(records, taxids):
        if t:
            oracle.set_lcas_sequence(db, pm, s, t, flags=1 if contaminant else 0)
    return ext, db.kdb, counts_text(db.kdb)


def outputs(d):
    """what set_lcas wrote: (database.kdb, taxDB, database.kdb.counts) bytes; database0.kdb stays as it was (-M -o)"""
    return tuple(open(os.path.join(d, n), "rb").read() for n in ("database.kdb", "taxDB", "database.kdb.counts"))
