"""Synthetic KrakenUniq workloads (numpy, host side): genomes, taxonomy, database.kdb / database.idx images, reads.

This is workload generation for tests and for the small bench configurations — it is not on the classification
path.  File layouts follow the reference byte for byte (SURVEY.md App. B):

* database.kdb  — ``JFLISTDN`` header (krakendb.cpp:60-78,177) + packed {key, u32 taxon} records sorted by
  (bin_key, key) (db_sort.cpp:80-116); the key takes ceil(2k / 8) little-endian bytes, so a record is 12 bytes for
  k = 29..31 and 8 to 11 bytes for k = 13..28;
* database.idx  — ``KRAKIX2``/``KRAKIDX`` + nt byte + 4^nt+1 u64 offsets (krakendb.cpp:118-148,534-544);
* taxDB         — ``taxid \\t parent \\t name \\t rank`` (taxdb.hpp:563-605).
"""
from __future__ import annotations

import numpy as np

INDEX2_XOR_MASK = 0xE37E28C4271B5A2D  # krakendb.cpp:45
_CODE = np.full(256, 4, np.uint8)
for _i, _c in enumerate("ACGT"):
    _CODE[ord(_c)] = _i
    _CODE[ord(_c.lower())] = _i
_BASES = np.frombuffer(b"ACGT", np.uint8)
_U = np.uint64


def encode(seq: np.ndarray | bytes) -> np.ndarray:
    """ASCII → 0..3, 4 = ambiguous (krakenutil.cpp:253-273)."""
    a = np.frombuffer(seq, np.uint8) if isinstance(seq, (bytes, bytearray)) else np.asarray(seq, np.uint8)
    return _CODE[a]


def decode(codes: np.ndarray) -> np.ndarray:
    return _BASES[np.asarray(codes, np.uint8)]


def forward_kmers(codes: np.ndarray, k: int):
    """All k-mer windows of a code array (first base in the most significant bits, krakenutil.cpp:250).
    Returns (kmers u64[n-k+1], valid bool[n-k+1]); windows touching an ambiguous base are invalid."""
    n = len(codes) - k + 1
    if n <= 0:
        return np.zeros(0, np.uint64), np.zeros(0, bool)
    km = np.zeros(n, np.uint64)
    bad = np.zeros(n, bool)
    for j in range(k):
        c = codes[j:j + n]
        km = (km << _U(2)) | (c & 3).astype(np.uint64)
        bad |= c > 3
    return km, ~bad


def revcomp(kmers: np.ndarray, n: int) -> np.ndarray:
    """krakendb.cpp:218-225"""
    x = np.asarray(kmers, np.uint64)
    x = ((x >> _U(2)) & _U(0x3333333333333333)) | ((x & _U(0x3333333333333333)) << _U(2))
    x = ((x >> _U(4)) & _U(0x0F0F0F0F0F0F0F0F)) | ((x & _U(0x0F0F0F0F0F0F0F0F)) << _U(4))
    x = ((x >> _U(8)) & _U(0x00FF00FF00FF00FF)) | ((x & _U(0x00FF00FF00FF00FF)) << _U(8))
    x = ((x >> _U(16)) & _U(0x0000FFFF0000FFFF)) | ((x & _U(0x0000FFFF0000FFFF)) << _U(16))
    x = (x >> _U(32)) | (x << _U(32))
    return (~x) >> _U(64 - 2 * n)


def canonical(kmers: np.ndarray, n: int) -> np.ndarray:
    """krakendb.cpp:238-246"""
    return np.minimum(kmers, revcomp(kmers, n))


def bin_key(kmers: np.ndarray, k: int, nt: int, idx_type: int = 2) -> np.ndarray:
    """krakendb.cpp:200-215"""
    mask = _U((1 << (2 * nt)) - 1)
    xor = _U((0 if idx_type == 1 else INDEX2_XOR_MASK) & ((1 << (2 * nt)) - 1))
    x = np.asarray(kmers, np.uint64).copy()
    best = np.full(len(x), np.iinfo(np.uint64).max, np.uint64)
    for _ in range(k - nt + 1):
        best = np.minimum(best, xor ^ canonical(x & mask, nt))
        x >>= _U(2)
    return best


def kdb_header(k: int, key_ct: int) -> np.ndarray:
    """Jellyfish-1 style header with every ignored field zero (SURVEY App. A16)."""
    key_bits = 2 * k
    size = 72 + 2 * (4 + 8 * key_bits)
    h = np.zeros(size, np.uint8)
    h[:8] = np.frombuffer(b"JFLISTDN", np.uint8)
    h[8:16] = np.frombuffer(np.uint64(key_bits).tobytes(), np.uint8)
    h[16:24] = np.frombuffer(np.uint64(4).tobytes(), np.uint8)
    h[48:56] = np.frombuffer(np.uint64(key_ct).tobytes(), np.uint8)
    return h


_REC = np.dtype([("key", "<u8"), ("taxon", "<u4")])  # packed: itemsize 12, the records of k = 29..31


def key_len(k: int) -> int:
    """bytes of a key in database.kdb (krakendb.cpp:76)"""
    return (2 * k + 7) // 8


def pack_records(keys: np.ndarray, vals: np.ndarray, k: int) -> np.ndarray:
    """packed {key_len-byte key, u32 value} records, little-endian, as one uint8 array"""
    kl = key_len(k)
    assert 1 <= kl <= 8
    keys = np.ascontiguousarray(keys, "<u8")
    vals = np.ascontiguousarray(vals, "<u4")
    rec = np.zeros((len(keys), kl + 4), np.uint8)
    rec[:, :kl] = keys.view(np.uint8).reshape(-1, 8)[:, :kl]
    rec[:, kl:] = vals.view(np.uint8).reshape(-1, 4)
    return rec.reshape(-1)


def build_db_images(kmers: np.ndarray, taxa: np.ndarray, k: int = 31, nt: int = 8, idx_type: int = 2):
    """(canonical k-mer, taxon) pairs → (database.kdb image, database.idx image) as uint8 arrays, for any k <= 31
    (records of key_len(k) + 4 bytes)."""
    assert 1 <= k <= 31 and nt <= k
    kmers = np.asarray(kmers, np.uint64)
    taxa = np.asarray(taxa, np.uint32)
    bins = bin_key(kmers, k, nt, idx_type)
    order = np.lexsort((kmers, bins))
    kdb = np.concatenate([kdb_header(k, len(kmers)), pack_records(kmers[order], taxa[order], k)])
    n_bins = 1 << (2 * nt)
    counts = np.bincount(bins.astype(np.int64), minlength=n_bins)
    offsets = np.zeros(n_bins + 1, np.uint64)
    np.cumsum(counts, out=offsets[1:])
    magic = b"KRAKIDX" if idx_type == 1 else b"KRAKIX2"
    idx = np.concatenate([np.frombuffer(magic, np.uint8), np.array([nt], np.uint8), offsets.view(np.uint8)])
    return kdb, idx


def unsorted_jdb_image(kmers: np.ndarray, k: int = 31) -> np.ndarray:
    """A `database.jdb` as Jellyfish would dump it (unsorted keys, zero values) for the reference's db_sort."""
    kmers = np.asarray(kmers, np.uint64)
    return np.concatenate([kdb_header(k, len(kmers)), pack_records(kmers, np.zeros(len(kmers), np.uint32), k)])


def parse_kdb(kdb: np.ndarray):
    """→ (k, keys u64[n], taxa u32[n]) from a database.kdb image of any record size."""
    key_bits = int(np.frombuffer(kdb[8:16].tobytes(), np.uint64)[0])
    key_ct = int(np.frombuffer(kdb[48:56].tobytes(), np.uint64)[0])
    header = 72 + 2 * (4 + 8 * key_bits)
    kl = key_len(key_bits // 2)
    rec = np.frombuffer(kdb[header:header + (kl + 4) * key_ct].tobytes(), np.uint8).reshape(key_ct, kl + 4)
    keys = np.zeros((key_ct, 8), np.uint8)
    keys[:, :kl] = rec[:, :kl]
    taxa = np.ascontiguousarray(rec[:, kl:]).view("<u4").reshape(-1)
    return key_bits // 2, keys.view("<u8").reshape(-1).astype(np.uint64), taxa.astype(np.uint32)


class Taxonomy:
    """taxid → parent table + the Parent_map view the classifier uses (taxdb.hpp:383-398: root → 0)."""

    def __init__(self, rows):
        # rows: list of (taxid, parent_taxid, name, rank); the root has parent == taxid
        self.rows = list(rows)

    def parent_map(self):
        ids = {r[0] for r in self.rows}
        taxid = np.array([r[0] for r in self.rows if r[0] != 0], np.uint32)
        parent = np.array([(0 if (r[1] == r[0] or r[1] not in ids) else r[1]) for r in self.rows if r[0] != 0],
                          np.uint32)
        return taxid, parent

    def write(self, path):
        with open(path, "w") as f:
            for t, p, name, rank in self.rows:
                f.write(f"{t}\t{p}\t{name}\t{rank}\n")

    @staticmethod
    def read(path):
        rows = []
        with open(path) as f:
            for line in f:
                line = line.rstrip("\n")
                if not line:
                    continue
                t, p, name, rank = (line.split("\t") + ["", ""])[:4]
                rows.append((int(t), int(p), name, rank))
        return Taxonomy(rows)

    def lca(self, a, b):
        """plain tree LCA used only to label synthetic database k-mers (set_lcas.cpp:461 analogue)"""
        if a == 0 or b == 0:
            return a or b
        par = {r[0]: r[1] for r in self.rows}
        path = set()
        while a and a not in path:
            path.add(a)
            a = par.get(a, 0) if par.get(a, 0) != a else 0
        seen = set()
        while b and b not in seen:
            if b in path:
                return b
            seen.add(b)
            b = par.get(b, 0) if par.get(b, 0) != b else 0
        return 1


def make_taxonomy(n_species: int, n_genera: int = 0, n_families: int = 0, first_id: int = 100) -> Taxonomy:
    """root(1) → families → genera → species; ids ascending from first_id.  Returns the Taxonomy; species ids
    are returned by `species_ids(tax)`."""
    n_genera = n_genera or max(1, n_species // 3)
    n_families = n_families or max(1, n_genera // 3)
    rows = [(1, 1, "root", "no rank")]
    nid = first_id
    fam = []
    for i in range(n_families):
        rows.append((nid, 1, f"family{i}", "family"))
        fam.append(nid)
        nid += 1
    gen = []
    for i in range(n_genera):
        rows.append((nid, fam[i % n_families], f"genus{i}", "genus"))
        gen.append(nid)
        nid += 1
    for i in range(n_species):
        rows.append((nid, gen[i % n_genera], f"species{i}", "species"))
        nid += 1
    return Taxonomy(rows)


def add_upper_ranks(rows):
    """rows with superkingdom, kingdom, phylum, class and order nodes (ids 2..17) between the root and the families that
    hang from it, so that every rank code of the MetaPhlAn-style report occurs"""
    upper = [(2, 1, "Bacteria", "superkingdom"), (3, 2, "Kingdom one", "kingdom"), (4, 3, "Phylum a", "phylum"),
             (5, 3, "Phylum b", "phylum")]
    upper += [(6 + i, 4 + i % 2, f"Class {i}", "class") for i in range(4)]
    upper += [(10 + i, 6 + i % 4, f"Order {i}", "order") for i in range(8)]
    out, n_fam = [], 0
    for t, p, name, rank in rows:
        if rank == "family" and p == 1:
            p = 10 + n_fam % 8
            n_fam += 1
        out.append((t, p, name, rank))
    return out[:1] + upper + out[1:]


def species_ids(tax: Taxonomy):
    return [r[0] for r in tax.rows if r[3] == "species"]


def random_genomes(rng: np.random.Generator, n: int, length: int, shared_frac: float = 0.15):
    """n random genomes (code arrays); a `shared_frac` slice of genome i is copied from genome i-1 so that some
    k-mers belong to several taxa (→ LCA labels in the database)."""
    g = [rng.integers(0, 4, length, dtype=np.uint8) for _ in range(n)]
    sh = int(length * shared_frac)
    for i in range(1, n):
        if sh > 0:
            a = int(rng.integers(0, length - sh))
            b = int(rng.integers(0, length - sh))
            g[i][b:b + sh] = g[i - 1][a:a + sh]
    return g


def label_kmers(genomes, taxids, tax: Taxonomy, k: int = 31):
    """canonical k-mers of all genomes with the LCA of their owners → (kmers u64 sorted, taxa u32)."""
    ks, ts = [], []
    for g, t in zip(genomes, taxids):
        km, ok = forward_kmers(g, k)
        c = canonical(km[ok], k)
        c = np.unique(c)
        ks.append(c)
        ts.append(np.full(len(c), t, np.uint32))
    allk = np.concatenate(ks)
    allt = np.concatenate(ts)
    order = np.argsort(allk, kind="stable")
    allk, allt = allk[order], allt[order]
    uk, start, cnt = np.unique(allk, return_index=True, return_counts=True)
    ut = allt[start].copy()
    for i in np.nonzero(cnt > 1)[0]:
        t = 0
        for v in np.unique(allt[start[i]:start[i] + cnt[i]]):
            t = tax.lca(t, int(v))
        ut[i] = t
    return uk, ut


def sample_reads(rng: np.random.Generator, genomes, n_reads: int, read_len: int = 150, sub_rate: float = 0.01,
                 n_frac: float = 0.0, random_frac: float = 0.2, revcomp_frac: float = 0.5):
    """Reads as one uint8 ASCII buffer + offsets u64[n_reads+1]."""
    out = np.zeros(n_reads * read_len, np.uint8)
    comp = np.array([3, 2, 1, 0], np.uint8)
    for i in range(n_reads):
        if rng.random() < random_frac:
            r = rng.integers(0, 4, read_len, dtype=np.uint8)
        else:
            g = genomes[int(rng.integers(0, len(genomes)))]
            s = int(rng.integers(0, len(g) - read_len + 1))
            r = g[s:s + read_len].copy()
            if sub_rate > 0:
                m = rng.random(read_len) < sub_rate
                r[m] = (r[m] + rng.integers(1, 4, int(m.sum()), dtype=np.uint8)) & 3
            if rng.random() < revcomp_frac:
                r = comp[r[::-1]]
        a = decode(r).copy()
        if n_frac > 0 and rng.random() < n_frac:
            a[int(rng.integers(0, read_len))] = ord("N")
        out[i * read_len:(i + 1) * read_len] = a
    offsets = (np.arange(n_reads + 1, dtype=np.uint64) * np.uint64(read_len))
    return out, offsets


def pack_reads(seqs):
    """list of bytes → (uint8 buffer, offsets u64[n+1])"""
    offsets = np.zeros(len(seqs) + 1, np.uint64)
    np.cumsum([len(s) for s in seqs], out=offsets[1:])
    buf = np.frombuffer(b"".join(seqs), np.uint8).copy() if seqs else np.zeros(0, np.uint8)
    return buf, offsets


def work_unit_ids(offsets: np.ndarray, work_unit_size: int = 500000, carry_nt: int = 0, first_unit: int = 0):
    """Work-unit id of every read, following process_file (classify.cpp:506-521): consecutive reads are added
    to a unit until its total length reaches `work_unit_size`.  Returns (unit_id u32[n], carry_nt, next_unit)
    so that batches can be chained like one input stream."""
    lens = np.diff(np.asarray(offsets, np.uint64)).astype(np.int64)
    ids = np.zeros(len(lens), np.uint32)
    unit, tot = first_unit, carry_nt
    for i, ln in enumerate(lens.tolist()):
        ids[i] = unit
        tot += ln
        if tot >= work_unit_size:
            unit += 1
            tot = 0
    return ids, tot, unit
