"""ctypes bindings for the CPU oracle — TEST INFRASTRUCTURE ONLY.

Two libraries live behind this module:

* ``oracle/libkuq_oracle.so`` — the plain-C restatement (``kuq_oracle.c``), class :class:`Oracle`.
* ``oracle/_ref/libkuref.so`` — the UNMODIFIED reference classes behind a thin veneer (``ref_shim.cpp``),
  class :class:`RefShim`, plus the reference executables ``oracle/_ref/{classify,db_sort,set_lcas}``.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` legs may import
this module (as the checker, never as the thing measured or shipped).  Nothing under ``krakenuniq_b200/`` does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "libkuq_oracle.so")
REF_DIR = os.path.join(HERE, "_ref")
REF_SO = os.path.join(REF_DIR, "libkuref.so")
AMBIG = 0xFFFFFFFF

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)


def _p(arr, typ):
    return arr.ctypes.data_as(typ)


def build_oracle():
    """(Re)build libkuq_oracle.so with gcc.  Building the checker is not using it."""
    subprocess.run(["make", "-C", HERE, "-s"], check=True)
    return ORACLE_SO


def build_reference():
    """Build oracle/_ref from the reference sources named by KUQ_REFERENCE_SRC."""
    subprocess.run([os.path.join(HERE, "build_ref.sh")], check=True)


def have_reference():
    return os.path.exists(REF_SO) and os.path.exists(os.path.join(REF_DIR, "classify"))


class _DB(C.Structure):
    _fields_ = [("pairs", C.c_void_p), ("key_ct", C.c_uint64), ("k", C.c_uint), ("key_bits", C.c_uint),
                ("key_len", C.c_uint), ("pair_sz", C.c_uint), ("offsets", C.c_void_p), ("nt", C.c_uint),
                ("idx_type", C.c_int)]


class Oracle:
    """The plain-C restatement (oracle/kuq_oracle.c)."""

    def __init__(self):
        if not os.path.exists(ORACLE_SO) or os.path.getmtime(ORACLE_SO) < os.path.getmtime(
                os.path.join(HERE, "kuq_oracle.c")):
            build_oracle()
        L = self.L = C.CDLL(ORACLE_SO)
        L.kuqo_fmix64.restype = C.c_uint64
        L.kuqo_fmix64.argtypes = [C.c_uint64]
        L.kuqo_revcomp.restype = C.c_uint64
        L.kuqo_revcomp.argtypes = [C.c_uint64, C.c_uint]
        L.kuqo_canonical.restype = C.c_uint64
        L.kuqo_canonical.argtypes = [C.c_uint64, C.c_uint]
        L.kuqo_bin_key.restype = C.c_uint64
        L.kuqo_bin_key.argtypes = [C.c_uint64, C.c_uint, C.c_uint, C.c_int]
        L.kuqo_scan.restype = C.c_uint32
        L.kuqo_scan.argtypes = [C.c_char_p, C.c_size_t, C.c_uint, u64p, u8p]
        L.kuqo_db_open.restype = C.c_int
        L.kuqo_db_open.argtypes = [C.POINTER(_DB), C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
        L.kuqo_kmer_query.restype = C.c_int
        L.kuqo_kmer_query.argtypes = [C.POINTER(_DB), C.c_uint64, u32p]
        L.kuqo_parent_map_new.restype = C.c_void_p
        L.kuqo_parent_map_new.argtypes = [u32p, u32p, C.c_uint32]
        L.kuqo_parent_map_free.argtypes = [C.c_void_p]
        L.kuqo_lca.restype = C.c_uint32
        L.kuqo_lca.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        L.kuqo_resolve_tree.restype = C.c_uint32
        L.kuqo_resolve_tree.argtypes = [C.c_void_p, u32p, u32p, C.c_uint32]
        L.kuqo_hll_new.restype = C.c_void_p
        L.kuqo_hll_free.argtypes = [C.c_void_p]
        L.kuqo_hll_insert.argtypes = [C.c_void_p, C.c_uint64]
        L.kuqo_hll_merge.argtypes = [C.c_void_p, C.c_void_p]
        L.kuqo_hll_cardinality.restype = C.c_uint64
        L.kuqo_hll_cardinality.argtypes = [C.c_void_p]
        L.kuqo_hll_is_sparse.restype = C.c_int
        L.kuqo_hll_is_sparse.argtypes = [C.c_void_p]
        L.kuqo_hll_n_observed.restype = C.c_uint64
        L.kuqo_hll_n_observed.argtypes = [C.c_void_p]
        L.kuqo_hll_sparse_size.restype = C.c_uint32
        L.kuqo_hll_sparse_size.argtypes = [C.c_void_p]
        L.kuqo_hll_registers.argtypes = [C.c_void_p, u8p]
        L.kuqo_ertl_dense.restype = C.c_uint64
        L.kuqo_ertl_dense.argtypes = [u8p, C.c_uint64]
        L.kuqo_encode_hash32.restype = C.c_uint32
        L.kuqo_encode_hash32.argtypes = [C.c_uint64]
        L.kuqo_classify_read.restype = C.c_uint32
        L.kuqo_classify_read.argtypes = [C.POINTER(_DB), C.c_void_p, C.c_char_p, C.c_size_t, u32p, u32p]
        L.kuqo_hitlist_string.restype = C.c_size_t
        L.kuqo_hitlist_string.argtypes = [u32p, C.c_uint32, C.c_char_p, C.c_size_t]
        L.kuqo_run_new.restype = C.c_void_p
        L.kuqo_run_new.argtypes = [C.POINTER(_DB), C.c_void_p, C.c_uint64, C.c_int]
        L.kuqo_run_free.argtypes = [C.c_void_p]
        L.kuqo_run_classify.restype = C.c_int
        L.kuqo_run_classify.argtypes = [C.c_void_p, C.c_char_p, u64p, C.c_uint32, u32p, u32p, u64p]
        L.kuqo_run_finish.argtypes = [C.c_void_p]
        L.kuqo_run_n_taxa.restype = C.c_uint32
        L.kuqo_run_n_taxa.argtypes = [C.c_void_p]
        L.kuqo_run_counts.argtypes = [C.c_void_p, u32p, u64p, u64p, u64p, u8p, u8p]
        L.kuqo_run_add_db.restype = C.c_int
        L.kuqo_run_add_db.argtypes = [C.c_void_p, C.POINTER(_DB)]
        L.kuqo_run_clade.restype = C.c_uint64
        L.kuqo_run_clade.argtypes = [C.c_void_p, u32p, C.c_uint32, u64p, u64p]

    # -- scalar helpers -------------------------------------------------------------------------------
    def fmix64(self, x):
        return self.L.kuqo_fmix64(x)

    def revcomp(self, kmer, n):
        return self.L.kuqo_revcomp(kmer, n)

    def canonical(self, kmer, n):
        return self.L.kuqo_canonical(kmer, n)

    def bin_key(self, kmer, k, nt, idx_type=2):
        return self.L.kuqo_bin_key(kmer, k, nt, idx_type)

    def scan(self, seq: bytes, k: int):
        cap = max(len(seq) - k + 2, 1)
        kmers = np.zeros(cap, np.uint64)
        amb = np.zeros(cap, np.uint8)
        n = self.L.kuqo_scan(seq, len(seq), k, _p(kmers, u64p), _p(amb, u8p))
        return kmers[:n].copy(), amb[:n].copy()

    def encode_hash32(self, h):
        return self.L.kuqo_encode_hash32(h)

    def ertl_dense(self, regs: np.ndarray, n_observed: int):
        regs = np.ascontiguousarray(regs, np.uint8)
        assert regs.size == 4096
        return self.L.kuqo_ertl_dense(_p(regs, u8p), n_observed)

    # -- database / taxonomy ----------------------------------------------------------------------------
    def open_db(self, kdb: np.ndarray, idx: np.ndarray):
        return OracleDB(self, kdb, idx)

    def parent_map(self, taxid, parent):
        return OracleParentMap(self, taxid, parent)

    def hll(self):
        return OracleHLL(self)

    def hitlist_string(self, codes: np.ndarray) -> str:
        codes = np.ascontiguousarray(codes, np.uint32)
        cap = 24 * (len(codes) + 1)
        buf = C.create_string_buffer(cap)
        n = self.L.kuqo_hitlist_string(_p(codes, u32p), len(codes), buf, cap)
        return buf.raw[:n].decode()

    def classify_read(self, db, pm, seq: bytes):
        codes = np.zeros(max(len(seq), 1) + 2, np.uint32)
        nw = C.c_uint32(0)
        call = self.L.kuqo_classify_read(C.byref(db.s), pm.h, seq, len(seq), _p(codes, u32p), C.byref(nw))
        return call, codes[:nw.value].copy()

    def db_sort(self, jdb: np.ndarray, nt: int, zero_vals=False):
        """db_sort [-z] -n nt: unsorted Jellyfish-style image → (database.kdb image, KRAKIX2 index image)"""
        jdb = np.ascontiguousarray(jdb, np.uint8)
        kdb = np.zeros(jdb.size, np.uint8)
        idx = np.zeros(8 + 8 * (4 ** nt + 1), np.uint8)
        self.L.kuqo_db_sort.restype = C.c_int
        self.L.kuqo_db_sort.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p]
        rc = self.L.kuqo_db_sort(jdb.ctypes.data, jdb.size, nt, 1 if zero_vals else 0, kdb.ctypes.data, idx.ctypes.data)
        if rc != 0:
            raise ValueError(f"kuqo_db_sort failed: {rc}")
        return kdb, idx

    def set_lcas_sequence(self, db: "OracleDB", pm, seq: bytes, taxid: int, flags: int = 0) -> int:
        """set_lcas for one library sequence; updates db.kdb (the image the OracleDB was opened on) in place.
        flags: 1 = -T, 2 = -R"""
        f = self.L.kuqo_set_lcas_sequence_flags
        f.restype = C.c_uint64
        f.argtypes = [C.POINTER(_DB), C.c_void_p, C.c_char_p, C.c_size_t, C.c_uint32, C.c_uint32]
        return f(C.byref(db.s), pm.h, seq, len(seq), taxid, flags)

    def run(self, db, pm, work_unit_size=500000, mode=0):
        return OracleRun(self, db, pm, work_unit_size, mode)


class OracleDB:
    def __init__(self, o: Oracle, kdb: np.ndarray, idx: np.ndarray):
        self.o = o
        self.kdb = np.ascontiguousarray(kdb, np.uint8)     # keep the images alive
        self.idx = np.ascontiguousarray(idx, np.uint8)
        self.s = _DB()
        rc = o.L.kuqo_db_open(C.byref(self.s), self.kdb.ctypes.data, self.kdb.size, self.idx.ctypes.data,
                              self.idx.size)
        if rc != 0:
            raise ValueError(f"kuqo_db_open failed: {rc}")
        self.k, self.nt, self.idx_type, self.key_ct = self.s.k, self.s.nt, self.s.idx_type, self.s.key_ct

    def query(self, canon: int):
        t = C.c_uint32(0)
        found = self.o.L.kuqo_kmer_query(C.byref(self.s), canon, C.byref(t))
        return (True, t.value) if found else (False, 0)


class OracleParentMap:
    def __init__(self, o: Oracle, taxid, parent):
        self.o = o
        t = np.ascontiguousarray(taxid, np.uint32)
        p = np.ascontiguousarray(parent, np.uint32)
        self.h = C.c_void_p(o.L.kuqo_parent_map_new(_p(t, u32p), _p(p, u32p), len(t)))

    def __del__(self):
        try:
            self.o.L.kuqo_parent_map_free(self.h)
        except Exception:
            pass

    def lca(self, a, b):
        return self.o.L.kuqo_lca(self.h, a, b)

    def resolve_tree(self, hits: dict):
        t = np.array(list(hits.keys()), np.uint32)
        c = np.array(list(hits.values()), np.uint32)
        return self.o.L.kuqo_resolve_tree(self.h, _p(t, u32p), _p(c, u32p), len(t))


class OracleHLL:
    def __init__(self, o: Oracle):
        self.o = o
        self.h = C.c_void_p(o.L.kuqo_hll_new())

    def __del__(self):
        try:
            self.o.L.kuqo_hll_free(self.h)
        except Exception:
            pass

    def insert(self, items):
        for x in np.asarray(items, np.uint64).tolist():
            self.o.L.kuqo_hll_insert(self.h, x)

    def merge(self, other: "OracleHLL"):
        self.o.L.kuqo_hll_merge(self.h, other.h)

    def cardinality(self):
        return self.o.L.kuqo_hll_cardinality(self.h)

    def is_sparse(self):
        return bool(self.o.L.kuqo_hll_is_sparse(self.h))

    def n_observed(self):
        return self.o.L.kuqo_hll_n_observed(self.h)

    def sparse_size(self):
        return self.o.L.kuqo_hll_sparse_size(self.h)

    def registers(self):
        r = np.zeros(4096, np.uint8)
        self.o.L.kuqo_hll_registers(self.h, _p(r, u8p))
        return r


class OracleRun:
    """process_file() work-unit loop over in-memory reads (mode 0 = preload rule, 1 = chunked rule)."""

    def __init__(self, o: Oracle, db: OracleDB, pm: OracleParentMap, work_unit_size, mode):
        self.o, self.db, self.pm = o, db, pm
        self.h = C.c_void_p(o.L.kuqo_run_new(C.byref(db.s), pm.h, work_unit_size, mode))

    def __del__(self):
        try:
            self.o.L.kuqo_run_free(self.h)
        except Exception:
            pass

    def add_db(self, db: "OracleDB"):
        """a further database, tried after the earlier ones for every k-mer (classify -d a -d b)"""
        self._more = getattr(self, "_more", []) + [db]
        if self.o.L.kuqo_run_add_db(self.h, C.byref(db.s)) != 0:
            raise ValueError("databases must share k")

    def set_exact(self, on=True):
        """classifyExact: exact distinct counts instead of HLL estimates"""
        self.o.L.kuqo_run_set_exact.argtypes = [C.c_void_p, C.c_int]
        self.o.L.kuqo_run_set_exact.restype = None
        self.o.L.kuqo_run_set_exact(self.h, 1 if on else 0)

    def set_quick(self, min_hits: int):
        """classify -q -m min_hits (0 = off)"""
        self.o.L.kuqo_run_set_quick.argtypes = [C.c_void_p, C.c_uint32]
        self.o.L.kuqo_run_set_quick.restype = None
        self.o.L.kuqo_run_set_quick(self.h, min_hits)

    def classify(self, bases: np.ndarray, offsets: np.ndarray, want_codes=True):
        bases = np.ascontiguousarray(bases, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.uint64)
        n = len(offsets) - 1
        calls = np.zeros(n, np.uint32)
        code_off = np.zeros(n + 1, np.uint64)
        codes = np.zeros(int(offsets[-1] - offsets[0]) + n + 1, np.uint32) if want_codes else None
        buf = bases.tobytes() if bases.size else b"\0"
        self.o.L.kuqo_run_classify(self.h, buf, _p(offsets, u64p), n, _p(calls, u32p),
                                   _p(codes, u32p) if want_codes else None, _p(code_off, u64p))
        if want_codes:
            codes = codes[:int(code_off[-1])].copy()
        return calls, codes, code_off

    def finish(self):
        self.o.L.kuqo_run_finish(self.h)

    def counts(self, want_regs=False):
        n = self.o.L.kuqo_run_n_taxa(self.h)
        taxid = np.zeros(n, np.uint32)
        n_reads = np.zeros(n, np.uint64)
        n_kmers = np.zeros(n, np.uint64)
        est = np.zeros(n, np.uint64)
        sparse = np.zeros(n, np.uint8)
        regs = np.zeros((n, 4096), np.uint8) if want_regs else None
        self.o.L.kuqo_run_counts(self.h, _p(taxid, u32p), _p(n_reads, u64p), _p(n_kmers, u64p), _p(est, u64p),
                                 _p(sparse, u8p), _p(regs, u8p) if want_regs else None)
        out = dict(taxid=taxid, n_reads=n_reads, n_kmers=n_kmers, unique=est, sparse=sparse)
        if want_regs:
            out["regs"] = regs
        return out


    def clade(self, taxa):
        """(unique estimate, reads, kmers) of the union of the listed taxa (TaxReport clade roll-up)."""
        t = np.ascontiguousarray(taxa, np.uint32)
        r, k = C.c_uint64(0), C.c_uint64(0)
        u = self.o.L.kuqo_run_clade(self.h, _p(t, u32p), len(t), C.byref(r), C.byref(k))
        return u, r.value, k.value


class RefShim:
    """The reference's own classes (oracle/_ref/libkuref.so).  KmerScanner's k is process-global (31 here)."""

    def __init__(self):
        if not os.path.exists(REF_SO):
            raise FileNotFoundError(REF_SO)
        L = self.L = C.CDLL(REF_SO)
        L.kuref_murmur_fmix.restype = C.c_uint64
        L.kuref_murmur_fmix.argtypes = [C.c_uint64]
        L.kuref_db_open.restype = C.c_void_p
        L.kuref_db_open.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        for name in ("kuref_db_k", "kuref_db_index_nt", "kuref_db_index_type"):
            getattr(L, name).restype = C.c_uint32
            getattr(L, name).argtypes = [C.c_void_p]
        L.kuref_revcomp.restype = C.c_uint64
        L.kuref_revcomp.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32]
        L.kuref_canonical.restype = C.c_uint64
        L.kuref_canonical.argtypes = [C.c_void_p, C.c_uint64]
        L.kuref_bin_key.restype = C.c_uint64
        L.kuref_bin_key.argtypes = [C.c_void_p, C.c_uint64]
        L.kuref_bin_key_nt.restype = C.c_uint64
        L.kuref_bin_key_nt.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32]
        L.kuref_kmer_query.restype = C.c_uint64
        L.kuref_kmer_query.argtypes = [C.c_void_p, C.c_uint64]
        L.kuref_kmer_query_stateful.argtypes = [C.c_void_p, u64p, C.c_uint32, u32p]
        L.kuref_scan.restype = C.c_uint32
        L.kuref_scan.argtypes = [C.c_char_p, C.c_uint64, C.c_uint32, u64p, u8p]
        L.kuref_lca.restype = C.c_uint32
        L.kuref_lca.argtypes = [u32p, u32p, C.c_uint32, C.c_uint32, C.c_uint32]
        L.kuref_parent_map_new.restype = C.c_void_p
        L.kuref_parent_map_new.argtypes = [u32p, u32p, C.c_uint32]
        L.kuref_parent_map_free.argtypes = [C.c_void_p]
        L.kuref_lca_pm.restype = C.c_uint32
        L.kuref_lca_pm.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        L.kuref_resolve_tree.restype = C.c_uint32
        L.kuref_resolve_tree.argtypes = [C.c_void_p, u32p, u32p, C.c_uint32]
        L.kuref_hll_new.restype = C.c_void_p
        L.kuref_hll_new_dense.restype = C.c_void_p
        L.kuref_hll_new_dense.argtypes = [C.c_uint32]
        L.kuref_hll_free.argtypes = [C.c_void_p]
        L.kuref_hll_insert.argtypes = [C.c_void_p, u64p, C.c_uint64]
        L.kuref_hll_merge.argtypes = [C.c_void_p, C.c_void_p]
        L.kuref_hll_merge_move.argtypes = [C.c_void_p, C.c_void_p]
        L.kuref_hll_cardinality.restype = C.c_uint64
        L.kuref_hll_cardinality.argtypes = [C.c_void_p]
        L.kuref_hll_n_observed.restype = C.c_uint64
        L.kuref_hll_n_observed.argtypes = [C.c_void_p]
        L.kuref_get_rank64.restype = C.c_uint32
        L.kuref_get_rank64.argtypes = [C.c_uint64, C.c_uint32]
        L.kuref_get_encoded_rank.restype = C.c_uint32
        L.kuref_get_encoded_rank.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]

    def open_db(self, kdb: np.ndarray, idx: np.ndarray):
        return RefDB(self, kdb, idx)

    def scan(self, seq: bytes, k=31):
        cap = max(len(seq) - k + 2, 1)
        kmers = np.zeros(cap, np.uint64)
        amb = np.zeros(cap, np.uint8)
        n = self.L.kuref_scan(seq, len(seq), k, _p(kmers, u64p), _p(amb, u8p))
        if n == 0xFFFFFFFF:
            raise RuntimeError("KmerScanner::k already fixed to another value in this process")
        return kmers[:n].copy(), amb[:n].copy()

    def parent_map(self, taxid, parent):
        return RefParentMap(self, taxid, parent)


class RefDB:
    def __init__(self, r: RefShim, kdb, idx):
        self.r = r
        self.kdb = np.ascontiguousarray(kdb, np.uint8).copy()
        self.idx = np.ascontiguousarray(idx, np.uint8).copy()
        self.h = C.c_void_p(r.L.kuref_db_open(self.kdb.ctypes.data, self.kdb.size, self.idx.ctypes.data))

    def canonical(self, kmer):
        return self.r.L.kuref_canonical(self.h, kmer)

    def revcomp(self, kmer, n):
        return self.r.L.kuref_revcomp(self.h, kmer, n)

    def bin_key(self, kmer):
        return self.r.L.kuref_bin_key(self.h, kmer)

    def bin_key_nt(self, kmer, nt):
        return self.r.L.kuref_bin_key_nt(self.h, kmer, nt)

    def query(self, canon):
        v = self.r.L.kuref_kmer_query(self.h, canon)
        return (True, v - 1) if v else (False, 0)

    def query_stateful(self, canon: np.ndarray):
        canon = np.ascontiguousarray(canon, np.uint64)
        out = np.zeros(len(canon), np.uint32)
        self.r.L.kuref_kmer_query_stateful(self.h, _p(canon, u64p), len(canon), _p(out, u32p))
        return out


class RefParentMap:
    def __init__(self, r: RefShim, taxid, parent):
        self.r = r
        t = np.ascontiguousarray(taxid, np.uint32)
        p = np.ascontiguousarray(parent, np.uint32)
        self.h = C.c_void_p(r.L.kuref_parent_map_new(_p(t, u32p), _p(p, u32p), len(t)))

    def __del__(self):
        try:
            self.r.L.kuref_parent_map_free(self.h)
        except Exception:
            pass

    def lca(self, a, b):
        return self.r.L.kuref_lca_pm(self.h, a, b)

    def resolve_tree(self, hits: dict):
        t = np.array(list(hits.keys()), np.uint32)
        c = np.array(list(hits.values()), np.uint32)
        return self.r.L.kuref_resolve_tree(self.h, _p(t, u32p), _p(c, u32p), len(t))


class RefHLL:
    def __init__(self, r: RefShim, dense_p=None):
        self.r = r
        self.h = C.c_void_p(r.L.kuref_hll_new() if dense_p is None else r.L.kuref_hll_new_dense(dense_p))

    def __del__(self):
        try:
            self.r.L.kuref_hll_free(self.h)
        except Exception:
            pass

    def insert(self, items):
        a = np.ascontiguousarray(items, np.uint64)
        self.r.L.kuref_hll_insert(self.h, _p(a, u64p), len(a))

    def merge(self, other: "RefHLL", move=False):
        (self.r.L.kuref_hll_merge_move if move else self.r.L.kuref_hll_merge)(self.h, other.h)

    def cardinality(self):
        return self.r.L.kuref_hll_cardinality(self.h)

    def n_observed(self):
        return self.r.L.kuref_hll_n_observed(self.h)


def run_ref_tool(tool: str, args, cwd=None, stdin=None):
    """Run one of the reference executables built into oracle/_ref/ (classify, db_sort, set_lcas, classifyExact)."""
    exe = os.path.join(REF_DIR, tool)
    return subprocess.run([exe] + [str(a) for a in args], cwd=cwd, stdin=stdin, capture_output=True, text=True)
