"""ctypes binding of libkuq.so (include/kuq.h) — the host-side mirror of the reference's classify driver objects.

`Classifier` plays the role of the globals `KrakenDatabases` / `Parent_map` / `taxon_counts` of
src/classify.cpp:78-113 and of its per-read function `classify_sequence()` (:897-1012): stage a database, set
the taxonomy, push batches of reads, read per-read calls / hit lists and the per-taxon counters back.

There is no CPU path here: if libkuq.so is missing or no sm_90 device is present this module raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import build as _build

AMBIG = 0xFFFFFFFF
CODE_FOUND_ZERO = 0xFFFFFFFD      # KUQ_CODE_FOUND_ZERO: the first database holding the k-mer stores taxon 0
LOOKUP_FILL_EMPTY = 2             # KUQ_LOOKUP_FILL_EMPTY (lookup_device only_hits)
HLL_PRELOAD, HLL_CHUNKED, HLL_DENSE_ONLY, HLL_EXACT = 0, 1, 2, 3
F_WANT_CODES, F_NO_RUNS, F_NO_COUNTS, F_STATS = 1, 2, 4, 8
EXTRACT_SUBTREE, EXTRACT_INVERT, EXTRACT_OTHERS, EXTRACT_CLASSIFIED_ONLY = 1, 2, 4, 8     # kuq_set_extract flags

u8p, u32p, u64p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)


class KuqError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libkuq error {code}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("n_slots", C.c_uint32), ("max_reads_per_batch", C.c_uint32),
                ("max_bases_per_batch", C.c_uint64), ("work_unit_size", C.c_uint64), ("hll_mode", C.c_uint32),
                ("reserved0", C.c_uint32), ("sparse_set_slots", C.c_uint64)]


class Run(C.Structure):
    _fields_ = [("code", C.c_uint32), ("count", C.c_uint32)]


class BatchResult(C.Structure):
    _fields_ = [("n_reads", C.c_uint32), ("reserved0", C.c_uint32), ("call", u32p), ("n_windows", u32p),
                ("run_start", u32p), ("run_count", u32p), ("runs", C.POINTER(Run)), ("n_runs", C.c_uint64),
                ("codes", u32p), ("n_classified", C.c_uint64), ("kernel_ms", C.c_double),
                ("filtered_call", u32p), ("filter_hits", u32p), ("filter_total", u32p),
                ("extract_sel", C.POINTER(C.c_uint8)), ("n_extract", C.c_uint64)]


class DeviceResult(C.Structure):
    _fields_ = [("d_call", C.c_void_p), ("d_n_windows", C.c_void_p), ("d_codes", C.c_void_p),
                ("d_run_start", C.c_void_p), ("d_run_count", C.c_void_p), ("d_runs", C.c_void_p),
                ("d_n_runs", C.c_void_p)]


LAYOUT_VARIANTS = 25
LAYOUT_SHAPES = ["thread per window", "product k_lookup<MODE_LOOKUP>", "index prefetch, 8 CTAs/SM", "index prefetch, 6 CTAs/SM",
                 "2 windows per thread, 8 CTAs/SM", "2 windows per thread, 6 CTAs/SM", "2 windows per thread, 4 CTAs/SM",
                 "4 windows per thread, 4 CTAs/SM", "product k_lookup<MODE_LOOKUP>, lean", "product k_lookup<MODE_FUSED>",
                 "product k_lookup<MODE_FUSED>, lean", "thread per window, if-chain narrowing",
                 "thread per window, product parameter block", "thread per window, L2::256B on round 1",
                 "tree layout", "tree layout, L2::256B on the header"]


class LayoutResult(C.Structure):                     # kuq_layout_result
    _fields_ = [("n_records", C.c_uint64), ("n_positions", C.c_uint64), ("n_windows", C.c_uint64),
                ("sum_probes", C.c_uint64), ("bin_class", C.c_uint64 * 6), ("transcode_ms", C.c_double),
                ("n_variants", C.c_uint32), ("rec_bytes", C.c_uint32 * LAYOUT_VARIANTS),
                ("arity", C.c_uint32 * LAYOUT_VARIANTS), ("window", C.c_uint32 * LAYOUT_VARIANTS),
                ("shape", C.c_uint32 * LAYOUT_VARIANTS),
                ("best_ms", C.c_double * LAYOUT_VARIANTS), ("mean_ms", C.c_double * LAYOUT_VARIANTS),
                ("mismatches", C.c_uint64 * LAYOUT_VARIANTS), ("tree_ms", C.c_double), ("tree_unordered", C.c_uint64)]


class StatePtrs(C.Structure):
    _fields_ = [("d_regs", C.c_void_p), ("regs_bytes", C.c_uint64), ("d_n_kmers", C.c_void_p),
                ("d_n_reads", C.c_void_p), ("d_dense_flag", C.c_void_p), ("n_sketch", C.c_uint32),
                ("n_taxa", C.c_uint32)]


_LIB = None


def lib_path():
    return _build.LIB


def load_library(rebuild_if_stale: bool = False):
    """Load libkuq.so; raises if it is not there (no silent fallback)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if rebuild_if_stale:
        _build.build()
    if not os.path.exists(_build.LIB):
        raise FileNotFoundError(f"{_build.LIB} is missing: run `python -m krakenuniq_b200.build` "
                                "(the CUDA extension is the only implementation; there is no CPU path)")
    L = C.CDLL(_build.LIB)
    vp = C.c_void_p
    sigs = {
        "kuq_config_default": (None, [C.POINTER(Config)]),
        "kuq_create": (C.c_int, [C.POINTER(Config), C.POINTER(vp)]),
        "kuq_destroy": (None, [vp]),
        "kuq_strerror": (C.c_char_p, [C.c_int]),
        "kuq_last_error": (C.c_char_p, [vp]),
        "kuq_version": (C.c_char_p, []),
        "kuq_device_count": (C.c_int, []),
        "kuq_stage_db": (C.c_int, [vp, vp, C.c_uint64, vp, C.c_uint64, C.c_uint64, C.c_uint64]),
        "kuq_stage_db_append": (C.c_int, [vp, vp, C.c_uint64, vp, C.c_uint64]),
        "kuq_stage_db_append_range": (C.c_int, [vp, vp, C.c_uint64, vp, C.c_uint64, C.c_uint64, C.c_uint64]),
        "kuq_db_runs": (C.c_int, [vp, u32p]),
        "kuq_attach_db_device": (C.c_int, [vp, vp, C.c_uint64, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64,
                                           C.c_uint64]),
        "kuq_db_taxids": (C.c_int, [vp, u32p, u64p, C.c_uint32, u32p]),
        "kuq_set_db_taxid_universe": (C.c_int, [vp, u32p, C.c_uint32]),
        "kuq_mark_zero_hits": (C.c_int, [vp, C.c_int]),
        "kuq_db_sort": (C.c_int, [C.c_int, vp, C.c_uint64, C.c_uint32, C.c_int, vp, vp, C.c_char_p, C.c_uint64]),
        "kuq_db_sort_budget": (C.c_int, [C.c_int, vp, C.c_uint64, C.c_uint32, C.c_int, C.c_uint64, vp, vp, u32p, C.c_char_p,
                                         C.c_uint64]),
        "kuq_db_sort_devices": (C.c_int, [C.POINTER(C.c_int), C.c_uint32, vp, C.c_uint64, C.c_uint32, C.c_int, C.c_uint64,
                                          vp, vp, u32p, C.c_char_p, C.c_uint64]),
        "kuq_db_value_counts": (C.c_int, [vp, u32p, u64p, C.c_uint32, u32p]),
        "kuq_set_lcas_batch": (C.c_int, [vp, vp, u64p, C.c_uint32, u32p, C.c_uint32, u64p]),
        "kuq_export_db_values": (C.c_int, [vp, vp, C.c_uint64]),
        "kuq_set_quick_mode": (C.c_int, [vp, C.c_uint32, C.c_int]),
        "kuq_set_taxonomy": (C.c_int, [vp, u32p, u32p, C.c_uint32]),
        "kuq_set_threshold": (C.c_int, [vp, C.c_double, u32p, u32p, C.c_uint32]),
        "kuq_set_extract": (C.c_int, [vp, u32p, C.c_uint32, C.c_uint32, u32p, u32p, C.c_uint32]),
        "kuq_extract_taxa": (C.c_int, [u32p, C.c_uint32, C.c_uint32, u32p, u32p, C.c_uint32, u32p, C.c_uint32, u32p]),
        "kuq_classify_batch": (C.c_int, [vp, vp, u64p, C.c_uint32, u32p, C.c_uint32, C.POINTER(BatchResult)]),
        "kuq_submit_batch": (C.c_int, [vp, C.c_uint32, vp, u64p, C.c_uint32, u32p, C.c_uint32]),
        "kuq_wait_batch": (C.c_int, [vp, C.c_uint32, C.POINTER(BatchResult)]),
        "kuq_lookup_batch": (C.c_int, [vp, vp, u64p, C.c_uint32, u32p, u32p]),
        "kuq_resolve_batch": (C.c_int, [vp, vp, u64p, C.c_uint32, u32p, u32p, C.c_uint32, C.POINTER(BatchResult)]),
        "kuq_host_alloc": (vp, [C.c_uint64]),
        "kuq_host_free": (None, [vp]),
        "kuq_classify_device": (C.c_int, [vp, C.c_uint32, vp, vp, C.c_uint32, C.c_uint64, vp, C.c_uint32]),
        "kuq_lookup_device": (C.c_int, [vp, C.c_uint32, vp, vp, C.c_uint32, C.c_uint64, vp, C.c_uint32]),
        "kuq_resolve_device": (C.c_int, [vp, C.c_uint32, vp, vp, C.c_uint32, C.c_uint64, vp, vp, C.c_uint32]),
        "kuq_lookup_device_peers": (C.c_int, [vp, C.c_uint32, vp, vp, C.c_uint32, C.c_uint64, C.POINTER(vp), u64p,
                                             C.c_uint32]),
        "kuq_lookup_device_peers_run": (C.c_int, [vp, C.c_uint32, vp, vp, C.c_uint32, C.c_uint64, C.POINTER(vp), u64p,
                                                 C.c_uint32, C.c_uint32]),
        "kuq_device_alloc": (vp, [vp, C.c_uint64]),
        "kuq_device_free": (None, [vp, vp]),
        "kuq_device_memset": (C.c_int, [vp, C.c_uint32, vp, C.c_int, C.c_uint64]),
        "kuq_ipc_export": (C.c_int, [vp, vp, u8p]),
        "kuq_ipc_open": (C.c_int, [vp, u8p, C.POINTER(vp)]),
        "kuq_ipc_close": (C.c_int, [vp, vp]),
        "kuq_sync_slot": (C.c_int, [vp, C.c_uint32]),
        "kuq_copy_to_device": (C.c_int, [vp, C.c_uint32, vp, vp, C.c_uint64]),
        "kuq_device_free_bytes": (C.c_uint64, [vp]),
        "kuq_collect_device_batch": (C.c_int, [vp, C.c_uint32, C.POINTER(BatchResult)]),
        "kuq_slot_device_result": (C.c_int, [vp, C.c_uint32, C.POINTER(DeviceResult)]),
        "kuq_slot_stream": (vp, [vp, C.c_uint32]),
        "kuq_slot_stats": (C.c_int, [vp, C.c_uint32, u64p, u64p]),
        "kuq_launch_count": (C.c_uint64, [vp]),
        "kuq_last_kernel_ms": (C.c_double, [vp, C.c_uint32]),
        "kuq_last_stage_ms": (C.c_int, [vp, C.c_uint32, C.POINTER(C.c_double)]),
        "kuq_finish": (C.c_int, [vp]),
        "kuq_counts_size": (C.c_int, [vp, u32p]),
        "kuq_read_counts": (C.c_int, [vp, u32p, u64p, u64p, u64p, u8p, C.c_uint32]),
        "kuq_clade_counts": (C.c_int, [vp, u32p, C.c_uint32, u64p, u64p, u64p]),
        "kuq_clade_counts_tree": (C.c_int, [vp, u32p, C.c_uint32, u64p, u64p, u64p]),
        "kuq_get_registers": (C.c_int, [vp, C.c_uint32, u8p]),
        "kuq_state_ptrs_get": (C.c_int, [vp, C.POINTER(StatePtrs)]),
        "kuq_unit_table_rows": (C.c_int, [vp, u32p]),
        "kuq_dense_taxids": (C.c_int, [vp, u32p, C.c_uint32, u32p]),
        "kuq_sparse_export": (C.c_int, [vp, vp, C.c_uint64, u64p]),
        "kuq_sparse_import": (C.c_int, [vp, vp, C.c_uint64]),
        "kuq_reset_counts": (C.c_int, [vp]),
        "kuq_sparse_tier_info": (C.c_int, [vp, u64p, u64p, u64p, C.POINTER(C.c_double)]),
        "kuq_exact_info": (C.c_int, [vp, u64p, u64p, u64p]),
        "kuq_exact_export": (C.c_int, [vp, vp, C.c_uint64, u64p]),
        "kuq_exact_import": (C.c_int, [vp, vp, C.c_uint64]),
        "kuq_exact_owner": (C.c_uint32, [C.c_uint64, C.c_uint32]),
        "kuq_exact_export_partitioned": (C.c_int, [vp, C.c_uint32, vp, C.c_uint64, u64p]),
        "kuq_exact_export_partitioned_alloc": (C.c_int, [vp, C.c_uint32, C.POINTER(vp), u64p]),
        "kuq_exact_replace": (C.c_int, [vp, vp, C.c_uint64]),
        "kuq_exact_summary": (C.c_int, [vp, vp, vp]),
        "kuq_set_exact_summary": (C.c_int, [vp, vp, vp]),
        "kuq_exact_partition": (C.c_int, [C.POINTER(vp), C.c_uint32]),
        "kuq_exact_rollup_passes": (C.c_int, [vp, u32p]),
        "kuq_set_exact_spill": (C.c_int, [vp, C.c_uint64]),
        "kuq_exact_spill_info": (C.c_int, [vp, u64p, u64p]),
        "kuq_exact_settle": (C.c_int, [C.POINTER(vp), C.c_uint32]),
        "kuq_merge_counters_into": (C.c_int, [vp, vp]),
        "kuq_set_shard_counting": (C.c_int, [vp, C.c_int]),
        "kuq_set_stats": (C.c_int, [vp, C.c_int]),
        "kuq_merge_into": (C.c_int, [vp, vp]),
        "kuq_enable_peer_access": (C.c_int, [vp, vp]),
        "kuq_stream_open": (C.c_int, [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint64]),
        "kuq_stream_load": (C.c_int, [vp, C.c_uint32, vp, C.c_uint64, vp, C.c_uint64, C.c_uint64]),
        "kuq_stream_use": (C.c_int, [vp, C.c_uint32]),
        "kuq_stream_check": (C.c_int, [vp]),
        "kuq_host_register": (C.c_int, [vp, C.c_uint64]),
        "kuq_host_unregister": (C.c_int, [vp]),
        "kuq_signal_peers": (C.c_int, [vp, C.c_uint32, C.POINTER(vp), C.c_uint32, C.c_uint32, C.c_uint64]),
        "kuq_wait_flags": (C.c_int, [vp, C.c_uint32, vp, C.c_uint32, C.c_uint64, C.c_uint32]),
        "kuq_sparse_export_partitioned": (C.c_int, [vp, C.c_uint32, vp, C.c_uint64, u64p]),
        "kuq_sparse_export_partitioned_alloc": (C.c_int, [vp, C.c_uint32, C.POINTER(vp), u64p]),
        "kuq_sparse_replace": (C.c_int, [vp, vp, C.c_uint64]),
        "kuq_sparse_summary": (C.c_int, [vp, vp, vp]),
        "kuq_set_sparse_summary": (C.c_int, [vp, vp, vp]),
        "kuq_clade_partial": (C.c_int, [vp, u32p, C.c_uint32, u64p, u64p, C.POINTER(C.c_int), u32p]),
        "kuq_ertl_sparse": (C.c_uint64, [u32p, C.c_uint64]),
        "kuq_ertl_dense_hist": (C.c_uint64, [u32p, C.c_uint64]),
        "kuq_scan_device": (C.c_int, [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, C.c_uint32, C.c_uint64, vp, vp]),
        "kuq_ertl_dense": (C.c_uint64, [u8p, C.c_uint64]),
        "kuq_layout_experiment": (C.c_int, [vp, C.c_uint32, C.c_uint64, C.c_uint32, C.POINTER(LayoutResult)]),
        "kuq_random_gather_peak": (C.c_int, [C.c_int, C.c_uint64, C.c_uint64, C.c_uint32, C.POINTER(C.c_double),
                                            C.POINTER(C.c_double), C.POINTER(C.c_double)]),
        "kuq_harvest_keep_device": (C.c_int, [C.c_int, vp, C.c_uint64, vp, C.c_uint64, vp, C.c_uint32, vp, vp]),
        "kuq_kmer_set_create": (C.c_int, [C.c_int, C.c_uint32, C.c_uint64, C.POINTER(vp), C.c_char_p, C.c_uint64]),
        "kuq_kmer_set_add": (C.c_int, [vp, vp, u64p, C.c_uint32]),
        "kuq_kmer_set_next": (C.c_int, [vp, vp, C.c_uint64, u64p]),
        "kuq_kmer_set_info": (C.c_int, [vp, u64p, u32p]),
        "kuq_kmer_set_stats": (C.c_int, [vp, C.POINTER(C.c_double), u64p, u64p, u64p, C.POINTER(C.c_int)]),
        "kuq_kmer_set_last_error": (C.c_char_p, [vp]),
        "kuq_kmer_set_destroy": (None, [vp]),
        "kuq_count_unique_create": (C.c_int, [C.c_int, C.c_uint32, C.c_uint32, C.c_uint64, C.POINTER(vp), C.c_char_p,
                                              C.c_uint64]),
        "kuq_count_unique_add": (C.c_int, [vp, vp, u64p, C.c_uint32]),
        "kuq_count_unique_result": (C.c_int, [vp, u64p, u64p, vp]),
        "kuq_count_unique_stats": (C.c_int, [vp, C.POINTER(C.c_double), u64p, u64p]),
        "kuq_count_unique_last_error": (C.c_char_p, [vp]),
        "kuq_count_unique_destroy": (None, [vp]),
    }
    for name, (res, args) in sigs.items():
        f = getattr(L, name)            # AttributeError here = the library does not export what kuq.h declares
        f.restype, f.argtypes = res, args
    _LIB = L
    return L


def exported_symbols():
    """Names include/kuq.h declares; used by the CPU tests to check the library exports them all."""
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kuq.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(kuq_[a-z0-9_]+)\s*\(", hdr)))


def extract_taxa(taxa, flags, taxid=(), parent=()):
    """the taxa kuq_set_extract selects (kuq_extract_taxa; no device needed), ascending"""
    L = load_library()
    l = np.ascontiguousarray(taxa, np.uint32)
    t = np.ascontiguousarray(taxid, np.uint32)
    p = np.ascontiguousarray(parent, np.uint32)
    n = C.c_uint32(0)
    rc = L.kuq_extract_taxa(_p(l, u32p), len(l), int(flags), _p(t, u32p), _p(p, u32p), len(t), None, 0, C.byref(n))
    if rc:
        raise KuqError(rc, "kuq_extract_taxa: " + L.kuq_strerror(rc).decode())
    out = np.zeros(max(1, n.value), np.uint32)
    rc = L.kuq_extract_taxa(_p(l, u32p), len(l), int(flags), _p(t, u32p), _p(p, u32p), len(t), _p(out, u32p), n.value, C.byref(n))
    if rc:
        raise KuqError(rc, "kuq_extract_taxa: " + L.kuq_strerror(rc).decode())
    return out[:n.value]


def _p(a, t):
    return a.ctypes.data_as(t)


class Classifier:
    """One GPU's classification context (kuq_ctx)."""

    def __init__(self, device=0, n_slots=2, max_reads=1 << 20, max_bases=192 << 20, work_unit_size=500000,
                 hll_mode=HLL_PRELOAD, sparse_set_slots=1 << 26):
        self.L = load_library()
        cfg = Config()
        self.L.kuq_config_default(C.byref(cfg))
        cfg.device, cfg.n_slots = device, n_slots
        cfg.max_reads_per_batch, cfg.max_bases_per_batch = max_reads, max_bases
        cfg.work_unit_size, cfg.hll_mode, cfg.sparse_set_slots = work_unit_size, hll_mode, sparse_set_slots
        self.cfg = cfg
        h = C.c_void_p()
        rc = self.L.kuq_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise KuqError(rc, self.L.kuq_strerror(rc).decode())
        self.h = h
        self._keep = []

    def close(self):
        if getattr(self, "h", None):
            self.L.kuq_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise KuqError(rc, f"{self.L.kuq_strerror(rc).decode()}: {self.L.kuq_last_error(self.h).decode()}")

    # ---- database / taxonomy -------------------------------------------------------------------------------
    def stage_db(self, kdb: np.ndarray, idx: np.ndarray, bin_lo=0, bin_hi=0):
        kdb = np.ascontiguousarray(kdb).view(np.uint8) if not isinstance(kdb, np.memmap) else kdb
        idx = np.ascontiguousarray(idx).view(np.uint8) if not isinstance(idx, np.memmap) else idx
        self._ck(self.L.kuq_stage_db(self.h, kdb.ctypes.data, kdb.size, idx.ctypes.data, idx.size, bin_lo, bin_hi))

    def stage_db_append(self, kdb: np.ndarray, idx: np.ndarray):
        """one more whole database, asked after those staged already (classify -d a -d b; kuq_stage_db_append).
        Same k; nt and index type may differ.  stage_db drops the appended databases again."""
        kdb = np.ascontiguousarray(kdb).view(np.uint8) if not isinstance(kdb, np.memmap) else kdb
        idx = np.ascontiguousarray(idx).view(np.uint8) if not isinstance(idx, np.memmap) else idx
        self._ck(self.L.kuq_stage_db_append(self.h, kdb.ctypes.data, kdb.size, idx.ctypes.data, idx.size))

    def stage_db_append_range(self, kdb: np.ndarray, idx: np.ndarray, bin_lo=0, bin_hi=0):
        """minimizer bins [bin_lo, bin_hi) of one more database (kuq_stage_db_append_range): (0, 0) = all of it,
        bin_lo == bin_hi != 0 = an empty slice"""
        kdb = np.ascontiguousarray(kdb).view(np.uint8) if not isinstance(kdb, np.memmap) else kdb
        idx = np.ascontiguousarray(idx).view(np.uint8) if not isinstance(idx, np.memmap) else idx
        self._ck(self.L.kuq_stage_db_append_range(self.h, kdb.ctypes.data, kdb.size, idx.ctypes.data, idx.size,
                                                  int(bin_lo), int(bin_hi)))

    def db_runs(self):
        n = C.c_uint32(0)
        self._ck(self.L.kuq_db_runs(self.h, C.byref(n)))
        return n.value

    def stage_db_files(self, kdb_path, idx_path, bin_lo=0, bin_hi=0):
        self.stage_db(np.memmap(kdb_path, np.uint8, "r"), np.memmap(idx_path, np.uint8, "r"), bin_lo, bin_hi)

    def attach_db_device(self, d_pairs_ptr, key_ct, d_offsets_ptr, k, nt, idx_type=2, bin_lo=0, bin_hi=0):
        self._ck(self.L.kuq_attach_db_device(self.h, d_pairs_ptr, key_ct, d_offsets_ptr, k, nt, idx_type, bin_lo,
                                             bin_hi))

    def db_taxids(self):
        n = C.c_uint32(0)
        self._ck(self.L.kuq_db_taxids(self.h, None, None, 0, C.byref(n)))
        t = np.zeros(n.value, np.uint32)
        c = np.zeros(n.value, np.uint64)
        if n.value:
            self._ck(self.L.kuq_db_taxids(self.h, _p(t, u32p), _p(c, u64p), n.value, C.byref(n)))
        return t, c

    def set_quick_mode(self, min_hits, stop_at_last_hit=True):
        """classify -q -m min_hits (0 = off); stop_at_last_hit=False gives the -x path's rule (kuq_set_quick_mode)"""
        self._ck(self.L.kuq_set_quick_mode(self.h, int(min_hits), 1 if stop_at_last_hit else 0))

    def set_lcas(self, bases: np.ndarray, piece_offsets: np.ndarray, taxids, flags=0) -> int:
        """kuq_set_lcas_batch: fold the pieces' taxids into the staged database's values; returns #k-mers not found.
        flags: 1 = set_lcas -T, 2 = -R"""
        bases = np.ascontiguousarray(bases, np.uint8)
        offs = np.ascontiguousarray(piece_offsets, np.uint64)
        t = np.ascontiguousarray(taxids, np.uint32)
        missing = C.c_uint64(0)
        buf = bases if bases.size else np.zeros(1, np.uint8)
        self._ck(self.L.kuq_set_lcas_batch(self.h, buf.ctypes.data, _p(offs, u64p), len(offs) - 1, _p(t, u32p), flags, C.byref(missing)))
        return missing.value

    def export_db_values(self, kdb: np.ndarray):
        """kuq_export_db_values: write the device record values (taxids) into the host image `kdb` in place"""
        assert kdb.dtype == np.uint8 and kdb.flags["C_CONTIGUOUS"]
        self._ck(self.L.kuq_export_db_values(self.h, kdb.ctypes.data, kdb.size))

    def db_value_counts(self):
        """kuq_db_value_counts: (taxids ascending, records holding each) of the staged records' values as they are now"""
        n = C.c_uint32(0)
        self._ck(self.L.kuq_db_value_counts(self.h, None, None, 0, C.byref(n)))
        t = np.zeros(n.value, np.uint32)
        c = np.zeros(n.value, np.uint64)
        if n.value:
            self._ck(self.L.kuq_db_value_counts(self.h, _p(t, u32p), _p(c, u64p), n.value, C.byref(n)))
        return t, c

    def mark_zero_hits(self, on=True):
        """several databases: lookups report a stored taxon 0 as CODE_FOUND_ZERO (kuq_mark_zero_hits)"""
        self._ck(self.L.kuq_mark_zero_hits(self.h, 1 if on else 0))

    def set_db_taxid_universe(self, taxids):
        t = np.ascontiguousarray(taxids, np.uint32)
        self._ck(self.L.kuq_set_db_taxid_universe(self.h, _p(t, u32p), len(t)))

    def set_taxonomy(self, taxid, parent):
        t = np.ascontiguousarray(taxid, np.uint32)
        p = np.ascontiguousarray(parent, np.uint32)
        self._ck(self.L.kuq_set_taxonomy(self.h, _p(t, u32p), _p(p, u32p), len(t)))

    def set_threshold(self, threshold, taxid, parent):
        """krakenuniq-filter --threshold on every later batch, from the taxDB rows in file order (kuq_set_threshold);
        results gain filtered_call, filter_hits and filter_total"""
        t = np.ascontiguousarray(taxid, np.uint32)
        p = np.ascontiguousarray(parent, np.uint32)
        self._ck(self.L.kuq_set_threshold(self.h, float(threshold), _p(t, u32p), _p(p, u32p), len(t)))

    def set_extract(self, taxa, flags, taxid=(), parent=()):
        """krakenuniq-extract-reads' read selection on every later batch (kuq_set_extract; flags: EXTRACT_*); results gain
        extract_sel and n_extract"""
        l = np.ascontiguousarray(taxa, np.uint32)
        t = np.ascontiguousarray(taxid, np.uint32)
        p = np.ascontiguousarray(parent, np.uint32)
        self._ck(self.L.kuq_set_extract(self.h, _p(l, u32p), len(l), int(flags), _p(t, u32p), _p(p, u32p), len(t)))

    # ---- host-buffer classification ---------------------------------------------------------------------------
    def _result(self, res: BatchResult, offsets, copy=True):
        n = res.n_reads
        as_np = lambda ptr, cnt, dt: (np.ctypeslib.as_array(ptr, shape=(cnt,)).view(dt) if cnt else np.zeros(0, dt))
        out = dict(call=as_np(res.call, n, np.uint32), n_windows=as_np(res.n_windows, n, np.uint32),
                   n_classified=int(res.n_classified), kernel_ms=res.kernel_ms, n_runs=int(res.n_runs))
        if res.n_runs or res.run_start:
            out["run_start"] = as_np(res.run_start, n, np.uint32)
            out["run_count"] = as_np(res.run_count, n, np.uint32)
            runs = np.ctypeslib.as_array(C.cast(res.runs, u32p), shape=(int(res.n_runs) * 2,)) if res.n_runs else \
                np.zeros(0, np.uint32)
            out["runs"] = runs.reshape(-1, 2)
        if res.extract_sel:
            out["extract_sel"] = as_np(res.extract_sel, n, np.uint8)
            out["n_extract"] = int(res.n_extract)
        if res.filtered_call:
            out["filtered_call"] = as_np(res.filtered_call, n, np.uint32)
            out["filter_hits"] = as_np(res.filter_hits, n, np.uint32)
            out["filter_total"] = as_np(res.filter_total, n, np.uint32)
        if res.codes:
            total = int(offsets[-1] - offsets[0])
            out["codes"] = as_np(res.codes, total, np.uint32)
        if copy:
            out = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in out.items()}
        return out

    def classify(self, bases: np.ndarray, offsets: np.ndarray, unit_id=None, flags=0):
        """kuq_classify_batch: returns dict(call, n_windows, run_start, run_count, runs[, codes])."""
        bases = np.ascontiguousarray(bases, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.uint64)
        n = len(offsets) - 1
        u = np.ascontiguousarray(unit_id, np.uint32) if unit_id is not None else None
        res = BatchResult()
        self._ck(self.L.kuq_classify_batch(self.h, bases.ctypes.data if bases.size else None, _p(offsets, u64p), n,
                                           _p(u, u32p) if u is not None else None, flags, C.byref(res)))
        return self._result(res, offsets)

    def lookup(self, bases: np.ndarray, offsets: np.ndarray):
        """kuq_lookup_batch: per-window dense ids of the staged range (host arrays) + window counts"""
        bases = np.ascontiguousarray(bases, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.uint64)
        n = len(offsets) - 1
        total = int(offsets[-1] - offsets[0])
        codes = np.zeros(max(total, 1), np.uint32)
        nwin = np.zeros(max(n, 1), np.uint32)
        self._ck(self.L.kuq_lookup_batch(self.h, bases.ctypes.data if bases.size else None, _p(offsets, u64p), n,
                                         _p(codes, u32p), _p(nwin, u32p)))
        return codes[:total], nwin[:n]

    def resolve(self, bases: np.ndarray, offsets: np.ndarray, codes: np.ndarray, unit_id=None, flags=0):
        """kuq_resolve_batch: calls / hit lists / counters from merged per-window dense ids"""
        bases = np.ascontiguousarray(bases, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.uint64)
        codes = np.ascontiguousarray(codes, np.uint32)
        n = len(offsets) - 1
        u = np.ascontiguousarray(unit_id, np.uint32) if unit_id is not None else None
        res = BatchResult()
        self._ck(self.L.kuq_resolve_batch(self.h, bases.ctypes.data if bases.size else None, _p(offsets, u64p), n,
                                          _p(codes, u32p), _p(u, u32p) if u is not None else None, flags, C.byref(res)))
        return self._result(res, offsets)

    def submit(self, slot, bases_ptr, offsets: np.ndarray, unit_id=None, flags=0):
        n = len(offsets) - 1
        u = np.ascontiguousarray(unit_id, np.uint32) if unit_id is not None else None
        self._ck(self.L.kuq_submit_batch(self.h, slot, bases_ptr, _p(offsets, u64p), n,
                                         _p(u, u32p) if u is not None else None, flags))

    def wait(self, slot, offsets=None, copy=False):
        res = BatchResult()
        self._ck(self.L.kuq_wait_batch(self.h, slot, C.byref(res)))
        return self._result(res, offsets if offsets is not None else np.zeros(2, np.uint64), copy=copy)

    # ---- device-buffer classification ---------------------------------------------------------------------------
    def classify_device(self, slot, d_bases, d_offsets, n_reads, total_bases, d_unit=None, flags=0):
        self._ck(self.L.kuq_classify_device(self.h, slot, d_bases, d_offsets, n_reads, total_bases, d_unit, flags))

    def lookup_device(self, slot, d_bases, d_offsets, n_reads, total_bases, d_codes_out, only_hits=0):
        """per-window dense ids into d_codes_out.  only_hits: 0 = every window, 1 = hits only, 2 = LOOKUP_FILL_EMPTY
        (hits only, and windows already coded non-zero are skipped: the later databases of a streamed run)."""
        self._ck(self.L.kuq_lookup_device(self.h, slot, d_bases, d_offsets, n_reads, total_bases, d_codes_out,
                                          only_hits))

    def resolve_device(self, slot, d_bases, d_offsets, n_reads, total_bases, d_codes_in, d_unit=None, flags=0):
        self._ck(self.L.kuq_resolve_device(self.h, slot, d_bases, d_offsets, n_reads, total_bases, d_codes_in, d_unit,
                                           flags))

    def lookup_device_peers(self, slot, d_bases, d_offsets, n_reads, total_bases, peer_ptrs, base_bounds):
        n = len(peer_ptrs)
        arr = (C.c_void_p * n)(*[C.c_void_p(int(x)) for x in peer_ptrs])
        bounds = np.ascontiguousarray(base_bounds, np.uint64)
        assert len(bounds) == n + 1
        self._ck(self.L.kuq_lookup_device_peers(self.h, slot, d_bases, d_offsets, n_reads, total_bases, arr,
                                                _p(bounds, u64p), n))

    def collect_device(self, slot, offsets=None):
        """kuq_collect_device_batch: the results of the slot's last device call, like wait()"""
        res = BatchResult()
        self._ck(self.L.kuq_collect_device_batch(self.h, slot, C.byref(res)))
        return self._result(res, offsets if offsets is not None else np.zeros(2, np.uint64))

    def lookup_device_peers_run(self, slot, d_bases, d_offsets, n_reads, total_bases, peer_ptrs, base_bounds, run):
        """one run (kuq_db_runs) of the in-order lookup of databases sharded by minimizer range, hits stored into the
        resolving GPU's buffer (kuq_lookup_device_peers_run)"""
        n = len(peer_ptrs)
        arr = (C.c_void_p * n)(*[C.c_void_p(int(x)) for x in peer_ptrs])
        bounds = np.ascontiguousarray(base_bounds, np.uint64)
        assert len(bounds) == n + 1
        self._ck(self.L.kuq_lookup_device_peers_run(self.h, slot, d_bases, d_offsets, n_reads, total_bases, arr,
                                                    _p(bounds, u64p), n, int(run)))

    def device_alloc(self, nbytes):
        p = self.L.kuq_device_alloc(self.h, nbytes)
        if not p:
            raise KuqError(-8, "device allocation failed")
        return p

    def device_free(self, p):
        self.L.kuq_device_free(self.h, p)

    def device_memset(self, slot, p, value, nbytes):
        self._ck(self.L.kuq_device_memset(self.h, slot, p, value, nbytes))

    def ipc_export(self, p) -> bytes:
        h = np.zeros(64, np.uint8)
        self._ck(self.L.kuq_ipc_export(self.h, p, _p(h, u8p)))
        return h.tobytes()

    def ipc_open(self, handle: bytes):
        h = np.frombuffer(handle, np.uint8).copy()
        out = C.c_void_p()
        self._ck(self.L.kuq_ipc_open(self.h, _p(h, u8p), C.byref(out)))
        return out.value

    def ipc_close(self, p):
        self._ck(self.L.kuq_ipc_close(self.h, p))

    def sync(self, slot):
        self._ck(self.L.kuq_sync_slot(self.h, slot))

    def device_result(self, slot):
        r = DeviceResult()
        self._ck(self.L.kuq_slot_device_result(self.h, slot, C.byref(r)))
        return r

    def slot_stats(self, slot):
        a, b = C.c_uint64(0), C.c_uint64(0)
        self._ck(self.L.kuq_slot_stats(self.h, slot, C.byref(a), C.byref(b)))
        return a.value, b.value

    def slot_stream(self, slot):
        return self.L.kuq_slot_stream(self.h, slot)

    def launch_count(self):
        return int(self.L.kuq_launch_count(self.h))

    def last_kernel_ms(self, slot):
        return float(self.L.kuq_last_kernel_ms(self.h, slot))

    def last_stage_ms(self, slot):
        a = (C.c_double * 3)()
        self._ck(self.L.kuq_last_stage_ms(self.h, slot, a))
        return [a[0], a[1], a[2]]

    # ---- results ---------------------------------------------------------------------------------------------
    def finish(self):
        self._ck(self.L.kuq_finish(self.h))

    def counts(self):
        n = C.c_uint32(0)
        self._ck(self.L.kuq_counts_size(self.h, C.byref(n)))
        m = n.value
        taxid, nr, nk, un, sp = (np.zeros(m, np.uint32), np.zeros(m, np.uint64), np.zeros(m, np.uint64),
                                 np.zeros(m, np.uint64), np.zeros(m, np.uint8))
        if m:
            self._ck(self.L.kuq_read_counts(self.h, _p(taxid, u32p), _p(nr, u64p), _p(nk, u64p), _p(un, u64p),
                                            _p(sp, u8p), m))
        return dict(taxid=taxid, n_reads=nr, n_kmers=nk, unique=un, sparse=sp)

    def clade(self, taxids):
        t = np.ascontiguousarray(taxids, np.uint32)
        r, k, u = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._ck(self.L.kuq_clade_counts(self.h, _p(t, u32p), len(t), C.byref(r), C.byref(k), C.byref(u)))
        return u.value, r.value, k.value

    def registers(self, taxid):
        r = np.zeros(4096, np.uint8)
        self._ck(self.L.kuq_get_registers(self.h, int(taxid), _p(r, u8p)))
        return r

    def unit_table_rows(self):
        """units a preloaded batch holds before (unit, taxon) pairs spill into the per-batch hash map"""
        n = np.zeros(1, np.uint32)
        self._ck(self.L.kuq_unit_table_rows(self.h, _p(n, u32p)))
        return int(n[0])

    def state_ptrs(self):
        s = StatePtrs()
        self._ck(self.L.kuq_state_ptrs_get(self.h, C.byref(s)))
        return s

    def dense_taxids(self):
        n = C.c_uint32(0)
        self._ck(self.L.kuq_dense_taxids(self.h, None, 0, C.byref(n)))
        t = np.zeros(n.value, np.uint32)
        self._ck(self.L.kuq_dense_taxids(self.h, _p(t, u32p), n.value, C.byref(n)))
        return t

    def sparse_export(self, d_out=None, cap=0):
        n = C.c_uint64(0)
        self._ck(self.L.kuq_sparse_export(self.h, d_out, cap, C.byref(n)))
        return n.value

    def sparse_import(self, d_keys, n):
        self._ck(self.L.kuq_sparse_import(self.h, d_keys, n))

    def stream_open(self, k, nt, idx_type, max_records, max_bins):
        self._ck(self.L.kuq_stream_open(self.h, k, nt, idx_type, max_records, max_bins))

    def stream_load(self, buf, host_records_ptr, n_records, host_offsets_ptr, bin_lo, bin_hi):
        self._ck(self.L.kuq_stream_load(self.h, buf, host_records_ptr, n_records, host_offsets_ptr, bin_lo, bin_hi))

    def stream_use(self, buf):
        self._ck(self.L.kuq_stream_use(self.h, buf))

    def stream_check(self):
        self._ck(self.L.kuq_stream_check(self.h))

    def merge_from(self, other):
        """kuq_merge_into(self, other): fold another context's per-taxon state (another GPU of this process) into this one"""
        self._ck(self.L.kuq_merge_into(self.h, other.h))

    def set_stats(self, on=True):
        self._ck(self.L.kuq_set_stats(self.h, 1 if on else 0))

    def set_shard_counting(self, on=True):
        self._ck(self.L.kuq_set_shard_counting(self.h, 1 if on else 0))

    def signal_peers(self, slot, flag_ptrs, my_index, value):
        arr = (C.c_void_p * len(flag_ptrs))(*flag_ptrs)
        self._ck(self.L.kuq_signal_peers(self.h, slot, arr, len(flag_ptrs), my_index, value))

    def wait_flags(self, slot, d_flags, n, value, timeout_ms=0):
        self._ck(self.L.kuq_wait_flags(self.h, slot, d_flags, n, value, timeout_ms))

    def sparse_export_partitioned(self, n_parts, d_out=None, cap=0):
        counts = np.zeros(n_parts, np.uint64)
        self._ck(self.L.kuq_sparse_export_partitioned(self.h, n_parts, d_out, cap, _p(counts, u64p)))
        return counts

    def sparse_export_partitioned_alloc(self, n_parts):
        """→ (device pointer of the keys grouped by part — release with device_free —, counts per part)"""
        counts = np.zeros(n_parts, np.uint64)
        ptr = C.c_void_p()
        self._ck(self.L.kuq_sparse_export_partitioned_alloc(self.h, n_parts, C.byref(ptr), _p(counts, u64p)))
        return ptr.value, counts

    def sparse_replace(self, d_keys, n):
        self._ck(self.L.kuq_sparse_replace(self.h, d_keys, n))

    def sparse_summary(self, d_hist, d_distinct):
        self._ck(self.L.kuq_sparse_summary(self.h, d_hist, d_distinct))

    def set_sparse_summary(self, d_hist, d_distinct):
        self._ck(self.L.kuq_set_sparse_summary(self.h, d_hist, d_distinct))

    def clade_counts_tree(self, taxids):
        """kuq_clade_counts_tree: (reads, kmers, unique) arrays for clade(taxid) = the taxon and all its descendants"""
        t = np.ascontiguousarray(taxids, np.uint32)
        r, k, u = (np.zeros(len(t), np.uint64) for _ in range(3))
        self._ck(self.L.kuq_clade_counts_tree(self.h, _p(t, u32p), len(t), _p(r, u64p), _p(k, u64p), _p(u, u64p)))
        return r, k, u

    def clade_partial(self, taxids):
        """(reads, kmers, is_dense, hist64) of the listed taxa's merged sketch on THIS GPU (see kuq.h)"""
        t = np.ascontiguousarray(taxids, np.uint32)
        r, k, dflag = C.c_uint64(0), C.c_uint64(0), C.c_int(0)
        hist = np.zeros(64, np.uint32)
        self._ck(self.L.kuq_clade_partial(self.h, _p(t, u32p), len(t), C.byref(r), C.byref(k), C.byref(dflag), _p(hist, u32p)))
        return r.value, k.value, bool(dflag.value), hist

    def scan_device(self, slot, k, nt, idx_type, d_bases, d_offsets, n_reads, total_bases, d_canon, d_bins):
        self._ck(self.L.kuq_scan_device(self.h, slot, k, nt, idx_type, d_bases, d_offsets, n_reads, total_bases, d_canon, d_bins))

    def sparse_tier_info(self):
        a, b, c, d = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_double()
        self._ck(self.L.kuq_sparse_tier_info(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return {"slots": a.value, "keys": b.value, "times_grown": c.value, "last_harvest_ms": d.value}

    def exact_info(self):
        """kuq_exact_info: capacity, pairs held and growths of the exact k-mer set (HLL_EXACT)"""
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._ck(self.L.kuq_exact_info(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return {"slots": a.value, "pairs": b.value, "times_grown": c.value}

    def exact_export(self, d_out=None, cap=0):
        """kuq_exact_export: pairs (16 B: k-mer + 1, dense taxon + 1) into device memory; without a buffer → their number"""
        n = C.c_uint64(0)
        self._ck(self.L.kuq_exact_export(self.h, d_out, cap, C.byref(n)))
        return n.value

    def exact_import(self, d_pairs, n):
        self._ck(self.L.kuq_exact_import(self.h, d_pairs, n))

    def exact_owner(self, kmer, n_parts):
        """kuq_exact_owner: the part (0..n_parts-1) that owns a canonical k-mer in the partitioned exact set"""
        return int(self.L.kuq_exact_owner(int(kmer), n_parts))

    def exact_export_partitioned(self, n_parts, d_out=None, cap=0):
        """kuq_exact_export_partitioned: pairs grouped by owner, parts back to back; → pairs per part"""
        counts = np.zeros(n_parts, np.uint64)
        self._ck(self.L.kuq_exact_export_partitioned(self.h, n_parts, d_out, cap, _p(counts, u64p)))
        return counts

    def exact_export_partitioned_alloc(self, n_parts):
        """→ (device pointer of the pairs grouped by owner — release with device_free —, pairs per part)"""
        counts = np.zeros(n_parts, np.uint64)
        ptr = C.c_void_p()
        self._ck(self.L.kuq_exact_export_partitioned_alloc(self.h, n_parts, C.byref(ptr), _p(counts, u64p)))
        return ptr.value, counts

    def exact_replace(self, d_pairs, n):
        self._ck(self.L.kuq_exact_replace(self.h, d_pairs, n))

    def exact_summary(self, d_count, d_books):
        """kuq_exact_summary: per-taxon set sizes ([n_sketch] uint64) and roll-up books ([n_taxa] int64) of this part"""
        self._ck(self.L.kuq_exact_summary(self.h, d_count, d_books))

    def set_exact_summary(self, d_count, d_books):
        self._ck(self.L.kuq_set_exact_summary(self.h, d_count, d_books))

    def exact_rollup_passes(self):
        n = np.zeros(1, np.uint32)
        self._ck(self.L.kuq_exact_rollup_passes(self.h, _p(n, u32p)))
        return int(n[0])

    def merge_counters_from(self, other):
        """kuq_merge_counters_into(self, other): kuq_merge_into without the sparse-tier keys and the exact pairs"""
        self._ck(self.L.kuq_merge_counters_into(self.h, other.h))

    @staticmethod
    def exact_partition(classifiers):
        """kuq_exact_partition: the exact sets of these contexts (one process) spread over them by k-mer owner; the summed
        summary is installed on the first one"""
        arr = (C.c_void_p * len(classifiers))(*[c.h for c in classifiers])
        classifiers[0]._ck(classifiers[0].L.kuq_exact_partition(arr, len(classifiers)))

    def set_exact_spill(self, host_budget_bytes):
        """kuq_set_exact_spill: a table that cannot grow spills to host memory, up to this many bytes of pairs over all
        contexts of the process (0 = fail with KUQ_E_NOMEM instead)"""
        self._ck(self.L.kuq_set_exact_spill(self.h, int(host_budget_bytes)))

    def exact_spill_info(self):
        """kuq_exact_spill_info: (times the table spilled since the last reset, pairs held in host memory now)"""
        a, b = C.c_uint64(), C.c_uint64()
        self._ck(self.L.kuq_exact_spill_info(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    @staticmethod
    def exact_settle(classifiers):
        """kuq_exact_settle: the spilled exact sets of these contexts counted part by part on all of them; the summed
        summary is installed on the first one"""
        arr = (C.c_void_p * len(classifiers))(*[c.h for c in classifiers])
        classifiers[0]._ck(classifiers[0].L.kuq_exact_settle(arr, len(classifiers)))

    def layout_experiment(self, slot, n_positions, reps=5):
        """kuq_layout_experiment: record layout x search shape of the bin search, timed on the windows of the slot's
        last batch and checked against the ids the product wrote for it"""
        r = LayoutResult()
        self._ck(self.L.kuq_layout_experiment(self.h, slot, n_positions, reps, C.byref(r)))
        out = {"n_records": r.n_records, "n_positions": r.n_positions, "n_windows": r.n_windows,
               "probes_per_window": r.sum_probes / max(r.n_windows, 1), "transcode_ms": r.transcode_ms,
               "tree_ms": r.tree_ms, "tree_unordered_bins": r.tree_unordered,
               "windows_by_bin_size": dict(zip(["<=8", "<=16", "<=64", "<=256", "<=1024", ">1024"], list(r.bin_class))),
               "variants": []}
        for v in range(r.n_variants):
            out["variants"].append({"record_bytes": r.rec_bytes[v], "arity": r.arity[v], "scan_window": r.window[v],
                                    "shape": LAYOUT_SHAPES[r.shape[v]],
                                    "best_ms": r.best_ms[v], "mean_ms": r.mean_ms[v], "mismatches": r.mismatches[v]})
        return out

    def reset_counts(self):
        """Start a new run on the staged database: the context then answers like a freshly staged one (kuq.h)"""
        self._ck(self.L.kuq_reset_counts(self.h))


def ertl_dense(regs: np.ndarray, n_observed: int) -> int:
    L = load_library()
    regs = np.ascontiguousarray(regs, np.uint8)
    return int(L.kuq_ertl_dense(_p(regs, u8p), n_observed))


def ertl_sparse(hist64: np.ndarray, n_observed: int) -> int:
    L = load_library()
    h = np.ascontiguousarray(hist64, np.uint32)
    return int(L.kuq_ertl_sparse(_p(h, u32p), n_observed))


def ertl_dense_hist(hist64: np.ndarray, n_observed: int) -> int:
    L = load_library()
    h = np.ascontiguousarray(hist64, np.uint32)
    return int(L.kuq_ertl_dense_hist(_p(h, u32p), n_observed))


def random_gather_peak(device=0, buffer_bytes=16 << 30, n_sectors=1 << 30, bytes_per_access=32):
    """kuq_random_gather_peak: (G sectors/s, GB/s of 32-byte sectors, kernel ms) — SURVEY.md §8(d)'s second roofline"""
    L = load_library()
    gs, gb, ms = C.c_double(), C.c_double(), C.c_double()
    rc = L.kuq_random_gather_peak(device, buffer_bytes, n_sectors, bytes_per_access, C.byref(gs), C.byref(gb), C.byref(ms))
    if rc != 0:
        raise KuqError(rc, L.kuq_strerror(rc).decode())
    return gs.value, gb.value, ms.value


def harvest_keep_device(d_pairs, n_rec, d_secondaries, n_secondaries, d_dense_flag, n_sketch, d_distinct, d_n_kept, device=0):
    """kuq_harvest_keep_device: the record-tier harvest of kuq_finish on caller-owned device buffers (pointers)"""
    L = load_library()
    rc = L.kuq_harvest_keep_device(device, d_pairs, n_rec, d_secondaries, n_secondaries, d_dense_flag, n_sketch, d_distinct, d_n_kept)
    if rc != 0:
        raise KuqError(rc, L.kuq_strerror(rc).decode())


def decode_runs(res, i):
    """hit list of read i as [(code, count), ...] from a classify() result"""
    s, c = int(res["run_start"][i]), int(res["run_count"][i])
    return [(int(a), int(b)) for a, b in res["runs"][s:s + c]]


def db_sort(jdb: np.ndarray, nt: int, zero_vals=False, device=0, budget=0, with_passes=False, devices=None):
    """kuq_db_sort_budget: unsorted Jellyfish-style image → (database.kdb image, KRAKIX2 index image), on the GPU within
    `budget` bytes of device memory (0 → KUQ_DB_SORT_BUDGET, else 3/4 of the free memory).  with_passes: also return
    the number of passes (1 = in one piece, else the number of minimizer ranges).  devices: a list of device ordinals
    (kuq_db_sort_devices; repeats allowed), each a worker of a sort in passes, instead of `device` alone."""
    L = load_library()
    jdb = np.ascontiguousarray(jdb, np.uint8)
    key_bits = int(np.frombuffer(jdb[8:16].tobytes(), np.uint64)[0])
    key_ct = int(np.frombuffer(jdb[48:56].tobytes(), np.uint64)[0])
    size = 72 + 2 * (4 + 8 * key_bits) + key_ct * ((key_bits + 7) // 8 + 4)
    kdb = np.zeros(size, np.uint8)
    idx = np.zeros(8 + 8 * (4 ** nt + 1), np.uint8)
    err = C.create_string_buffer(512)
    passes = C.c_uint32(0)
    if devices is None:
        rc = L.kuq_db_sort_budget(device, jdb.ctypes.data, jdb.size, nt, 1 if zero_vals else 0, budget, kdb.ctypes.data,
                                  idx.ctypes.data, C.byref(passes), err, 512)
    else:
        devs = (C.c_int * len(devices))(*devices)
        rc = L.kuq_db_sort_devices(devs, len(devices), jdb.ctypes.data, jdb.size, nt, 1 if zero_vals else 0, budget,
                                   kdb.ctypes.data, idx.ctypes.data, C.byref(passes), err, 512)
    if rc != 0:
        raise KuqError(rc, err.value.decode() or L.kuq_strerror(rc).decode())
    return (kdb, idx, passes.value) if with_passes else (kdb, idx)


def kdb_header(k: int, key_ct: int) -> np.ndarray:
    """header of a Jellyfish-1 style k-mer file (SURVEY App. A16): JFLISTDN, key_bits = 2k, val_len = 4, key_ct"""
    h = np.zeros(72 + 2 * (4 + 8 * 2 * k), np.uint8)
    h[:8] = np.frombuffer(b"JFLISTDN", np.uint8)
    h[8:24] = np.array([2 * k, 4], "<u8").view(np.uint8)
    h[48:56] = np.array([key_ct], "<u8").view(np.uint8)
    return h


class KmerSet:
    """kuq_kmer_set_*: the canonical k-mer set of a library with its counts (step 1 of build_db.sh) on the GPU."""

    def __init__(self, k, budget=None, device=0):
        self.L = load_library()
        self.k, self.rec = k, (2 * k + 7) // 8 + 4
        h, err = C.c_void_p(), C.create_string_buffer(1024)
        rc = self.L.kuq_kmer_set_create(device, k, budget or 0, C.byref(h), err, 1024)
        if rc != 0:
            raise KuqError(rc, err.value.decode() or self.L.kuq_strerror(rc).decode())
        self.h = h

    def _ck(self, rc):
        if rc != 0:
            raise KuqError(rc, f"{self.L.kuq_strerror(rc).decode()}: {self.L.kuq_kmer_set_last_error(self.h).decode()}")

    def add(self, bases: np.ndarray, offsets: np.ndarray):
        bases = np.ascontiguousarray(bases, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.uint64)
        buf = bases if bases.size else np.zeros(1, np.uint8)
        self._ck(self.L.kuq_kmer_set_add(self.h, buf.ctypes.data, _p(offsets, u64p), len(offsets) - 1))

    def next(self, out: np.ndarray) -> int:
        """fill `out` (uint8, a multiple of the record size) with the next records; returns how many (0 = done)"""
        n = C.c_uint64(0)
        self._ck(self.L.kuq_kmer_set_next(self.h, out.ctypes.data, out.size // self.rec, C.byref(n)))
        return n.value

    def info(self):
        """(records produced so far, planned passes)"""
        n, p = C.c_uint64(0), C.c_uint32(0)
        self._ck(self.L.kuq_kmer_set_info(self.h, C.byref(n), C.byref(p)))
        return n.value, p.value

    def stats(self):
        ms, w, est, peak, dev = (C.c_double * 5)(), C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_int()
        self._ck(self.L.kuq_kmer_set_stats(self.h, ms, C.byref(w), C.byref(est), C.byref(peak), C.byref(dev)))
        return {"stage_ms": dict(zip(["pack_hist", "extract", "sort", "collapse", "d2h"], list(ms))), "windows": w.value,
                "ws_estimate_bytes": est.value, "peak_bytes": peak.value, "library_in_hbm": bool(dev.value)}

    def close(self):
        if getattr(self, "h", None):
            self.L.kuq_kmer_set_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def kmer_set(bases: np.ndarray, offsets: np.ndarray, k: int, budget=None, batch=None, device=0):
    """The k-mer file `kmer_set count -m k -C` writes (database_0) for the sequences bases[offsets[r]:offsets[r+1]]:
    header + one record per distinct canonical k-mer with its count, ascending.  batch = bases per device batch
    (KUQ_KMER_SET_BATCH).  Returns (image uint8, number of passes)."""
    old = os.environ.get("KUQ_KMER_SET_BATCH")
    if batch:
        os.environ["KUQ_KMER_SET_BATCH"] = str(int(batch))
    try:
        ks = KmerSet(k, budget, device)
    finally:
        if batch:
            if old is None:
                del os.environ["KUQ_KMER_SET_BATCH"]
            else:
                os.environ["KUQ_KMER_SET_BATCH"] = old
    try:
        ks.add(bases, offsets)
        parts, buf = [], np.zeros((1 << 20) * ks.rec, np.uint8)
        while True:
            n = ks.next(buf)
            if not n:
                break
            parts.append(buf[:n * ks.rec].copy())
        key_ct, passes = ks.info()
    finally:
        ks.close()
    return np.concatenate([kdb_header(k, key_ct)] + parts), passes


class CountUnique:
    """kuq_count_unique_*: count_unique's HyperLogLog estimate of a library's distinct forward k-mers on the GPU."""

    def __init__(self, k, p=14, batch=None, device=0):
        self.L = load_library()
        self.k, self.p = k, p
        h, err = C.c_void_p(), C.create_string_buffer(1024)
        rc = self.L.kuq_count_unique_create(device, k, p, int(batch or 0), C.byref(h), err, 1024)
        if rc != 0:
            raise KuqError(rc, err.value.decode() or self.L.kuq_strerror(rc).decode())
        self.h = h

    def _ck(self, rc):
        if rc != 0:
            raise KuqError(rc, f"{self.L.kuq_strerror(rc).decode()}: {self.L.kuq_count_unique_last_error(self.h).decode()}")

    def add(self, bases: np.ndarray, offsets: np.ndarray):
        bases = np.ascontiguousarray(bases, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.uint64)
        buf = bases if bases.size else np.zeros(1, np.uint8)
        self._ck(self.L.kuq_count_unique_add(self.h, buf.ctypes.data, _p(offsets, u64p), len(offsets) - 1))

    def result(self):
        """(estimate count_unique prints, valid windows, registers uint8[2^p])"""
        est, n = C.c_uint64(0), C.c_uint64(0)
        regs = np.zeros(1 << self.p, np.uint8)
        self._ck(self.L.kuq_count_unique_result(self.h, C.byref(est), C.byref(n), regs.ctypes.data))
        return est.value, n.value, regs

    def stats(self):
        ms, w, b = C.c_double(), C.c_uint64(), C.c_uint64()
        self._ck(self.L.kuq_count_unique_stats(self.h, C.byref(ms), C.byref(w), C.byref(b)))
        return {"sketch_ms": ms.value, "windows": w.value, "bases": b.value}

    def close(self):
        if getattr(self, "h", None):
            self.L.kuq_count_unique_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def count_unique(bases: np.ndarray, offsets: np.ndarray, k: int, p: int, batch=None, device=0):
    """What `count_unique -k k -p p` computes for the sequences bases[offsets[r]:offsets[r+1]] (FastaReader's
    sequences): (estimate, n_observed, registers uint8[2^p]).  batch = bases per device batch (None: 256 Mi)."""
    cu = CountUnique(k, p, batch, device)
    try:
        cu.add(bases, offsets)
        return cu.result()
    finally:
        cu.close()
