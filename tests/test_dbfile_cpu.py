"""kuq_dbfile.h, the one reader of database.kdb / database.idx, compiled for the host: every field of images built by
synth.build_db_images, and every refusal with its code and message.  Then classify, which checks every database right
after mapping it: a truncated index is refused with the library's message and EX_DATAERR before any device is looked
for, so this runs without a GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import build, synth

HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "krakenuniq_b200", "csrc", "kuq_dbfile.h")
KUQ_E_DB_FORMAT, KUQ_E_UNSUPPORTED_K = -4, -5

SHIM = r'''
#include "%s"
extern "C" int parse(const void *kdb, uint64_t kdb_bytes, const void *idx, uint64_t idx_bytes, uint64_t *out, char *msg,
                     size_t cap) {
  DbFile f;
  std::string err;
  const int rc = parse_db(kdb, kdb_bytes, idx, idx_bytes, f, err);
  snprintf(msg, cap, "%%s", err.c_str());
  if (rc) return rc;
  const uint64_t v[] = {f.key_bits, f.val_len, f.key_ct, f.k, f.key_len, f.pair_sz, f.header_bytes,
                        (uint64_t)(f.records - (const uint8_t *)kdb), (uint64_t)((const uint8_t *)f.offsets - (const uint8_t *)idx),
                        f.nt, f.idx_type, f.n_bins};
  memcpy(out, v, sizeof v);
  return rc;
}
extern "C" uint64_t mask(uint32_t k) { return kmer_mask(k); }
extern "C" uint64_t header_bytes(uint64_t key_bits) { return kdb_header_bytes(key_bits); }
'''
FIELDS = ("key_bits", "val_len", "key_ct", "k", "key_len", "pair_sz", "header_bytes", "records_at", "offsets_at", "nt",
          "idx_type", "n_bins")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("dbfile")
    (d / "s.cpp").write_text(SHIM % HDR)
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC", "-x", "c++", str(d / "s.cpp"),
                    "-o", str(d / "s.so")], check=True)
    so = ctypes.CDLL(str(d / "s.so"))
    so.mask.restype = so.header_bytes.restype = ctypes.c_uint64
    return so


def parse(lib, kdb, idx, kdb_bytes=None, idx_bytes=None):
    """→ (code, message, {field: value})"""
    kdb, idx = np.ascontiguousarray(kdb, np.uint8), np.ascontiguousarray(idx, np.uint8)
    out = np.zeros(len(FIELDS), np.uint64)
    msg = ctypes.create_string_buffer(256)
    rc = lib.parse(kdb.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint64(len(kdb) if kdb_bytes is None else kdb_bytes),
                   idx.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint64(len(idx) if idx_bytes is None else idx_bytes),
                   out.ctypes.data_as(ctypes.c_void_p), msg, ctypes.c_size_t(len(msg)))
    return rc, msg.value.decode(), dict(zip(FIELDS, (int(x) for x in out)))


def images(k, nt, idx_type, n=500, seed=0):
    rng = np.random.default_rng(seed)
    kmers = np.unique(synth.canonical(rng.integers(0, 1 << (2 * k), n, dtype=np.uint64), k))
    return synth.build_db_images(kmers, rng.integers(1, 1000, len(kmers)).astype(np.uint32), k=k, nt=nt, idx_type=idx_type)


@pytest.mark.parametrize("idx_type", [1, 2])
@pytest.mark.parametrize("k,nt", [(31, 5), (31, 8), (31, 11), (21, 5), (21, 8), (21, 11), (15, 5), (15, 8), (15, 11)])
def test_fields(lib, k, nt, idx_type):
    kdb, idx = images(k, nt, idx_type)
    rc, msg, f = parse(lib, kdb, idx)
    assert rc == 0 and msg == "", msg
    key_len = (2 * k + 7) // 8
    n_bins = 1 << (2 * nt)
    key_ct = (len(kdb) - len(synth.kdb_header(k, 0))) // (key_len + 4)
    assert f == dict(key_bits=2 * k, val_len=4, key_ct=key_ct, k=k, key_len=key_len, pair_sz=key_len + 4,
                     header_bytes=len(synth.kdb_header(k, 0)), records_at=len(synth.kdb_header(k, 0)), offsets_at=8, nt=nt,
                     idx_type=idx_type, n_bins=n_bins)
    offsets = np.frombuffer(idx[8:].tobytes(), np.uint64)
    assert len(offsets) == n_bins + 1 and offsets[-1] == key_ct


@pytest.mark.parametrize("k", [15, 21, 31])
def test_fields_nt15(lib, k):
    """An index of 4^15 + 1 offsets is 8 GiB: the parse reads none of them, so a header with that size declared will do."""
    kdb, _ = images(k, 5, 2)
    idx = np.frombuffer(b"KRAKIX2" + bytes([15]) + bytes(8), np.uint8)
    rc, msg, f = parse(lib, kdb, idx, idx_bytes=8 + 8 * ((1 << 30) + 1))
    assert rc == 0, msg
    assert (f["k"], f["nt"], f["idx_type"], f["n_bins"]) == (k, 15, 2, 1 << 30)
    rc, msg, _ = parse(lib, kdb, idx, idx_bytes=8 + 8 * (1 << 30))
    assert (rc, msg) == (KUQ_E_DB_FORMAT, "index file truncated")


def _set(a, at, value, width=8):
    a = a.copy()
    a[at:at + width] = np.frombuffer(int(value).to_bytes(width, "little"), np.uint8)
    return a


def test_refusals(lib):
    kdb, idx = images(31, 8, 2)
    hdr = len(synth.kdb_header(31, 0))
    cases = [
        (kdb[:55], idx, KUQ_E_DB_FORMAT, "database in improper format"),
        (_set(kdb, 0, int.from_bytes(b"JFLISTDX", "little")), idx, KUQ_E_DB_FORMAT, "database in improper format"),
        (_set(kdb, 16, 8), idx, KUQ_E_DB_FORMAT, "can only handle 4 byte DB values"),
        (_set(kdb, 8, 64), idx, KUQ_E_UNSUPPORTED_K, "k = 32 (key_len 8): k-mers up to 31 bases are supported"),
        (_set(kdb, 8, 63), idx, KUQ_E_UNSUPPORTED_K, "k = 31 (key_len 8): k-mers up to 31 bases are supported"),
        (kdb[:-1], idx, KUQ_E_DB_FORMAT, "database file truncated"),
        (kdb[:hdr - 1], idx, KUQ_E_DB_FORMAT, "database file truncated"),
        (kdb, idx[:7], KUQ_E_DB_FORMAT, "illegal Kraken DB index format"),
        (kdb, _set(idx, 0, int.from_bytes(b"KRAKIX3", "little"), 7), KUQ_E_DB_FORMAT, "illegal Kraken DB index format"),
        (kdb, _set(idx, 7, 0, 1), KUQ_E_DB_FORMAT, "index minimizer length 0 out of range"),
        (kdb, _set(idx, 7, 16, 1), KUQ_E_DB_FORMAT, "index minimizer length 16 out of range"),
        (kdb, idx[:-1], KUQ_E_DB_FORMAT, "index file truncated"),
    ]
    for i, (a, b, code, message) in enumerate(cases):
        rc, msg, _ = parse(lib, a, b)
        assert (rc, msg) == (code, message), i
    kdb5, _ = images(5, 5, 2, n=20)                              # nt == k is allowed, nt > k is not
    rc, msg, _ = parse(lib, kdb5, images(5, 5, 1, n=20)[1])
    assert rc == 0, msg
    rc, msg, _ = parse(lib, _set(kdb5, 8, 8), images(5, 5, 1, n=20)[1])
    assert (rc, msg) == (KUQ_E_DB_FORMAT, "index minimizer length 5 out of range")


def test_helpers(lib):
    assert [lib.mask(k) for k in (1, 15, 31, 32)] == [3, (1 << 30) - 1, (1 << 62) - 1, (1 << 64) - 1]
    assert [lib.header_bytes(b) for b in (2, 42, 62)] == [len(synth.kdb_header(k, 0)) for k in (1, 21, 31)]


@pytest.mark.parametrize("tool", ["classify", "classifyExact"])
@pytest.mark.parametrize("reads", [True, False])
def test_classify_refuses_a_truncated_index_before_any_device(tmp_path, tool, reads):
    """KUQ_HBM_BUDGET=4096 makes the database too large for the budget, so the streamed layout would plan its ranges from
    the index.  No device is visible: a run that got as far as the devices would exit EX_UNAVAILABLE (69) instead.
    Without reads (`-M`, the page-cache warm-up) the databases are checked all the same."""
    kdb, idx = images(31, 8, 2)
    kdb.tofile(tmp_path / "db.kdb")
    idx[:-8].tofile(tmp_path / "db.idx")
    synth.make_taxonomy(4).write(str(tmp_path / "taxDB"))
    (tmp_path / "r.fa").write_bytes(b">r\n" + b"ACGT" * 20 + b"\n")
    exe = os.path.join(os.path.dirname(build.build_classify()), tool)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", KUQ_HBM_BUDGET="4096")
    r = subprocess.run([exe, "-d", "db.kdb", "-i", "db.idx", "-a", "taxDB", "-M"] + (["r.fa"] if reads else []), cwd=tmp_path,
                       env=env, capture_output=True, text=True)
    assert r.returncode == 65 and "classify: index file truncated" in r.stderr, r.stderr
    idx.tofile(tmp_path / "db.idx")                              # the whole index gets as far as the devices
    if reads:
        r = subprocess.run([exe, "-d", "db.kdb", "-i", "db.idx", "-a", "taxDB", "r.fa"], cwd=tmp_path, env=env,
                           capture_output=True, text=True)
        assert r.returncode == 69, r.stderr
