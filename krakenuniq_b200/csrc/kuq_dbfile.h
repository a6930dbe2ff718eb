// The one reader of a Kraken database's files (database.kdb + database.idx, krakendb.cpp:60-78,141-147,176-177,534-544)
// for the library and every tool: where the header's fields and the records lie, and what makes an image malformed.
//
// database.kdb: "JFLISTDN", key_bits at byte 8, val_len at 16, key_ct at 48, a header of 72 + 2 * (4 + 8 * key_bits)
// bytes, then key_ct records of key_len key bytes and a 4-byte value.  database.idx: "KRAKIDX" or "KRAKIX2" (bins XORed
// with a mask), the minimizer length nt in byte 7, then the 4^nt + 1 running record counts of the bins.
#ifndef KUQ_DBFILE_H
#define KUQ_DBFILE_H
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>

#include "../../include/kuq.h"

inline uint64_t kdb_header_bytes(uint64_t key_bits) { return 72 + 2 * (4 + 8 * key_bits); }
inline uint64_t kdb_key_len(uint64_t key_bits) { return key_bits / 8 + !!(key_bits % 8); }
inline uint64_t kmer_mask(uint32_t k) { return k >= 32 ? ~0ull : ((1ull << (2 * k)) - 1); }

// The .kdb header as it stands, unchecked (db_sort reads unsorted Jellyfish dumps with checks of its own).  The image
// must hold at least 56 bytes.
struct KdbFile {
  uint64_t key_bits, val_len, key_ct;
  uint32_t k;
  uint64_t key_len, pair_sz;   // pair_sz: the file's record size, key_len + 4 (pair_size(), krakendb.cpp:76,176)
  uint64_t header_bytes;
  const uint8_t *records;      // the first record
};
inline KdbFile kdb_view(const void *image) {
  const uint8_t *p = (const uint8_t *)image;
  KdbFile h;
  memcpy(&h.key_bits, p + 8, 8);
  memcpy(&h.val_len, p + 16, 8);
  memcpy(&h.key_ct, p + 48, 8);
  h.k = (uint32_t)(h.key_bits / 2);
  h.key_len = kdb_key_len(h.key_bits);
  h.pair_sz = h.key_len + 4;
  h.header_bytes = kdb_header_bytes(h.key_bits);
  h.records = p + h.header_bytes;
  return h;
}

// A validated database: the .kdb view plus its index.
struct DbFile : KdbFile {
  const uint64_t *offsets;     // 4^nt + 1 cumulative record offsets
  uint32_t nt, idx_type;       // idx_type 1: KRAKIDX, 2: KRAKIX2
  uint64_t n_bins;             // 4^nt
};

// Returns KUQ_OK with f filled, or a KUQ_E_* code with the message in err.
inline int parse_db(const void *kdb_image, uint64_t kdb_bytes, const void *idx_image, uint64_t idx_bytes, DbFile &f,
                    std::string &err) {
  char msg[128];
  auto fail = [&](int code, const char *m) { err = m; return code; };
  if (kdb_bytes < 56 || memcmp(kdb_image, "JFLISTDN", 8) != 0)                    // krakendb.cpp:32,67-68
    return fail(KUQ_E_DB_FORMAT, "database in improper format");
  static_cast<KdbFile &>(f) = kdb_view(kdb_image);
  if (f.val_len != 4) return fail(KUQ_E_DB_FORMAT, "can only handle 4 byte DB values");   // :73-74
  if (f.key_bits > 62) {
    snprintf(msg, sizeof msg, "k = %u (key_len %llu): k-mers up to 31 bases are supported", f.k, (unsigned long long)f.key_len);
    return fail(KUQ_E_UNSUPPORTED_K, msg);
  }
  if (kdb_bytes < f.header_bytes + f.key_ct * f.pair_sz) return fail(KUQ_E_DB_FORMAT, "database file truncated");
  const uint8_t *q = (const uint8_t *)idx_image;
  if (idx_bytes < 8) return fail(KUQ_E_DB_FORMAT, "illegal Kraken DB index format");
  if (memcmp(q, "KRAKIDX", 7) == 0) f.idx_type = 1;
  else if (memcmp(q, "KRAKIX2", 7) == 0) f.idx_type = 2;
  else return fail(KUQ_E_DB_FORMAT, "illegal Kraken DB index format");             // :541
  f.nt = q[7];
  if (f.nt < 1 || f.nt > 15 || f.nt > f.k) {
    snprintf(msg, sizeof msg, "index minimizer length %u out of range", f.nt);
    return fail(KUQ_E_DB_FORMAT, msg);
  }
  f.n_bins = 1ull << (2 * f.nt);
  if (idx_bytes < 8 + 8 * (f.n_bins + 1)) return fail(KUQ_E_DB_FORMAT, "index file truncated");
  f.offsets = (const uint64_t *)(q + 8);
  return KUQ_OK;
}

#endif
