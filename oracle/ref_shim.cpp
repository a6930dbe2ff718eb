// oracle/ref_shim.cpp — TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// A thin extern "C" veneer over the UNMODIFIED reference classes, compiled by oracle/build_ref.sh together with
// the reference's own krakendb.cpp / krakenutil.cpp / hyperloglogplus.cpp (from where $KUQ_REFERENCE_SRC says they
// lie) into oracle/_ref/libkuref.so.  It lets the tests pin oracle/kuq_oracle.c — and through it
// the CUDA path — against the real reference function by function (known-answer tests), because the reference
// itself ships no golden vectors (SURVEY.md §4, §8(c)).
//
// Every entry point names the reference function it forwards to.  Nothing here re-implements an algorithm.
#include <cstdint>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>
#include "krakendb.hpp"          // KrakenDB, KrakenDBIndex        (src/krakendb.hpp:30-140)
#include "krakenutil.hpp"        // KmerScanner, lca, resolve_tree (src/krakenutil.hpp:38-69)
#include "hyperloglogplus.hpp"   // HyperLogLogPlusMinus           (src/hyperloglogplus.hpp:62-121)

using namespace kraken;

// Non-inline free functions of hyperloglogplus.cpp (:131-161) that its header does not declare.
uint8_t getRank(const uint64_t hash_value, const uint8_t p);
uint8_t getEncodedRank(const uint32_t encoded_hash_value, const uint8_t pPrime, const uint8_t p);

namespace {
struct RefDB {
  KrakenDB *db;          // never deleted: ~KrakenDB munmaps an uninitialised pointer (src/krakendb.cpp:81-83)
  KrakenDBIndex *idx;
};
typedef std::unordered_map<uint32_t, uint32_t> umap;
umap make_map(const uint32_t *keys, const uint32_t *vals, uint32_t n) {
  umap m;
  for (uint32_t i = 0; i < n; i++) m[keys[i]] = vals[i];
  return m;
}
}  // namespace

extern "C" {

// murmurhash3_finalizer — src/hyperloglogplus.cpp:830-838
uint64_t kuref_murmur_fmix(uint64_t key) { return murmurhash3_finalizer(key); }

// ---- KrakenDB over in-memory file images (src/krakendb.cpp:60-78, 534-544) ------------------------------
// kdb_image / idx_image are byte-for-byte database.kdb / database.idx contents; they must outlive the handle.
void *kuref_db_open(char *kdb_image, uint64_t kdb_bytes, char *idx_image) {
  RefDB *h = new RefDB;
  h->db = new KrakenDB(kdb_image, kdb_bytes);
  h->idx = new KrakenDBIndex(idx_image);
  h->db->set_index(h->idx);
  return h;
}
uint32_t kuref_db_k(void *h) { return ((RefDB *)h)->db->get_k(); }
uint32_t kuref_db_index_nt(void *h) { return ((RefDB *)h)->idx->indexed_nt(); }
uint32_t kuref_db_index_type(void *h) { return ((RefDB *)h)->idx->index_type(); }
// KrakenDB::reverse_complement(kmer, n) — src/krakendb.cpp:218-225
uint64_t kuref_revcomp(void *h, uint64_t kmer, uint32_t n) { return ((RefDB *)h)->db->reverse_complement(kmer, (uint8_t)n); }
// KrakenDB::canonical_representation(kmer) — src/krakendb.cpp:243-246
uint64_t kuref_canonical(void *h, uint64_t kmer) { return ((RefDB *)h)->db->canonical_representation(kmer); }
// KrakenDB::bin_key(kmer) — src/krakendb.cpp:200-215
uint64_t kuref_bin_key(void *h, uint64_t kmer) { return ((RefDB *)h)->db->bin_key(kmer); }
// KrakenDB::bin_key(kmer, nt) — src/krakendb.cpp:182-196 (always the type-2 XOR mask)
uint64_t kuref_bin_key_nt(void *h, uint64_t kmer, uint32_t nt) { return ((RefDB *)h)->db->bin_key(kmer, nt); }
// KrakenDB::kmer_query(kmer) stateless form — src/krakendb.cpp:322-325.  Returns 1 + *taxon when found, 0 on miss
// (so a stored taxon 0 is distinguishable from a miss: SURVEY §7.3 item 8).
uint64_t kuref_kmer_query(void *h, uint64_t canon) {
  uint32_t *p = ((RefDB *)h)->db->kmer_query(canon);
  return p ? 1ull + *p : 0ull;
}
// The stateful call sequence classify_sequence makes (src/classify.cpp:911,928-936): one db_status per read.
// taxa_out[i] = taxon (0 on miss) for canon[i], fed in order with the cached-range shortcut active.
void kuref_kmer_query_stateful(void *h, const uint64_t *canon, uint32_t n, uint32_t *taxa_out) {
  uint64_t cur_bin = 0;
  int64_t cur_min = 1, cur_max = 0;   // db_status ctor, src/classify.cpp:115-120
  for (uint32_t i = 0; i < n; i++) {
    uint32_t *p = ((RefDB *)h)->db->kmer_query(canon[i], &cur_bin, &cur_min, &cur_max);
    taxa_out[i] = p ? *p : 0;
  }
}

// ---- KmerScanner (src/krakenutil.cpp:205-282).  k is process-global and settable once (:229-237). -------
// Returns the number of k-mers produced; kmers_out/ambig_out must hold max(len-k+1, 0) + 1 entries.
uint32_t kuref_scan(const char *seq, uint64_t len, uint32_t k, uint64_t *kmers_out, uint8_t *ambig_out) {
  KmerScanner::set_k((uint8_t)k);
  if (KmerScanner::get_k() != k) return 0xFFFFFFFFu;  // k already fixed to another value in this process
  std::string s(seq, len);
  uint32_t n = 0;
  if (s.size() >= k) {                 // guard of classify_sequence, src/classify.cpp:913
    KmerScanner scanner(s);
    uint64_t *kp;
    while ((kp = scanner.next_kmer()) != NULL) {
      kmers_out[n] = *kp;
      ambig_out[n] = scanner.ambig_kmer() ? 1 : 0;
      n++;
    }
  }
  return n;
}

// ---- lca / resolve_tree (src/krakenutil.cpp:90-118, 149-200) ---------------------------------------------
uint32_t kuref_lca(const uint32_t *pm_keys, const uint32_t *pm_vals, uint32_t pm_n, uint32_t a, uint32_t b) {
  umap pm = make_map(pm_keys, pm_vals, pm_n);
  return lca(pm, a, b);
}
void *kuref_parent_map_new(const uint32_t *pm_keys, const uint32_t *pm_vals, uint32_t pm_n) {
  return new umap(make_map(pm_keys, pm_vals, pm_n));
}
void kuref_parent_map_free(void *pm) { delete (umap *)pm; }
uint32_t kuref_lca_pm(void *pm, uint32_t a, uint32_t b) { return lca(*(umap *)pm, a, b); }
uint32_t kuref_resolve_tree(void *pm, const uint32_t *hit_taxa, const uint32_t *hit_counts, uint32_t n_hits) {
  umap hc = make_map(hit_taxa, hit_counts, n_hits);
  return resolve_tree(hc, *(umap *)pm);
}

// ---- HyperLogLogPlusMinus<uint64_t> (src/hyperloglogplus.cpp:427-753) ------------------------------------
typedef HyperLogLogPlusMinus<uint64_t> HLL;
void *kuref_hll_new(void) { return new HLL(); }                            // default ctor: p=12, sparse (readcounts.hpp:40)
void *kuref_hll_new_dense(uint32_t p) { return new HLL((uint8_t)p, false); }
void kuref_hll_free(void *h) { delete (HLL *)h; }
void kuref_hll_insert(void *h, const uint64_t *items, uint64_t n) {        // insert(), :485-523
  for (uint64_t i = 0; i < n; i++) ((HLL *)h)->insert(items[i]);
}
void kuref_hll_merge(void *dst, void *src) { *(HLL *)dst += *(const HLL *)src; }   // merge(const&), :627-665
void kuref_hll_merge_move(void *dst, void *src) { *(HLL *)dst += std::move(*(HLL *)src); }  // merge(&&), :586-625
uint64_t kuref_hll_cardinality(void *h) { return ((HLL *)h)->ertlCardinality(); }    // :722-753
uint64_t kuref_hll_n_observed(void *h) { return ((HLL *)h)->nObserved(); }
// getRank(uint64_t hash, p) — src/hyperloglogplus.cpp:140-147
uint32_t kuref_get_rank64(uint64_t hash, uint32_t p) { return getRank(hash, (uint8_t)p); }
// getEncodedRank(encoded, pPrime, p) — src/hyperloglogplus.cpp:152-161
uint32_t kuref_get_encoded_rank(uint32_t encoded, uint32_t p_prime, uint32_t p) {
  return getEncodedRank(encoded, (uint8_t)p_prime, (uint8_t)p);
}

}  // extern "C"
