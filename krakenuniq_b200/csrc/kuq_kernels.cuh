// kuq_kernels.cuh — sm_90a kernels of the KrakenUniq classification hot path (device side of libkuq.so).
//
// The per-read path of the reference's classify_sequence() (src/classify.cpp:897-1012) as three stages:
//
//  k_scan     read blocks --TMA bulk copy--> shared memory    (cp.async.bulk + mbarrier, double buffered)
//   (warp     2-bit packing + ambiguity mask   KmerScanner::next_kmer   src/krakenutil.cpp:239-282
//    per      canonical k-mer                  canonical_representation src/krakendb.cpp:238-246
//    read)    rolling minimizer                bin_key                  src/krakendb.cpp:200-215
//             → scratch: canonical k-mer + bin per window (12 B, coalesced)
//   or, for the fused call, k_pack (thread per 16 bases) + k_pack_reads (thread per read): 2-bit codes, ambiguity and
//   read-start masks per 32 text positions (16 B) — the lookup computes each window itself from two such blocks
//  k_lookup   index fetch + bin search         kmer_query               src/krakendb.cpp:250-321, :586-593
//   (thread   HLL register update              ReadCounts::add_kmer     src/readcounts.hpp:71-74,
//    per                                                                 hyperloglogplus.cpp:485-523
//    window)  → scratch: dense taxon id per window
//  k_resolve  hit aggregation + tree resolve   resolve_tree / lca       src/krakenutil.cpp:90-118,149-200
//   (warp     per-taxon counters               classify.cpp:939,968
//    per      run-length hit list              hitlist_string           src/classify.cpp:826-861
//    read)
//
// k_scan is ALU/shuffle work with no dependent memory access; k_lookup is the random-HBM stage and is written
// thread-per-window with a small register footprint so that ~48 warps per SM keep enough probes in flight;
// consecutive threads hold consecutive windows of a read, so windows sharing a minimizer touch the same index
// sector and the same pivots (coalesced by the load unit).  No tensor cores: the path is integer compares on
// randomly addressed HBM (SURVEY.md §8(d)).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kuq_buffers.cuh"

struct kuq_layout_result;

namespace kuq {

constexpr uint32_t AMBIG = 0xFFFFFFFFu;
// MODE_LOOKUP with flag 16: the key IS in the database but stores taxon 0 (an un-LCA'd record).  With several
// databases that still ends the search (classify.cpp:928-936), so the lookup has to tell it from a miss.
constexpr uint32_t FOUND_ZERO = 0xFFFFFFFDu;
constexpr int CTA_THREADS = 256;
constexpr int CTA_WARPS = CTA_THREADS / 32;
constexpr int CHUNK_READS = 64;            // reads per CTA work item
constexpr int STAGE_BYTES = 24 * 1024;     // bytes of read text per shared-memory stage
constexpr int N_STAGES = 2;
constexpr uint32_t HLL_P = 12;
constexpr uint32_t HLL_M = 4096;
// Record flag in the key word's free top bit (keys hold 2k <= 62 bits; the reference masks the rest away,
// krakendb.cpp:283-284): "a counted hit has seen this record since the last harvest" — the sparse HLL tier of hits.
constexpr uint32_t SEEN_BIT = 0x80000000u;
// Second record flag (bit 62, free for k <= 31): "this record's (taxon, encoded hash) is a key of the sparse tier".
// Only one record per (taxon, code) carries it — the primary of its collision group (kuq_api.cu, build_collisions).
constexpr uint32_t KEPT_BIT = 0x40000000u;
// Params::flags bit of a fused call that keeps records at their first sighting (keep mode): the lookup sets KEPT_BIT
// itself instead of SEEN_BIT, and marks the window whose atomic made the record kept with KEEP_NEW in codes_dense;
// k_resolve counts those windows into distinct[taxon] and *n_new_kept.  Secondaries of collision groups can become kept
// too; settle_kept (kuq_api.cu) hands their flag to the primary and takes the duplicate count back.
constexpr uint32_t F_KEEP = 64u;
constexpr uint32_t KEEP_NEW = 0x80000000u;   // never part of a dense id; AMBIG carries it too, so test AMBIG first
constexpr int SEARCH_WINDOW = 8;           // records scanned linearly once the bisection window is this small
constexpr uint32_t MAX_DBS = 8;            // databases one launch of the in-order lookup asks (Params::dbs)

enum Mode { MODE_FUSED = 0, MODE_LOOKUP = 1, MODE_RESOLVE = 2 };

struct DbView {
  const uint8_t *pairs;      // records of the staged range, on-disk layout: {u64 key, u32 value} packed to 12 B
  const uint64_t *offsets;   // offsets[b - bin_lo] = absolute record index of the first record of bin b
  uint64_t rec_base;         // absolute record index of pairs[0]
  uint64_t key_mask;         // (1 << 2k) - 1
  uint32_t bin_lo, bin_hi;   // staged minimizer range [bin_lo, bin_hi)
  uint32_t k, nt;
  uint32_t xor_mask;         // INDEX2_XOR_MASK & (4^nt - 1) for KRAKIX2, 0 for KRAKIDX (krakendb.cpp:45,203-206)
  uint32_t n_mini;           // k - nt + 1 minimizer candidates per k-mer (krakendb.cpp:208)
};

struct TaxView {
  const uint32_t *parent;    // dense id → dense id of the parent (0 = none), Parent_map of taxdb.hpp:383-398
  const uint16_t *depth;     // dense id → steps to the end of its parent chain (0 or the node of taxid 1)
  const uint32_t *raw;       // dense id → taxid
  uint32_t n_taxa;
  uint32_t n_sketch;         // dense ids < n_sketch own HLL registers / k-mer counters
};

struct SparseSet {           // device set of (dense taxon, encoded hash) pairs: the sparse HLL tier
  unsigned long long *slots; // 0 = empty; key = (taxon + 1) << 32 | code
  uint64_t mask;             // capacity - 1 (power of two)
  unsigned long long *n_used;
  uint32_t *distinct;        // [n_sketch] distinct codes per taxon (set keys + kept records)
};

// The sparse tier lives in two places: the slots of the set, and the staged records that carry KEPT_BIT.  Readouts
// scan one source per launch; a source with n == 0 launches nothing.
struct KeySource {
  const unsigned long long *slots;   // set slots, or nullptr for the record tier
  const uint8_t *pairs;              // records of the staged range (slots == nullptr)
  uint64_t n;                        // slots / records
  uint32_t hi_mask;                  // key bits of the record's high word
};

#ifdef __CUDACC__
// Owner and roll-up pass of a canonical k-mer of the exact set (kuq.h, kuq_exact_owner): a splitmix64 finalizer of the
// k-mer alone.  The table's slot hash mixes (k-mer, taxon) with another function, so an owner's part of a table does
// not crowd into a subset of its slots; the owner takes the high word, the roll-up passes the low word, so a context
// that holds one owner's part still splits evenly over the passes.
__host__ __device__ __forceinline__ uint64_t exact_kmer_hash(uint64_t kmer) {
  uint64_t x = kmer ^ 0x2545F4914F6CDD1Dull;
  x ^= x >> 30;
  x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27;
  x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}
__host__ __device__ __forceinline__ uint32_t exact_owner(uint64_t kmer, uint32_t n_parts) {
  return (uint32_t)(((exact_kmer_hash(kmer) >> 32) * n_parts) >> 32);
}
__host__ __device__ __forceinline__ uint32_t exact_pass(uint64_t kmer, uint32_t n_pass) {
  return (uint32_t)(((exact_kmer_hash(kmer) & 0xFFFFFFFFull) * n_pass) >> 32);
}

// murmurhash3_finalizer (hyperloglogplus.cpp:830-838)
__device__ __forceinline__ uint64_t fmix64(uint64_t key) {
  key += 1;
  key ^= key >> 33;
  key *= 0xff51afd7ed558ccdull;
  key ^= key >> 33;
  key *= 0xc4ceb9fe1a85ec53ull;
  key ^= key >> 33;
  return key;
}

// encodeHashIn32Bit(h, pPrime=25, p=12), hyperloglogplus.cpp:181-204
__device__ __forceinline__ uint32_t encode_hash32(uint64_t hash) {
  uint32_t idx = (uint32_t)((hash >> 39) << 7);
  if ((idx << 12) == 0) {
    uint64_t rest = hash << 25;
    uint32_t add_rank = rest ? (uint32_t)__clzll((long long)rest) + 1 : 40;
    return idx | (add_rank << 1) | 1;
  }
  return idx;
}

// KrakenDB::reverse_complement (krakendb.cpp:218-225): reverse the 2-bit groups, complement, shift down.
__device__ __forceinline__ uint64_t revcomp64(uint64_t x, uint32_t n) {
  x = __brevll(x);                                                              // reverses bits inside groups too
  x = ((x >> 1) & 0x5555555555555555ull) | ((x & 0x5555555555555555ull) << 1);  // ... so swap them back
  return (~x) >> (64 - 2 * n);
}
// One character → 2-bit code (A=0 C=1 G=2 T=3, case-insensitive, krakenutil.cpp:254-264); false = not ACGT.
__device__ __forceinline__ bool base_code(uint32_t c, uint32_t &code) {
  const uint32_t uc = c & 0xDFu;
  const bool ok = (uc == 'A') | (uc == 'C') | (uc == 'G') | (uc == 'T');
  code = ok ? (((c >> 1) ^ (c >> 2)) & 3u) : 0u;
  return ok;
}
// k-mer of the window that starts at base `lane` of the 128-bit string a:b (first base in bits 63:62 of a), k <= 31:
// the window's bases [lane, lane + k) in its top bits
__device__ __forceinline__ uint64_t window_top(uint64_t a, uint64_t b, uint32_t lane) {
  return lane ? (a << (2 * lane)) | (b >> (64 - 2 * lane)) : a;
}
// canonical k-mer (krakendb.cpp:238-246)
__device__ __forceinline__ uint64_t canonical_kmer(uint64_t top, uint32_t k) {
  const uint64_t kmer = top >> (64 - 2 * k);
  const uint64_t rc = revcomp64(kmer, k);
  return kmer < rc ? kmer : rc;
}

// set-key of a record: (taxon + 1) << 32 | encodeHashIn32Bit(hash(k-mer))
__device__ __forceinline__ unsigned long long record_key(const uint32_t *w, uint32_t hiw, uint32_t hi_mask) {
  const uint64_t kmer = ((uint64_t)(hiw & hi_mask) << 32) | w[0];
  return ((unsigned long long)(w[2] + 1) << 32) | encode_hash32(fmix64(kmer));
}

// item i of a key source: a set slot (0 = empty) or the key of a kept record (0 = not kept)
__device__ __forceinline__ unsigned long long source_key(const KeySource &s, uint64_t i) {
  if (s.slots) return s.slots[i];
  const uint32_t *w = reinterpret_cast<const uint32_t *>(s.pairs + i * 12);
  const uint32_t hiw = w[1];
  return (hiw & KEPT_BIT) ? record_key(w, hiw, s.hi_mask) : 0ull;
}
#endif

// Per-batch bookkeeping of the reference's per-work-unit sketches (classify.cpp:525: one ReadCounts map per work
// unit).  A (unit, taxon) sketch converts from sparse to dense iff an insert finds >= 1024 distinct encoded hashes
// already stored (hyperloglogplus.cpp:496-498), so only pairs with > 1024 inserts need their distinct count.
constexpr uint32_t UNIT_CODES = 2048;               // distinct-code table of one candidate pair (k_unit_decide)
constexpr uint32_t UNIT_DECIDE_CTAS_PER_SM = 4;
struct UnitMap {
  unsigned long long *keys;   // 0 = empty; (unit + 1) << 32 | taxon   (open addressing, per batch)
  uint32_t *inserts;          // N(unit, taxon): add_kmer calls
  uint32_t mask;              // capacity - 1
  uint32_t *cand;             // map slots of the candidate pairs (N >= 1025, taxon not already known dense)
  uint32_t *n_cand;           // [0] number of candidate pairs of the batch, [1] != 0: unit ids not ascending
  uint32_t *codes;            // k_unit_decide: per CTA, UNIT_CODES distinct codes + UNIT_CODES occurrence counts
  // fast path for the insert counts: units of a batch are (nearly always) consecutive ids, so N(unit, taxon) lives in a
  // dense table direct[(unit - unit_id[0]) * n_sketch + taxon] — one fire-and-forget atomic per (read, taxon), no probe.
  // Pairs outside the table (rows >= direct_rows) use the hash map above; k_unit_mark moves the candidates there.
  uint32_t *direct;
  uint32_t direct_rows;
};

// classifyExact (EXACT_COUNTING, classify.cpp:46-49): the per-taxon container is a set of canonical k-mers.  All
// sets of a run share one open-addressing table of 16-byte entries, filled with 128-bit compare-and-swap.
struct alignas(16) ExactPair {
  unsigned long long kmer1;    // canonical k-mer + 1 (0 = empty slot)
  unsigned long long taxon1;   // dense taxon id + 1
};
struct ExactSet {
  ExactPair *slots;
  uint64_t mask;               // capacity - 1 (power of two)
  unsigned long long *count;   // [n_sketch] distinct k-mers per taxon == khset size (readcounts.hpp:127-130)
};

// 2-bit packed copy of a batch (k_pack): block j holds the text positions [32j, 32j + 32), indexed like bases / 32
struct __align__(16) PackedBlock {
  uint64_t codes;              // 2-bit codes, position 32j in bits 63:62 (non-ACGT bases as A)
  uint32_t amb;                // bit l = position 32j + l is not ACGT (or lies outside the batch's text)
  uint32_t start;              // bit l = a read starts at 32j + l (also set at offsets[n_reads])
};
struct PackView {
  PackedBlock *blocks;
  uint32_t *side;              // bit l = position 32j + l belongs to a read holding '\n' / '\r': its windows are in scratch
};

struct Params {
  DbView db;
  TaxView tax;
  // batch
  const char *bases;            // 16-byte aligned, >= 32 bytes of slack after the last base
  const uint64_t *offsets;      // [n_reads + 1], relative to bases
  const uint32_t *unit_id;      // [n_reads] or nullptr
  char *clean;                  // scratch of the same size as bases for reads containing '\n' / '\r'
  uint32_t n_reads;
  uint32_t n_chunks;
  uint32_t flags;
  uint32_t hll_mode;
  // outputs
  uint32_t *call;               // [n_reads] taxid
  uint32_t *n_windows;          // [n_reads]
  uint32_t *codes;              // per window, indexed like bases (taxids; only with flag 1)
  uint64_t total_bases;
  // scratch between the stages (indexed like bases)
  uint64_t *canon;              // canonical k-mer of the window
  uint32_t *bins;               // minimizer bin, or BIN_AMBIG / BIN_NONE
  uint32_t *codes_dense;        // dense taxon id of the window (0 = miss) or AMBIG
  const uint32_t *codes_in;     // MODE_RESOLVE: merged dense ids
  PackView pack;                // the fused path's windows (see windows_packed)
  uint32_t packed;              // this call's windows come from `pack` (canon / bins hold only those of side reads)
  uint32_t *run_start;
  uint32_t *run_count;
  uint2 *runs;
  unsigned long long *run_cursor;
  uint64_t runs_capacity;       // entries of runs[]
  unsigned long long *n_classified;
  uint32_t *chunk_counter;      // dynamic chunk scheduler
  uint32_t *error_flag;
  uint32_t only_hits;           // MODE_LOOKUP: write hits only (peer-memory merge)
  // MODE_LOOKUP over NVLink: text positions [peer_bounds[j], peer_bounds[j+1]) belong to the reads GPU j resolves;
  // their hits are stored straight into that GPU's buffer (peer memory mapped through CUDA IPC)
  uint32_t n_peers;
  uint32_t *peer_codes[8];
  uint64_t peer_bounds[9];
  // MODE_LOOKUP over several databases (launch_lookup_multi): dbs[0, n_dbs) of one (k, nt, index type) are asked in
  // order; db = dbs[0] gives k_scan its window parameters.  only_hits 2 (fill empty): windows coded non-zero already are
  // skipped before any index fetch.  With n_peers (databases sharded by minimizer range over the GPUs), a window whose
  // bin lies in [run_lo, run_hi) — the bins this GPU holds of the launch's databases — is asked here and its hit stored
  // into the buffer of the GPU that resolves the read; fill empty then reads that GPU's word first.
  DbView dbs[MAX_DBS];
  uint32_t n_dbs;
  uint32_t run_lo, run_hi;
  unsigned long long *stats;    // flag 8: [0] += looked-up windows, [1] += sum of ceil(log2(bin size + 1))
  // per-taxon state
  uint8_t *regs;                // [n_sketch][4096]
  unsigned long long *n_kmers;  // [n_sketch]
  unsigned long long *n_reads_ctr; // [n_taxa]
  uint8_t *dense_flag;          // [n_sketch]
  const uint8_t *reg_floor;     // [n_sketch]: at most the smallest register of each sketch (launch_reg_floor)
  SparseSet sparse;
  unsigned long long *n_new_kept;  // F_KEEP: records the batch made kept (k_resolve adds them)
  UnitMap units;
  // pool for the hit tables of reads with more than 32 distinct taxa (2 u64 per entry)
  unsigned long long *ovf_mem;
  unsigned long long *ovf_cursor;
  uint64_t ovf_capacity;
  // quick mode (classify -q -m quick_min; 0 = off).  quick_stop: the read ends at its quick_min-th hit
  // (classify.cpp:943-944); otherwise every k-mer counts and only the call rule changes (the -x path, :701-738)
  uint32_t quick_min;
  uint32_t quick_stop;
  ExactSet exact;               // hll_mode 3 (KUQ_HLL_EXACT)
  // set_lcas: 1 = -T (values lca_keep[] stick, pieces with such a taxid overwrite), 2 = -R (values become 0)
  uint32_t lca_flags;
  uint32_t lca_keep[2];         // dense ids of taxids 32630 / 81077 (0 = not in the taxonomy)
  // confidence filter (kuq_set_threshold; fcall == nullptr = off).  Filter ids: the dense ids, then taxa of the
  // filter's parent map F that have no dense id (fextra[id - tax.n_taxa] = their taxids)
  const uint32_t *fparent;      // filter id → filter id of F[t]; meaningful where fdepth > 0
  const uint32_t *fdepth;       // filter id → F-steps to the end of its chain (0 = no F entry)
  const uint32_t *fextra;
  double fmin;                  // threshold - 1e-5
  uint32_t *fcall;              // [n_reads] taxid the call moves up to
  uint32_t *fhits;              // [n_reads] hits at or below the last weighed node ...
  uint32_t *ftotal;             // [n_reads] ... and the read's unambiguous k-mers (0 / 0: no node weighed)
};

// The fused lookup computes its windows itself from the packed copy of the batch; exact counting and quick-stop runs
// (and the lookup / resolve halves) read k_scan's scratch.  The caller sets p.packed from this before launch_classify.
bool windows_packed(int mode, const Params &p);
// returns #kernels launched; stage_events[0] / [1] (optional) are recorded after k_scan (or k_pack + k_pack_reads) /
// k_lookup
int launch_classify(int mode, const Params &p, int n_sm, cudaStream_t stream, cudaEvent_t *stage_events);
// canon / bins of the text positions [0, n_pos) from the packed copy the last fused call left in p.pack (side reads'
// windows are in scratch already): the scratch layout k_scan writes, for kuq_layout_experiment
void launch_unpack_windows(const Params &p, uint64_t n_pos, int n_sm, cudaStream_t stream);
int classify_smem_bytes();
int device_sm_count();
// ertlCardinality's estimator body (hyperloglogplus.cpp:738-752) from the register histogram C[0..q+1] of m registers:
// min(n_observed, round(estimate)) in the reference's order of operations (kuq_api.cu)
uint64_t ertl_from_hist(const int *C, size_t q, size_t m, uint64_t n_observed);
// set_lcas: k_scan + k_set_lcas over library pieces (p.unit_id = dense taxid per piece, p.stats[0] += k-mers not found)
int launch_set_lcas(const Params &p, int n_sm, cudaStream_t stream);
int launch_scan_only(const Params &p, int n_sm, cudaStream_t stream);
int launch_lookup_only(const Params &p, int n_sm, cudaStream_t stream, int fused, int lean);
// several databases: [k_scan with p.db's parameters when `scan`] + the in-order lookup over p.dbs into p.codes_dense;
// p.chunk_counter must be 0 when `scan`.  Returns #kernels launched.
int launch_lookup_multi(const Params &p, int n_sm, cudaStream_t stream, bool scan);
// db_sort on devices[0, n_dev) (kuq_dbbuild.cu; the current device is devices[0]): returns a KUQ_* code, *n_passes =
// per-range sorts (1 = in one piece)
int dbsort_device(const int *devices, uint32_t n_dev, const uint8_t *jdb_image, uint64_t jdb_bytes, uint32_t nt,
                  int zero_vals, uint64_t budget, uint8_t *kdb_out, uint8_t *idx_out, uint32_t *n_passes, char *err,
                  size_t err_cap);
// records per dense id of n 12-byte records, added to counts[0, n_ids); *bad = 1 when a value is n_ids or more
void launch_value_counts(const uint8_t *pairs, uint64_t n, uint32_t n_ids, unsigned long long *counts, uint32_t *bad,
                         cudaStream_t st);

// database staging helpers
void launch_collect_taxids(const uint8_t *pairs, uint64_t n_rec, uint32_t *keys, unsigned long long *counts,
                           uint32_t cap_mask, uint32_t *overflow, cudaStream_t stream);
void launch_remap_values(uint8_t *pairs, uint64_t n_rec, const uint32_t *keys, const uint32_t *dense,
                         uint32_t cap_mask, uint32_t *missing, uint64_t key_mask, cudaStream_t stream);
// records of key_len (1..7) + 4 bytes (k <= 28) → 12-byte records at wide12; narrow: 4-byte aligned, 16 bytes of slack
void launch_widen_records(const uint8_t *narrow, uint64_t n_rec, uint32_t key_len, uint8_t *wide12, cudaStream_t stream);
// flagged records → keys of the set: mode 0 count (stats[0]), 1 insert + clear, 2 clear SEEN_BIT and KEPT_BIT,
// 3 kept records → set (not counted again)
void launch_harvest_seen(uint8_t *pairs, uint64_t n_rec, uint64_t key_mask, const uint8_t *dense_flag, const SparseSet &set,
                         unsigned long long *stats, uint32_t *error_flag, int mode, cudaStream_t stream);
// flagged records → kept records (no set): secondaries hand their flag to their primaries, then one pass over the
// records sets KEPT_BIT, counts distinct[taxon] and clears SEEN_BIT (*n_kept += records that became kept).  pairs:
// 4-byte aligned; dense_flag has n_sketch entries, and every record's taxon is below n_sketch.
void launch_harvest_keep(uint8_t *pairs, uint64_t n_rec, const uint2 *secondaries, uint64_t n_secondaries, const uint8_t *dense_flag,
                         uint32_t n_sketch, uint32_t *distinct, unsigned long long *n_kept, cudaStream_t stream);
// after keep-mode calls: a kept secondary hands KEPT_BIT to its primary; where the primary had it already the code was
// counted twice, so distinct[taxon] drops by one and *n_dup grows by one
void launch_settle_kept(uint8_t *pairs, const uint2 *secondaries, uint64_t n_secondaries, uint32_t *distinct,
                        unsigned long long *n_dup, cudaStream_t stream);
// kuq_collisions.cu: (secondary, primary) record pairs of every (taxon, code) group of the staged records
int build_collisions(const uint8_t *pairs, uint64_t n_rec, uint64_t key_mask, const uint64_t *records_of_taxon, uint32_t n_sketch,
                     uint64_t max_entries, DevBuf<uint2> &list_out, uint64_t *n_out, int n_sm, cudaStream_t stream);
// the items of old_slots[0, old_cap) into a grown table without counting them again
void launch_rehash(const unsigned long long *old_slots, uint64_t old_cap, const SparseSet &s, uint32_t *error_flag, cudaStream_t stream);
void launch_rehash(const ExactPair *old_slots, uint64_t old_cap, const ExactSet &e, uint32_t *error_flag, cudaStream_t stream);
// floor[t] = the smallest of sketch t's registers
void launch_reg_floor(const uint8_t *regs, uint32_t n_sketch, uint8_t *floor, cudaStream_t stream);
void launch_register_histograms(const uint8_t *regs, uint32_t n_sketch, uint32_t *hist /*[n_sketch][64]*/,
                                cudaStream_t stream);
void launch_clade_max(const uint8_t *regs, const uint32_t *members, uint32_t n_members, uint8_t *out4096,
                      cudaStream_t stream);
void launch_fill_u32(uint32_t *p, uint64_t n, uint32_t v, cudaStream_t stream);
// HLL mode rule, per batch: mark candidate (unit, taxon) pairs, count their distinct codes, flag dense taxa
int launch_unit_accounting(const Params &p, int n_sm, cudaStream_t stream);
void launch_unit_clear(const UnitMap &u, uint32_t n_sketch, int n_sm, cudaStream_t stream);
// chunked rule: one global sketch per taxon converts once it holds >= 1025 distinct codes
void launch_flag_dense_global(const uint32_t *distinct, uint8_t *dense_flag, uint32_t n_sketch, cudaStream_t stream);
// kuq_set_extract: one byte per read (bit 0 selected XOR invert, bit 1 no Kraken line) and the batch's selected reads
// added to *count; members = the selected taxids, ascending
void launch_extract_select(const uint32_t *call, const uint32_t *fcall, uint32_t n_reads, const uint32_t *members,
                           uint32_t n_members, uint32_t flags, uint8_t *sel, uint32_t *count, cudaStream_t stream);
// histogram of encoded ranks over one source of the sparse tier, per taxon: hist[t][64] (+ hist[t][63] unused)
void launch_sparse_histograms(const KeySource &src, const uint8_t *dense_flag, uint32_t *hist, cudaStream_t stream);
// distinct codes of the union of the member taxa (member[t] != 0): rank histogram hist64 via a scratch set
// exact mode: distinct k-mers over the member taxa (set union of ReadCounts::operator+=, readcounts.hpp:76-81)
void launch_exact_union(const ExactSet &e, const uint8_t *member, unsigned long long *scratch_set, uint64_t scratch_mask,
                        unsigned long long *n_distinct, uint32_t *overflow, cudaStream_t stream);
// occupied slots [lo, hi) compacted into out (order unspecified); *n_out += their number, also beyond out_cap
void launch_exact_export(const ExactPair *slots, uint64_t lo, uint64_t hi, ExactPair *out, uint64_t out_cap,
                         unsigned long long *n_out, cudaStream_t stream);
// pairs (layout of ExactPair) into e; count[taxon] grows by the pairs that were new
void launch_exact_import(const ExactPair *pairs, uint64_t n, const ExactSet &e, uint32_t *error_flag, cudaStream_t stream);
// occupied slots [lo, hi) grouped by the owner of their k-mer (exact_owner, at most EXACT_MAX_PARTS parts): pass 0 adds
// the pairs per part to counters[part]; pass 1 scatters them through the cursors counters[part], bounded by part_end
constexpr uint32_t EXACT_MAX_PARTS = 64;
void launch_exact_parts(const ExactPair *slots, uint64_t lo, uint64_t hi, uint32_t n_parts, unsigned long long *counters,
                        ExactPair *out, const unsigned long long *part_end, uint32_t *error_flag, int pass, cudaStream_t stream);
void launch_sparse_union(const KeySource &src, const uint8_t *member,
                         unsigned long long *scratch_set, uint64_t scratch_mask, uint32_t *hist64, uint32_t *overflow,
                         cudaStream_t stream);

void launch_sparse_export(const KeySource &src, const uint8_t *dense_flag,
                          unsigned long long *out, uint64_t out_cap, unsigned long long *n_out, cudaStream_t stream);
void launch_sparse_import(const unsigned long long *keys, uint64_t n, const SparseSet &s, const uint8_t *dense_flag,
                          uint32_t *error_flag, cudaStream_t stream);

void launch_merge_state(uint8_t *regs, const uint8_t *regs2, unsigned long long *n_kmers, const unsigned long long *n_kmers2,
                        uint32_t n_sketch, unsigned long long *n_reads, const unsigned long long *n_reads2, uint32_t n_taxa,
                        uint8_t *dense, const uint8_t *dense2, cudaStream_t stream);
// cross-GPU flags (kuq_signal_peers / kuq_wait_flags) and the partitioned export of the sparse tier
void launch_signal_peers(unsigned long long *const *flag_ptrs, uint32_t n, uint32_t my_index, unsigned long long value,
                         cudaStream_t stream);
void launch_wait_flags(const unsigned long long *flags, uint32_t n, unsigned long long value, unsigned long long timeout_ns,
                       uint32_t *error_flag, cudaStream_t stream);
// keys of the still-sparse taxa grouped by owner part: src 0 = slots of the local set, src 1 = flagged records (pass 1
// clears the flags); pass 0 counts into counters[part], pass 1 scatters through counters[part] (cursors), bounded by part_end
void launch_keys_parts(int src, const unsigned long long *slots, uint8_t *pairs, uint64_t n_items, uint64_t key_mask,
                       const uint8_t *dense_flag, uint32_t n_parts, unsigned long long *counters, unsigned long long *out,
                       const unsigned long long *part_end, uint32_t *error_flag, int pass, cudaStream_t stream);

// kuq_clades.cu: all clades of the report at once
void launch_clade_max_batch(const uint8_t *regs, const uint32_t *d_offs, const uint32_t *d_members, uint32_t n_clades,
                            uint8_t *d_out, cudaStream_t stream);
int sparse_clade_dups(const KeySource &set_keys, const KeySource &kept_keys, const uint8_t *dense_flag, uint64_t n_keys_upper,
                      const uint32_t *d_pre_of_taxon, const uint32_t *d_node_of_pre, const uint32_t *d_parent_c,
                      const uint32_t *d_depth_c, const int32_t *d_sid_of_node, uint32_t *d_dup, int n_sm, cudaStream_t stream);
// exact mode: d_books[lca] -= 1 for every two pairs of the table with one k-mer that are adjacent in (k-mer, preorder)
// order, their LCA in the taxonomy (d_parent / d_depth of the context, 0 = none).  Taxa with pre_of_taxon NONE are left
// out.  In passes over parts of the k-mer space (exact_pass) sized to `budget` bytes of scratch.  0 = ok, 1 = not
// enough device memory for one pass, 2 = CUDA error.
int exact_clade_dups(const ExactPair *slots, uint64_t n_slots, uint64_t n_pairs, const uint32_t *d_pre_of_taxon,
                     const uint32_t *d_parent, const uint16_t *d_depth, unsigned long long *d_books, uint64_t budget, int n_sm,
                     cudaStream_t stream, uint32_t *passes_out);
// kuq_layout_exp.cu: record-layout / search-shape experiment (0 ok, 1 no memory, 2 CUDA error, 3 taxon ids > 24 bits);
// `product` = parameters of a k_lookup<MODE_LOOKUP> launch on the same database (scratch / output pointers are set there)
int layout_experiment(const Params &product, uint64_t n_records, const uint64_t *canon, const uint32_t *bins, const uint32_t *ref,
                      uint64_t n_pos, int n_sm, cudaStream_t st, uint32_t reps, int allow_fused, ::kuq_layout_result *res);

}  // namespace kuq
