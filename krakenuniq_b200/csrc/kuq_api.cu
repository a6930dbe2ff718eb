// kuq_api.cu — host side of libkuq.so: the C ABI declared in include/kuq.h.
//
// Owns HBM (database range, taxonomy arrays, per-taxon state), the batch slots (stream + device and pinned
// host staging) and the host-side pieces of the path that are not data parallel: database header validation
// (kuq_dbfile.h), dense taxon numbering, work-unit cutting (classify.cpp:514-520) and the
// double-precision Ertl estimator (hyperloglogplus.cpp:722-753).  There is no CPU classification path: without
// an sm_90 device kuq_create fails with KUQ_E_NO_DEVICE.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <type_traits>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/kuq.h"
#include "kuq_batches.h"
#include "kuq_bounce.cuh"
#include "kuq_dbfile.h"
#include "kuq_kernels.cuh"

using namespace kuq;

namespace {

constexpr uint64_t INDEX2_XOR_MASK = 0xe37e28c4271b5a2dULL;   // krakendb.cpp:45
constexpr uint32_t SLACK = 64;                                // bytes readable past the end of a bases buffer
constexpr uint32_t UMAP_CAP = 1u << 21;                       // (unit, taxon) pairs per batch

struct Slot {
  Stream stream;
  Event ev_k0, ev_k1, ev_stage[2], ev_sync;
  double stage_ms[3] = {0, 0, 0};
  // device
  DevBuf<char> d_bases, d_clean;
  DevBuf<uint64_t> d_offsets;
  DevBuf<uint32_t> d_unit, d_call, d_nwin, d_codes;
  // HLL mode rule bookkeeping (KUQ_HLL_PRELOAD), allocated on first use
  DevBuf<unsigned long long> u_keys;
  DevBuf<uint32_t> u_inserts, u_cand, u_ncand, u_direct, u_codes;
  uint32_t u_direct_rows = 0;
  DevBuf<uint64_t> d_canon;                    // scratch between the stages
  DevBuf<uint32_t> d_bins, d_dense, d_codes_in;
  DevBuf<PackedBlock> d_pack;                  // the fused path's 2-bit copy of the batch (k_pack)
  DevBuf<uint32_t> d_side;
  bool windows_packed = false;                 // the last call's windows are in d_pack, not in d_canon / d_bins
  DevBuf<unsigned long long> d_ovf;            // hit-table pool for reads with > 32 distinct taxa
  uint64_t ovf_entries = 0;
  DevBuf<uint32_t> d_run_start, d_run_count;
  DevBuf<uint2> d_runs;
  uint64_t runs_cap = 0;
  DevBuf<unsigned long long> d_scalars;        // [0] run cursor, [1] n_classified, [2] chunk counter(u32) [3] error(u32)
  // pinned host
  HostBuf<uint32_t> h_call, h_nwin, h_run_start, h_run_count, h_codes;
  HostBuf<uint32_t> h_unit;
  // confidence filter (kuq_set_threshold): filtered call, hits and total per read, allocated when it is set
  DevBuf<uint32_t> d_fcall, d_fhits, d_ftotal;
  HostBuf<uint32_t> h_fcall, h_fhits, h_ftotal;
  // read selection (kuq_set_extract): one byte per read, then the batch's selected reads (u32 at extract_count_at)
  DevBuf<uint8_t> d_xsel;
  HostBuf<uint8_t> h_xsel;
  HostBuf<kuq_run> h_runs;
  uint64_t h_runs_cap = 0;
  HostBuf<unsigned long long> h_scalars;
  // in-flight batch
  bool busy = false;
  bool timed = false;      // the timing events of this slot have been recorded at least once
  uint32_t n_reads = 0, flags = 0;
  uint64_t total_bases = 0;
  double kernel_ms = 0;
  bool external = false;   // inputs are caller-owned device buffers
  const char *x_bases = nullptr;
};

}  // namespace

// One open-addressing table in HBM: the sparse-tier set (8-byte keys (taxon + 1) << 32 | code) or the exact k-mer set
// (16-byte ExactPairs).  A context has at most one of them.
template <typename Item, typename Count>
struct DevTable {
  DevBuf<Item> slots;
  DevBuf<Count> count;                    // [n_sketch] items per taxon
  uint64_t cap = 0;                       // slots, a power of two
  uint64_t upper = 0;                     // upper bound of the items since the last exact count (reserve_room)
  uint64_t grown = 0;                     // times the slots were re-allocated
};
using SparseTable = DevTable<unsigned long long, uint32_t>;
using ExactTable = DevTable<ExactPair, unsigned long long>;

struct CountsHost {
  std::vector<unsigned long long> n_kmers, n_reads;
  std::vector<uint32_t> hist;      // [n_sketch][64]
  std::vector<uint8_t> dense_flag;
  std::vector<uint32_t> distinct;
  std::vector<uint32_t> sparse_hist;   // [n_sketch][64] rank histogram of the sparse tier
  std::vector<unsigned long long> exact;   // KUQ_HLL_EXACT: [n_sketch] distinct k-mers per taxon
};

// The DbView inputs of one staged minimizer range: its records (12-byte layout) and index slice on the device
struct DbRange {
  uint8_t *pairs = nullptr;
  const uint64_t *offsets = nullptr;
  uint64_t key_ct = 0, rec_base = 0, bin_lo = 0, bin_hi = 0;
  uint32_t nt = 0, idx_type = 0;
};

// One staged database or minimizer range of one.  Its records are owned here when they were staged from a host image
// (own_pairs), else they are the caller's (kuq_attach_db_device) or a stream buffer's.
struct StagedDb {
  DbRange range;
  DevBuf<uint8_t> own_pairs;
  DevBuf<uint64_t> own_offsets;
  // device hash of the range's taxids (keys = taxid + 1), and the distinct taxids (ascending) with their record counts
  DevBuf<uint32_t> d_tx_keys, d_tx_dense;
  DevBuf<unsigned long long> d_tx_counts;
  uint32_t tx_cap = 0;
  std::vector<uint32_t> taxids;
  std::vector<uint64_t> counts;
  bool remapped = false;                  // the record values are dense ids
};

struct kuq_ctx {
  kuq_config cfg;
  CountsHost snap;                 // host copy of the per-taxon state, valid until the next batch
  bool snap_valid = false;
  int device = 0;
  int n_sm = 132;
  std::string err;
  std::vector<Slot> slots;
  uint64_t launches = 0;
  Stream aux;

  // the staged databases (or minimizer ranges of them) in the order they are asked (kuq_stage_db_append_range), all of
  // the same k; none = no database staged.  dbs[0] is the range the record tier works on.
  uint32_t k = 0;
  std::vector<StagedDb> dbs;
  std::vector<uint32_t> universe;         // taxids of all records of the database (optional)

  // taxonomy
  bool tax_set = false, finalized = false;
  uint32_t quick_min = 0;                 // kuq_set_quick_mode: classify -q -m quick_min (0 = off)
  bool quick_stop = false;                // reads end at their quick_min-th hit (preloaded path) or not (-x path)
  bool mark_zero_hits = false;            // kuq_mark_zero_hits: lookups report stored taxon 0 as KUQ_CODE_FOUND_ZERO
  std::vector<uint32_t> tax_ids, tax_parents;
  std::vector<uint32_t> raw_of_dense;
  std::vector<uint32_t> parent_dense;     // host copy of d_parent (dense id of the parent, 0 = none)
  std::unordered_map<uint32_t, uint32_t> dense_of_raw;
  uint32_t n_taxa = 0, n_sketch = 0;
  DevBuf<uint32_t> d_parent, d_raw;
  DevBuf<uint16_t> d_depth;
  // kuq_set_threshold: krakenuniq-filter's parent map F (taxid → parent) with the F-depth of every node; uploaded in
  // filter ids (Params::fparent) once the dense numbering exists
  bool filter_set = false;
  double threshold = 0;
  std::unordered_map<uint32_t, uint32_t> f_parent, f_depth;
  DevBuf<uint32_t> d_fparent, d_fdepth, d_fextra;
  // kuq_set_extract: the selected taxids, ascending, and the KUQ_EXTRACT_* flags
  bool extract_set = false;
  uint32_t extract_flags = 0, n_members = 0;
  DevBuf<uint32_t> d_members;

  // per-taxon state
  DevBuf<uint8_t> d_regs, d_dense_flag;
  DevBuf<uint8_t> d_reg_floor;            // [n_sketch]: lower bound of each sketch's registers (refresh_reg_floor)
  DevBuf<unsigned long long> d_n_kmers, d_n_reads;
  DevBuf<unsigned long long> d_sparse_used;
  SparseTable sparse;                     // the sparse-tier set; count[] includes the keys of kept records
  ExactTable exact;                       // KUQ_HLL_EXACT: the (taxon, k-mer) table and the per-taxon set sizes
  bool exact_partitioned = false;         // kuq_exact_replace / kuq_exact_partition: the table holds one owner's part
  bool merged_exact = false;              // kuq_set_exact_summary: merged_exact_count / merged_books hold sums over parts
  std::vector<unsigned long long> merged_exact_count;
  std::vector<long long> merged_books;
  std::vector<uint32_t> exact_pre;        // preorder of every sketch taxon in the taxonomy (exact roll-up), built once
  DevBuf<uint32_t> d_exact_pre;
  uint32_t exact_rollup_passes = 0;       // k-mer passes of the last exact roll-up
  // kuq_set_exact_spill: a table that cannot grow moves its pairs to host memory, grouped by owner part
  // (exact_owner(k-mer, EXACT_MAX_PARTS)), and kuq_exact_settle counts the parts at the end
  uint64_t spill_budget = 0;              // bytes of spilled pairs the process may hold (0 = no spilling)
  uint64_t spills = 0;                    // times the table spilled since the last reset
  uint64_t spilled_pairs = 0;             // pairs held in spill_parts (their bytes are taken from the budget)
  std::vector<std::vector<ExactPair>> spill_parts[EXACT_MAX_PARTS];   // pieces of each part, one per round that had some

  // database streamed through HBM range by range (kuq_stream_*): two device buffers, one copy stream
  struct StreamBuf {
    DevBuf<uint8_t> d_pairs;
    DevBuf<uint64_t> d_offsets;
    Event ready;
    DbRange range;                        // what kuq_stream_use makes dbs[0]'s range
    bool loaded = false;
  } sbuf[2];
  bool stream_open = false;
  uint64_t stream_cap_records = 0, stream_cap_bins = 0;
  Stream copy_stream;
  DevBuf<uint32_t> d_stream_missing;
  uint64_t stream_pair_sz = 12;           // record size of the streamed database's file (key_len + 4)
  DevBuf<uint8_t> d_stream_land;          // k <= 28: landing zone of stream_land_rec file records, widened from there
  uint64_t stream_land_rec = 0;
  bool shard_counting = false;            // kuq_set_shard_counting: hits are counted by the GPU that finds them
  uint32_t extra_flags = 0;               // kuq_set_stats: KUQ_F_STATS for calls that take no flags
  DevBuf<uint32_t> d_sync_err;            // set by a kuq_wait_flags that timed out
  bool merged_summary = false;            // kuq_set_sparse_summary: snap.sparse_hist / distinct hold cross-GPU sums
  std::vector<uint32_t> merged_hist, merged_distinct;
  bool seen_dirty = false;                // counted hits flagged records since the last harvest (SEEN_BIT)
  // record tier of the sparse HLL tier (KEPT_BIT): a resident range keeps its hits' keys in the records themselves
  DevBuf<uint2> d_secondaries;            // (secondary, primary) record pairs of the (taxon, code) groups of the range
  uint64_t n_secondaries = 0;
  int collisions = 0;                     // that table: 0 = not built yet, 1 = built, -1 = none (harvests fill the set)
  double collisions_ms = 0;               // time the table took to build
  bool kept = false;                      // some staged records carry KEPT_BIT
  uint64_t kept_keys = 0;                 // keys held by kept records (included in sparse.count)
  bool set_has_hits = false;              // the set holds keys of hits, which kept records could duplicate
  bool keep_dirty = false;                // fused calls kept records at their first sighting (F_KEEP) since settle_kept
  double harvest_ms = 0;                  // device time of the last harvest
  // the harvest's counters and timing events, made at the first harvest (or keep-mode call) and kept: a cudaMalloc /
  // cudaFree pair per harvest held the device idle at the end of every run.  [0], [1]: the harvest's; [2]: records that
  // keep-mode calls made kept since settle_kept (k_resolve counts them)
  DevBuf<unsigned long long> d_harvest_stat;
  Event harvest_ev[2];
  bool lca_mode = false;                  // kuq_set_lcas_batch ran: record values are LCA results, not classifiable
  WorkUnits units;                        // the open work unit across batches (kuq_batches.h)
};

namespace {

void stream_close(kuq_ctx *ctx);
int harvest_seen(kuq_ctx *ctx, bool discard, bool to_set = false);
int settle_kept(kuq_ctx *ctx);

// Records of a database with k <= 28 are shorter than the 12 bytes they take in HBM; they pass through a device landing
// zone of this many records on their way there.  64 MiB unless KUQ_LANDING_BYTES says otherwise (a small zone cuts a
// small database into many pieces, which is what tests of the piece arithmetic want).
uint64_t landing_records(uint64_t pair_sz) {
  uint64_t bytes = 64ull << 20;
  if (const char *e = getenv("KUQ_LANDING_BYTES")) bytes = strtoull(e, nullptr, 10);
  return std::max<uint64_t>(1, bytes / pair_sz);
}

int fail(kuq_ctx *c, int code, const char *fmt, ...) {
  if (c) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    c->err = buf;
  }
  return code;
}

#define CU(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if (e__ != cudaSuccess)                                                                        \
      return fail(ctx, KUQ_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

void free_db(kuq_ctx *ctx) {
  ctx->dbs.clear();
  ctx->d_secondaries.reset();
  ctx->n_secondaries = 0; ctx->collisions = 0;
}

// the record tier's range: the first staged one, or an empty range when none is staged
const DbRange &first_range(const kuq_ctx *ctx) {
  static const DbRange none;
  return ctx->dbs.empty() ? none : ctx->dbs[0].range;
}

}  // namespace

namespace kuq {
// ---- Ertl estimator (hyperloglogplus.cpp:373-422,738-752), same operation order as the reference ----------
double ertl_sigma(double x) {
  if (x == 1.0) return INFINITY;
  double prev, sigma_x = x, y = 1.0;
  do { prev = sigma_x; x *= x; sigma_x += x * y; y += y; } while (sigma_x != prev);
  return sigma_x;
}
double ertl_tau(double x) {
  if (x == 0.0 || x == 1.0) return 0.0;
  double prev, y = 1.0, tau_x = 1 - x;
  do { prev = tau_x; x = std::sqrt(x); y /= 2.0; tau_x -= std::pow(1 - x, 2) * y; } while (tau_x != prev);
  return tau_x / 3.0;
}
uint64_t ertl_from_hist(const int *C, size_t q, size_t m, uint64_t n_observed) {
  double est_denominator = m * ertl_tau(1.0 - double(C[q + 1]) / double(m));
  for (int k = (int)q; k >= 1; --k) { est_denominator += C[k]; est_denominator *= 0.5; }
  est_denominator += m * ertl_sigma(double(C[0]) / double(m));
  double m_sq_alpha_inf = (m / (2.0 * std::log(2))) * m;
  double est = m_sq_alpha_inf / est_denominator;
  return (double(n_observed) < est) ? n_observed : (uint64_t)std::round(est);
}
}  // namespace kuq

namespace {

uint64_t ertl_dense_hist(const uint32_t *hist64, uint64_t n_observed) {
  int C[66];
  for (int i = 0; i < 64; i++) C[i] = (int)hist64[i];
  C[64] = C[65] = 0;
  return ertl_from_hist(C, 64 - HLL_P, HLL_M, n_observed);
}
// ertlCardinality of a sparse sketch (hyperloglogplus.cpp:726-729): q = 64 - 25, m = 2^25, C from
// sparseRegisterHistogram (:356-366): hist64[r] = distinct codes of encoded rank r, C[0] = m - |S|.
uint64_t ertl_sparse_hist(const uint32_t *hist64, uint64_t n_codes, uint64_t n_observed) {
  int C[66];
  memset(C, 0, sizeof C);
  for (int i = 1; i <= 40; i++) C[i] = (int)hist64[i];
  const size_t m = 1u << 25;
  C[0] = (int)(m - n_codes);
  return ertl_from_hist(C, 64 - 25, m, n_observed);
}

int alloc_slot(kuq_ctx *ctx, Slot &s) {
  const uint64_t mr = ctx->cfg.max_reads_per_batch, mb = ctx->cfg.max_bases_per_batch;
  CU(s.stream.alloc(cudaStreamNonBlocking));
  CU(s.ev_k0.alloc(cudaEventDefault));
  CU(s.ev_k1.alloc(cudaEventDefault));
  CU(s.ev_stage[0].alloc(cudaEventDefault));
  CU(s.ev_stage[1].alloc(cudaEventDefault));
  CU(s.ev_sync.alloc(cudaEventDisableTiming));
  CU(s.d_bases.alloc(mb + SLACK));
  CU(s.d_clean.alloc(mb + SLACK));
  CU(s.d_offsets.alloc(mr + 4));   // + slack: offsets slices are bulk-copied in 16-byte units
  CU(s.d_unit.alloc(mr));
  CU(s.d_call.alloc(mr));
  CU(s.d_nwin.alloc(mr));
  CU(s.d_codes.alloc(mb + SLACK));
  CU(s.d_canon.alloc(mb + SLACK));
  CU(s.d_bins.alloc(mb + SLACK));
  CU(s.d_pack.alloc((mb + SLACK) / 32 + 3));   // blocks up to the one after the last text position
  CU(s.d_side.alloc((mb + SLACK) / 32 + 3));
  CU(s.d_dense.alloc(mb + SLACK));
  // worst case one table of < 4 * windows entries per read: 4 entries (64 B) per base always suffices, but reads that
  // need it are rare: a pool of max(bases / 4, 1 Mi) entries + the largest single table
  s.ovf_entries = std::max<uint64_t>(mb / 4, 1ull << 20);
  CU(s.d_ovf.alloc(2 * s.ovf_entries));
  CU(s.d_run_start.alloc(mr));
  CU(s.d_run_count.alloc(mr));
  // every resolving warp may leave one partly used block of 256 run slots behind (k_resolve)
  s.runs_cap = mb + SLACK + 256ull * (uint64_t)ctx->n_sm * 64;
  if (s.runs_cap > 0xFFFFFF00ull) s.runs_cap = 0xFFFFFF00ull;   // run indices are 32-bit
  CU(s.d_runs.alloc(s.runs_cap));
  CU(s.d_scalars.alloc(8));
  CU(cudaMemset(s.d_scalars, 0, 8 * 8));           // kuq_sync_slot reads the error word even before the first batch
  CU(s.h_call.alloc(mr));
  CU(s.h_nwin.alloc(mr));
  CU(s.h_run_start.alloc(mr));
  CU(s.h_run_count.alloc(mr));
  CU(s.h_unit.alloc(mr));
  CU(s.h_scalars.alloc(8));
  s.h_runs_cap = std::max<uint64_t>(mr * 8, 1024);
  CU(s.h_runs.alloc(s.h_runs_cap));
  return KUQ_OK;
}

int check_slot(kuq_ctx *ctx, uint32_t slot) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  if (slot >= ctx->slots.size()) return fail(ctx, KUQ_E_INVALID_ARG, "slot %u out of range (%zu slots)", slot, ctx->slots.size());
  return KUQ_OK;
}

// Scan the records of a staged range for their distinct taxids (+counts): count_taxons (krakendb.cpp:90-113) on the GPU.
// The device hash (keys, dense ids to be filled, counts) and the sorted taxids / counts go to the range's fields.
int collect_taxids(kuq_ctx *ctx, StagedDb &db) {
  DevBuf<uint32_t> &d_keys = db.d_tx_keys, &d_dense = db.d_tx_dense;
  DevBuf<unsigned long long> &d_counts = db.d_tx_counts;
  uint32_t cap = 1u << 16;
  for (;;) {
    d_keys.reset(); d_counts.reset(); d_dense.reset();
    CU(d_keys.alloc(cap));
    CU(d_counts.alloc(cap));
    CU(d_dense.alloc(cap));
    CU(cudaMemsetAsync(d_keys, 0, cap * 4ull, ctx->aux));
    CU(cudaMemsetAsync(d_counts, 0, cap * 8ull, ctx->aux));
    DevBuf<uint32_t> d_over;
    CU(d_over.alloc(1));
    CU(cudaMemsetAsync(d_over, 0, 4, ctx->aux));
    launch_collect_taxids(db.range.pairs, db.range.key_ct, d_keys, d_counts, cap - 1, d_over, ctx->aux);
    ctx->launches++;
    uint32_t over = 0;
    CU(cudaMemcpyAsync(&over, d_over, 4, cudaMemcpyDeviceToHost, ctx->aux));
    CU(cudaStreamSynchronize(ctx->aux));
    d_over.reset();
    if (over == 2) return fail(ctx, KUQ_E_DB_FORMAT, "taxid 0xFFFFFFFF is reserved");
    std::vector<uint32_t> keys(cap);
    std::vector<unsigned long long> counts(cap);
    CU(cudaMemcpy(keys.data(), d_keys, cap * 4ull, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(counts.data(), d_counts, cap * 8ull, cudaMemcpyDeviceToHost));
    uint64_t used = 0;
    for (uint32_t i = 0; i < cap; i++) used += keys[i] != 0;
    if (over == 1 || used * 2 > cap) {            // too full: the probe chains got long or overflowed
      if (cap >= (1u << 28)) return fail(ctx, KUQ_E_CAPACITY, "more than 2^27 distinct taxids in the database");
      cap <<= 2;
      continue;
    }
    std::vector<std::pair<uint32_t, uint64_t>> v;
    v.reserve(used);
    for (uint32_t i = 0; i < cap; i++) if (keys[i]) v.emplace_back(keys[i] - 1, counts[i]);
    std::sort(v.begin(), v.end());
    db.taxids.clear(); db.counts.clear();
    for (auto &pr : v) { db.taxids.push_back(pr.first); db.counts.push_back(pr.second); }
    db.tx_cap = cap;
    return KUQ_OK;
  }
}

// ---- the two device tables: the sparse-tier set and the exact k-mer set ---------------------------------------------
// What differs between them is supplied by the overloads below: the device view (whose counter the kernels add to),
// the kernels that re-insert and import items, the slot cap and the messages.  The routines after them are written
// once over both tables.
// KUQ_EXACT_MAX_SLOTS caps the slots the exact set may grow to, as if the device had no room for more: tests use it to
// build, on one card, runs whose union exceeds one context's table (0 / unset = no cap)
uint64_t max_slots(const SparseTable &) { return 0; }
uint64_t max_slots(const ExactTable &) {
  const char *e = getenv("KUQ_EXACT_MAX_SLOTS");
  return e ? strtoull(e, nullptr, 10) : 0;
}
SparseSet set_view(const kuq_ctx *ctx, const SparseTable &t) {
  return SparseSet{t.slots, t.cap ? t.cap - 1 : 0, ctx->d_sparse_used, t.count};
}
ExactSet set_view(const kuq_ctx *, const ExactTable &t) { return ExactSet{t.slots, t.cap ? t.cap - 1 : 0, t.count}; }
void launch_import(kuq_ctx *ctx, const unsigned long long *keys, uint64_t n, const SparseSet &s, uint32_t *err) {
  launch_sparse_import(keys, n, s, ctx->d_dense_flag, err, ctx->aux);
}
void launch_import(kuq_ctx *ctx, const ExactPair *pairs, uint64_t n, const ExactSet &e, uint32_t *err) {
  launch_exact_import(pairs, n, e, err, ctx->aux);
}
// The messages of each table.  printf arguments: no_room_to_grow takes (slots now, slots wanted, GiB wanted), the two
// `saturated` messages take the slots.
struct TableText {
  const char *name, *items, *no_room_to_grow, *saturated_importing, *saturated_building, *overran;
};
const TableText SPARSE_TEXT{"sparse-tier set", "keys", "sparse-tier set: no room to grow from %llu to %llu slots",
                            "sparse-tier set saturated while importing", "sparse-tier set saturated while importing",
                            "internal: partitioned export overran a segment"};
const TableText EXACT_TEXT{"exact k-mer set", "pairs", "exact k-mer set: no room to grow from %llu to %llu slots (%.2f GiB)",
                           "exact k-mer set saturated while importing (%llu slots)",
                           "exact k-mer set saturated while building a part (%llu slots)", "internal: partitioned export overran a part"};
const TableText &text(const SparseTable &) { return SPARSE_TEXT; }
const TableText &text(const ExactTable &) { return EXACT_TEXT; }
// a table of `cap` slots for `incoming` items could not be allocated
int no_room_for(kuq_ctx *ctx, const SparseTable &, uint64_t, uint64_t cap) {
  (void)cudaGetLastError();
  return fail(ctx, KUQ_E_NOMEM, "sparse-tier set: no room for %llu slots", (unsigned long long)cap);
}
int no_room_for(kuq_ctx *ctx, const ExactTable &, uint64_t incoming, uint64_t cap) {
  (void)cudaGetLastError();
  return fail(ctx, KUQ_E_NOMEM, "exact k-mer set: no room for a part of %llu pairs (%llu slots, %.2f GiB) on device %d",
              (unsigned long long)incoming, (unsigned long long)cap, cap * 16.0 / (1ull << 30), ctx->device);
}

// Runs `launch(d_err)` on ctx->aux with a zeroed device word that its kernels set when the table they fill is full, and
// turns a set word into KUQ_E_CAPACITY with the message (fmt, args).
template <typename Launch, typename... Args>
int run_saturating(kuq_ctx *ctx, Launch launch, const char *fmt, Args... args) {
  DevBuf<uint32_t> d_err;
  CU(d_err.alloc(1));
  CU(cudaMemsetAsync(d_err, 0, 4, ctx->aux));
  launch(d_err);
  ctx->launches++;
  uint32_t err = 0;
  CU(cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, ctx->aux));
  CU(cudaStreamSynchronize(ctx->aux));
  return err ? fail(ctx, KUQ_E_CAPACITY, fmt, args...) : KUQ_OK;
}

// the table's per-taxon counter on the host, and the items in the table: every item was counted once, under its taxon
template <typename Table, typename Count>
int table_counts(kuq_ctx *ctx, const Table &t, std::vector<Count> &count, uint64_t *n) {
  count.resize(ctx->n_sketch);
  CU(cudaMemcpy(count.data(), t.count, ctx->n_sketch * sizeof count[0], cudaMemcpyDeviceToHost));
  *n = 0;
  for (auto v : count) *n += v;
  return KUQ_OK;
}
template <typename Table>
int table_items(kuq_ctx *ctx, const Table &t, uint64_t *n) {
  std::vector<std::remove_pointer_t<decltype(t.count.get())>> count;
  return table_counts(ctx, t, count, n);
}

// slots for n items at a load of at most tenths / 10: `cap`, doubled as often as that needs
uint64_t slots_for(uint64_t n, uint64_t cap, uint64_t tenths) {
  cap = std::max<uint64_t>(cap, 1);
  while (n * 10 > cap * tenths) cap <<= 1;
  return cap;
}

// Re-allocate the table with `cap` slots and re-insert its items (not counted again).  All slots must be idle.
template <typename Table>
int grow_table(kuq_ctx *ctx, Table &t, uint64_t cap) {
  decltype(t.slots) bigger;
  const uint64_t max = max_slots(t), old_cap = t.cap;
  if ((max && cap > max) || bigger.alloc(cap) != cudaSuccess) {
    (void)cudaGetLastError();
    return fail(ctx, KUQ_E_NOMEM, text(t).no_room_to_grow, (unsigned long long)t.cap, (unsigned long long)cap,
                cap * (double)sizeof *t.slots.get() / (1ull << 30));
  }
  CU(cudaMemsetAsync(bigger, 0, cap * sizeof *t.slots.get(), ctx->aux));
  decltype(t.slots) old = std::move(t.slots);
  t.slots = std::move(bigger);
  t.cap = cap;
  const int rc = run_saturating(ctx, [&](uint32_t *err) { launch_rehash(old, old_cap, set_view(ctx, t), err, ctx->aux); },
                                "%s saturated while growing to %llu slots", text(t).name, (unsigned long long)cap);
  if (rc) {
    t.slots = std::move(old);
    t.cap = old_cap;
    return rc;
  }
  t.grown++;
  return KUQ_OK;
}

// The one growth rule of both tables: `used` items in the table and `incoming` more to come; when they could pass a
// load factor of 0.8, the table grows to a load of at most 0.6.  t.upper becomes their sum.  All slots must be idle.
template <typename Table>
int make_room(kuq_ctx *ctx, Table &t, uint64_t used, uint64_t incoming) {
  t.upper = used;
  if ((used + incoming) * 10 > t.cap * 8) {
    int rc = grow_table(ctx, t, slots_for(used + incoming, t.cap, 6));
    if (rc) return rc;
  }
  t.upper += incoming;
  return KUQ_OK;
}

// Room for `incoming` more items, made BEFORE a batch instead of failing in the middle of it: t.upper bounds the items
// since the last exact count, and only when the bound could pass the load of make_room does `fill` read the exact count
// back (all slots drained first).
template <typename Table, typename Fill>
int reserve_room(kuq_ctx *ctx, Table &t, uint64_t incoming, Fill fill) {
  if ((t.upper + incoming) * 10 <= t.cap * 8) { t.upper += incoming; return KUQ_OK; }
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  uint64_t used = 0;
  int rc = fill(&used);
  if (rc) return rc;
  return make_room(ctx, t, used, incoming);
}

// Items (the table's layout) into the table; its counter grows by the items that were new.  The caller made room.
template <typename Table, typename Item>
int import_items(kuq_ctx *ctx, Table &t, const Item *items, uint64_t n, bool building = false) {
  if (!n) return KUQ_OK;
  return run_saturating(ctx, [&](uint32_t *err) { launch_import(ctx, items, n, set_view(ctx, t), err); },
                        building ? text(t).saturated_building : text(t).saturated_importing, (unsigned long long)t.cap);
}

template <typename Table>
int clear_table(kuq_ctx *ctx, Table &t) {
  CU(cudaMemsetAsync(t.slots, 0, t.cap * sizeof *t.slots, ctx->aux));
  CU(cudaMemsetAsync(t.count, 0, ctx->n_sketch * sizeof *t.count, ctx->aux));
  CU(cudaStreamSynchronize(ctx->aux));
  t.upper = 0;
  return KUQ_OK;
}

// A fresh table for `incoming` items at a load of at most tenths / 10 from `start` slots up (the slot cap applies as to
// growth), zeroed, with a zeroed per-taxon counter.  On ctx's device.
template <typename Table>
int alloc_table(kuq_ctx *ctx, uint64_t incoming, uint64_t start, uint64_t tenths, Table &t) {
  const uint64_t cap = slots_for(incoming, start, tenths), max = max_slots(t);
  if ((max && cap > max) || t.slots.alloc(cap) != cudaSuccess || t.count.alloc(ctx->n_sketch) != cudaSuccess) {
    t = Table{};
    return no_room_for(ctx, t, incoming, cap);
  }
  t.cap = cap;
  return clear_table(ctx, t);
}

// the built table replaces the context's; `upper` bounds its items
template <typename Table>
void install_table(Table &t, Table &built, uint64_t upper) {
  built.grown = t.grown + (built.cap != t.cap);
  built.upper = upper;
  t = std::move(built);
}

// The table's items become the received ones (the old ones were exported before), in a table sized for them at a load
// of at most tenths / 10 from `start` slots up.  A table of another size replaces the old slots after they are freed,
// so the peak is the received items and the new table.  When that fails, the context keeps an empty table of the old
// size.  All slots must be idle.
template <typename Table, typename Item>
int replace_table(kuq_ctx *ctx, Table &t, const Item *items, uint64_t n, uint64_t start, uint64_t tenths) {
  const uint64_t old_cap = t.cap, cap = slots_for(n, start, tenths), max = max_slots(t);
  int rc = KUQ_OK;
  if (cap != old_cap) {
    t.slots.reset();
    if ((max && cap > max) || t.slots.alloc(cap) != cudaSuccess) rc = no_room_for(ctx, t, n, cap);
  }
  t.cap = cap;
  if (!rc) rc = clear_table(ctx, t);
  if (!rc) rc = import_items(ctx, t, items, n, true);
  if (!rc) {
    t.grown += cap != old_cap;
    t.upper = n;
    return KUQ_OK;
  }
  t.cap = old_cap;
  if (cap != old_cap && t.slots.alloc(old_cap) != cudaSuccess) {
    (void)cudaGetLastError();
    t.cap = t.upper = 0;
    return rc;
  }
  clear_table(ctx, t);
  return rc;
}

// The table's occupied slots compacted into out (cap items; out == nullptr only counts) by `launch(out, cap, d_n)`;
// *n = their number.  All slots idle.
template <typename Item, typename Launch>
int export_items(kuq_ctx *ctx, Item *out, uint64_t cap, uint64_t *n, const char *items, Launch launch) {
  DevBuf<unsigned long long> d_n;
  CU(d_n.alloc(1));
  CU(cudaMemsetAsync(d_n, 0, 8, ctx->aux));
  launch(out, out ? cap : 0, d_n);
  unsigned long long cnt = 0;
  CU(cudaMemcpyAsync(&cnt, d_n, 8, cudaMemcpyDeviceToHost, ctx->aux));
  CU(cudaStreamSynchronize(ctx->aux));
  *n = cnt;
  if (out && cnt > cap) return fail(ctx, KUQ_E_CAPACITY, "need room for %llu %s", cnt, items);
  return KUQ_OK;
}

// The partitioned export: items grouped by owner part into out (cap items), parts back to back; counts[part] = items per
// part.  `scan(counters, out, part_end, err, pass)` launches the table's parts kernels: pass 0 counts per part, pass 1
// scatters through the part cursors, bounded by the part ends.  out == nullptr only counts, unless alloc_out asks the
// library to size the buffer after the counting pass and hand it out.  All slots idle.
template <typename Item, typename Scan>
int export_parts(kuq_ctx *ctx, uint32_t n_parts, uint32_t max_parts, Item *out, uint64_t cap, uint64_t *counts, Item **alloc_out,
                 const TableText &tx, Scan scan) {
  const uint32_t P = max_parts;
  DevBuf<unsigned long long> d_cnt;
  CU(d_cnt.alloc(2 * P + 1));                    // [0, P) counts / cursors, [P, 2P) part ends, [2P] error word
  CU(cudaMemsetAsync(d_cnt, 0, (2 * P + 1) * 8ull, ctx->aux));
  uint32_t *d_err = reinterpret_cast<uint32_t *>(d_cnt + 2 * P);
  scan(d_cnt, nullptr, nullptr, d_err, 0);
  std::vector<unsigned long long> h(2 * P, 0);
  CU(cudaMemcpyAsync(h.data(), d_cnt, P * 8ull, cudaMemcpyDeviceToHost, ctx->aux));
  CU(cudaStreamSynchronize(ctx->aux));
  uint64_t total = 0;
  for (uint32_t j = 0; j < n_parts; j++) { counts[j] = h[j]; total += h[j]; }
  DevBuf<Item> owned;                            // alloc_out's buffer until it is handed out
  if (alloc_out) {
    if (owned.alloc(std::max<uint64_t>(total, 1)) != cudaSuccess) {
      (void)cudaGetLastError();
      return fail(ctx, KUQ_E_NOMEM, "no room for %llu exported %s", (unsigned long long)total, tx.items);
    }
    out = owned;
    cap = total;
  }
  if (!out) return KUQ_OK;                       // counts only: nothing was consumed
  int rc = KUQ_OK;
  if (total > cap) {
    rc = fail(ctx, KUQ_E_CAPACITY, "need room for %llu %s", (unsigned long long)total, tx.items);
  } else {
    unsigned long long at = 0;
    for (uint32_t j = 0; j < P; j++) {
      const unsigned long long c = j < n_parts ? h[j] : 0;
      h[j] = at;
      h[P + j] = at + c;
      at += c;
    }
    CU(cudaMemcpyAsync(d_cnt, h.data(), 2 * P * 8ull, cudaMemcpyHostToDevice, ctx->aux));
    scan(d_cnt, out, d_cnt + P, d_err, 1);
    uint32_t err = 0;
    CU(cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, ctx->aux));
    CU(cudaStreamSynchronize(ctx->aux));
    if (err) rc = fail(ctx, KUQ_E_CAPACITY, tx.overran);
  }
  if (alloc_out && !rc) *alloc_out = owned.release();
  return rc;
}

// kuq_sparse_tier_info / kuq_exact_info: the table's slots, items and growths
template <typename Table>
int table_info(kuq_ctx *ctx, const Table &t, uint64_t *slots, uint64_t *items, uint64_t *times_grown) {
  if (slots) *slots = t.cap;
  if (times_grown) *times_grown = t.grown;
  if (!items) return KUQ_OK;
  *items = 0;
  if (!t.count) return KUQ_OK;
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  if (ctx->keep_dirty) {                         // duplicates of collision groups out first
    int rc = settle_kept(ctx);
    if (rc) return rc;
  }
  return table_items(ctx, t, items);
}

// Misses and the resolve half insert (taxon, code) pairs straight into the set — at most one per window of the batch.
int reserve_direct_inserts(kuq_ctx *ctx, uint64_t windows) {
  if (!ctx->sparse.slots) return KUQ_OK;
  auto fill = [ctx](uint64_t *used) -> int {
    uint64_t n = 0;
    int rc = table_items(ctx, ctx->sparse, &n);
    if (rc) return rc;
    // keys of kept records live in the records, not in the set; those of keep-mode calls since the last settle_kept are
    // counted in count[] and in d_harvest_stat[2] alike (duplicates of collision groups included)
    unsigned long long pending = 0;
    if (ctx->keep_dirty) CU(cudaMemcpy(&pending, ctx->d_harvest_stat + 2, 8, cudaMemcpyDeviceToHost));
    *used = n - std::min<uint64_t>(n, ctx->kept_keys + pending);
    return KUQ_OK;
  };
  return reserve_room(ctx, ctx->sparse, windows, fill);
}

// A batch adds at most one pair per non-ambiguous window; an import at most one per incoming pair.
int reserve_exact_inserts(kuq_ctx *ctx, uint64_t incoming) {
  if (!ctx->exact.slots) return KUQ_OK;
  return reserve_room(ctx, ctx->exact, incoming, [ctx](uint64_t *used) { return table_items(ctx, ctx->exact, used); });
}

// Occupied slots [lo, hi) of the exact table into out (cap pairs; cap 0 only counts); *n = their number.  All slots idle.
int exact_export_range(kuq_ctx *ctx, uint64_t lo, uint64_t hi, ExactPair *out, uint64_t cap, uint64_t *n) {
  return export_items(ctx, out, cap, n, "pairs", [&](ExactPair *o, uint64_t c, unsigned long long *d_n) {
    launch_exact_export(ctx->exact.slots, lo, hi, o, c, d_n, ctx->aux);
    ctx->launches++;
  });
}

// Slots [lo, hi) of the exact table grouped by owner (exact_owner) into out, parts back to back (export_parts).
int exact_parts(kuq_ctx *ctx, uint64_t lo, uint64_t hi, uint32_t n_parts, ExactPair *out, uint64_t cap, uint64_t *counts,
                ExactPair **alloc_out = nullptr) {
  return export_parts(ctx, n_parts, EXACT_MAX_PARTS, out, cap, counts, alloc_out, EXACT_TEXT,
                      [&](unsigned long long *cnt, ExactPair *o, const unsigned long long *end, uint32_t *err, int pass) {
                        launch_exact_parts(ctx->exact.slots, lo, hi, n_parts, cnt, o, end, err, pass, ctx->aux);
                        ctx->launches++;
                      });
}

// pairs of another context (ExactPair layout) into the table, grown first when they need room.  All slots idle.
int exact_import(kuq_ctx *ctx, const ExactPair *d_pairs, uint64_t n) {
  int rc = reserve_exact_inserts(ctx, n);
  if (rc) return rc;
  ctx->snap_valid = false;
  return import_items(ctx, ctx->exact, d_pairs, n);
}

// a batch's kernels found the set they insert into full (error code 4)
int batch_set_saturated(kuq_ctx *ctx) {
  if (ctx->cfg.hll_mode == KUQ_HLL_EXACT)
    return fail(ctx, KUQ_E_CAPACITY, "exact k-mer set saturated (%llu slots)", (unsigned long long)ctx->exact.cap);
  return fail(ctx, KUQ_E_CAPACITY, "sparse-tier set saturated: raise kuq_config.sparse_set_slots (now %llu)", (unsigned long long)ctx->sparse.cap);
}

// Slots of a table per round when its pairs move between contexts or to the host: 2^22 (64 MiB of pairs), or
// KUQ_EXACT_MERGE_SLOTS, so that tests of the rounds can use small tables
uint64_t exact_round_slots() {
  uint64_t round_slots = 1ull << 22;
  if (const char *e = getenv("KUQ_EXACT_MERGE_SLOTS")) round_slots = std::max<uint64_t>(1, strtoull(e, nullptr, 10));
  return round_slots;
}

// src's exact pairs go to the tables of dsts[0, n) in rounds over at most 2^22 slots of src's table (64 MiB of pairs per
// round on each side; KUQ_EXACT_MERGE_SLOTS overrides it, so that tests of the rounds can use small tables).
// `gather(lo, hi, buf, cap, counts)` compacts the slots [lo, hi) into buf on src's device, grouped by destination with
// counts[o] pairs for dsts[o]; each group is copied peer to peer when its destination is on another device and handed
// to `take(o, pairs, m)` there.  Peak per device: one round on each side.  Errors are reported on `report`.  The slots
// of all contexts must be idle.
template <typename Gather, typename Take>
int move_rounds(kuq_ctx *report, const char *no_room, kuq_ctx *src, kuq_ctx *const *dsts, uint32_t n, Gather gather, Take take) {
  kuq_ctx *ctx = report;
  const uint64_t chunk = std::min(exact_round_slots(), src->exact.cap);
  DevBuf<ExactPair> send;
  std::vector<DevBuf<ExactPair>> recv(n);
  int rc = KUQ_OK;
  for (uint32_t o = 0; o <= n && !rc; o++) {     // the round buffer on src's device, then one on each other destination's
    kuq_ctx *c = o < n ? dsts[o] : src;
    DevBuf<ExactPair> &buf = o < n ? recv[o] : send;
    if (o < n && c->device == src->device) continue;
    CU(cudaSetDevice(c->device));
    if (buf.alloc(std::max<uint64_t>(chunk, 1)) != cudaSuccess) {
      (void)cudaGetLastError();
      rc = fail(ctx, KUQ_E_NOMEM, no_room, (unsigned long long)chunk, c->device);
    }
  }
  std::vector<uint64_t> counts(n);
  for (uint64_t lo = 0; lo < src->exact.cap && !rc; lo += chunk) {
    CU(cudaSetDevice(src->device));
    rc = gather(lo, std::min(lo + chunk, src->exact.cap), send, chunk, counts.data());
    if (rc) { report->err = src->err; break; }
    uint64_t off = 0;
    for (uint32_t o = 0; o < n && !rc; o++) {
      const uint64_t m = counts[o];
      const ExactPair *from = send + off;
      off += m;
      if (!m) continue;
      kuq_ctx *dst = dsts[o];
      CU(cudaSetDevice(dst->device));
      if (recv[o]) {
        CU(cudaMemcpyPeer(recv[o], dst->device, from, src->device, m * 16));
        from = recv[o];
      }
      rc = take(o, from, m);
      if (rc && dst != report) report->err = dst->err;
    }
  }
  cudaSetDevice(report->device);
  return rc;
}

// kuq_merge_into under KUQ_HLL_EXACT: src's pairs move to dst's table in rounds (move_rounds), imported on dst's device
// (count[] grows by the pairs dst did not hold yet).  Union does not depend on order, so dst ends with the set one
// context would have built.  The slots of both contexts must be idle.
int merge_exact_pairs(kuq_ctx *dst, kuq_ctx *src) {
  if (!src->exact.slots || !dst->exact.slots) return KUQ_OK;
  return move_rounds(
      dst, "exact k-mer set merge: no room for %llu pairs on device %d", src, &dst, 1,
      [src](uint64_t lo, uint64_t hi, ExactPair *buf, uint64_t cap, uint64_t *counts) { return exact_export_range(src, lo, hi, buf, cap, counts); },
      [dst](uint32_t, const ExactPair *pairs, uint64_t m) { return exact_import(dst, pairs, m); });
}

// ---- the exact set spilled to host memory (kuq_set_exact_spill, kuq_exact_settle) -----------------------------------
// Bytes of spilled pairs held by all contexts of the process; a spill takes its bytes before it copies anything.
std::atomic<uint64_t> g_spill_bytes{0};

bool take_spill_bytes(uint64_t bytes, uint64_t budget) {
  uint64_t cur = g_spill_bytes.load();
  do {
    if (cur + bytes > budget) return false;
  } while (!g_spill_bytes.compare_exchange_weak(cur, cur + bytes));
  return true;
}

// the context's host parts go, and their bytes return to the budget
void drop_spill(kuq_ctx *ctx) {
  g_spill_bytes -= ctx->spilled_pairs * sizeof(ExactPair);
  ctx->spilled_pairs = 0;
  for (auto &part : ctx->spill_parts) std::vector<std::vector<ExactPair>>().swap(part);
}

int refuse_spilled(kuq_ctx *ctx, const char *call) {
  return fail(ctx, KUQ_E_STATE, "%s: the exact k-mer set has spilled %llu pairs to host memory and the device holds only part of "
                                "it: count it with kuq_exact_settle first", call, (unsigned long long)ctx->spilled_pairs);
}

// A device and a pinned buffer of `chunk` pairs for rounds between the host parts and a table.  The card may be full, so
// `chunk` halves until both can be allocated (down to 1024 pairs); false when even that fails.
bool round_buffers(uint64_t &chunk, DevBuf<ExactPair> &d_buf, HostBuf<ExactPair> &h_buf) {
  for (;; chunk /= 2) {
    if (d_buf.alloc(chunk) == cudaSuccess && h_buf.alloc(chunk) == cudaSuccess) return true;
    (void)cudaGetLastError();
    d_buf.reset();
    if (chunk <= 1024) return false;
  }
}

// Every pair of the table to the context's host parts, then the table is emptied (counts included) at the same
// capacity.  Rounds over exact_round_slots() slots: the round's pairs grouped by owner part (the partitioned export's
// kernel over a slot range) into a device buffer, through a pinned buffer into the parts.  The card is full when this
// runs, so the round buffer halves until it can be allocated.  All slots idle.
int spill_exact(kuq_ctx *ctx) {
  ExactTable &t = ctx->exact;
  uint64_t n = 0;
  int rc = table_items(ctx, t, &n);
  if (rc || !n) return rc;
  const uint64_t bytes = n * sizeof(ExactPair);
  if (!take_spill_bytes(bytes, ctx->spill_budget))
    return fail(ctx, KUQ_E_NOMEM, "exact k-mer set: spilling %llu pairs (%.2f GiB) to host memory would pass the host budget of "
                                  "%llu bytes (KUQ_EXACT_HOST_BUDGET), of which the process holds %llu already",
                (unsigned long long)n, bytes / double(1ull << 30), (unsigned long long)ctx->spill_budget,
                (unsigned long long)g_spill_bytes.load());
  uint64_t chunk = std::min(exact_round_slots(), t.cap), moved = 0;
  DevBuf<ExactPair> d_buf;
  HostBuf<ExactPair> h_buf;
  if (!round_buffers(chunk, d_buf, h_buf))
    rc = fail(ctx, KUQ_E_NOMEM, "exact k-mer set: no memory for a spill round of %llu pairs on device %d", (unsigned long long)chunk, ctx->device);
  uint64_t counts[EXACT_MAX_PARTS];
  for (uint64_t lo = 0; lo < t.cap && !rc; lo += chunk) {
    rc = exact_parts(ctx, lo, std::min(lo + chunk, t.cap), EXACT_MAX_PARTS, d_buf, chunk, counts);
    uint64_t m = 0;
    for (uint32_t j = 0; j < EXACT_MAX_PARTS && !rc; j++) m += counts[j];
    if (rc || !m) continue;
    if (cudaMemcpyAsync(h_buf, d_buf, m * sizeof(ExactPair), cudaMemcpyDeviceToHost, ctx->aux) != cudaSuccess ||
        cudaStreamSynchronize(ctx->aux) != cudaSuccess) {
      rc = fail(ctx, KUQ_E_CUDA, "exact k-mer set: spill copy failed: %s", cudaGetErrorString(cudaGetLastError()));
      break;
    }
    const ExactPair *at = h_buf;
    for (uint32_t j = 0; j < EXACT_MAX_PARTS; j++) {
      if (counts[j]) ctx->spill_parts[j].emplace_back(at, at + counts[j]);
      at += counts[j];
    }
    moved += m;
  }
  // the budget holds what the parts hold; pairs still in the table after a failure stay there, and a set union does not
  // mind holding a pair twice
  ctx->spilled_pairs += moved;
  g_spill_bytes -= (n - std::min(n, moved)) * sizeof(ExactPair);
  if (rc) return rc;
  if (moved != n) return fail(ctx, KUQ_E_CAPACITY, "internal: the spill moved %llu of %llu pairs", (unsigned long long)moved, (unsigned long long)n);
  ctx->snap_valid = false;
  return clear_table(ctx, t);
}

// Room for a batch's pairs (one per window).  A table that cannot grow spills when kuq_set_exact_spill allows it and
// then takes the batch at its capacity.
int reserve_batch_pairs(kuq_ctx *ctx, uint64_t windows) {
  int rc = reserve_exact_inserts(ctx, windows);
  if (rc != KUQ_E_NOMEM || !ctx->spill_budget) return rc;
  rc = spill_exact(ctx);
  if (rc) return rc;
  ctx->spills++;
  rc = make_room(ctx, ctx->exact, 0, windows);
  if (rc)
    return fail(ctx, KUQ_E_NOMEM, "exact k-mer set: an empty table of %llu slots cannot take a batch of up to %llu pairs, which needs "
                                  "%llu slots: smaller batches, or more device memory",
                (unsigned long long)ctx->exact.cap, (unsigned long long)windows,
                (unsigned long long)slots_for(windows, ctx->exact.cap, 6));
  return KUQ_OK;
}

// kuq_set_extract's slot buffer: one selection byte per read, then the batch's count of selected reads (u32)
uint64_t extract_count_at(const kuq_ctx *ctx) { return (ctx->cfg.max_reads_per_batch + 15ull) & ~15ull; }

// krakenuniq-filter's parent map in filter ids: a taxon's dense id, or for taxa of F without one (parents without a
// taxonomy row, taxa the taxonomy does not have) n_taxa + their index in d_fextra.
int upload_filter(kuq_ctx *ctx) {
  std::unordered_map<uint32_t, uint32_t> extra;
  std::vector<uint32_t> extra_raw;
  auto id_of = [&](uint32_t t) {
    auto it = ctx->dense_of_raw.find(t);
    if (it != ctx->dense_of_raw.end()) return it->second;
    auto ins = extra.emplace(t, ctx->n_taxa + (uint32_t)extra_raw.size());
    if (ins.second) extra_raw.push_back(t);
    return ins.first->second;
  };
  for (auto &kv : ctx->f_parent) { id_of(kv.first); id_of(kv.second); }
  const uint64_t n = (uint64_t)ctx->n_taxa + extra_raw.size();
  std::vector<uint32_t> parent(n, 0), depth(n, 0);
  for (auto &kv : ctx->f_parent) {
    const uint32_t i = id_of(kv.first);
    parent[i] = id_of(kv.second);
    depth[i] = ctx->f_depth[kv.first];
  }
  extra_raw.push_back(0);                             // never an empty allocation
  CU(ctx->d_fparent.alloc(n));
  CU(ctx->d_fdepth.alloc(n));
  CU(ctx->d_fextra.alloc(extra_raw.size()));
  CU(cudaMemcpy(ctx->d_fparent, parent.data(), n * 4, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(ctx->d_fdepth, depth.data(), n * 4, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(ctx->d_fextra, extra_raw.data(), extra_raw.size() * 4, cudaMemcpyHostToDevice));
  return KUQ_OK;
}

// Dense numbering: 0 = "no taxon", 1 = taxid 1 (the reference's hard-wired root, krakenutil.cpp:96,106), then every
// taxid stored in database records (these own HLL sketches), then the remaining taxonomy nodes; each group
// ascending by taxid.  Builds the flattened Parent_map and uploads everything.
int finalize(kuq_ctx *ctx) {
  if (ctx->finalized) return KUQ_OK;
  if (ctx->dbs.empty()) return fail(ctx, KUQ_E_STATE, "no database staged");
  if (!ctx->tax_set) return fail(ctx, KUQ_E_STATE, "no taxonomy set");
  std::vector<uint32_t> staged;
  for (auto &e : ctx->dbs) staged.insert(staged.end(), e.taxids.begin(), e.taxids.end());
  std::vector<uint32_t> dbt = ctx->universe.empty() ? staged : ctx->universe;
  std::sort(dbt.begin(), dbt.end());
  dbt.erase(std::unique(dbt.begin(), dbt.end()), dbt.end());
  std::vector<uint32_t> &raw = ctx->raw_of_dense;
  raw.clear();
  ctx->dense_of_raw.clear();
  raw.push_back(0);
  raw.push_back(1);
  for (uint32_t t : dbt) if (t > 1) raw.push_back(t);
  ctx->n_sketch = (uint32_t)raw.size();
  for (uint32_t i = 0; i < raw.size(); i++) ctx->dense_of_raw[raw[i]] = i;
  std::vector<uint32_t> rest;
  for (uint32_t t : ctx->tax_ids) if (!ctx->dense_of_raw.count(t)) rest.push_back(t);
  for (uint32_t t : ctx->tax_parents) if (t && !ctx->dense_of_raw.count(t)) rest.push_back(t);   // parents without a row
  std::sort(rest.begin(), rest.end());
  rest.erase(std::unique(rest.begin(), rest.end()), rest.end());
  for (uint32_t t : rest) { ctx->dense_of_raw[t] = (uint32_t)raw.size(); raw.push_back(t); }
  ctx->n_taxa = (uint32_t)raw.size();
  // staged taxids must all be numbered
  for (uint32_t t : staged)
    if (!ctx->dense_of_raw.count(t) || ctx->dense_of_raw[t] >= ctx->n_sketch)
      return fail(ctx, KUQ_E_STATE, "staged records hold taxid %u that is not in the declared taxid universe", t);

  // Parent_map (taxdb.hpp:383-398): every taxonomy row has an entry; rows whose parent is themselves / 0 map to
  // 0.  A parent id WITHOUT a row of its own is still walked to by resolve_tree/lca (then the walk stops:
  // "No parent for ..." krakenutil.cpp:166-169), so such ids got a dense id above with parent 0.
  std::vector<uint32_t> parent(ctx->n_taxa, 0);
  for (size_t i = 0; i < ctx->tax_ids.size(); i++) {
    uint32_t t = ctx->tax_ids[i], p = ctx->tax_parents[i];
    if (t == 0) continue;
    parent[ctx->dense_of_raw[t]] = (p == t || p == 0) ? 0 : ctx->dense_of_raw[p];
  }
  // depth = steps until the chain ends at 0 or at dense 1 (lca() stops at taxid 1, krakenutil.cpp:96,106)
  std::vector<uint16_t> depth(ctx->n_taxa, 0);
  std::vector<uint8_t> state(ctx->n_taxa, 0);   // 0 new, 1 on stack, 2 done
  state[0] = state[1] = 2;
  std::vector<uint32_t> stack;
  for (uint32_t i = 2; i < ctx->n_taxa; i++) {
    if (state[i]) continue;
    uint32_t x = i;
    stack.clear();
    while (state[x] == 0) { state[x] = 1; stack.push_back(x); x = parent[x]; }
    if (state[x] == 1) return fail(ctx, KUQ_E_TAXONOMY, "cycle in the taxonomy at taxid %u", raw[x]);
    uint32_t d = depth[x];
    while (!stack.empty()) {
      uint32_t y = stack.back(); stack.pop_back();
      d++;
      if (d > 65000) return fail(ctx, KUQ_E_TAXONOMY, "taxonomy deeper than 65000 levels");
      depth[y] = (uint16_t)d; state[y] = 2;
    }
  }
  ctx->parent_dense = parent;
  CU(ctx->d_parent.alloc(ctx->n_taxa));
  CU(ctx->d_raw.alloc(ctx->n_taxa));
  CU(ctx->d_depth.alloc(ctx->n_taxa));
  CU(cudaMemcpy(ctx->d_parent, parent.data(), ctx->n_taxa * 4ull, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(ctx->d_raw, raw.data(), ctx->n_taxa * 4ull, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(ctx->d_depth, depth.data(), ctx->n_taxa * 2ull, cudaMemcpyHostToDevice));
  CU(ctx->d_regs.alloc((uint64_t)ctx->n_sketch * HLL_M));
  CU(ctx->d_dense_flag.alloc(ctx->n_sketch));
  CU(ctx->d_reg_floor.alloc(ctx->n_sketch));
  CU(ctx->d_n_kmers.alloc(ctx->n_sketch));
  CU(ctx->d_n_reads.alloc(ctx->n_taxa));
  CU(cudaMemset(ctx->d_regs, 0, (uint64_t)ctx->n_sketch * HLL_M));
  CU(cudaMemset(ctx->d_dense_flag, 0, ctx->n_sketch));
  CU(cudaMemset(ctx->d_reg_floor, 0, ctx->n_sketch));
  CU(cudaMemset(ctx->d_n_kmers, 0, ctx->n_sketch * 8ull));
  CU(cudaMemset(ctx->d_n_reads, 0, ctx->n_taxa * 8ull));
  if (ctx->cfg.hll_mode == KUQ_HLL_EXACT) {
    ctx->exact.cap = ctx->cfg.sparse_set_slots;            // entries of 16 B; grows before batches that could fill it
    CU(ctx->exact.slots.alloc(ctx->exact.cap));
    CU(ctx->exact.count.alloc(ctx->n_sketch));
    int rc = clear_table(ctx, ctx->exact);
    if (rc) return rc;
  } else if (ctx->cfg.hll_mode != KUQ_HLL_DENSE_ONLY) {
    ctx->sparse.cap = ctx->cfg.sparse_set_slots;
    CU(ctx->sparse.slots.alloc(ctx->sparse.cap));
    CU(ctx->d_sparse_used.alloc(1));
    CU(ctx->sparse.count.alloc(ctx->n_sketch));
    CU(cudaMemset(ctx->d_sparse_used, 0, 8));
    int rc = clear_table(ctx, ctx->sparse);
    if (rc) return rc;
  }
  ctx->finalized = true;
  return ctx->filter_set ? upload_filter(ctx) : KUQ_OK;
}

// rewrite the record values of each staged range taxid → dense id, once per range
int remap_values(kuq_ctx *ctx, StagedDb &db) {
  const uint32_t tx_cap = db.tx_cap;
  std::vector<uint32_t> keys(tx_cap), dense(tx_cap, 0);
  CU(cudaMemcpy(keys.data(), db.d_tx_keys, tx_cap * 4ull, cudaMemcpyDeviceToHost));
  for (uint32_t i = 0; i < tx_cap; i++)
    if (keys[i]) {
      auto it = ctx->dense_of_raw.find(keys[i] - 1);
      if (it == ctx->dense_of_raw.end() || it->second >= ctx->n_sketch)
        return fail(ctx, KUQ_E_STATE, "staged records hold taxid %u outside the numbered universe", keys[i] - 1);
      dense[i] = it->second;
    }
  CU(cudaMemcpy(db.d_tx_dense, dense.data(), tx_cap * 4ull, cudaMemcpyHostToDevice));
  DevBuf<uint32_t> d_missing;
  CU(d_missing.alloc(1));
  CU(cudaMemset(d_missing, 0, 4));
  launch_remap_values(db.range.pairs, db.range.key_ct, db.d_tx_keys, db.d_tx_dense, tx_cap - 1, d_missing, kmer_mask(ctx->k), ctx->aux);
  ctx->launches++;
  uint32_t missing = 0;
  CU(cudaMemcpyAsync(&missing, d_missing, 4, cudaMemcpyDeviceToHost, ctx->aux));
  CU(cudaStreamSynchronize(ctx->aux));
  if (missing) return fail(ctx, KUQ_E_STATE, "internal: a record value was missing from the taxid table");
  return KUQ_OK;
}
int remap_db(kuq_ctx *ctx) {
  for (auto &e : ctx->dbs) {
    if (e.remapped) continue;
    int rc = remap_values(ctx, e);
    if (rc) return rc;
    e.remapped = true;
  }
  return KUQ_OK;
}

// Preorder of the context's taxonomy (roots: taxa whose parent is 0, as in kuq_clade_counts_tree), kept for the sketch
// taxa on host and device.  Taxa no root reaches (a malformed chain) stay NONE and are left out of the roll-up.
int exact_preorder(kuq_ctx *ctx) {
  if (ctx->d_exact_pre) return KUQ_OK;
  const uint32_t NT = ctx->n_taxa, NONE = 0xFFFFFFFFu;
  const std::vector<uint32_t> &par = ctx->parent_dense;
  std::vector<uint32_t> first(NT + 1, 0), child(NT), pre(NT, NONE), stack;
  for (uint32_t x = 1; x < NT; x++) if (par[x]) first[par[x] + 1]++;
  for (uint32_t x = 0; x < NT; x++) first[x + 1] += first[x];
  {
    std::vector<uint32_t> fill(first.begin(), first.end() - 1);
    for (uint32_t x = 1; x < NT; x++) if (par[x]) child[fill[par[x]]++] = x;
  }
  uint32_t counter = 0;
  for (uint32_t r = 0; r < NT; r++) {
    if (r != 0 && par[r] != 0) continue;
    stack.push_back(r);
    while (!stack.empty()) {
      const uint32_t x = stack.back();
      stack.pop_back();
      if (pre[x] != NONE) continue;
      pre[x] = counter++;
      if (x == 0) continue;                      // dense 0 ("no taxon") is a root of its own
      for (uint32_t i = first[x]; i < first[x + 1]; i++) stack.push_back(child[i]);
    }
  }
  pre.resize(ctx->n_sketch);
  CU(ctx->d_exact_pre.alloc(ctx->n_sketch));
  CU(cudaMemcpy(ctx->d_exact_pre, pre.data(), ctx->n_sketch * 4ull, cudaMemcpyHostToDevice));
  ctx->exact_pre.swap(pre);
  return KUQ_OK;
}

// Books of the exact roll-up, one signed counter per taxon of the taxonomy: books[d] = pairs of taxon d − the adjacent
// equal-k-mer pairs (sorted by (k-mer, preorder)) whose LCA is d.  Summed over a subtree they give its distinct k-mers;
// summed over contexts that hold disjoint parts of the k-mer space they give the books of the union.  The +1 per pair
// comes from count[] instead of one atomic per pair on the device (most pairs of a run go to a few taxa: the misses to
// taxon 0).  Scratch: KUQ_EXACT_ROLLUP_BUDGET bytes, else 80 % of the free device memory.  All slots idle.
int exact_books(kuq_ctx *ctx, std::vector<long long> &books) {
  int rc = exact_preorder(ctx);
  if (rc) return rc;
  std::vector<unsigned long long> count;
  uint64_t n_pairs = 0;
  rc = table_counts(ctx, ctx->exact, count, &n_pairs);
  if (rc) return rc;
  DevBuf<unsigned long long> d_books;
  CU(d_books.alloc(ctx->n_taxa));
  CU(cudaMemsetAsync(d_books, 0, ctx->n_taxa * 8ull, ctx->aux));
  uint64_t budget = 0;
  if (const char *e = getenv("KUQ_EXACT_ROLLUP_BUDGET")) budget = strtoull(e, nullptr, 10);
  if (!budget) {
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    budget = (uint64_t)(free_b * 0.8);
  }
  const int src = exact_clade_dups(ctx->exact.slots, ctx->exact.cap, n_pairs, ctx->d_exact_pre, ctx->d_parent, ctx->d_depth, d_books,
                                   std::max<uint64_t>(budget, 1), ctx->n_sm, ctx->aux, &ctx->exact_rollup_passes);
  ctx->launches += 3ull * std::max<uint32_t>(ctx->exact_rollup_passes, 1);
  std::vector<unsigned long long> dups(ctx->n_taxa, 0);
  cudaError_t ce = cudaSuccess;
  if (src == 0) ce = cudaMemcpy(dups.data(), d_books, ctx->n_taxa * 8ull, cudaMemcpyDeviceToHost);
  d_books.reset();
  if (src == 1) return fail(ctx, KUQ_E_NOMEM, "exact clade roll-up: no device memory for one pass of the sort (budget %llu bytes)", (unsigned long long)budget);
  if (src == 2 || ce != cudaSuccess) return fail(ctx, KUQ_E_CUDA, "exact clade roll-up failed: %s", cudaGetErrorString(cudaGetLastError()));
  books.assign(ctx->n_taxa, 0);
  for (uint32_t d = 0; d < ctx->n_taxa; d++) books[d] = (long long)dups[d];
  for (uint32_t d = 0; d < ctx->n_sketch; d++)
    if (ctx->exact_pre[d] != 0xFFFFFFFFu) books[d] += (long long)count[d];
  return KUQ_OK;
}

// Build the collision table of the staged range once, the first time keep mode or a harvest can use the record tier.
int ensure_collisions(kuq_ctx *ctx) {
  if (ctx->collisions) return KUQ_OK;
  ctx->collisions = -1;
  if (ctx->stream_open || ctx->lca_mode || ctx->dbs.empty() || !ctx->dbs[0].remapped) return KUQ_OK;
  const StagedDb &db = ctx->dbs[0];
  std::vector<uint64_t> per_taxon(ctx->n_sketch, 0);
  for (size_t i = 0; i < db.taxids.size(); i++) per_taxon[ctx->dense_of_raw[db.taxids[i]]] += db.counts[i];
  const auto t0 = std::chrono::steady_clock::now();
  // a table above 1/32 of the records (a taxon far above 2^25 records) is not worth it: the set path stays
  const int rc = build_collisions(db.range.pairs, db.range.key_ct, kmer_mask(ctx->k), per_taxon.data(), ctx->n_sketch,
                                  db.range.key_ct / 32 + 1024, ctx->d_secondaries, &ctx->n_secondaries, ctx->n_sm, ctx->aux);
  ctx->launches += 3;
  ctx->collisions_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  if (rc == 2) return fail(ctx, KUQ_E_CUDA, "building the collision table of the record tier failed: %s", cudaGetErrorString(cudaGetLastError()));
  if (rc == 0) ctx->collisions = 1;
  if (getenv("KUQ_TIMING"))
    fprintf(stderr, "[timing] collision table: %llu secondaries of %llu records, %.1f ms%s\n", (unsigned long long)ctx->n_secondaries,
            (unsigned long long)db.range.key_ct, ctx->collisions_ms, rc ? " (not built: harvests fill the set)" : "");
  return KUQ_OK;
}

int harvest_state(kuq_ctx *ctx) {
  if (ctx->d_harvest_stat) return KUQ_OK;
  CU(ctx->d_harvest_stat.alloc(3));
  CU(cudaMemset(ctx->d_harvest_stat, 0, 3 * 8));
  CU(ctx->harvest_ev[0].alloc(cudaEventDefault)); CU(ctx->harvest_ev[1].alloc(cudaEventDefault));
  return KUQ_OK;
}

// Params::reg_floor for a counting launch about to run on `stream`: every sketch's smallest register, so that windows
// whose hash rank cannot raise a register skip the register load (hll_update).  Registers only grow while kernels
// run, so a floor taken before the launch stays a lower bound through it, whichever slot refreshed it last; between
// launches they may be cleared (kuq_reset_counts) or rewritten through kuq_state_ptrs_get, hence a refresh per launch.
// The pass reads every register: when that is more bytes than the launch's bases the floor is 0 instead (no skip).
int refresh_reg_floor(kuq_ctx *ctx, uint64_t total_bases, cudaStream_t stream) {
  if (!ctx->d_reg_floor) return KUQ_OK;
  if ((uint64_t)ctx->n_sketch * HLL_M <= total_bases) {
    launch_reg_floor(ctx->d_regs, ctx->n_sketch, ctx->d_reg_floor, stream);
    ctx->launches++;
  } else {
    CU(cudaMemsetAsync(ctx->d_reg_floor, 0, ctx->n_sketch, stream));
  }
  CU(cudaGetLastError());
  return KUQ_OK;
}

// Keep mode (F_KEEP): a fused call whose counted hits would become kept records at the next harvest anyway (preload
// rule, a resident range with its collision table, a set without keys of hits, no flags pending) keeps them in the
// lookup, and the harvest shrinks to settle_kept.  KUQ_KEEP_AT_HARVEST=1 keeps the flag-and-harvest path instead (A/B
// runs and tests compare both in one build).
int use_keep_mode(kuq_ctx *ctx, int mode, const Params &p, bool *keep) {
  *keep = false;
  if (mode != MODE_FUSED || !p.n_reads || (p.flags & 4u) || ctx->cfg.hll_mode != KUQ_HLL_PRELOAD || !ctx->sparse.slots ||
      ctx->set_has_hits || ctx->stream_open || ctx->seen_dirty || (ctx->quick_min && ctx->quick_stop))
    return KUQ_OK;
  const char *env = getenv("KUQ_KEEP_AT_HARVEST");
  if (env && *env && strcmp(env, "0") != 0) return KUQ_OK;
  int rc = ensure_collisions(ctx);
  if (rc) return rc;
  if (ctx->collisions != 1) return KUQ_OK;
  rc = harvest_state(ctx);
  if (rc) return rc;
  *keep = true;
  return KUQ_OK;
}

// After keep-mode calls: kept secondaries hand KEPT_BIT to their primaries (k_settle_kept takes the duplicates back out of
// distinct[]) and the records those calls kept join kept_keys — the state the flag-and-harvest path leaves.  All slots
// must be idle.
int settle_kept(kuq_ctx *ctx) {
  ctx->keep_dirty = false;
  unsigned long long *d_stat = ctx->d_harvest_stat;
  CU(cudaMemsetAsync(d_stat, 0, 8, ctx->aux));
  CU(cudaEventRecord(ctx->harvest_ev[0], ctx->aux));
  launch_settle_kept(first_range(ctx).pairs, ctx->d_secondaries, ctx->n_secondaries, ctx->sparse.count, d_stat, ctx->aux);
  if (ctx->n_secondaries) ctx->launches++;
  CU(cudaEventRecord(ctx->harvest_ev[1], ctx->aux));
  unsigned long long st[3] = {0, 0, 0};
  CU(cudaMemcpyAsync(st, d_stat, 24, cudaMemcpyDeviceToHost, ctx->aux));
  CU(cudaMemsetAsync(d_stat + 2, 0, 8, ctx->aux));
  CU(cudaStreamSynchronize(ctx->aux));
  float ms = 0;
  cudaEventElapsedTime(&ms, ctx->harvest_ev[0], ctx->harvest_ev[1]);
  ctx->harvest_ms = ms;
  ctx->kept_keys += st[2] - st[0];
  ctx->snap_valid = false;
  if (getenv("KUQ_TIMING"))
    fprintf(stderr, "[timing] settle: %llu records kept at sighting, %llu of them duplicates (%llu kept), %.3f ms\n", st[2], st[0],
            (unsigned long long)ctx->kept_keys, ms);
  return KUQ_OK;
}

// The keys of the kept records move into the set (mode 3), which is the only store from here on: the records are about
// to leave HBM, or the set is about to receive keys of hits that kept records could duplicate.  All slots must be idle.
int spill_kept(kuq_ctx *ctx) {
  if (!ctx->kept) return KUQ_OK;
  uint64_t used = 0;
  int rc = table_items(ctx, ctx->sparse, &used);
  if (!rc) rc = make_room(ctx, ctx->sparse, used, 0);
  if (rc) return rc;
  const DbRange &r = first_range(ctx);
  rc = run_saturating(
      ctx, [&](uint32_t *err) { launch_harvest_seen(r.pairs, r.key_ct, kmer_mask(ctx->k), ctx->d_dense_flag, set_view(ctx, ctx->sparse), nullptr, err, 3, ctx->aux); },
      "sparse-tier set saturated while taking over the kept records (%llu slots)", (unsigned long long)ctx->sparse.cap);
  ctx->kept = false;
  ctx->kept_keys = 0;
  ctx->set_has_hits = true;
  ctx->snap_valid = false;
  return rc;
}

// Sparse HLL tier of the hits: the fused lookup only flags the records it counted (SEEN_BIT); here the flags of the
// staged range become (taxon, encoded hash) keys — the union the reference builds with `taxon_counts[t] += ...` over
// sparse sketches (hyperloglogplus.cpp:600-603) — and are cleared.  Two stores:
//  * record tier (a resident range whose set holds no keys of hits): the key is a function of the record and the
//    database does not change while it is resident, so the primary record of the key's (taxon, code) group is marked
//    KEPT_BIT and the taxon's distinct count grows by one — one streaming pass, no hash-set insert;
//  * the set (ranges that leave HBM, `to_set`, and contexts whose set receives keys of hits from elsewhere): count →
//    grow the set if it would pass a load factor of 0.8 → insert.  The number of keys is known before they are
//    inserted, so the set grows here instead of failing mid-batch.
// `discard` drops every flag of both kinds instead (the keys were exported, or the counts are reset).
int harvest_seen(kuq_ctx *ctx, bool discard, bool to_set) {
  if (!ctx->seen_dirty && !ctx->keep_dirty && !(ctx->kept && (discard || to_set))) return KUQ_OK;
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  double settle_ms = 0;
  if (discard && ctx->keep_dirty) {              // the flags are dropped below (kept is set): settle_kept would be wasted,
    ctx->keep_dirty = false;                     // only its counter of records kept since then starts over
    CU(cudaMemsetAsync(ctx->d_harvest_stat + 2, 0, 8, ctx->aux));
  }
  if (ctx->keep_dirty) {
    int rc = settle_kept(ctx);
    if (rc) return rc;
    settle_ms = ctx->harvest_ms;
  }
  if (to_set && !discard) { int rc = spill_kept(ctx); if (rc) return rc; }
  if (!ctx->seen_dirty && !(ctx->kept && discard)) return KUQ_OK;
  ctx->seen_dirty = false;
  const DbRange &r = first_range(ctx);
  if (!r.pairs || !r.key_ct) return KUQ_OK;
  bool keep = !discard && !to_set && ctx->sparse.slots && !ctx->set_has_hits && !ctx->stream_open;
  if (keep) {
    int rc = ensure_collisions(ctx);
    if (rc) return rc;
    keep = ctx->collisions == 1;
  }
  const uint64_t key_mask = kmer_mask(ctx->k);
  SparseSet ss = set_view(ctx, ctx->sparse);
  { int rc = harvest_state(ctx); if (rc) return rc; }
  unsigned long long *d_stat = ctx->d_harvest_stat;
  cudaEvent_t e0 = ctx->harvest_ev[0], e1 = ctx->harvest_ev[1];
  CU(cudaMemsetAsync(d_stat, 0, 16, ctx->aux));
  CU(cudaEventRecord(e0, ctx->aux));
  if (discard || !ctx->sparse.slots) {
    launch_harvest_seen(r.pairs, r.key_ct, key_mask, ctx->d_dense_flag, ss, d_stat, reinterpret_cast<uint32_t *>(d_stat + 1), 2, ctx->aux);
    ctx->launches++;
    ctx->kept = false;
    ctx->kept_keys = 0;
  } else if (keep) {
    launch_harvest_keep(r.pairs, r.key_ct, ctx->d_secondaries, ctx->n_secondaries, ctx->d_dense_flag, ctx->n_sketch,
                        ctx->sparse.count, d_stat, ctx->aux);
    ctx->launches += ctx->n_secondaries ? 2 : 1;
    ctx->kept = true;
  } else {
    launch_harvest_seen(r.pairs, r.key_ct, key_mask, ctx->d_dense_flag, ss, d_stat, reinterpret_cast<uint32_t *>(d_stat + 1), 0, ctx->aux);
    ctx->launches++;
    unsigned long long n_new = 0;
    uint64_t used = 0;
    CU(cudaMemcpyAsync(&n_new, d_stat, 8, cudaMemcpyDeviceToHost, ctx->aux));
    CU(cudaStreamSynchronize(ctx->aux));
    int grc = table_items(ctx, ctx->sparse, &used);
    if (!grc) grc = make_room(ctx, ctx->sparse, used, n_new);
    if (grc) return grc;
    ss = set_view(ctx, ctx->sparse);
    if (n_new) ctx->set_has_hits = true;
    // Insert in record order.  (Round 2 also tried staging the keys by table slice so that the inserts of a slice are
    // L2-resident: read-only probes got faster, but NEW keys did not (each one still costs a DRAM sector fetch and a
    // dirty sector write-back), and new keys are what a harvest mostly sees.)
    launch_harvest_seen(r.pairs, r.key_ct, key_mask, ctx->d_dense_flag, ss, d_stat, reinterpret_cast<uint32_t *>(d_stat + 1), 1, ctx->aux);
    ctx->launches++;
    CU(cudaStreamSynchronize(ctx->aux));
    if (getenv("KUQ_TIMING")) fprintf(stderr, "[timing] harvest: %llu flagged records, %llu slots\n", n_new, (unsigned long long)ctx->sparse.cap);
  }
  CU(cudaEventRecord(e1, ctx->aux));
  unsigned long long st[2] = {0, 0};
  CU(cudaMemcpyAsync(st, d_stat, 16, cudaMemcpyDeviceToHost, ctx->aux));
  CU(cudaStreamSynchronize(ctx->aux));
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  ctx->harvest_ms = settle_ms + ms;
  ctx->snap_valid = false;
  if (keep) {
    ctx->kept_keys += st[0];
    if (getenv("KUQ_TIMING")) fprintf(stderr, "[timing] harvest: %llu records became kept (%llu kept), %.2f ms\n", st[0], (unsigned long long)ctx->kept_keys, ms);
    return KUQ_OK;
  }
  if ((uint32_t)st[1]) return fail(ctx, KUQ_E_CAPACITY, "sparse-tier set saturated during the harvest (%llu slots)", (unsigned long long)ctx->sparse.cap);
  return KUQ_OK;
}

KeySource set_keys(const kuq_ctx *ctx) {
  KeySource k{ctx->sparse.slots, nullptr, ctx->sparse.slots ? ctx->sparse.cap : 0, 0};
  return k;
}
KeySource kept_keys(const kuq_ctx *ctx) {
  const DbRange &r = first_range(ctx);
  KeySource k{nullptr, r.pairs, ctx->kept ? r.key_ct : 0, (uint32_t)(kmer_mask(ctx->k) >> 32)};
  return k;
}

int ensure_ready(kuq_ctx *ctx) {
  int rc = finalize(ctx);
  if (rc) return rc;
  return remap_db(ctx);
}

// dense (unit, taxon) table: the units a batch can hold when the library cuts them, at most 64 Mi counters
uint64_t unit_table_rows(const kuq_ctx *ctx) {
  const uint64_t rows = ctx->cfg.max_bases_per_batch / std::max<uint64_t>(ctx->cfg.work_unit_size, 1) + 8;
  return std::min<uint64_t>(rows, (64ull << 20) / std::max<uint32_t>(ctx->n_sketch, 1));
}

void set_unit_ptrs(Params &p, Slot &s);
int prepare_unit_map(kuq_ctx *ctx, Slot &s) {
  if (ctx->cfg.hll_mode != KUQ_HLL_PRELOAD) return KUQ_OK;
  if (!s.u_keys) {
    CU(s.u_keys.alloc(UMAP_CAP));
    CU(s.u_inserts.alloc(UMAP_CAP));
    CU(s.u_cand.alloc(UMAP_CAP));             // every candidate is a distinct map slot
    CU(s.u_ncand.alloc(2));
    CU(s.u_codes.alloc((size_t)ctx->n_sm * UNIT_DECIDE_CTAS_PER_SM * 2 * UNIT_CODES));
    const uint64_t rows = unit_table_rows(ctx);
    s.u_direct_rows = (uint32_t)rows;
    if (rows) CU(s.u_direct.alloc(rows * ctx->n_sketch));
  }
  Params tmp;
  set_unit_ptrs(tmp, s);
  launch_unit_clear(tmp.units, ctx->n_sketch, ctx->n_sm, s.stream);
  ctx->launches++;
  return KUQ_OK;
}

// process_file's unit cutting (kuq_batches.h): reads join the open unit until its length reaches -u.
void cut_units(kuq_ctx *ctx, const uint64_t *offsets, uint32_t n, uint32_t *unit) {
  for (uint32_t i = 0; i < n; i++) {
    unit[i] = ctx->units.id;
    ctx->units.add(offsets[i + 1] - offsets[i], ctx->cfg.work_unit_size);
  }
}

void set_unit_ptrs(Params &p, Slot &s) {
  p.units.keys = s.u_keys;
  p.units.inserts = s.u_inserts;
  p.units.cand = s.u_cand;
  p.units.mask = UMAP_CAP - 1;
  p.units.n_cand = s.u_ncand;
  p.units.codes = s.u_codes;
  p.units.direct = s.u_direct;
  p.units.direct_rows = s.u_direct_rows;
}

DbView db_view(const kuq_ctx *ctx, const DbRange &r) {
  DbView v;
  v.pairs = r.pairs;
  v.offsets = r.offsets;
  v.rec_base = r.rec_base;
  v.key_mask = kmer_mask(ctx->k);
  v.bin_lo = (uint32_t)r.bin_lo;
  v.bin_hi = (uint32_t)r.bin_hi;
  v.k = ctx->k;
  v.nt = r.nt;
  v.xor_mask = (uint32_t)((r.idx_type == 1 ? 0ull : INDEX2_XOR_MASK) & ((1ull << (2 * r.nt)) - 1));
  v.n_mini = ctx->k - r.nt + 1;
  return v;
}

void fill_params(kuq_ctx *ctx, Slot &s, Params &p, const char *d_bases, const uint64_t *d_offsets,
                 const uint32_t *d_unit, uint32_t n_reads, uint32_t flags) {
  memset(&p, 0, sizeof p);
  p.db = db_view(ctx, first_range(ctx));
  p.tax.parent = ctx->d_parent;
  p.tax.depth = ctx->d_depth;
  p.tax.raw = ctx->d_raw;
  p.tax.n_taxa = ctx->n_taxa;
  p.tax.n_sketch = ctx->n_sketch;
  p.bases = d_bases;
  p.offsets = d_offsets;
  p.unit_id = d_unit;
  p.clean = s.d_clean;
  p.n_reads = n_reads;
  p.n_chunks = (n_reads + CHUNK_READS - 1) / CHUNK_READS;
  p.flags = flags & ~F_KEEP;                 // launch_on_slot decides keep mode
  p.hll_mode = ctx->cfg.hll_mode;
  p.call = s.d_call;
  p.n_windows = s.d_nwin;
  p.codes = s.d_codes;
  p.total_bases = s.total_bases;
  p.canon = s.d_canon;
  p.bins = s.d_bins;
  p.pack.blocks = s.d_pack;
  p.pack.side = s.d_side;
  p.codes_dense = s.d_dense;
  p.run_start = s.d_run_start;
  p.run_count = s.d_run_count;
  p.runs = s.d_runs;
  p.run_cursor = s.d_scalars;
  p.runs_capacity = s.runs_cap;
  p.n_classified = s.d_scalars + 1;
  p.chunk_counter = reinterpret_cast<uint32_t *>(s.d_scalars + 2);
  p.error_flag = reinterpret_cast<uint32_t *>(s.d_scalars + 3);
  p.stats = s.d_scalars + 4;
  p.ovf_mem = s.d_ovf;
  p.ovf_cursor = s.d_scalars + 6;
  p.ovf_capacity = s.ovf_entries;
  p.regs = ctx->d_regs;
  p.n_kmers = ctx->d_n_kmers;
  p.n_reads_ctr = ctx->d_n_reads;
  p.dense_flag = ctx->d_dense_flag;
  p.reg_floor = ctx->d_reg_floor;
  p.sparse = set_view(ctx, ctx->sparse);
  p.exact = set_view(ctx, ctx->exact);
  set_unit_ptrs(p, s);
  if (ctx->filter_set) {
    p.fparent = ctx->d_fparent;
    p.fdepth = ctx->d_fdepth;
    p.fextra = ctx->d_fextra;
    p.fmin = ctx->threshold - 1e-5;                  // krakenuniq-filter:126, in double like the script
    p.fcall = s.d_fcall;
    p.fhits = s.d_fhits;
    p.ftotal = s.d_ftotal;
  }
}

// The staged databases in the order they are asked, each with its own minimizer range.  A run = consecutive databases
// with the same window parameters (nt, index type).
std::vector<DbView> db_views(const kuq_ctx *ctx) {
  std::vector<DbView> v;
  for (auto &e : ctx->dbs) v.push_back(db_view(ctx, e.range));
  return v;
}
bool same_run(const DbView &a, const DbView &b) { return a.nt == b.nt && a.xor_mask == b.xor_mask; }
uint32_t count_runs(const kuq_ctx *ctx) {
  const std::vector<DbView> v = db_views(ctx);
  uint32_t n = 1;
  for (size_t i = 1; i < v.size(); i++) n += !same_run(v[i], v[i - 1]);
  return n;
}

// The in-order lookup over every staged database (kuq_stage_db_append_range) into p0.codes_dense: one launch per run of
// consecutive databases with the same (nt, index type), at most MAX_DBS per launch; runs after the first fill only the
// windows no earlier run answered, and k_scan runs again where the window parameters change.  run >= 0: only that run,
// its first launch with `only_hits` and a k_scan of its own (kuq_lookup_device_peers_run, one run per call).
int launch_multi_lookup(kuq_ctx *ctx, Slot &s, const Params &p0, uint32_t only_hits, int run = -1) {
  const std::vector<DbView> v = db_views(ctx);
  const DbView *scanned = nullptr;
  int r = -1;
  for (size_t i = 0; i < v.size();) {
    if (i == 0 || !same_run(v[i], v[i - 1])) r++;
    Params q = p0;
    q.db = v[i];
    q.n_dbs = 0;
    while (i < v.size() && q.n_dbs < MAX_DBS && same_run(v[i], q.db)) q.dbs[q.n_dbs++] = v[i++];
    if (run >= 0 && r != run) continue;
    q.run_lo = q.run_hi = 0;                           // the bins this launch's databases hold (empty slices aside)
    for (uint32_t d = 0; d < q.n_dbs; d++) {
      if (q.dbs[d].bin_lo >= q.dbs[d].bin_hi) continue;
      if (q.run_lo >= q.run_hi) { q.run_lo = q.dbs[d].bin_lo; q.run_hi = q.dbs[d].bin_hi; continue; }
      q.run_lo = std::min(q.run_lo, q.dbs[d].bin_lo);
      q.run_hi = std::max(q.run_hi, q.dbs[d].bin_hi);
    }
    q.only_hits = scanned ? KUQ_LOOKUP_FILL_EMPTY : only_hits;
    const bool scan = !scanned || scanned->nt != q.db.nt || scanned->xor_mask != q.db.xor_mask;
    if (scan) CU(cudaMemsetAsync(q.chunk_counter, 0, 4, s.stream));
    ctx->launches += launch_lookup_multi(q, ctx->n_sm, s.stream, scan);
    scanned = &v[i - 1];
  }
  return KUQ_OK;
}

// run >= 0: one run of the in-order lookup with peer scatter (kuq_lookup_device_peers_run)
int launch_on_slot(kuq_ctx *ctx, Slot &s, int mode, Params &p, int run = -1) {
  if (ctx->lca_mode) return fail(ctx, KUQ_E_STATE, "this context built a database (kuq_set_lcas_batch): stage it anew to classify");
  // several databases (or a fill-empty lookup): the in-order lookup, then — for a classification — the resolve half
  // over the slot's merged codes
  const bool multi = (ctx->dbs.size() > 1 && mode != MODE_RESOLVE) || (mode == MODE_LOOKUP && p.only_hits == KUQ_LOOKUP_FILL_EMPTY) ||
                     run >= 0;
  if (multi && ((p.n_peers && run < 0) || ctx->shard_counting))
    return fail(ctx, KUQ_E_STATE, "shard counting and kuq_lookup_device_peers take one database (several: kuq_lookup_device_peers_run)");
  uint32_t *multi_out = p.codes_dense;
  const uint32_t multi_only_hits = mode == MODE_LOOKUP ? p.only_hits : 0;
  if (multi && mode == MODE_FUSED) {
    // the merged codes live in the slot's output-code buffer: the resolve half reads them (codes_in) before k_resolve
    // writes its per-window taxids there
    multi_out = s.d_codes;
    p.codes_in = s.d_codes;
    mode = MODE_RESOLVE;
  }
  ctx->snap_valid = false;
  p.flags |= ctx->extra_flags;
  if (mode == MODE_LOOKUP && ctx->mark_zero_hits) p.flags |= 16u;
  if (ctx->shard_counting && mode != MODE_FUSED && !ctx->mark_zero_hits && !ctx->quick_min &&
      ctx->cfg.hll_mode != KUQ_HLL_EXACT) {
    p.flags |= 32u;
    if (mode == MODE_LOOKUP && p.n_reads && ctx->cfg.hll_mode <= KUQ_HLL_CHUNKED) ctx->seen_dirty = true;
  }
  ctx->merged_summary = false;
  ctx->merged_exact = false;
  if (mode != MODE_LOOKUP && ctx->quick_min) {           // "Q:hits" replaces the hit list (classify.cpp:989-990)
    p.quick_min = ctx->quick_min;
    p.quick_stop = ctx->quick_stop;
    p.flags |= KUQ_F_NO_RUNS;
    s.flags |= KUQ_F_NO_RUNS;
  }
  // the fused path's only direct inserts are misses (taxon 0): harvests of the record tier do not grow the set, so room
  // for them is made before the batch as well
  if ((mode == MODE_RESOLVE || mode == MODE_FUSED) && !(p.flags & 4u) && ctx->cfg.hll_mode <= KUQ_HLL_CHUNKED && p.n_reads) {
    if (mode == MODE_RESOLVE && !(p.flags & 32u) && !ctx->set_has_hits) {
      // the resolve half inserts the keys of hits into the set, which kept records could duplicate
      int hrc = harvest_seen(ctx, false, true);
      if (hrc) return hrc;
      ctx->set_has_hits = true;
    }
    int rrc = reserve_direct_inserts(ctx, s.total_bases);
    if (rrc) return rrc;
    p.sparse = set_view(ctx, ctx->sparse);             // the set may have moved
  }
  // exact counting: the batch's windows go into the (taxon, k-mer) table, which grows before the batch when they could
  // fill it, or spills to host memory when it cannot grow (kuq_set_exact_spill)
  if ((mode == MODE_RESOLVE || mode == MODE_FUSED) && !(p.flags & 4u) && ctx->cfg.hll_mode == KUQ_HLL_EXACT && p.n_reads) {
    int rrc = reserve_batch_pairs(ctx, s.total_bases);
    if (rrc) return rrc;
    p.exact = set_view(ctx, ctx->exact);
  }
  const bool units = mode != MODE_LOOKUP && ctx->cfg.hll_mode == KUQ_HLL_PRELOAD && p.unit_id && !(p.flags & 4u);
  if (units) {
    int rc = prepare_unit_map(ctx, s);
    if (rc) return rc;
    set_unit_ptrs(p, s);                 // the map is allocated on first use
  } else if (ctx->cfg.hll_mode == KUQ_HLL_PRELOAD) {
    p.unit_id = nullptr;                 // no per-unit bookkeeping for this call
  }
  bool keep = false;
  { int krc = use_keep_mode(ctx, mode, p, &keep); if (krc) return krc; }
  if (keep) {
    p.flags |= F_KEEP;
    p.n_new_kept = ctx->d_harvest_stat + 2;
    ctx->kept = true;
    ctx->keep_dirty = true;
  }
  p.packed = windows_packed(mode, p) ? 1u : 0u;
  if (p.n_reads) s.windows_packed = p.packed != 0;
  if (p.n_reads && !(p.flags & 4u)) {
    int frc = refresh_reg_floor(ctx, s.total_bases, s.stream);
    if (frc) return frc;
  }
  CU(cudaMemsetAsync(s.d_scalars, 0, 8 * 8, s.stream));
  CU(cudaEventRecord(s.ev_k0, s.stream));
  CU(cudaEventRecord(s.ev_stage[0], s.stream));
  CU(cudaEventRecord(s.ev_stage[1], s.stream));
  if (p.n_reads && multi) {
    Params q = p;
    q.codes_dense = multi_out;
    int mrc = launch_multi_lookup(ctx, s, q, multi_only_hits, run);
    if (mrc) return mrc;
    if (mode != MODE_LOOKUP) CU(cudaMemsetAsync(p.chunk_counter, 0, 4, s.stream));   // k_scan of the resolve half
  }
  if (p.n_reads && !(multi && mode == MODE_LOOKUP)) {
    cudaEvent_t stage[2] = {s.ev_stage[0], s.ev_stage[1]};
    ctx->launches += launch_classify(mode, p, ctx->n_sm, s.stream, stage);
  }
  if (p.n_reads && mode != MODE_LOOKUP && ctx->extract_set) {          // after whichever resolve wrote the calls
    CU(cudaMemsetAsync(s.d_xsel + extract_count_at(ctx), 0, 4, s.stream));
    launch_extract_select(p.call, p.fcall, p.n_reads, ctx->d_members, ctx->n_members, ctx->extract_flags, s.d_xsel,
                          reinterpret_cast<uint32_t *>(s.d_xsel + extract_count_at(ctx)), s.stream);
    ctx->launches++;
  }
  // the fused path flags the records of its counted hits (k_lookup); quick / exact runs go through the other halves
  if (p.n_reads && mode == MODE_FUSED && !(p.flags & 4u) && ctx->cfg.hll_mode <= KUQ_HLL_CHUNKED &&
      !(ctx->quick_min && ctx->quick_stop) && !keep)
    ctx->seen_dirty = true;
  CU(cudaEventRecord(s.ev_k1, s.stream));
  s.timed = true;
  // HLL mode rule: which taxa have a sketch that converted to dense (SURVEY.md App. C)
  if (p.n_reads && mode != MODE_LOOKUP && !(p.flags & 4u)) {
    if (units) ctx->launches += launch_unit_accounting(p, ctx->n_sm, s.stream);
    else if (ctx->cfg.hll_mode == KUQ_HLL_CHUNKED) {
      launch_flag_dense_global(ctx->sparse.count, ctx->d_dense_flag, ctx->n_sketch, s.stream);
      ctx->launches++;
    }
  }
  CU(cudaGetLastError());
  return KUQ_OK;
}

}  // namespace

// ===========================================================================================================
extern "C" {

const char *kuq_version(void) { return "libkuq 0.2.0 sm_90a"; }

int kuq_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
  int usable = 0;
  for (int d = 0; d < n; d++) {
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, d) == cudaSuccess && prop.major == 9 && prop.minor == 0) usable = d + 1;
  }
  return usable;
}

const char *kuq_strerror(int code) {
  switch (code) {
    case KUQ_OK: return "ok";
    case KUQ_E_INVALID_ARG: return "invalid argument";
    case KUQ_E_CUDA: return "CUDA error";
    case KUQ_E_NO_DEVICE: return "no sm_90 CUDA device (libkuq has no CPU path)";
    case KUQ_E_DB_FORMAT: return "database in improper format";
    case KUQ_E_UNSUPPORTED_K: return "unsupported k (k-mers of up to 31 bases)";
    case KUQ_E_STATE: return "call order / state error";
    case KUQ_E_CAPACITY: return "capacity exceeded";
    case KUQ_E_NOMEM: return "out of memory";
    case KUQ_E_TAXA_OVERFLOW: return "hit-table pool exhausted (too many reads with more than 32 distinct taxa in one batch)";
    case KUQ_E_TAXONOMY: return "malformed taxonomy";
    default: return "unknown error";
  }
}

const char *kuq_last_error(const kuq_ctx *ctx) { return ctx ? ctx->err.c_str() : ""; }

void kuq_config_default(kuq_config *cfg) {
  if (!cfg) return;
  memset(cfg, 0, sizeof *cfg);
  cfg->device = 0;
  cfg->n_slots = 2;
  cfg->max_reads_per_batch = 1u << 20;
  cfg->max_bases_per_batch = 160ull << 20;
  cfg->work_unit_size = 500000;           // DEF_WORK_UNIT_SIZE, classify.cpp:38
  cfg->hll_mode = KUQ_HLL_PRELOAD;
  cfg->sparse_set_slots = 1ull << 26;
}

int kuq_create(const kuq_config *cfg_in, kuq_ctx **out) {
  if (!out) return KUQ_E_INVALID_ARG;
  *out = nullptr;
  kuq_config cfg;
  kuq_config_default(&cfg);
  if (cfg_in) {
    cfg = *cfg_in;
    kuq_config d;
    kuq_config_default(&d);
    if (!cfg.n_slots) cfg.n_slots = d.n_slots;
    if (!cfg.max_reads_per_batch) cfg.max_reads_per_batch = d.max_reads_per_batch;
    if (!cfg.max_bases_per_batch) cfg.max_bases_per_batch = d.max_bases_per_batch;
    if (!cfg.work_unit_size) cfg.work_unit_size = d.work_unit_size;
    if (!cfg.sparse_set_slots) cfg.sparse_set_slots = d.sparse_set_slots;
  }
  if (cfg.hll_mode > KUQ_HLL_EXACT || cfg.n_slots > 16) return KUQ_E_INVALID_ARG;
  // round the sparse set to a power of two
  uint64_t sc = 1024;
  while (sc < cfg.sparse_set_slots) sc <<= 1;
  cfg.sparse_set_slots = sc;
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= cfg.device || cfg.device < 0) return KUQ_E_NO_DEVICE;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, cfg.device) != cudaSuccess) return KUQ_E_NO_DEVICE;
  if (prop.major != 9 || prop.minor != 0) return KUQ_E_NO_DEVICE;     // kernels are built for sm_90a only
  if (cudaSetDevice(cfg.device) != cudaSuccess) return KUQ_E_NO_DEVICE;
  kuq_ctx *ctx = new kuq_ctx();
  ctx->cfg = cfg;
  ctx->device = cfg.device;
  ctx->n_sm = prop.multiProcessorCount;
  if (ctx->aux.alloc(cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return KUQ_E_CUDA; }
  ctx->slots.resize(cfg.n_slots);
  for (auto &s : ctx->slots) {
    int rc = alloc_slot(ctx, s);
    if (rc) {
      fprintf(stderr, "libkuq: %s\n", ctx->err.c_str());
      kuq_destroy(ctx);
      return rc == KUQ_E_CUDA ? KUQ_E_NOMEM : rc;
    }
  }
  *out = ctx;
  return KUQ_OK;
}

void kuq_destroy(kuq_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  drop_spill(ctx);
  delete ctx;
}

void *kuq_host_alloc(uint64_t bytes) {
  void *p = nullptr;
  // portable: pinned for every CUDA context of the process, whichever thread / device it was allocated from (a buffer
  // that the copying context does not know as pinned silently takes the pageable path: 6 GB/s instead of 50)
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
  return p;
}
void kuq_host_free(void *p) { if (p) cudaFreeHost(p); }

// ---- database -------------------------------------------------------------------------------------------------
namespace {
int parse_images(kuq_ctx *ctx, const void *kdb_image, uint64_t kdb_bytes, const void *idx_image, uint64_t idx_bytes, DbFile &f) {
  std::string err;
  const int rc = parse_db(kdb_image, kdb_bytes, idx_image, idx_bytes, f, err);
  return rc ? fail(ctx, rc, "%s", err.c_str()) : KUQ_OK;
}

// records [offsets[bin_lo], offsets[bin_hi]) of f → d_pairs (12-byte layout), offsets [bin_lo, bin_hi] → d_offsets.
// Bulk H2D through pinned bounce buffers (kuq_bounce.cuh) on the aux stream.  Records shorter than 12 bytes (k <= 28)
// travel as they are in the file: each piece lands in one bounded device buffer and k_widen_records writes it into
// d_pairs in the 12-byte layout, behind the copy on the same stream.
int upload_db(kuq_ctx *ctx, const DbFile &f, uint64_t bin_lo, uint64_t bin_hi, uint8_t *d_pairs, uint64_t *d_offsets) {
  const uint64_t pair_sz = f.pair_sz, rec_lo = f.offsets[bin_lo], n_rec = f.offsets[bin_hi] - rec_lo;
  {
    PinnedBounce bounce;
    CU(bounce.init());
    DevBuf<uint8_t> d_land;
    const uint64_t land_rec = pair_sz == 12 ? 0 : std::min(landing_records(pair_sz), PinnedBounce::CH / pair_sz);
    if (land_rec && n_rec) CU(d_land.alloc(land_rec * pair_sz + SLACK));
    // rec_sz = 0: bytes are copied to d_dst as they are; else they are records of rec_sz bytes, widened into d_dst
    auto piece_copy = [&](uint8_t *d_dst, const uint8_t *h_src, uint64_t bytes, uint64_t rec_sz) -> int {
      if (!rec_sz) {
        CU(bounce.to_device(d_dst, h_src, bytes, ctx->aux));
      } else {
        for (uint64_t off = 0, step = land_rec * rec_sz; off < bytes; off += step) {
          const uint64_t n = std::min(step, bytes - off);
          CU(bounce.h2d(d_land, h_src + off, n, ctx->aux));       // in order behind the last widening
          launch_widen_records(d_land, n / rec_sz, (uint32_t)(rec_sz - 4), d_dst + off / rec_sz * 12, ctx->aux);
          ctx->launches++;
          CU(cudaGetLastError());
        }
      }
      CU(cudaStreamSynchronize(ctx->aux));
      return KUQ_OK;
    };
    int crc = piece_copy(d_pairs, f.records + rec_lo * pair_sz, n_rec * pair_sz, pair_sz == 12 ? 0 : pair_sz);
    if (!crc) crc = piece_copy(reinterpret_cast<uint8_t *>(d_offsets), reinterpret_cast<const uint8_t *>(f.offsets + bin_lo),
                               (bin_hi - bin_lo + 1) * 8, 0);
    if (crc) return crc;
  }
  return KUQ_OK;
}
}  // namespace

namespace {
// Bins [bin_lo, bin_hi) of f (validated by the caller; may be empty) join the staged databases; `first`: they replace
// whatever the context held.  The taxonomy numbering survives a re-stage (chunked mode) as long as the new range only
// holds numbered taxids; the sparse-tier keys of the old records leave with them into the set.  A range that fails to
// stage is not kept.
int stage_range(kuq_ctx *ctx, const DbFile &f, uint64_t bin_lo, uint64_t bin_hi, bool first) {
  const uint64_t rec_lo = f.offsets[bin_lo], rec_hi = f.offsets[bin_hi];
  if (rec_hi < rec_lo || rec_hi > f.key_ct) return fail(ctx, KUQ_E_DB_FORMAT, "index offsets inconsistent with key count");
  if (first) {
    { int hrc = harvest_seen(ctx, false, true); if (hrc) return hrc; }
    stream_close(ctx);
    free_db(ctx);
    ctx->k = f.k;
  }
  ctx->dbs.emplace_back();
  StagedDb &e = ctx->dbs.back();
  auto drop = [&](int code) { ctx->dbs.pop_back(); return code; };
  const uint64_t key_ct = rec_hi - rec_lo;
  if (e.own_pairs.alloc(key_ct * 12 + SLACK) != cudaSuccess || e.own_offsets.alloc(bin_hi - bin_lo + 1) != cudaSuccess) {
    (void)cudaGetLastError();
    return drop(fail(ctx, KUQ_E_NOMEM, "no room for database %zu (%llu records)", ctx->dbs.size(), (unsigned long long)key_ct));
  }
  e.range = DbRange{e.own_pairs, e.own_offsets, key_ct, rec_lo, bin_lo, bin_hi, f.nt, f.idx_type};
  int rc = upload_db(ctx, f, bin_lo, bin_hi, e.own_pairs, e.own_offsets);
  if (!rc) rc = collect_taxids(ctx, e);
  if (rc) return drop(rc);
  if (ctx->finalized) return remap_db(ctx);
  return KUQ_OK;
}
}  // namespace

int kuq_stage_db(kuq_ctx *ctx, const void *kdb_image, uint64_t kdb_bytes, const void *idx_image, uint64_t idx_bytes,
                 uint64_t bin_lo, uint64_t bin_hi) {
  if (!ctx || !kdb_image || !idx_image) return KUQ_E_INVALID_ARG;
  CU(cudaSetDevice(ctx->device));
  DbFile f;
  int rc = parse_images(ctx, kdb_image, kdb_bytes, idx_image, idx_bytes, f);
  if (rc) return rc;
  if (bin_hi == 0 || bin_hi > f.n_bins) bin_hi = f.n_bins;
  if (bin_lo >= bin_hi) return fail(ctx, KUQ_E_INVALID_ARG, "empty minimizer range");
  return stage_range(ctx, f, bin_lo, bin_hi, true);
}

int kuq_stage_db_append_range(kuq_ctx *ctx, const void *kdb_image, uint64_t kdb_bytes, const void *idx_image,
                              uint64_t idx_bytes, uint64_t bin_lo, uint64_t bin_hi) {
  if (!ctx || !kdb_image || !idx_image) return KUQ_E_INVALID_ARG;
  CU(cudaSetDevice(ctx->device));
  DbFile f;
  int rc = parse_images(ctx, kdb_image, kdb_bytes, idx_image, idx_bytes, f);
  if (rc) return rc;
  if (bin_hi == 0) bin_hi = f.n_bins;                // (0, 0) = the whole database; lo == hi != 0 = an empty slice
  if (bin_lo > bin_hi || bin_hi > f.n_bins)
    return fail(ctx, KUQ_E_INVALID_ARG, "minimizer range [%llu, %llu) outside the %llu bins of nt = %u", (unsigned long long)bin_lo,
                (unsigned long long)bin_hi, (unsigned long long)f.n_bins, f.nt);
  const bool first = ctx->dbs.empty() || ctx->stream_open;
  if (!first) {
    if (f.k != ctx->k) return fail(ctx, KUQ_E_INVALID_ARG, "the databases differ in k: %u vs %u", ctx->k, f.k);
    if (f.offsets[f.n_bins] != f.key_ct) return fail(ctx, KUQ_E_DB_FORMAT, "index offsets inconsistent with key count");
  }
  return stage_range(ctx, f, bin_lo, bin_hi, first);
}

int kuq_stage_db_append(kuq_ctx *ctx, const void *kdb_image, uint64_t kdb_bytes, const void *idx_image, uint64_t idx_bytes) {
  return kuq_stage_db_append_range(ctx, kdb_image, kdb_bytes, idx_image, idx_bytes, 0, 0);
}

int kuq_db_runs(kuq_ctx *ctx, uint32_t *n_runs) {
  if (!ctx || !n_runs) return KUQ_E_INVALID_ARG;
  if (ctx->dbs.empty()) return fail(ctx, KUQ_E_STATE, "no database staged");
  *n_runs = count_runs(ctx);
  return KUQ_OK;
}

int kuq_attach_db_device(kuq_ctx *ctx, void *d_pairs, uint64_t key_ct, const uint64_t *d_offsets, uint32_t k,
                         uint32_t nt, uint32_t idx_type, uint64_t bin_lo, uint64_t bin_hi) {
  if (!ctx || !d_pairs || !d_offsets) return KUQ_E_INVALID_ARG;
  if (k < 29 || k > 31) return fail(ctx, KUQ_E_UNSUPPORTED_K, "k = %u: only 8-byte keys (k = 29..31)", k);
  if (nt < 1 || nt > 15 || (idx_type != 1 && idx_type != 2)) return fail(ctx, KUQ_E_INVALID_ARG, "bad index parameters");
  CU(cudaSetDevice(ctx->device));
  uint64_t n_bins = 1ull << (2 * nt);
  if (bin_hi == 0 || bin_hi > n_bins) bin_hi = n_bins;
  if (bin_lo >= bin_hi) return fail(ctx, KUQ_E_INVALID_ARG, "empty minimizer range");
  { int hrc = harvest_seen(ctx, false, true); if (hrc) return hrc; }
  free_db(ctx);
  ctx->k = k;
  uint64_t first = 0;
  CU(cudaMemcpy(&first, d_offsets, 8, cudaMemcpyDeviceToHost));
  ctx->dbs.emplace_back();
  ctx->dbs[0].range = DbRange{(uint8_t *)d_pairs, d_offsets, key_ct, first, bin_lo, bin_hi, nt, idx_type};
  int rc = collect_taxids(ctx, ctx->dbs[0]);
  if (rc) return rc;
  if (ctx->finalized) return remap_db(ctx);
  return KUQ_OK;
}

int kuq_db_taxids(kuq_ctx *ctx, uint32_t *taxid, uint64_t *count, uint32_t cap, uint32_t *n) {
  if (!ctx || !n) return KUQ_E_INVALID_ARG;
  if (ctx->dbs.empty()) return fail(ctx, KUQ_E_STATE, "no database staged");
  std::vector<std::pair<uint32_t, uint64_t>> all;          // over every staged range (counts summed)
  for (auto &e : ctx->dbs)
    for (size_t i = 0; i < e.taxids.size(); i++) all.emplace_back(e.taxids[i], e.counts[i]);
  std::sort(all.begin(), all.end());
  std::vector<std::pair<uint32_t, uint64_t>> u;
  for (auto &pr : all) {
    if (!u.empty() && u.back().first == pr.first) u.back().second += pr.second;
    else u.push_back(pr);
  }
  *n = (uint32_t)u.size();
  if (cap == 0) return KUQ_OK;
  if (cap < *n) return fail(ctx, KUQ_E_CAPACITY, "need room for %u taxids", *n);
  for (uint32_t i = 0; i < *n; i++) {
    if (taxid) taxid[i] = u[i].first;
    if (count) count[i] = u[i].second;
  }
  return KUQ_OK;
}

int kuq_set_db_taxid_universe(kuq_ctx *ctx, const uint32_t *taxid, uint32_t n) {
  if (!ctx || (!taxid && n)) return KUQ_E_INVALID_ARG;
  if (ctx->finalized) return fail(ctx, KUQ_E_STATE, "taxid universe must be declared before the first classification");
  ctx->universe.assign(taxid, taxid + n);
  return KUQ_OK;
}

int kuq_set_quick_mode(kuq_ctx *ctx, uint32_t min_hits, int stop_at_last_hit) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  for (auto &s : ctx->slots)
    if (s.busy) return fail(ctx, KUQ_E_STATE, "quick mode cannot change while a batch is in flight");
  if (min_hits && ctx->cfg.hll_mode == KUQ_HLL_EXACT) return fail(ctx, KUQ_E_INVALID_ARG, "quick mode is not available with KUQ_HLL_EXACT");
  ctx->quick_min = min_hits;
  ctx->quick_stop = min_hits && stop_at_last_hit;
  return KUQ_OK;
}

int kuq_mark_zero_hits(kuq_ctx *ctx, int on) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  ctx->mark_zero_hits = on != 0;
  return KUQ_OK;
}

int kuq_set_taxonomy(kuq_ctx *ctx, const uint32_t *taxid, const uint32_t *parent, uint32_t n) {
  if (!ctx || ((!taxid || !parent) && n)) return KUQ_E_INVALID_ARG;
  if (ctx->finalized) return fail(ctx, KUQ_E_STATE, "taxonomy already in use; create a new context to change it");
  // later rows overwrite earlier ones, like Parent_map[taxid] = parent
  std::unordered_map<uint32_t, uint32_t> m;
  for (uint32_t i = 0; i < n; i++) m[taxid[i]] = parent[i];
  ctx->tax_ids.clear(); ctx->tax_parents.clear();
  for (auto &kv : m) { ctx->tax_ids.push_back(kv.first); ctx->tax_parents.push_back(kv.second); }
  ctx->tax_set = true;
  return KUQ_OK;
}

int kuq_set_threshold(kuq_ctx *ctx, double threshold, const uint32_t *taxid, const uint32_t *parent, uint32_t n) {
  if (!ctx || ((!taxid || !parent) && n)) return KUQ_E_INVALID_ARG;
  if (!(threshold >= 0 && threshold <= 1)) return fail(ctx, KUQ_E_INVALID_ARG, "threshold must be in the interval [0,1]");
  if (!ctx->tax_set) return fail(ctx, KUQ_E_STATE, "kuq_set_threshold: set the taxonomy first");
  if (ctx->filter_set) return fail(ctx, KUQ_E_STATE, "the threshold is already set");
  for (auto &s : ctx->slots)
    if (s.busy) return fail(ctx, KUQ_E_STATE, "the threshold cannot be set while a batch is in flight");
  // F (krakenuniq-filter:136-146): rows in file order, `$parent_map{$taxID} = $parentTaxID unless $parentTaxID == $taxID`
  std::unordered_map<uint32_t, uint32_t> F, depth;
  for (uint32_t i = 0; i < n; i++)
    if (parent[i] != taxid[i]) F[taxid[i]] = parent[i];
  if (F.count(0)) return fail(ctx, KUQ_E_TAXONOMY, "taxid 0 has parent %u in the taxonomy: the filter would divide by zero", F[0]);
  // F-depth = steps until a node without an F entry; a cycle would keep the script's loops going forever
  std::vector<uint32_t> stack;
  std::unordered_map<uint32_t, bool> on_stack;
  for (auto &kv : F) {
    uint32_t x = kv.first;
    stack.clear();
    while (F.count(x) && !depth.count(x)) {
      if (on_stack[x]) return fail(ctx, KUQ_E_TAXONOMY, "cycle in the parents of the taxonomy at taxid %u", x);
      on_stack[x] = true;
      stack.push_back(x);
      x = F[x];
    }
    uint32_t d = F.count(x) ? depth[x] : 0;
    while (!stack.empty()) { depth[stack.back()] = ++d; on_stack[stack.back()] = false; stack.pop_back(); }
  }
  CU(cudaSetDevice(ctx->device));
  const uint64_t mr = ctx->cfg.max_reads_per_batch;
  for (auto &s : ctx->slots) {
    CU(s.d_fcall.alloc(mr));
    CU(s.d_fhits.alloc(mr));
    CU(s.d_ftotal.alloc(mr));
    CU(s.h_fcall.alloc(mr));
    CU(s.h_fhits.alloc(mr));
    CU(s.h_ftotal.alloc(mr));
  }
  ctx->f_parent.swap(F);
  ctx->f_depth.swap(depth);
  ctx->threshold = threshold;
  ctx->filter_set = true;
  return ctx->finalized ? upload_filter(ctx) : KUQ_OK;
}

namespace {
// get_children (krakenuniq-extract-reads:48-58,65-76) over the child multigraph of the rows: the listed taxa and, with
// KUQ_EXTRACT_SUBTREE, everything reachable from them, ascending.  A depth-first walk that meets a node still on its
// path has found a cycle: KUQ_E_TAXONOMY, *cycle_at = that node.
int extract_members(const uint32_t *list, uint32_t n_list, uint32_t flags, const uint32_t *taxid, const uint32_t *parent,
                    uint32_t n_rows, std::vector<uint32_t> &out, uint32_t *cycle_at) {
  std::unordered_set<uint32_t> members(list, list + n_list);
  if (flags & KUQ_EXTRACT_SUBTREE) {
    std::unordered_map<uint32_t, std::vector<uint32_t>> children;
    for (uint32_t i = 0; i < n_rows; i++)
      if (taxid[i] != parent[i]) children[parent[i]].push_back(taxid[i]);
    std::unordered_map<uint32_t, uint8_t> state;          // 1 = on the walk's path, 2 = done
    std::vector<std::pair<uint32_t, size_t>> path;
    for (uint32_t i = 0; i < n_list; i++) {
      if (state[list[i]]) continue;
      path.assign(1, {list[i], 0});
      state[list[i]] = 1;
      while (!path.empty()) {
        const uint32_t node = path.back().first;
        auto it = children.find(node);
        if (it == children.end() || path.back().second == it->second.size()) { state[node] = 2; path.pop_back(); continue; }
        const uint32_t c = it->second[path.back().second++];
        uint8_t &st = state[c];
        if (st == 1) { *cycle_at = c; return KUQ_E_TAXONOMY; }
        if (st == 2) continue;
        st = 1;
        members.insert(c);
        path.push_back({c, 0});
      }
    }
  }
  out.assign(members.begin(), members.end());
  std::sort(out.begin(), out.end());
  return KUQ_OK;
}
}  // namespace

int kuq_extract_taxa(const uint32_t *list, uint32_t n_list, uint32_t flags, const uint32_t *taxid, const uint32_t *parent,
                     uint32_t n_rows, uint32_t *out, uint32_t cap, uint32_t *n_out) {
  if ((!list && n_list) || ((!taxid || !parent) && n_rows) || !n_out || (!out && cap)) return KUQ_E_INVALID_ARG;
  std::vector<uint32_t> m;
  uint32_t at = 0;
  const int rc = extract_members(list, n_list, flags, taxid, parent, n_rows, m, &at);
  if (rc) return rc;
  *n_out = (uint32_t)m.size();
  if (cap) std::copy(m.begin(), m.begin() + std::min<size_t>(cap, m.size()), out);
  return KUQ_OK;
}

int kuq_set_extract(kuq_ctx *ctx, const uint32_t *list, uint32_t n_list, uint32_t flags, const uint32_t *taxid,
                    const uint32_t *parent, uint32_t n_rows) {
  if (!ctx || (!list && n_list) || ((!taxid || !parent) && n_rows)) return KUQ_E_INVALID_ARG;
  if (flags & ~(KUQ_EXTRACT_SUBTREE | KUQ_EXTRACT_INVERT | KUQ_EXTRACT_OTHERS | KUQ_EXTRACT_CLASSIFIED_ONLY))
    return fail(ctx, KUQ_E_INVALID_ARG, "unknown kuq_set_extract flags 0x%x", flags);
  if (!ctx->tax_set) return fail(ctx, KUQ_E_STATE, "kuq_set_extract: set the taxonomy first");
  if (ctx->extract_set) return fail(ctx, KUQ_E_STATE, "the extraction is already set");
  for (auto &s : ctx->slots)
    if (s.busy) return fail(ctx, KUQ_E_STATE, "the extraction cannot be set while a batch is in flight");
  std::vector<uint32_t> sorted;
  uint32_t at = 0;
  if (extract_members(list, n_list, flags, taxid, parent, n_rows, sorted, &at))
    return fail(ctx, KUQ_E_TAXONOMY, "cycle in the children of the taxonomy at taxid %u", at);
  const uint32_t n_members = (uint32_t)sorted.size();
  sorted.push_back(0);                                  // never an empty allocation
  CU(cudaSetDevice(ctx->device));
  CU(ctx->d_members.alloc(sorted.size()));
  CU(cudaMemcpy(ctx->d_members, sorted.data(), sorted.size() * 4, cudaMemcpyHostToDevice));
  for (auto &s : ctx->slots) {
    CU(s.d_xsel.alloc(extract_count_at(ctx) + 16));
    CU(s.h_xsel.alloc(extract_count_at(ctx) + 16));
  }
  ctx->n_members = n_members;
  ctx->extract_flags = flags;
  ctx->extract_set = true;
  return KUQ_OK;
}

// ---- classification -------------------------------------------------------------------------------------------
namespace {
// D2H of a batch's fixed-size results; the variable-size hit lists follow in kuq_wait_batch
int copy_results(kuq_ctx *ctx, Slot &s) {
  const uint64_t n = s.n_reads;
  if (n) {
    CU(cudaMemcpyAsync(s.h_call, s.d_call, n * 4, cudaMemcpyDeviceToHost, s.stream));
    CU(cudaMemcpyAsync(s.h_nwin, s.d_nwin, n * 4, cudaMemcpyDeviceToHost, s.stream));
    if (!(s.flags & KUQ_F_NO_RUNS) || ctx->quick_min) {
      CU(cudaMemcpyAsync(s.h_run_start, s.d_run_start, n * 4, cudaMemcpyDeviceToHost, s.stream));
      CU(cudaMemcpyAsync(s.h_run_count, s.d_run_count, n * 4, cudaMemcpyDeviceToHost, s.stream));
    }
    if (ctx->filter_set) {
      CU(cudaMemcpyAsync(s.h_fcall, s.d_fcall, n * 4, cudaMemcpyDeviceToHost, s.stream));
      CU(cudaMemcpyAsync(s.h_fhits, s.d_fhits, n * 4, cudaMemcpyDeviceToHost, s.stream));
      CU(cudaMemcpyAsync(s.h_ftotal, s.d_ftotal, n * 4, cudaMemcpyDeviceToHost, s.stream));
    }
    if (ctx->extract_set) {
      CU(cudaMemcpyAsync(s.h_xsel, s.d_xsel, n, cudaMemcpyDeviceToHost, s.stream));
      CU(cudaMemcpyAsync(s.h_xsel + extract_count_at(ctx), s.d_xsel + extract_count_at(ctx), 4, cudaMemcpyDeviceToHost, s.stream));
    }
  }
  CU(cudaMemcpyAsync(s.h_scalars, s.d_scalars, 8 * 8, cudaMemcpyDeviceToHost, s.stream));
  return KUQ_OK;
}

// copy one batch of reads (host) into the slot; returns the total number of bases
int upload_reads(kuq_ctx *ctx, Slot &s, const char *bases, const uint64_t *read_offsets, uint32_t n_reads, uint64_t *total_out) {
  if (n_reads > ctx->cfg.max_reads_per_batch) return fail(ctx, KUQ_E_CAPACITY, "%u reads > slot capacity %u", n_reads, ctx->cfg.max_reads_per_batch);
  const uint64_t base0 = n_reads ? read_offsets[0] : 0;
  const uint64_t total = n_reads ? read_offsets[n_reads] - base0 : 0;
  if (total > ctx->cfg.max_bases_per_batch) return fail(ctx, KUQ_E_CAPACITY, "%llu bases > slot capacity %llu", (unsigned long long)total, (unsigned long long)ctx->cfg.max_bases_per_batch);
  if (total >= (1ull << 32)) return fail(ctx, KUQ_E_CAPACITY, "batches are limited to 4 Gbases");
  *total_out = total;
  if (!n_reads) return KUQ_OK;
  CU(cudaMemcpyAsync(s.d_bases, bases + base0, total, cudaMemcpyHostToDevice, s.stream));
  CU(cudaMemsetAsync(s.d_bases + total, 'N', SLACK, s.stream));
  if (base0 == 0) {
    CU(cudaMemcpyAsync(s.d_offsets, read_offsets, (n_reads + 1ull) * 8, cudaMemcpyHostToDevice, s.stream));
  } else {
    std::vector<uint64_t> tmp(n_reads + 1);
    for (uint32_t i = 0; i <= n_reads; i++) tmp[i] = read_offsets[i] - base0;
    CU(cudaMemcpy(s.d_offsets, tmp.data(), (n_reads + 1ull) * 8, cudaMemcpyHostToDevice));
  }
  return KUQ_OK;
}
}  // namespace

int kuq_lookup_batch(kuq_ctx *ctx, const char *bases, const uint64_t *read_offsets, uint32_t n_reads,
                     uint32_t *codes_out, uint32_t *n_windows_out) {
  int rc = check_slot(ctx, 0);
  if (rc) return rc;
  if (n_reads && (!bases || !read_offsets || !codes_out)) return fail(ctx, KUQ_E_INVALID_ARG, "NULL batch buffers");
  CU(cudaSetDevice(ctx->device));
  Slot &s = ctx->slots[0];
  if (s.busy) return fail(ctx, KUQ_E_STATE, "slot 0 still has an unread batch");
  rc = ensure_ready(ctx);
  if (rc) return rc;
  uint64_t total = 0;
  rc = upload_reads(ctx, s, bases, read_offsets, n_reads, &total);
  if (rc) return rc;
  s.n_reads = n_reads; s.flags = 0; s.total_bases = total; s.external = false;
  Params p;
  fill_params(ctx, s, p, s.d_bases, s.d_offsets, nullptr, n_reads, 0);
  // positions without a window are not written by the kernels: give the caller zeros there
  CU(cudaMemsetAsync(s.d_dense, 0, total * 4, s.stream));
  rc = launch_on_slot(ctx, s, MODE_LOOKUP, p);
  if (rc) return rc;
  if (n_reads) {
    CU(cudaMemcpyAsync(codes_out, s.d_dense, total * 4, cudaMemcpyDeviceToHost, s.stream));
    if (n_windows_out) CU(cudaMemcpyAsync(n_windows_out, s.d_nwin, n_reads * 4ull, cudaMemcpyDeviceToHost, s.stream));
  }
  CU(cudaStreamSynchronize(s.stream));
  return KUQ_OK;
}

int kuq_resolve_batch(kuq_ctx *ctx, const char *bases, const uint64_t *read_offsets, uint32_t n_reads,
                      const uint32_t *codes_in, const uint32_t *unit_id, uint32_t flags, kuq_batch_result *out) {
  int rc = check_slot(ctx, 0);
  if (rc) return rc;
  if (!out || (n_reads && (!bases || !read_offsets || !codes_in))) return fail(ctx, KUQ_E_INVALID_ARG, "NULL batch buffers");
  CU(cudaSetDevice(ctx->device));
  Slot &s = ctx->slots[0];
  if (s.busy) return fail(ctx, KUQ_E_STATE, "slot 0 still has an unread batch");
  rc = ensure_ready(ctx);
  if (rc) return rc;
  uint64_t total = 0;
  rc = upload_reads(ctx, s, bases, read_offsets, n_reads, &total);
  if (rc) return rc;
  if (!s.d_codes_in) CU(s.d_codes_in.alloc(ctx->cfg.max_bases_per_batch + SLACK));
  if (n_reads) CU(cudaMemcpyAsync(s.d_codes_in, codes_in, total * 4, cudaMemcpyHostToDevice, s.stream));
  s.n_reads = n_reads; s.flags = flags; s.total_bases = total; s.external = false;
  const uint32_t *d_unit = nullptr;
  if (ctx->cfg.hll_mode == KUQ_HLL_PRELOAD && n_reads) {
    if (unit_id) memcpy(s.h_unit, unit_id, n_reads * 4ull);
    else cut_units(ctx, read_offsets, n_reads, s.h_unit);
    CU(cudaMemcpyAsync(s.d_unit, s.h_unit, n_reads * 4ull, cudaMemcpyHostToDevice, s.stream));
    d_unit = s.d_unit;
  }
  Params p;
  fill_params(ctx, s, p, s.d_bases, s.d_offsets, d_unit, n_reads, flags);
  p.codes_in = s.d_codes_in;
  rc = launch_on_slot(ctx, s, MODE_RESOLVE, p);
  if (rc) return rc;
  rc = copy_results(ctx, s);
  if (rc) return rc;
  s.busy = true;
  return kuq_wait_batch(ctx, 0, out);
}

int kuq_submit_batch(kuq_ctx *ctx, uint32_t slot, const char *bases, const uint64_t *read_offsets, uint32_t n_reads,
                     const uint32_t *unit_id, uint32_t flags) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (n_reads && (!bases || !read_offsets)) return fail(ctx, KUQ_E_INVALID_ARG, "NULL batch buffers");
  CU(cudaSetDevice(ctx->device));
  Slot &s = ctx->slots[slot];
  if (s.busy) return fail(ctx, KUQ_E_STATE, "slot %u still has an unread batch: call kuq_wait_batch first", slot);
  rc = ensure_ready(ctx);
  if (rc) return rc;
  uint64_t total = 0;
  rc = upload_reads(ctx, s, bases, read_offsets, n_reads, &total);
  if (rc) return rc;
  s.n_reads = n_reads; s.flags = flags; s.total_bases = total; s.external = false;
  const uint32_t *d_unit = nullptr;
  if (ctx->cfg.hll_mode == KUQ_HLL_PRELOAD && n_reads) {
    if (unit_id) memcpy(s.h_unit, unit_id, n_reads * 4ull);
    else cut_units(ctx, read_offsets, n_reads, s.h_unit);
    CU(cudaMemcpyAsync(s.d_unit, s.h_unit, n_reads * 4ull, cudaMemcpyHostToDevice, s.stream));
    d_unit = s.d_unit;
  }
  Params p;
  fill_params(ctx, s, p, s.d_bases, s.d_offsets, d_unit, n_reads, flags);
  rc = launch_on_slot(ctx, s, MODE_FUSED, p);
  if (rc) return rc;
  // D2H of the fixed-size results; the variable-size hit lists follow in kuq_wait_batch
  rc = copy_results(ctx, s);
  if (rc) return rc;
  s.busy = true;
  return KUQ_OK;
}

int kuq_wait_batch(kuq_ctx *ctx, uint32_t slot, kuq_batch_result *out) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (!out) return KUQ_E_INVALID_ARG;
  CU(cudaSetDevice(ctx->device));
  Slot &s = ctx->slots[slot];
  if (!s.busy) return fail(ctx, KUQ_E_STATE, "slot %u has no batch in flight", slot);
  CU(cudaStreamSynchronize(s.stream));
  s.busy = false;
  float ms = 0;
  if (s.timed) cudaEventElapsedTime(&ms, s.ev_k0, s.ev_k1);
  (void)cudaGetLastError();
  s.kernel_ms = ms;
  const uint32_t err = (uint32_t)(s.h_scalars[3] & 0xFFFFFFFFu);
  if (err == 1) return fail(ctx, KUQ_E_TAXA_OVERFLOW, "the batch exhausted the hit-table pool for reads with more than 32 distinct taxa: use smaller batches");
  if (err == 4) return batch_set_saturated(ctx);
  if (err == 5) return fail(ctx, KUQ_E_CAPACITY, "the hit lists of the batch need more run slots than the slot holds (%llu): use smaller batches", (unsigned long long)s.runs_cap);
  if (err) return fail(ctx, KUQ_E_CAPACITY, "per-batch work-unit bookkeeping overflowed (code %u): use smaller batches", err);
  const uint64_t n_runs = (s.flags & KUQ_F_NO_RUNS) ? 0 : s.h_scalars[0];
  if (n_runs) {
    if (n_runs > s.h_runs_cap) {
      s.h_runs_cap = n_runs + n_runs / 2;
      CU(s.h_runs.alloc(s.h_runs_cap));
    }
    CU(cudaMemcpyAsync(s.h_runs, s.d_runs, n_runs * 8, cudaMemcpyDeviceToHost, s.stream));
  }
  if ((s.flags & KUQ_F_WANT_CODES) && s.total_bases) {
    if (!s.h_codes) CU(s.h_codes.alloc(ctx->cfg.max_bases_per_batch));
    CU(cudaMemcpyAsync(s.h_codes, s.d_codes, s.total_bases * 4, cudaMemcpyDeviceToHost, s.stream));
  }
  CU(cudaStreamSynchronize(s.stream));
  memset(out, 0, sizeof *out);
  out->n_reads = s.n_reads;
  out->call = s.h_call;
  out->n_windows = s.h_nwin;
  out->run_start = s.h_run_start;
  out->run_count = s.h_run_count;
  out->runs = s.h_runs;
  out->n_runs = n_runs;
  out->codes = (s.flags & KUQ_F_WANT_CODES) ? s.h_codes.get() : nullptr;
  out->n_classified = s.h_scalars[1];
  out->kernel_ms = s.kernel_ms;
  if (ctx->filter_set) {
    out->filtered_call = s.h_fcall;
    out->filter_hits = s.h_fhits;
    out->filter_total = s.h_ftotal;
  }
  if (ctx->extract_set) {
    out->extract_sel = s.h_xsel;
    uint32_t n_sel = 0;
    if (s.n_reads) memcpy(&n_sel, s.h_xsel + extract_count_at(ctx), 4);
    out->n_extract = n_sel;
  }
  return KUQ_OK;
}

int kuq_classify_batch(kuq_ctx *ctx, const char *bases, const uint64_t *read_offsets, uint32_t n_reads,
                       const uint32_t *unit_id, uint32_t flags, kuq_batch_result *out) {
  int rc = kuq_submit_batch(ctx, 0, bases, read_offsets, n_reads, unit_id, flags);
  if (rc) return rc;
  return kuq_wait_batch(ctx, 0, out);
}

static int device_call(kuq_ctx *ctx, uint32_t slot, int mode, const char *d_bases, const uint64_t *d_offsets,
                       uint32_t n_reads, uint64_t total_bases, const uint32_t *d_unit, uint32_t flags,
                       uint32_t *d_codes_out, const uint32_t *d_codes_in, uint32_t only_hits) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (n_reads && (!d_bases || !d_offsets)) return fail(ctx, KUQ_E_INVALID_ARG, "NULL device buffers");
  if ((uintptr_t)d_bases & 15) return fail(ctx, KUQ_E_INVALID_ARG, "d_bases must be 16-byte aligned");
  CU(cudaSetDevice(ctx->device));
  rc = ensure_ready(ctx);
  if (rc) return rc;
  if (mode != MODE_LOOKUP && ctx->cfg.hll_mode == KUQ_HLL_PRELOAD && !d_unit && !(flags & KUQ_F_NO_COUNTS) && n_reads)
    return fail(ctx, KUQ_E_INVALID_ARG, "KUQ_HLL_PRELOAD needs the work-unit id of every read (d_unit_id) to "
                "reproduce the per-unit sketches; pass it, or create the context with KUQ_HLL_CHUNKED / KUQ_HLL_DENSE_ONLY");
  Slot &s = ctx->slots[slot];
  if (n_reads > ctx->cfg.max_reads_per_batch || total_bases > ctx->cfg.max_bases_per_batch)
    return fail(ctx, KUQ_E_CAPACITY, "batch exceeds the slot capacity");
  s.n_reads = n_reads; s.flags = flags; s.total_bases = total_bases; s.external = true;
  Params p;
  fill_params(ctx, s, p, d_bases, d_offsets, d_unit, n_reads, flags);
  if (mode == MODE_LOOKUP) { p.codes_dense = d_codes_out; p.only_hits = only_hits; }
  if (mode == MODE_RESOLVE) p.codes_in = d_codes_in;
  return launch_on_slot(ctx, s, mode, p);
}

int kuq_classify_device(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets,
                        uint32_t n_reads, uint64_t total_bases, const uint32_t *d_unit_id, uint32_t flags) {
  return device_call(ctx, slot, MODE_FUSED, d_bases, d_read_offsets, n_reads, total_bases, d_unit_id, flags, nullptr, nullptr, 0);
}
int kuq_lookup_device(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets,
                      uint32_t n_reads, uint64_t total_bases, uint32_t *d_codes_out, uint32_t only_hits) {
  if (!d_codes_out) return KUQ_E_INVALID_ARG;
  return device_call(ctx, slot, MODE_LOOKUP, d_bases, d_read_offsets, n_reads, total_bases, nullptr, 0, d_codes_out, nullptr, only_hits);
}
int kuq_resolve_device(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets,
                       uint32_t n_reads, uint64_t total_bases, const uint32_t *d_codes_in, const uint32_t *d_unit_id,
                       uint32_t flags) {
  if (!d_codes_in) return KUQ_E_INVALID_ARG;
  return device_call(ctx, slot, MODE_RESOLVE, d_bases, d_read_offsets, n_reads, total_bases, d_unit_id, flags, nullptr, d_codes_in, 0);
}

// run < 0: kuq_lookup_device_peers (one database, hits only); run >= 0: that run of the in-order lookup
static int peers_call(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets, uint32_t n_reads,
                      uint64_t total_bases, uint32_t *const *d_codes_peers, const uint64_t *base_bounds, uint32_t n_peers,
                      int run) {
  if (!d_codes_peers || !base_bounds || n_peers == 0 || n_peers > 8) return KUQ_E_INVALID_ARG;
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (n_reads && (!d_bases || !d_read_offsets)) return fail(ctx, KUQ_E_INVALID_ARG, "NULL device buffers");
  if ((uintptr_t)d_bases & 15) return fail(ctx, KUQ_E_INVALID_ARG, "d_bases must be 16-byte aligned");
  CU(cudaSetDevice(ctx->device));
  rc = ensure_ready(ctx);
  if (rc) return rc;
  Slot &s = ctx->slots[slot];
  if (n_reads > ctx->cfg.max_reads_per_batch || total_bases > ctx->cfg.max_bases_per_batch)
    return fail(ctx, KUQ_E_CAPACITY, "batch exceeds the slot capacity");
  s.n_reads = n_reads; s.flags = 0; s.total_bases = total_bases; s.external = true;
  Params p;
  fill_params(ctx, s, p, d_bases, d_read_offsets, nullptr, n_reads, 0);
  p.only_hits = run > 0 ? KUQ_LOOKUP_FILL_EMPTY : 1;
  p.n_peers = n_peers;
  for (uint32_t j = 0; j < n_peers; j++) { p.peer_codes[j] = d_codes_peers[j]; p.peer_bounds[j] = base_bounds[j]; }
  p.peer_bounds[n_peers] = base_bounds[n_peers];
  return launch_on_slot(ctx, s, MODE_LOOKUP, p, run);
}

int kuq_lookup_device_peers(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets,
                            uint32_t n_reads, uint64_t total_bases, uint32_t *const *d_codes_peers,
                            const uint64_t *base_bounds, uint32_t n_peers) {
  return peers_call(ctx, slot, d_bases, d_read_offsets, n_reads, total_bases, d_codes_peers, base_bounds, n_peers, -1);
}

int kuq_lookup_device_peers_run(kuq_ctx *ctx, uint32_t slot, const char *d_bases, const uint64_t *d_read_offsets,
                                uint32_t n_reads, uint64_t total_bases, uint32_t *const *d_codes_peers,
                                const uint64_t *base_bounds, uint32_t n_peers, uint32_t run) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  if (ctx->dbs.empty()) return fail(ctx, KUQ_E_STATE, "no database staged");
  const uint32_t n_runs = count_runs(ctx);
  if (run >= n_runs) return fail(ctx, KUQ_E_INVALID_ARG, "run %u of %u", run, n_runs);
  return peers_call(ctx, slot, d_bases, d_read_offsets, n_reads, total_bases, d_codes_peers, base_bounds, n_peers, (int)run);
}

// ---- device memory that can be shared with the other ranks of a node (CUDA IPC) --------------------------------
void *kuq_device_alloc(kuq_ctx *ctx, uint64_t bytes) {
  if (!ctx) return nullptr;
  if (cudaSetDevice(ctx->device) != cudaSuccess) return nullptr;
  void *p = nullptr;
  if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
  return p;
}
void kuq_device_free(kuq_ctx *ctx, void *p) {
  if (ctx) cudaSetDevice(ctx->device);
  if (p) cudaFree(p);
}
int kuq_device_memset(kuq_ctx *ctx, uint32_t slot, void *p, int value, uint64_t bytes) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  CU(cudaSetDevice(ctx->device));
  CU(cudaMemsetAsync(p, value, bytes, ctx->slots[slot].stream));
  return KUQ_OK;
}
int kuq_ipc_export(kuq_ctx *ctx, void *d_ptr, uint8_t handle64[64]) {
  if (!ctx || !d_ptr || !handle64) return KUQ_E_INVALID_ARG;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  CU(cudaSetDevice(ctx->device));
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, d_ptr));
  memcpy(handle64, &h, 64);
  return KUQ_OK;
}
int kuq_ipc_open(kuq_ctx *ctx, const uint8_t handle64[64], void **d_ptr_out) {
  if (!ctx || !handle64 || !d_ptr_out) return KUQ_E_INVALID_ARG;
  CU(cudaSetDevice(ctx->device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  CU(cudaIpcOpenMemHandle(d_ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
  return KUQ_OK;
}
int kuq_ipc_close(kuq_ctx *ctx, void *d_ptr) {
  if (!ctx || !d_ptr) return KUQ_E_INVALID_ARG;
  CU(cudaSetDevice(ctx->device));
  CU(cudaIpcCloseMemHandle(d_ptr));
  return KUQ_OK;
}

int kuq_copy_to_device(kuq_ctx *ctx, uint32_t slot, void *d_dst, const void *h_src, uint64_t bytes) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (!bytes) return KUQ_OK;
  if (!d_dst || !h_src) return KUQ_E_INVALID_ARG;
  CU(cudaSetDevice(ctx->device));
  CU(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, ctx->slots[slot].stream));
  return KUQ_OK;
}

uint64_t kuq_device_free_bytes(kuq_ctx *ctx) {
  if (!ctx || cudaSetDevice(ctx->device) != cudaSuccess) return 0;
  size_t fr = 0, tot = 0;
  if (cudaMemGetInfo(&fr, &tot) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
  return fr;
}

// after kuq_classify_device / kuq_resolve_device on `slot`: bring the batch's results to the slot's pinned host
// buffers and wait — the device-input counterpart of kuq_classify_batch's second half
int kuq_collect_device_batch(kuq_ctx *ctx, uint32_t slot, kuq_batch_result *out) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (!out) return KUQ_E_INVALID_ARG;
  CU(cudaSetDevice(ctx->device));
  Slot &s = ctx->slots[slot];
  if (s.busy) return fail(ctx, KUQ_E_STATE, "slot %u still has an unread batch", slot);
  rc = copy_results(ctx, s);
  if (rc) return rc;
  s.busy = true;
  return kuq_wait_batch(ctx, slot, out);
}

int kuq_sync_slot(kuq_ctx *ctx, uint32_t slot) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  Slot &s = ctx->slots[slot];
  CU(cudaStreamSynchronize(s.stream));
  float ms = 0;
  if (s.timed && cudaEventElapsedTime(&ms, s.ev_k0, s.ev_k1) == cudaSuccess) s.kernel_ms = ms;
  (void)cudaGetLastError();      // never leave a stale error code behind for the next CUDA user of this process
  uint32_t err = 0;
  if (ctx->d_sync_err) {
    CU(cudaMemcpy(&err, ctx->d_sync_err, 4, cudaMemcpyDeviceToHost));
    if (err) return fail(ctx, KUQ_E_STATE, "kuq_wait_flags timed out: a peer GPU never signalled (code %u)", err);
  }
  CU(cudaMemcpy(&err, reinterpret_cast<uint32_t *>(s.d_scalars + 3), 4, cudaMemcpyDeviceToHost));
  if (err == 1) return fail(ctx, KUQ_E_TAXA_OVERFLOW, "the batch exhausted the hit-table pool for reads with more than 32 distinct taxa: use smaller batches");
  if (err == 4) return batch_set_saturated(ctx);
  if (err == 5) return fail(ctx, KUQ_E_CAPACITY, "the hit lists of the batch need more run slots than the slot holds (%llu): use smaller batches", (unsigned long long)s.runs_cap);
  if (err) return fail(ctx, KUQ_E_CAPACITY, "per-batch work-unit bookkeeping overflowed (code %u): use smaller batches", err);
  return KUQ_OK;
}

int kuq_slot_device_result(kuq_ctx *ctx, uint32_t slot, kuq_device_result *out) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (!out) return KUQ_E_INVALID_ARG;
  Slot &s = ctx->slots[slot];
  out->d_call = s.d_call;
  out->d_n_windows = s.d_nwin;
  out->d_codes = s.d_codes;
  out->d_run_start = s.d_run_start;
  out->d_run_count = s.d_run_count;
  out->d_runs = reinterpret_cast<const kuq_run *>(s.d_runs.get());
  out->d_n_runs = reinterpret_cast<const uint64_t *>(s.d_scalars.get());
  return KUQ_OK;
}

int kuq_slot_stats(kuq_ctx *ctx, uint32_t slot, uint64_t *n_lookups, uint64_t *sum_probes) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  Slot &s = ctx->slots[slot];
  CU(cudaStreamSynchronize(s.stream));
  unsigned long long v[2];
  CU(cudaMemcpy(v, s.d_scalars + 4, 16, cudaMemcpyDeviceToHost));
  if (n_lookups) *n_lookups = v[0];
  if (sum_probes) *sum_probes = v[1];
  return KUQ_OK;
}

void *kuq_slot_stream(kuq_ctx *ctx, uint32_t slot) {
  if (!ctx || slot >= ctx->slots.size()) return nullptr;
  return (void *)ctx->slots[slot].stream.get();
}
uint64_t kuq_launch_count(const kuq_ctx *ctx) { return ctx ? ctx->launches : 0; }
double kuq_last_kernel_ms(kuq_ctx *ctx, uint32_t slot) {
  if (!ctx || slot >= ctx->slots.size()) return -1;
  return ctx->slots[slot].kernel_ms;
}
int kuq_last_stage_ms(kuq_ctx *ctx, uint32_t slot, double *ms3) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (!ms3) return KUQ_E_INVALID_ARG;
  Slot &s = ctx->slots[slot];
  CU(cudaStreamSynchronize(s.stream));
  float a = 0, b = 0, c = 0;
  if (s.timed) {
    cudaEventElapsedTime(&a, s.ev_k0, s.ev_stage[0]);
    cudaEventElapsedTime(&b, s.ev_stage[0], s.ev_stage[1]);
    cudaEventElapsedTime(&c, s.ev_stage[1], s.ev_k1);
  }
  (void)cudaGetLastError();
  ms3[0] = a; ms3[1] = b; ms3[2] = c;
  return KUQ_OK;
}

// ---- per-taxon results ------------------------------------------------------------------------------------------
int kuq_finish(kuq_ctx *ctx) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  ctx->units.new_file();
  return harvest_seen(ctx, false);
}

namespace {
int fetch_counts(kuq_ctx *ctx, CountsHost &h) {
  if (!ctx->finalized) return fail(ctx, KUQ_E_STATE, "nothing classified yet");
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  { int hrc = harvest_seen(ctx, false); if (hrc) return hrc; }
  ctx->snap_valid = false;
  h.n_kmers.resize(ctx->n_sketch);
  h.n_reads.resize(ctx->n_taxa);
  h.hist.resize((size_t)ctx->n_sketch * 64);
  h.dense_flag.assign(ctx->n_sketch, 1);
  h.distinct.assign(ctx->n_sketch, 0);
  CU(cudaMemcpy(h.n_kmers.data(), ctx->d_n_kmers, ctx->n_sketch * 8ull, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(h.n_reads.data(), ctx->d_n_reads, ctx->n_taxa * 8ull, cudaMemcpyDeviceToHost));
  {
    DevBuf<uint32_t> d_hist;
    CU(d_hist.alloc((uint64_t)ctx->n_sketch * 64));
    launch_register_histograms(ctx->d_regs, ctx->n_sketch, d_hist, ctx->aux);
    ctx->launches++;
    CU(cudaMemcpyAsync(h.hist.data(), d_hist, (uint64_t)ctx->n_sketch * 64 * 4, cudaMemcpyDeviceToHost, ctx->aux));
    CU(cudaStreamSynchronize(ctx->aux));
  }
  if (ctx->cfg.hll_mode == KUQ_HLL_EXACT) {
    h.exact.resize(ctx->n_sketch);
    CU(cudaMemcpy(h.exact.data(), ctx->exact.count, ctx->n_sketch * 8ull, cudaMemcpyDeviceToHost));
    if (ctx->merged_exact) h.exact = ctx->merged_exact_count;   // sums over the k-mer parts (kuq_set_exact_summary)
  } else if (ctx->cfg.hll_mode != KUQ_HLL_DENSE_ONLY) {
    if (ctx->cfg.hll_mode == KUQ_HLL_CHUNKED) {
      launch_flag_dense_global(ctx->sparse.count, ctx->d_dense_flag, ctx->n_sketch, ctx->aux);
      ctx->launches++;
    }
    DevBuf<uint32_t> d_sh;
    CU(d_sh.alloc((uint64_t)ctx->n_sketch * 64));
    CU(cudaMemsetAsync(d_sh, 0, (uint64_t)ctx->n_sketch * 64 * 4, ctx->aux));
    launch_sparse_histograms(set_keys(ctx), ctx->d_dense_flag, d_sh, ctx->aux);
    launch_sparse_histograms(kept_keys(ctx), ctx->d_dense_flag, d_sh, ctx->aux);
    ctx->launches += ctx->kept ? 2 : 1;
    h.sparse_hist.resize((size_t)ctx->n_sketch * 64);
    CU(cudaMemcpyAsync(h.sparse_hist.data(), d_sh, (uint64_t)ctx->n_sketch * 64 * 4, cudaMemcpyDeviceToHost, ctx->aux));
    CU(cudaMemcpyAsync(h.dense_flag.data(), ctx->d_dense_flag, ctx->n_sketch, cudaMemcpyDeviceToHost, ctx->aux));
    CU(cudaMemcpyAsync(h.distinct.data(), ctx->sparse.count, ctx->n_sketch * 4ull, cudaMemcpyDeviceToHost, ctx->aux));
    CU(cudaStreamSynchronize(ctx->aux));
    if (ctx->merged_summary) {             // sums over the code partitions of all GPUs (kuq_set_sparse_summary)
      h.sparse_hist = ctx->merged_hist;
      h.distinct = ctx->merged_distinct;
    }
  }
  if (&h == &ctx->snap) ctx->snap_valid = true;
  return KUQ_OK;
}
}  // namespace

namespace {
// Histogram of the merged sketch of the member taxa (dense ids with k-mers): register-value histogram of the
// register-wise max when any member is dense, else rank histogram of the union of the members' sparse code sets.
// With a cross-GPU summary installed (kuq_set_sparse_summary) the local set is one code partition: the union
// histogram of several sparse members is then a PARTIAL result the caller sums over GPUs (allow_partial).
int clade_hist(kuq_ctx *ctx, const std::vector<uint32_t> &members, uint32_t *hist64, int *is_dense, bool allow_partial) {
  const CountsHost &h = ctx->snap;
  memset(hist64, 0, 64 * sizeof(uint32_t));
  bool any_dense = ctx->cfg.hll_mode == KUQ_HLL_DENSE_ONLY;
  uint64_t sum_distinct = 0;
  for (uint32_t d : members) { any_dense |= h.dense_flag[d] != 0; sum_distinct += h.distinct[d]; }
  *is_dense = any_dense ? 1 : 0;
  if (members.empty()) return KUQ_OK;
  if (members.size() == 1 && !(allow_partial && ctx->merged_summary && !any_dense)) {
    // a clade with a single contributing taxon has that taxon's sketch
    const uint32_t d = members[0];
    memcpy(hist64, any_dense ? &h.hist[(size_t)d * 64] : &h.sparse_hist[(size_t)d * 64], 64 * sizeof(uint32_t));
    return KUQ_OK;
  }
  if (!any_dense) {
    if (ctx->merged_summary && !allow_partial)
      return fail(ctx, KUQ_E_STATE, "the sparse tier is partitioned over GPUs: sum kuq_clade_partial over the GPUs instead");
    std::vector<uint8_t> member(ctx->n_sketch, 0);
    for (uint32_t d : members) member[d] = 1;
    uint64_t cap = 1024;
    while (cap < 2 * sum_distinct + 16) cap <<= 1;
    DevBuf<uint8_t> d_member;
    DevBuf<unsigned long long> d_set;
    DevBuf<uint32_t> d_hist;
    CU(d_member.alloc(ctx->n_sketch));
    CU(d_set.alloc(cap));
    CU(d_hist.alloc(65));
    CU(cudaMemcpyAsync(d_member, member.data(), ctx->n_sketch, cudaMemcpyHostToDevice, ctx->aux));
    CU(cudaMemsetAsync(d_set, 0, cap * 8, ctx->aux));
    CU(cudaMemsetAsync(d_hist, 0, 65 * 4, ctx->aux));
    launch_sparse_union(set_keys(ctx), d_member, d_set, cap - 1, d_hist, d_hist + 64, ctx->aux);
    launch_sparse_union(kept_keys(ctx), d_member, d_set, cap - 1, d_hist, d_hist + 64, ctx->aux);
    ctx->launches += ctx->kept ? 2 : 1;
    uint32_t hist[65];
    CU(cudaMemcpyAsync(hist, d_hist, sizeof hist, cudaMemcpyDeviceToHost, ctx->aux));
    CU(cudaStreamSynchronize(ctx->aux));
    if (hist[64]) return fail(ctx, KUQ_E_CAPACITY, "internal: clade union scratch overflow");
    memcpy(hist64, hist, 64 * sizeof(uint32_t));
    return KUQ_OK;
  }
  DevBuf<uint32_t> d_members, d_hist;
  DevBuf<uint8_t> d_out;
  CU(d_members.alloc(members.size()));
  CU(d_out.alloc(HLL_M));
  CU(d_hist.alloc(64));
  CU(cudaMemcpyAsync(d_members, members.data(), members.size() * 4, cudaMemcpyHostToDevice, ctx->aux));
  launch_clade_max(ctx->d_regs, d_members, (uint32_t)members.size(), d_out, ctx->aux);
  launch_register_histograms(d_out, 1, d_hist, ctx->aux);
  ctx->launches += 2;
  CU(cudaMemcpyAsync(hist64, d_hist, 64 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->aux));
  CU(cudaStreamSynchronize(ctx->aux));
  return KUQ_OK;
}
}  // namespace

uint64_t kuq_ertl_sparse(const uint32_t *hist64, uint64_t n_observed);

int kuq_counts_size(kuq_ctx *ctx, uint32_t *n) {
  if (!ctx || !n) return KUQ_E_INVALID_ARG;
  CountsHost &h = ctx->snap;
  int rc = ctx->snap_valid ? KUQ_OK : fetch_counts(ctx, h);
  if (rc) return rc;
  uint32_t c = 0;
  for (uint32_t d = 0; d < ctx->n_taxa; d++)
    if (h.n_reads[d] || (d < ctx->n_sketch && h.n_kmers[d])) c++;
  *n = c;
  return KUQ_OK;
}

int kuq_read_counts(kuq_ctx *ctx, uint32_t *taxid, uint64_t *n_reads, uint64_t *n_kmers, uint64_t *unique,
                    uint8_t *is_sparse, uint32_t cap) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  if (ctx->spilled_pairs) return refuse_spilled(ctx, "kuq_read_counts");
  CountsHost &h = ctx->snap;
  int rc = ctx->snap_valid ? KUQ_OK : fetch_counts(ctx, h);
  if (rc) return rc;
  std::vector<std::pair<uint32_t, uint32_t>> rows;   // (taxid, dense)
  for (uint32_t d = 0; d < ctx->n_taxa; d++)
    if (h.n_reads[d] || (d < ctx->n_sketch && h.n_kmers[d])) rows.emplace_back(ctx->raw_of_dense[d], d);
  std::sort(rows.begin(), rows.end());
  if (rows.size() > cap) return fail(ctx, KUQ_E_CAPACITY, "need room for %zu rows", rows.size());
  for (size_t i = 0; i < rows.size(); i++) {
    uint32_t d = rows[i].second;
    uint64_t nk = d < ctx->n_sketch ? h.n_kmers[d] : 0;
    if (taxid) taxid[i] = rows[i].first;
    if (n_reads) n_reads[i] = h.n_reads[d];
    if (n_kmers) n_kmers[i] = nk;
    // the sketch the reference would hold: dense registers if some per-unit (or the global) sketch converted,
    // else the union of the encoded hashes (sparse tier)
    const bool exact = ctx->cfg.hll_mode == KUQ_HLL_EXACT;
    // A taxon outside the database (no sketch here) that is the call of some read, e.g. the LCA of tied hits, has a
    // READCOUNTS entry in the reference all the same: an empty sketch, which is sparse.
    const bool sparse = !exact && ctx->cfg.hll_mode != KUQ_HLL_DENSE_ONLY &&
                        (d < ctx->n_sketch ? !h.dense_flag[d] : h.n_reads[d] > 0);
    uint64_t u = 0;
    if (exact) u = d < ctx->n_sketch ? h.exact[d] : 0;     // khset size, readcounts.hpp:127-130
    else if (d < ctx->n_sketch && nk)
      u = sparse ? ertl_sparse_hist(&h.sparse_hist[(size_t)d * 64], h.distinct[d], nk)
                 : ertl_dense_hist(&h.hist[(size_t)d * 64], nk);
    if (unique) unique[i] = u;
    if (is_sparse) is_sparse[i] = sparse ? 1 : 0;
  }
  return KUQ_OK;
}

int kuq_clade_counts(kuq_ctx *ctx, const uint32_t *taxids, uint32_t n, uint64_t *n_reads, uint64_t *n_kmers,
                     uint64_t *unique) {
  if (!ctx || (!taxids && n)) return KUQ_E_INVALID_ARG;
  if (!ctx->finalized) return fail(ctx, KUQ_E_STATE, "nothing classified yet");
  if (ctx->spilled_pairs) return refuse_spilled(ctx, "kuq_clade_counts");
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  if (!ctx->snap_valid) {
    int rc = fetch_counts(ctx, ctx->snap);
    if (rc) return rc;
  }
  const CountsHost &h = ctx->snap;
  std::vector<uint32_t> members;
  uint64_t reads = 0, kmers = 0;
  for (uint32_t i = 0; i < n; i++) {
    auto it = ctx->dense_of_raw.find(taxids[i]);
    if (it == ctx->dense_of_raw.end()) continue;
    const uint32_t d = it->second;
    reads += h.n_reads[d];
    if (d < ctx->n_sketch && h.n_kmers[d]) { kmers += h.n_kmers[d]; members.push_back(d); }
  }
  uint64_t u = 0;
  if (ctx->cfg.hll_mode == KUQ_HLL_EXACT) {
    if (ctx->exact_partitioned)
      return fail(ctx, KUQ_E_STATE, "the exact k-mer set is partitioned by k-mer over contexts and this one holds one part: "
                                    "a union over a member list would be partial (use kuq_clade_counts_tree after "
                                    "kuq_set_exact_summary)");
    // the clade's container is the union of the members' k-mer sets (readcounts.hpp:76-81)
    uint64_t sum = 0;
    for (uint32_t d : members) sum += h.exact[d];
    if (members.size() == 1) {
      u = sum;
    } else if (!members.empty()) {
      std::vector<uint8_t> member(ctx->n_sketch, 0);
      for (uint32_t d : members) member[d] = 1;
      uint64_t cap = 1024;
      while (cap < 2 * sum + 16) cap <<= 1;
      DevBuf<uint8_t> d_member;
      DevBuf<unsigned long long> d_set, d_cnt;
      CU(d_member.alloc(ctx->n_sketch));
      CU(d_set.alloc(cap));
      CU(d_cnt.alloc(2));
      CU(cudaMemcpyAsync(d_member, member.data(), ctx->n_sketch, cudaMemcpyHostToDevice, ctx->aux));
      CU(cudaMemsetAsync(d_set, 0, cap * 8, ctx->aux));
      CU(cudaMemsetAsync(d_cnt, 0, 16, ctx->aux));
      launch_exact_union(set_view(ctx, ctx->exact), d_member, d_set, cap - 1, d_cnt, reinterpret_cast<uint32_t *>(d_cnt + 1), ctx->aux);
      ctx->launches++;
      unsigned long long out[2];
      CU(cudaMemcpyAsync(out, d_cnt, 16, cudaMemcpyDeviceToHost, ctx->aux));
      CU(cudaStreamSynchronize(ctx->aux));
      if (out[1]) return fail(ctx, KUQ_E_CAPACITY, "internal: clade union scratch overflow");
      u = out[0];
    }
    if (n_reads) *n_reads = reads;
    if (n_kmers) *n_kmers = kmers;
    if (unique) *unique = u;
    return KUQ_OK;
  }
  // clade sketch = merge of the members' sketches: dense as soon as one member is dense
  // (hyperloglogplus.cpp:604-621), else the union of the sparse sets (:600-603)
  uint32_t hist[64];
  int is_dense = 0;
  int rc = clade_hist(ctx, members, hist, &is_dense, /*allow_partial=*/false);
  if (rc) return rc;
  if (!members.empty()) u = is_dense ? ertl_dense_hist(hist, kmers) : kuq_ertl_sparse(hist, kmers);
  if (n_reads) *n_reads = reads;
  if (n_kmers) *n_kmers = kmers;
  if (unique) *unique = u;
  return KUQ_OK;
}

int kuq_clade_partial(kuq_ctx *ctx, const uint32_t *taxids, uint32_t n, uint64_t *n_reads, uint64_t *n_kmers, int *is_dense,
                      uint32_t *hist64) {
  if (!ctx || (!taxids && n) || !hist64 || !is_dense) return KUQ_E_INVALID_ARG;
  if (!ctx->finalized) return fail(ctx, KUQ_E_STATE, "nothing classified yet");
  if (ctx->cfg.hll_mode == KUQ_HLL_EXACT) return fail(ctx, KUQ_E_STATE, "kuq_clade_partial is about sketches (not KUQ_HLL_EXACT)");
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  if (!ctx->snap_valid) {
    int rc = fetch_counts(ctx, ctx->snap);
    if (rc) return rc;
  }
  const CountsHost &h = ctx->snap;
  std::vector<uint32_t> members;
  uint64_t reads = 0, kmers = 0;
  for (uint32_t i = 0; i < n; i++) {
    auto it = ctx->dense_of_raw.find(taxids[i]);
    if (it == ctx->dense_of_raw.end()) continue;
    const uint32_t d = it->second;
    reads += h.n_reads[d];
    if (d < ctx->n_sketch && h.n_kmers[d]) { kmers += h.n_kmers[d]; members.push_back(d); }
  }
  if (n_reads) *n_reads = reads;
  if (n_kmers) *n_kmers = kmers;
  return clade_hist(ctx, members, hist64, is_dense, /*allow_partial=*/true);
}

// All clades at once (kuq.h).  Host: one pass up the tree for the counters and for which clades are dense / sparse /
// carried by a single taxon; device: kuq_clades.cu.
int kuq_clade_counts_tree(kuq_ctx *ctx, const uint32_t *taxids, uint32_t n, uint64_t *n_reads, uint64_t *n_kmers,
                          uint64_t *unique) {
  if (!ctx || (!taxids && n)) return KUQ_E_INVALID_ARG;
  if (!ctx->finalized) return fail(ctx, KUQ_E_STATE, "nothing classified yet");
  if (ctx->spilled_pairs) return refuse_spilled(ctx, "kuq_clade_counts_tree");
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  if (!ctx->snap_valid) {
    int rc = fetch_counts(ctx, ctx->snap);
    if (rc) return rc;
  }
  const CountsHost &h = ctx->snap;
  const uint32_t NT = ctx->n_taxa, NS = ctx->n_sketch;
  const std::vector<uint32_t> &par = ctx->parent_dense;
  const uint32_t NONE = 0xFFFFFFFFu;
  auto has_kmers = [&](uint32_t d) { return d < NS && h.n_kmers[d] != 0; };
  // ---- the nodes on a path from a counted taxon to its root, children before parents ----------------------------
  std::vector<uint32_t> cid(NT, NONE), nodes;
  for (uint32_t d = 0; d < NT; d++) {
    if (!(h.n_reads[d] || has_kmers(d))) continue;
    for (uint32_t x = d; cid[x] == NONE;) {
      cid[x] = (uint32_t)nodes.size();
      nodes.push_back(x);
      if (x == 0 || par[x] == 0) break;
      x = par[x];
    }
  }
  const uint32_t NC = (uint32_t)nodes.size();
  std::vector<uint32_t> parent_c(NC, NONE), depth_c(NC, 0), order(NC);
  for (uint32_t c = 0; c < NC; c++) {
    const uint32_t x = nodes[c];
    if (x != 0 && par[x] != 0) parent_c[c] = cid[par[x]];
  }
  {  // depth in the compact forest (roots 0); a node's chain was appended root-last, so walk it explicitly
    std::vector<uint32_t> chain;
    std::vector<uint8_t> done(NC, 0);
    for (uint32_t c = 0; c < NC; c++) {
      chain.clear();
      uint32_t x = c;
      while (x != NONE && !done[x]) { chain.push_back(x); x = parent_c[x]; }
      uint32_t d = x == NONE ? 0 : depth_c[x] + 1;
      for (size_t i = chain.size(); i-- > 0;) { depth_c[chain[i]] = d++; done[chain[i]] = 1; }
    }
    for (uint32_t c = 0; c < NC; c++) order[c] = c;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return depth_c[a] > depth_c[b]; });
  }
  const bool all_dense = ctx->cfg.hll_mode == KUQ_HLL_DENSE_ONLY;
  std::vector<uint64_t> c_reads(NC, 0), c_kmers(NC, 0);
  std::vector<uint32_t> c_members(NC, 0), c_single(NC, NONE);
  std::vector<uint8_t> c_dense(NC, 0);
  for (uint32_t c = 0; c < NC; c++) {
    const uint32_t d = nodes[c];
    c_reads[c] = h.n_reads[d];
    if (has_kmers(d)) { c_kmers[c] = h.n_kmers[d]; c_members[c] = 1; c_single[c] = d; c_dense[c] = all_dense || h.dense_flag[d]; }
  }
  for (uint32_t c : order) {
    const uint32_t q = parent_c[c];
    if (q == NONE) continue;
    c_reads[q] += c_reads[c];
    c_kmers[q] += c_kmers[c];
    if (c_members[c]) {
      if (c_members[q] == 0) c_single[q] = c_single[c];
      c_members[q] += c_members[c];
      c_dense[q] |= c_dense[c];
    }
  }
  // ---- what was asked for ---------------------------------------------------------------------------------------
  std::vector<uint32_t> req(n, NONE);
  std::vector<uint8_t> wanted(NC, 0);
  for (uint32_t i = 0; i < n; i++) {
    auto it = ctx->dense_of_raw.find(taxids[i]);
    if (it != ctx->dense_of_raw.end() && cid[it->second] != NONE) { req[i] = cid[it->second]; wanted[req[i]] = 1; }
  }
  std::vector<uint64_t> c_unique(NC, 0);
  const bool exact = ctx->cfg.hll_mode == KUQ_HLL_EXACT;
  const bool per_clade = !exact && ctx->merged_summary;
  bool sparse_fallback = false;
  std::vector<uint32_t> dense_list, sparse_multi;          // compact ids
  // ---- exact counting: every clade from the books of one sort (exact_books), or from their sums over the parts ------
  if (exact) {
    std::vector<long long> own;
    const std::vector<long long> *books = &ctx->merged_books;
    if (!ctx->merged_exact) {
      if (ctx->exact_partitioned)
        return fail(ctx, KUQ_E_STATE, "the exact k-mer set is partitioned by k-mer over contexts: install the books summed "
                                      "over all parts first (kuq_exact_summary, kuq_set_exact_summary)");
      int rc = exact_books(ctx, own);
      if (rc) return rc;
      books = &own;
    }
    std::vector<long long> acc(NC, 0);
    for (uint32_t c = 0; c < NC; c++) acc[c] = (*books)[nodes[c]];
    for (uint32_t c : order)
      if (parent_c[c] != NONE) acc[parent_c[c]] += acc[c];
    for (uint32_t c = 0; c < NC; c++) c_unique[c] = (uint64_t)std::max<long long>(acc[c], 0);
  }
  if (!per_clade && !exact) {
    for (uint32_t c = 0; c < NC; c++) {
      if (c_members[c] == 0) continue;
      if (c_members[c] == 1) {
        if (!wanted[c]) continue;
        const uint32_t d = c_single[c];
        c_unique[c] = c_dense[c] ? ertl_dense_hist(&h.hist[(size_t)d * 64], c_kmers[c]) : kuq_ertl_sparse(&h.sparse_hist[(size_t)d * 64], c_kmers[c]);
      } else if (c_dense[c]) {
        if (wanted[c]) dense_list.push_back(c);
      } else {
        sparse_multi.push_back(c);                          // needed for the sums up the tree whether asked for or not
      }
    }
  }
  // ---- dense clades: register-wise max of the members, in chunks ---------------------------------------------------
  if (!dense_list.empty()) {
    std::vector<uint32_t> dix(NC, NONE);
    for (uint32_t i = 0; i < dense_list.size(); i++) dix[dense_list[i]] = i;
    std::vector<uint32_t> offs(dense_list.size() + 1, 0), mem;
    for (int pass = 0; pass < 2; pass++) {
      std::vector<uint32_t> fill(offs.begin(), offs.end() - 1);
      for (uint32_t c = 0; c < NC; c++) {
        if (!has_kmers(nodes[c])) continue;
        for (uint32_t x = c; x != NONE; x = parent_c[x])
          if (dix[x] != NONE) { if (pass == 0) offs[dix[x] + 1]++; else mem[fill[dix[x]]++] = nodes[c]; }
      }
      if (pass == 0) { for (size_t i = 1; i < offs.size(); i++) offs[i] += offs[i - 1]; mem.resize(offs.back()); }
    }
    const uint32_t CH = 8192;                                // clades per launch: 32 MB of folded registers
    DevBuf<uint32_t> d_offs, d_mem, d_hist;
    DevBuf<uint8_t> d_out;
    std::vector<uint32_t> hist((size_t)CH * 64), loc;
    CU(d_offs.alloc(CH + 1));
    CU(d_mem.alloc(std::max<size_t>(mem.size(), 1)));
    CU(d_out.alloc((uint64_t)CH * HLL_M));
    CU(d_hist.alloc((uint64_t)CH * 64));
    CU(cudaMemcpyAsync(d_mem, mem.data(), mem.size() * 4, cudaMemcpyHostToDevice, ctx->aux));
    for (uint32_t a = 0; a < dense_list.size(); a += CH) {
      const uint32_t m = std::min<uint32_t>(CH, (uint32_t)dense_list.size() - a);
      loc.assign(offs.begin() + a, offs.begin() + a + m + 1);           // absolute offsets into d_mem
      CU(cudaMemcpyAsync(d_offs, loc.data(), (m + 1) * 4ull, cudaMemcpyHostToDevice, ctx->aux));
      launch_clade_max_batch(ctx->d_regs, d_offs, d_mem, m, d_out, ctx->aux);
      launch_register_histograms(d_out, m, d_hist, ctx->aux);
      ctx->launches += 2;
      CU(cudaMemcpyAsync(hist.data(), d_hist, (uint64_t)m * 64 * 4, cudaMemcpyDeviceToHost, ctx->aux));
      CU(cudaStreamSynchronize(ctx->aux));
      for (uint32_t i = 0; i < m; i++) {
        const uint32_t c = dense_list[a + i];
        c_unique[c] = ertl_dense_hist(&hist[(size_t)i * 64], c_kmers[c]);
      }
    }
  }
  // ---- sparse clades with several members: distinct codes of every subtree from one sort ------------------------------
  if (!sparse_multi.empty()) {
    std::vector<int32_t> sid(NC, -1);
    for (uint32_t i = 0; i < sparse_multi.size(); i++) sid[sparse_multi[i]] = (int32_t)i;
    // preorder numbers: children lists from the parent pointers, explicit stack
    std::vector<uint32_t> first_child(NC + 1, 0), child(NC), pre(NC, NONE), node_of_pre(NC, 0);
    for (uint32_t c = 0; c < NC; c++) if (parent_c[c] != NONE) first_child[parent_c[c] + 1]++;
    for (uint32_t c = 0; c < NC; c++) first_child[c + 1] += first_child[c];
    {
      std::vector<uint32_t> fill(first_child.begin(), first_child.end() - 1);
      for (uint32_t c = 0; c < NC; c++) if (parent_c[c] != NONE) child[fill[parent_c[c]]++] = c;
      std::vector<uint32_t> stack;
      uint32_t counter = 0;
      for (uint32_t r = 0; r < NC; r++) {
        if (parent_c[r] != NONE) continue;
        stack.push_back(r);
        while (!stack.empty()) {
          const uint32_t x = stack.back();
          stack.pop_back();
          pre[x] = counter;
          node_of_pre[counter++] = x;
          for (uint32_t i = first_child[x]; i < first_child[x + 1]; i++) stack.push_back(child[i]);
        }
      }
    }
    std::vector<uint32_t> pre_of_taxon(NS, NONE);
    uint64_t n_keys = 0;
    for (uint32_t c = 0; c < NC; c++) {
      const uint32_t d = nodes[c];
      if (d < NS) { pre_of_taxon[d] = pre[c]; if (has_kmers(d) && !h.dense_flag[d]) n_keys += h.distinct[d]; }
    }
    std::vector<uint32_t> dup(sparse_multi.size() * 64, 0);
    int src = 0;
    cudaError_t ce = cudaSuccess;
    {
      DevBuf<uint32_t> d_pre, d_nop, d_par, d_dep, d_dup;
      DevBuf<int32_t> d_sid;
      CU(d_pre.alloc(NS)); CU(d_nop.alloc(NC)); CU(d_par.alloc(NC)); CU(d_dep.alloc(NC)); CU(d_sid.alloc(NC));
      CU(d_dup.alloc(sparse_multi.size() * 64));
      CU(cudaMemcpyAsync(d_pre, pre_of_taxon.data(), NS * 4ull, cudaMemcpyHostToDevice, ctx->aux));
      CU(cudaMemcpyAsync(d_nop, node_of_pre.data(), NC * 4ull, cudaMemcpyHostToDevice, ctx->aux));
      CU(cudaMemcpyAsync(d_par, parent_c.data(), NC * 4ull, cudaMemcpyHostToDevice, ctx->aux));
      CU(cudaMemcpyAsync(d_dep, depth_c.data(), NC * 4ull, cudaMemcpyHostToDevice, ctx->aux));
      CU(cudaMemcpyAsync(d_sid, sid.data(), NC * 4ull, cudaMemcpyHostToDevice, ctx->aux));
      CU(cudaMemsetAsync(d_dup, 0, sparse_multi.size() * 64 * 4ull, ctx->aux));
      src = sparse_clade_dups(set_keys(ctx), kept_keys(ctx), ctx->d_dense_flag, n_keys, d_pre, d_nop, d_par, d_dep, d_sid, d_dup,
                              ctx->n_sm, ctx->aux);
      ctx->launches += 3;
      if (src == 0) {
        ce = cudaMemcpyAsync(dup.data(), d_dup, dup.size() * 4, cudaMemcpyDeviceToHost, ctx->aux);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(ctx->aux);
      }
    }
    if (src == 2 || ce != cudaSuccess) return fail(ctx, KUQ_E_CUDA, "clade roll-up (sparse tier) failed: %s", cudaGetErrorString(cudaGetLastError()));
    if (src == 1) {
      sparse_fallback = true;                                // no room for the sort: one union per clade instead
    } else {
      // rank histogram of every sparse subtree: own codes + children's − the pairs booked at the node
      std::vector<std::vector<uint32_t>> H(NC);
      for (uint32_t c : order) {
        if (c_members[c] == 0 || c_dense[c]) continue;
        std::vector<uint32_t> &hc = H[c];
        if (hc.empty()) hc.assign(64, 0);
        const uint32_t d = nodes[c];
        if (has_kmers(d)) for (int r = 0; r < 64; r++) hc[r] += h.sparse_hist[(size_t)d * 64 + r];
        if (sid[c] >= 0) for (int r = 0; r < 64; r++) hc[r] -= dup[(size_t)sid[c] * 64 + r];
        if (wanted[c] && c_members[c] > 1) c_unique[c] = kuq_ertl_sparse(hc.data(), c_kmers[c]);
        const uint32_t q = parent_c[c];
        if (q != NONE && !c_dense[q]) {
          std::vector<uint32_t> &hq = H[q];
          if (hq.empty()) hq.assign(64, 0);
          for (int r = 0; r < 64; r++) hq[r] += hc[r];
        }
        std::vector<uint32_t>().swap(hc);
      }
    }
  }
  // ---- exact counting / partitioned sparse tier / no memory for the sort: one merge per clade ------------------------
  if (per_clade || sparse_fallback) {
    std::vector<std::vector<uint32_t>> lists(NC);
    for (uint32_t c = 0; c < NC; c++) {
      if (!(h.n_reads[nodes[c]] || has_kmers(nodes[c]))) continue;
      for (uint32_t x = c; x != NONE; x = parent_c[x])
        if (wanted[x] && (per_clade || (c_members[x] > 1 && !c_dense[x]))) lists[x].push_back(ctx->raw_of_dense[nodes[c]]);
    }
    for (uint32_t c = 0; c < NC; c++) {
      if (lists[c].empty()) continue;
      uint64_t r = 0, k = 0, u = 0;
      int rc = kuq_clade_counts(ctx, lists[c].data(), (uint32_t)lists[c].size(), &r, &k, &u);
      if (rc) return rc;
      c_unique[c] = u;
    }
  }
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t c = req[i];
    if (n_reads) n_reads[i] = c == NONE ? 0 : c_reads[c];
    if (n_kmers) n_kmers[i] = c == NONE ? 0 : c_kmers[c];
    if (unique) unique[i] = c == NONE ? 0 : c_unique[c];
  }
  return KUQ_OK;
}

uint64_t kuq_ertl_dense_hist(const uint32_t *hist64, uint64_t n_observed) { return ertl_dense_hist(hist64, n_observed); }

int kuq_get_registers(kuq_ctx *ctx, uint32_t taxid, uint8_t *regs) {
  if (!ctx || !regs) return KUQ_E_INVALID_ARG;
  if (!ctx->finalized) return fail(ctx, KUQ_E_STATE, "nothing classified yet");
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  memset(regs, 0, HLL_M);
  auto it = ctx->dense_of_raw.find(taxid);
  if (it == ctx->dense_of_raw.end() || it->second >= ctx->n_sketch) return KUQ_OK;
  CU(cudaMemcpy(regs, ctx->d_regs + (size_t)it->second * HLL_M, HLL_M, cudaMemcpyDeviceToHost));
  return KUQ_OK;
}

int kuq_state_ptrs_get(kuq_ctx *ctx, kuq_state_ptrs *out) {
  if (!ctx || !out) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  out->d_regs = ctx->d_regs;
  out->regs_bytes = (uint64_t)ctx->n_sketch * HLL_M;
  out->d_n_kmers = reinterpret_cast<uint64_t *>(ctx->d_n_kmers.get());
  out->d_n_reads = reinterpret_cast<uint64_t *>(ctx->d_n_reads.get());
  out->d_dense_flag = ctx->d_dense_flag;
  out->n_sketch = ctx->n_sketch;
  out->n_taxa = ctx->n_taxa;
  return KUQ_OK;
}

int kuq_unit_table_rows(kuq_ctx *ctx, uint32_t *rows) {
  if (!ctx || !rows) return KUQ_E_INVALID_ARG;
  int rc = finalize(ctx);
  if (rc) return rc;
  *rows = (uint32_t)unit_table_rows(ctx);
  return KUQ_OK;
}

int kuq_sparse_export(kuq_ctx *ctx, uint64_t *d_keys_out, uint64_t cap, uint64_t *n) {
  if (!ctx || !n) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  *n = 0;
  if (!ctx->sparse.slots) return KUQ_OK;                    // KUQ_HLL_DENSE_ONLY: no sparse tier
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  rc = harvest_seen(ctx, false);
  if (rc) return rc;
  return export_items(ctx, reinterpret_cast<unsigned long long *>(d_keys_out), cap, n, "keys",
                      [ctx](unsigned long long *out, uint64_t c, unsigned long long *d_n) {
                        for (const KeySource &src : {set_keys(ctx), kept_keys(ctx)}) launch_sparse_export(src, ctx->d_dense_flag, out, c, d_n, ctx->aux);
                        ctx->launches += ctx->kept ? 2 : 1;
                      });
}

// ---- database sharded over GPUs: who counts, step flags, partitioned merge of the sparse tier ---------------------
int kuq_set_shard_counting(kuq_ctx *ctx, int on) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  for (auto &s : ctx->slots)
    if (s.busy) return fail(ctx, KUQ_E_STATE, "cannot change while a batch is in flight");
  ctx->shard_counting = on != 0;
  return KUQ_OK;
}

// ---- a database larger than HBM: ranges streamed from pinned host memory, copy overlapped with the lookups -------------
extern "C++" {
namespace {
uint32_t host_hash_u32(uint32_t x) {                        // == hash_u32 of kuq_kernels.cu
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}
void stream_close(kuq_ctx *ctx) {
  for (auto &b : ctx->sbuf) b = kuq_ctx::StreamBuf();
  ctx->copy_stream.reset();
  ctx->d_stream_missing.reset();
  ctx->d_stream_land.reset();
  if (ctx->stream_open) ctx->dbs.clear();
  ctx->stream_open = false;
}
}  // namespace
}  // extern "C++"

int kuq_stream_open(kuq_ctx *ctx, uint32_t k, uint32_t nt, uint32_t idx_type, uint64_t max_records, uint64_t max_bins) {
  if (!ctx || !max_records || !max_bins) return KUQ_E_INVALID_ARG;
  if (k > 31) return fail(ctx, KUQ_E_UNSUPPORTED_K, "k = %u: k-mers up to 31 bases are supported", k);
  if (nt < 1 || nt > 15 || nt > k || (idx_type != 1 && idx_type != 2)) return fail(ctx, KUQ_E_INVALID_ARG, "bad index parameters");
  if (ctx->universe.empty()) return fail(ctx, KUQ_E_STATE, "declare the taxids of the whole database first (kuq_set_db_taxid_universe)");
  if (!ctx->tax_set) return fail(ctx, KUQ_E_STATE, "no taxonomy set");
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));   // a re-open frees the buffers they may still read
  { int hrc = harvest_seen(ctx, false, true); if (hrc) return hrc; }
  free_db(ctx);
  stream_close(ctx);
  ctx->k = k;
  ctx->dbs.emplace_back();
  StagedDb &db = ctx->dbs[0];
  db.range.nt = nt; db.range.idx_type = idx_type;
  db.taxids = ctx->universe;
  std::sort(db.taxids.begin(), db.taxids.end());
  db.taxids.erase(std::unique(db.taxids.begin(), db.taxids.end()), db.taxids.end());
  db.counts.assign(db.taxids.size(), 0);
  int rc = finalize(ctx);
  if (rc) { ctx->dbs.clear(); return rc; }
  // device table taxid → dense id over the whole universe (what collect_taxids builds per staged range otherwise)
  uint32_t cap = 1u << 16;
  while ((uint64_t)cap < 4ull * db.taxids.size()) cap <<= 1;
  std::vector<uint32_t> keys(cap, 0), dense(cap, 0);
  for (uint32_t t : db.taxids) {
    uint32_t slot = host_hash_u32(t) & (cap - 1);
    while (keys[slot]) slot = (slot + 1) & (cap - 1);
    keys[slot] = t + 1;
    dense[slot] = ctx->dense_of_raw[t];
  }
  CU(db.d_tx_keys.alloc(cap));
  CU(db.d_tx_dense.alloc(cap));
  CU(cudaMemcpy(db.d_tx_keys, keys.data(), cap * 4ull, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(db.d_tx_dense, dense.data(), cap * 4ull, cudaMemcpyHostToDevice));
  db.tx_cap = cap;
  db.remapped = true;                            // each range is remapped as it arrives
  CU(ctx->copy_stream.alloc(cudaStreamNonBlocking));
  CU(ctx->d_stream_missing.alloc(1));
  CU(cudaMemset(ctx->d_stream_missing, 0, 4));
  for (auto &b : ctx->sbuf) {
    CU(b.d_pairs.alloc(max_records * 12 + SLACK));
    CU(b.d_offsets.alloc(max_bins + 1));
    CU(b.ready.alloc(cudaEventDisableTiming));
  }
  ctx->stream_pair_sz = (2 * k + 7) / 8 + 4;     // the file's record size: key_len + 4 (krakendb.cpp:76,176)
  ctx->stream_land_rec = 0;
  if (ctx->stream_pair_sz != 12) {               // k <= 28: one landing zone, the pieces of both buffers pass through in turn
    ctx->stream_land_rec = std::min(landing_records(ctx->stream_pair_sz), max_records);
    CU(ctx->d_stream_land.alloc(ctx->stream_land_rec * ctx->stream_pair_sz + SLACK));
  }
  ctx->stream_cap_records = max_records;
  ctx->stream_cap_bins = max_bins;
  ctx->stream_open = true;
  return KUQ_OK;
}

int kuq_stream_load(kuq_ctx *ctx, uint32_t buf, const void *host_records, uint64_t n_records, const uint64_t *host_offsets,
                    uint64_t bin_lo, uint64_t bin_hi) {
  if (!ctx || buf > 1 || !host_offsets || (!host_records && n_records)) return KUQ_E_INVALID_ARG;
  if (!ctx->stream_open) return fail(ctx, KUQ_E_STATE, "kuq_stream_open first");
  if (bin_lo >= bin_hi || bin_hi - bin_lo > ctx->stream_cap_bins || n_records > ctx->stream_cap_records)
    return fail(ctx, KUQ_E_CAPACITY, "range of %llu records / %llu bins exceeds the stream buffers", (unsigned long long)n_records,
                (unsigned long long)(bin_hi - bin_lo));
  CU(cudaSetDevice(ctx->device));
  kuq_ctx::StreamBuf &b = ctx->sbuf[buf];
  if (!b.d_pairs) return fail(ctx, KUQ_E_STATE, "the range buffers were released (kuq_stream_close): kuq_stream_open first");
  // whoever still reads this buffer was queued before this call: the copy waits for the slots' streams as they stand
  if (ctx->seen_dirty) { int hrc = harvest_seen(ctx, false); if (hrc) return hrc; }
  for (auto &s : ctx->slots) {
    CU(cudaEventRecord(s.ev_sync, s.stream));
    CU(cudaStreamWaitEvent(ctx->copy_stream, s.ev_sync, 0));
  }
  if (ctx->stream_pair_sz == 12) {
    if (n_records) CU(cudaMemcpyAsync(b.d_pairs, host_records, n_records * 12, cudaMemcpyHostToDevice, ctx->copy_stream));
  } else {
    // records shorter than 12 bytes: piece by piece through the landing zone, each piece widened in stream order behind
    // its copy, so the next piece's copy waits for that (on the device, like everything else here)
    const uint64_t sz = ctx->stream_pair_sz;
    for (uint64_t r = 0; r < n_records; r += ctx->stream_land_rec) {
      const uint64_t n = std::min(ctx->stream_land_rec, n_records - r);
      CU(cudaMemcpyAsync(ctx->d_stream_land, (const uint8_t *)host_records + r * sz, n * sz, cudaMemcpyHostToDevice, ctx->copy_stream));
      launch_widen_records(ctx->d_stream_land, n, (uint32_t)(sz - 4), b.d_pairs + r * 12, ctx->copy_stream);
      ctx->launches++;
    }
    CU(cudaGetLastError());
  }
  CU(cudaMemcpyAsync(b.d_offsets, host_offsets, (bin_hi - bin_lo + 1) * 8, cudaMemcpyHostToDevice, ctx->copy_stream));
  const StagedDb &db = ctx->dbs[0];
  launch_remap_values(b.d_pairs, n_records, db.d_tx_keys, db.d_tx_dense, db.tx_cap - 1, ctx->d_stream_missing, kmer_mask(ctx->k),
                      ctx->copy_stream);
  ctx->launches++;
  CU(cudaEventRecord(b.ready, ctx->copy_stream));
  b.range = DbRange{b.d_pairs, b.d_offsets, n_records, host_offsets[0], bin_lo, bin_hi, db.range.nt, db.range.idx_type};
  b.loaded = true;
  return KUQ_OK;
}

int kuq_stream_use(kuq_ctx *ctx, uint32_t buf) {
  if (!ctx || buf > 1) return KUQ_E_INVALID_ARG;
  if (!ctx->stream_open || !ctx->sbuf[buf].loaded) return fail(ctx, KUQ_E_STATE, "stream buffer %u holds no range", buf);
  CU(cudaSetDevice(ctx->device));
  if (ctx->seen_dirty) { int hrc = harvest_seen(ctx, false); if (hrc) return hrc; }
  kuq_ctx::StreamBuf &b = ctx->sbuf[buf];
  for (auto &s : ctx->slots) CU(cudaStreamWaitEvent(s.stream, b.ready, 0));
  ctx->dbs[0].range = b.range;
  return KUQ_OK;
}

int kuq_stream_close(kuq_ctx *ctx) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  if (!ctx->stream_open) return KUQ_OK;
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));   // the lookups that read the buffers
  CU(cudaStreamSynchronize(ctx->copy_stream));
  { int hrc = harvest_seen(ctx, false, true); if (hrc) return hrc; }  // flags in the records go before the records do
  for (auto &b : ctx->sbuf) b = kuq_ctx::StreamBuf();
  ctx->d_stream_land.reset();
  DbRange &r = ctx->dbs[0].range;
  r.pairs = nullptr; r.offsets = nullptr;
  r.key_ct = 0;
  return KUQ_OK;
}

int kuq_stream_check(kuq_ctx *ctx) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  if (!ctx->stream_open) return KUQ_OK;
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->copy_stream));
  uint32_t missing = 0;
  CU(cudaMemcpy(&missing, ctx->d_stream_missing, 4, cudaMemcpyDeviceToHost));
  if (missing) return fail(ctx, KUQ_E_STATE, "a streamed range holds a taxid outside the declared universe");
  return KUQ_OK;
}

int kuq_host_register(void *p, uint64_t bytes) {
  if (!p || !bytes) return KUQ_E_INVALID_ARG;
  // portable: the memory counts as pinned for every device, so each GPU streaming its ranges from one mapping overlaps
  // its copies with its lookups
  if (cudaHostRegister(p, bytes, cudaHostRegisterPortable) == cudaSuccess) return KUQ_OK;
  (void)cudaGetLastError();
  // a read-only mapping (mmap PROT_READ of database.kdb) can only be pinned read-only
  if (cudaHostRegister(p, bytes, cudaHostRegisterPortable | cudaHostRegisterReadOnly) == cudaSuccess) return KUQ_OK;
  (void)cudaGetLastError();
  return KUQ_E_CUDA;
}
int kuq_host_unregister(void *p) {
  if (!p) return KUQ_E_INVALID_ARG;
  if (cudaHostUnregister(p) != cudaSuccess) { (void)cudaGetLastError(); return KUQ_E_CUDA; }
  return KUQ_OK;
}

// Several GPUs in ONE process (the drop-in `classify` with replicas): fold the per-taxon state of `src` into `dst`.
// sets = false folds the counters, registers and dense flags only (kuq_merge_counters_into).
static int merge_into(kuq_ctx *dst, kuq_ctx *src, bool sets);
int kuq_merge_into(kuq_ctx *dst, kuq_ctx *src) { return merge_into(dst, src, true); }
int kuq_merge_counters_into(kuq_ctx *dst, kuq_ctx *src) { return merge_into(dst, src, false); }

static int merge_into(kuq_ctx *dst, kuq_ctx *src, bool sets) {
  kuq_ctx *ctx = dst;
  if (!dst || !src || dst == src) return KUQ_E_INVALID_ARG;
  if (!src->finalized) return KUQ_OK;                       // src never classified anything: nothing to add
  if (!dst->finalized) return fail(ctx, KUQ_E_STATE, "the destination context has not classified anything yet");
  if (dst->n_taxa != src->n_taxa || dst->n_sketch != src->n_sketch || dst->raw_of_dense != src->raw_of_dense ||
      dst->cfg.hll_mode != src->cfg.hll_mode)
    return fail(ctx, KUQ_E_STATE, "the contexts number their taxa differently (different database / taxonomy / HLL mode)");
  const bool exact = dst->cfg.hll_mode == KUQ_HLL_EXACT;
  if (exact && sets && (dst->spilled_pairs || src->spilled_pairs)) {
    int rc = refuse_spilled(dst->spilled_pairs ? dst : src, "kuq_merge_into");
    if (!dst->spilled_pairs) dst->err = src->err;
    return rc;
  }
  // src: flagged records → its set (skipping what dst already knows to be dense is a refinement left out)
  CU(cudaSetDevice(src->device));
  for (auto &s : src->slots) CU(cudaStreamSynchronize(s.stream));
  { int rc = harvest_seen(src, false); if (rc) { dst->err = src->err; return rc; } }
  uint64_t n_keys = 0;
  DevBuf<uint64_t> d_keys_src;                   // on src's device
  if (src->sparse.slots && !exact && sets) {
    int rc = kuq_sparse_export(src, nullptr, 0, &n_keys);
    if (rc) { dst->err = src->err; return rc; }
    if (n_keys) {
      if (d_keys_src.alloc(n_keys) != cudaSuccess) { (void)cudaGetLastError(); return fail(ctx, KUQ_E_NOMEM, "no room for %llu keys", (unsigned long long)n_keys); }
      uint64_t n2 = 0;
      rc = kuq_sparse_export(src, d_keys_src, n_keys, &n2);
      if (rc) { dst->err = src->err; return rc; }
      n_keys = n2;
    }
  }
  CU(cudaSetDevice(dst->device));
  for (auto &s : dst->slots) CU(cudaStreamSynchronize(s.stream));
  // the imported keys may duplicate keys of dst's kept records: dst's record tier moves into its set first
  { int rc = harvest_seen(dst, false, true); if (rc) return rc; }
  dst->snap_valid = false;
  dst->merged_summary = false;
  dst->merged_exact = false;
  {
    DevBuf<uint8_t> t_regs, t_dense;
    DevBuf<unsigned long long> t_nk, t_nr;
    const uint64_t reg_bytes = (uint64_t)dst->n_sketch * HLL_M;
    CU(t_regs.alloc(reg_bytes));
    CU(t_dense.alloc(dst->n_sketch));
    CU(t_nk.alloc(dst->n_sketch));
    CU(t_nr.alloc(dst->n_taxa));
    CU(cudaMemcpyPeer(t_regs, dst->device, src->d_regs, src->device, reg_bytes));
    CU(cudaMemcpyPeer(t_dense, dst->device, src->d_dense_flag, src->device, dst->n_sketch));
    CU(cudaMemcpyPeer(t_nk, dst->device, src->d_n_kmers, src->device, dst->n_sketch * 8ull));
    CU(cudaMemcpyPeer(t_nr, dst->device, src->d_n_reads, src->device, dst->n_taxa * 8ull));
    launch_merge_state(dst->d_regs, t_regs, dst->d_n_kmers, t_nk, dst->n_sketch, dst->d_n_reads, t_nr, dst->n_taxa, dst->d_dense_flag,
                       t_dense, dst->aux);
    dst->launches++;
    CU(cudaStreamSynchronize(dst->aux));
  }
  if (exact) return sets ? merge_exact_pairs(dst, src) : KUQ_OK;
  int rc = KUQ_OK;
  if (n_keys && dst->sparse.slots) {
    DevBuf<uint64_t> d_keys_dst;
    if (d_keys_dst.alloc(n_keys) != cudaSuccess) { (void)cudaGetLastError(); return fail(ctx, KUQ_E_NOMEM, "no room for %llu keys", (unsigned long long)n_keys); }
    CU(cudaMemcpyPeer(d_keys_dst, dst->device, d_keys_src, src->device, n_keys * 8));
    rc = kuq_sparse_import(dst, d_keys_dst, n_keys);        // grows dst's set first when the keys need room
  }
  return rc;
}

int kuq_enable_peer_access(kuq_ctx *ctx, kuq_ctx *peer) {
  if (!ctx || !peer) return KUQ_E_INVALID_ARG;
  if (ctx->device == peer->device) return KUQ_OK;
  CU(cudaSetDevice(ctx->device));
  int can = 0;
  CU(cudaDeviceCanAccessPeer(&can, ctx->device, peer->device));
  if (!can) return fail(ctx, KUQ_E_STATE, "device %d cannot map the memory of device %d", ctx->device, peer->device);
  cudaError_t e = cudaDeviceEnablePeerAccess(peer->device, 0);
  if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(ctx, KUQ_E_CUDA, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e));
  (void)cudaGetLastError();
  return KUQ_OK;
}

int kuq_set_stats(kuq_ctx *ctx, int on) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  ctx->extra_flags = on ? KUQ_F_STATS : 0u;
  return KUQ_OK;
}

int kuq_signal_peers(kuq_ctx *ctx, uint32_t slot, uint64_t *const *d_flag_peers, uint32_t n_peers, uint32_t my_index,
                     uint64_t value) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (!d_flag_peers || n_peers == 0 || n_peers > 8 || my_index >= 8) return fail(ctx, KUQ_E_INVALID_ARG, "1..8 peers");
  CU(cudaSetDevice(ctx->device));
  launch_signal_peers(reinterpret_cast<unsigned long long *const *>(d_flag_peers), n_peers, my_index, value, ctx->slots[slot].stream);
  ctx->launches++;
  CU(cudaGetLastError());
  return KUQ_OK;
}

int kuq_wait_flags(kuq_ctx *ctx, uint32_t slot, const uint64_t *d_flags, uint32_t n, uint64_t value, uint32_t timeout_ms) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (!d_flags || n == 0 || n > 32) return fail(ctx, KUQ_E_INVALID_ARG, "1..32 flags");
  CU(cudaSetDevice(ctx->device));
  if (!ctx->d_sync_err) {
    CU(ctx->d_sync_err.alloc(1));
    CU(cudaMemset(ctx->d_sync_err, 0, 4));
  }
  launch_wait_flags(reinterpret_cast<const unsigned long long *>(d_flags), n, value, (unsigned long long)(timeout_ms ? timeout_ms : 20000) * 1000000ull,
                    ctx->d_sync_err, ctx->slots[slot].stream);
  ctx->launches++;
  CU(cudaGetLastError());
  return KUQ_OK;
}

static int export_partitioned(kuq_ctx *ctx, uint32_t n_parts, uint64_t *d_keys_out, uint64_t cap, uint64_t *counts, uint64_t **alloc_out);

int kuq_sparse_export_partitioned(kuq_ctx *ctx, uint32_t n_parts, uint64_t *d_keys_out, uint64_t cap, uint64_t *counts) {
  return export_partitioned(ctx, n_parts, d_keys_out, cap, counts, nullptr);
}
int kuq_sparse_export_partitioned_alloc(kuq_ctx *ctx, uint32_t n_parts, uint64_t **d_keys_out, uint64_t *counts) {
  if (!d_keys_out) return KUQ_E_INVALID_ARG;
  *d_keys_out = nullptr;
  return export_partitioned(ctx, n_parts, nullptr, 0, counts, d_keys_out);
}

static int export_partitioned(kuq_ctx *ctx, uint32_t n_parts, uint64_t *d_keys_out, uint64_t cap, uint64_t *counts, uint64_t **alloc_out) {
  if (!ctx || !counts || n_parts == 0 || n_parts > 8) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  for (uint32_t j = 0; j < n_parts; j++) counts[j] = 0;
  if (!ctx->sparse.slots) return KUQ_OK;
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  if (ctx->keep_dirty) { rc = settle_kept(ctx); if (rc) return rc; }   // one kept record per key
  // Two sources: the keys already in the local set (misses, resolve-half inserts, earlier harvests) and the records —
  // flagged since the last harvest, or kept.  The flagged records are NOT inserted locally first: their keys go straight
  // into the export buffer (and the flags are cleared) — after the exchange every key is inserted exactly once, by its
  // owner.
  const uint64_t key_mask = kmer_mask(ctx->k);
  const DbRange &r = first_range(ctx);
  const bool records = (ctx->seen_dirty || ctx->kept) && r.pairs && r.key_ct;
  return export_parts(ctx, n_parts, 8, reinterpret_cast<unsigned long long *>(d_keys_out), cap, counts,
                      reinterpret_cast<unsigned long long **>(alloc_out), SPARSE_TEXT,
                      [&](unsigned long long *cnt, unsigned long long *out, const unsigned long long *end, uint32_t *err, int pass) {
                        launch_keys_parts(0, ctx->sparse.slots, nullptr, ctx->sparse.cap, key_mask, ctx->d_dense_flag, n_parts, cnt, out,
                                          end, err, pass, ctx->aux);
                        ctx->launches++;
                        if (!records) return;
                        launch_keys_parts(1, nullptr, r.pairs, r.key_ct, key_mask, ctx->d_dense_flag, n_parts, cnt, out, end,
                                          err, pass, ctx->aux);
                        ctx->launches++;
                        // the flags are gone: their keys live in the export buffer now (the kept records drop their flag
                        // when the merged keys replace the set)
                        if (pass == 1) ctx->seen_dirty = false;
                      });
}

int kuq_sparse_replace(kuq_ctx *ctx, const uint64_t *d_keys, uint64_t n) {
  if (!ctx || (!d_keys && n)) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  if (!ctx->sparse.slots) return KUQ_OK;
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  rc = harvest_seen(ctx, true);                  // anything still flagged or kept was exported before; drop the flags
  if (rc) return rc;
  ctx->snap_valid = false;
  // at a load of at most 0.7, from the current size up
  rc = replace_table(ctx, ctx->sparse, reinterpret_cast<const unsigned long long *>(d_keys), n, ctx->sparse.cap, 7);
  if (!rc && n) ctx->set_has_hits = true;
  return rc;
}

int kuq_sparse_summary(kuq_ctx *ctx, uint32_t *d_hist_out, uint32_t *d_distinct_out) {
  if (!ctx || !d_hist_out || !d_distinct_out) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  rc = harvest_seen(ctx, false);
  if (rc) return rc;
  CU(cudaMemsetAsync(d_hist_out, 0, (uint64_t)ctx->n_sketch * 64 * 4, ctx->aux));
  if (ctx->sparse.slots) {
    launch_sparse_histograms(set_keys(ctx), ctx->d_dense_flag, d_hist_out, ctx->aux);
    launch_sparse_histograms(kept_keys(ctx), ctx->d_dense_flag, d_hist_out, ctx->aux);
    ctx->launches += ctx->kept ? 2 : 1;
    CU(cudaMemcpyAsync(d_distinct_out, ctx->sparse.count, ctx->n_sketch * 4ull, cudaMemcpyDeviceToDevice, ctx->aux));
  } else {
    CU(cudaMemsetAsync(d_distinct_out, 0, ctx->n_sketch * 4ull, ctx->aux));
  }
  CU(cudaStreamSynchronize(ctx->aux));
  return KUQ_OK;
}

int kuq_set_sparse_summary(kuq_ctx *ctx, const uint32_t *d_hist, const uint32_t *d_distinct) {
  if (!ctx || !d_hist || !d_distinct) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  CU(cudaSetDevice(ctx->device));
  ctx->merged_hist.resize((size_t)ctx->n_sketch * 64);
  ctx->merged_distinct.resize(ctx->n_sketch);
  CU(cudaMemcpy(ctx->merged_hist.data(), d_hist, (uint64_t)ctx->n_sketch * 64 * 4, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(ctx->merged_distinct.data(), d_distinct, ctx->n_sketch * 4ull, cudaMemcpyDeviceToHost));
  ctx->merged_summary = true;
  ctx->snap_valid = false;
  return KUQ_OK;
}

uint64_t kuq_ertl_sparse(const uint32_t *hist64, uint64_t n_observed) {
  uint64_t n_codes = 0;
  for (int i = 0; i < 64; i++) n_codes += hist64[i];
  return ertl_sparse_hist(hist64, n_codes, n_observed);
}

int kuq_scan_device(kuq_ctx *ctx, uint32_t slot, uint32_t k, uint32_t nt, uint32_t idx_type, const char *d_bases,
                    const uint64_t *d_read_offsets, uint32_t n_reads, uint64_t total_bases, uint64_t *d_canon_out,
                    uint32_t *d_bins_out) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (!d_bases || !d_read_offsets || !d_canon_out || !d_bins_out) return fail(ctx, KUQ_E_INVALID_ARG, "NULL device buffers");
  if ((uintptr_t)d_bases & 15) return fail(ctx, KUQ_E_INVALID_ARG, "d_bases must be 16-byte aligned");
  if (k < 2 || k > 31 || nt < 1 || nt > 15 || nt > k || (idx_type != 1 && idx_type != 2)) return fail(ctx, KUQ_E_INVALID_ARG, "bad k / minimizer length / index type");
  CU(cudaSetDevice(ctx->device));
  Slot &s = ctx->slots[slot];
  if (n_reads > ctx->cfg.max_reads_per_batch || total_bases > ctx->cfg.max_bases_per_batch)
    return fail(ctx, KUQ_E_CAPACITY, "batch exceeds the slot capacity");
  Params p;
  memset(&p, 0, sizeof p);
  p.db.k = k; p.db.nt = nt;
  p.db.key_mask = (1ull << (2 * k)) - 1;
  p.db.xor_mask = (uint32_t)((idx_type == 1 ? 0ull : INDEX2_XOR_MASK) & ((1ull << (2 * nt)) - 1));
  p.db.n_mini = k - nt + 1;
  p.bases = d_bases; p.offsets = d_read_offsets; p.clean = s.d_clean;
  p.n_reads = n_reads; p.n_chunks = (n_reads + CHUNK_READS - 1) / CHUNK_READS;
  p.total_bases = total_bases;
  p.n_windows = s.d_nwin; p.canon = d_canon_out; p.bins = d_bins_out;
  p.chunk_counter = reinterpret_cast<uint32_t *>(s.d_scalars + 2);
  p.error_flag = reinterpret_cast<uint32_t *>(s.d_scalars + 3);
  CU(cudaMemsetAsync(s.d_scalars, 0, 8 * 8, s.stream));
  ctx->launches += launch_scan_only(p, ctx->n_sm, s.stream);
  CU(cudaGetLastError());
  return KUQ_OK;
}

int kuq_layout_experiment(kuq_ctx *ctx, uint32_t slot, uint64_t n_positions, uint32_t reps, kuq_layout_result *out) {
  int rc = check_slot(ctx, slot);
  if (rc) return rc;
  if (!out) return fail(ctx, KUQ_E_INVALID_ARG, "NULL result");
  CU(cudaSetDevice(ctx->device));
  rc = ensure_ready(ctx);
  if (rc) return rc;
  const DbRange &r = first_range(ctx);
  if (ctx->stream_open || !r.pairs) return fail(ctx, KUQ_E_STATE, "the experiment needs a staged (not streamed) database");
  if (ctx->k != 31 || r.nt != 15) return fail(ctx, KUQ_E_INVALID_ARG, "the 8-byte record code is defined for k = 31, m = 15");
  Slot &s = ctx->slots[slot];
  if (!s.timed || n_positions == 0 || n_positions > s.total_bases)
    return fail(ctx, KUQ_E_STATE, "run a batch on the slot first; n_positions must not exceed its text length");
  Params p;
  fill_params(ctx, s, p, nullptr, nullptr, nullptr, 0, 0);
  // a fused call leaves its windows packed: the variants read scratch
  if (s.windows_packed) launch_unpack_windows(p, n_positions, ctx->n_sm, s.stream);
  rc = refresh_reg_floor(ctx, s.total_bases, s.stream);     // the fused variants count
  if (rc) return rc;
  const int erc = layout_experiment(p, r.key_ct, s.d_canon, s.d_bins, s.d_dense, n_positions, ctx->n_sm, s.stream, reps,
                                    ctx->cfg.hll_mode == KUQ_HLL_DENSE_ONLY && s.windows_packed, out);
  ctx->snap_valid = false;
  ctx->launches += 3 + (s.windows_packed ? 1 : 0) + (uint64_t)KUQ_LAYOUT_VARIANTS * (reps + 2ull);
  if (erc == 1) return fail(ctx, KUQ_E_NOMEM, "not enough free device memory for the transcoded and tree-ordered records");
  if (erc == 3) return fail(ctx, KUQ_E_CAPACITY, "dense taxon ids need more than 24 bits");
  if (erc) return fail(ctx, KUQ_E_CUDA, "layout experiment: %s", cudaGetErrorString(cudaGetLastError()));
  return KUQ_OK;
}

int kuq_sparse_tier_info(kuq_ctx *ctx, uint64_t *slots, uint64_t *keys, uint64_t *times_grown, double *last_harvest_ms) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  if (last_harvest_ms) *last_harvest_ms = ctx->harvest_ms;
  return table_info(ctx, ctx->sparse, slots, keys, times_grown);
}

int kuq_sparse_import(kuq_ctx *ctx, const uint64_t *d_keys, uint64_t n) {
  if (!ctx || (!d_keys && n)) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  if (!ctx->sparse.slots || !n) return KUQ_OK;
  ctx->snap_valid = false;
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  rc = harvest_seen(ctx, false, true);           // imported keys may duplicate kept ones: the set becomes the store
  if (rc) return rc;
  // make room first: the import kernel cannot grow the set (a context that classified few reads or none has a small
  // set and may receive the keys of all the others)
  uint64_t used = 0;
  rc = table_items(ctx, ctx->sparse, &used);
  if (!rc) rc = make_room(ctx, ctx->sparse, used, n);
  if (rc) return rc;
  ctx->set_has_hits = true;
  return import_items(ctx, ctx->sparse, reinterpret_cast<const unsigned long long *>(d_keys), n);
}

int kuq_exact_info(kuq_ctx *ctx, uint64_t *slots, uint64_t *pairs, uint64_t *times_grown) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  return table_info(ctx, ctx->exact, slots, pairs, times_grown);
}

int kuq_exact_export(kuq_ctx *ctx, void *d_pairs_out, uint64_t cap, uint64_t *n) {
  if (!ctx || !n) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  *n = 0;
  if (!ctx->exact.slots) return KUQ_OK;                           // not KUQ_HLL_EXACT
  if (ctx->spilled_pairs) return refuse_spilled(ctx, "kuq_exact_export");
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  return exact_export_range(ctx, 0, ctx->exact.cap, static_cast<ExactPair *>(d_pairs_out), d_pairs_out ? cap : 0, n);
}

int kuq_exact_import(kuq_ctx *ctx, const void *d_pairs, uint64_t n) {
  if (!ctx || (!d_pairs && n)) return KUQ_E_INVALID_ARG;
  if ((uintptr_t)d_pairs & 15) return fail(ctx, KUQ_E_INVALID_ARG, "d_pairs must be 16-byte aligned");
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  if (!ctx->exact.slots) return fail(ctx, KUQ_E_STATE, "kuq_exact_import needs a KUQ_HLL_EXACT context");
  if (!n) return KUQ_OK;
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  return exact_import(ctx, static_cast<const ExactPair *>(d_pairs), n);
}

uint32_t kuq_exact_owner(uint64_t kmer, uint32_t n_parts) { return n_parts ? exact_owner(kmer, n_parts) : 0; }

static int exact_export_partitioned(kuq_ctx *ctx, uint32_t n_parts, void *d_pairs_out, uint64_t cap, uint64_t *counts, void **alloc_out) {
  if (!ctx || !counts || n_parts == 0 || n_parts > EXACT_MAX_PARTS) return KUQ_E_INVALID_ARG;
  if (d_pairs_out && ((uintptr_t)d_pairs_out & 15)) return fail(ctx, KUQ_E_INVALID_ARG, "d_pairs_out must be 16-byte aligned");
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  for (uint32_t j = 0; j < n_parts; j++) counts[j] = 0;
  if (!ctx->exact.slots) return fail(ctx, KUQ_E_STATE, "kuq_exact_export_partitioned needs a KUQ_HLL_EXACT context");
  if (ctx->spilled_pairs) return refuse_spilled(ctx, "kuq_exact_export_partitioned");
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  return exact_parts(ctx, 0, ctx->exact.cap, n_parts, static_cast<ExactPair *>(d_pairs_out), cap, counts,
                     reinterpret_cast<ExactPair **>(alloc_out));
}

int kuq_exact_export_partitioned(kuq_ctx *ctx, uint32_t n_parts, void *d_pairs_out, uint64_t cap, uint64_t *counts) {
  return exact_export_partitioned(ctx, n_parts, d_pairs_out, cap, counts, nullptr);
}
int kuq_exact_export_partitioned_alloc(kuq_ctx *ctx, uint32_t n_parts, void **d_pairs_out, uint64_t *counts) {
  if (!d_pairs_out) return KUQ_E_INVALID_ARG;
  *d_pairs_out = nullptr;
  return exact_export_partitioned(ctx, n_parts, nullptr, 0, counts, d_pairs_out);
}

int kuq_exact_replace(kuq_ctx *ctx, const void *d_pairs, uint64_t n) {
  if (!ctx || (!d_pairs && n)) return KUQ_E_INVALID_ARG;
  if ((uintptr_t)d_pairs & 15) return fail(ctx, KUQ_E_INVALID_ARG, "d_pairs must be 16-byte aligned");
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  if (!ctx->exact.slots) return fail(ctx, KUQ_E_STATE, "kuq_exact_replace needs a KUQ_HLL_EXACT context");
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  // a part of its own size: at a load of at most 0.6, from 1024 slots up
  rc = replace_table(ctx, ctx->exact, static_cast<const ExactPair *>(d_pairs), n, 1024, 6);
  if (rc) return rc;
  ctx->exact_partitioned = true;                 // from now on the table holds one owner's part
  ctx->merged_exact = false;
  ctx->snap_valid = false;
  return KUQ_OK;
}

int kuq_exact_summary(kuq_ctx *ctx, uint64_t *d_count_out, int64_t *d_books_out) {
  if (!ctx || !d_count_out || !d_books_out) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  if (!ctx->exact.slots) return fail(ctx, KUQ_E_STATE, "kuq_exact_summary needs a KUQ_HLL_EXACT context");
  if (ctx->spilled_pairs) return refuse_spilled(ctx, "kuq_exact_summary");
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  std::vector<long long> books;
  rc = exact_books(ctx, books);
  if (rc) return rc;
  CU(cudaMemcpy(d_count_out, ctx->exact.count, ctx->n_sketch * 8ull, cudaMemcpyDeviceToDevice));
  CU(cudaMemcpy(d_books_out, books.data(), ctx->n_taxa * 8ull, cudaMemcpyHostToDevice));
  return KUQ_OK;
}

static int set_exact_summary(kuq_ctx *ctx, std::vector<unsigned long long> &count, std::vector<long long> &books) {
  ctx->merged_exact_count.swap(count);
  ctx->merged_books.swap(books);
  ctx->merged_exact = true;
  ctx->snap_valid = false;
  return KUQ_OK;
}

int kuq_set_exact_summary(kuq_ctx *ctx, const uint64_t *d_count, const int64_t *d_books) {
  if (!ctx || !d_count || !d_books) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  if (!ctx->exact.slots) return fail(ctx, KUQ_E_STATE, "kuq_set_exact_summary needs a KUQ_HLL_EXACT context");
  CU(cudaSetDevice(ctx->device));
  std::vector<unsigned long long> count(ctx->n_sketch);
  std::vector<long long> books(ctx->n_taxa);
  CU(cudaMemcpy(count.data(), d_count, ctx->n_sketch * 8ull, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(books.data(), d_books, ctx->n_taxa * 8ull, cudaMemcpyDeviceToHost));
  return set_exact_summary(ctx, count, books);
}

// In one process: every context's pairs go to the context that owns their k-mer, in rounds over slot ranges of each
// source table (KUQ_EXACT_MERGE_SLOTS, as kuq_merge_into), peer to peer between devices.  Each owner builds its part
// in a new table beside its old one, sized to the pairs all sources send it; the old tables go when every round is done.
// Peak per device: its old table + its new part + one round of pairs on each side.  Then the books and counters of
// the parts are summed on the host and installed on ctxs[0] (kuq_set_exact_summary).
int kuq_exact_partition(kuq_ctx *const *ctxs, uint32_t n) {
  if (!ctxs || n == 0 || n > EXACT_MAX_PARTS) return KUQ_E_INVALID_ARG;
  kuq_ctx *ctx = ctxs[0];
  for (uint32_t g = 0; g < n; g++) {
    if (!ctxs[g]) return KUQ_E_INVALID_ARG;
    for (uint32_t h = 0; h < g; h++) if (ctxs[h] == ctxs[g]) return KUQ_E_INVALID_ARG;
  }
  for (uint32_t g = 0; g < n; g++) {
    kuq_ctx *c = ctxs[g];
    int rc = ensure_ready(c);
    if (rc) { if (g) ctx->err = c->err; return rc; }
    if (!c->exact.slots) return fail(ctx, KUQ_E_STATE, "kuq_exact_partition needs KUQ_HLL_EXACT contexts");
    if (c->spilled_pairs) { rc = refuse_spilled(c, "kuq_exact_partition"); if (g) ctx->err = c->err; return rc; }
    if (c->n_taxa != ctx->n_taxa || c->n_sketch != ctx->n_sketch || c->raw_of_dense != ctx->raw_of_dense)
      return fail(ctx, KUQ_E_STATE, "the contexts number their taxa differently (different database / taxonomy)");
    CU(cudaSetDevice(c->device));
    for (auto &s : c->slots) CU(cudaStreamSynchronize(s.stream));
  }
  // 1. pairs per (source, owner): the owner's part is at most their sum (pairs held by several sources collapse)
  std::vector<uint64_t> want(n, 0), counts(n);
  for (uint32_t g = 0; g < n; g++) {
    CU(cudaSetDevice(ctxs[g]->device));
    int rc = exact_parts(ctxs[g], 0, ctxs[g]->exact.cap, n, nullptr, 0, counts.data());
    if (rc) { if (g) ctx->err = ctxs[g]->err; return rc; }
    for (uint32_t o = 0; o < n; o++) want[o] += counts[o];
  }
  // 2. the new parts, at a load of at most 0.6 from 1024 slots up
  std::vector<ExactTable> part(n);
  int rc = KUQ_OK;
  for (uint32_t g = 0; g < n && !rc; g++) {
    CU(cudaSetDevice(ctxs[g]->device));
    rc = alloc_table(ctxs[g], want[g], 1024, 6, part[g]);
    if (rc) ctx->err = ctxs[g]->err;
  }
  // 3. rounds: a slot range of one source, grouped by owner, each group imported by its owner
  for (uint32_t g = 0; g < n && !rc; g++) {
    kuq_ctx *src = ctxs[g];
    rc = move_rounds(
        ctx, "exact k-mer set partition: no room for a round of %llu pairs on device %d", src, ctxs, n,
        [src, n](uint64_t lo, uint64_t hi, ExactPair *buf, uint64_t cap, uint64_t *cnt) { return exact_parts(src, lo, hi, n, buf, cap, cnt); },
        [&](uint32_t o, const ExactPair *pairs, uint64_t m) { return import_items(ctxs[o], part[o], pairs, m, true); });
  }
  if (rc) {
    cudaSetDevice(ctx->device);
    return rc;
  }
  // 4. the parts replace the tables: from now on each holds one owner's part
  for (uint32_t g = 0; g < n; g++) {
    CU(cudaSetDevice(ctxs[g]->device));
    install_table(ctxs[g]->exact, part[g], want[g]);
    ctxs[g]->exact_partitioned = true;
    ctxs[g]->merged_exact = false;
    ctxs[g]->snap_valid = false;
  }
  // 5. counters and books summed over the parts, installed on the first context
  std::vector<unsigned long long> count_sum(ctx->n_sketch, 0), cnt(ctx->n_sketch);
  std::vector<long long> books_sum(ctx->n_taxa, 0), books;
  for (uint32_t g = 0; g < n; g++) {
    kuq_ctx *c = ctxs[g];
    CU(cudaSetDevice(c->device));
    rc = exact_books(c, books);
    if (rc) { ctx->err = c->err; cudaSetDevice(ctx->device); return rc; }
    CU(cudaMemcpy(cnt.data(), c->exact.count, c->n_sketch * 8ull, cudaMemcpyDeviceToHost));
    for (uint32_t d = 0; d < ctx->n_sketch; d++) count_sum[d] += cnt[d];
    for (uint32_t d = 0; d < ctx->n_taxa; d++) books_sum[d] += books[d];
  }
  CU(cudaSetDevice(ctx->device));
  return set_exact_summary(ctx, count_sum, books_sum);
}

int kuq_exact_rollup_passes(kuq_ctx *ctx, uint32_t *passes) {
  if (!ctx || !passes) return KUQ_E_INVALID_ARG;
  *passes = ctx->exact_rollup_passes;
  return KUQ_OK;
}

int kuq_set_exact_spill(kuq_ctx *ctx, uint64_t host_budget_bytes) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  if (ctx->cfg.hll_mode != KUQ_HLL_EXACT) return fail(ctx, KUQ_E_STATE, "kuq_set_exact_spill needs a KUQ_HLL_EXACT context");
  ctx->spill_budget = host_budget_bytes;
  return KUQ_OK;
}

int kuq_exact_spill_info(kuq_ctx *ctx, uint64_t *spills, uint64_t *pairs_on_host) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  if (spills) *spills = ctx->spills;
  if (pairs_on_host) *pairs_on_host = ctx->spilled_pairs;
  return KUQ_OK;
}

// 1. every context spills what its table holds; 2. the EXACT_MAX_PARTS parts of all contexts are cut into groups of
// consecutive parts that fit one table; 3. one host thread per context imports each of its groups into its emptied
// table in rounds (duplicates from successive spills and from other contexts collapse) and adds the group's counters
// and roll-up books to its sums; 4. the sums are installed on ctxs[0] and the host parts go.
int kuq_exact_settle(kuq_ctx *const *ctxs, uint32_t n) {
  if (!ctxs || n == 0) return KUQ_E_INVALID_ARG;
  kuq_ctx *ctx = ctxs[0];
  for (uint32_t g = 0; g < n; g++) {
    if (!ctxs[g]) return KUQ_E_INVALID_ARG;
    for (uint32_t h = 0; h < g; h++) if (ctxs[h] == ctxs[g]) return KUQ_E_INVALID_ARG;
  }
  int max_device = 0;
  for (uint32_t g = 0; g < n; g++) {
    kuq_ctx *c = ctxs[g];
    int rc = ensure_ready(c);
    if (rc) { if (g) ctx->err = c->err; return rc; }
    if (!c->exact.slots) return fail(ctx, KUQ_E_STATE, "kuq_exact_settle needs KUQ_HLL_EXACT contexts");
    if (c->n_taxa != ctx->n_taxa || c->n_sketch != ctx->n_sketch || c->raw_of_dense != ctx->raw_of_dense)
      return fail(ctx, KUQ_E_STATE, "the contexts number their taxa differently (different database / taxonomy)");
    max_device = std::max(max_device, c->device);
  }
  // 1. the pairs still on the devices join the host parts
  for (uint32_t g = 0; g < n; g++) {
    kuq_ctx *c = ctxs[g];
    CU(cudaSetDevice(c->device));
    for (auto &s : c->slots) CU(cudaStreamSynchronize(s.stream));
    int rc = spill_exact(c);
    if (rc) { if (g) ctx->err = c->err; cudaSetDevice(ctx->device); return rc; }
  }
  // 2. a table smaller than the largest grows to it (it is empty now) where its device keeps room beside the new table
  //    for a round buffer and for half the new table's bytes of sort scratch (the roll-up sorts in passes when it has
  //    less than its 32 B per pair); each table takes pairs up to the load of make_room.  Groups of consecutive parts whose spilled pairs fit the largest table; a part
  //    larger than that is a group of its own, which fits only if its duplicates collapse enough.
  uint64_t big = 0;
  for (uint32_t g = 0; g < n; g++) big = std::max(big, ctxs[g]->exact.cap);
  std::vector<uint64_t> room(n);
  for (uint32_t g = 0; g < n; g++) {
    kuq_ctx *c = ctxs[g];
    CU(cudaSetDevice(c->device));
    size_t free_b = 0, total_b = 0;
    const uint64_t headroom = std::min(exact_round_slots(), big) * sizeof(ExactPair) + big * sizeof(ExactPair) / 2;
    if (c->exact.cap < big && cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && free_b >= big * sizeof(ExactPair) + headroom &&
        grow_table(c, c->exact, big) != KUQ_OK)
      c->err.clear();
    (void)cudaGetLastError();
    room[g] = c->exact.cap * 8 / 10;
  }
  const uint64_t room_max = *std::max_element(room.begin(), room.end());
  uint64_t part_pairs[EXACT_MAX_PARTS] = {};
  for (uint32_t g = 0; g < n; g++)
    for (uint32_t j = 0; j < EXACT_MAX_PARTS; j++)
      for (auto &piece : ctxs[g]->spill_parts[j]) part_pairs[j] += piece.size();
  struct Group { uint32_t lo, hi; uint64_t pairs; };
  std::vector<Group> groups;
  for (uint32_t j = 0; j < EXACT_MAX_PARTS; j++) {
    if (!part_pairs[j]) continue;
    if (groups.empty() || groups.back().pairs + part_pairs[j] > room_max) groups.push_back(Group{j, j, 0});
    groups.back().hi = j + 1;
    groups.back().pairs += part_pairs[j];
  }
  // 3. each group to the context with the fewest pairs so far among those whose table takes it (the largest if none)
  std::vector<std::vector<Group>> work(n);
  std::vector<uint64_t> load(n, 0);
  for (const Group &gr : groups) {
    uint32_t best = n;
    for (uint32_t g = 0; g < n; g++)
      if (room[g] >= std::min(gr.pairs, room_max) && (best == n || load[g] < load[best])) best = g;
    work[best].push_back(gr);
    load[best] += gr.pairs;
  }
  std::vector<std::vector<unsigned long long>> count_sum(n, std::vector<unsigned long long>(ctx->n_sketch, 0));
  std::vector<std::vector<long long>> books_sum(n, std::vector<long long>(ctx->n_taxa, 0));
  std::vector<int> status(n, KUQ_OK);
  // the roll-up's sort sizes its scratch to the device's free memory: one sort at a time per device
  std::vector<std::mutex> device_lock(max_device + 1);
  auto settle_groups = [&](uint32_t g) -> int {
    kuq_ctx *ctx = ctxs[g];                      // errors are reported on this context (CU)
    if (work[g].empty()) return KUQ_OK;
    CU(cudaSetDevice(ctx->device));
    uint64_t chunk = std::min(exact_round_slots(), std::max<uint64_t>(room[g], 1));
    DevBuf<ExactPair> d_buf;
    HostBuf<ExactPair> h_buf;
    if (!round_buffers(chunk, d_buf, h_buf))
      return fail(ctx, KUQ_E_NOMEM, "exact k-mer set settle: no memory for a round of %llu pairs on device %d",
                  (unsigned long long)chunk, ctx->device);
    std::vector<unsigned long long> cnt(ctx->n_sketch);
    std::vector<long long> books;
    for (const Group &gr : work[g]) {
      int rc = clear_table(ctx, ctx->exact);
      // the group's pieces in rounds of up to `chunk` pairs: pieces are packed into the pinned buffer, and a piece
      // larger than it is cut
      uint64_t fill = 0;
      auto flush = [&]() -> int {
        if (!fill) return KUQ_OK;
        CU(cudaMemcpyAsync(d_buf, h_buf, fill * sizeof(ExactPair), cudaMemcpyHostToDevice, ctx->aux));
        CU(cudaStreamSynchronize(ctx->aux));
        const uint64_t m = fill;
        fill = 0;
        return exact_import(ctx, d_buf, m);
      };
      for (uint32_t j = gr.lo; j < gr.hi && !rc; j++)
        for (uint32_t s = 0; s < n && !rc; s++)
          for (auto &piece : ctxs[s]->spill_parts[j]) {
            for (uint64_t at = 0; at < piece.size() && !rc;) {
              const uint64_t m = std::min<uint64_t>(piece.size() - at, chunk - fill);
              memcpy(h_buf + fill, piece.data() + at, m * sizeof(ExactPair));
              fill += m;
              at += m;
              if (fill == chunk) rc = flush();
            }
            if (rc) break;
          }
      if (!rc) rc = flush();
      if (rc == KUQ_E_NOMEM)
        return fail(ctx, KUQ_E_NOMEM, "exact k-mer set settle: parts %u to %u (%llu spilled pairs) do not fit the table of %llu "
                                      "slots on device %d: %s", gr.lo, gr.hi - 1, (unsigned long long)gr.pairs,
                    (unsigned long long)ctx->exact.cap, ctx->device, ctx->err.c_str());
      if (rc) return rc;
      {
        std::lock_guard<std::mutex> lock(device_lock[ctx->device]);
        rc = exact_books(ctx, books);
      }
      if (rc) return rc;
      CU(cudaMemcpy(cnt.data(), ctx->exact.count, ctx->n_sketch * 8ull, cudaMemcpyDeviceToHost));
      for (uint32_t d = 0; d < ctx->n_sketch; d++) count_sum[g][d] += cnt[d];
      for (uint32_t d = 0; d < ctx->n_taxa; d++) books_sum[g][d] += books[d];
    }
    return KUQ_OK;
  };
  {
    std::vector<std::thread> threads;
    for (uint32_t g = 1; g < n; g++) threads.emplace_back([&, g] { status[g] = settle_groups(g); });
    status[0] = settle_groups(0);
    for (auto &t : threads) t.join();
  }
  // 4. a failure keeps every host part, so the set is not lost: the contexts stay spilled (their readouts refuse) and the
  //    settle step can run again once there is more device memory (the pairs in the tables are spilled again, and a set
  //    union does not mind them twice)
  CU(cudaSetDevice(ctx->device));
  for (uint32_t g = 0; g < n; g++)
    if (status[g]) {
      if (g) ctx->err = ctxs[g]->err;
      return status[g];
    }
  // the host parts go; every table holds one group at most from now on
  for (uint32_t g = 0; g < n; g++) {
    kuq_ctx *c = ctxs[g];
    drop_spill(c);
    c->exact_partitioned = true;
    c->merged_exact = false;
    c->snap_valid = false;
  }
  for (uint32_t g = 1; g < n; g++) {
    for (uint32_t d = 0; d < ctx->n_sketch; d++) count_sum[0][d] += count_sum[g][d];
    for (uint32_t d = 0; d < ctx->n_taxa; d++) books_sum[0][d] += books_sum[g][d];
  }
  return set_exact_summary(ctx, count_sum[0], books_sum[0]);
}

int kuq_dense_taxids(kuq_ctx *ctx, uint32_t *taxid_of_dense, uint32_t cap, uint32_t *n) {
  if (!ctx || !n) return KUQ_E_INVALID_ARG;
  int rc = ensure_ready(ctx);
  if (rc) return rc;
  *n = ctx->n_taxa;
  if (cap == 0) return KUQ_OK;
  if (cap < ctx->n_taxa) return fail(ctx, KUQ_E_CAPACITY, "need room for %u ids", ctx->n_taxa);
  memcpy(taxid_of_dense, ctx->raw_of_dense.data(), ctx->n_taxa * 4ull);
  return KUQ_OK;
}

int kuq_reset_counts(kuq_ctx *ctx) {
  if (!ctx) return KUQ_E_INVALID_ARG;
  ctx->snap_valid = false;
  drop_spill(ctx);
  ctx->spills = 0;
  if (!ctx->finalized) return KUQ_OK;
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  // the SEEN / KEPT bits of the records go in one discarding pass, skipped when no record can carry one
  int rc = harvest_seen(ctx, true);
  if (rc) return rc;
  ctx->kept = false;
  ctx->kept_keys = 0;
  CU(cudaMemset(ctx->d_regs, 0, (uint64_t)ctx->n_sketch * HLL_M));
  CU(cudaMemset(ctx->d_reg_floor, 0, ctx->n_sketch));
  CU(cudaMemset(ctx->d_dense_flag, 0, ctx->n_sketch));
  CU(cudaMemset(ctx->d_n_kmers, 0, ctx->n_sketch * 8ull));
  CU(cudaMemset(ctx->d_n_reads, 0, ctx->n_taxa * 8ull));
  if (ctx->sparse.slots) {
    CU(cudaMemset(ctx->d_sparse_used, 0, 8));
    rc = clear_table(ctx, ctx->sparse);
    if (rc) return rc;
  }
  if (ctx->exact.slots) {
    rc = clear_table(ctx, ctx->exact);
    if (rc) return rc;
  }
  ctx->set_has_hits = false;
  ctx->merged_summary = false;
  ctx->merged_hist.clear();
  ctx->merged_distinct.clear();
  ctx->exact_partitioned = false;
  ctx->merged_exact = false;
  ctx->merged_exact_count.clear();
  ctx->merged_books.clear();
  ctx->units = WorkUnits();
  return KUQ_OK;
}

uint64_t kuq_ertl_dense(const uint8_t *regs, uint64_t n_observed) {
  int C[66];
  memset(C, 0, sizeof C);
  for (uint32_t i = 0; i < HLL_M; i++) C[regs[i] > 65 ? 65 : regs[i]]++;
  return ertl_from_hist(C, 64 - HLL_P, HLL_M, n_observed);
}

int kuq_harvest_keep_device(int device, void *d_pairs, uint64_t n_rec, const void *d_secondaries, uint64_t n_secondaries,
                            const uint8_t *d_dense_flag, uint32_t n_sketch, uint32_t *d_distinct, uint64_t *d_n_kept) {
  if ((reinterpret_cast<uintptr_t>(d_pairs) & 3) || (n_rec && (!d_pairs || !d_dense_flag || !d_distinct || !d_n_kept)) ||
      (n_secondaries && !d_secondaries))
    return KUQ_E_INVALID_ARG;
  if (cudaSetDevice(device) != cudaSuccess) { (void)cudaGetLastError(); return KUQ_E_NO_DEVICE; }
  launch_harvest_keep(static_cast<uint8_t *>(d_pairs), n_rec, static_cast<const uint2 *>(d_secondaries), n_secondaries, d_dense_flag,
                      n_sketch, d_distinct, reinterpret_cast<unsigned long long *>(d_n_kept), 0);
  if (cudaDeviceSynchronize() != cudaSuccess || cudaGetLastError() != cudaSuccess) return KUQ_E_CUDA;
  return KUQ_OK;
}

// ---- database build (SURVEY.md §8 f4; ROUND 1: compiled, not yet run on hardware) ---------------------------------
int kuq_db_sort_devices(const int *devices, uint32_t n_devices, const void *jdb_image, uint64_t jdb_bytes, uint32_t nt,
                        int zero_vals, uint64_t budget, void *kdb_out, void *idx_out, uint32_t *n_passes, char *err,
                        uint64_t err_cap) {
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
    if (err && err_cap) snprintf(err, err_cap, "db_sort: no CUDA device (there is no CPU path)");
    (void)cudaGetLastError();
    return KUQ_E_NO_DEVICE;
  }
  if (!devices || !n_devices) return KUQ_E_INVALID_ARG;
  for (uint32_t i = 0; i < n_devices; i++)
    if (devices[i] < 0 || devices[i] >= n_dev || cudaSetDevice(devices[i]) != cudaSuccess) return KUQ_E_INVALID_ARG;
  if (cudaSetDevice(devices[0]) != cudaSuccess) return KUQ_E_INVALID_ARG;
  uint32_t passes = 0;
  int rc = dbsort_device(devices, n_devices, (const uint8_t *)jdb_image, jdb_bytes, nt, zero_vals, budget, (uint8_t *)kdb_out,
                         (uint8_t *)idx_out, &passes, err, err_cap);
  if (n_passes) *n_passes = passes;
  return rc;
}

int kuq_db_sort_budget(int device, const void *jdb_image, uint64_t jdb_bytes, uint32_t nt, int zero_vals, uint64_t budget,
                       void *kdb_out, void *idx_out, uint32_t *n_passes, char *err, uint64_t err_cap) {
  return kuq_db_sort_devices(&device, 1, jdb_image, jdb_bytes, nt, zero_vals, budget, kdb_out, idx_out, n_passes, err, err_cap);
}

int kuq_db_sort(int device, const void *jdb_image, uint64_t jdb_bytes, uint32_t nt, int zero_vals, void *kdb_out,
                void *idx_out, char *err, uint64_t err_cap) {
  return kuq_db_sort_budget(device, jdb_image, jdb_bytes, nt, zero_vals, 0, kdb_out, idx_out, NULL, err, err_cap);
}

int kuq_set_lcas_batch(kuq_ctx *ctx, const char *bases, const uint64_t *piece_offsets, uint32_t n_pieces,
                       const uint32_t *taxid, uint32_t flags, uint64_t *n_missing) {
  int rc = check_slot(ctx, 0);
  if (rc) return rc;
  if (n_pieces && (!bases || !piece_offsets || !taxid)) return fail(ctx, KUQ_E_INVALID_ARG, "NULL batch buffers");
  CU(cudaSetDevice(ctx->device));
  Slot &s = ctx->slots[0];
  if (s.busy) return fail(ctx, KUQ_E_STATE, "slot 0 still has an unread batch");
  rc = ensure_ready(ctx);
  if (rc) return rc;
  if (n_pieces > ctx->cfg.max_reads_per_batch) return fail(ctx, KUQ_E_CAPACITY, "%u pieces > slot capacity %u", n_pieces, ctx->cfg.max_reads_per_batch);
  for (uint32_t i = 0; i < n_pieces; i++) {
    // the reference skips sequences whose taxid the taxonomy does not hold (set_lcas.cpp:336-341): the caller's job
    auto it = ctx->dense_of_raw.find(taxid[i]);
    if (taxid[i] == 0 || it == ctx->dense_of_raw.end())
      return fail(ctx, KUQ_E_INVALID_ARG, "piece %u: taxid %u is not in the taxonomy", i, taxid[i]);
    s.h_unit[i] = it->second;
  }
  if (flags & KUQ_LCA_FORCE_CONTAMINANT) {
    // first-come-first-kept between the two contaminant taxids is the one order dependence of -T: one kind per batch
    bool c1 = false, c2 = false;
    for (uint32_t i = 0; i < n_pieces; i++) { c1 |= taxid[i] == 32630u; c2 |= taxid[i] == 81077u; }
    if (c1 && c2) return fail(ctx, KUQ_E_INVALID_ARG, "with KUQ_LCA_FORCE_CONTAMINANT a batch may hold pieces of taxid 32630 or of 81077, not both");
  }
  uint64_t total = 0;
  rc = upload_reads(ctx, s, bases, piece_offsets, n_pieces, &total);
  if (rc) return rc;
  s.n_reads = n_pieces; s.flags = 0; s.total_bases = total; s.external = false;
  if (n_pieces) CU(cudaMemcpyAsync(s.d_unit, s.h_unit, n_pieces * 4ull, cudaMemcpyHostToDevice, s.stream));
  Params p;
  fill_params(ctx, s, p, s.d_bases, s.d_offsets, s.d_unit, n_pieces, 0);
  p.lca_flags = flags & 3u;
  {
    auto c1 = ctx->dense_of_raw.find(32630u), c2 = ctx->dense_of_raw.find(81077u);   // set_lcas.cpp:88-89
    p.lca_keep[0] = c1 == ctx->dense_of_raw.end() ? 0 : c1->second;
    p.lca_keep[1] = c2 == ctx->dense_of_raw.end() ? 0 : c2->second;
  }
  CU(cudaMemsetAsync(s.d_scalars, 0, 8 * 8, s.stream));
  ctx->lca_mode = true;
  ctx->snap_valid = false;
  ctx->launches += launch_set_lcas(p, ctx->n_sm, s.stream);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(s.h_scalars, s.d_scalars, 8 * 8, cudaMemcpyDeviceToHost, s.stream));
  CU(cudaStreamSynchronize(s.stream));
  if (n_missing) *n_missing = s.h_scalars[4];
  return KUQ_OK;
}

int kuq_db_value_counts(kuq_ctx *ctx, uint32_t *taxid, uint64_t *count, uint32_t cap, uint32_t *n) {
  if (!ctx || !n) return KUQ_E_INVALID_ARG;
  if (ctx->dbs.empty()) return fail(ctx, KUQ_E_STATE, "no database staged");
  if (ctx->dbs.size() > 1) return fail(ctx, KUQ_E_STATE, "several databases staged: count them one at a time");
  const StagedDb &db = ctx->dbs[0];
  std::vector<std::pair<uint32_t, uint64_t>> u;
  if (!db.remapped) {
    // the values are still the taxids they were staged with, and staging counted them (collect_taxids)
    for (size_t i = 0; i < db.taxids.size(); i++) u.emplace_back(db.taxids[i], db.counts[i]);
  } else {
    CU(cudaSetDevice(ctx->device));
    for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
    DevBuf<unsigned long long> d_counts;
    DevBuf<uint32_t> d_bad;
    CU(d_counts.alloc(ctx->n_taxa));
    CU(d_bad.alloc(1));
    CU(cudaMemsetAsync(d_counts, 0, ctx->n_taxa * 8ull, ctx->aux));
    CU(cudaMemsetAsync(d_bad, 0, 4, ctx->aux));
    launch_value_counts(db.range.pairs, db.range.key_ct, ctx->n_taxa, d_counts, d_bad, ctx->aux);
    CU(cudaGetLastError());
    ctx->launches++;
    std::vector<unsigned long long> c(ctx->n_taxa);
    uint32_t bad = 0;
    CU(cudaMemcpyAsync(c.data(), d_counts, ctx->n_taxa * 8ull, cudaMemcpyDeviceToHost, ctx->aux));
    CU(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, ctx->aux));
    CU(cudaStreamSynchronize(ctx->aux));
    if (bad) return fail(ctx, KUQ_E_STATE, "a record holds a dense id outside the %u taxa", ctx->n_taxa);
    for (uint32_t d = 0; d < ctx->n_taxa; d++)
      if (c[d]) u.emplace_back(ctx->raw_of_dense[d], c[d]);
    std::sort(u.begin(), u.end());
  }
  *n = (uint32_t)u.size();
  if (cap == 0) return KUQ_OK;
  if (cap < *n) return fail(ctx, KUQ_E_CAPACITY, "need room for %u taxids", *n);
  for (uint32_t i = 0; i < *n; i++) {
    if (taxid) taxid[i] = u[i].first;
    if (count) count[i] = u[i].second;
  }
  return KUQ_OK;
}

int kuq_export_db_values(kuq_ctx *ctx, void *kdb_image, uint64_t kdb_bytes) {
  if (!ctx || !kdb_image) return KUQ_E_INVALID_ARG;
  if (ctx->dbs.empty() || !ctx->dbs[0].own_pairs) return fail(ctx, KUQ_E_STATE, "no database staged from a host image");
  const StagedDb &db = ctx->dbs[0];
  CU(cudaSetDevice(ctx->device));
  for (auto &s : ctx->slots) CU(cudaStreamSynchronize(s.stream));
  const uint64_t key_bits = 2ull * ctx->k, header = kdb_header_bytes(key_bits);
  const uint64_t key_len = kdb_key_len(key_bits), pair_sz = key_len + 4;           // the file's records, not HBM's 12 bytes
  const uint64_t rec_base = db.range.rec_base, key_ct = db.range.key_ct;
  if (kdb_bytes < header + (rec_base + key_ct) * pair_sz)
    return fail(ctx, KUQ_E_INVALID_ARG, "image too small for %llu records", (unsigned long long)(rec_base + key_ct));
  std::vector<uint8_t> rec(key_ct * 12);
  CU(cudaMemcpy(rec.data(), db.range.pairs, rec.size(), cudaMemcpyDeviceToHost));
  uint8_t *out = (uint8_t *)kdb_image + header + rec_base * pair_sz;              // a staged range: its records only
  for (uint64_t i = 0; i < key_ct; i++) {
    uint32_t v;
    memcpy(&v, rec.data() + i * 12 + 8, 4);
    if (db.remapped) {                                      // dense id → taxid
      if (v >= ctx->n_taxa) return fail(ctx, KUQ_E_STATE, "record %llu holds an unknown dense id %u", (unsigned long long)i, v);
      v = ctx->raw_of_dense[v];
    }
    memcpy(out + i * pair_sz + key_len, &v, 4);
  }
  return KUQ_OK;
}

}  // extern "C"
