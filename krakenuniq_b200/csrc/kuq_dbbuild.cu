// db_sort on the GPU — SURVEY.md §8 row f4 (db_sort.cpp:41-116, make_index krakendb.cpp:118-148).
// Checked against the CPU statement of the same tool, oracle/kuq_oracle.c:kuqo_db_sort, which is pinned byte for byte
// against the reference executable.
//
// The reference bins the records by bin_key(key) and qsorts every bin by key.  Keys are distinct, so the result is
// THE order by (bin, key): one stable LSD radix sort by key followed by one by bin.  The two sorts are CUB's
// DeviceRadixSort (library code; database build is not the hot path north_star names), the kernels around them —
// minimizer of every stored key, bin histogram, record gather — are ours.  Records never move during the sorts:
// only (key, index) and (bin, index) pairs do, and one gather at the end writes the 12-byte records.
//
// A database whose one-piece working set does not fit the byte budget is sorted in passes over the host images:
//   A. the record body streams through the device once for the bin histogram, whose running sum is database.idx;
//   B. it streams once more and every chunk is grouped, stably, by minimizer range (kuq_ranges.h cuts the ranges
//      from the index); each range's slice goes to that range's cursor in the output image;
//   C. each range's records come back to the device, get the two sorts of the one-piece path, and return in place.
// Within a range the records keep input order until C, so repeated keys come out as in the one-piece sort.
// With several workers (devices, or one device listed more than once) A and B run on one contiguous input slice each,
// and a range's records are laid out slice after slice (per-slice cursors from each slice's histogram), which keeps
// that order; C sorts one contiguous group of ranges per worker.  Workers write disjoint bytes of the host images.
#include "../../include/kuq.h"
#include "kuq_bounce.cuh"
#include "kuq_dbfile.h"
#include "kuq_kernels.cuh"
#include "kuq_minimizer.cuh"
#include "kuq_ranges.h"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <cstdarg>
#include <cstdio>
#include <cstring>

namespace kuq {
namespace {

typedef unsigned long long ull;

__device__ __forceinline__ uint64_t record_key(const uint8_t *r, uint32_t key_len) {
  uint64_t key = 0;
  for (uint32_t b = 0; b < key_len; b++) key |= (uint64_t)r[b] << (8 * b);  // memcpy(&kmer, pair, key_len), :99-100
  return key;
}

// one thread per record: key, its bin (relative to bin_lo), its position; the bin histogram on the way if asked
// (make_index :126-134)
__global__ void k_dbs_keys(const uint8_t *pairs, uint64_t n, uint32_t key_len, uint32_t k, uint32_t nt, uint32_t bin_lo,
                           ull *keys, uint32_t *bins, ull *index, ull *bin_counts) {
  const uint32_t pair_sz = key_len + 4;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t key = record_key(pairs + i * pair_sz, key_len);
    const uint32_t bin = bin_key_of(key, k, nt);
    keys[i] = key;
    bins[i] = bin - bin_lo;
    index[i] = i;
    if (bin_counts) atomicAdd(bin_counts + bin + 1, 1ull);                     // offsets[b + 1] after the scan
  }
}

// pass A: the bin histogram alone
__global__ void k_dbs_hist(const uint8_t *pairs, uint64_t n, uint32_t key_len, uint32_t k, uint32_t nt, ull *bin_counts) {
  const uint32_t pair_sz = key_len + 4;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    atomicAdd(bin_counts + bin_key_of(record_key(pairs + i * pair_sz, key_len), k, nt) + 1, 1ull);
}

// pass B: the range of each record (range r starts at bin starts[r]; every record's bin lies in some range), its
// position, and the chunk's record count per range
__global__ void k_dbs_range_of(const uint8_t *pairs, uint64_t n, uint32_t key_len, uint32_t k, uint32_t nt,
                               const uint32_t *starts, uint32_t n_ranges, uint32_t *rid, ull *index, ull *range_counts) {
  const uint32_t pair_sz = key_len + 4;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t bin = bin_key_of(record_key(pairs + i * pair_sz, key_len), k, nt);
    uint32_t lo = 0, hi = n_ranges;                                            // last start <= bin
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (__ldg(starts + mid) <= bin) lo = mid; else hi = mid;
    }
    rid[i] = lo;
    index[i] = i;
    atomicAdd(range_counts + lo, 1ull);
  }
}

// per-slice cursors: records of one input slice in each range, from the slice's own running bin counts (off[b] =
// records in bins < b); range r holds bins [starts[r], starts[r + 1]), the last one up to n_bins — the bins
// k_dbs_range_of sends to it
__global__ void k_dbs_range_counts(const ull *off, uint64_t n_bins, const uint32_t *starts, uint32_t n_ranges, ull *counts) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_ranges; r += gridDim.x * blockDim.x)
    counts[r] = off[r + 1 < n_ranges ? starts[r + 1] : n_bins] - off[starts[r]];
}

// records per value (kuq_db_value_counts): values are dense ids < n_ids.  Each warp groups its lanes by value
// (__match_any_sync) and one lane adds the group's size, so a value most records hold (0, a dominant species) costs
// one atomic per warp, not 32.  SHARED: the block counts into its own 32-bit counters in shared memory first (the grid
// is sized so that no block sees 2^32 records) and adds them to the global ones at its end.  *bad = 1 when a value is
// not below n_ids.
template <bool SHARED>
__global__ void k_value_counts(const uint8_t *pairs, uint64_t n, uint32_t n_ids, ull *counts, uint32_t *bad) {
  extern __shared__ uint32_t sh_counts[];
  if (SHARED) {
    for (uint32_t i = threadIdx.x; i < n_ids; i += blockDim.x) sh_counts[i] = 0;
    __syncthreads();
  }
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;                    // a multiple of 32: whole warps loop
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); w < n; w += stride) {
    const uint64_t i = w + lane;
    const bool ok = i < n;
    uint32_t v = ok ? *reinterpret_cast<const uint32_t *>(pairs + i * 12 + 8) : 0xFFFFFFFFu;
    if (ok && v >= n_ids) { *bad = 1; v = 0xFFFFFFFFu; }
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, v);
    if (v != 0xFFFFFFFFu && lane == (uint32_t)(__ffs(peers) - 1)) {
      if (SHARED) atomicAdd(sh_counts + v, (uint32_t)__popc(peers));
      else atomicAdd(counts + v, (ull)__popc(peers));
    }
  }
  if (SHARED) {
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n_ids; i += blockDim.x)
      if (sh_counts[i]) atomicAdd(counts + i, (ull)sh_counts[i]);
  }
}

__global__ void k_dbs_gather_bins(const uint32_t *bins, const ull *index, uint64_t n, uint32_t *out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    out[i] = bins[index[i]];
}

// output record i = input record index[i]; -z zeroes the value (db_sort.cpp:105-106)
__global__ void k_dbs_emit(const uint8_t *in, const ull *index, uint64_t n, uint32_t key_len, int zero_vals, uint8_t *out) {
  const uint32_t pair_sz = key_len + 4;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t *src = in + index[i] * pair_sz;
    uint8_t *dst = out + i * pair_sz;
    for (uint32_t b = 0; b < key_len; b++) dst[b] = src[b];
    for (uint32_t b = 0; b < 4; b++) dst[key_len + b] = zero_vals ? (uint8_t)0 : src[key_len + b];
  }
}

int seterr(int code, char *err, size_t cap, const char *fmt, ...) {
  if (err && cap) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(err, cap, fmt, ap);
    va_end(ap);
  }
  return code;
}

// count items and 16 bytes more
template <typename T>
cudaError_t get(DevBuf<T> &b, uint64_t count) { return b.alloc(count + 16 / sizeof(T)); }

#define DB_CU(call)                                                                                      \
  do {                                                                                                   \
    cudaError_t e__ = (call);                                                                            \
    if (e__ != cudaSuccess) return seterr(KUQ_E_DB_FORMAT, err, err_cap, "db_sort: %s: %s", #call, cudaGetErrorString(e__)); \
  } while (0)

struct Geometry {
  uint32_t k, nt, key_len;
  uint64_t key_bits, pair_sz, header, n, entries;
};

int bits_for(uint64_t span) {       // radix bits of values in [0, span)
  int b = 1;
  while ((1ull << b) < span) b++;
  return b;
}

// ---- the two-sort core: records [0, n) of a slice whose bins start at bin_lo → sorted by (bin, key) ----------------
const uint64_t CORE_REC = 44;        // device bytes per record besides its two copies: keys x2, index x2, bins x3
// Planned bytes per record of a pass-C range besides its two copies: CORE_REC plus CUB's alternate key and value
// arrays of the key sort (16 B) and its look-back state; the plan is checked against CUB's queried size.
const uint64_t PASS_C_REC = CORE_REC + 20;
const uint64_t RESERVE = 1ull << 18; // budget kept back from the pass-C plan for CUB's fixed-size state

struct Core {
  DevBuf<uint8_t> in, out, tmp;
  DevBuf<ull> keys, keys2, idx, idx2;
  DevBuf<uint32_t> bins, bins2, bins3;
  size_t tmp_bytes = 0;
};

// CUB's temporary bytes for the two sorts of n records with bins of bin_bits bits
cudaError_t core_tmp(uint64_t n, int key_bits, int bin_bits, size_t *bytes) {
  size_t a = 0, b = 0;
  *bytes = 0;
  if (!n) return cudaSuccess;
  cudaError_t rc = cub::DeviceRadixSort::SortPairs((void *)nullptr, a, (ull *)nullptr, (ull *)nullptr, (ull *)nullptr,
                                                   (ull *)nullptr, (int64_t)n, 0, key_bits);
  if (rc == cudaSuccess)
    rc = cub::DeviceRadixSort::SortPairs((void *)nullptr, b, (uint32_t *)nullptr, (uint32_t *)nullptr, (ull *)nullptr,
                                         (ull *)nullptr, (int64_t)n, 0, bin_bits);
  *bytes = a > b ? a : b;
  return rc;
}

uint64_t core_bytes(uint64_t n, uint64_t pair_sz, size_t tmp) { return n * (2 * pair_sz + CORE_REC) + tmp + 10 * 16; }

cudaError_t core_alloc(Core &c, uint64_t n, uint64_t pair_sz, size_t tmp) {
  cudaError_t rc;
  if ((rc = get(c.in, n * pair_sz)) || (rc = get(c.out, n * pair_sz)) || (rc = get(c.keys, n)) || (rc = get(c.keys2, n)) ||
      (rc = get(c.idx, n)) || (rc = get(c.idx2, n)) || (rc = get(c.bins, n)) || (rc = get(c.bins2, n)) || (rc = get(c.bins3, n)) ||
      (rc = get(c.tmp, tmp)))
    return rc;
  c.tmp_bytes = tmp;
  return cudaSuccess;
}

// c.in[0, n) → c.out sorted by (bin, key), -z applied; the bins lie in [bin_lo, bin_lo + 2^bin_bits).  hist (optional)
// receives the bin histogram at hist[bin + 1].
cudaError_t core_sort(Core &c, uint64_t n, const Geometry &g, uint32_t bin_lo, int bin_bits, int zero_vals, ull *hist,
                      cudaStream_t st) {
  if (!n) return cudaSuccess;
  const int grid = device_sm_count() * 8;
  k_dbs_keys<<<grid, 256, 0, st>>>(c.in, n, g.key_len, g.k, g.nt, bin_lo, c.keys, c.bins, c.idx, hist);
  // by key (pair_cmp, db_sort.cpp:118-128) ...
  size_t need = c.tmp_bytes;
  cudaError_t rc = cub::DeviceRadixSort::SortPairs(c.tmp.get(), need, c.keys.get(), c.keys2.get(), c.idx.get(), c.idx2.get(), (int64_t)n, 0,
                                                   (int)g.key_bits, st);
  if (rc != cudaSuccess) return rc;
  // ... then, stably, by bin (:96-107): the order inside a bin stays the key order
  k_dbs_gather_bins<<<grid, 256, 0, st>>>(c.bins, c.idx2, n, c.bins2);
  need = c.tmp_bytes;
  rc = cub::DeviceRadixSort::SortPairs(c.tmp.get(), need, c.bins2.get(), c.bins3.get(), c.idx2.get(), c.idx.get(), (int64_t)n, 0, bin_bits, st);
  if (rc != cudaSuccess) return rc;
  k_dbs_emit<<<grid, 256, 0, st>>>(c.in, c.idx, n, g.key_len, zero_vals, c.out);
  return cudaGetLastError();
}

uint64_t largest_bin(const uint64_t *offsets, uint64_t entries) {
  uint64_t m = 0;
  for (uint64_t b = 0; b < entries; b++) m = std::max(m, offsets[b + 1] - offsets[b]);
  return m;
}

// One worker of a sort in passes: a device, its stream and bounce buffers, and the slice [s0, s1) of the input records
// whose histogram (pass A) and grouping (pass B) it does.  Several workers may share a device.
struct Worker {
  int dev = 0;
  Stream st;
  PinnedBounce *bounce = nullptr;
  uint64_t s0 = 0, s1 = 0;
  DevBuf<ull> d_off;                       // pass A → cursors: the running bin counts of the slice
  std::vector<uint64_t> off;               // their host copy (worker 0 writes the index instead)
  std::vector<uint64_t> cursor;            // per range: where the slice's records of the range go in the output
  std::vector<uint64_t> cnt;               // per range: the slice's records of the range
  size_t group_first = 0, group_end = 0;   // pass C: ranges [group_first, group_end)
  int rc = KUQ_OK;
  char msg[512] = "";
  ~Worker() {                              // the bounce's events belong to the worker's device
    int cur = dev;
    cudaGetDevice(&cur);
    cudaSetDevice(dev);
    delete bounce;
    cudaSetDevice(cur);
  }
};

// f(worker, err, err_cap) on every worker at once, one host thread each on its device; the first failure's code and
// message
template <typename F>
int on_workers(std::vector<Worker> &W, F f, char *err, size_t err_cap) {
  std::vector<std::thread> th;
  for (auto &w : W)
    th.emplace_back([&w, &f] {
      w.rc = cudaSetDevice(w.dev) == cudaSuccess ? f(w, w.msg, sizeof w.msg)
                                                 : seterr(KUQ_E_NO_DEVICE, w.msg, sizeof w.msg, "db_sort: device %d not usable", w.dev);
    });
  for (auto &t : th) t.join();
  for (auto &w : W)
    if (w.rc) return seterr(w.rc, err, err_cap, "%s", w.msg);
  return KUQ_OK;
}

}  // namespace

// Host images in, host images out (kdb_out: header + key_ct * pair size bytes — what db_sort.cpp:70-72 writes;
// idx_out: 8 + 8 * (4^nt + 1) bytes), on devices[0, n_dev) (the current device is devices[0]).  budget = bytes of
// device memory per worker (0 → KUQ_DB_SORT_BUDGET, else 3/4 of each device's free memory shared among the workers on
// it).  Returns KUQ_OK, KUQ_E_CAPACITY (a bin or the histogram does not fit the budget) or KUQ_E_DB_FORMAT (+ err).
int dbsort_device(const int *devices, uint32_t n_dev, const uint8_t *jdb, uint64_t jdb_bytes, uint32_t nt, int zero_vals,
                  uint64_t budget, uint8_t *kdb_out, uint8_t *idx_out, uint32_t *n_passes, char *err, size_t err_cap) {
  if (!jdb || !kdb_out || !idx_out) return seterr(KUQ_E_DB_FORMAT, err, err_cap, "db_sort: NULL image");
  if (jdb_bytes < 56 || memcmp(jdb, "JFLISTDN", 8) != 0)
    return seterr(KUQ_E_DB_FORMAT, err, err_cap, "db_sort: not a Jellyfish-style database (krakendb.cpp:67)");
  if (nt < 1 || nt > 15) return seterr(KUQ_E_DB_FORMAT, err, err_cap, "db_sort: -n must be 1..15");
  const KdbFile h = kdb_view(jdb);
  const uint64_t key_bits = h.key_bits;
  if (h.val_len != 4) return seterr(KUQ_E_DB_FORMAT, err, err_cap, "db_sort: can only handle 4 byte DB values (krakendb.cpp:73-74)");
  if (key_bits < 2 * nt || key_bits > 64)
    return seterr(KUQ_E_DB_FORMAT, err, err_cap, "db_sort: key_bits %llu out of range", (unsigned long long)key_bits);
  Geometry g;
  g.k = h.k;
  g.nt = nt;
  g.key_len = (uint32_t)h.key_len;
  g.key_bits = key_bits;
  g.pair_sz = h.pair_sz;
  g.header = h.header_bytes;
  g.n = h.key_ct;
  g.entries = 1ull << (2 * nt);
  if (jdb_bytes < g.header + g.n * g.pair_sz) return seterr(KUQ_E_DB_FORMAT, err, err_cap, "db_sort: image shorter than its header says");
  const uint64_t n = g.n, pair_sz = g.pair_sz, entries = g.entries;
  // one_budget decides whether the sort fits the first device in one piece; budget is then what every worker of the
  // passes may use, the same for all so that the plan does not depend on the devices
  uint64_t one_budget = budget;
  if (!budget) {
    const char *s = getenv("KUQ_DB_SORT_BUDGET");
    one_budget = budget = s && *s ? strtoull(s, nullptr, 10) : 0;
    if (!budget) {
      budget = UINT64_MAX;
      for (uint32_t w = 0; w < n_dev; w++) {
        size_t free_b = 0, total_b = 0;
        DB_CU(cudaSetDevice(devices[w]));
        DB_CU(cudaMemGetInfo(&free_b, &total_b));
        uint32_t sharing = 0;
        for (uint32_t v = 0; v < n_dev; v++) sharing += devices[v] == devices[w];
        if (w == 0) one_budget = free_b / 4 * 3;
        budget = std::min<uint64_t>(budget, free_b / 4 * 3 / sharing);
      }
      DB_CU(cudaSetDevice(devices[0]));
    }
  }
  memcpy(kdb_out, jdb, g.header);                                              // db_sort.cpp:56-58,71
  memcpy(idx_out, "KRAKIX2", 7);                                               // krakendb.cpp:144-147
  idx_out[7] = (uint8_t)nt;
  const uint8_t *body = jdb + g.header;
  uint8_t *obody = kdb_out + g.header;
  const uint64_t idx_dev = (entries + 1) * 8 + 16;
  size_t tmp = 0, scan_tmp = 0;
  DB_CU(core_tmp(n, (int)key_bits, 2 * nt, &tmp));
  DB_CU(cub::DeviceScan::InclusiveSum((void *)nullptr, scan_tmp, (ull *)nullptr, (ull *)nullptr, (int64_t)(entries + 1)));
  *n_passes = 1;

  // ---- in one piece on the first device: the whole input and the index on the device ----
  if (core_bytes(n, pair_sz, std::max(tmp, scan_tmp)) + idx_dev <= one_budget) {
    PinnedBounce bounce;
    DB_CU(bounce.init());
    cudaStream_t st = 0;
    Core c;
    DevBuf<ull> d_off;
    DB_CU(core_alloc(c, n, pair_sz, std::max(tmp, scan_tmp)));
    DB_CU(get(d_off, entries + 1));
    DB_CU(bounce.to_device(c.in, body, n * pair_sz, st));
    DB_CU(cudaMemsetAsync(d_off, 0, (entries + 1) * 8, st));
    DB_CU(core_sort(c, n, g, 0, 2 * nt, zero_vals, d_off, st));
    // offsets = running sum of the bin sizes (make_index :136-139)
    size_t need = c.tmp_bytes;
    DB_CU(cub::DeviceScan::InclusiveSum(c.tmp.get(), need, d_off.get(), d_off.get(), (int64_t)(entries + 1), st));
    DB_CU(bounce.to_host(obody, c.out, n * pair_sz, st));
    DB_CU(bounce.to_host(idx_out + 8, d_off, (entries + 1) * 8, st));
    return KUQ_OK;
  }

  // ---- in passes: worker w holds the contiguous slice [n * w / G, n * (w + 1) / G) of the input records ----
  std::vector<Worker> W(n_dev);
  for (uint32_t w = 0; w < n_dev; w++) {
    W[w].dev = devices[w];
    W[w].s0 = (uint64_t)((unsigned __int128)n * w / n_dev);
    W[w].s1 = (uint64_t)((unsigned __int128)n * (w + 1) / n_dev);
  }
  int rc = on_workers(W, [&](Worker &w, char *err, size_t err_cap) -> int {
    w.bounce = new PinnedBounce;
    DB_CU(w.bounce->init());
    DB_CU(w.st.alloc(cudaStreamNonBlocking));
    return KUQ_OK;
  }, err, err_cap);
  if (rc) return rc;

  // ---- pass A: each slice's bin histogram, streamed, and its running sum; the sum over the slices is the index ----
  rc = on_workers(W, [&](Worker &w, char *err, size_t err_cap) -> int {
    const uint64_t m_all = w.s1 - w.s0;
    uint64_t chunk = std::max<uint64_t>(1, std::min(m_all, PinnedBounce::CH / pair_sz));
    while (chunk > 1 && idx_dev + scan_tmp + chunk * pair_sz + 32 > budget) chunk /= 2;
    if (idx_dev + scan_tmp + chunk * pair_sz + 32 > budget)
      return seterr(KUQ_E_CAPACITY, err, err_cap, "db_sort: the bin histogram of -n %u (%llu bytes) does not fit KUQ_DB_SORT_BUDGET = %llu bytes",
                    nt, (unsigned long long)idx_dev, (unsigned long long)budget);
    const int grid = device_sm_count() * 8;
    DevBuf<uint8_t> d_chunk, d_tmp;
    DB_CU(get(d_chunk, chunk * pair_sz));
    DB_CU(get(w.d_off, entries + 1));
    DB_CU(get(d_tmp, scan_tmp));
    DB_CU(cudaMemsetAsync(w.d_off, 0, (entries + 1) * 8, w.st));
    for (uint64_t s = w.s0; s < w.s1; s += chunk) {
      const uint64_t m = std::min(chunk, w.s1 - s);
      DB_CU(w.bounce->h2d(d_chunk, body + s * pair_sz, m * pair_sz, w.st));   // the host copy of the next overlaps this kernel
      k_dbs_hist<<<grid, 256, 0, w.st>>>(d_chunk, m, g.key_len, g.k, nt, w.d_off);
      DB_CU(cudaGetLastError());
    }
    size_t need = scan_tmp;
    DB_CU(cub::DeviceScan::InclusiveSum(d_tmp.get(), need, w.d_off.get(), w.d_off.get(), (int64_t)(entries + 1), w.st));
    if (&w != &W[0]) w.off.resize(entries + 1);
    DB_CU(w.bounce->to_host(&w == &W[0] ? (void *)(idx_out + 8) : (void *)w.off.data(), w.d_off, (entries + 1) * 8, w.st));
    return KUQ_OK;
  }, err, err_cap);
  if (rc) return rc;
  uint64_t *offsets = reinterpret_cast<uint64_t *>(idx_out + 8);
  if (n_dev > 1) {                                                             // the running sums add up
    std::vector<std::thread> th;
    const uint64_t per = (entries + 1 + PinnedBounce::NT - 1) / PinnedBounce::NT;
    for (uint64_t a = 0; a < entries + 1; a += per)
      th.emplace_back([&, a] {
        for (uint32_t w = 1; w < n_dev; w++)
          for (uint64_t b = a; b < std::min(entries + 1, a + per); b++) offsets[b] += W[w].off[b];
      });
    for (auto &t : th) t.join();
    for (auto &w : W) std::vector<uint64_t>().swap(w.off);
  }

  // ---- the ranges of pass C: planned from the index, checked against CUB's queried temporary size ----
  std::vector<std::pair<uint64_t, uint64_t>> ranges;
  uint64_t max_rec = 0;
  size_t ctmp = 0;
  {
    uint64_t plan_budget = budget > RESERVE ? budget - RESERVE : 0;
    for (int attempt = 0;; attempt++) {
      if (!plan_ranges(offsets, entries, plan_budget, 2 * pair_sz + PASS_C_REC, ranges))
        return seterr(KUQ_E_CAPACITY, err, err_cap, "db_sort: a minimizer bin of %llu records does not fit KUQ_DB_SORT_BUDGET = %llu bytes",
                      (unsigned long long)largest_bin(offsets, entries), (unsigned long long)budget);
      int max_bits = 1;
      max_rec = 0;
      for (auto &r : ranges) {
        max_rec = std::max(max_rec, offsets[r.second] - offsets[r.first]);
        max_bits = std::max(max_bits, bits_for(r.second - r.first));
      }
      DB_CU(core_tmp(max_rec, (int)key_bits, max_bits, &ctmp));
      const uint64_t need = core_bytes(max_rec, pair_sz, ctmp);
      if (need <= budget) break;
      if (attempt == 8 || need - budget >= plan_budget)
        return seterr(KUQ_E_CAPACITY, err, err_cap, "db_sort: a range of %llu records needs %llu bytes, more than KUQ_DB_SORT_BUDGET = %llu",
                      (unsigned long long)max_rec, (unsigned long long)need, (unsigned long long)budget);
      plan_budget -= need - budget;
    }
  }
  const uint32_t R = (uint32_t)ranges.size();
  std::vector<uint32_t> starts(R);
  for (uint32_t r = 0; r < R; r++) starts[r] = (uint32_t)ranges[r].first;

  // ---- cursors: each slice's records per range (on its device, from its running sums); a range's records are laid
  // out slice after slice, so that they keep input order across the slices ----
  if (R) {
    rc = on_workers(W, [&](Worker &w, char *err, size_t err_cap) -> int {
      DevBuf<uint32_t> d_starts;
      DevBuf<ull> d_cnt;
      DB_CU(get(d_starts, R));
      DB_CU(get(d_cnt, R));
      DB_CU(cudaMemcpyAsync(d_starts, starts.data(), R * 4ull, cudaMemcpyHostToDevice, w.st));
      k_dbs_range_counts<<<(R + 255) / 256, 256, 0, w.st>>>(w.d_off, entries, d_starts, R, d_cnt);
      DB_CU(cudaGetLastError());
      w.cnt.resize(R);
      DB_CU(cudaMemcpyAsync(w.cnt.data(), d_cnt, R * 8ull, cudaMemcpyDeviceToHost, w.st));
      DB_CU(cudaStreamSynchronize(w.st));
      w.d_off.reset();
      return KUQ_OK;
    }, err, err_cap);
    if (rc) return rc;
  }
  for (uint32_t r = 0; r < R; r++) {
    uint64_t at = offsets[ranges[r].first];
    for (auto &w : W) { w.cursor.push_back(at); at += w.cnt[r]; }
  }

  // ---- pass B: each worker groups every chunk of its slice by range, stably; each range's part goes to the slice's
  // cursor in that range ----
  rc = on_workers(W, [&](Worker &w, char *err, size_t err_cap) -> int {
    const uint64_t n_w = w.s1 - w.s0;
    if (!n_w) return KUQ_OK;
    const int grid = device_sm_count() * 8;
    const int rbits = bits_for(R);
    auto stream_need = [&](uint64_t c, size_t *sort_tmp) -> cudaError_t {
      *sort_tmp = 0;
      return cub::DeviceRadixSort::SortPairs((void *)nullptr, *sort_tmp, (uint32_t *)nullptr, (uint32_t *)nullptr, (ull *)nullptr,
                                             (ull *)nullptr, (int64_t)c, 0, rbits);
    };
    auto fits = [&](uint64_t c, size_t t) { return c * (2 * pair_sz + 24) + t + (uint64_t)R * 12 + 8 * 16 <= budget; };
    uint64_t chunk = std::min(n_w, PinnedBounce::CH / pair_sz);
    size_t stmp = 0;
    DB_CU(stream_need(chunk, &stmp));
    while (chunk > 1 && !fits(chunk, stmp)) { chunk /= 2; DB_CU(stream_need(chunk, &stmp)); }
    if (!fits(chunk, stmp))
      return seterr(KUQ_E_CAPACITY, err, err_cap, "db_sort: %u ranges do not fit KUQ_DB_SORT_BUDGET = %llu bytes", R,
                    (unsigned long long)budget);
    DevBuf<uint8_t> d_chunk, d_grp, d_tmp;
    DevBuf<uint32_t> d_rid, d_rid2, d_starts;
    DevBuf<ull> d_idx, d_idx2, d_cnt;
    DB_CU(get(d_chunk, chunk * pair_sz));
    DB_CU(get(d_grp, chunk * pair_sz));
    DB_CU(get(d_rid, chunk));
    DB_CU(get(d_rid2, chunk));
    DB_CU(get(d_idx, chunk));
    DB_CU(get(d_idx2, chunk));
    DB_CU(get(d_starts, R));
    DB_CU(get(d_cnt, R));
    DB_CU(get(d_tmp, stmp));
    std::vector<uint64_t> &cursor = w.cursor;
    std::vector<uint64_t> cnt(R), pos(R);
    DB_CU(cudaMemcpyAsync(d_starts, starts.data(), R * 4ull, cudaMemcpyHostToDevice, w.st));
    const uint8_t *in = body + w.s0 * pair_sz;
    DB_CU(w.bounce->h2d(d_chunk, in, chunk * pair_sz, w.st));
    for (uint64_t s = 0; s < n_w; s += chunk) {
      const uint64_t m = std::min(chunk, n_w - s);
      DB_CU(cudaMemsetAsync(d_cnt, 0, R * 8ull, w.st));
      k_dbs_range_of<<<grid, 256, 0, w.st>>>(d_chunk, m, g.key_len, g.k, nt, d_starts, R, d_rid, d_idx, d_cnt);
      size_t need = stmp;
      DB_CU(cub::DeviceRadixSort::SortPairs(d_tmp.get(), need, d_rid.get(), d_rid2.get(), d_idx.get(), d_idx2.get(), (int64_t)m, 0, rbits, w.st));
      k_dbs_emit<<<grid, 256, 0, w.st>>>(d_chunk, d_idx2, m, g.key_len, 0, d_grp);
      DB_CU(cudaGetLastError());
      if (s + m < n_w)                                               // the host copy of the next chunk overlaps these kernels
        DB_CU(w.bounce->h2d(d_chunk, in + (s + m) * pair_sz, std::min(chunk, n_w - s - m) * pair_sz, w.st));
      DB_CU(cudaMemcpyAsync(cnt.data(), d_cnt, R * 8ull, cudaMemcpyDeviceToHost, w.st));
      const uint8_t *grp = nullptr;
      DB_CU(w.bounce->d2h(&grp, d_grp, m * pair_sz, w.st));
      uint64_t at = 0;
      for (uint32_t r = 0; r < R; r++) { pos[r] = at; at += cnt[r]; }
      std::vector<std::thread> th;
      const uint32_t per = (R + PinnedBounce::NT - 1) / PinnedBounce::NT;
      for (uint32_t a = 0; a < R; a += per)
        th.emplace_back([&, a] {
          for (uint32_t r = a; r < std::min(R, a + per); r++)
            if (cnt[r]) memcpy(obody + cursor[r] * pair_sz, grp + pos[r] * pair_sz, cnt[r] * pair_sz);
        });
      for (auto &x : th) x.join();
      for (uint32_t r = 0; r < R; r++) cursor[r] += cnt[r];
    }
    return KUQ_OK;
  }, err, err_cap);
  if (rc) return rc;

  // ---- pass C: the ranges split into contiguous groups, one per worker; each range sorted in place ----
  {
    const std::vector<size_t> first = group_ranges(offsets, ranges, (int)n_dev, 2 * pair_sz + PASS_C_REC);
    for (uint32_t w = 0; w < n_dev; w++) { W[w].group_first = first[w]; W[w].group_end = first[w + 1]; }
  }
  rc = on_workers(W, [&](Worker &w, char *err, size_t err_cap) -> int {
    if (w.group_first == w.group_end) return KUQ_OK;
    Core c;
    DB_CU(core_alloc(c, max_rec, pair_sz, ctmp));
    for (size_t i = w.group_first; i < w.group_end; i++) {
      const auto &r = ranges[i];
      const uint64_t a = offsets[r.first], m = offsets[r.second] - a;
      DB_CU(w.bounce->to_device(c.in, obody + a * pair_sz, m * pair_sz, w.st));
      DB_CU(core_sort(c, m, g, (uint32_t)r.first, bits_for(r.second - r.first), zero_vals, nullptr, w.st));
      DB_CU(w.bounce->to_host(obody + a * pair_sz, c.out, m * pair_sz, w.st));
    }
    return KUQ_OK;
  }, err, err_cap);
  if (rc) return rc;
  *n_passes = R ? R : 1;
  return KUQ_OK;
}

// records per dense id of n 12-byte records, added to counts[0, n_ids); *bad = 1 when a value is n_ids or more
void launch_value_counts(const uint8_t *pairs, uint64_t n, uint32_t n_ids, unsigned long long *counts, uint32_t *bad,
                         cudaStream_t st) {
  if (!n) return;
  const uint32_t SHARED_IDS = 12288;      // 48 KiB of 32-bit counters: as much shared memory as a block gets by default
  uint64_t grid = std::min<uint64_t>((uint64_t)device_sm_count() * 4, (n + 255) / 256);
  grid = std::max<uint64_t>(grid, (n >> 31) + 1);   // fewer than 2^31 records per block: its 32-bit counters hold
  if (n_ids <= SHARED_IDS)
    k_value_counts<true><<<(unsigned)grid, 256, n_ids * 4, st>>>(pairs, n, n_ids, counts, bad);
  else
    k_value_counts<false><<<(unsigned)grid, 256, 0, st>>>(pairs, n, n_ids, counts, bad);
}

}  // namespace kuq
