// k-mer set of a FASTA library on the GPU: step 1 of build_db.sh (scripts/build_db.sh:116-147), which the reference
// hands to `jellyfish count -m k -C` of Jellyfish 1.  Output = one record per distinct canonical k-mer of the
// library's scanner windows (KmerScanner, krakenutil.cpp:239-282; canonical_representation, krakendb.cpp:238-246) with
// its number of occurrences, in ascending key order.  Jellyfish writes hash order; only db_shrink reads the order.
//
//  add    (per batch of sequences, pieces of a long sequence overlap by k - 1 like set_lcas's)
//    k_ks_mark + k_ks_pack     sequence starts, 2-bit codes and non-ACGT mask per 32 positions (k_pack's conversion)
//    k_ks_windows              valid-window mask per 32 positions → the packed library (12 B per 32 bases), and the
//                              histogram of the top 16 bits of every valid window's canonical k-mer
//  next   (per pass = a run of histogram buckets whose windows fit the HBM budget)
//    k_ks_extract              windows whose bucket is in the pass's range → keys (warp ballot, one atomic per warp)
//    CUB DeviceRadixSort::SortKeys over the low 2k bits
//    k_ks_heads_count / k_ks_heads_write + CUB scan of the tile counts: position of every run of equal keys
//    k_ks_emit                 (key, count) → database records of key_len(k) + 4 bytes, chunk by chunk to the host
//
// The packed library stays in HBM when it fits next to the working set of a pass that holds every window; otherwise it
// lives in pinned host memory and is streamed back once per pass on a copy stream, double-buffered against extraction.
#include "kuq_kernels.cuh"
#include "kuq_kmerpack.cuh"
#include "../../include/kuq.h"

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

namespace kuq {

// bit of position pos[i] (relative to the batch) in mask[], i < n: sequence starts (with the end of the text), or the
// starts of the windows the scanner skips
__global__ void k_ks_mark(const uint64_t *pos, uint32_t n, uint32_t *mask) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    atomicOr(mask + (pos[i] >> 5), 1u << (pos[i] & 31));
}

// One thread converts 16 bases (one 16-byte load), two lanes make a block of 32: blocks [0, nb].  Positions at or past
// len are ambiguous.  text: 16-byte aligned with 16 bytes of slack.
__global__ void __launch_bounds__(256) k_ks_pack(const char *text, uint64_t len, uint64_t nb, uint64_t *codes, uint32_t *amb) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t h_end = (nb + 1) * 2, stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t h0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~31ull; h0 < h_end; h0 += stride) {
    const uint64_t h = h0 + lane, pos0 = h * 16;
    uint32_t code32 = 0, amb16 = 0xFFFFu;
    if (h < h_end && pos0 < len) {
      const uint4 v = __ldg(reinterpret_cast<const uint4 *>(text + pos0));
      const uint32_t wd[4] = {v.x, v.y, v.z, v.w};
      amb16 = 0;
#pragma unroll
      for (int i = 0; i < 16; i++) {
        uint32_t code;
        const bool ok = base_code((wd[i >> 2] >> (8 * (i & 3))) & 0xFFu, code);
        code32 |= code << (2 * (15 - i));
        amb16 |= ok ? 0u : 1u << i;
      }
      if (len - pos0 < 16) amb16 |= 0xFFFFu & ~((1u << (len - pos0)) - 1);
    }
    const uint32_t code_o = __shfl_xor_sync(0xFFFFFFFFu, code32, 1), amb_o = __shfl_xor_sync(0xFFFFFFFFu, amb16, 1);
    if (!(lane & 1) && h < h_end) {
      codes[h >> 1] = ((uint64_t)code32 << 32) | code_o;
      amb[h >> 1] = amb16 | (amb_o << 16);
    }
  }
}

void ks_scanner_skips(const char *s, uint64_t len, uint32_t k, std::vector<char> &clean, std::vector<uint64_t> &drop_ends) {
  // the automaton clean_read replays for classification
  clean.clear();
  drop_ends.clear();
  int loaded = 0;
  bool skip = false;
  for (uint64_t i = 0; i < len; i++) {
    const char c = s[i];
    if (c == '\n' || c == '\r') {
      if (skip) loaded--;
      skip = true;
      continue;
    }
    bool emit = false;
    if (!skip && ++loaded == (int)k) { emit = true; loaded = (int)k - 1; }
    skip = false;
    if (!emit && clean.size() >= k - 1) drop_ends.push_back(clean.size());
    clean.push_back(c);
  }
}

cudaError_t KsStager::init(uint32_t k_, uint64_t batch_cap_, uint64_t max_seqs_) {
  k = k_;
  batch_cap = batch_cap_;
  max_seqs = max_seqs_;
  n_sm = device_sm_count();
  const uint64_t nb_cap = batch_cap / 32 + 2;
  cudaError_t e = cudaSuccess;
  for (int b = 0; b < 2 && e == cudaSuccess; b++) {
    if ((e = staged[b].alloc(cudaEventDisableTiming)) != cudaSuccess || (e = h_text[b].alloc(batch_cap)) != cudaSuccess) break;
    e = h_offs[b].alloc(max_seqs + 1);
  }
  if (e == cudaSuccess) e = d_text.alloc(batch_cap + 32);
  if (e == cudaSuccess) e = d_offs.alloc(max_seqs + 1);
  if (e == cudaSuccess) e = d_codes.alloc(nb_cap + 1);
  if (e == cudaSuccess) e = d_amb.alloc(nb_cap + 1);
  if (e == cudaSuccess) e = d_start.alloc(nb_cap + 2);
  if (e == cudaSuccess) e = d_drop.alloc(nb_cap + 2);
  if (e != cudaSuccess) { (void)cudaGetLastError(); return e; }
  h_offs[0][0] = 0;
  return cudaSuccess;
}

void KsStager::release_device() {
  d_text.reset(); d_offs.reset(); d_codes.reset(); d_amb.reset(); d_start.reset(); d_drop.reset(); d_drops.reset();
  drop_cap = 0;
  for (int b = 0; b < 2; b++) { h_text[b].reset(); h_offs[b].reset(); }
}

// Sequence boundary (seq_start .. fill is one piece): keep it when it holds a window
void KsStager::close_piece() {
  if (fill - seq_start >= k) h_offs[cur][++n_seqs] = fill;
  else fill = seq_start;
  seq_start = fill;
}

// append bases of the open sequence; a full batch cuts it, the next piece starts with the last k - 1 bases
int KsStager::append(const char *p, uint64_t n) {
  while (n) {
    if (fill == batch_cap) {
      const uint64_t piece = fill - seq_start, c = std::min<uint64_t>(piece, k - 1);
      carry.assign(h_text[cur] + fill - c, h_text[cur] + fill);
      close_piece();
      int rc = flush();
      if (rc) return rc;
      memcpy(h_text[cur], carry.data(), c);
      fill = c;
    }
    const uint64_t take = std::min(n, batch_cap - fill);
    memcpy(h_text[cur] + fill, p, take);
    fill += take;
    p += take;
    n -= take;
  }
  return 0;
}

int KsStager::add_clean(const char *c, uint64_t n, const std::vector<uint64_t> &ends) {
  if (n < k) return 0;                             // no window
  if (full()) {
    int rc = flush();
    if (rc) return rc;
  }
  seq_start = fill;
  uint64_t done = 0;
  for (uint64_t e : ends) {
    int rc = append(c + done, e + 1 - done);
    if (rc) return rc;
    done = e + 1;
    drops.push_back(fill - k);                     // base e sits at fill - 1 with its k - 1 predecessors in the piece
  }
  int rc = append(c + done, n - done);
  if (rc) return rc;
  close_piece();
  return 0;
}

int KsStager::add_sequence(const char *s, uint64_t n) {
  if (n < k) return 0;
  if (!memchr(s, '\n', n) && !memchr(s, '\r', n)) {
    static const std::vector<uint64_t> none;
    return add_clean(s, n, none);
  }
  ks_scanner_skips(s, n, k, clean, drop_ends);
  return add_clean(clean.data(), clean.size(), drop_ends);
}

cudaError_t KsStager::stage(cudaStream_t st) {
  const int b = cur;
  len = fill;
  nb = (len + 31) / 32;
  const uint64_t n = n_seqs;
  cudaError_t e;
  if ((e = cudaMemcpyAsync(d_text, h_text[b], len, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
  if ((e = cudaMemcpyAsync(d_offs, h_offs[b], (n + 1) * 8, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
  if ((e = cudaEventRecord(staged[b], st)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(d_start, 0, (nb + 2) * 4, st)) != cudaSuccess) return e;
  k_ks_mark<<<(unsigned)std::min<uint64_t>((n + 256) / 256, (uint64_t)n_sm * 8), 256, 0, st>>>(d_offs, (uint32_t)n + 1, d_start);
  const uint64_t nd = drops.size();
  has_drops = nd != 0;
  if (nd) {                                         // sequences with line breaks (rare): the windows the scanner skips
    if (nd > drop_cap) {
      drop_cap = std::max<uint64_t>(nd, 1 << 16);
      if ((e = d_drops.alloc(drop_cap)) != cudaSuccess) { drop_cap = 0; return e; }
    }
    if ((e = cudaMemcpyAsync(d_drops, drops.data(), nd * 8, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;   // pageable: staged now
    if ((e = cudaMemsetAsync(d_drop, 0, (nb + 2) * 4, st)) != cudaSuccess) return e;
    k_ks_mark<<<(unsigned)std::min<uint64_t>((nd + 255) / 256, (uint64_t)n_sm * 8), 256, 0, st>>>(d_drops, (uint32_t)nd, d_drop);
    drops.clear();
  }
  k_ks_pack<<<(unsigned)std::min<uint64_t>((2 * (nb + 1) + 255) / 256, (uint64_t)n_sm * 16), 256, 0, st>>>(d_text, len, nb, d_codes, d_amb);
  return cudaGetLastError();
}

cudaError_t KsStager::next() {
  cur ^= 1;
  const cudaError_t e = cudaEventSynchronize(staged[cur]);
  fill = seq_start = 0;
  n_seqs = 0;
  h_offs[cur][0] = 0;
  return e;
}

namespace {

constexpr uint32_t HIST_BITS = 16;                 // histogram over the top 16 bits of the canonical k-mer
constexpr uint32_t N_BUCKETS = 1u << HIST_BITS;
constexpr int TILE_THREADS = 256, TILE_ITEMS = 8, TILE = TILE_THREADS * TILE_ITEMS;
constexpr uint64_t CHUNK_RECORDS = 1ull << 22;     // records per device → host copy
constexpr uint64_t DEFAULT_BATCH = 256ull << 20;   // bases per batch

__host__ __device__ __forceinline__ uint32_t bucket_of(uint64_t canon, uint32_t k) {
  return 2 * k > HIST_BITS ? (uint32_t)(canon >> (2 * k - HIST_BITS)) : (uint32_t)canon;
}

// Warp per block j < nb, lane = window start 32j + lane (valid: ks_window_ok).  Writes the library segment (codes[0..nb], valid[0..nb)) and counts every valid window's canonical k-mer into hist.
__global__ void __launch_bounds__(256) k_ks_windows(const uint64_t *codes, const uint32_t *amb, const uint32_t *start,
                                                    const uint32_t *drop, uint64_t nb, uint32_t k, uint64_t *lib_codes,
                                                    uint32_t *lib_valid, unsigned long long *hist) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < nb; j += warps) {
    const uint64_t a = codes[j], b = codes[j + 1];
    const bool ok = ks_window_ok(amb, start, drop, j, lane, k);
    const uint32_t valid = __ballot_sync(0xFFFFFFFFu, ok);
    if (ok) atomicAdd(hist + bucket_of(canonical_kmer(window_top(a, b, lane), k), k), 1ull);
    if (lane == 0) {
      lib_codes[j] = a;
      lib_valid[j] = valid;
      if (j == nb - 1) lib_codes[nb] = b;
    }
  }
}

// Warp per block: the valid windows whose bucket lies in [blo, bhi), compacted into keys (one atomic per warp).
__global__ void __launch_bounds__(256) k_ks_extract(const uint64_t *lib_codes, const uint32_t *lib_valid, uint64_t nb, uint32_t k,
                                                    uint32_t blo, uint32_t bhi, unsigned long long *keys,
                                                    unsigned long long *cursor, uint64_t cap) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < nb; j += warps) {
    const uint32_t valid = __ldg(lib_valid + j);
    if (!valid) continue;                                           // warp-uniform
    const uint64_t canon = canonical_kmer(window_top(__ldg(lib_codes + j), __ldg(lib_codes + j + 1), lane), k);
    const uint32_t bk = bucket_of(canon, k);
    const bool keep = ((valid >> lane) & 1u) && bk >= blo && bk < bhi;
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, keep);
    if (!m) continue;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(cursor, (unsigned long long)__popc(m));
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    const uint64_t at = base + __popc(m & ((1u << lane) - 1));
    if (keep && at < cap) keys[at] = canon;
  }
}

// Run heads of the sorted keys (i = 0 or keys[i] != keys[i - 1]): per tile of TILE keys, their number ...
__global__ void __launch_bounds__(TILE_THREADS) k_ks_heads_count(const unsigned long long *keys, uint64_t n,
                                                                 unsigned long long *tile_counts) {
  typedef cub::BlockReduce<uint32_t, TILE_THREADS> Reduce;
  __shared__ typename Reduce::TempStorage tmp;
  const uint64_t base = (uint64_t)blockIdx.x * TILE;
  uint32_t c = 0;
#pragma unroll
  for (int q = 0; q < TILE_ITEMS; q++) {
    const uint64_t i = base + q * TILE_THREADS + threadIdx.x;
    c += i < n && (i == 0 || keys[i] != keys[i - 1]);
  }
  const uint32_t total = Reduce(tmp).Sum(c);
  if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
}

// ... and, after an exclusive scan of those counts, the position of every head: pos[run] = i
__global__ void __launch_bounds__(TILE_THREADS) k_ks_heads_write(const unsigned long long *keys, uint64_t n,
                                                                 const unsigned long long *tile_off, unsigned long long *pos) {
  typedef cub::BlockScan<uint32_t, TILE_THREADS> Scan;
  __shared__ typename Scan::TempStorage tmp;
  const uint64_t i0 = (uint64_t)blockIdx.x * TILE + (uint64_t)threadIdx.x * TILE_ITEMS;   // blocked: 8 keys per thread
  uint32_t heads = 0;
#pragma unroll
  for (int q = 0; q < TILE_ITEMS; q++) {
    const uint64_t i = i0 + q;
    heads |= (uint32_t)(i < n && (i == 0 || keys[i] != keys[i - 1])) << q;
  }
  uint32_t before;
  Scan(tmp).ExclusiveSum((uint32_t)__popc(heads), before);
  unsigned long long at = tile_off[blockIdx.x] + before;
#pragma unroll
  for (int q = 0; q < TILE_ITEMS; q++)
    if ((heads >> q) & 1u) pos[at++] = i0 + q;
}

// Records [r0, r1): key = keys[pos[r]], count = pos[r + 1] - pos[r] saturated at 2^32 - 1, in the file's layout
// (key_len little-endian key bytes + u32 value; the inverse of k_widen_records)
__global__ void k_ks_emit(const unsigned long long *keys, const unsigned long long *pos, uint64_t r0, uint64_t r1,
                          uint32_t key_len, uint8_t *out) {
  const uint32_t rec = key_len + 4;
  for (uint64_t r = r0 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < r1; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t p = pos[r], cnt = pos[r + 1] - p;
    const uint64_t key = keys[p];
    const uint32_t val = cnt > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)cnt;
    uint8_t *o = out + (r - r0) * rec;
    for (uint32_t b = 0; b < key_len; b++) o[b] = (uint8_t)(key >> (8 * b));
    for (uint32_t b = 0; b < 4; b++) o[key_len + b] = (uint8_t)(val >> (8 * b));
  }
}

uint64_t env_u64(const char *name, uint64_t dflt) {
  const char *s = getenv(name);
  if (!s || !*s) return dflt;
  char *end = nullptr;
  const unsigned long long v = strtoull(s, &end, 10);
  return (end && *end == 0 && v) ? (uint64_t)v : dflt;
}

uint64_t seg_bytes(uint64_t nb) { return 8 * (nb + 1) + 4 * nb; }   // codes[nb + 1], valid[nb]

}  // namespace
}  // namespace kuq

using namespace kuq;

struct kuq_kmer_set {
  int device = 0;
  uint32_t k = 0, key_len = 0;
  uint64_t budget = 0, batch_cap = 0, max_seqs = 0;
  std::string err;
  cudaStream_t st = nullptr, cp = nullptr;
  int n_sm = 0;
  // device memory of the set and its byte count; free device memory at creation and its low point during the passes
  std::map<void *, uint64_t> dev;
  uint64_t dev_bytes = 0, free0 = 0, free_min = 0;
  // batches
  KsStager in;
  uint8_t *d_spill = nullptr;
  unsigned long long *d_hist = nullptr, *d_cursor = nullptr;
  uint64_t positions = 0;
  // the packed library
  struct Segment {
    uint64_t nb;
    uint8_t *dev, *host;
  };
  std::vector<Segment> segs;
  bool lib_on_device = true;
  uint64_t lib_dev_bytes = 0, max_seg_bytes = 0;
  // passes
  bool planned = false;
  struct Pass {
    uint32_t lo, hi;
    uint64_t n;
  };
  std::vector<Pass> passes;
  uint64_t ws_estimate = 0, cap = 0, windows = 0;
  unsigned long long *d_keys[2] = {nullptr, nullptr}, *d_tiles = nullptr, *d_tile_off = nullptr;
  void *d_tmp = nullptr;
  uint64_t tmp_bytes = 0, sort_tmp = 0, scan_tmp = 0;
  uint8_t *d_chunk = nullptr, *h_chunk = nullptr;
  uint8_t *d_stream[2] = {nullptr, nullptr};
  cudaEvent_t ready[2] = {nullptr, nullptr}, freed[2] = {nullptr, nullptr};
  unsigned long long *h_scalar = nullptr;
  size_t pass_idx = 0;
  bool pass_ready = false;
  unsigned long long *sorted = nullptr, *pos = nullptr;
  uint64_t pass_runs = 0, run_cursor = 0, key_ct = 0;
  // stage timing: (stage, start, end) event pairs, summed by kuq_kmer_set_stats
  std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> timers;
  double stage_ms[5] = {0, 0, 0, 0, 0};

  int fail(int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    err = buf;
    return code;
  }
  template <typename T>
  cudaError_t alloc(T **p, uint64_t bytes) {
    cudaError_t e = cudaMalloc((void **)p, bytes ? bytes : 1);
    if (e != cudaSuccess) { (void)cudaGetLastError(); return e; }
    dev[*p] = bytes;
    dev_bytes += bytes;
    return e;
  }
  template <typename T>
  void release(T *&p) {
    if (!p) return;
    auto it = dev.find((void *)p);
    if (it != dev.end()) { dev_bytes -= it->second; dev.erase(it); }
    cudaFree((void *)p);
    p = nullptr;
  }
  void mark(int stage, bool begin) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) { (void)cudaGetLastError(); return; }
    cudaEventRecord(e, st);
    if (begin) timers.push_back({stage, {e, nullptr}});
    else timers.back().second.second = e;
  }
};

#define KS_CU(call)                                                                                       \
  do {                                                                                                    \
    cudaError_t e__ = (call);                                                                             \
    if (e__ != cudaSuccess) return h->fail(KUQ_E_CUDA, "%s: %s", #call, cudaGetErrorString(e__)); \
  } while (0)
#define KS_ALLOC(p, bytes)                                                                                     \
  do {                                                                                                         \
    if (h->alloc(&(p), (bytes)) != cudaSuccess)                                                               \
      return h->fail(KUQ_E_NOMEM, "cannot allocate %llu bytes of device memory", (unsigned long long)(bytes)); \
  } while (0)

namespace {

// device bytes one pass over n windows needs besides the library: two key buffers (the second holds the run positions
// after the sort), tile counts / offsets, CUB's temporary storage, the records of one copy-back chunk
uint64_t pass_bytes(const kuq_kmer_set *h, uint64_t n, uint64_t *sort_tmp = nullptr, uint64_t *scan_tmp = nullptr) {
  const uint64_t tiles = (n + TILE - 1) / TILE;
  size_t a = 0, b = 0;
  cub::DoubleBuffer<unsigned long long> db(nullptr, nullptr);
  cub::DeviceRadixSort::SortKeys(nullptr, a, db, (int64_t)std::max<uint64_t>(n, 1), 0, (int)(2 * h->k));
  cub::DeviceScan::ExclusiveSum(nullptr, b, (unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                (int64_t)(tiles + 1));
  if (sort_tmp) *sort_tmp = a;
  if (scan_tmp) *scan_tmp = b;
  return 2 * 8 * (n + 1) + 2 * 8 * (tiles + 1) + std::max<uint64_t>(a, b) + std::min(n, CHUNK_RECORDS) * (h->key_len + 4);
}

int copy_segment_to_host(kuq_kmer_set *h, kuq_kmer_set::Segment &s) {
  const uint64_t bytes = seg_bytes(s.nb);
  KS_CU(cudaHostAlloc((void **)&s.host, bytes, cudaHostAllocDefault));
  KS_CU(cudaMemcpyAsync(s.host, s.dev, bytes, cudaMemcpyDeviceToHost, h->st));
  return 0;
}

// the open batch → packed segment + histogram, asynchronously on h->st
int flush(kuq_kmer_set *h) {
  KsStager &in = h->in;
  if (in.empty()) { in.fill = in.seq_start = 0; return 0; }
  h->mark(0, true);
  KS_CU(in.stage(h->st));
  const uint64_t len = in.len, nb = in.nb;
  // placement: the library stays in HBM while it fits next to a pass holding every window seen so far
  h->positions += len;
  const uint64_t sb = seg_bytes(nb);
  if (h->lib_on_device && h->lib_dev_bytes + sb + pass_bytes(h, h->positions) > h->budget) {
    for (auto &s : h->segs) {
      int rc = copy_segment_to_host(h, s);
      if (rc) return rc;
    }
    KS_CU(cudaStreamSynchronize(h->st));
    for (auto &s : h->segs) h->release(s.dev);
    h->lib_on_device = false;
    h->lib_dev_bytes = 0;
  }
  kuq_kmer_set::Segment s{nb, nullptr, nullptr};
  uint8_t *dst = h->d_spill;
  if (h->lib_on_device) {
    KS_ALLOC(s.dev, sb);
    dst = s.dev;
    h->lib_dev_bytes += sb;
  }
  k_ks_windows<<<(unsigned)std::min<uint64_t>((nb + 7) / 8, (uint64_t)h->n_sm * 16), 256, 0, h->st>>>(
      in.d_codes, in.d_amb, in.d_start, in.has_drops ? in.d_drop.get() : nullptr, nb, h->k, (uint64_t *)dst,
      (uint32_t *)(dst + 8 * (nb + 1)), h->d_hist);
  KS_CU(cudaGetLastError());
  if (!h->lib_on_device) {
    s.dev = h->d_spill;
    int rc = copy_segment_to_host(h, s);
    s.dev = nullptr;
    if (rc) return rc;
  }
  h->max_seg_bytes = std::max(h->max_seg_bytes, sb);
  h->segs.push_back(s);
  h->mark(0, false);
  KS_CU(in.next());
  return 0;
}

int plan(kuq_kmer_set *h) {
  int rc = flush(h);
  if (rc) return rc;
  KS_CU(cudaStreamSynchronize(h->st));
  h->in.release_device();
  h->release(h->d_spill);
  std::vector<unsigned long long> hist(N_BUCKETS);
  KS_CU(cudaMemcpy(hist.data(), h->d_hist, N_BUCKETS * 8, cudaMemcpyDeviceToHost));
  uint64_t total = 0, biggest = 0;
  for (auto c : hist) { total += c; biggest = std::max<uint64_t>(biggest, c); }
  h->windows = total;
  // capacity: the most windows a pass can hold next to the library (or its two stream buffers)
  const uint64_t fixed = h->dev_bytes + (h->lib_on_device ? 0 : 2 * h->max_seg_bytes);
  const uint64_t avail = h->budget > fixed ? h->budget - fixed : 0;
  uint64_t lo = 0, hi = std::max<uint64_t>(total, 1);
  if (pass_bytes(h, hi) <= avail) lo = hi;
  while (lo < hi) {
    const uint64_t mid = lo + (hi - lo + 1) / 2;
    if (pass_bytes(h, mid) <= avail) lo = mid; else hi = mid - 1;
  }
  h->cap = lo;
  if (biggest > h->cap)
    return h->fail(KUQ_E_CAPACITY,
                   "one k-mer bucket holds %llu windows but a pass under the HBM budget of %llu bytes holds at "
                   "most %llu; raise KUQ_KMER_SET_BUDGET",
                   (unsigned long long)biggest, (unsigned long long)h->budget, (unsigned long long)h->cap);
  uint64_t max_n = 0;
  for (uint32_t b = 0; b < N_BUCKETS;) {
    kuq_kmer_set::Pass p{b, b, 0};
    while (p.hi < N_BUCKETS && p.n + hist[p.hi] <= h->cap) p.n += hist[p.hi++];
    b = p.hi;
    if (p.n) h->passes.push_back(p);
    max_n = std::max(max_n, p.n);
  }
  if (h->passes.size() > 1) {                       // a pass's range is a run of buckets: cover [0, N_BUCKETS) whole
    h->passes.front().lo = 0;
    for (size_t i = 1; i < h->passes.size(); i++) h->passes[i].lo = h->passes[i - 1].hi;
    h->passes.back().hi = N_BUCKETS;
  } else if (h->passes.size() == 1) {
    h->passes[0].lo = 0;
    h->passes[0].hi = N_BUCKETS;
  }
  h->planned = true;
  if (h->passes.empty()) { h->ws_estimate = h->dev_bytes; return 0; }
  h->ws_estimate = fixed + pass_bytes(h, max_n, &h->sort_tmp, &h->scan_tmp);
  h->tmp_bytes = std::max(h->sort_tmp, h->scan_tmp);
  const uint64_t tiles = (max_n + TILE - 1) / TILE;
  KS_ALLOC(h->d_keys[0], 8 * (max_n + 1));
  KS_ALLOC(h->d_keys[1], 8 * (max_n + 1));
  KS_ALLOC(h->d_tiles, 8 * (tiles + 1));
  KS_ALLOC(h->d_tile_off, 8 * (tiles + 1));
  KS_ALLOC(h->d_tmp, h->tmp_bytes);
  const uint64_t chunk = std::min(max_n, CHUNK_RECORDS) * (h->key_len + 4);
  KS_ALLOC(h->d_chunk, chunk);
  KS_CU(cudaHostAlloc((void **)&h->h_chunk, chunk, cudaHostAllocDefault));
  if (!h->lib_on_device) {
    KS_ALLOC(h->d_stream[0], h->max_seg_bytes);
    KS_ALLOC(h->d_stream[1], h->max_seg_bytes);
  }
  return 0;
}

int run_pass(kuq_kmer_set *h) {
  const kuq_kmer_set::Pass &p = h->passes[h->pass_idx];
  const int grid_x = h->n_sm * 16;
  h->mark(1, true);
  KS_CU(cudaMemsetAsync(h->d_cursor, 0, 8, h->st));
  uint32_t i_host = 0;
  for (auto &s : h->segs) {
    const uint8_t *src = s.dev;
    if (!src) {                                     // host segment: stream it in on the copy stream
      const int b = i_host++ & 1;
      KS_CU(cudaStreamWaitEvent(h->cp, h->freed[b], 0));
      KS_CU(cudaMemcpyAsync(h->d_stream[b], s.host, seg_bytes(s.nb), cudaMemcpyHostToDevice, h->cp));
      KS_CU(cudaEventRecord(h->ready[b], h->cp));
      KS_CU(cudaStreamWaitEvent(h->st, h->ready[b], 0));
      src = h->d_stream[b];
    }
    k_ks_extract<<<(unsigned)std::min<uint64_t>((s.nb + 7) / 8, (uint64_t)grid_x), 256, 0, h->st>>>(
        (const uint64_t *)src, (const uint32_t *)(src + 8 * (s.nb + 1)), s.nb, h->k, p.lo, p.hi, h->d_keys[0], h->d_cursor, p.n);
    if (!s.dev) KS_CU(cudaEventRecord(h->freed[(i_host - 1) & 1], h->st));
  }
  KS_CU(cudaGetLastError());
  h->mark(1, false);
  KS_CU(cudaMemcpyAsync(h->h_scalar, h->d_cursor, 8, cudaMemcpyDeviceToHost, h->st));
  KS_CU(cudaStreamSynchronize(h->st));
  if (*h->h_scalar != p.n)
    return h->fail(KUQ_E_STATE, "pass %zu extracted %llu windows, the histogram says %llu", h->pass_idx,
                   (unsigned long long)*h->h_scalar, (unsigned long long)p.n);
  const uint64_t n = p.n;
  h->mark(2, true);
  cub::DoubleBuffer<unsigned long long> db(h->d_keys[0], h->d_keys[1]);
  size_t tb = h->tmp_bytes;
  KS_CU(cub::DeviceRadixSort::SortKeys(h->d_tmp, tb, db, (int64_t)n, 0, (int)(2 * h->k), h->st));
  h->mark(2, false);
  size_t free_b = 0, total_b = 0;
  KS_CU(cudaMemGetInfo(&free_b, &total_b));          // every buffer of the pass exists now
  h->free_min = std::min<uint64_t>(h->free_min, free_b);
  h->sorted = db.Current();
  h->pos = db.Alternate();
  h->mark(3, true);
  const uint64_t tiles = (n + TILE - 1) / TILE;
  KS_CU(cudaMemsetAsync(h->d_tiles + tiles, 0, 8, h->st));
  k_ks_heads_count<<<(unsigned)tiles, TILE_THREADS, 0, h->st>>>(h->sorted, n, h->d_tiles);
  tb = h->tmp_bytes;
  KS_CU(cub::DeviceScan::ExclusiveSum(h->d_tmp, tb, h->d_tiles, h->d_tile_off, (int64_t)(tiles + 1), h->st));
  k_ks_heads_write<<<(unsigned)tiles, TILE_THREADS, 0, h->st>>>(h->sorted, n, h->d_tile_off, h->pos);
  KS_CU(cudaGetLastError());
  KS_CU(cudaMemcpyAsync(h->h_scalar, h->d_tile_off + tiles, 8, cudaMemcpyDeviceToHost, h->st));
  KS_CU(cudaStreamSynchronize(h->st));
  h->pass_runs = *h->h_scalar;
  *h->h_scalar = n;                                  // pos[n_runs] = n closes the last run
  KS_CU(cudaMemcpyAsync(h->pos + h->pass_runs, h->h_scalar, 8, cudaMemcpyHostToDevice, h->st));
  h->mark(3, false);
  h->run_cursor = 0;
  h->key_ct += h->pass_runs;
  h->pass_ready = true;
  return 0;
}

}  // namespace

extern "C" {

int kuq_kmer_set_create(int device, uint32_t k, uint64_t budget, kuq_kmer_set **out, char *err, uint64_t err_cap) {
  auto say = [&](int code, const char *msg) {
    if (err && err_cap) snprintf(err, err_cap, "%s", msg);
    return code;
  };
  if (!out) return say(KUQ_E_INVALID_ARG, "NULL handle pointer");
  *out = nullptr;
  if (k < 1 || k > 31) return say(KUQ_E_UNSUPPORTED_K, "k must be 1..31");
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
    (void)cudaGetLastError();
    return say(KUQ_E_NO_DEVICE, "no CUDA device (there is no CPU path)");
  }
  if (device < 0 || device >= n_dev || cudaSetDevice(device) != cudaSuccess) return say(KUQ_E_INVALID_ARG, "bad device ordinal");
  kuq_kmer_set *h = new kuq_kmer_set;
  h->device = device;
  h->k = k;
  h->key_len = (2 * k + 7) / 8;
  h->n_sm = device_sm_count();
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { delete h; return say(KUQ_E_CUDA, "cudaMemGetInfo failed"); }
  h->free0 = h->free_min = free_b;
  h->budget = budget ? budget : env_u64("KUQ_KMER_SET_BUDGET", free_b / 4 * 3);
  h->batch_cap = std::max<uint64_t>(env_u64("KUQ_KMER_SET_BATCH", DEFAULT_BATCH), 2 * k + 32);
  h->max_seqs = std::min<uint64_t>(h->batch_cap / k + 2, 1ull << 22);
  h->in.flush = [h] { return flush(h); };
  auto bail = [&](int code) {
    std::string m = h->err;
    kuq_kmer_set_destroy(h);
    return say(code, m.c_str());
  };
  const uint64_t nb = h->batch_cap / 32 + 2;
  if (cudaStreamCreateWithFlags(&h->st, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&h->cp, cudaStreamNonBlocking) != cudaSuccess)
    return bail(h->fail(KUQ_E_CUDA, "cannot create streams"));
  for (int b = 0; b < 2; b++) {
    if (cudaEventCreateWithFlags(&h->ready[b], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->freed[b], cudaEventDisableTiming) != cudaSuccess)
      return bail(h->fail(KUQ_E_CUDA, "cannot create events"));
    cudaEventRecord(h->freed[b], h->cp);
  }
  if (h->in.init(k, h->batch_cap, h->max_seqs) != cudaSuccess)
    return bail(h->fail(KUQ_E_NOMEM, "cannot allocate the batch staging buffers"));
  if (cudaHostAlloc((void **)&h->h_scalar, 8, cudaHostAllocDefault) != cudaSuccess)
    return bail(h->fail(KUQ_E_NOMEM, "cannot allocate pinned memory"));
  if (h->alloc(&h->d_spill, seg_bytes(nb)) || h->alloc(&h->d_hist, 8ull * N_BUCKETS) || h->alloc(&h->d_cursor, 8))
    return bail(h->fail(KUQ_E_NOMEM, "cannot allocate the batch buffers on the device"));
  if (cudaMemsetAsync(h->d_hist, 0, 8ull * N_BUCKETS, h->st) != cudaSuccess) return bail(h->fail(KUQ_E_CUDA, "memset failed"));
  *out = h;
  return KUQ_OK;
}

int kuq_kmer_set_add(kuq_kmer_set *h, const char *bases, const uint64_t *offsets, uint32_t n_seqs) {
  if (!h) return KUQ_E_INVALID_ARG;
  if (h->planned) return h->fail(KUQ_E_STATE, "sequences added after the first kuq_kmer_set_next / _info");
  if (n_seqs && (!bases || !offsets)) return h->fail(KUQ_E_INVALID_ARG, "NULL sequence buffers");
  KS_CU(cudaSetDevice(h->device));
  for (uint32_t r = 0; r < n_seqs; r++) {
    if (offsets[r + 1] < offsets[r]) return h->fail(KUQ_E_INVALID_ARG, "offsets decrease at sequence %u", r);
    int rc = h->in.add_sequence(bases + offsets[r], offsets[r + 1] - offsets[r]);
    if (rc) return rc;
  }
  return KUQ_OK;
}

int kuq_kmer_set_next(kuq_kmer_set *h, void *records_out, uint64_t cap_records, uint64_t *n_out) {
  if (!h || !n_out || (cap_records && !records_out)) return KUQ_E_INVALID_ARG;
  *n_out = 0;
  KS_CU(cudaSetDevice(h->device));
  if (!h->planned) {
    int rc = plan(h);
    if (rc) return rc;
  }
  const uint32_t rec = h->key_len + 4;
  uint8_t *out = (uint8_t *)records_out;
  while (*n_out < cap_records && h->pass_idx < h->passes.size()) {
    if (!h->pass_ready) {
      int rc = run_pass(h);
      if (rc) return rc;
    }
    const uint64_t take = std::min(std::min(cap_records - *n_out, h->pass_runs - h->run_cursor), CHUNK_RECORDS);
    if (take) {
      h->mark(3, true);
      k_ks_emit<<<(unsigned)std::min<uint64_t>((take + 255) / 256, (uint64_t)h->n_sm * 16), 256, 0, h->st>>>(
          h->sorted, h->pos, h->run_cursor, h->run_cursor + take, h->key_len, h->d_chunk);
      KS_CU(cudaGetLastError());
      h->mark(3, false);
      h->mark(4, true);
      KS_CU(cudaMemcpyAsync(h->h_chunk, h->d_chunk, take * rec, cudaMemcpyDeviceToHost, h->st));
      h->mark(4, false);
      KS_CU(cudaStreamSynchronize(h->st));
      memcpy(out + *n_out * rec, h->h_chunk, take * rec);
      h->run_cursor += take;
      *n_out += take;
    }
    if (h->run_cursor == h->pass_runs) {
      h->pass_idx++;
      h->pass_ready = false;
    }
  }
  return KUQ_OK;
}

int kuq_kmer_set_info(kuq_kmer_set *h, uint64_t *key_ct, uint32_t *n_passes) {
  if (!h) return KUQ_E_INVALID_ARG;
  KS_CU(cudaSetDevice(h->device));
  if (!h->planned) {
    int rc = plan(h);
    if (rc) return rc;
  }
  if (key_ct) *key_ct = h->key_ct;
  if (n_passes) *n_passes = (uint32_t)h->passes.size();
  return KUQ_OK;
}

int kuq_kmer_set_stats(kuq_kmer_set *h, double *stage_ms5, uint64_t *windows, uint64_t *ws_estimate, uint64_t *peak_bytes,
                       int *lib_on_device) {
  if (!h) return KUQ_E_INVALID_ARG;
  KS_CU(cudaSetDevice(h->device));
  KS_CU(cudaStreamSynchronize(h->st));
  for (auto &t : h->timers) {
    float ms = 0;
    if (t.second.second && cudaEventElapsedTime(&ms, t.second.first, t.second.second) == cudaSuccess) h->stage_ms[t.first] += ms;
    cudaEventDestroy(t.second.first);
    if (t.second.second) cudaEventDestroy(t.second.second);
  }
  (void)cudaGetLastError();
  h->timers.clear();
  if (stage_ms5) memcpy(stage_ms5, h->stage_ms, sizeof h->stage_ms);
  if (windows) *windows = h->windows;
  if (ws_estimate) *ws_estimate = h->ws_estimate;
  if (peak_bytes) *peak_bytes = h->free0 - h->free_min;
  if (lib_on_device) *lib_on_device = h->lib_on_device ? 1 : 0;
  return KUQ_OK;
}

const char *kuq_kmer_set_last_error(const kuq_kmer_set *h) { return h ? h->err.c_str() : ""; }

void kuq_kmer_set_destroy(kuq_kmer_set *h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->st) cudaStreamSynchronize(h->st);
  if (h->cp) cudaStreamSynchronize(h->cp);
  for (auto &t : h->timers) {
    cudaEventDestroy(t.second.first);
    if (t.second.second) cudaEventDestroy(t.second.second);
  }
  for (auto &s : h->segs) {
    if (s.host) cudaFreeHost(s.host);
  }
  for (auto &kv : h->dev) cudaFree(kv.first);
  for (int b = 0; b < 2; b++)
    for (cudaEvent_t e : {h->ready[b], h->freed[b]})
      if (e) cudaEventDestroy(e);
  if (h->h_chunk) cudaFreeHost(h->h_chunk);
  if (h->h_scalar) cudaFreeHost(h->h_scalar);
  if (h->st) cudaStreamDestroy(h->st);
  if (h->cp) cudaStreamDestroy(h->cp);
  (void)cudaGetLastError();
  delete h;
}

}  // extern "C"
