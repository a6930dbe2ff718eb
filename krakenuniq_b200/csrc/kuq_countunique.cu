// Distinct k-mers of a FASTA library by HyperLogLog on the GPU: count_unique (src/count_unique.cpp:51-79), which
// krakenuniq-build runs to size Jellyfish's hash when --jellyfish-hash-size is not given (scripts/build_db.sh:125-129).
//
// count_unique cuts every sequence into pieces [i, i + 50000 + k - 1), i = 0, 50000, ..., runs a fresh KmerScanner over
// each, inserts every unambiguous forward k-mer into a dense sketch at precision p (4..18) and merges the pieces'
// sketches: the registers are the max over all pieces, n_observed counts every valid window.  Pieces overlap by k - 1
// bases, so over a sequence without line breaks they yield each window of the sequence once, and such a sequence is
// staged whole.  A sequence holding '\n' / '\r' is staged piece by piece as the scanner reads each one: it may read past
// the piece's end and yield a window the next piece yields again, which counts twice in n_observed.
//
//  add      (per batch, KsStager of kuq_kmerpack.cuh: 2-bit codes, non-ACGT mask, sequence starts, skipped windows)
//    k_cu_sketch<SMEM>   warp per 32 window starts: fmix64 of each valid window's forward k-mer, register max at run-time
//                        p, popcount of the valid windows into n_observed.  p <= 15: the block's own registers in
//                        shared memory, merged into the global ones with atomicMax at its end; p >= 16: the global
//                        registers, read before the atomicMax (late in a pass few ranks raise a register)
//  result   k_cu_hist    64-bin rank histogram of the registers → ertlCardinality on the host
#include "kuq_kernels.cuh"
#include "kuq_kmerpack.cuh"
#include "../../include/kuq.h"

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

namespace kuq {
namespace {

constexpr uint64_t PIECE = 50000;                  // SKIP_LEN, count_unique.cpp:26
constexpr uint64_t DEFAULT_BATCH = 256ull << 20;   // bases per batch
constexpr uint32_t SMEM_MAX_P = 15;                // 2^15 u32 registers = 128 KB of shared memory
constexpr int SKETCH_THREADS = 512;

template <bool SMEM>
__global__ void __launch_bounds__(SKETCH_THREADS) k_cu_sketch(const uint64_t *codes, const uint32_t *amb, const uint32_t *start,
                                                              const uint32_t *drop, uint64_t nb, uint32_t k, uint32_t p,
                                                              uint32_t *regs, unsigned long long *n_observed) {
  extern __shared__ uint32_t s_regs[];
  const uint32_t m = 1u << p, lane = threadIdx.x & 31;
  if (SMEM) {
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) s_regs[i] = 0;
    __syncthreads();
  }
  uint32_t *M = SMEM ? s_regs : regs;
  const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  uint32_t seen = 0;
  for (uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < nb; j += warps) {
    if (!ks_window_ok(amb, start, drop, j, lane, k)) continue;
    seen++;
    const uint64_t kmer = window_top(__ldg(codes + j), __ldg(codes + j + 1), lane) >> (64 - 2 * k);
    const uint64_t h = fmix64(kmer);                                       // hyperloglogplus.cpp:485-523
    const uint32_t idx = (uint32_t)(h >> (64 - p));
    const uint64_t w = h << p;
    const uint32_t rank = w ? (uint32_t)__clzll((long long)w) + 1 : 64 - p + 1;
    if (rank > *(volatile uint32_t *)(M + idx)) atomicMax(M + idx, rank);   // registers only grow: a stale read costs an atomic
  }
  seen = __reduce_add_sync(0xFFFFFFFFu, seen);
  if (lane == 0 && seen) atomicAdd(n_observed, (unsigned long long)seen);
  if (SMEM) {
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
      const uint32_t v = s_regs[i];
      if (v > regs[i]) atomicMax(regs + i, v);
    }
  }
}

// hist[r] = registers of rank r (ranks are at most 64 - 4 + 1)
__global__ void __launch_bounds__(256) k_cu_hist(const uint32_t *regs, uint32_t m, uint32_t *hist) {
  __shared__ uint32_t s[64];
  if (threadIdx.x < 64) s[threadIdx.x] = 0;
  __syncthreads();
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) atomicAdd(s + min(regs[i], 63u), 1u);
  __syncthreads();
  if (threadIdx.x < 64 && s[threadIdx.x]) atomicAdd(hist + threadIdx.x, s[threadIdx.x]);
}

// KmerScanner(seq, pos1, pos2) + next_kmer until NULL (krakenutil.cpp:208-282) over s[0, len): the characters it reads
// without line breaks (clean) and the clean positions where a window it does not yield ends (drop_ends).  Each call
// starts only while curr_pos < pos2 but reads on until k bases are loaded, past pos2 into the next piece and, at the
// end of the sequence, onto the string's terminating '\0' (ambiguous).  Positions past that are read as '\0' too; the
// reference reads memory beyond its string there.
void scan_piece(const char *s, uint64_t len, uint64_t pos1, uint64_t pos2, uint32_t k, std::vector<char> &clean,
                std::vector<uint64_t> &drop_ends) {
  clean.clear();
  drop_ends.clear();
  uint64_t curr = pos2 - pos1 + 1 < k ? pos2 : pos1;
  int64_t loaded = 0;
  uint64_t next_end = k - 1;                       // first clean window end not yet classified
  while (curr < pos2) {
    bool skip = false;
    if (loaded) loaded--;
    while (loaded < (int64_t)k) {
      if (skip) skip = false;
      else loaded++;
      const char c = curr < len ? s[curr] : '\0';
      curr++;
      if (c == '\n' || c == '\r') {
        --loaded;
        skip = true;
        continue;
      }
      clean.push_back(c);
    }
    const uint64_t end = clean.size() - 1;         // the window yielded: the last k characters read
    for (; next_end < end; next_end++) drop_ends.push_back(next_end);
    next_end = end + 1;
  }
  for (; next_end < clean.size(); next_end++) drop_ends.push_back(next_end);
}

}  // namespace
}  // namespace kuq

using namespace kuq;

struct kuq_count_unique {
  int device = 0;
  uint32_t k = 0, p = 0;
  std::string err;
  Stream st;
  KsStager in;
  DevBuf<uint32_t> d_regs, d_hist;
  DevBuf<unsigned long long> d_count;
  HostBuf<unsigned long long> h_count;
  int grid = 0;
  uint64_t bases = 0, windows = 0;
  std::vector<char> clean;
  std::vector<uint64_t> drop_ends;
  // (start, end) events of every sketch launch, summed by kuq_count_unique_stats
  std::vector<std::pair<Event, Event>> timers;
  double sketch_ms = 0;

  int fail(int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    err = buf;
    return code;
  }
};

#define CU_CU(call)                                                                                       \
  do {                                                                                                    \
    cudaError_t e__ = (call);                                                                             \
    if (e__ != cudaSuccess) return h->fail(KUQ_E_CUDA, "%s: %s", #call, cudaGetErrorString(e__)); \
  } while (0)

namespace {

// the open batch → the sketch, asynchronously on h->st
int flush(kuq_count_unique *h) {
  KsStager &in = h->in;
  if (in.empty()) { in.fill = in.seq_start = 0; return 0; }
  CU_CU(in.stage(h->st));
  h->bases += in.len;
  std::pair<Event, Event> t;
  CU_CU(t.first.alloc(cudaEventDefault));
  CU_CU(t.second.alloc(cudaEventDefault));
  CU_CU(cudaEventRecord(t.first, h->st));
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((in.nb + 15) / 16, (uint64_t)h->grid));
  const uint32_t *drop = in.has_drops ? in.d_drop.get() : nullptr;
  if (h->p <= SMEM_MAX_P)
    k_cu_sketch<true><<<grid, SKETCH_THREADS, 4u << h->p, h->st>>>(in.d_codes, in.d_amb, in.d_start, drop, in.nb, h->k, h->p,
                                                                    h->d_regs, h->d_count);
  else
    k_cu_sketch<false><<<grid, SKETCH_THREADS, 0, h->st>>>(in.d_codes, in.d_amb, in.d_start, drop, in.nb, h->k, h->p, h->d_regs,
                                                           h->d_count);
  CU_CU(cudaGetLastError());
  CU_CU(cudaEventRecord(t.second, h->st));
  h->timers.push_back(std::move(t));
  CU_CU(in.next());
  return 0;
}

int sum_timers(kuq_count_unique *h) {
  CU_CU(cudaStreamSynchronize(h->st));
  for (auto &t : h->timers) {
    float ms = 0;
    CU_CU(cudaEventElapsedTime(&ms, t.first, t.second));
    h->sketch_ms += ms;
  }
  h->timers.clear();
  return 0;
}

}  // namespace

extern "C" {

int kuq_count_unique_create(int device, uint32_t k, uint32_t p, uint64_t batch_bases, kuq_count_unique **out, char *err,
                            uint64_t err_cap) {
  auto say = [&](int code, const char *msg) {
    if (err && err_cap) snprintf(err, err_cap, "%s", msg);
    return code;
  };
  if (!out) return say(KUQ_E_INVALID_ARG, "NULL handle pointer");
  *out = nullptr;
  if (k < 1 || k > 31) return say(KUQ_E_UNSUPPORTED_K, "k must be 1..31");
  if (p < 4 || p > 18) return say(KUQ_E_INVALID_ARG, "precision (number of register = 2^precision) must be between 4 and 18");
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
    (void)cudaGetLastError();
    return say(KUQ_E_NO_DEVICE, "no CUDA device (there is no CPU path)");
  }
  if (device < 0 || device >= n_dev || cudaSetDevice(device) != cudaSuccess) return say(KUQ_E_INVALID_ARG, "bad device ordinal");
  kuq_count_unique *h = new kuq_count_unique;
  h->device = device;
  h->k = k;
  h->p = p;
  auto bail = [&](int code, const char *msg) {
    kuq_count_unique_destroy(h);
    return say(code, msg);
  };
  const uint64_t batch = std::max<uint64_t>(batch_bases ? batch_bases : DEFAULT_BATCH, 2 * k + 32);
  h->in.flush = [h] { return flush(h); };
  if (h->st.alloc(cudaStreamNonBlocking) != cudaSuccess) return bail(KUQ_E_CUDA, "cannot create a stream");
  if (h->in.init(k, batch, std::min<uint64_t>(batch / k + 2, 1ull << 22)) != cudaSuccess ||
      h->d_regs.alloc(1ull << p) != cudaSuccess || h->d_hist.alloc(64) != cudaSuccess || h->d_count.alloc(1) != cudaSuccess ||
      h->h_count.alloc(1) != cudaSuccess)
    return bail(KUQ_E_NOMEM, "cannot allocate the batch and sketch buffers");
  const int smem = p <= SMEM_MAX_P ? 4 << p : 0;
  int per_sm = 0;
  cudaError_t e = p <= SMEM_MAX_P ? cudaFuncSetAttribute(k_cu_sketch<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)
                                  : cudaSuccess;
  if (e == cudaSuccess)
    e = p <= SMEM_MAX_P ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_cu_sketch<true>, SKETCH_THREADS, smem)
                        : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_cu_sketch<false>, SKETCH_THREADS, 0);
  if (e != cudaSuccess || per_sm < 1) return bail(KUQ_E_CUDA, "cannot size the sketch kernel's grid");
  h->grid = per_sm * h->in.n_sm;
  if (cudaMemsetAsync(h->d_regs, 0, 4ull << p, h->st) != cudaSuccess || cudaMemsetAsync(h->d_count, 0, 8, h->st) != cudaSuccess)
    return bail(KUQ_E_CUDA, "memset failed");
  *out = h;
  return KUQ_OK;
}

int kuq_count_unique_add(kuq_count_unique *h, const char *bases, const uint64_t *offsets, uint32_t n_seqs) {
  if (!h) return KUQ_E_INVALID_ARG;
  if (n_seqs && (!bases || !offsets)) return h->fail(KUQ_E_INVALID_ARG, "NULL sequence buffers");
  CU_CU(cudaSetDevice(h->device));
  for (uint32_t r = 0; r < n_seqs; r++) {
    if (offsets[r + 1] < offsets[r]) return h->fail(KUQ_E_INVALID_ARG, "offsets decrease at sequence %u", r);
    const char *s = bases + offsets[r];
    const uint64_t len = offsets[r + 1] - offsets[r];
    int rc = 0;
    if (!memchr(s, '\n', len) && !memchr(s, '\r', len)) {
      rc = h->in.add_sequence(s, len);
    } else {
      for (uint64_t i = 0; i < len && !rc; i += PIECE) {
        scan_piece(s, len, i, std::min(i + PIECE + h->k - 1, len), h->k, h->clean, h->drop_ends);
        rc = h->in.add_clean(h->clean.data(), h->clean.size(), h->drop_ends);
      }
    }
    if (rc) return rc;
  }
  return KUQ_OK;
}

int kuq_count_unique_result(kuq_count_unique *h, uint64_t *estimate, uint64_t *n_observed, uint8_t *regs_out) {
  if (!h) return KUQ_E_INVALID_ARG;
  CU_CU(cudaSetDevice(h->device));
  int rc = flush(h);
  if (rc) return rc;
  const uint32_t m = 1u << h->p;
  CU_CU(cudaMemsetAsync(h->d_hist, 0, 64 * 4, h->st));
  k_cu_hist<<<(unsigned)std::min<uint32_t>((m + 255) / 256, 128), 256, 0, h->st>>>(h->d_regs, m, h->d_hist);
  CU_CU(cudaGetLastError());
  uint32_t hist[64];
  std::vector<uint32_t> regs(regs_out ? m : 0);
  CU_CU(cudaMemcpyAsync(hist, h->d_hist, sizeof hist, cudaMemcpyDeviceToHost, h->st));
  CU_CU(cudaMemcpyAsync(h->h_count, h->d_count, 8, cudaMemcpyDeviceToHost, h->st));
  if (regs_out) CU_CU(cudaMemcpyAsync(regs.data(), h->d_regs, 4ull * m, cudaMemcpyDeviceToHost, h->st));
  CU_CU(cudaStreamSynchronize(h->st));
  h->windows = *h->h_count;
  if (regs_out)
    for (uint32_t i = 0; i < m; i++) regs_out[i] = (uint8_t)regs[i];
  if (n_observed) *n_observed = h->windows;
  if (estimate) {
    // no valid window: the main counter stays sparse and empty (hyperloglogplus.cpp:592-593), its estimate is 0
    int C[66] = {0};
    for (int i = 0; i < 64; i++) C[i] = (int)hist[i];
    *estimate = h->windows ? ertl_from_hist(C, 64 - h->p, m, h->windows) : 0;
  }
  return KUQ_OK;
}

int kuq_count_unique_stats(kuq_count_unique *h, double *sketch_ms, uint64_t *windows, uint64_t *bases) {
  if (!h) return KUQ_E_INVALID_ARG;
  CU_CU(cudaSetDevice(h->device));
  int rc = sum_timers(h);
  if (rc) return rc;
  if (sketch_ms) *sketch_ms = h->sketch_ms;
  if (windows) *windows = h->windows;
  if (bases) *bases = h->bases;
  return KUQ_OK;
}

const char *kuq_count_unique_last_error(const kuq_count_unique *h) { return h ? h->err.c_str() : ""; }

void kuq_count_unique_destroy(kuq_count_unique *h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->st) cudaStreamSynchronize(h->st);
  (void)cudaGetLastError();
  delete h;
}

}  // extern "C"
