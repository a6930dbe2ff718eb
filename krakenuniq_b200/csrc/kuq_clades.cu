// kuq_clades.cu — device side of kuq_clade_counts_tree: the sketches of ALL clades of the taxonomy in a few launches
// (the report of the reference rolls every taxon's ReadCounts into each ancestor, TaxReport, taxdb.hpp:928-982, with
// ReadCounts::operator+= = HLL merge, readcounts.hpp:76-88 / hyperloglogplus.cpp:596-621).
//
//  dense clades  (some member's sketch is dense → register-wise max of the members' registers, :604-621):
//      one CTA per clade folds its members' 4 KB register arrays; register histograms of all clades in one launch.
//  sparse clades (no dense member → union of the members' code sets, :600-603): the number of distinct codes of
//      every subtree at once.  Keys (taxon, code) of the sparse tier (set slots and kept records) are sorted by (code, preorder(taxon)); the
//      taxa of a subtree are a preorder interval, so the occurrences of one code inside a subtree are a run of that
//      sorted sequence and   distinct(subtree u) = keys in u − adjacent equal-code pairs inside u,
//      and a pair lies inside u exactly when its taxa's lowest common ancestor does.  The kernel books every
//      adjacent pair at its LCA (per encoded rank, because the estimator wants the rank histogram of the union);
//      the host sums the books up the tree.
//  exact mode (KUQ_HLL_EXACT): the same identity over the (k-mer, taxon) pairs of the exact table, sorted by
//      (k-mer, preorder), in passes over parts of the k-mer space when scratch is short (exact_clade_dups).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include <cub/cub.cuh>
#include <cuda/std/tuple>

#include "kuq_kernels.cuh"

namespace kuq {
namespace {

constexpr uint32_t NONE32 = 0xFFFFFFFFu;

__device__ __forceinline__ uint32_t enc_rank(uint32_t e) {          // getEncodedRank(enc, 25, 12), hyperloglogplus.cpp:152-161
  if (e & 1) return 13 + ((e >> 1) & 0x3F);
  const uint32_t r = e << 12;
  return (r ? (uint32_t)__clz(r) : 20u) + 1;
}

// out[c][0..4096) = max over the members of clade c; 256 threads x 16 bytes
__global__ void __launch_bounds__(256) k_clade_max_batch(const uint8_t *__restrict__ regs, const uint32_t *__restrict__ offs,
                                                         const uint32_t *__restrict__ members, uint8_t *__restrict__ out) {
  const uint32_t c = blockIdx.x;
  uint4 acc = make_uint4(0, 0, 0, 0);
  for (uint32_t i = offs[c]; i < offs[c + 1]; i++) {
    const uint4 v = __ldg(reinterpret_cast<const uint4 *>(regs + (size_t)members[i] * HLL_M) + threadIdx.x);
    acc.x = __vmaxu4(acc.x, v.x); acc.y = __vmaxu4(acc.y, v.y); acc.z = __vmaxu4(acc.z, v.z); acc.w = __vmaxu4(acc.w, v.w);
  }
  reinterpret_cast<uint4 *>(out + (size_t)c * HLL_M)[threadIdx.x] = acc;
}

// keys of the taxa that are still sparse and belong to the tree → (code << 32 | preorder of the taxon)
__global__ void __launch_bounds__(256) k_clade_sort_keys(const KeySource src,
                                                         const uint8_t *__restrict__ dense_flag, const uint32_t *__restrict__ pre_of_taxon,
                                                         unsigned long long *__restrict__ out, uint64_t out_cap,
                                                         unsigned long long *cursor) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t n_round = (src.n + stride - 1) / stride * stride;        // whole warps stay in the loop (ballot below)
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
    unsigned long long sk = 0;
    bool have = false;
    if (i < src.n) {
      const unsigned long long key = source_key(src, i);
      if (key) {
        const uint32_t taxon = (uint32_t)(key >> 32) - 1;
        if (!dense_flag[taxon]) {
          const uint32_t pre = pre_of_taxon[taxon];
          if (pre != NONE32) { sk = ((unsigned long long)(uint32_t)key << 32) | pre; have = true; }
        }
      }
    }
    const uint32_t vote = __ballot_sync(0xFFFFFFFFu, have);
    if (vote) {
      const uint32_t lane = threadIdx.x & 31;
      unsigned long long base = 0;
      if (lane == 0) base = atomicAdd(cursor, (unsigned long long)__popc(vote));
      base = __shfl_sync(0xFFFFFFFFu, base, 0);
      if (have) {
        const unsigned long long at = base + __popc(vote & ((1u << lane) - 1));
        if (at < out_cap) out[at] = sk;
      }
    }
  }
}

// adjacent equal codes: book the pair at the lowest common ancestor of its two taxa
__global__ void __launch_bounds__(256) k_clade_dups(const unsigned long long *__restrict__ sorted, uint64_t n,
                                                    const uint32_t *__restrict__ node_of_pre, const uint32_t *__restrict__ parent_c,
                                                    const uint32_t *__restrict__ depth_c, const int32_t *__restrict__ sid_of_node,
                                                    uint32_t *dup) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x + 1; i < n; i += stride) {
    const unsigned long long a = sorted[i - 1], b = sorted[i];
    if ((a >> 32) != (b >> 32)) continue;
    uint32_t x = node_of_pre[(uint32_t)a], y = node_of_pre[(uint32_t)b];
    uint32_t dx = depth_c[x], dy = depth_c[y];
    while (dx > dy && x != NONE32) { x = parent_c[x]; dx--; }
    while (dy > dx && y != NONE32) { y = parent_c[y]; dy--; }
    while (x != y && x != NONE32 && y != NONE32) { x = parent_c[x]; y = parent_c[y]; }
    if (x == NONE32 || y == NONE32 || x != y) continue;               // different trees: no clade holds both
    const int32_t s = sid_of_node[x];
    if (s >= 0) atomicAdd(dup + (size_t)s * 64 + min(enc_rank((uint32_t)(a >> 32)), 63u), 1u);
  }
}

// ---- exact mode: the same identity over (k-mer, taxon) pairs --------------------------------------------------------
// distinct(subtree u) = pairs of taxa in u − adjacent equal-k-mer pairs whose LCA lies in u, with the pairs sorted by
// (k-mer, preorder of the taxon).  The pairs of one k-mer all fall in one pass of the k-mer space, so passes add up.
struct ExactItem {
  unsigned long long kmer;     // canonical k-mer (62 bits at most): sort key, most significant
  uint32_t pre;                // preorder of the taxon: sort key
  uint32_t taxon;              // dense taxon id, carried along
};
struct ExactItemDecomposer {
  __host__ __device__ cuda::std::tuple<unsigned long long &, uint32_t &> operator()(ExactItem &it) const { return {it.kmer, it.pre}; }
};

// the occupied slots whose k-mer falls in this pass and whose taxon lies in the tree → items; one cursor atomic per warp
__global__ void __launch_bounds__(256) k_exact_sort_items(const ExactPair *__restrict__ slots, uint64_t n_slots, uint32_t n_pass,
                                                          uint32_t pass, const uint32_t *__restrict__ pre_of_taxon,
                                                          ExactItem *__restrict__ out, uint64_t out_cap, unsigned long long *cursor) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t n_round = (n_slots + stride - 1) / stride * stride;      // whole warps stay in the loop (ballot below)
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
    ExactItem it{0ull, NONE32, 0u};
    bool have = false;
    if (i < n_slots) {
      const ExactPair pr = slots[i];
      if (pr.kmer1 && (n_pass == 1 || exact_pass(pr.kmer1 - 1, n_pass) == pass)) {
        it.kmer = pr.kmer1 - 1;
        it.taxon = (uint32_t)(pr.taxon1 - 1);
        it.pre = pre_of_taxon[it.taxon];
        have = it.pre != NONE32;
      }
    }
    const uint32_t vote = __ballot_sync(0xFFFFFFFFu, have);
    if (vote) {
      const uint32_t lane = threadIdx.x & 31;
      unsigned long long base = 0;
      if (lane == 0) base = atomicAdd(cursor, (unsigned long long)__popc(vote));
      base = __shfl_sync(0xFFFFFFFFu, base, 0);
      if (have) {
        const unsigned long long at = base + __popc(vote & ((1u << lane) - 1));
        if (at < out_cap) out[at] = it;
      }
    }
  }
}

// adjacent items with one k-mer: −1 at the LCA of their taxa in the context's taxonomy (parent 0 = none; the walk is
// bounded by the depth, so a malformed chain cannot hold it)
__global__ void __launch_bounds__(256) k_exact_dups(const ExactItem *__restrict__ sorted, uint64_t n, const uint32_t *__restrict__ parent,
                                                    const uint16_t *__restrict__ depth, unsigned long long *books) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x + 1; i < n; i += stride) {
    const ExactItem a = sorted[i - 1], b = sorted[i];
    if (a.kmer != b.kmer) continue;
    uint32_t x = a.taxon, y = b.taxon, dx = depth[x], dy = depth[y];
    while (dx > dy) { x = parent[x]; dx--; }
    while (dy > dx) { y = parent[y]; dy--; }
    for (uint32_t s = 0; x != y && s <= dx; s++) { x = parent[x]; y = parent[y]; }
    if (x == y && x != 0) atomicAdd(books + x, ~0ull);                  // two's complement −1
  }
}

}  // namespace

int exact_clade_dups(const ExactPair *slots, uint64_t n_slots, uint64_t n_pairs, const uint32_t *d_pre_of_taxon,
                     const uint32_t *d_parent, const uint16_t *d_depth, unsigned long long *d_books, uint64_t budget, int n_sm,
                     cudaStream_t stream, uint32_t *passes_out) {
  *passes_out = 0;
  if (n_pairs < 2) return 0;
  // scratch per item: two sort buffers of 16 B and CUB's temporary storage (a few bytes per item); 48 B with margin
  const uint64_t per_item = 48;
  uint64_t n_pass = std::max<uint64_t>(1, (n_pairs * per_item + budget - 1) / std::max<uint64_t>(budget, 1));
  if (n_pass > (1ull << 20)) return 1;
  auto pass_cap = [&](uint64_t want) { return std::min<uint64_t>(n_pairs, want + want / 16 + 4096); };
  uint64_t cap = pass_cap((n_pairs + n_pass - 1) / n_pass);
  DevBuf<ExactItem> buf[2];
  DevBuf<unsigned long long> cursor;
  DevBuf<uint8_t> temp;
  size_t temp_bytes = 0;
  auto reserve = [&](uint64_t c) -> int {                                // 0 ok, 1 no memory, 2 CUDA error
    buf[0].reset(); buf[1].reset(); temp.reset();
    cub::DoubleBuffer<ExactItem> keys(nullptr, nullptr);
    temp_bytes = 0;
    if (cub::DeviceRadixSort::SortKeys(nullptr, temp_bytes, keys, (int64_t)c, ExactItemDecomposer{}, 0, 94, stream) != cudaSuccess) {
      (void)cudaGetLastError();
      return 2;
    }
    if (buf[0].alloc(c) != cudaSuccess || buf[1].alloc(c) != cudaSuccess || temp.alloc(temp_bytes ? temp_bytes : 1) != cudaSuccess) {
      (void)cudaGetLastError();
      return 1;
    }
    cap = c;
    return 0;
  };
  if (cursor.alloc(1) != cudaSuccess) { (void)cudaGetLastError(); return 1; }
  int rc = reserve(cap);
  const int grid = n_sm * 8;
  for (uint32_t pass = 0; pass < n_pass && !rc; pass++) {
    unsigned long long n = 0;
    for (int attempt = 0; attempt < 2 && !rc; attempt++) {
      cudaMemsetAsync(cursor, 0, 8, stream);
      k_exact_sort_items<<<grid, 256, 0, stream>>>(slots, n_slots, (uint32_t)n_pass, pass, d_pre_of_taxon, buf[0], cap, cursor);
      cudaMemcpyAsync(&n, cursor, 8, cudaMemcpyDeviceToHost, stream);
      if (cudaStreamSynchronize(stream) != cudaSuccess) { (void)cudaGetLastError(); rc = 2; break; }
      if (n <= cap) break;
      rc = attempt ? 2 : reserve(n);                                     // an unlucky pass: room for all of its items
    }
    if (rc || n < 2) continue;
    cub::DoubleBuffer<ExactItem> keys(buf[0], buf[1]);
    if (cub::DeviceRadixSort::SortKeys(temp.get(), temp_bytes, keys, (int64_t)n, ExactItemDecomposer{}, 0, 94, stream) != cudaSuccess) rc = 2;
    if (!rc) k_exact_dups<<<grid, 256, 0, stream>>>(keys.Current(), n, d_parent, d_depth, d_books);
    if (cudaStreamSynchronize(stream) != cudaSuccess || cudaGetLastError() != cudaSuccess) rc = 2;
  }
  *passes_out = (uint32_t)n_pass;
  return rc;
}

void launch_clade_max_batch(const uint8_t *regs, const uint32_t *d_offs, const uint32_t *d_members, uint32_t n_clades,
                            uint8_t *d_out, cudaStream_t stream) {
  if (n_clades) k_clade_max_batch<<<n_clades, 256, 0, stream>>>(regs, d_offs, d_members, d_out);
}

// 0 = ok, 1 = not enough device memory (the caller falls back to one union per clade), 2 = CUDA error
int sparse_clade_dups(const KeySource &set_keys, const KeySource &kept_keys, const uint8_t *dense_flag, uint64_t n_keys_upper,
                      const uint32_t *d_pre_of_taxon, const uint32_t *d_node_of_pre, const uint32_t *d_parent_c,
                      const uint32_t *d_depth_c, const int32_t *d_sid_of_node, uint32_t *d_dup, int n_sm, cudaStream_t stream) {
  if (n_keys_upper < 2 || set_keys.n + kept_keys.n == 0) return 0;
  DevBuf<unsigned long long> buf[2], cursor;
  DevBuf<uint8_t> temp;
  size_t temp_bytes = 0;
  int rc = 0;
  cub::DoubleBuffer<unsigned long long> keys(nullptr, nullptr);
  if (cub::DeviceRadixSort::SortKeys(nullptr, temp_bytes, keys, (int64_t)n_keys_upper, 0, 64, stream) != cudaSuccess) {
    (void)cudaGetLastError();
    return 2;
  }
  if (buf[0].alloc(n_keys_upper) != cudaSuccess || buf[1].alloc(n_keys_upper) != cudaSuccess || cursor.alloc(1) != cudaSuccess ||
      temp.alloc(temp_bytes ? temp_bytes : 1) != cudaSuccess) {
    (void)cudaGetLastError();
    return 1;
  }
  cudaMemsetAsync(cursor, 0, 8, stream);
  for (const KeySource *src : {&set_keys, &kept_keys})
    if (src->n) k_clade_sort_keys<<<n_sm * 8, 256, 0, stream>>>(*src, dense_flag, d_pre_of_taxon, buf[0], n_keys_upper, cursor);
  unsigned long long n = 0;
  cudaMemcpyAsync(&n, cursor, 8, cudaMemcpyDeviceToHost, stream);
  if (cudaStreamSynchronize(stream) != cudaSuccess) { (void)cudaGetLastError(); return 2; }
  if (n > n_keys_upper) return 2;                                      // more keys than the per-taxon counters promised
  if (n >= 2) {
    keys = cub::DoubleBuffer<unsigned long long>(buf[0], buf[1]);
    if (cub::DeviceRadixSort::SortKeys(temp.get(), temp_bytes, keys, (int64_t)n, 0, 64, stream) != cudaSuccess) rc = 2;
    if (!rc) k_clade_dups<<<n_sm * 8, 256, 0, stream>>>(keys.Current(), n, d_node_of_pre, d_parent_c, d_depth_c, d_sid_of_node, d_dup);
    if (cudaStreamSynchronize(stream) != cudaSuccess || cudaGetLastError() != cudaSuccess) rc = 2;
  }
  return rc;
}

}  // namespace kuq
