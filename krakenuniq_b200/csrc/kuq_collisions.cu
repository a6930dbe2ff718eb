// kuq_collisions.cu — the collision table behind the record tier of the sparse HLL tier (KEPT_BIT).
//
// Two records of one taxon can share a sparse-tier key: the code keeps about the top 25 bits of the k-mer's hash.
// Each such group has one primary (its lowest record index); the table lists the other members, the secondaries, as
// (secondary, primary) pairs.  Built once per staged range: group the records by (taxon, code) with a radix sort of
// (key, record index), in passes over taxon ranges when the sort's buffers do not fit beside everything else.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include <cub/cub.cuh>

#include "kuq_kernels.cuh"

namespace kuq {
namespace {

// (taxon − t_lo, code) and the record index of every record of a taxon in [t_lo, t_hi)
__global__ void __launch_bounds__(256) k_collide_gather(const uint8_t *__restrict__ pairs, uint64_t n_rec, uint32_t hi_mask,
                                                        uint32_t t_lo, uint32_t t_hi, unsigned long long *__restrict__ keys,
                                                        uint32_t *__restrict__ idx, unsigned long long *cursor) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t n_round = (n_rec + stride - 1) / stride * stride;          // whole warps stay in the loop (ballot below)
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
    unsigned long long key = 0;
    bool have = false;
    if (i < n_rec) {
      const uint32_t *w = reinterpret_cast<const uint32_t *>(pairs + i * 12);
      const uint32_t taxon = w[2];
      if (taxon >= t_lo && taxon < t_hi) {
        key = ((unsigned long long)(taxon - t_lo) << 32) | (uint32_t)record_key(w, w[1], hi_mask);
        have = true;
      }
    }
    const uint32_t vote = __ballot_sync(0xFFFFFFFFu, have);
    if (!vote) continue;
    const uint32_t lane = threadIdx.x & 31;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(cursor, (unsigned long long)__popc(vote));
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    if (have) {
      const unsigned long long at = base + __popc(vote & ((1u << lane) - 1));
      keys[at] = key;
      idx[at] = (uint32_t)i;
    }
  }
}

// groups of equal keys in the sorted sequence: the first position of a group of >= 2 emits its secondaries
__global__ void __launch_bounds__(256) k_collide_emit(const unsigned long long *__restrict__ keys, const uint32_t *__restrict__ idx,
                                                      uint64_t n, uint2 *out, uint64_t cap, unsigned long long *n_out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (i > 0 && keys[i - 1] == k) continue;
    if (i + 1 >= n || keys[i + 1] != k) continue;                          // a group of one: no secondary
    uint64_t e = i + 1;
    uint32_t prim = idx[i];
    while (e < n && keys[e] == k) prim = min(prim, idx[e++]);
    for (uint64_t q = i; q < e; q++) {
      if (idx[q] == prim) continue;
      const unsigned long long at = atomicAdd(n_out, 1ull);
      if (at < cap) out[at] = make_uint2(idx[q], prim);
    }
  }
}

}  // namespace

// 0 = ok (list_out / *n_out: device list of (secondary, primary), empty when there is none), 1 = no table (more than 2^32
// records, no memory for the sort, a taxon too large for one pass, or more than `max_entries` secondaries), 2 = CUDA error
int build_collisions(const uint8_t *pairs, uint64_t n_rec, uint64_t key_mask, const uint64_t *records_of_taxon, uint32_t n_sketch,
                     uint64_t max_entries, DevBuf<uint2> &list_out, uint64_t *n_out, int n_sm, cudaStream_t stream) {
  list_out.reset();
  *n_out = 0;
  if (n_rec >= (1ull << 32)) return 1;
  const uint32_t hi_mask = (uint32_t)(key_mask >> 32);
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { (void)cudaGetLastError(); return 2; }
  const uint64_t list_bytes = (max_entries + 1) * sizeof(uint2);
  // per record of a pass: two key buffers + two index buffers; keep a quarter of the free memory for the sort's
  // temporaries and for the other users of the device
  const uint64_t usable = free_b / 4 * 3 > list_bytes ? free_b / 4 * 3 - list_bytes : 0;
  const uint64_t pass_max = std::min<uint64_t>(usable / 24, n_rec);
  // taxon ranges: consecutive dense ids while their records fit one pass (taxon 0 = "no taxon" is never counted)
  std::vector<uint32_t> cuts{1};
  uint64_t in_pass = 0, biggest = 0;
  for (uint32_t t = 1; t < n_sketch; t++) {
    const uint64_t c = records_of_taxon[t];
    if (c > pass_max) return 1;
    if (in_pass + c > pass_max) { biggest = std::max(biggest, in_pass); cuts.push_back(t); in_pass = 0; }
    in_pass += c;
  }
  biggest = std::max(biggest, in_pass);
  cuts.push_back(n_sketch);
  if (biggest == 0) return 0;
  DevBuf<unsigned long long> kbuf[2], cnt;
  DevBuf<uint32_t> ibuf[2];
  DevBuf<uint2> list;
  DevBuf<uint8_t> temp;
  size_t temp_bytes = 0;
  auto error = [](int rc) {
    (void)cudaGetLastError();
    return rc;
  };
  {
    cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    if (cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, k, v, (int64_t)biggest, 0, 64, stream) != cudaSuccess) return error(2);
  }
  if (kbuf[0].alloc(biggest) != cudaSuccess || kbuf[1].alloc(biggest) != cudaSuccess || ibuf[0].alloc(biggest) != cudaSuccess ||
      ibuf[1].alloc(biggest) != cudaSuccess || cnt.alloc(2) != cudaSuccess || temp.alloc(temp_bytes ? temp_bytes : 1) != cudaSuccess ||
      list.alloc(max_entries + 1) != cudaSuccess)
    return error(1);
  if (cudaMemsetAsync(cnt + 1, 0, 8, stream) != cudaSuccess) return error(2);
  const int grid = n_sm * 8;
  for (size_t p = 0; p + 1 < cuts.size(); p++) {
    const uint32_t t_lo = cuts[p], t_hi = cuts[p + 1];
    unsigned long long n = 0;
    if (cudaMemsetAsync(cnt, 0, 8, stream) != cudaSuccess) return error(2);
    k_collide_gather<<<grid, 256, 0, stream>>>(pairs, n_rec, hi_mask, t_lo, t_hi, kbuf[0], ibuf[0], cnt);
    if (cudaMemcpyAsync(&n, cnt, 8, cudaMemcpyDeviceToHost, stream) != cudaSuccess || cudaStreamSynchronize(stream) != cudaSuccess)
      return error(2);
    if (n > biggest) return error(2);                      // more records than the per-taxon counts promised
    if (n < 2) continue;
    const int end_bit = 32 + (32 - __builtin_clz(std::max<uint32_t>(t_hi - t_lo - 1, 1)));
    cub::DoubleBuffer<unsigned long long> k(kbuf[0], kbuf[1]);
    cub::DoubleBuffer<uint32_t> v(ibuf[0], ibuf[1]);
    if (cub::DeviceRadixSort::SortPairs(temp.get(), temp_bytes, k, v, (int64_t)n, 0, end_bit, stream) != cudaSuccess) return error(2);
    k_collide_emit<<<grid, 256, 0, stream>>>(k.Current(), v.Current(), n, list, max_entries, cnt + 1);
  }
  unsigned long long n_list = 0;
  if (cudaMemcpyAsync(&n_list, cnt + 1, 8, cudaMemcpyDeviceToHost, stream) != cudaSuccess ||
      cudaStreamSynchronize(stream) != cudaSuccess || cudaGetLastError() != cudaSuccess)
    return error(2);
  if (n_list > max_entries) return error(1);
  if (n_list == 0) list.reset();
  list_out = std::move(list);
  *n_out = n_list;
  return 0;
}

}  // namespace kuq
