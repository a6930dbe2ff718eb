// kuq_layout_exp.cu — measurement aid, not part of the classification path: how would k_lookup's bin search
// (kmer_query, src/krakendb.cpp:250-321) behave with another record layout or another search shape?
//
// The product keeps the on-disk layout in HBM: 12-byte {u64 key, u32 value} records, 4-byte aligned, so a key is two
// 32-bit loads and one key in eight straddles a 32-byte sector.  The experiment transcodes the staged records ONCE
// into 8-byte "minimizer-relative" records and runs a lookup-only kernel (no sketches, no record flags) over the
// windows a batch left in a slot's scratch, for every combination of
//     record layout  12 B (as staged)  |  8 B (below)
//     narrowing      4-, 8- or 16-ary  (pivots fetched per dependent round: 3, 7, 15)
//     final scan     <= 8 or <= 16 records
// and checks every variant's per-window result against the ids the product wrote for the same batch.
//
// 8-byte record: all records of a bin share their minimizer, i.e. 30 of the k-mer's 62 bits are known from the bin
// once the minimizer's position (0..16) and orientation are known (k = 31, m = 15; a 15-mer is never its own reverse
// complement).  low word  = the 16 bases outside the minimizer, high word = orient | pos << 1 | dense taxon << 6.
// The first position (from the k-mer's low end, the order of bin_key's loop, krakendb.cpp:208-213) whose canonical
// 15-mer equals the bin's is used on both sides, so equal k-mers have equal codes and the map is injective.
// Records stay in key order: a pivot's key is rebuilt from its code and the bin's minimizer for the narrowing
// rounds; the final scan compares codes.
//
// Tree layout (tree_slot): a second copy of the 12-byte records with every bin reordered so that its search pivots sit
// together at the bin's head — index, one shared header, one short leaf instead of index, two rounds of pivots spread
// over the bin, scan.  Its control keeps the on-disk layout and only asks L2 for 256-byte blocks on the first round.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "../../include/kuq.h"
#include "kuq_kernels.cuh"

namespace kuq {
namespace {

constexpr uint32_t X_BIN_NONE = 0xFFFFFFFFu, X_BIN_AMBIG = 0xFFFFFFFEu;   // k_scan's scratch markers
constexpr uint32_t MASK30 = 0x3FFFFFFFu;

__device__ __forceinline__ uint32_t revcomp15(uint32_t x) {               // krakendb.cpp:218-225 for n = 15
  x = __brev(x);
  x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
  return (~x) >> 2;
}

__device__ __forceinline__ uint64_t key12(const uint8_t *pairs, uint64_t pos, uint64_t key_mask) {
  const uint32_t *p = reinterpret_cast<const uint32_t *>(pairs + pos * 12);
  const uint32_t lo = __ldg(p), hi = __ldg(p + 1);
  return (((uint64_t)hi << 32) | lo) & key_mask;
}

// key of an 8-byte record of the bin whose canonical minimizer is mm (reverse complement mm_rc)
__device__ __forceinline__ uint64_t rebuild8(unsigned long long rec, uint32_t mm, uint32_t mm_rc) {
  const uint32_t rest = (uint32_t)rec, hi = (uint32_t)(rec >> 32);
  const uint32_t sh = (hi >> 1) & 31u;                       // pos
  const uint64_t mmer = (hi & 1u) ? mm_rc : mm;
  const uint32_t s2 = 2 * sh;
  const uint64_t low = (uint64_t)rest & ((1ull << s2) - 1);
  const uint64_t high = (uint64_t)rest >> s2;
  return (high << (s2 + 30)) | (mmer << s2) | low;
}

__global__ void __launch_bounds__(256) k_transcode8(const uint8_t *__restrict__ pairs, uint64_t n_rec, uint64_t key_mask,
                                                    uint32_t xor_mask, unsigned long long *__restrict__ out, uint32_t *err) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rec; r += stride) {
    const uint64_t key = key12(pairs, r, key_mask);
    const uint32_t val = __ldg(reinterpret_cast<const uint32_t *>(pairs + r * 12) + 2);
    if (val >> 24) atomicExch(err, 1u);
    uint32_t best = 0xFFFFFFFFu, pos = 0, orient = 0;
#pragma unroll
    for (uint32_t i = 0; i < 17; i++) {
      const uint32_t m = (uint32_t)(key >> (2 * i)) & MASK30, rc = revcomp15(m);
      const uint32_t t = xor_mask ^ min(m, rc);
      if (t < best) { best = t; pos = i; orient = rc < m ? 1u : 0u; }
    }
    const uint32_t s2 = 2 * pos;
    const uint32_t rest = (uint32_t)(((key >> (s2 + 30)) << s2) | (key & ((1ull << s2) - 1)));
    const uint32_t hi = orient | (pos << 1) | (val << 6);
    out[r] = ((unsigned long long)hi << 32) | rest;
  }
}

// key of a 12-byte record through a load that asks L2 to fetch the whole aligned 256-byte block around it
__device__ __forceinline__ uint64_t key12_pf(const uint8_t *pairs, uint64_t pos, uint64_t key_mask) {
  const uint32_t *p = reinterpret_cast<const uint32_t *>(pairs + pos * 12);
  uint32_t lo, hi;
  asm("ld.global.nc.L2::256B.u32 %0, [%1];" : "=r"(lo) : "l"(p));
  asm("ld.global.nc.L2::256B.u32 %0, [%1];" : "=r"(hi) : "l"(p + 1));
  return (((uint64_t)hi << 32) | lo) & key_mask;
}

// Lookup-only variant of k_lookup: same grid-stride loop and scratch prefetch; REC = record bytes, ARITY - 1 pivots per
// narrowing round, final scan of <= W records.
// FORM 1 (4-ary only): the narrowing step as an if / else-if chain instead of a count of pivots <= key
// FORM 2 (12 B only): the first round's pivots through key12_pf, so that most of a small bin is in L2 after one trip
template <int REC, int ARITY, int W, int FORM = 0>
__global__ void __launch_bounds__(256, 8) k_lookup_variant(const DbView db, const unsigned long long *__restrict__ rec8,
                                                           const uint64_t *__restrict__ canon_a, const uint32_t *__restrict__ bins_a,
                                                           uint32_t *__restrict__ out, uint64_t n_pos) {
  static_assert(ARITY <= W, "a narrowing round needs n / ARITY >= 1");
  const uint32_t hi_mask = (uint32_t)(db.key_mask >> 32);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t bin_n = g < n_pos ? __ldg(bins_a + g) : X_BIN_NONE;
  uint64_t canon_n = g < n_pos ? __ldg(canon_a + g) : 0ull;
  for (; g < n_pos; g += stride) {
    const uint32_t bin = bin_n;
    const uint64_t canon = canon_n;
    if (g + stride < n_pos) { bin_n = __ldg(bins_a + g + stride); canon_n = __ldg(canon_a + g + stride); }
    if (bin == X_BIN_NONE) continue;
    if (bin == X_BIN_AMBIG) { out[g] = AMBIG; continue; }
    uint32_t taxon = 0;
    if (bin >= db.bin_lo && bin < db.bin_hi) {
      const uint64_t *o = db.offsets + (bin - db.bin_lo);
      const uint64_t o0 = __ldg(o), o1 = __ldg(o + 1);
      uint64_t lo = o0 - db.rec_base;
      uint32_t n = (uint32_t)(o1 - o0);
      const uint32_t mm = bin ^ db.xor_mask, mm_rc = revcomp15(mm);
      bool first = true;
      while (n > (uint32_t)W) {
        const uint32_t q = n / ARITY;
        uint64_t piv[ARITY - 1];
#pragma unroll
        for (int j = 0; j < ARITY - 1; j++) {
          if (REC == 12 && FORM == 2 && first) piv[j] = key12_pf(db.pairs, lo + (uint64_t)(j + 1) * q, db.key_mask);
          else if (REC == 12) piv[j] = key12(db.pairs, lo + (uint64_t)(j + 1) * q, db.key_mask);
          else piv[j] = rebuild8(__ldg(rec8 + lo + (uint64_t)(j + 1) * q), mm, mm_rc);
        }
        first = false;
        if (FORM == 1 && ARITY == 4) {
          if (canon >= piv[2]) { lo += 3 * q; n -= 3 * q; }
          else if (canon >= piv[1]) { lo += 2 * q; n = q; }
          else if (canon >= piv[0]) { lo += q; n = q; }
          else { n = q; }
        } else {
          uint32_t c = 0;                                      // pivots <= canon: the part that can hold the key
#pragma unroll
          for (int j = 0; j < ARITY - 1; j++) c += canon >= piv[j] ? 1u : 0u;
          lo += (uint64_t)c * q;
          n = (c == (uint32_t)(ARITY - 1)) ? n - (ARITY - 1) * q : q;
        }
      }
      if (n) {
        if (REC == 12) {
          const uint32_t *b = reinterpret_cast<const uint32_t *>(db.pairs + lo * 12);
          const uint32_t clo = (uint32_t)canon, chi = (uint32_t)(canon >> 32);
          uint32_t lw[W];                                      // all loads in flight before the first compare
#pragma unroll
          for (int t = 0; t < W; t++) lw[t] = ((uint32_t)t < n) ? __ldg(b + 3 * t) : 0;
          uint32_t m = 0;
#pragma unroll
          for (int t = 0; t < W; t++) m |= ((uint32_t)t < n && lw[t] == clo) ? (1u << t) : 0u;
          while (m) {
            const int t = __ffs(m) - 1;
            m &= m - 1;
            if ((__ldg(b + 3 * t + 1) & hi_mask) == chi) { taxon = __ldg(b + 3 * t + 2); m = 0; }
          }
        } else {
          // code of the query: first position whose 15-mer is the bin's minimizer in either orientation
          uint32_t pos = 0, orient = 0;
#pragma unroll
          for (int i = 16; i >= 0; i--) {
            const uint32_t x = (uint32_t)(canon >> (2 * i)) & MASK30;
            if (x == mm) { pos = (uint32_t)i; orient = 0; }
            else if (x == mm_rc) { pos = (uint32_t)i; orient = 1; }
          }
          const uint32_t s2 = 2 * pos;
          const uint32_t rest = (uint32_t)(((canon >> (s2 + 30)) << s2) | (canon & ((1ull << s2) - 1)));
          const uint32_t tag = orient | (pos << 1);
          const uint32_t *b = reinterpret_cast<const uint32_t *>(rec8 + lo);
          uint32_t lw[W];
#pragma unroll
          for (int t = 0; t < W; t++) lw[t] = ((uint32_t)t < n) ? __ldg(b + 2 * t) : 0;
          uint32_t m = 0;
#pragma unroll
          for (int t = 0; t < W; t++) m |= ((uint32_t)t < n && lw[t] == rest) ? (1u << t) : 0u;
          while (m) {
            const int t = __ffs(m) - 1;
            m &= m - 1;
            const uint32_t hw = __ldg(b + 2 * t + 1);
            if ((hw & 63u) == tag) { taxon = (hw >> 6) & 0xFFFFFFu; m = 0; }
          }
        }
      }
    }
    out[g] = taxon;
  }
}

// The 12 B / 4-ary / scan <= 8 variant again, but fed like the product kernel: the whole Params block as a grid
// constant, loop bounds from p.offsets, no __restrict__ — isolates what the parameter passing costs.
__global__ void __launch_bounds__(256, 8) k_lookup_params(const __grid_constant__ Params p) {
  const DbView &db = p.db;
  const uint32_t hi_mask = (uint32_t)(db.key_mask >> 32);
  const uint64_t g_begin = p.offsets[0], g_end = p.offsets[p.n_reads];
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t g = g_begin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t bin_n = g < g_end ? __ldg(p.bins + g) : X_BIN_NONE;
  uint64_t canon_n = g < g_end ? __ldg(p.canon + g) : 0ull;
  for (; g < g_end; g += stride) {
    const uint32_t bin = bin_n;
    const uint64_t canon = canon_n;
    if (g + stride < g_end) { bin_n = __ldg(p.bins + g + stride); canon_n = __ldg(p.canon + g + stride); }
    if (bin == X_BIN_NONE) continue;
    if (bin == X_BIN_AMBIG) { p.codes_dense[g] = AMBIG; continue; }
    uint32_t taxon = 0;
    if (bin >= db.bin_lo && bin < db.bin_hi) {
      const uint64_t *o = db.offsets + (bin - db.bin_lo);
      const uint64_t o0 = __ldg(o), o1 = __ldg(o + 1);
      uint64_t lo = o0 - db.rec_base;
      uint32_t n = (uint32_t)(o1 - o0);
      while (n > 8u) {
        const uint32_t q = n >> 2;
        const uint64_t k1 = key12(db.pairs, lo + q, db.key_mask);
        const uint64_t k2 = key12(db.pairs, lo + 2 * q, db.key_mask);
        const uint64_t k3 = key12(db.pairs, lo + 3 * q, db.key_mask);
        const uint32_t c = (canon >= k1 ? 1u : 0u) + (canon >= k2 ? 1u : 0u) + (canon >= k3 ? 1u : 0u);
        lo += (uint64_t)c * q;
        n = (c == 3u) ? n - 3 * q : q;
      }
      if (n) {
        const uint32_t *b = reinterpret_cast<const uint32_t *>(db.pairs + lo * 12);
        const uint32_t clo = (uint32_t)canon, chi = (uint32_t)(canon >> 32);
        uint32_t lw[8];
#pragma unroll
        for (int t = 0; t < 8; t++) lw[t] = ((uint32_t)t < n) ? __ldg(b + 3 * t) : 0;
        uint32_t m = 0;
#pragma unroll
        for (int t = 0; t < 8; t++) m |= ((uint32_t)t < n && lw[t] == clo) ? (1u << t) : 0u;
        while (m) {
          const int t = __ffs(m) - 1;
          m &= m - 1;
          if ((__ldg(b + 3 * t + 1) & hi_mask) == chi) { taxon = __ldg(b + 3 * t + 2); m = 0; }
        }
      }
    }
    p.codes_dense[g] = taxon;
  }
}

// the product's search on 12-byte records (4-ary narrowing, scan of <= 8) as a function, for the shapes below
__device__ __forceinline__ uint32_t search12(const DbView &db, uint32_t hi_mask, uint64_t canon, uint64_t o0, uint64_t o1) {
  uint64_t lo = o0 - db.rec_base;
  uint32_t n = (uint32_t)(o1 - o0);
  while (n > 8u) {
    const uint32_t q = n >> 2;
    const uint64_t k1 = key12(db.pairs, lo + q, db.key_mask);
    const uint64_t k2 = key12(db.pairs, lo + 2 * q, db.key_mask);
    const uint64_t k3 = key12(db.pairs, lo + 3 * q, db.key_mask);
    if (canon >= k3) { lo += 3 * q; n -= 3 * q; }
    else if (canon >= k2) { lo += 2 * q; n = q; }
    else if (canon >= k1) { lo += q; n = q; }
    else { n = q; }
  }
  uint32_t taxon = 0;
  if (n) {
    const uint32_t *b = reinterpret_cast<const uint32_t *>(db.pairs + lo * 12);
    const uint32_t clo = (uint32_t)canon, chi = (uint32_t)(canon >> 32);
    uint32_t lw[8];
#pragma unroll
    for (int t = 0; t < 8; t++) lw[t] = ((uint32_t)t < n) ? __ldg(b + 3 * t) : 0;
    uint32_t m = 0;
#pragma unroll
    for (int t = 0; t < 8; t++) m |= ((uint32_t)t < n && lw[t] == clo) ? (1u << t) : 0u;
    while (m) {
      const int t = __ffs(m) - 1;
      m &= m - 1;
      if ((__ldg(b + 3 * t + 1) & hi_mask) == chi) { taxon = __ldg(b + 3 * t + 2); m = 0; }
    }
  }
  return taxon;
}

// Shape "index prefetch": the scratch of a thread's window i + 2 and the index entry of window i + 1 are in flight
// while window i is searched — one level less in the dependent chain index -> pivots -> scan of every window.
template <int MINB>
__global__ void __launch_bounds__(256, MINB) k_lookup_pf(const DbView db, const uint64_t *__restrict__ canon_a,
                                                         const uint32_t *__restrict__ bins_a, uint32_t *__restrict__ out,
                                                         uint64_t n_pos) {
  const uint32_t hi_mask = (uint32_t)(db.key_mask >> 32);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t bin_c = g < n_pos ? __ldg(bins_a + g) : X_BIN_NONE;
  uint64_t canon_c = g < n_pos ? __ldg(canon_a + g) : 0ull;
  uint32_t bin_1 = g + stride < n_pos ? __ldg(bins_a + g + stride) : X_BIN_NONE;
  uint64_t canon_1 = g + stride < n_pos ? __ldg(canon_a + g + stride) : 0ull;
  uint64_t o0_c = 0, o1_c = 0;
  if (bin_c >= db.bin_lo && bin_c < db.bin_hi) {
    o0_c = __ldg(db.offsets + (bin_c - db.bin_lo));
    o1_c = __ldg(db.offsets + (bin_c - db.bin_lo) + 1);
  }
  for (; g < n_pos; g += stride) {
    uint32_t bin_2 = X_BIN_NONE;
    uint64_t canon_2 = 0;
    if (g + 2 * stride < n_pos) { bin_2 = __ldg(bins_a + g + 2 * stride); canon_2 = __ldg(canon_a + g + 2 * stride); }
    uint64_t o0_1 = 0, o1_1 = 0;
    if (bin_1 >= db.bin_lo && bin_1 < db.bin_hi) {
      o0_1 = __ldg(db.offsets + (bin_1 - db.bin_lo));
      o1_1 = __ldg(db.offsets + (bin_1 - db.bin_lo) + 1);
    }
    if (bin_c == X_BIN_AMBIG) out[g] = AMBIG;
    else if (bin_c != X_BIN_NONE) out[g] = search12(db, hi_mask, canon_c, o0_c, o1_c);   // o0 == o1 == 0 outside the range
    bin_c = bin_1; canon_c = canon_1; o0_c = o0_1; o1_c = o1_1;
    bin_1 = bin_2; canon_1 = canon_2;
  }
}

// Shape "ILP": every thread searches ILP windows (text positions g, g + stride, ...) in lock step, so ILP times as many
// independent loads are in flight per thread at every level of the chain.
template <int ILP, int MINB>
__global__ void __launch_bounds__(256, MINB) k_lookup_ilp(const DbView db, const uint64_t *__restrict__ canon_a,
                                                          const uint32_t *__restrict__ bins_a, uint32_t *__restrict__ out,
                                                          uint64_t n_pos) {
  const uint32_t hi_mask = (uint32_t)(db.key_mask >> 32);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t g0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g0 < n_pos; g0 += stride * ILP) {
    uint32_t bin[ILP], n[ILP], taxon[ILP];
    uint64_t canon[ILP], lo[ILP];
#pragma unroll
    for (int j = 0; j < ILP; j++) {
      const uint64_t g = g0 + (uint64_t)j * stride;
      bin[j] = g < n_pos ? __ldg(bins_a + g) : X_BIN_NONE;
      canon[j] = g < n_pos ? __ldg(canon_a + g) : 0ull;
    }
    {
      uint64_t o0[ILP], o1[ILP];
#pragma unroll
      for (int j = 0; j < ILP; j++) {
        const bool in = bin[j] >= db.bin_lo && bin[j] < db.bin_hi;
        o0[j] = in ? __ldg(db.offsets + (bin[j] - db.bin_lo)) : 0ull;
        o1[j] = in ? __ldg(db.offsets + (bin[j] - db.bin_lo) + 1) : 0ull;
      }
#pragma unroll
      for (int j = 0; j < ILP; j++) { lo[j] = o0[j] - db.rec_base; n[j] = (uint32_t)(o1[j] - o0[j]); taxon[j] = 0; }
    }
    bool more = false;
#pragma unroll
    for (int j = 0; j < ILP; j++) more = more || n[j] > 8u;
    while (more) {
      uint64_t k1[ILP], k2[ILP], k3[ILP];
#pragma unroll
      for (int j = 0; j < ILP; j++) {
        const uint32_t q = n[j] >> 2;
        const bool act = n[j] > 8u;
        k1[j] = act ? key12(db.pairs, lo[j] + q, db.key_mask) : 0ull;
        k2[j] = act ? key12(db.pairs, lo[j] + 2 * q, db.key_mask) : 0ull;
        k3[j] = act ? key12(db.pairs, lo[j] + 3 * q, db.key_mask) : 0ull;
      }
      more = false;
#pragma unroll
      for (int j = 0; j < ILP; j++) {
        if (n[j] > 8u) {
          const uint32_t q = n[j] >> 2;
          if (canon[j] >= k3[j]) { lo[j] += 3 * q; n[j] -= 3 * q; }
          else if (canon[j] >= k2[j]) { lo[j] += 2 * q; n[j] = q; }
          else if (canon[j] >= k1[j]) { lo[j] += q; n[j] = q; }
          else { n[j] = q; }
        }
        more = more || n[j] > 8u;
      }
    }
    uint32_t lw[ILP][8];
#pragma unroll
    for (int j = 0; j < ILP; j++) {
      const uint32_t *b = reinterpret_cast<const uint32_t *>(db.pairs + lo[j] * 12);
#pragma unroll
      for (int t = 0; t < 8; t++) lw[j][t] = ((uint32_t)t < n[j]) ? __ldg(b + 3 * t) : 0;
    }
#pragma unroll
    for (int j = 0; j < ILP; j++) {
      const uint32_t *b = reinterpret_cast<const uint32_t *>(db.pairs + lo[j] * 12);
      const uint32_t clo = (uint32_t)canon[j], chi = (uint32_t)(canon[j] >> 32);
      uint32_t m = 0;
#pragma unroll
      for (int t = 0; t < 8; t++) m |= ((uint32_t)t < n[j] && lw[j][t] == clo) ? (1u << t) : 0u;
      while (m) {
        const int t = __ffs(m) - 1;
        m &= m - 1;
        if ((__ldg(b + 3 * t + 1) & hi_mask) == chi) { taxon[j] = __ldg(b + 3 * t + 2); m = 0; }
      }
    }
#pragma unroll
    for (int j = 0; j < ILP; j++) {
      const uint64_t g = g0 + (uint64_t)j * stride;
      if (g < n_pos && bin[j] != X_BIN_NONE) out[g] = bin[j] == X_BIN_AMBIG ? AMBIG : taxon[j];
    }
  }
}

// Two-level search tree per bin, a pure function of the bin's record count n (no per-bin metadata):
//   n <= 8           sorted, as staged
//   9 <= n < 36      [3 pivots at sorted positions floor((c + 1) n / 4)][4 leaves in key order]
//   n >= 36          [those 3 pivots][3 pivots per quarter, at floor((d + 1) m / 4) of the quarter's m records, in
//                    quarter order][16 leaves in key order]
// Below 36 records one level leaves at most 8 records per leaf (the scan window) already; from 36 on a quarter holds
// at least 8 records, so its 3 pivots are distinct and a leaf holds at most 8 records up to about 140.
constexpr uint32_t TREE_MIN = 9, TREE_TWO = 36;

// stored position of the record at sorted position i of a bin of n records
__host__ __device__ inline uint32_t tree_slot(uint32_t n, uint32_t i) {
  if (n < TREE_MIN) return i;
  uint32_t c = 0;                                          // level-1 pivots before i
  while (c < 3 && (uint32_t)(((uint64_t)(c + 1) * n) >> 2) < i) c++;
  if (c < 3 && i == (uint32_t)(((uint64_t)(c + 1) * n) >> 2)) return c;
  const uint32_t q0 = c ? (uint32_t)(((uint64_t)c * n) >> 2) + 1 : 0, q1 = (uint32_t)(((uint64_t)(c + 1) * n) >> 2);
  if (n < TREE_TWO) return 3 + i - c;
  const uint32_t m = q1 - q0, j = i - q0;
  uint32_t d = 0;                                          // level-2 pivots of the quarter before i
  while (d < 3 && (uint32_t)(((uint64_t)(d + 1) * m) >> 2) < j) d++;
  if (d < 3 && j == (uint32_t)(((uint64_t)(d + 1) * m) >> 2)) return 3 + 3 * c + d;
  return 15 + i - 4 * c - d;
}

// out-of-place copy of the staged records into the tree layout, one thread per bin; bad counts bins whose keys are not
// strictly increasing (the layout would not be a search tree there)
__global__ void __launch_bounds__(256) k_tree_copy(const DbView db, uint8_t *__restrict__ tree, unsigned long long *bad) {
  const uint64_t n_bins = db.bin_hi - db.bin_lo, stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b < n_bins; b += stride) {
    const uint64_t lo = __ldg(db.offsets + b) - db.rec_base;
    const uint32_t n = (uint32_t)(__ldg(db.offsets + b + 1) - __ldg(db.offsets + b));
    uint64_t prev = 0;
    for (uint32_t i = 0; i < n; i++) {
      const uint32_t *s = reinterpret_cast<const uint32_t *>(db.pairs + (lo + i) * 12);
      uint32_t *d = reinterpret_cast<uint32_t *>(tree + (lo + tree_slot(n, i)) * 12);
      d[0] = s[0]; d[1] = s[1]; d[2] = s[2];
      const uint64_t key = key12(db.pairs, lo + i, db.key_mask);
      if (i && key <= prev) atomicAdd(bad, 1ull);
      prev = key;
    }
  }
}

template <bool PF>
__device__ __forceinline__ uint64_t tree_key(const uint8_t *pairs, uint64_t pos, uint64_t key_mask) {
  return PF ? key12_pf(pairs, pos, key_mask) : key12(pairs, pos, key_mask);
}

// narrows [lo, lo + n) of a bin of n > 8 records in the tree layout to the leaf that can hold canon, or to the one
// pivot equal to it (n = 1); PF: the header loads ask L2 for the 256-byte block
template <bool PF>
__device__ __forceinline__ void tree_narrow(const uint8_t *pairs, uint64_t key_mask, uint64_t canon, uint64_t &lo, uint32_t &n) {
  const uint64_t k0 = tree_key<PF>(pairs, lo, key_mask), k1 = tree_key<PF>(pairs, lo + 1, key_mask),
                 k2 = tree_key<PF>(pairs, lo + 2, key_mask);
  const uint32_t c = (canon > k0 ? 1u : 0u) + (canon > k1 ? 1u : 0u) + (canon > k2 ? 1u : 0u);
  if (canon == k0 || canon == k1 || canon == k2) { lo += c; n = 1; return; }   // keys increase: pivot c is the equal one
  const uint32_t q0 = c ? (uint32_t)(((uint64_t)c * n) >> 2) + 1 : 0, q1 = (uint32_t)(((uint64_t)(c + 1) * n) >> 2);
  if (n < TREE_TWO) { lo += 3 + q0 - c; n = q1 - q0; return; }
  const uint64_t h = lo + 3 + 3 * c;
  const uint64_t l0 = key12(pairs, h, key_mask), l1 = key12(pairs, h + 1, key_mask), l2 = key12(pairs, h + 2, key_mask);
  const uint32_t d = (canon > l0 ? 1u : 0u) + (canon > l1 ? 1u : 0u) + (canon > l2 ? 1u : 0u);
  if (canon == l0 || canon == l1 || canon == l2) { lo = h + d; n = 1; return; }
  const uint32_t m = q1 - q0;
  const uint32_t s = q0 + (d ? (uint32_t)(((uint64_t)d * m) >> 2) + 1 : 0), e = q0 + (uint32_t)(((uint64_t)(d + 1) * m) >> 2);
  lo += 15 + s - 4 * c - d;
  n = e - s;
}

// shape 0 (12 B, 4-ary, scan <= 8) on the tree layout: the tree's two levels, then the 4-ary narrowing inside a leaf
// of more than 8 records (bins of more than about 140)
template <bool PF>
__global__ void __launch_bounds__(256, 8) k_lookup_tree(const DbView db, const uint8_t *__restrict__ tree,
                                                        const uint64_t *__restrict__ canon_a, const uint32_t *__restrict__ bins_a,
                                                        uint32_t *__restrict__ out, uint64_t n_pos) {
  const uint32_t hi_mask = (uint32_t)(db.key_mask >> 32);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t bin_n = g < n_pos ? __ldg(bins_a + g) : X_BIN_NONE;
  uint64_t canon_n = g < n_pos ? __ldg(canon_a + g) : 0ull;
  for (; g < n_pos; g += stride) {
    const uint32_t bin = bin_n;
    const uint64_t canon = canon_n;
    if (g + stride < n_pos) { bin_n = __ldg(bins_a + g + stride); canon_n = __ldg(canon_a + g + stride); }
    if (bin == X_BIN_NONE) continue;
    if (bin == X_BIN_AMBIG) { out[g] = AMBIG; continue; }
    uint32_t taxon = 0;
    if (bin >= db.bin_lo && bin < db.bin_hi) {
      const uint64_t *o = db.offsets + (bin - db.bin_lo);
      const uint64_t o0 = __ldg(o), o1 = __ldg(o + 1);
      uint64_t lo = o0 - db.rec_base;
      uint32_t n = (uint32_t)(o1 - o0);
      if (n > 8u) tree_narrow<PF>(tree, db.key_mask, canon, lo, n);
      while (n > 8u) {
        const uint32_t q = n >> 2;
        const uint64_t k1 = key12(tree, lo + q, db.key_mask), k2 = key12(tree, lo + 2 * q, db.key_mask),
                       k3 = key12(tree, lo + 3 * q, db.key_mask);
        const uint32_t c = (canon >= k1 ? 1u : 0u) + (canon >= k2 ? 1u : 0u) + (canon >= k3 ? 1u : 0u);
        lo += (uint64_t)c * q;
        n = (c == 3u) ? n - 3 * q : q;
      }
      if (n) {
        const uint32_t *b = reinterpret_cast<const uint32_t *>(tree + lo * 12);
        const uint32_t clo = (uint32_t)canon, chi = (uint32_t)(canon >> 32);
        uint32_t lw[8];
#pragma unroll
        for (int t = 0; t < 8; t++) lw[t] = ((uint32_t)t < n) ? __ldg(b + 3 * t) : 0;
        uint32_t m = 0;
#pragma unroll
        for (int t = 0; t < 8; t++) m |= ((uint32_t)t < n && lw[t] == clo) ? (1u << t) : 0u;
        while (m) {
          const int t = __ffs(m) - 1;
          m &= m - 1;
          if ((__ldg(b + 3 * t + 1) & hi_mask) == chi) { taxon = __ldg(b + 3 * t + 2); m = 0; }
        }
      }
    }
    out[g] = taxon;
  }
}

// counters: [0] looked-up windows, [1] sum of ceil(log2(n + 1)), [2..7] windows by bin size class, [8] mismatches
__global__ void __launch_bounds__(256) k_layout_stats(const DbView db, const uint32_t *__restrict__ bins_a, uint64_t n_pos,
                                                      unsigned long long *counters) {
  __shared__ unsigned long long acc[8];
  if (threadIdx.x < 8) acc[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_pos; g += stride) {
    const uint32_t bin = __ldg(bins_a + g);
    if (bin == X_BIN_NONE || bin == X_BIN_AMBIG || bin < db.bin_lo || bin >= db.bin_hi) continue;
    const uint64_t *o = db.offsets + (bin - db.bin_lo);
    const uint32_t n = (uint32_t)(__ldg(o + 1) - __ldg(o));
    const int cls = n <= 8 ? 2 : n <= 16 ? 3 : n <= 64 ? 4 : n <= 256 ? 5 : n <= 1024 ? 6 : 7;
    atomicAdd(&acc[0], 1ull);
    atomicAdd(&acc[1], (unsigned long long)(n ? 32 - __clz(n) : 0));
    atomicAdd(&acc[cls], 1ull);
  }
  __syncthreads();
  if (threadIdx.x < 8 && acc[threadIdx.x]) atomicAdd(counters + threadIdx.x, acc[threadIdx.x]);
}

__global__ void __launch_bounds__(256) k_layout_check(const DbView db, const uint32_t *__restrict__ bins_a,
                                                      const uint32_t *__restrict__ ref, const uint32_t *__restrict__ out,
                                                      uint64_t n_pos, unsigned long long *mismatches) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  unsigned long long bad = 0;
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_pos; g += stride) {
    const uint32_t bin = __ldg(bins_a + g);
    if (bin == X_BIN_NONE) continue;
    if (bin != X_BIN_AMBIG && (bin < db.bin_lo || bin >= db.bin_hi)) continue;   // window of another range
    uint32_t want = __ldg(ref + g);
    if (want != AMBIG) want &= ~KEEP_NEW;                  // a fused call in keep mode marks some hits (F_KEEP)
    if (want != __ldg(out + g)) bad++;
  }
  if (bad) atomicAdd(mismatches, bad);
}

// shape: 0 = thread per window (the product's shape), 1 = the product's own k_lookup<MODE_LOOKUP> with its run-time
// switches, 2 / 3 = index prefetch at 8 / 6 CTAs per SM, 4 / 5 / 6 = two windows per thread at 8 / 6 / 4 CTAs per SM,
// 7 = four windows at 4, 8 = the product's k_lookup<MODE_LOOKUP> with the switches compiled out (LEAN), 9 / 10 = the
// product's k_lookup<MODE_FUSED> (search + sketch update) with run-time switches / LEAN, 11 = shape 0 with the
// narrowing step written as an if / else-if chain, 12 = shape 0 fed through the product's Params block, 13 = shape 0
// with the first round's pivots loaded through key12_pf, 14 / 15 = shape 0 on the tree layout (k_tree_copy) with the
// header loaded plainly / through key12_pf
struct Variant { int rec, arity, window, shape; };
constexpr Variant VARIANTS[KUQ_LAYOUT_VARIANTS] = {
    {12, 4, 8, 0}, {12, 8, 8, 0}, {12, 4, 16, 0}, {12, 8, 16, 0}, {12, 16, 16, 0}, {8, 4, 8, 0}, {8, 8, 8, 0}, {8, 4, 16, 0},
    {8, 8, 16, 0}, {8, 16, 16, 0}, {12, 4, 8, 1}, {12, 4, 8, 2}, {12, 4, 8, 3}, {12, 4, 8, 4}, {12, 4, 8, 5}, {12, 4, 8, 6},
    {12, 4, 8, 7}, {12, 4, 8, 8}, {12, 4, 8, 9}, {12, 4, 8, 10}, {12, 4, 8, 11}, {12, 4, 8, 12}, {12, 4, 8, 13},
    {12, 4, 8, 14}, {12, 4, 8, 15}};

void launch_variant(int v, int grid, cudaStream_t st, const Params &product, int n_sm, const unsigned long long *rec8,
                    const uint8_t *tree, const uint64_t *canon, const uint32_t *bins, uint32_t *out, uint64_t n_pos) {
  const DbView &db = product.db;
  switch (v) {
    case 0: k_lookup_variant<12, 4, 8><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 1: k_lookup_variant<12, 8, 8><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 2: k_lookup_variant<12, 4, 16><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 3: k_lookup_variant<12, 8, 16><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 4: k_lookup_variant<12, 16, 16><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 5: k_lookup_variant<8, 4, 8><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 6: k_lookup_variant<8, 8, 8><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 7: k_lookup_variant<8, 4, 16><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 8: k_lookup_variant<8, 8, 16><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 9: k_lookup_variant<8, 16, 16><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 10: launch_lookup_only(product, n_sm, st, 0, 0); break;
    case 11: k_lookup_pf<8><<<grid, 256, 0, st>>>(db, canon, bins, out, n_pos); break;
    case 12: k_lookup_pf<6><<<std::min(grid, n_sm * 6 * 8), 256, 0, st>>>(db, canon, bins, out, n_pos); break;
    case 13: k_lookup_ilp<2, 8><<<grid, 256, 0, st>>>(db, canon, bins, out, n_pos); break;
    case 14: k_lookup_ilp<2, 6><<<std::min(grid, n_sm * 6 * 8), 256, 0, st>>>(db, canon, bins, out, n_pos); break;
    case 15: k_lookup_ilp<2, 4><<<std::min(grid, n_sm * 4 * 8), 256, 0, st>>>(db, canon, bins, out, n_pos); break;
    case 16: k_lookup_ilp<4, 4><<<std::min(grid, n_sm * 4 * 8), 256, 0, st>>>(db, canon, bins, out, n_pos); break;
    case 17: launch_lookup_only(product, n_sm, st, 0, 1); break;
    case 18: launch_lookup_only(product, n_sm, st, 1, 0); break;
    case 19: launch_lookup_only(product, n_sm, st, 1, 1); break;
    case 20: k_lookup_variant<12, 4, 8, 1><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 21: k_lookup_params<<<grid, 256, 0, st>>>(product); break;
    case 22: k_lookup_variant<12, 4, 8, 2><<<grid, 256, 0, st>>>(db, rec8, canon, bins, out, n_pos); break;
    case 23: k_lookup_tree<false><<<grid, 256, 0, st>>>(db, tree, canon, bins, out, n_pos); break;
    default: k_lookup_tree<true><<<grid, 256, 0, st>>>(db, tree, canon, bins, out, n_pos); break;
  }
}

}  // namespace

// 0 = ok, 1 = out of device memory, 2 = CUDA error, 3 = dense taxon ids need more than 24 bits
int layout_experiment(const Params &product_in, uint64_t n_records, const uint64_t *canon, const uint32_t *bins, const uint32_t *ref,
                      uint64_t n_pos, int n_sm, cudaStream_t st, uint32_t reps, int allow_fused, kuq_layout_result *res) {
  const DbView &db = product_in.db;
  memset(res, 0, sizeof *res);
  res->n_records = n_records;
  res->n_positions = n_pos;
  res->n_variants = KUQ_LAYOUT_VARIANTS;
  unsigned long long *rec8 = nullptr, *counters = nullptr;
  uint64_t *two = nullptr;                     // {0, n_pos}: the text range of the product kernel's launch
  uint32_t *out = nullptr, *err = nullptr;
  uint8_t *tree = nullptr;                     // the records in the tree layout (k_tree_copy)
  cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr, e3 = nullptr;
  int rc = 0;
  auto cleanup = [&]() {
    cudaFree(rec8); cudaFree(counters); cudaFree(out); cudaFree(err); cudaFree(two); cudaFree(tree);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (e2) cudaEventDestroy(e2);
    if (e3) cudaEventDestroy(e3);
  };
  if (cudaMalloc((void **)&rec8, std::max<uint64_t>(n_records, 1) * 8) != cudaSuccess ||
      cudaMalloc((void **)&out, std::max<uint64_t>(n_pos, 1) * 4) != cudaSuccess ||
      cudaMalloc((void **)&counters, 16 * 8) != cudaSuccess || cudaMalloc((void **)&err, 4) != cudaSuccess ||
      cudaMalloc((void **)&two, 16) != cudaSuccess || cudaMalloc((void **)&tree, std::max<uint64_t>(n_records, 1) * 12) != cudaSuccess) {
    (void)cudaGetLastError();
    cleanup();
    return 1;
  }
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventCreate(&e2);
  cudaEventCreate(&e3);
  cudaMemsetAsync(counters, 0, 16 * 8, st);
  cudaMemsetAsync(err, 0, 4, st);
  const uint64_t h_two[2] = {0, n_pos};
  cudaMemcpyAsync(two, h_two, 16, cudaMemcpyHostToDevice, st);
  Params product = product_in;                 // a plain lookup of one range: ids of all windows into `out`, no sketch work
  product.offsets = two;
  product.n_reads = 1;
  product.total_bases = n_pos;
  product.canon = const_cast<uint64_t *>(canon);
  product.bins = const_cast<uint32_t *>(bins);
  product.flags = 0;
  product.only_hits = 0;
  product.n_peers = 0;
  const int tgrid = n_sm * 8;
  cudaEventRecord(e0, st);
  k_transcode8<<<tgrid, 256, 0, st>>>(db.pairs, n_records, db.key_mask, db.xor_mask, rec8, err);
  cudaEventRecord(e1, st);
  const int lgrid = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)n_sm * 8 * 8, (n_pos + 255) / 256));
  k_layout_stats<<<lgrid, 256, 0, st>>>(db, bins, n_pos, counters);
  cudaEventRecord(e2, st);
  k_tree_copy<<<tgrid, 256, 0, st>>>(db, tree, counters + 9);
  cudaEventRecord(e3, st);
  uint32_t h_err = 0;
  unsigned long long h_cnt[16];
  cudaMemcpyAsync(&h_err, err, 4, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(h_cnt, counters, sizeof h_cnt, cudaMemcpyDeviceToHost, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) { (void)cudaGetLastError(); cleanup(); return 2; }
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  res->transcode_ms = ms;
  cudaEventElapsedTime(&ms, e2, e3);
  res->tree_ms = ms;
  res->tree_unordered = h_cnt[9];
  if (h_err) { cleanup(); return 3; }
  res->n_windows = h_cnt[0];
  res->sum_probes = h_cnt[1];
  for (int i = 0; i < 6; i++) res->bin_class[i] = h_cnt[2 + i];
  if (reps == 0) reps = 1;
  for (int v = 0; v < KUQ_LAYOUT_VARIANTS; v++) {
    res->rec_bytes[v] = (uint32_t)VARIANTS[v].rec;
    res->arity[v] = (uint32_t)VARIANTS[v].arity;
    res->window[v] = (uint32_t)VARIANTS[v].window;
    res->shape[v] = (uint32_t)VARIANTS[v].shape;
    product.codes_dense = out;
    if (VARIANTS[v].shape >= 9 && !allow_fused) continue;      // would count into sketches that are not dense-only
    cudaMemsetAsync(out, 0xEE, std::max<uint64_t>(n_pos, 1) * 4, st);
    launch_variant(v, lgrid, st, product, n_sm, rec8, tree, canon, bins, out, n_pos);   // warm-up (and the checked result)
    double best = 1e30, sum = 0;
    for (uint32_t r = 0; r < reps; r++) {
      cudaEventRecord(e0, st);
      launch_variant(v, lgrid, st, product, n_sm, rec8, tree, canon, bins, out, n_pos);
      cudaEventRecord(e1, st);
      if (cudaEventSynchronize(e1) != cudaSuccess) { rc = 2; break; }
      cudaEventElapsedTime(&ms, e0, e1);
      best = std::min<double>(best, ms);
      sum += ms;
    }
    if (rc) break;
    res->best_ms[v] = best;
    res->mean_ms[v] = sum / reps;
    cudaMemsetAsync(counters + 8, 0, 8, st);
    k_layout_check<<<lgrid, 256, 0, st>>>(db, bins, ref, out, n_pos, counters + 8);
    unsigned long long bad = 0;
    cudaMemcpyAsync(&bad, counters + 8, 8, cudaMemcpyDeviceToHost, st);
    if (cudaStreamSynchronize(st) != cudaSuccess) { rc = 2; break; }
    res->mismatches[v] = bad;
  }
  if (cudaGetLastError() != cudaSuccess) rc = 2;
  cleanup();
  return rc;
}

}  // namespace kuq
