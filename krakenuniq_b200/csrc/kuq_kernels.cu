// kuq_kernels.cu — see kuq_kernels.cuh for the map from kernel stages to reference functions.
// Design history: round 1 first fused all stages into one persistent warp-per-read kernel; at 128 registers it ran
// at 25 % occupancy and was bound by exposed latency, so the path is now three stages that
// each keep a small register footprint.  The lookup and resolve halves hand windows over through HBM scratch (12 B per
// window, streamed); the fused call hands over a 2-bit packed copy of the batch (16 B per 32 positions) and the
// thread-per-window lookup computes its window from it.
#include "../../include/kuq.h"
#include "kuq_kernels.cuh"

namespace kuq {

// ------------------------------------------------------------------------------------------------------
// small PTX wrappers: mbarrier + 1-D TMA bulk copy (global → shared), sm_90a
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// cp.async.bulk: one thread moves `bytes` (multiple of 16, 16-byte aligned on both sides) and signals `bar`.
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ------------------------------------------------------------------------------------------------------
// bit arithmetic
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t revcomp32(uint32_t x, uint32_t n) {   // n <= 15
  x = __brev(x);
  x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
  return (~x) >> (32 - 2 * n);
}
// 12-byte records are only 4-byte aligned: a key is two 32-bit loads.
__device__ __forceinline__ uint64_t load_key(const uint8_t *pairs, uint64_t pos, uint64_t key_mask) {
  const uint32_t *p = reinterpret_cast<const uint32_t *>(pairs + pos * 12);
  uint32_t lo = __ldg(p), hi = __ldg(p + 1);
  return (((uint64_t)hi << 32) | lo) & key_mask;                                // krakendb.cpp:283-284
}
__device__ __forceinline__ uint32_t load_val(const uint8_t *pairs, uint64_t pos) {
  return __ldg(reinterpret_cast<const uint32_t *>(pairs + pos * 12) + 2);
}

// HyperLogLogPlusMinus::insert, dense branch (hyperloglogplus.cpp:514-521): M[idx] = max(M[idx], rank).
// Registers are bytes; a byte-wide max is a CAS on the enclosing word, reached only when the plain load says the
// register would grow (after warm-up almost never: P[grow] ~ 1/n).  A stale load can only be too small, which
// costs a redundant CAS, never a lost update.
// floor[taxon] is at most every register of the sketch (refreshed before each counting launch, registers only grow
// during one): a rank that low cannot raise any register, so most windows skip the register load, a dependent L2
// trip once the taxon is known.  Once a sketch has seen a few hashes per register that is most windows (rank <= 3 for
// 7 in 8 of them).
__device__ __forceinline__ void hll_update(uint8_t *regs, const uint8_t *floor, uint32_t taxon, uint64_t hash) {
  uint32_t idx = (uint32_t)(hash >> (64 - HLL_P));
  uint64_t rest = hash << HLL_P;
  uint32_t rank = rest ? (uint32_t)__clzll((long long)rest) + 1 : (64 - HLL_P + 1);   // getRank, :140-147
  if (rank <= __ldg(floor + taxon)) return;
  uint8_t *reg = regs + (size_t)taxon * HLL_M + idx;
  if (*reinterpret_cast<volatile uint8_t *>(reg) >= rank) return;
  uint32_t *word = reinterpret_cast<uint32_t *>(reinterpret_cast<uintptr_t>(reg) & ~(uintptr_t)3);
  uint32_t shift = (uint32_t)(reinterpret_cast<uintptr_t>(reg) & 3) * 8;
  uint32_t old = *reinterpret_cast<volatile uint32_t *>(word);
  while (((old >> shift) & 0xFF) < rank) {
    uint32_t upd = (old & ~(0xFFu << shift)) | (rank << shift);
    uint32_t prev = atomicCAS(word, old, upd);
    if (prev == old) break;
    old = prev;
  }
}

__device__ __forceinline__ uint64_t mix64(uint64_t x) {   // table hash for the device sets (not reference arithmetic)
  x ^= x >> 31;
  x *= 0x7fb5d329728ea185ull;
  x ^= x >> 27;
  x *= 0x81dadef4bc2dd44dull;
  x ^= x >> 33;
  return x;
}

// Insert into the (taxon, code) set behind the sparse HLL tier.  Returns 1 when the key is new, 0 when it was
// there already, -1 when the table is saturated (the host turns that into KUQ_E_CAPACITY).
__device__ __forceinline__ int sparse_insert(const SparseSet &s, uint32_t taxon, uint32_t code) {
  unsigned long long key = ((unsigned long long)(taxon + 1) << 32) | code;
  uint64_t slot = mix64(key) & s.mask;
  for (uint32_t probe = 0; probe < 512; probe++) {
    unsigned long long cur = __ldcg(s.slots + slot);          // L2 is where the CAS of other threads lands
    if (cur == key) return 0;
    if (cur == 0) {
      unsigned long long prev = atomicCAS(s.slots + slot, 0ull, key);
      if (prev == 0) return 1;
      if (prev == key) return 0;
    }
    slot = (slot + 1) & s.mask;
  }
  return -1;
}

// ------------------------------------------------------------------------------------------------------
// taxonomy walks on the flattened parent array
// ------------------------------------------------------------------------------------------------------
// lca(), krakenutil.cpp:90-118, in dense ids.  Dense id 1 is ALWAYS the node of taxid 1 (the reference's
// hard-wired root: loops run `while (a > 1)`), dense id 0 is "no taxon".  depth[] counts the steps of a node's
// parent chain until it ends (at 0, or at node 1), so both chains can be levelled first.
__device__ uint32_t lca_dense(const TaxView &t, uint32_t a, uint32_t b) {
  if (a == 0 || b == 0) return a ? a : b;
  uint32_t da = a <= 1 ? 0 : t.depth[a], db = b <= 1 ? 0 : t.depth[b];
  while (da > db) { a = t.parent[a]; da--; }
  while (db > da) { b = t.parent[b]; db--; }
  while (a != b && a > 1 && b > 1) {
    a = t.parent[a];
    b = t.parent[b];
  }
  return (a == b && a > 1) ? a : 1u;
}

// ------------------------------------------------------------------------------------------------------
// one read, one warp
// ------------------------------------------------------------------------------------------------------
struct Block64 {         // 32 bases: 2-bit codes, first base in bits 63:62; amb bit l = base l is not ACGT
  uint64_t codes;
  uint32_t amb;
  uint32_t mark;         // bit l = a window ENDS at base l (only for cleaned reads, see clean_read)
  bool skip;             // the block holds a '\n' / '\r' (not set for cleaned reads)
};


// Convert 32 characters (lane = position) — krakenutil.cpp:253-273.  Positions >= len read as ambiguous.
__device__ __forceinline__ Block64 load_block(const char *seq, uint32_t len, uint32_t blk, uint32_t lane, bool marks) {
  uint32_t pos = blk * 32 + lane;
  uint32_t c = pos < len ? (uint32_t)(uint8_t)seq[pos] : (uint32_t)'N';
  uint32_t mk = 0;
  if (marks) { mk = c >> 7; c &= 0x7Fu; }
  uint32_t code;
  const bool ok = base_code(c, code);
  uint32_t sh = 2 * (15 - (lane & 15));
  uint32_t hi = __reduce_or_sync(0xFFFFFFFFu, lane < 16 ? code << sh : 0u);
  uint32_t lo = __reduce_or_sync(0xFFFFFFFFu, lane >= 16 ? code << sh : 0u);
  Block64 b;
  b.codes = ((uint64_t)hi << 32) | lo;
  b.amb = __ballot_sync(0xFFFFFFFFu, !ok);
  b.mark = marks ? __ballot_sync(0xFFFFFFFFu, mk != 0) : 0u;
  // a skipped character is first of all a non-ACGT one: blocks without any (the common case) need no second vote
  b.skip = !marks && b.amb != 0 && __any_sync(0xFFFFFFFFu, !ok && (c == '\n' || c == '\r'));
  return b;
}

constexpr uint32_t BIN_NONE = 0xFFFFFFFFu;    // scratch marker: no window at this position
constexpr uint32_t BIN_AMBIG = 0xFFFFFFFEu;   // scratch marker: window with a non-ACGT base


// The windows of one slot of 32 (lane = window start in the 64 bases a:b): canonical k-mer (→ canon) and minimizer bin,
// or BIN_AMBIG for a window with a non-ACGT base.  Warp-uniform: the minimizer takes shuffles.
// FAST = the (k, m) = (31, 15) of every published KrakenUniq database, with the window arithmetic as constants.
template <bool FAST>
__device__ __forceinline__ uint32_t window_bin(const DbView &db, uint64_t a, uint64_t b, uint64_t amb64, uint32_t lane,
                                               uint64_t &canon) {
  const uint32_t k = FAST ? 31u : db.k, nt = FAST ? 15u : db.nt;
  const uint32_t n_mini = FAST ? 17u : db.n_mini;
  const uint64_t hi = window_top(a, b, lane);
  canon = canonical_kmer(hi, k);
  const bool amb = ((amb64 >> lane) & ((1ull << k) - 1)) != 0;   // any non-ACGT base in the window, :275,280-282
  // minimizer = min over the k-nt+1 nt-mers of (xor_mask ^ canonical(nt-mer)) (krakendb.cpp:200-215).
  // Candidate of position q (0..63 relative to the slot): lane holds q = lane (m0) and q = 32+lane (m1).
  uint32_t f0 = (uint32_t)(hi >> (64 - 2 * nt));
  uint32_t r0 = revcomp32(f0, nt);
  uint32_t m0 = db.xor_mask ^ (f0 < r0 ? f0 : r0);
  uint32_t f1 = (uint32_t)((b << (2 * lane)) >> (64 - 2 * nt));
  uint32_t r1 = revcomp32(f1, nt);
  uint32_t m1 = db.xor_mask ^ (f1 < r1 ? f1 : r1);
  // sliding-window minimum of width n_mini by doubling: after the loop m0 holds min over [q, q+n_mini)
  uint32_t w = 1;
#pragma unroll
  for (int step = 0; step < 5; step++) {                  // n_mini <= 31 → at most 4 doublings
    if (2 * w > n_mini) break;
    uint32_t src = (lane + w) & 31;
    uint32_t x0 = __shfl_sync(0xFFFFFFFFu, m0, src), x1 = __shfl_sync(0xFFFFFFFFu, m1, src);
    bool wrap = lane + w >= 32;
    m0 = min(m0, wrap ? x1 : x0);
    m1 = min(m1, wrap ? 0xFFFFFFFFu : x1);
    w *= 2;
  }
  if (w < n_mini) {                                       // [q, q+n_mini) = [q, q+w) U [q+n_mini-w, q+n_mini)
    uint32_t d = n_mini - w;
    uint32_t src = (lane + d) & 31;
    uint32_t x0 = __shfl_sync(0xFFFFFFFFu, m0, src), x1 = __shfl_sync(0xFFFFFFFFu, m1, src);
    m0 = min(m0, lane + d >= 32 ? x1 : x0);
  }
  return amb ? BIN_AMBIG : m0;
}

// Stage 1 for one read (one warp, one slot of 32 windows at a time): canonical k-mer and minimizer bin of every
// window → scratch.  Pure ALU + shuffles, no dependent memory access.
// Returns false (having possibly written a prefix of the read's windows, all of which the caller rewrites) when it
// meets a skipped character: the read then goes through clean_read.
template <bool FAST>
__device__ bool scan_read(const Params &p, uint32_t r, const char *seq, uint32_t len, uint32_t raw_len,
                          uint64_t out_base, uint32_t lane, bool marks) {
  const DbView &db = p.db;
  const uint32_t k = FAST ? 31u : db.k;
  // candidate windows; every one of them is a scanner window unless the read was cleaned (marks), in which case
  // only the marked ones are (the scanner drops a window per skipped character, see clean_read)
  const uint32_t nwin = len >= k ? len - k + 1 : 0;           // classify.cpp:913-914
  uint32_t n_out = 0;                                         // windows emitted so far
  if (nwin > 0) {
    Block64 A = load_block(seq, len, 0, lane, marks);
    if (A.skip) return false;
    const uint32_t nslots = (nwin + 31) / 32;
    for (uint32_t s = 0; s < nslots; s++) {
      Block64 B = load_block(seq, len, s + 1, lane, marks);
      if (B.skip) return false;
      const uint32_t i = s * 32 + lane;
      bool valid = i < nwin;
      if (marks) valid = valid && (((((uint64_t)B.mark << 32) | A.mark) >> (lane + k - 1)) & 1);
      const uint32_t vmask = __ballot_sync(0xFFFFFFFFu, valid);
      const uint32_t oi = n_out + __popc(vmask & ((1u << lane) - 1));   // output slot of this window
      n_out += __popc(vmask);
      // window i: bases [i, i+k) of the 128-bit string A:B
      uint64_t canon;
      const uint32_t bin = window_bin<FAST>(db, A.codes, B.codes, ((uint64_t)B.amb << 32) | A.amb, lane, canon);
      if (valid) {
        p.bins[out_base + oi] = bin;
        p.canon[out_base + oi] = canon;
      }
      A = B;
    }
  }
  // positions of the read's text that carry no window
  for (uint32_t q = n_out + lane; q < raw_len; q += 32) p.bins[out_base + q] = BIN_NONE;
  if (lane == 0) p.n_windows[r] = n_out;
  return true;
}

// A read that contains '\n' / '\r' (CRLF input, SURVEY App. A9).  KmerScanner::next_kmer (krakenutil.cpp:239-278)
// "skips" such a character by undoing the loaded_nt increment (:265-269), but the base that follows a skipped
// character is then loaded WITHOUT being counted (skip_pos, :246-247), and every further skipped character of a
// run decrements loaded_nt once more.  Net effect: each skipped character makes the scanner swallow one extra
// base, i.e. one k-mer window is never produced.  If the text ends while a call is still loading, the scanner
// reads the string terminator as an ambiguous base and produces one last (ambiguous) window.
// The warp's lane 0 replays that automaton once (rare path) and writes the cleaned bases to scratch, setting bit 7
// of the base each produced window ENDS at; process_read then only keeps the marked windows.
__device__ uint32_t clean_read(const char *seq, uint32_t len, char *dst, uint32_t k, uint32_t lane) {
  uint32_t n = 0;
  if (lane == 0) {
    int loaded = 0;
    bool skipflag = false;
    int64_t last_emit = -1;
    for (uint32_t i = 0; i < len; i++) {
      char c = seq[i];
      if (c == '\n' || c == '\r') {
        if (skipflag) loaded--;
        skipflag = true;
      } else {
        uint8_t o = ((uint8_t)c & 0x80) ? (uint8_t)'N' : (uint8_t)c;   // bit 7 is the window mark
        if (!skipflag) {
          loaded++;
          if (loaded == (int)k) { o |= 0x80; loaded = (int)k - 1; last_emit = i; }
        }
        skipflag = false;
        dst[n++] = (char)o;
      }
    }
    if (len >= k && last_emit + 1 < (int64_t)len) {     // a call is still loading: one last, ambiguous window
      uint32_t target = n + 1 > k ? n + 1 : k;          // <= len because at least one character was skipped
      while (n < target) dst[n++] = 'N';
      dst[n - 1] = (char)((uint8_t)'N' | 0x80);
    }
  }
  n = __shfl_sync(0xFFFFFFFFu, n, 0);
  __syncwarp();
  return n;
}

// ------------------------------------------------------------------------------------------------------
// the persistent kernel
// ------------------------------------------------------------------------------------------------------
struct __align__(16) SharedState {
  uint64_t off[N_STAGES][CHUNK_READS + 2];   // read offsets of the chunk (bulk-copied with the bases)
  uint64_t bar[N_STAGES];
  uint64_t a0[N_STAGES];                     // global byte offset the stage's text starts at
  uint32_t chunk[N_STAGES];
  uint32_t staged[N_STAGES];
  uint32_t next_read[N_STAGES];              // warps take the reads of a chunk from this counter
};

// Stage 1: persistent CTAs; one thread pulls the next chunk of reads (offsets slice + text) into shared memory
// with TMA bulk copies while the warps still scan the previous chunk.
__global__ void __launch_bounds__(CTA_THREADS, 4) k_scan(const __grid_constant__ Params p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t *stage_buf = smem;                                                   // N_STAGES x STAGE_BYTES
  SharedState *ss = reinterpret_cast<SharedState *>(smem + N_STAGES * STAGE_BYTES);
  const uint32_t tid = threadIdx.x, lane = tid & 31;

  auto fetch = [&](uint32_t st) {
    uint32_t c = atomicAdd(p.chunk_counter, 1u);
    ss->chunk[st] = c;
    ss->staged[st] = 0;
    ss->next_read[st] = 0;
    if (c < p.n_chunks) {
      const uint32_t r0 = c * CHUNK_READS, r1 = min(r0 + CHUNK_READS, p.n_reads);
      const uint32_t n_off = (r1 - r0 + 2) & ~1u;                  // even count → multiple of 16 bytes
      const uint64_t b0 = p.offsets[r0], b1 = p.offsets[r1];
      const uint64_t a0 = b0 & ~15ull, a1 = (b1 + 15) & ~15ull;
      ss->a0[st] = a0;
      uint32_t bytes = n_off * 8;
      const bool text = a1 - a0 <= (uint64_t)STAGE_BYTES && a1 > a0;
      if (text) bytes += (uint32_t)(a1 - a0);
      mbar_expect_tx(&ss->bar[st], bytes);
      tma_load_1d(&ss->off[st][0], p.offsets + r0, n_off * 8, &ss->bar[st]);
      if (text) {
        tma_load_1d(stage_buf + st * STAGE_BYTES, p.bases + a0, (uint32_t)(a1 - a0), &ss->bar[st]);
        ss->staged[st] = 1;
      }
    }
  };

  if (tid == 0) {
    for (int s = 0; s < N_STAGES; s++) mbar_init(&ss->bar[s], 1);
    mbar_fence_init();
    fetch(0);
  }
  __syncthreads();
  uint32_t phase[N_STAGES] = {0, 0};
  const bool fast = p.db.k == 31 && p.db.nt == 15;
  for (uint32_t it = 0;; it++) {
    const uint32_t st = it & 1;
    const uint32_t c = ss->chunk[st];
    if (c >= p.n_chunks) break;
    if (tid == 0) fetch(st ^ 1);        // the other stage was released by the barrier that ended the last round
    const bool staged = ss->staged[st] != 0;
    const uint64_t a0 = ss->a0[st];
    mbar_wait(&ss->bar[st], phase[st]);
    phase[st] ^= 1;
    const uint32_t r0 = c * CHUNK_READS, r1 = min(r0 + CHUNK_READS, p.n_reads);
    for (;;) {
      uint32_t q = 0;
      if (lane == 0) q = atomicAdd(&ss->next_read[st], 1u);
      q = __shfl_sync(0xFFFFFFFFu, q, 0);
      const uint32_t r = r0 + q;
      if (r >= r1) break;
      const uint64_t b0 = ss->off[st][q], b1 = ss->off[st][q + 1];
      const uint32_t raw_len = (uint32_t)(b1 - b0);
      uint32_t len = raw_len;
      const char *seq = staged ? reinterpret_cast<const char *>(stage_buf + st * STAGE_BYTES + (b0 - a0))
                               : p.bases + b0;
      const bool done = fast ? scan_read<true>(p, r, seq, len, raw_len, b0, lane, false)
                             : scan_read<false>(p, r, seq, len, raw_len, b0, lane, false);
      if (!done) {   // the read holds '\n' / '\r' (rare: CRLF input): replay the scanner, then rescan the cleaned copy
        len = clean_read(seq, len, p.clean + b0, p.db.k, lane);
        scan_read<false>(p, r, p.clean + b0, len, raw_len, b0, lane, true);
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------------
// the fused path's stage 1: a 2-bit packed copy of the batch instead of 12 bytes of scratch per window
// ------------------------------------------------------------------------------------------------------
// blocks [g_begin / 32, g_end / 32 + 2): every block a window of the text starts in, and the block after it
__device__ __forceinline__ uint64_t pack_block_end(uint64_t g_end) { return ((g_end + 31) >> 5) + 1; }

// Position-parallel: one thread converts 16 bases (one 16-byte load), two lanes make a block.  Positions outside the
// batch's text are ambiguous; start bits are cleared (k_pack_reads sets them).  Blocks holding '\n' / '\r' keep those
// positions in `side` and are counted in p.chunk_counter (k_scan's chunk scheduler, idle on this path).
__global__ void __launch_bounds__(256) k_pack(const __grid_constant__ Params p) {
  const uint64_t g_begin = p.offsets[0], g_end = p.offsets[p.n_reads];
  const uint64_t h_begin = (g_begin >> 5) * 2, h_end = pack_block_end(g_end) * 2;   // half blocks of 16 bases
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  // warp-uniform trip count: the two lanes of a block meet in a shuffle
  for (uint64_t h0 = h_begin + (((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~31ull); h0 < h_end; h0 += stride) {
    const uint64_t h = h0 + lane, pos0 = h * 16;
    uint32_t code32 = 0, amb16 = 0xFFFFu, crlf16 = 0;
    if (h < h_end && pos0 < g_end && pos0 + 16 > g_begin) {
      const uint4 v = __ldg(reinterpret_cast<const uint4 *>(p.bases + pos0));   // bases: 16-byte aligned, 64 B of slack
      const uint32_t wd[4] = {v.x, v.y, v.z, v.w};
      amb16 = 0;
#pragma unroll
      for (int i = 0; i < 16; i++) {
        const uint32_t c = (wd[i >> 2] >> (8 * (i & 3))) & 0xFFu;
        uint32_t code;
        const bool ok = base_code(c, code);
        code32 |= code << (2 * (15 - i));
        amb16 |= ok ? 0u : 1u << i;
        crlf16 |= (c == '\n' || c == '\r') ? 1u << i : 0u;
      }
      // bases outside [g_begin, g_end) belong to no read of the batch
      const uint32_t lo = g_begin > pos0 ? (uint32_t)(g_begin - pos0) : 0u;
      const uint32_t hi = g_end - pos0 < 16 ? (uint32_t)(g_end - pos0) : 16u;
      const uint32_t in = (0xFFFFu >> (16 - hi)) & ~((1u << lo) - 1);
      amb16 |= ~in & 0xFFFFu;
      crlf16 &= in;
    }
    const uint32_t code_o = __shfl_xor_sync(0xFFFFFFFFu, code32, 1);
    const uint32_t amb_o = __shfl_xor_sync(0xFFFFFFFFu, amb16, 1);
    const uint32_t crlf_o = __shfl_xor_sync(0xFFFFFFFFu, crlf16, 1);
    if (!(lane & 1) && h < h_end) {
      const uint64_t j = h >> 1;
      PackedBlock b;
      b.codes = ((uint64_t)code32 << 32) | code_o;
      b.amb = amb16 | (amb_o << 16);
      b.start = 0;
      p.pack.blocks[j] = b;
      const uint32_t crlf = crlf16 | (crlf_o << 16);
      p.pack.side[j] = crlf;
      if (crlf) atomicAdd(p.chunk_counter, 1u);
    }
  }
}

// Read-parallel, after k_pack: read start bits (and the one at offsets[n_reads]), window counts, and the reads that
// hold '\n' / '\r': those go through the scanner replay of k_scan (clean_read + scan_read on the cleaned copy), which
// writes their windows to scratch at the text positions the resolve reads them from; all their positions become side.
__global__ void __launch_bounds__(256) k_pack_reads(const __grid_constant__ Params p) {
  const uint32_t lane = threadIdx.x & 31, k = p.db.k;
  const bool any_crlf = *reinterpret_cast<volatile uint32_t *>(p.chunk_counter) != 0;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t r0 = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; r0 <= p.n_reads; r0 += stride) {   // warp-uniform
    const uint32_t r = r0 + lane;
    uint64_t b0 = 0, b1 = 0;
    bool side = false;
    if (r <= p.n_reads) {
      b0 = p.offsets[r];
      atomicOr(&p.pack.blocks[b0 >> 5].start, 1u << (b0 & 31));
      if (r < p.n_reads) {
        b1 = p.offsets[r + 1];
        // '\n' / '\r' inside [b0, b1) (k_pack left only those bits in side; neighbours only add bits of their own reads)
        for (uint64_t j = b0 >> 5; any_crlf && b1 > b0 && j <= (b1 - 1) >> 5 && !side; j++) {
          uint64_t m = p.pack.side[j];
          const uint64_t base = j << 5;
          if (b0 > base) m &= ~0ull << (b0 - base);
          if (b1 < base + 32) m &= (1ull << (b1 - base)) - 1;
          side = m != 0;
        }
        const uint64_t len = b1 - b0;
        if (!side) p.n_windows[r] = len >= k ? (uint32_t)(len - k + 1) : 0u;      // classify.cpp:913-914
      }
    }
    for (uint32_t todo = __ballot_sync(0xFFFFFFFFu, side); todo; todo &= todo - 1) {
      const int src = __ffs(todo) - 1;
      const uint64_t s0 = __shfl_sync(0xFFFFFFFFu, b0, src), s1 = __shfl_sync(0xFFFFFFFFu, b1, src);
      const uint32_t raw_len = (uint32_t)(s1 - s0);
      const uint32_t len = clean_read(p.bases + s0, raw_len, p.clean + s0, k, lane);
      scan_read<false>(p, r0 + src, p.clean + s0, len, raw_len, s0, lane, true);
      for (uint64_t j = (s0 >> 5) + lane; j <= (s1 - 1) >> 5; j += 32) {
        const uint64_t base = j << 5;
        uint64_t m = 0xFFFFFFFFull;
        if (s0 > base) m &= ~0ull << (s0 - base);
        if (s1 < base + 32) m &= (1ull << (s1 - base)) - 1;
        atomicOr(p.pack.side + j, (uint32_t)m);
      }
    }
  }
}

__device__ __forceinline__ PackedBlock load_packed(const PackedBlock *b) {
  const uint4 v = __ldg(reinterpret_cast<const uint4 *>(b));
  PackedBlock r;
  r.codes = ((uint64_t)v.y << 32) | v.x;
  r.amb = v.z;
  r.start = v.w;
  return r;
}

// Window of text position 32j + lane from the packed blocks a = j and b = j + 1 (warp-uniform, see window_bin): its
// bin (BIN_NONE when a read starts inside (g, g + k), i.e. the read ends before the window does) and canonical k-mer.
template <bool FAST>
__device__ __forceinline__ uint32_t packed_window(const DbView &db, const PackedBlock &a, const PackedBlock &b, uint32_t lane,
                                                  uint64_t &canon) {
  const uint32_t k = FAST ? 31u : db.k;
  const uint32_t bin = window_bin<FAST>(db, a.codes, b.codes, ((uint64_t)b.amb << 32) | a.amb, lane, canon);
  const uint64_t starts = ((uint64_t)b.start << 32) | a.start;
  return ((starts >> (lane + 1)) & ((1ull << (k - 1)) - 1)) ? BIN_NONE : bin;
}

// canonical k-mer of the window at text position g of a call whose windows are packed (or of scratch otherwise)
__device__ __forceinline__ uint64_t window_canon(const Params &p, uint64_t g) {
  const uint64_t j = g >> 5;
  const uint32_t l = (uint32_t)g & 31u;
  if (!p.packed || ((p.pack.side[j] >> l) & 1u)) return p.canon[g];
  return canonical_kmer(window_top(p.pack.blocks[j].codes, p.pack.blocks[j + 1].codes, l), p.db.k);
}

// scratch (canon / bins) of the positions [0, n_pos) from the packed blocks; side positions hold their windows already
template <bool FAST>
__global__ void __launch_bounds__(256) k_unpack_windows(const __grid_constant__ Params p, uint64_t n_pos) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < (n_pos + 31) >> 5; j += warps) {
    uint64_t canon;
    const uint32_t bin = packed_window<FAST>(p.db, load_packed(p.pack.blocks + j), load_packed(p.pack.blocks + j + 1), lane, canon);
    const uint64_t g = (j << 5) + lane;
    if (g < n_pos && !((p.pack.side[j] >> lane) & 1u)) {
      p.bins[g] = bin;
      p.canon[g] = canon;
    }
  }
}

void launch_unpack_windows(const Params &p, uint64_t n_pos, int n_sm, cudaStream_t stream) {
  const int grid = (int)max((uint64_t)1, min((uint64_t)n_sm * 8, (n_pos + 255) / 256));
  if (p.db.k == 31 && p.db.nt == 15) k_unpack_windows<true><<<grid, 256, 0, stream>>>(p, n_pos);
  else k_unpack_windows<false><<<grid, 256, 0, stream>>>(p, n_pos);
}

// Stage 2: one thread per text position.  Index fetch (KrakenDBIndex::at, krakendb.cpp:586-593), bin search
// (kmer_query, :280-299: 4-ary narrowing while the bin is large, then a scan of <= 8 records) and — unless the
// lookups belong to one range of a sharded database — the HLL insert of ReadCounts::add_kmer (classify.cpp:939).
// Threads of a warp hold consecutive windows of a read: windows that share a minimizer read the same index
// sector and the same pivots, which the load unit coalesces.
// LEAN = the launch uses none of: probe statistics (flag 8), stored-zero marking (16), shard counting (32), hits-only
// output, peer buffers.  Those are launch-uniform run-time switches; compiled out, the common path of the fused kernel
// is a third shorter.
template <int MODE, bool LEAN>
__device__ __forceinline__ void lookup_window(const Params &p, uint64_t g, uint32_t bin, uint64_t canon) {
  const DbView &db = p.db;
  const uint32_t flags = LEAN ? (p.flags & (4u | F_KEEP)) : p.flags;
  const uint32_t only_hits = LEAN ? 0u : p.only_hits;
  const uint32_t n_peers = LEAN ? 0u : p.n_peers;
  const uint32_t hi_mask = (uint32_t)(db.key_mask >> 32);
  const bool counting = (MODE == MODE_FUSED) && !(flags & 4u);
  const bool keep = counting && (flags & F_KEEP);
  // hits of the fused path reach the sparse tier through the record flag (see below); dense-only / exact runs have
  // no sparse tier
  // flag 32 (database sharded over GPUs, one database): the GPU that FINDS a hit owns its sketch work — register
  // update and record flag happen in the lookup half, and the resolve half (on the GPU that owns the read) only adds
  // the misses (taxon 0).  Valid because every looked-up window is counted exactly once in that layout.
  const bool shard_counting = (flags & 32u) != 0;
  const bool mark_seen = (counting || (MODE == MODE_LOOKUP && shard_counting)) && p.hll_mode <= 1u;
  {
    if (bin == BIN_NONE) return;
    if (bin == BIN_AMBIG) {
      if (!only_hits && !(MODE == MODE_LOOKUP && n_peers)) p.codes_dense[g] = AMBIG;
      return;
    }
    uint32_t taxon = 0, kept_new = 0;
    if (MODE == MODE_RESOLVE) {
      taxon = p.codes_in[g];                                 // merged dense ids of all database ranges
      if (taxon == FOUND_ZERO) taxon = 0;                    // a stored taxon 0 counts like a miss from here on
    } else if (bin >= db.bin_lo && bin < db.bin_hi) {
      const uint64_t *o = db.offsets + (bin - db.bin_lo);
      const uint64_t o0 = __ldg(o), o1 = __ldg(o + 1);
      uint64_t lo = o0 - db.rec_base;
      uint32_t n = (uint32_t)(o1 - o0);
      if (flags & 8u) {   // measurement aid: algorithmic probe count of SURVEY.md §8(d)
        atomicAdd(p.stats, 1ull);
        atomicAdd(p.stats + 1, (unsigned long long)(n ? 32 - __clz(n) : 0));
      }
      while (n > (uint32_t)SEARCH_WINDOW) {
        const uint32_t q = n >> 2;
        const uint64_t k1 = load_key(db.pairs, lo + q, db.key_mask);
        const uint64_t k2 = load_key(db.pairs, lo + 2 * q, db.key_mask);
        const uint64_t k3 = load_key(db.pairs, lo + 3 * q, db.key_mask);
        // pivots <= the key: the quarter that can hold it (branch-free; the lanes of a warp disagree here all the time)
        const uint32_t c = (canon >= k1 ? 1u : 0u) + (canon >= k2 ? 1u : 0u) + (canon >= k3 ? 1u : 0u);
        lo += (uint64_t)c * q;
        n = (c == 3u) ? n - 3 * q : q;
      }
      if (n) {
        // compare the low key words of the window first, confirm the (rare) matches on the high word
        const uint32_t *b = reinterpret_cast<const uint32_t *>(db.pairs + lo * 12);
        const uint32_t clo = (uint32_t)canon, chi = (uint32_t)(canon >> 32);
        uint32_t lw[SEARCH_WINDOW];
#pragma unroll
        for (int t = 0; t < SEARCH_WINDOW; t++) lw[t] = ((uint32_t)t < n) ? __ldg(b + 3 * t) : 0;
        uint32_t m = 0;
#pragma unroll
        for (int t = 0; t < SEARCH_WINDOW; t++) m |= ((uint32_t)t < n && lw[t] == clo) ? (1u << t) : 0u;
        while (m) {
          const int t = __ffs(m) - 1;
          m &= m - 1;
          const uint32_t hiw = __ldg(b + 3 * t + 1);
          if ((hiw & hi_mask) == chi) {
            taxon = __ldg(b + 3 * t + 2);                        // value = dense id
            if (MODE == MODE_LOOKUP && taxon == 0 && (flags & 16u)) taxon = FOUND_ZERO;
            // Sparse HLL tier of a hit (hyperloglogplus.cpp:499-512): the (taxon, encoded hash) pair is a function
            // of the RECORD, so instead of probing a hash set per window the record itself is flagged in the free
            // top bit of its key word — the sector is in L1/L2 already, the flag costs no DRAM read, and only the
            // first sighting of a record issues the atomic.  The harvest turns flagged records into sparse-tier
            // keys once per run; a record whose key is kept already (KEPT_BIT) needs no flag.  A stale
            // (non-coherent) load can only miss a flag another thread just set: the atomicOr is then redundant,
            // never wrong.
            // Keep mode (F_KEEP) skips the flag and the harvest: the record becomes kept here, unless its taxon is dense
            // already (as keep_record decides).  Other windows may sight the record in this step too: only the one whose
            // atomic found KEPT_BIT clear counts it, through its code (k_resolve).
            if (mark_seen && taxon != 0 && taxon != FOUND_ZERO && !(hiw & (SEEN_BIT | KEPT_BIT))) {
              uint32_t *w = const_cast<uint32_t *>(b + 3 * t + 1);
              if (!keep) atomicOr(w, SEEN_BIT);
              else if (!p.dense_flag[taxon] && !(atomicOr(w, KEPT_BIT) & KEPT_BIT)) kept_new = KEEP_NEW;
            }
            m = 0;
          }
        }
      }
    } else if (flags & 8u) {
      atomicAdd(p.stats + 3, 1ull);                          // a window of another range: nothing fetched here
    }
    // only_hits: several DB ranges (GPUs) write their hits into one zero-initialised buffer, possibly over
    // NVLink; a key lives in exactly one range (classify.cpp:447), so no two writers touch the same word.
    if (MODE == MODE_LOOKUP && n_peers) {
      // fused lookup + scatter: the hit goes to the GPU that resolves this read, as a peer store over NVLink
      if (taxon != 0) {
        uint32_t j = 0;
        while (j + 1 < n_peers && g >= p.peer_bounds[j + 1]) j++;
        p.peer_codes[j][g] = taxon;
      }
    } else if (MODE == MODE_RESOLVE || !only_hits || taxon != 0) {
      p.codes_dense[g] = taxon | kept_new;
    }
    if (MODE == MODE_LOOKUP && shard_counting) {
      if (taxon != 0 && taxon != FOUND_ZERO) hll_update(p.regs, p.reg_floor, taxon, fmix64(canon));
    } else if ((counting || (MODE == MODE_RESOLVE && !(flags & 4u))) && !(MODE == MODE_RESOLVE && shard_counting && taxon != 0)) {
      const uint64_t h = fmix64(canon);
      hll_update(p.regs, p.reg_floor, taxon, h);
      // direct set insert: misses (taxon 0 has no record to flag) and the resolve half, which only sees merged ids
      if (p.hll_mode != 2u && !(mark_seen && taxon != 0) && !p.dense_flag[taxon]) {
        const int ins = sparse_insert(p.sparse, taxon, encode_hash32(h));
        if (ins > 0) atomicAdd(p.sparse.distinct + taxon, 1u);
        else if (ins < 0) atomicExch(p.error_flag, 4u);       // set saturated
      }
    }
  }
}

// Several databases (classify -d A -d B, classify.cpp:928-936): the window asks p.dbs[0], p.dbs[1], ... in order and
// the first database that holds the key answers — a stored taxon 0 too, written as FOUND_ZERO so that it also ends the
// search of later launches.  Same bin search as lookup_window (kept apart so that the fused kernels stay as they are).
// only_hits 1 writes hits only; 2 (fill empty) skips a window an earlier launch coded already, before any index fetch.
__device__ __forceinline__ bool search_bin(const DbView &db, uint32_t bin, uint64_t canon, uint32_t &value) {
  const uint64_t *o = db.offsets + (bin - db.bin_lo);
  const uint64_t o0 = __ldg(o), o1 = __ldg(o + 1);
  uint64_t lo = o0 - db.rec_base;
  uint32_t n = (uint32_t)(o1 - o0);
  while (n > (uint32_t)SEARCH_WINDOW) {
    const uint32_t q = n >> 2;
    const uint64_t k1 = load_key(db.pairs, lo + q, db.key_mask);
    const uint64_t k2 = load_key(db.pairs, lo + 2 * q, db.key_mask);
    const uint64_t k3 = load_key(db.pairs, lo + 3 * q, db.key_mask);
    const uint32_t c = (canon >= k1 ? 1u : 0u) + (canon >= k2 ? 1u : 0u) + (canon >= k3 ? 1u : 0u);
    lo += (uint64_t)c * q;
    n = (c == 3u) ? n - 3 * q : q;
  }
  const uint32_t *b = reinterpret_cast<const uint32_t *>(db.pairs + lo * 12);
  const uint32_t clo = (uint32_t)canon, chi = (uint32_t)(canon >> 32), hi_mask = (uint32_t)(db.key_mask >> 32);
  for (uint32_t t = 0; t < n; t++) {
    if (__ldg(b + 3 * t) != clo || (__ldg(b + 3 * t + 1) & hi_mask) != chi) continue;
    value = __ldg(b + 3 * t + 2);
    return true;
  }
  return false;
}

// A word another GPU may have stored over NVLink in an earlier phase: a coherent system-scope load, never the
// non-coherent read-only path.
__device__ __forceinline__ uint32_t load_relaxed_sys(const uint32_t *a) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(a) : "memory");
  return v;
}

__device__ __forceinline__ void lookup_window_multi(const Params &p, uint64_t g, uint32_t bin, uint64_t canon) {
  if (bin == BIN_NONE) return;
  uint32_t *out = p.codes_dense + g;
  if (p.n_peers) {
    // databases sharded by minimizer range: ambiguous windows are the resolving GPU's own business, windows of other
    // GPUs' ranges are skipped before anything is loaded, and the hit goes to the GPU that resolves the read
    if (bin == BIN_AMBIG || bin < p.run_lo || bin >= p.run_hi) return;
    uint32_t j = 0;
    while (j + 1 < p.n_peers && g >= p.peer_bounds[j + 1]) j++;
    out = p.peer_codes[j] + g;
    if (p.only_hits == 2u && load_relaxed_sys(out) != 0) return;     // answered by an earlier run, on any GPU
  } else {
    if (p.only_hits == 2u && *out != 0) return;
    if (bin == BIN_AMBIG) {
      if (!p.only_hits) *out = AMBIG;
      return;
    }
  }
  uint32_t taxon = 0;
#pragma unroll
  for (uint32_t d = 0; d < MAX_DBS; d++) {            // constant indices: the views stay in the parameter bank
    if (d >= p.n_dbs) break;
    const DbView &db = p.dbs[d];
    if (bin < db.bin_lo || bin >= db.bin_hi) continue;
    if (p.flags & 8u) {                                // one fetch per database asked
      const uint64_t *o = db.offsets + (bin - db.bin_lo);
      const uint32_t n = (uint32_t)(__ldg(o + 1) - __ldg(o));
      atomicAdd(p.stats, 1ull);
      atomicAdd(p.stats + 1, (unsigned long long)(n ? 32 - __clz(n) : 0));
    }
    uint32_t v;
    if (search_bin(db, bin, canon, v)) {
      taxon = v ? v : FOUND_ZERO;
      break;
    }
  }
  if (!p.only_hits || taxon != 0) *out = taxon;
}

// MODE_FUSED computes its windows from the packed blocks (FAST: k = 31, m = 15, see window_bin) instead of reading
// 12 bytes of scratch per position: a warp takes 32 consecutive positions (one block) at a time, from a contiguous
// range of blocks, so block j + 1 of one step is block j of the next.  Side positions (reads with '\n' / '\r') read
// their windows from scratch.  The other modes read k_scan's scratch.
// The generic-k fused path needs a few registers more than 32 (6 CTAs per SM, 40 registers, no spills).
// MULTI: MODE_LOOKUP over p.dbs (lookup_window_multi).
template <int MODE, bool LEAN, bool FAST = false, bool MULTI = false>
__global__ void __launch_bounds__(256, (MODE == MODE_FUSED && !FAST) ? 6 : 8) k_lookup(const __grid_constant__ Params p) {
  // only the text of this call's reads (the scratch beyond it may hold windows of an earlier call on the slot)
  const uint64_t g_begin = p.offsets[0], g_end = p.offsets[p.n_reads];
  if constexpr (MODE == MODE_FUSED) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t j_begin = g_begin >> 5, n_blk = ((g_end + 31) >> 5) - j_begin;
    const uint64_t per = (n_blk + warps - 1) / warps;
    uint64_t j = j_begin + warp * per;
    const uint64_t j_end = min(j + per, j_begin + n_blk);
    if (j >= j_end) return;
    PackedBlock a = load_packed(p.pack.blocks + j), b = load_packed(p.pack.blocks + j + 1);
    for (; j < j_end; j++) {
      const PackedBlock c = load_packed(p.pack.blocks + j + 2);
      const uint32_t side = p.pack.side[j];
      const uint64_t g = (j << 5) + lane;
      uint64_t canon;
      uint32_t bin = packed_window<FAST>(p.db, a, b, lane, canon);
      if ((side >> lane) & 1u) { bin = p.bins[g]; canon = p.canon[g]; }
      if (g < g_begin || g >= g_end) bin = BIN_NONE;
      lookup_window<MODE, LEAN>(p, g, bin, canon);
      a = b;
      b = c;
    }
  } else {
    // the scratch of the NEXT position of this thread is fetched while the current window is searched: the grid-stride
    // loop would otherwise start every window with an exposed (streaming, but still ~1 us) load
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    uint64_t g = g_begin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t bin_n = g < g_end ? __ldg(p.bins + g) : BIN_NONE;
    uint64_t canon_n = g < g_end ? __ldg(p.canon + g) : 0ull;
    for (; g < g_end; g += stride) {
      const uint32_t bin = bin_n;
      const uint64_t canon = canon_n;
      if (g + stride < g_end) { bin_n = __ldg(p.bins + g + stride); canon_n = __ldg(p.canon + g + stride); }
      if constexpr (MULTI) lookup_window_multi(p, g, bin, canon);
      else lookup_window<MODE, LEAN>(p, g, bin, canon);
    }
  }
}

// ---- per-batch (unit, taxon) map ----------------------------------------------------------------------------
// Linear probing gives up after UMAP_PROBES slots (error 2, KUQ_E_CAPACITY).  classify's batches hold at most the
// dense table's rows of units, so the map holds only candidates (< 300 k pairs, under 15 % load) and a run that long
// does not occur; a map that a C ABI caller overfills fails in microseconds, not in a scan of all 2 Mi slots per insert.
constexpr uint32_t UMAP_PROBES = 4096;
__device__ __forceinline__ uint32_t umap_slot(const UnitMap &u, uint32_t unit, uint32_t taxon, bool insert) {
  const unsigned long long key = ((unsigned long long)(unit + 1) << 32) | taxon;
  uint32_t slot = (uint32_t)mix64(key) & u.mask;
  for (uint32_t probe = 0; probe < UMAP_PROBES; probe++) {
    unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(u.keys + slot);
    if (cur == key) return slot;
    if (cur == 0) {
      if (!insert) return 0xFFFFFFFFu;
      unsigned long long prev = atomicCAS(u.keys + slot, 0ull, key);
      if (prev == 0 || prev == key) return slot;
    }
    slot = (slot + 1) & u.mask;
  }
  return 0xFFFFFFFFu;
}

// Reads that hit more than 32 distinct taxa (long reads, contigs): the hit list moves to a hash table in HBM taken from
// a per-batch pool ({taxon+1 << 32 | count, score} per entry).  Same arithmetic as the register path, just slower.
struct OverflowPool {
  unsigned long long *mem;        // 2 words per entry
  unsigned long long *cursor;     // entries handed out
  uint64_t capacity;              // entries
};

// FILTER: *tab_out / *cap_out = the read's table (nullptr when the pool is exhausted), which the filter walks next
template <bool FILTER = false>
__device__ uint32_t resolve_overflow(const Params &p, const OverflowPool &pool, const uint32_t *codes_src, uint64_t out_base,
                                     uint32_t nwin, uint32_t unit, bool counting, bool units, uint32_t lane,
                                     unsigned long long **tab_out = nullptr, uint32_t *cap_out = nullptr) {
  // capacity: next power of two >= 2 * (upper bound of distinct taxa); distinct taxa <= windows
  // (and <= taxa that own a sketch: only database values can be hits)
  const uint32_t most = min(nwin, p.tax.n_sketch);
  uint32_t cap = 64;
  while (cap < 2 * most) cap <<= 1;
  unsigned long long start = 0;
  if (lane == 0) start = atomicAdd(pool.cursor, (unsigned long long)cap);
  start = __shfl_sync(0xFFFFFFFFu, start, 0);
  if (start + cap > pool.capacity) {
    if (lane == 0) atomicExch(p.error_flag, 1u);
    return 0;
  }
  unsigned long long *tab = pool.mem + 2 * start;
  if constexpr (FILTER) { *tab_out = tab; *cap_out = cap; }
  for (uint32_t i = lane; i < cap; i += 32) { tab[2 * i] = 0; tab[2 * i + 1] = 0; }
  __syncwarp();
  auto find = [&](uint32_t t) -> int {              // slot of taxon t or -1
    uint32_t s = (uint32_t)mix64(t) & (cap - 1);
    for (uint32_t probe = 0; probe < cap; probe++) {
      const unsigned long long e = *reinterpret_cast<volatile unsigned long long *>(tab + 2 * s);
      if (e == 0) return -1;
      if ((uint32_t)(e >> 32) == t + 1) return (int)s;
      s = (s + 1) & (cap - 1);
    }
    return -1;
  };
  // hit_counts[taxon]++ over all windows
  for (uint32_t i = lane; i < nwin; i += 32) {
    uint32_t t = codes_src[out_base + i];
    if (t == AMBIG || t == 0) continue;
    if (t & KEEP_NEW) {                               // rare path: the record's new distinct code is booked right here
      t &= ~KEEP_NEW;
      if (counting) atomicAdd(p.sparse.distinct + t, 1u);
    }
    uint32_t s = (uint32_t)mix64(t) & (cap - 1);
    for (;;) {
      unsigned long long e = *reinterpret_cast<volatile unsigned long long *>(tab + 2 * s);
      if (e == 0) {
        e = atomicCAS(tab + 2 * s, 0ull, ((unsigned long long)(t + 1) << 32) | 1ull);
        if (e == 0) break;
      }
      if ((uint32_t)(e >> 32) == t + 1) { atomicAdd(tab + 2 * s, 1ull); break; }
      s = (s + 1) & (cap - 1);
    }
  }
  __syncwarp();
  // score(t) = sum of hit counts along t's root path (krakenutil.cpp:156-177)
  uint32_t best = 0;
  for (uint32_t s = lane; s < cap; s += 32) {
    const unsigned long long e = tab[2 * s];
    if (!e) continue;
    const uint32_t t = (uint32_t)(e >> 32) - 1, c = (uint32_t)e;
    if (counting) {
      atomicAdd(p.n_kmers + t, (unsigned long long)c);
      if (units) {
        const uint32_t row = unit - p.unit_id[0];
        if (row < p.units.direct_rows) {
          atomicAdd(p.units.direct + (size_t)row * p.tax.n_sketch + t, c);
        } else {
          uint32_t sl = umap_slot(p.units, unit, t, true);
          if (sl == 0xFFFFFFFFu) atomicExch(p.error_flag, 2u);
          else atomicAdd(p.units.inserts + sl, c);
        }
      }
    }
    uint32_t score = 0;
    for (uint32_t node = t; node; node = __ldg(p.tax.parent + node)) {
      int q = find(node);
      if (q >= 0) score += (uint32_t)tab[2 * q];
    }
    tab[2 * s + 1] = score;
    best = max(best, score);
  }
  best = __reduce_max_sync(0xFFFFFFFFu, best);
  __syncwarp();
  if (best == 0) return 0;
  // ties → LCA of all tied taxa, folded in ascending taxid order (std::set iteration, krakenutil.cpp:190-196)
  uint32_t acc = 0;
  unsigned long long last = 0;          // raw taxid + 1 of the last folded taxon
  for (;;) {
    unsigned long long mn = ~0ull;      // smallest (raw+1) << 32 | dense among the tied entries above `last`
    for (uint32_t s = lane; s < cap; s += 32) {
      const unsigned long long e = tab[2 * s];
      if (!e || (uint32_t)tab[2 * s + 1] != best) continue;
      const uint32_t t = (uint32_t)(e >> 32) - 1;
      const unsigned long long r1 = (unsigned long long)__ldg(p.tax.raw + t) + 1;
      if (r1 > last) mn = min(mn, (r1 << 32) | t);
    }
    for (int o = 16; o; o >>= 1) mn = min(mn, __shfl_xor_sync(0xFFFFFFFFu, mn, o));
    if (mn == ~0ull) break;
    const uint32_t t = (uint32_t)mn;
    acc = acc ? lca_dense(p.tax, acc, t) : t;
    last = mn >> 32;
  }
  return acc;
}

// ---- confidence filter (krakenuniq-filter, scripts/krakenuniq-filter:88-133) ----------------------------------
// The deepest node that the F-chains of filter ids a and b (F-depths da, db) share, as its F-depth + 1; 0 = none.
__device__ __forceinline__ uint32_t f_common(const Params &p, uint32_t a, uint32_t da, uint32_t b, uint32_t db) {
  for (; da > db; da--) a = __ldg(p.fparent + a);
  for (; db > da; db--) b = __ldg(p.fparent + b);
  for (; a != b; da--) {
    if (!da) return 0;
    a = __ldg(p.fparent + a);
    b = __ldg(p.fparent + b);
  }
  return da + 1;
}

// Read r's filtered call, warp-collective.  The hit taxa are lane j's (my_t, my_c) for j < n_hits plus the entries of
// the overflow table tab (cap slots; nullptr = none); `total` starts as the misses (QUICK: the "Q:<hits>" value, with
// no taxa at all).  hit_sums[a] of a node a on the call's F-chain is the sum of the counts of the hit taxa whose chain
// shares a node with the call's at a's depth or above: their common node, found once per taxon, decides every step.
template <bool QUICK>
__device__ void filter_read(const Params &p, uint32_t r, uint32_t call, uint32_t lane, uint32_t my_t, uint32_t my_c,
                            uint32_t n_hits, uint32_t total, unsigned long long *tab, uint32_t cap) {
  const uint32_t dc = __ldg(p.fdepth + call);
  uint32_t mine = 0;                                            // lane's register entry: common depth + 1
  if (!QUICK) {
    uint32_t sum = lane < n_hits ? my_c : 0;
    if (dc && lane < n_hits) mine = f_common(p, my_t, __ldg(p.fdepth + my_t), call, dc);
    if (tab) {
      for (uint32_t s = lane; s < cap; s += 32) {
        const unsigned long long e = tab[2 * s];
        if (!e) continue;
        const uint32_t t = (uint32_t)(e >> 32) - 1;
        sum += (uint32_t)e;
        if (dc) tab[2 * s + 1] = f_common(p, t, __ldg(p.fdepth + t), call, dc);   // the score is no longer needed
      }
    }
    total += __reduce_add_sync(0xFFFFFFFFu, sum);
  }
  uint32_t node = call, hits = 0, den = 0;
  for (uint32_t d = dc; d; d--) {                               // while F[node] is defined
    uint32_t h = 0;
    if (!QUICK) {
      h = mine > d ? my_c : 0;
      if (tab)
        for (uint32_t s = lane; s < cap; s += 32) {
          const unsigned long long e = tab[2 * s];
          if (e && (uint32_t)tab[2 * s + 1] > d) h += (uint32_t)e;
        }
      h = __reduce_add_sync(0xFFFFFFFFu, h);
    }
    hits = h;
    den = total;
    if ((double)h / (double)total >= p.fmin) break;
    node = __ldg(p.fparent + node);
  }
  if (lane == 0) {
    p.fcall[r] = node < p.tax.n_taxa ? __ldg(p.tax.raw + node) : __ldg(p.fextra + node - p.tax.n_taxa);
    p.fhits[r] = hits;
    p.ftotal[r] = den;
  }
}

// Stage 3: one warp per read.  hit_counts (classify.cpp:941-942), resolve_tree / lca (krakenutil.cpp:90-118,
// 149-200), the per-taxon counters (classify.cpp:939,968) and the run-length encoded hit list (:826-861).
constexpr int RUN_BUF = 96;      // runs buffered per warp before they are flushed to global memory
constexpr uint32_t RUN_BLOCK = 256;   // run slots a warp takes from the global cursor at a time

// QUICK (classify -q): no resolve_tree; hits = min(#hits, quick_min) goes to run_count[] ("Q:hits", :989-990) and the
// call is the taxon of the last unambiguous window once quick_min hits were seen (:963-964 after k_quick_cut ended
// the read at that hit; :705-721,737-738 on the -x path, where the last window of the whole read decides).
// FILTER: also the confidence filter of every read (filter_read), a separate instantiation so that runs without one
// execute the kernels they always did.
template <bool QUICK, bool FILTER = false>
__global__ void __launch_bounds__(256, 4) k_resolve(const __grid_constant__ Params p) {
  __shared__ uint2 s_runs[CTA_WARPS][RUN_BUF];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t warps_total = gridDim.x * CTA_WARPS;
  const bool counting = !(p.flags & 4u);
  const bool want_runs = !(p.flags & 2u);
  const uint32_t *codes_src = p.codes_dense;
  // Same-address atomics serialise in L2 (about one per few cycles): a million reads per batch must not each hit
  // the run cursor, n_kmers[0] and n_reads[0].  Each warp therefore allocates run slots in blocks of RUN_BLOCK
  // and keeps the hot counters in registers until it is done.
  uint32_t blk_next = 0, blk_end = 0;                           // this warp's block of run slots
  uint32_t acc_miss = 0, acc_unclassified = 0, acc_classified = 0, acc_kept = 0;
  uint32_t unit_cur = 0xFFFFFFFFu, unit_miss = 0;               // misses of the current work unit, not yet booked
  const bool units = counting && p.hll_mode == 0u && p.unit_id;
  const uint32_t unit_row0 = units ? p.unit_id[0] : 0u;
  auto book_unit = [&](uint32_t unit, uint32_t taxon, uint32_t cnt) {          // N(unit, taxon) += cnt
    const uint32_t row = unit - unit_row0;
    if (row < p.units.direct_rows) {
      atomicAdd(p.units.direct + (size_t)row * p.tax.n_sketch + taxon, cnt);
    } else {
      const uint32_t sl = umap_slot(p.units, unit, taxon, true);
      if (sl == 0xFFFFFFFFu) atomicExch(p.error_flag, 2u);
      else atomicAdd(p.units.inserts + sl, cnt);
    }
  };
  auto flush_unit = [&]() {
    if (lane == 0 && unit_miss) book_unit(unit_cur, 0, unit_miss);
    unit_miss = 0;
  };
  // each warp takes a contiguous range of reads: consecutive reads share their work unit and their run block
  const uint32_t per_warp = (p.n_reads + warps_total - 1) / warps_total;
  const uint32_t r_begin = (blockIdx.x * CTA_WARPS + warp) * per_warp;
  const uint32_t r_end = min(r_begin + per_warp, p.n_reads);
  // A warp works through its reads one after the other and every read is a chain of dependent loads (offset →
  // codes → taxonomy → counters), so the kernel is latency bound (round 1: 36 % warps active, 6 % DRAM).  The loads
  // that do not depend on the read's outcome are therefore issued one read ahead: while read r is resolved, the
  // codes of read r+1 (first PRE_SLOTS x 32 windows) and the offset / window count / unit of read r+2 are in flight.
  constexpr int PRE_SLOTS = 4;
  const bool want_codes = (p.flags & 1u) != 0;
  uint64_t base_a = 0, base_b = 0;                              // read r, read r+1
  uint32_t nwin_a = 0, nwin_b = 0, unit_a = 0, unit_b = 0;
  uint32_t pre[PRE_SLOTS];
#pragma unroll
  for (int j = 0; j < PRE_SLOTS; j++) pre[j] = 0;
  if (r_begin < r_end) {
    base_a = p.offsets[r_begin]; nwin_a = p.n_windows[r_begin];
    if (units) unit_a = p.unit_id[r_begin];
#pragma unroll
    for (int j = 0; j < PRE_SLOTS; j++) { const uint32_t i = j * 32 + lane; pre[j] = i < nwin_a ? codes_src[base_a + i] : 0u; }
  }
  if (r_begin + 1 < r_end) {
    base_b = p.offsets[r_begin + 1]; nwin_b = p.n_windows[r_begin + 1];
    if (units) unit_b = p.unit_id[r_begin + 1];
  }
  for (uint32_t r = r_begin; r < r_end; r++) {
    const uint64_t out_base = base_a;
    const uint32_t nwin = nwin_a;
    const uint32_t unit = unit_a;
    uint32_t cur[PRE_SLOTS];
#pragma unroll
    for (int j = 0; j < PRE_SLOTS; j++) cur[j] = pre[j];
    base_a = base_b; nwin_a = nwin_b; unit_a = unit_b;
    if (r + 1 < r_end) {
#pragma unroll
      for (int j = 0; j < PRE_SLOTS; j++) { const uint32_t i = j * 32 + lane; pre[j] = i < nwin_a ? codes_src[base_a + i] : 0u; }
    }
    if (r + 2 < r_end) {
      base_b = p.offsets[r + 2]; nwin_b = p.n_windows[r + 2];
      if (units) unit_b = p.unit_id[r + 2];
    }
    uint32_t my_t = 0, my_c = 0;                                // hit list: lane j holds entry j (dense id, count)
    uint32_t my_k = 0;                                          // F_KEEP: windows of entry j that made their record kept
    uint32_t n_hits = 0, n_miss = 0, n_runs = 0;
    uint32_t carry_code = 0;
    bool overflow = false;
    uint32_t q_hits = 0, q_last = 0;                            // QUICK: hits seen, taxon of the last unambiguous window
    const uint32_t nslots = (nwin + 31) / 32;
    // one slot of 32 windows; c = dense id of the lane's window, 0 = miss, AMBIG.  Runs of the hit list break where
    // the DENSE code changes (dense id <-> taxid is one to one); taxids are looked up per run when the list is flushed
    auto do_slot = [&](uint32_t s, uint32_t c) {
      const uint32_t i = s * 32 + lane;
      const bool valid = i < nwin;
      const bool amb = valid && c == AMBIG;
      const bool look = valid && !amb;
      const uint32_t taxon = look ? c & ~KEEP_NEW : 0;
      const uint32_t kept_m = __ballot_sync(0xFFFFFFFFu, look && (c & KEEP_NEW));
      acc_kept += __popc(kept_m);
      const uint32_t out_code = amb ? AMBIG : taxon;
      if (want_codes && valid) p.codes[out_base + i] = amb ? AMBIG : (taxon ? __ldg(p.tax.raw + taxon) : 0u);
      // runs of the hit list
      uint32_t prev = __shfl_up_sync(0xFFFFFFFFu, out_code, 1);
      if (lane == 0) prev = carry_code;
      const bool brk = valid && (i == 0 || out_code != prev);
      const uint32_t bm = __ballot_sync(0xFFFFFFFFu, brk);
      if (want_runs && brk) {
        const uint32_t idx = n_runs + __popc(bm & ((1u << lane) - 1));
        if (idx < RUN_BUF) s_runs[warp][idx] = make_uint2(out_code, i);   // (dense code, start); lengths at flush
      }
      n_runs += __popc(bm);
      carry_code = __shfl_sync(0xFFFFFFFFu, out_code, 31);
      // hit_counts[taxon]++, aggregated per distinct taxon of the slot
      n_miss += __popc(__ballot_sync(0xFFFFFFFFu, look && taxon == 0));
      uint32_t rem = __ballot_sync(0xFFFFFFFFu, look && taxon != 0);
      if (QUICK) {
        q_hits += __popc(rem);
        const uint32_t lm = __ballot_sync(0xFFFFFFFFu, look);
        if (lm) q_last = __shfl_sync(0xFFFFFFFFu, taxon, 31 - __clz(lm));
      }
      while (rem) {
        const int ldr = __ffs(rem) - 1;
        const uint32_t t = __shfl_sync(0xFFFFFFFFu, taxon, ldr);
        const uint32_t same = __ballot_sync(0xFFFFFFFFu, look && taxon == t) & rem;
        const uint32_t cnt = __popc(same), kcnt = __popc(same & kept_m);
        rem &= ~same;
        const uint32_t pos = __ballot_sync(0xFFFFFFFFu, lane < n_hits && my_t == t);
        if (pos) {
          if (lane == (uint32_t)(__ffs(pos) - 1)) { my_c += cnt; my_k += kcnt; }
        } else if (n_hits < 32) {
          if (lane == n_hits) { my_t = t; my_c = cnt; my_k = kcnt; }
          n_hits++;
        } else {
          overflow = true;
        }
      }
    };
#pragma unroll
    for (int j = 0; j < PRE_SLOTS; j++)
      if ((uint32_t)j < nslots) do_slot((uint32_t)j, cur[j]);
    for (uint32_t s = PRE_SLOTS; s < nslots; s++) {
      const uint32_t i = s * 32 + lane;
      do_slot(s, i < nwin ? codes_src[out_base + i] : 0u);
    }

    // ---- resolve_tree (krakenutil.cpp:149-200) ------------------------------------------------------------
    uint32_t call = 0;
    unsigned long long *ovf_tab = nullptr;                      // FILTER: the overflow table of the read
    uint32_t ovf_cap = 0;
    if (overflow) {
      OverflowPool pool{p.ovf_mem, p.ovf_cursor, p.ovf_capacity};
      if constexpr (FILTER) call = resolve_overflow<true>(p, pool, codes_src, out_base, nwin, unit, counting, units, lane, &ovf_tab, &ovf_cap);
      else call = resolve_overflow(p, pool, codes_src, out_base, nwin, unit, counting, units, lane);
      n_hits = 0;                                               // counters were booked from the table
    } else if (!QUICK && n_hits == 1) {
      call = __shfl_sync(0xFFFFFFFFu, my_t, 0);                 // a single hit taxon is its own best path
    } else if (!QUICK && n_hits > 1) {
      // score(t) = sum of hit counts along t's root path (:156-177); lane j walks entry j
      uint32_t node = lane < n_hits ? my_t : 0;
      uint32_t score = 0;
      while (__any_sync(0xFFFFFFFFu, node != 0)) {
        for (uint32_t q = 0; q < n_hits; q++) {
          uint32_t tq = __shfl_sync(0xFFFFFFFFu, my_t, q);
          uint32_t cq = __shfl_sync(0xFFFFFFFFu, my_c, q);
          if (node == tq) score += cq;
        }
        if (node) node = __ldg(p.tax.parent + node);
      }
      uint32_t best = __reduce_max_sync(0xFFFFFFFFu, score);
      uint32_t tied = __ballot_sync(0xFFFFFFFFu, lane < n_hits && score == best);
      if (__popc(tied) == 1) {
        call = __shfl_sync(0xFFFFFFFFu, my_t, __ffs(tied) - 1);
      } else {
        // ties → LCA of all tied taxa, folded in ascending taxid order (std::set iteration, :190-196)
        uint32_t raw = (tied >> lane) & 1 ? __ldg(p.tax.raw + my_t) : 0xFFFFFFFFu;
        uint32_t acc = 0;
        uint32_t left = tied;
        while (left) {
          uint32_t cand = (left >> lane) & 1 ? raw : 0xFFFFFFFFu;
          uint32_t mn = __reduce_min_sync(0xFFFFFFFFu, cand);
          uint32_t who = __ballot_sync(0xFFFFFFFFu, cand == mn && ((left >> lane) & 1));
          int src = __ffs(who) - 1;
          uint32_t t = __shfl_sync(0xFFFFFFFFu, my_t, src);
          acc = acc ? lca_dense(p.tax, acc, t) : t;             // all lanes compute the same walk
          left &= ~(1u << src);
        }
        call = acc;
      }
    }
    if (QUICK) {
      const uint32_t hits = min(q_hits, p.quick_min);
      call = hits >= p.quick_min ? q_last : 0;
      if (lane == 0) p.run_count[r] = hits;
    }
    const uint32_t call_raw = call ? __ldg(p.tax.raw + call) : 0;
    if (lane == 0) p.call[r] = call_raw;
    if constexpr (FILTER)
      filter_read<QUICK>(p, r, call, lane, my_t, my_c, n_hits, QUICK ? min(q_hits, p.quick_min) : n_miss, ovf_tab, ovf_cap);
    // ---- counters: n_kmers per hit taxon (+ misses on taxon 0), n_reads of the call (classify.cpp:939,968) ---
    if (units) {
      // inserts per (work unit, taxon): the necessary condition for a per-unit sketch to convert
      if (unit != unit_cur) { flush_unit(); unit_cur = unit; }
      unit_miss += n_miss;
      if (lane < n_hits) book_unit(unit, my_t, my_c);
    }
    if (counting) {
      if (lane < n_hits) {
        atomicAdd(p.n_kmers + my_t, (unsigned long long)my_c);
        if (my_k) atomicAdd(p.sparse.distinct + my_t, my_k);
      }
      acc_miss += n_miss;
      if (call) {
        acc_classified++;
        if (lane == 0) atomicAdd(p.n_reads_ctr + call, 1ull);
      } else {
        acc_unclassified++;
      }
    }
    // ---- run-length encoded hit list ----------------------------------------------------------------------
    if (want_runs) {
      uint32_t start = 0;
      if (lane == 0) {
        if (n_runs > blk_end - blk_next) {                      // take a fresh block (the old tail stays a hole)
          const uint32_t take = n_runs > RUN_BLOCK ? n_runs : RUN_BLOCK;
          const unsigned long long got = atomicAdd(p.run_cursor, (unsigned long long)take);
          if (got + take > p.runs_capacity) {                   // run buffer exhausted: report, write nothing more
            atomicExch(p.error_flag, 5u);
            blk_next = blk_end = 0xFFFFFFFFu;
          } else {
            blk_next = (uint32_t)got;
            blk_end = blk_next + take;
          }
        }
        start = blk_next;
        if (blk_next != 0xFFFFFFFFu) blk_next += n_runs;
        p.run_start[r] = start;
        p.run_count[r] = n_runs;
      }
      start = __shfl_sync(0xFFFFFFFFu, start, 0);
      __syncwarp();
      if (start == 0xFFFFFFFFu) {
        // no room (KUQ_E_CAPACITY on the host side)
      } else if (n_runs <= RUN_BUF) {
        for (uint32_t j = lane; j < n_runs; j += 32) {
          const uint2 a = s_runs[warp][j];
          const uint32_t end = j + 1 < n_runs ? s_runs[warp][j + 1].y : nwin;
          const uint32_t code = (a.x == AMBIG || a.x == 0) ? a.x : __ldg(p.tax.raw + a.x);
          p.runs[start + j] = make_uint2(code, end - a.y);
        }
      } else {
        // long hit list (long read): recompute from the codes, walking the slots backwards so that each run
        // knows where the next one starts
        uint32_t next_start = nwin, later = 0;
        for (int s = (int)nslots - 1; s >= 0; s--) {
          uint32_t i = (uint32_t)s * 32 + lane;
          bool valid = i < nwin;
          auto code_at = [&](uint32_t w) {
            uint32_t c = codes_src[out_base + w];
            if (c != AMBIG) c &= ~KEEP_NEW;
            return c == AMBIG ? AMBIG : (c ? __ldg(p.tax.raw + c) : 0u);
          };
          uint32_t c = valid ? code_at(i) : 0;
          uint32_t prev = __shfl_up_sync(0xFFFFFFFFu, c, 1);
          if (lane == 0) prev = (s > 0) ? code_at(i - 1) : 0;
          bool brk = valid && (i == 0 || c != prev);
          uint32_t bm = __ballot_sync(0xFFFFFFFFu, brk);
          if (brk) {
            uint32_t after = lane == 31 ? 0u : (bm >> (lane + 1));
            uint32_t end = after ? (uint32_t)s * 32 + lane + (uint32_t)__ffs(after) : next_start;
            uint32_t idx = n_runs - later - (uint32_t)__popc(bm >> lane);
            p.runs[start + idx] = make_uint2(c, end - i);
          }
          if (bm) next_start = (uint32_t)s * 32 + (uint32_t)__ffs(bm) - 1;
          later += __popc(bm);
        }
      }
      __syncwarp();
    }
  }
  if (units) flush_unit();
  if (counting && lane == 0) {
    if (acc_miss) atomicAdd(p.n_kmers, (unsigned long long)acc_miss);
    if (acc_unclassified) atomicAdd(p.n_reads_ctr, (unsigned long long)acc_unclassified);
    if (acc_classified) atomicAdd(p.n_classified, (unsigned long long)acc_classified);
    if (acc_kept) atomicAdd(p.n_new_kept, (unsigned long long)acc_kept);
  }
}

// ---- HLL mode rule (SURVEY.md App. C) ------------------------------------------------------------------------
__global__ void k_unit_mark(const __grid_constant__ Params p) {
  const UnitMap &u = p.units;
  // dense table first: a pair with >= 1025 inserts moves to the hash map, where the candidate bookkeeping lives
  if (u.direct_rows) {
    const uint32_t row0 = p.unit_id[0];
    const uint64_t n = (uint64_t)u.direct_rows * p.tax.n_sketch;
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) {
      const uint32_t cnt = u.direct[e];
      if (cnt < 1025u) continue;
      const uint32_t taxon = (uint32_t)(e % p.tax.n_sketch), row = (uint32_t)(e / p.tax.n_sketch);
      if (p.dense_flag[taxon]) continue;
      const uint32_t sl = umap_slot(u, row0 + row, taxon, true);
      if (sl == 0xFFFFFFFFu) { atomicExch(p.error_flag, 2u); continue; }
      u.inserts[sl] = cnt;
      u.cand[atomicAdd(u.n_cand, 1u)] = sl;
    }
  }
  // the map's own pairs: units past the table (the pairs moved above are in rows < direct_rows and listed already)
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s <= u.mask; s += gridDim.x * blockDim.x) {
    const unsigned long long key = u.keys[s];
    if (!key) continue;
    const uint32_t taxon = (uint32_t)key;
    if ((uint32_t)(key >> 32) - 1u - p.unit_id[0] < u.direct_rows) continue;
    if (u.inserts[s] >= 1025u && !p.dense_flag[taxon]) u.cand[atomicAdd(u.n_cand, 1u)] = s;
  }
  // k_unit_decide finds a unit's reads by binary search, which needs ascending unit ids (classify's always are)
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r + 1 < p.n_reads; r += gridDim.x * blockDim.x)
    if (p.unit_id[r] > p.unit_id[r + 1]) { u.n_cand[1] = 1; break; }
}

// first index in [0, n) whose value is >= v, n if none; a[] ascending.  All lanes of the warp return it.
__device__ uint32_t warp_lower_bound(const uint32_t *a, uint32_t n, uint32_t v, uint32_t lane) {
  uint32_t lo = 0, hi = n;                              // the answer lies in [lo, hi]
  while (hi - lo > 32) {
    const uint32_t step = (hi - lo) / 32;
    const uint32_t below = __popc(__ballot_sync(0xFFFFFFFFu, a[lo + lane * step] < v));
    if (below == 0) return lo;
    if (below < 32) hi = lo + below * step;
    lo += (below - 1) * step + 1;
  }
  const uint32_t i = lo + lane;
  return lo + __popc(__ballot_sync(0xFFFFFFFFu, i < hi && a[i] < v));
}

// One block per candidate (unit, taxon) pair at a time: the distinct codes of the pair's inserts go to the block's own
// table of UNIT_CODES slots (u.codes, in L2).  Counting stops at 1025 codes; with 256 threads inserting at once the
// table then holds at most 1024 + 256 codes, so it never fills and no batch, however many candidates it has, runs out
// of room.  (The table is not in shared memory: this launch runs next to other slots' lookups in every preloaded batch,
// candidates or not, and should not take shared memory from them.)
// A (unit, taxon) sketch receiving inserts x_1..x_N converts iff D >= 1025, or D == 1024 and the 1024th distinct
// code arrives before the last insert (SURVEY.md §7.3): i.e. the last insert repeats a code seen earlier.
__global__ void __launch_bounds__(256) k_unit_decide(const __grid_constant__ Params p) {
  const UnitMap &u = p.units;
  const uint32_t n_cand = *reinterpret_cast<volatile uint32_t *>(u.n_cand);
  if (blockIdx.x >= n_cand) return;
  uint32_t *s_code = u.codes + (size_t)blockIdx.x * 2 * UNIT_CODES, *s_count = s_code + UNIT_CODES;
  __shared__ uint32_t s_distinct, s_lo, s_hi;
  __shared__ unsigned long long s_last;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const bool ascending = u.n_cand[1] == 0;
  volatile uint32_t *v_distinct = &s_distinct;
  const volatile uint8_t *v_dense = p.dense_flag;
  for (uint32_t c = blockIdx.x; c < n_cand; c += gridDim.x) {
    const uint32_t sl = u.cand[c];
    const unsigned long long key = u.keys[sl];
    const uint32_t unit = (uint32_t)(key >> 32) - 1u, taxon = (uint32_t)key;
    for (uint32_t j = threadIdx.x; j < UNIT_CODES; j += blockDim.x) { s_code[j] = 0; s_count[j] = 0; }
    if (warp == 0) {
      uint32_t lo = 0, hi = p.n_reads;
      if (ascending) {
        lo = warp_lower_bound(p.unit_id, p.n_reads, unit, lane);
        hi = unit == 0xFFFFFFFFu ? p.n_reads : warp_lower_bound(p.unit_id, p.n_reads, unit + 1, lane);
      }
      if (lane == 0) { s_lo = lo; s_hi = hi; s_distinct = 0; s_last = 0; }
    }
    __syncthreads();
    const uint32_t lo = s_lo, hi = s_hi;
    for (uint32_t r = lo + warp; r < hi; r += n_warps) {
      if (*v_distinct >= 1025u || v_dense[taxon]) break;            // decided (here, or by another pair of the taxon)
      if (!ascending && p.unit_id[r] != unit) continue;
      const uint64_t base = p.offsets[r];
      const uint32_t nwin = p.n_windows[r];
      for (uint32_t i = lane; i < nwin; i += 32) {
        if ((p.codes_dense[base + i] & ~KEEP_NEW) != taxon) continue;     // AMBIG & ~KEEP_NEW is no dense id
        atomicMax(&s_last, ((unsigned long long)r << 32) | i);
        if (*v_distinct >= 1025u) continue;
        const uint32_t code = encode_hash32(fmix64(window_canon(p, base + i)));     // never 0
        uint32_t q = (code * 0x9E3779B1u) >> 21;
        for (uint32_t probe = 0; probe < UNIT_CODES; probe++) {
          uint32_t cur = reinterpret_cast<volatile uint32_t *>(s_code)[q];   // (L1 bypassed: other threads CAS here)
          if (cur == 0) {
            cur = atomicCAS(s_code + q, 0u, code);
            if (cur == 0) { atomicAdd(&s_distinct, 1u); cur = code; }
          }
          if (cur == code) { atomicAdd(s_count + q, 1u); break; }
          q = (q + 1) & (UNIT_CODES - 1);
        }
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const uint32_t d = s_distinct;
      bool conv = d >= 1025u;
      if (!conv && d == 1024u) {
        const uint32_t r = (uint32_t)(s_last >> 32), i = (uint32_t)s_last;
        const uint32_t code = encode_hash32(fmix64(window_canon(p, p.offsets[r] + i)));
        uint32_t q = (code * 0x9E3779B1u) >> 21;
        const volatile uint32_t *v_code = s_code, *v_count = s_count;
        for (uint32_t probe = 0; probe < UNIT_CODES && v_code[q]; probe++) {
          if (v_code[q] == code) { conv = v_count[q] >= 2u; break; }
          q = (q + 1) & (UNIT_CODES - 1);
        }
      }
      if (conv) p.dense_flag[taxon] = 1;
    }
    __syncthreads();
  }
}

// one launch instead of several memsets: empty the per-batch (unit, taxon) map and its dense table
__global__ void __launch_bounds__(256) k_unit_clear(UnitMap u, uint32_t n_sketch) {
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (uint64_t)gridDim.x * blockDim.x;
  const uint4 z = make_uint4(0, 0, 0, 0);
  const uint64_t cap = (uint64_t)u.mask + 1;     // a power of two >= 1024
  for (uint64_t i = tid; i < cap / 2; i += nth) reinterpret_cast<uint4 *>(u.keys)[i] = z;
  for (uint64_t i = tid; i < cap / 4; i += nth) reinterpret_cast<uint4 *>(u.inserts)[i] = z;
  const uint64_t nd = (uint64_t)u.direct_rows * n_sketch;
  for (uint64_t i = tid; i < nd; i += nth) u.direct[i] = 0;
  if (tid == 0) { u.n_cand[0] = 0; u.n_cand[1] = 0; }
}
// SM count of the current device, for the grid-stride helpers below that have no context at hand
int device_sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 132;
  return n;
}

void launch_unit_clear(const UnitMap &u, uint32_t n_sketch, int n_sm, cudaStream_t stream) {
  k_unit_clear<<<n_sm * 8, 256, 0, stream>>>(u, n_sketch);
}

int launch_unit_accounting(const Params &p, int n_sm, cudaStream_t stream) {
  if (p.n_reads == 0) return 0;
  k_unit_mark<<<n_sm * 4, 256, 0, stream>>>(p);
  k_unit_decide<<<n_sm * UNIT_DECIDE_CTAS_PER_SM, 256, 0, stream>>>(p);     // blocks past the candidate count return at once
  return 2;
}

__global__ void k_flag_dense_global(const uint32_t *distinct, uint8_t *dense_flag, uint32_t n_sketch) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n_sketch && distinct[t] >= 1025u) dense_flag[t] = 1;
}
void launch_flag_dense_global(const uint32_t *distinct, uint8_t *dense_flag, uint32_t n_sketch, cudaStream_t stream) {
  if (n_sketch) k_flag_dense_global<<<(n_sketch + 255) / 256, 256, 0, stream>>>(distinct, dense_flag, n_sketch);
}

// krakenuniq-extract-reads' selection (:107-119) of each read's Kraken line: the line's taxid (the filtered call when a
// threshold is set) is looked up in the sorted member taxids; KUQ_EXTRACT_OTHERS takes every line.  One thread per read;
// each warp adds its selected reads to *count with one atomic.
__global__ void __launch_bounds__(256) k_extract_select(const uint32_t *__restrict__ call, const uint32_t *__restrict__ fcall,
                                                        uint32_t n_reads, const uint32_t *__restrict__ members,
                                                        uint32_t n_members, uint32_t flags, uint8_t *__restrict__ sel,
                                                        uint32_t *count) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  bool selected = false;
  if (r < n_reads) {
    const uint32_t c = __ldg(call + r);
    const bool line = c != 0 || !(flags & KUQ_EXTRACT_CLASSIFIED_ONLY);
    if (line) {
      if (flags & KUQ_EXTRACT_OTHERS) {
        selected = true;
      } else {
        const uint32_t t = fcall ? __ldg(fcall + r) : c;
        uint32_t lo = 0, hi = n_members;                 // first member >= t
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (__ldg(members + mid) < t) lo = mid + 1; else hi = mid;
        }
        selected = lo < n_members && __ldg(members + lo) == t;
      }
    }
    sel[r] = (uint8_t)((selected != ((flags & KUQ_EXTRACT_INVERT) != 0)) | (line ? 0 : 2));
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, selected);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(count, (uint32_t)__popc(m));
}
void launch_extract_select(const uint32_t *call, const uint32_t *fcall, uint32_t n_reads, const uint32_t *members,
                           uint32_t n_members, uint32_t flags, uint8_t *sel, uint32_t *count, cudaStream_t stream) {
  if (n_reads) k_extract_select<<<(n_reads + 255) / 256, 256, 0, stream>>>(call, fcall, n_reads, members, n_members, flags, sel, count);
}

// getEncodedRank(enc, 25, 12), hyperloglogplus.cpp:152-161
__device__ __forceinline__ uint32_t encoded_rank_dev(uint32_t e) {
  if (e & 1) return 13 + ((e >> 1) & 0x3F);
  uint32_t r = e << 12;
  return (r ? (uint32_t)__clz(r) : 20u) + 1;
}

// sparseRegisterHistogram (hyperloglogplus.cpp:356-366) for every taxon that stayed sparse: C[t][rank]++ over the
// distinct codes of t (the host derives C[0] = 2^25 - |S_t|)
__global__ void k_sparse_histograms(const KeySource src, const uint8_t *dense_flag, uint32_t *hist) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < src.n; i += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = source_key(src, i);
    if (!key) continue;
    const uint32_t taxon = (uint32_t)(key >> 32) - 1;
    if (dense_flag[taxon]) continue;
    atomicAdd(hist + (size_t)taxon * 64 + min(encoded_rank_dev((uint32_t)key), 63u), 1u);
  }
}
void launch_sparse_histograms(const KeySource &src, const uint8_t *dense_flag, uint32_t *hist, cudaStream_t stream) {
  if (src.n) k_sparse_histograms<<<device_sm_count() * 16, 256, 0, stream>>>(src, dense_flag, hist);
}

// union of the sparse code sets of the member taxa (sparse ∪ sparse merge, hyperloglogplus.cpp:600-603)
__global__ void k_sparse_union(const KeySource src, const uint8_t *member,
                               unsigned long long *scratch, uint64_t smask, uint32_t *hist64, uint32_t *overflow) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < src.n; i += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = source_key(src, i);
    if (!key) continue;
    const uint32_t taxon = (uint32_t)(key >> 32) - 1;
    if (!member[taxon]) continue;
    const uint32_t code = (uint32_t)key;
    const unsigned long long k2 = (1ull << 32) | code;
    uint64_t q = mix64(k2) & smask;
    for (uint64_t probe = 0; probe <= smask; probe++) {
      unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(scratch + q);
      if (cur == k2) break;
      if (cur == 0) {
        cur = atomicCAS(scratch + q, 0ull, k2);
        if (cur == 0) { atomicAdd(hist64 + min(encoded_rank_dev(code), 63u), 1u); break; }
        if (cur == k2) break;
      }
      q = (q + 1) & smask;
      if (probe == smask) atomicExch(overflow, 1u);
    }
  }
}
void launch_sparse_union(const KeySource &src, const uint8_t *member,
                         unsigned long long *scratch_set, uint64_t scratch_mask, uint32_t *hist64, uint32_t *overflow,
                         cudaStream_t stream) {
  if (src.n) k_sparse_union<<<device_sm_count() * 16, 256, 0, stream>>>(src, member, scratch_set, scratch_mask, hist64, overflow);
}

// The kept items of the active lanes go to out[*n_out ...]: one cursor atomic per warp.  *n_out counts them also beyond
// out_cap.
template <typename Item>
__device__ __forceinline__ void warp_append(bool keep, const Item &item, Item *out, uint64_t out_cap, unsigned long long *n_out) {
  const uint32_t m = __ballot_sync(__activemask(), keep);
  if (!keep) return;
  const uint32_t lane = threadIdx.x & 31;
  unsigned long long base = 0;
  const int leader = __ffs(m) - 1;
  if ((int)lane == leader) base = atomicAdd(n_out, (unsigned long long)__popc(m));
  base = __shfl_sync(m, base, leader);
  const unsigned long long pos = base + __popc(m & ((1u << lane) - 1));
  if (pos < out_cap) out[pos] = item;
}

// export / import of the sparse tier (cross-GPU union of the (taxon, code) sets)
__global__ void k_sparse_export(const KeySource src, const uint8_t *dense_flag,
                                unsigned long long *out, uint64_t out_cap, unsigned long long *n_out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < src.n; i += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = source_key(src, i);
    warp_append(key && !dense_flag[(uint32_t)(key >> 32) - 1], key, out, out_cap, n_out);
  }
}
__global__ void k_sparse_import(const unsigned long long *keys, uint64_t n, SparseSet s, const uint8_t *dense_flag,
                                uint32_t *error_flag) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = keys[i];
    if (!key) continue;
    const uint32_t taxon = (uint32_t)(key >> 32) - 1;
    if (dense_flag[taxon]) continue;
    const int ins = sparse_insert(s, taxon, (uint32_t)key);
    if (ins > 0) atomicAdd(s.distinct + taxon, 1u);
    else if (ins < 0) atomicExch(error_flag, 4u);
  }
}
void launch_sparse_export(const KeySource &src, const uint8_t *dense_flag,
                          unsigned long long *out, uint64_t out_cap, unsigned long long *n_out, cudaStream_t stream) {
  if (src.n) k_sparse_export<<<device_sm_count() * 16, 256, 0, stream>>>(src, dense_flag, out, out_cap, n_out);
}
void launch_sparse_import(const unsigned long long *keys, uint64_t n, const SparseSet &s, const uint8_t *dense_flag,
                          uint32_t *error_flag, cudaStream_t stream) {
  if (n) k_sparse_import<<<(int)min((uint64_t)device_sm_count() * 16, (n + 255) / 256), 256, 0, stream>>>(keys, n, s, dense_flag, error_flag);
}

// ---- exact counting (classifyExact) ---------------------------------------------------------------------------
// 1 = new pair, 0 = already there, -1 = table full.  Entries go 0 → final in one 128-bit CAS and never change again.
__device__ __forceinline__ int exact_insert(const ExactSet &e, uint32_t taxon, uint64_t canon) {
  const ExactPair want{canon + 1ull, (unsigned long long)taxon + 1ull};
  const ExactPair empty{0ull, 0ull};
  uint64_t s = mix64(canon * 0x9E3779B97F4A7C15ull + taxon) & e.mask;
  for (uint64_t probe = 0; probe <= e.mask; probe++) {
    const ulonglong2 seen = __ldcg(reinterpret_cast<const ulonglong2 *>(e.slots + s));    // one 16-byte load
    ExactPair cur{seen.x, seen.y};
    if (cur.kmer1 == 0 || cur.taxon1 == 0) {                // empty (or a load that raced with the writer): ask atomically
      cur = atomicCAS(e.slots + s, empty, want);
      if (cur.kmer1 == 0 && cur.taxon1 == 0) return 1;
    }
    if (cur.kmer1 == want.kmer1 && cur.taxon1 == want.taxon1) return 0;
    s = (s + 1) & e.mask;
  }
  return -1;
}

// add_kmer of the exact container (readcounts.hpp:71-74 with khset64_t): thread per text position, after the lookup
// wrote the window's dense taxon (0 for a miss) to codes_dense
__global__ void __launch_bounds__(256) k_exact_insert(const __grid_constant__ Params p) {
  const uint64_t g_begin = p.offsets[0], g_end = p.offsets[p.n_reads];
  for (uint64_t g = g_begin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < g_end;
       g += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t bin = __ldg(p.bins + g);
    if (bin == BIN_NONE || bin == BIN_AMBIG) continue;
    const uint32_t taxon = p.codes_dense[g];
    const int ins = exact_insert(p.exact, taxon, __ldg(p.canon + g));
    if (ins > 0) atomicAdd(p.exact.count + taxon, 1ull);
    else if (ins < 0) atomicExch(p.error_flag, 4u);
  }
}

// Slots of the two device tables: a sparse-tier key (0 = empty) or an exact pair (kmer1 0 = empty).
__device__ __forceinline__ bool occupied(unsigned long long key) { return key != 0; }
__device__ __forceinline__ bool occupied(const ExactPair &pr) { return pr.kmer1 != 0; }
__device__ __forceinline__ int reinsert(const SparseSet &s, unsigned long long key) {
  return sparse_insert(s, (uint32_t)(key >> 32) - 1, (uint32_t)key);
}
__device__ __forceinline__ int reinsert(const ExactSet &e, const ExactPair &pr) {
  return exact_insert(e, (uint32_t)(pr.taxon1 - 1), pr.kmer1 - 1);
}

// the items of an outgrown table into its successor with the table's own probe sequence; every item is counted already,
// so the per-taxon counters stay as they are
template <typename Set, typename Item>
__global__ void k_rehash(const Item *old_slots, uint64_t old_cap, Set s, uint32_t *error_flag) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < old_cap; i += (uint64_t)gridDim.x * blockDim.x) {
    const Item it = old_slots[i];
    if (!occupied(it)) continue;
    if (reinsert(s, it) < 0) atomicExch(error_flag, 4u);
  }
}
void launch_rehash(const unsigned long long *old_slots, uint64_t old_cap, const SparseSet &s, uint32_t *error_flag, cudaStream_t stream) {
  if (old_cap) k_rehash<<<device_sm_count() * 16, 256, 0, stream>>>(old_slots, old_cap, s, error_flag);
}
void launch_rehash(const ExactPair *old_slots, uint64_t old_cap, const ExactSet &e, uint32_t *error_flag, cudaStream_t stream) {
  if (old_cap) k_rehash<<<(int)min((uint64_t)device_sm_count() * 16, (old_cap + 255) / 256), 256, 0, stream>>>(old_slots, old_cap, e, error_flag);
}

// occupied slots [lo, hi) → dense pairs (out_cap 0 only counts them)
__global__ void k_exact_export(const ExactPair *slots, uint64_t lo, uint64_t hi, ExactPair *out, uint64_t out_cap,
                               unsigned long long *n_out) {
  for (uint64_t i = lo + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (uint64_t)gridDim.x * blockDim.x) {
    const ExactPair pr = slots[i];
    warp_append(occupied(pr), pr, out, out_cap, n_out);
  }
}
// pairs of another context into this table: only the ones it did not hold yet add to count[]
__global__ void k_exact_import(const ExactPair *pairs, uint64_t n, ExactSet e, uint32_t *error_flag) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const ExactPair pr = pairs[i];
    if (!pr.kmer1 || !pr.taxon1) continue;
    const uint32_t taxon = (uint32_t)(pr.taxon1 - 1);
    const int ins = exact_insert(e, taxon, pr.kmer1 - 1);
    if (ins > 0) atomicAdd(e.count + taxon, 1ull);
    else if (ins < 0) atomicExch(error_flag, 4u);
  }
}
void launch_exact_export(const ExactPair *slots, uint64_t lo, uint64_t hi, ExactPair *out, uint64_t out_cap,
                         unsigned long long *n_out, cudaStream_t stream) {
  if (hi > lo) k_exact_export<<<(int)min((uint64_t)device_sm_count() * 16, (hi - lo + 255) / 256), 256, 0, stream>>>(slots, lo, hi, out, out_cap, n_out);
}
void launch_exact_import(const ExactPair *pairs, uint64_t n, const ExactSet &e, uint32_t *error_flag, cudaStream_t stream) {
  if (n) k_exact_import<<<(int)min((uint64_t)device_sm_count() * 16, (n + 255) / 256), 256, 0, stream>>>(pairs, n, e, error_flag);
}

// distinct k-mers among the pairs whose taxon is a clade member
__global__ void k_exact_union(ExactSet e, const uint8_t *member, unsigned long long *scratch, uint64_t smask,
                              unsigned long long *n_distinct, uint32_t *overflow) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= e.mask; i += (uint64_t)gridDim.x * blockDim.x) {
    const ExactPair pr = e.slots[i];
    if (!pr.kmer1 || !member[pr.taxon1 - 1]) continue;
    uint64_t q = mix64(pr.kmer1) & smask;
    for (uint64_t probe = 0; probe <= smask; probe++) {
      unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(scratch + q);
      if (cur == pr.kmer1) break;
      if (cur == 0) {
        cur = atomicCAS(scratch + q, 0ull, pr.kmer1);
        if (cur == 0) { atomicAdd(n_distinct, 1ull); break; }
        if (cur == pr.kmer1) break;
      }
      q = (q + 1) & smask;
      if (probe == smask) atomicExch(overflow, 1u);
    }
  }
}
void launch_exact_union(const ExactSet &e, const uint8_t *member, unsigned long long *scratch_set, uint64_t scratch_mask,
                        unsigned long long *n_distinct, uint32_t *overflow, cudaStream_t stream) {
  if (e.slots) k_exact_union<<<device_sm_count() * 16, 256, 0, stream>>>(e, member, scratch_set, scratch_mask, n_distinct, overflow);
}

// Quick mode, preloaded path: the k-mer loop of classify_sequence leaves at the quick_min-th hit (classify.cpp:943-944),
// so the windows behind it are never looked at — no add_kmer, no hit.  One warp per read finds that window in the
// looked-up codes, shortens the read to it and wipes the later windows from the scan scratch; the counting pass
// (k_lookup<MODE_RESOLVE>), the per-unit accounting and k_resolve<true> then see the read the reference saw.
__global__ void __launch_bounds__(256) k_quick_cut(const __grid_constant__ Params p, const uint32_t *codes) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t warps_total = gridDim.x * (blockDim.x >> 5);
  for (uint32_t r = blockIdx.x * (blockDim.x >> 5) + warp; r < p.n_reads; r += warps_total) {
    const uint64_t base = p.offsets[r];
    const uint32_t nwin = p.n_windows[r];
    uint32_t seen = 0, cutoff = nwin;
    for (uint32_t s = 0; s * 32 < nwin; s++) {
      const uint32_t i = s * 32 + lane;
      const uint32_t c = i < nwin ? codes[base + i] : 0;
      const uint32_t bm = __ballot_sync(0xFFFFFFFFu, c != 0 && c != AMBIG && c != FOUND_ZERO);
      const uint32_t cnt = __popc(bm);
      if (seen + cnt >= p.quick_min) {
        uint32_t m = bm;
        for (uint32_t j = seen + 1; j < p.quick_min; j++) m &= m - 1;   // drop the hits before the quick_min-th
        cutoff = s * 32 + (uint32_t)__ffs(m) - 1;
        break;
      }
      seen += cnt;
    }
    if (cutoff < nwin) {
      for (uint32_t i = cutoff + 1 + lane; i < nwin; i += 32) p.bins[base + i] = BIN_NONE;
      if (lane == 0) p.n_windows[r] = cutoff + 1;
    }
  }
}

int classify_smem_bytes() { return N_STAGES * STAGE_BYTES + (int)sizeof(SharedState); }

// mode MODE_FUSED : scan → lookup (+HLL) → resolve            (whole database on this GPU)
//      MODE_LOOKUP: scan → lookup into p.codes_dense            (one range of a sharded / chunked database)
//      MODE_RESOLVE: scan → HLL from merged codes → resolve    (owner of the reads after the merge)
// picks the lean instantiation when the launch uses none of the rare switches (see k_lookup)
template <int MODE>
static void launch_lookup(const Params &q, int lgrid, cudaStream_t stream, bool lean) {
  if constexpr (MODE == MODE_FUSED) {
    if (q.db.k == 31 && q.db.nt == 15) {
      if (lean) k_lookup<MODE, true, true><<<lgrid, 256, 0, stream>>>(q);
      else k_lookup<MODE, false, true><<<lgrid, 256, 0, stream>>>(q);
      return;
    }
  }
  if (lean) k_lookup<MODE, true><<<lgrid, 256, 0, stream>>>(q);
  else k_lookup<MODE, false><<<lgrid, 256, 0, stream>>>(q);
}
template <int MODE>
static void launch_lookup(const Params &q, int lgrid, cudaStream_t stream) {
  launch_lookup<MODE>(q, lgrid, stream, !(q.flags & (8u | 16u | 32u)) && !q.only_hits && !q.n_peers);
}

bool windows_packed(int mode, const Params &p) {
  return mode == MODE_FUSED && p.hll_mode != 3u && !(p.quick_min != 0 && p.quick_stop);
}

int launch_classify(int mode, const Params &p, int n_sm, cudaStream_t stream, cudaEvent_t *stage_events) {
  const int smem = classify_smem_bytes();
  // per device (function attributes belong to the current context): cheap enough to set on every call
  cudaFuncSetAttribute(k_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  int launches = 0;
  if (p.n_reads == 0) return 0;
  if (windows_packed(mode, p)) {
    const uint64_t n_half = 2 * (p.total_bases / 32 + 2);
    k_pack<<<(int)min((uint64_t)n_sm * 8, (n_half + 255) / 256), 256, 0, stream>>>(p);
    k_pack_reads<<<(int)min((uint32_t)n_sm * 8, (p.n_reads + 256) / 256), 256, 0, stream>>>(p);
    launches += 2;
  } else {
    int grid = n_sm * 4;
    if ((uint32_t)grid > p.n_chunks) grid = (int)p.n_chunks;
    k_scan<<<grid, CTA_THREADS, smem, stream>>>(p);
    launches++;
  }
  if (stage_events) cudaEventRecord(stage_events[0], stream);
  const int lgrid = (int)min((uint64_t)n_sm * 8 * 8, (p.total_bases + 255) / 256);
  const bool quick = p.quick_min != 0 && mode != MODE_LOOKUP;
  const bool exact = p.hll_mode == 3u && mode != MODE_LOOKUP;
  if (exact) {
    // classifyExact: plain lookup (no sketch work), then the k-mer sets, then the usual resolve
    Params q = p;
    if (mode == MODE_FUSED) {
      q.only_hits = 0; q.n_peers = 0; q.flags &= ~16u;
      launch_lookup<MODE_LOOKUP>(q, lgrid, stream);
    } else {
      q.flags |= 4u;                                         // merged codes → codes_dense, no sketches
      launch_lookup<MODE_RESOLVE>(q, lgrid, stream);
    }
    if (!(p.flags & 4u)) { k_exact_insert<<<lgrid, 256, 0, stream>>>(p); launches++; }
  } else if (quick && p.quick_stop) {
    // lookup first, end every read at its quick_min-th hit, then count what is left
    Params q = p;
    if (mode == MODE_FUSED) {
      q.only_hits = 0; q.n_peers = 0; q.flags &= ~16u;
      launch_lookup<MODE_LOOKUP>(q, lgrid, stream);
      launches++;
      q.codes_in = p.codes_dense;
    }
    const int cgrid = (int)min((uint32_t)n_sm * 8, (p.n_reads + 7) / 8);
    k_quick_cut<<<cgrid, 256, 0, stream>>>(p, q.codes_in);
    q.flags = p.flags;
    launch_lookup<MODE_RESOLVE>(q, lgrid, stream);
    launches += 2;
  } else if (mode == MODE_FUSED) launch_lookup<MODE_FUSED>(p, lgrid, stream);
  else if (mode == MODE_LOOKUP) launch_lookup<MODE_LOOKUP>(p, lgrid, stream);
  else launch_lookup<MODE_RESOLVE>(p, lgrid, stream);
  if (exact || !(quick && p.quick_stop)) launches++;
  if (stage_events) cudaEventRecord(stage_events[1], stream);
  if (mode != MODE_LOOKUP) {
    const int rgrid = (int)min((uint32_t)n_sm * 4 * 2, (p.n_reads + CTA_WARPS - 1) / CTA_WARPS);
    if (p.fcall && quick) k_resolve<true, true><<<rgrid, 256, 0, stream>>>(p);
    else if (p.fcall) k_resolve<false, true><<<rgrid, 256, 0, stream>>>(p);
    else if (quick) k_resolve<true><<<rgrid, 256, 0, stream>>>(p);
    else k_resolve<false><<<rgrid, 256, 0, stream>>>(p);
    launches++;
  }
  return launches;
}

// ------------------------------------------------------------------------------------------------------
// set_lcas (set_lcas.cpp:429-476), SURVEY.md §8 f4.  ROUND 1: compiled, not yet run on hardware.
// Library sequences arrive cut into pieces (the reference's SKIP_LEN pieces, :363-364); unit_id[r] carries the dense
// taxid of piece r.  One warp per piece, lane = window: find the record of the canonical k-mer and fold the
// sequence's taxid into its value with lca() through a CAS loop.  lca over taxa of one tree is associative,
// commutative and idempotent (default ancestor 1), so the order in which pieces and sequences land does not matter.
// Under -T a contaminant taxid beats everything and sticks; with at most ONE of the two contaminant taxids per batch
// (the host side sees to that) the outcome is again independent of the order inside the batch.
// ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_set_lcas(const __grid_constant__ Params p) {
  const DbView &db = p.db;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t warps_total = gridDim.x * (blockDim.x >> 5);
  uint8_t *pairs = const_cast<uint8_t *>(db.pairs);
  for (uint32_t r = blockIdx.x * (blockDim.x >> 5) + warp; r < p.n_reads; r += warps_total) {
    const uint64_t base = p.offsets[r];
    const uint32_t nwin = p.n_windows[r];
    const uint32_t t = p.unit_id[r];
    for (uint32_t i = lane; i < nwin; i += 32) {
      const uint32_t bin = __ldg(p.bins + base + i);
      if (bin == BIN_NONE || bin == BIN_AMBIG) continue;                  // :434-435
      if (bin < db.bin_lo || bin >= db.bin_hi) continue;                  // another range of the database
      const uint64_t canon = __ldg(p.canon + base + i);
      const uint64_t *o = db.offsets + (bin - db.bin_lo);
      uint64_t lo = __ldg(o) - db.rec_base, hi = __ldg(o + 1) - db.rec_base;
      bool found = false;
      while (lo < hi) {
        const uint64_t mid = lo + ((hi - lo) >> 1);
        const uint64_t key = load_key(db.pairs, mid, db.key_mask);
        if (key < canon) lo = mid + 1;
        else if (key > canon) hi = mid;
        else { lo = mid; found = true; break; }
      }
      if (!found) { atomicAdd(p.stats, 1ull); continue; }                 // "kmer found in sequence that is not in database"
      uint32_t *val = reinterpret_cast<uint32_t *>(pairs + lo * 12) + 2;
      uint32_t old = *reinterpret_cast<volatile uint32_t *>(val);
      for (;;) {
        uint32_t nw;
        if (p.lca_flags & 2u) nw = 0;                                     // -R, :458-459
        else if (!(p.lca_flags & 1u)) nw = lca_dense(p.tax, t, old);      // :461
        else if (old != 0 && (old == p.lca_keep[0] || old == p.lca_keep[1])) nw = old;   // -T: contaminants stick, :465-466
        else if (t == p.lca_keep[0] || t == p.lca_keep[1]) nw = t;        // :467-470
        else nw = lca_dense(p.tax, t, old);                               // :472
        if (nw == old) break;
        const uint32_t prev = atomicCAS(val, old, nw);
        if (prev == old) break;
        old = prev;
      }
    }
  }
}

// stage 1 alone: canonical k-mer + minimizer bin of every window into p.canon / p.bins (database build, workload tools)
int launch_scan_only(const Params &p, int n_sm, cudaStream_t stream) {
  if (p.n_reads == 0) return 0;
  const int smem = classify_smem_bytes();
  cudaFuncSetAttribute(k_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  int grid = n_sm * 4;
  if ((uint32_t)grid > p.n_chunks) grid = (int)p.n_chunks;
  k_scan<<<grid, CTA_THREADS, smem, stream>>>(p);
  return 1;
}

// stage 2 alone over windows that are already there (kuq_layout_exp.cu times the product's kernel next to its
// variants): p.offsets = {first, last + 1} text positions with p.n_reads = 1
// fused = 1: k_lookup<MODE_FUSED> over the packed blocks of p (counts into the sketches of p); fused = 0: MODE_LOOKUP over
// scratch; lean: see k_lookup (the caller vouches for the flags)
int launch_lookup_only(const Params &p, int n_sm, cudaStream_t stream, int fused, int lean) {
  const int lgrid = (int)max((uint64_t)1, min((uint64_t)n_sm * 8 * 8, (p.total_bases + 255) / 256));
  if (fused) launch_lookup<MODE_FUSED>(p, lgrid, stream, lean != 0);
  else launch_lookup<MODE_LOOKUP>(p, lgrid, stream, lean != 0);
  return 1;
}

int launch_lookup_multi(const Params &p, int n_sm, cudaStream_t stream, bool scan) {
  if (p.n_reads == 0) return 0;
  const int launches = scan ? launch_scan_only(p, n_sm, stream) : 0;
  const int lgrid = (int)min((uint64_t)n_sm * 8 * 8, (p.total_bases + 255) / 256);
  k_lookup<MODE_LOOKUP, false, false, true><<<lgrid, 256, 0, stream>>>(p);
  return launches + 1;
}

// scan the pieces, then fold their taxids into the record values; returns #kernels launched
int launch_set_lcas(const Params &p, int n_sm, cudaStream_t stream) {
  if (p.n_reads == 0) return 0;
  const int smem = classify_smem_bytes();
  cudaFuncSetAttribute(k_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  int grid = n_sm * 4;
  if ((uint32_t)grid > p.n_chunks) grid = (int)p.n_chunks;
  k_scan<<<grid, CTA_THREADS, smem, stream>>>(p);
  const int rgrid = (int)min((uint32_t)n_sm * 8, (p.n_reads + 7) / 8);
  k_set_lcas<<<rgrid, 256, 0, stream>>>(p);
  return 2;
}

// ------------------------------------------------------------------------------------------------------
// database staging: distinct taxids + record counts (KrakenDB::count_taxons, krakendb.cpp:90-113) and the
// in-place rewrite taxid → dense id
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t hash_u32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

// keys[] holds taxid + 1 (0 = empty)
__global__ void k_collect_taxids(const uint8_t *pairs, uint64_t n_rec, uint32_t *keys, unsigned long long *counts,
                                 uint32_t cap_mask, uint32_t *overflow) {
  const uint32_t lane = threadIdx.x & 31;
  for (uint64_t base = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) - lane; base < n_rec;
       base += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t i = base + lane;
    bool in = i < n_rec;
    uint32_t v = in ? load_val(pairs, i) : 0;
    uint32_t active = __ballot_sync(0xFFFFFFFFu, in);
    if (!in) continue;
    uint32_t same = __match_any_sync(active, v);
    if (lane != (uint32_t)(__ffs(same) - 1)) continue;      // one lane per distinct value
    uint32_t key = v + 1;
    if (key == 0) { atomicExch(overflow, 2u); continue; }   // taxid 0xFFFFFFFF is reserved
    uint32_t slot = hash_u32(v) & cap_mask;
    for (uint32_t probe = 0; probe <= cap_mask; probe++) {
      uint32_t cur = keys[slot];
      if (cur == 0) cur = atomicCAS(keys + slot, 0u, key), cur = cur ? cur : key;
      if (cur == key) { atomicAdd(counts + slot, (unsigned long long)__popc(same)); break; }
      slot = (slot + 1) & cap_mask;
      if (probe == cap_mask) atomicExch(overflow, 1u);
    }
  }
}

__global__ void k_remap_values(uint8_t *pairs, uint64_t n_rec, const uint32_t *keys, const uint32_t *dense,
                               uint32_t cap_mask, uint32_t *missing, uint32_t hi_mask) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rec; i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t *vp = reinterpret_cast<uint32_t *>(pairs + i * 12) + 2;
    uint32_t v = *vp;
    uint32_t key = v + 1, slot = hash_u32(v) & cap_mask, d = 0xFFFFFFFFu;
    for (uint32_t probe = 0; probe <= cap_mask; probe++) {
      uint32_t cur = keys[slot];
      if (cur == key) { d = dense[slot]; break; }
      if (cur == 0) break;
      slot = (slot + 1) & cap_mask;
    }
    if (d == 0xFFFFFFFFu) { atomicExch(missing, 1u); d = 0; }
    *vp = d;
    // bits of the key word above 2k are ignored by the reference (krakendb.cpp:283-284) and serve as record flags
    // here (SEEN_BIT): start from zero
    if ((vp[-1] & ~hi_mask) != 0) vp[-1] &= hi_mask;
  }
}

// Flagged records → sparse-tier keys of the set (records that leave HBM, or contexts whose set receives hit keys from
// elsewhere): for every record a counted hit flagged, insert (taxon, encodeHashIn32Bit(hash(k-mer))) into the set
// unless the taxon went dense, and clear the flag.  mode 0 = count the records carrying `bit` of taxa that are not
// dense (stats[0]), 1 = insert + clear SEEN_BIT, 2 = clear SEEN_BIT and KEPT_BIT, 3 = move the kept records into the
// set: insert + clear KEPT_BIT, without counting (their keys are counted in `distinct` already).
__global__ void __launch_bounds__(256) k_harvest_seen(uint8_t *pairs, uint64_t n_rec, uint32_t hi_mask, const uint8_t *dense_flag,
                                                      SparseSet set, unsigned long long *stats, uint32_t *error_flag, int mode,
                                                      uint32_t bit) {
  unsigned long long n_local = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rec; i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t *w = reinterpret_cast<uint32_t *>(pairs + i * 12);
    const uint32_t hiw = w[1];
    if (!(hiw & bit)) continue;
    const uint32_t taxon = w[2];
    if (mode == 0) { n_local += dense_flag[taxon] ? 0 : 1; continue; }
    w[1] = hiw & ~bit;
    if (mode == 2 || dense_flag[taxon]) continue;
    const int ins = sparse_insert(set, taxon, (uint32_t)record_key(w, hiw, hi_mask));
    if (ins > 0 && mode == 1) atomicAdd(set.distinct + taxon, 1u);
    else if (ins < 0) atomicExch(error_flag, 4u);
  }
  if (mode == 0) {
    for (int o = 16; o; o >>= 1) n_local += __shfl_xor_sync(0xFFFFFFFFu, n_local, o);
    if ((threadIdx.x & 31) == 0 && n_local) atomicAdd(stats, n_local);
  }
}
void launch_harvest_seen(uint8_t *pairs, uint64_t n_rec, uint64_t key_mask, const uint8_t *dense_flag, const SparseSet &set,
                         unsigned long long *stats, uint32_t *error_flag, int mode, cudaStream_t stream) {
  if (!n_rec) return;
  const int grid = (int)min((uint64_t)device_sm_count() * 16, (n_rec + 255) / 256);
  const uint32_t bit = mode == 2 ? (SEEN_BIT | KEPT_BIT) : mode == 3 ? KEPT_BIT : SEEN_BIT;
  k_harvest_seen<<<grid, 256, 0, stream>>>(pairs, n_rec, (uint32_t)(key_mask >> 32), dense_flag, set, stats, error_flag, mode, bit);
}

// Harvest of a resident range without set inserts.  The sparse-tier key of a record is a function of the record, so
// "the key is in the tier" is one more record flag (KEPT_BIT), held by the primary of each (taxon, code) group.
// (a) k_fold_secondaries: a flagged secondary hands its flag to its primary.
// (b) k_harvest_keep, one streaming pass: a flagged record that is not kept yet (and whose taxon is not dense) becomes
//     kept and counts one distinct code of its taxon; every flag is cleared.  The per-taxon counts are gathered in a
//     shared-memory table per CTA (a few thousand taxa would otherwise take hundreds of millions of same-address global
//     atomics); taxa that do not find a slot there count globally.
__global__ void k_fold_secondaries(uint8_t *pairs, const uint2 *list, uint64_t n) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) {
    const uint2 sp = list[e];                              // (secondary, primary) record indices
    uint32_t *ws = reinterpret_cast<uint32_t *>(pairs + (uint64_t)sp.x * 12) + 1;
    const uint32_t hiw = *ws;
    if (!(hiw & SEEN_BIT)) continue;
    *ws = hiw & ~SEEN_BIT;                                 // a record is the secondary of one entry only
    atomicOr(reinterpret_cast<uint32_t *>(pairs + (uint64_t)sp.y * 12) + 1, SEEN_BIT);
  }
}

// Keep mode counts every record whose KEPT_BIT it set, secondaries included: the flag moves to the primary, and a
// primary that had it already (two members of the group were kept) held the code already.  Order-independent.
__global__ void k_settle_kept(uint8_t *pairs, const uint2 *list, uint64_t n, uint32_t *distinct, unsigned long long *n_dup) {
  unsigned long long dup = 0;
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) {
    const uint2 sp = list[e];                              // (secondary, primary) record indices
    uint32_t *ws = reinterpret_cast<uint32_t *>(pairs + (uint64_t)sp.x * 12) + 1;
    const uint32_t hiw = *ws;
    if (!(hiw & KEPT_BIT)) continue;
    *ws = hiw & ~KEPT_BIT;
    if (atomicOr(reinterpret_cast<uint32_t *>(pairs + (uint64_t)sp.y * 12) + 1, KEPT_BIT) & KEPT_BIT) {
      atomicSub(distinct + ws[1], 1u);                     // ws[1]: the taxon, the same for the whole group
      dup++;
    }
  }
  for (int o = 16; o; o >>= 1) dup += __shfl_xor_sync(0xFFFFFFFFu, dup, o);
  if ((threadIdx.x & 31) == 0 && dup) atomicAdd(n_dup, dup);
}
void launch_settle_kept(uint8_t *pairs, const uint2 *secondaries, uint64_t n_secondaries, uint32_t *distinct,
                        unsigned long long *n_dup, cudaStream_t stream) {
  if (!n_secondaries) return;
  k_settle_kept<<<(int)min((uint64_t)device_sm_count() * 8, (n_secondaries + 255) / 256), 256, 0, stream>>>(
      pairs, secondaries, n_secondaries, distinct, n_dup);
}

// k_harvest_keep streams the records in groups of 4 (48 bytes = three 16-byte loads, KEEP_UNROLL groups in flight per
// thread).  The records are 4-byte aligned only: the groups start at the first 16-byte aligned record, and the up to 3
// records before it and after the last whole group are handled one by one.  A group without a flagged record is not
// written; otherwise only the high words whose flags change are stored, so sectors without a flagged record stay clean.
// Per-taxon counts: with at most KEEP_DIRECT_TAXA taxa, each CTA holds one shared counter per taxon, indexed by the
// taxon (a dense taxon's counter holds KEEP_DENSE, so one shared load answers "dense?" too).  A hashed table of
// KEEP_SLOTS taxa would overflow into same-address global atomics once the records span more taxa than it holds (the
// bench's 2000 genomes do); that table remains for larger taxonomies.
constexpr int KEEP_SLOTS = 1024;
constexpr int KEEP_UNROLL = 2;
constexpr int KEEP_THREADS = 256;
constexpr uint32_t KEEP_DIRECT_TAXA = 16384;     // 64 KiB of counters per CTA
constexpr uint32_t KEEP_DENSE = 0xFFFFFFFFu;

// one flagged record's high word: SEEN cleared; neither KEPT nor of a dense taxon → KEPT, counted
template <bool DIRECT>
__device__ __forceinline__ uint32_t keep_record(uint32_t *s_tab, const uint8_t *dense_flag, uint32_t *distinct, uint32_t hiw,
                                                uint32_t taxon, unsigned long long &n_local) {
  if (hiw & KEPT_BIT) return hiw & ~SEEN_BIT;
  if (DIRECT) {
    if (s_tab[taxon] == KEEP_DENSE) return hiw & ~SEEN_BIT;
    atomicAdd(&s_tab[taxon], 1u);
  } else {
    if (dense_flag[taxon]) return hiw & ~SEEN_BIT;
    uint32_t *s_tax = s_tab, *s_cnt = s_tab + KEEP_SLOTS;
    uint32_t h = (taxon * 0x9E3779B1u) >> 22, probe = 0;
    for (; probe < 8; probe++, h = (h + 1) & (KEEP_SLOTS - 1)) {
      uint32_t cur = s_tax[h];
      if (cur == 0) cur = atomicCAS(&s_tax[h], 0u, taxon + 1), cur = cur ? cur : taxon + 1;
      if (cur == taxon + 1) { atomicAdd(&s_cnt[h], 1u); break; }
    }
    if (probe == 8) atomicAdd(distinct + taxon, 1u);
  }
  n_local++;
  return (hiw & ~SEEN_BIT) | KEPT_BIT;
}

template <bool DIRECT>
__global__ void __launch_bounds__(KEEP_THREADS) k_harvest_keep(uint8_t *pairs, uint64_t n_rec, const uint8_t *dense_flag,
                                                                uint32_t n_sketch, uint32_t *distinct, unsigned long long *n_kept) {
  extern __shared__ uint32_t s_tab[];             // DIRECT: [n_sketch] counters; else [KEEP_SLOTS] taxa + [KEEP_SLOTS] counts
  if (DIRECT) {
    for (uint32_t s = threadIdx.x; s < n_sketch; s += blockDim.x) s_tab[s] = dense_flag[s] ? KEEP_DENSE : 0u;
  } else {
    for (int s = threadIdx.x; s < 2 * KEEP_SLOTS; s += blockDim.x) s_tab[s] = 0;
  }
  __syncthreads();
  unsigned long long n_local = 0;
  // records before the first 16-byte boundary: 12 * head + (pairs mod 16) == 0 (mod 16), pairs 4-byte aligned
  const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(pairs) & 15u);
  const uint64_t head = min((uint64_t)(mis / 4u), n_rec);
  const uint64_t n_groups = (n_rec - head) / 4, tail = head + 4 * n_groups;
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid < head + (n_rec - tail)) {                     // the edges, one record per thread
    const uint64_t i = tid < head ? tid : tail + (tid - head);
    uint32_t *w = reinterpret_cast<uint32_t *>(pairs + i * 12);
    const uint32_t hiw = w[1];
    if (hiw & SEEN_BIT) w[1] = keep_record<DIRECT>(s_tab, dense_flag, distinct, hiw, w[2], n_local);
  }
  uint4 *groups = reinterpret_cast<uint4 *>(pairs + head * 12);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x * KEEP_UNROLL;
  for (uint64_t g0 = (uint64_t)blockIdx.x * blockDim.x * KEEP_UNROLL + threadIdx.x; g0 < n_groups; g0 += stride) {
    uint4 v[KEEP_UNROLL][3];
#pragma unroll
    for (int u = 0; u < KEEP_UNROLL; u++) {
      const uint64_t g = g0 + (uint64_t)u * blockDim.x;
      if (g < n_groups) {
        v[u][0] = groups[g * 3]; v[u][1] = groups[g * 3 + 1]; v[u][2] = groups[g * 3 + 2];
      } else {
        v[u][0] = v[u][1] = v[u][2] = make_uint4(0, 0, 0, 0);
      }
    }
#pragma unroll
    for (int u = 0; u < KEEP_UNROLL; u++) {
      // record r of the group: words 3r, 3r + 1 (high key word, flags), 3r + 2 (taxon)
      const uint32_t hi[4] = {v[u][0].y, v[u][1].x, v[u][1].w, v[u][2].z};
      const uint32_t tx[4] = {v[u][0].z, v[u][1].y, v[u][2].x, v[u][2].w};
      if (!((hi[0] | hi[1] | hi[2] | hi[3]) & SEEN_BIT)) continue;
      uint32_t *w = reinterpret_cast<uint32_t *>(groups + (g0 + (uint64_t)u * blockDim.x) * 3);
#pragma unroll
      for (int r = 0; r < 4; r++)
        if (hi[r] & SEEN_BIT) w[3 * r + 1] = keep_record<DIRECT>(s_tab, dense_flag, distinct, hi[r], tx[r], n_local);
    }
  }
  __syncthreads();
  if (DIRECT) {
    for (uint32_t s = threadIdx.x; s < n_sketch; s += blockDim.x)
      if (s_tab[s] && s_tab[s] != KEEP_DENSE) atomicAdd(distinct + s, s_tab[s]);
  } else {
    for (int s = threadIdx.x; s < KEEP_SLOTS; s += blockDim.x)
      if (s_tab[s]) atomicAdd(distinct + s_tab[s] - 1, s_tab[KEEP_SLOTS + s]);
  }
  for (int o = 16; o; o >>= 1) n_local += __shfl_xor_sync(0xFFFFFFFFu, n_local, o);
  if ((threadIdx.x & 31) == 0 && n_local) atomicAdd(n_kept, n_local);
}
void launch_harvest_keep(uint8_t *pairs, uint64_t n_rec, const uint2 *secondaries, uint64_t n_secondaries, const uint8_t *dense_flag,
                         uint32_t n_sketch, uint32_t *distinct, unsigned long long *n_kept, cudaStream_t stream) {
  if (!n_rec) return;
  const int n_sm = device_sm_count();
  if (n_secondaries)
    k_fold_secondaries<<<(int)min((uint64_t)n_sm * 8, (n_secondaries + 255) / 256), 256, 0, stream>>>(pairs, secondaries, n_secondaries);
  const bool direct = n_sketch <= KEEP_DIRECT_TAXA;
  const auto kernel = direct ? k_harvest_keep<true> : k_harvest_keep<false>;
  const size_t smem = direct ? 4ull * n_sketch : 8ull * KEEP_SLOTS;
  // per device (function attributes belong to the current context); the harvest runs once per run
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * KEEP_DIRECT_TAXA);
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, KEEP_THREADS, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  const uint64_t per_cta = (uint64_t)KEEP_THREADS * KEEP_UNROLL * 4;     // records per CTA per iteration
  const int grid = (int)min((uint64_t)n_sm * per_sm, (n_rec + per_cta - 1) / per_cta);     // >= 1: n_rec > 0
  kernel<<<grid, KEEP_THREADS, smem, stream>>>(pairs, n_rec, dense_flag, n_sketch, distinct, n_kept);
}

// C[taxon][v] = number of registers of the taxon holding v (registerHistogram, hyperloglogplus.cpp:337-354);
// the double-precision Ertl sum over it runs on the host.
__global__ void k_register_histograms(const uint8_t *regs, uint32_t n_sketch, uint32_t *hist) {
  __shared__ uint32_t h[64];
  for (uint32_t t = blockIdx.x; t < n_sketch; t += gridDim.x) {
    if (threadIdx.x < 64) h[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t *w = reinterpret_cast<const uint32_t *>(regs + (size_t)t * HLL_M);
    for (uint32_t i = threadIdx.x; i < HLL_M / 4; i += blockDim.x) {
      uint32_t x = w[i];
      atomicAdd(&h[x & 63], 1u);
      atomicAdd(&h[(x >> 8) & 63], 1u);
      atomicAdd(&h[(x >> 16) & 63], 1u);
      atomicAdd(&h[(x >> 24) & 63], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 64) hist[(size_t)t * 64 + threadIdx.x] = h[threadIdx.x];
    __syncthreads();
  }
}

// register-wise max over the sketches of the listed dense ids: the dense∪dense merge of the clade roll-up
// (hyperloglogplus.cpp:614-620)
__global__ void k_clade_max(const uint8_t *regs, const uint32_t *members, uint32_t n_members, uint8_t *out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;     // word index 0..1023
  if (i >= HLL_M / 4) return;
  uint32_t acc = 0;
  for (uint32_t m = 0; m < n_members; m++) {
    uint32_t x = reinterpret_cast<const uint32_t *>(regs + (size_t)members[m] * HLL_M)[i];
    acc = __vmaxu4(acc, x);
  }
  reinterpret_cast<uint32_t *>(out)[i] = acc;
}

__global__ void k_fill_u32(uint32_t *p, uint64_t n, uint32_t v) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = v;
}

void launch_collect_taxids(const uint8_t *pairs, uint64_t n_rec, uint32_t *keys, unsigned long long *counts,
                           uint32_t cap_mask, uint32_t *overflow, cudaStream_t stream) {
  if (!n_rec) return;
  int grid = (int)min((uint64_t)device_sm_count() * 8, (n_rec + 255) / 256);
  k_collect_taxids<<<grid, 256, 0, stream>>>(pairs, n_rec, keys, counts, cap_mask, overflow);
}
void launch_remap_values(uint8_t *pairs, uint64_t n_rec, const uint32_t *keys, const uint32_t *dense,
                         uint32_t cap_mask, uint32_t *missing, uint64_t key_mask, cudaStream_t stream) {
  if (!n_rec) return;
  int grid = (int)min((uint64_t)device_sm_count() * 8, (n_rec + 255) / 256);
  k_remap_values<<<grid, 256, 0, stream>>>(pairs, n_rec, keys, dense, cap_mask, missing, (uint32_t)(key_mask >> 32));
}
// Records of a database with k <= 28 ({key_len-byte key, u32 value}, key_len + 4 bytes each, packed) → the 12-byte
// {u64 key, u32 value} layout every other kernel reads.  Thread per record: the record's bytes come from the four aligned
// words that cover them (narrow must be 4-byte aligned with 16 readable bytes past the last record), funnel shifts
// line them up, the key is zero-extended (the flag bits 62 / 63 start clear) and the value copied.
__global__ void __launch_bounds__(256) k_widen_records(const uint8_t *__restrict__ narrow, uint64_t n, uint32_t key_len,
                                                        uint8_t *__restrict__ wide12) {
  const uint32_t *src = reinterpret_cast<const uint32_t *>(narrow);
  uint32_t *dst = reinterpret_cast<uint32_t *>(wide12);
  const uint64_t rec = key_len + 4;
  const uint64_t key_bytes_mask = (1ull << (8 * key_len)) - 1;        // key_len <= 7
  const uint32_t vw = key_len >> 2, vsh = 8 * (key_len & 3);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t off = i * rec;
    const uint32_t *w = src + (off >> 2);
    const uint32_t sh = 8 * (uint32_t)(off & 3);
    const uint32_t w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2), w3 = __ldg(w + 3);
    const uint32_t a[3] = {__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh)};
    const uint64_t key = (((uint64_t)a[1] << 32) | a[0]) & key_bytes_mask;
    dst[3 * i] = (uint32_t)key;
    dst[3 * i + 1] = (uint32_t)(key >> 32);
    dst[3 * i + 2] = __funnelshift_r(a[vw], a[vw + 1], vsh);
  }
}

void launch_widen_records(const uint8_t *narrow, uint64_t n_rec, uint32_t key_len, uint8_t *wide12, cudaStream_t stream) {
  if (!n_rec) return;
  int grid = (int)min((uint64_t)device_sm_count() * 8, (n_rec + 255) / 256);
  k_widen_records<<<grid, 256, 0, stream>>>(narrow, n_rec, key_len, wide12);
}
// one warp per sketch: byte-wise minimum of its 4096 registers
__global__ void __launch_bounds__(256) k_reg_floor(const uint8_t *__restrict__ regs, uint32_t n_sketch, uint8_t *__restrict__ floor) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < n_sketch; t += warps) {   // warp-uniform
    const uint4 *r = reinterpret_cast<const uint4 *>(regs + t * HLL_M);
    uint32_t m = 0xFFFFFFFFu;
    for (uint32_t i = lane; i < HLL_M / 16; i += 32) {
      const uint4 v = __ldcg(r + i);
      m = __vminu4(m, __vminu4(__vminu4(v.x, v.y), __vminu4(v.z, v.w)));
    }
    m = min(min(m & 0xFFu, (m >> 8) & 0xFFu), min((m >> 16) & 0xFFu, m >> 24));
    m = __reduce_min_sync(0xFFFFFFFFu, m);
    if (lane == 0) floor[t] = (uint8_t)m;
  }
}

void launch_reg_floor(const uint8_t *regs, uint32_t n_sketch, uint8_t *floor, cudaStream_t stream) {
  if (!n_sketch) return;
  k_reg_floor<<<min((n_sketch + 7) / 8, (uint32_t)device_sm_count() * 8), 256, 0, stream>>>(regs, n_sketch, floor);
}

void launch_register_histograms(const uint8_t *regs, uint32_t n_sketch, uint32_t *hist, cudaStream_t stream) {
  if (!n_sketch) return;
  k_register_histograms<<<min(n_sketch, (uint32_t)device_sm_count() * 16), 256, 0, stream>>>(regs, n_sketch, hist);
}
void launch_clade_max(const uint8_t *regs, const uint32_t *members, uint32_t n_members, uint8_t *out4096,
                      cudaStream_t stream) {
  k_clade_max<<<4, 256, 0, stream>>>(regs, members, n_members, out4096);
}
void launch_fill_u32(uint32_t *p, uint64_t n, uint32_t v, cudaStream_t stream) {
  if (!n) return;
  k_fill_u32<<<(int)min((uint64_t)device_sm_count() * 8, (n + 255) / 256), 256, 0, stream>>>(p, n, v);
}

// `taxon_counts[t] += other[t]` (classify.cpp:542-544) for the state of another context copied next to ours:
// registers max (hyperloglogplus.cpp:614-620), counters add (readcounts.hpp:76-88), dense anywhere = dense (:604-612)
__global__ void k_merge_state(uint32_t *regs, const uint32_t *regs2, uint64_t n_words, unsigned long long *n_kmers,
                              const unsigned long long *n_kmers2, uint32_t n_sketch, unsigned long long *n_reads,
                              const unsigned long long *n_reads2, uint32_t n_taxa, uint8_t *dense, const uint8_t *dense2) {
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = tid; i < n_words; i += nth) regs[i] = __vmaxu4(regs[i], regs2[i]);
  for (uint64_t i = tid; i < n_sketch; i += nth) { n_kmers[i] += n_kmers2[i]; dense[i] |= dense2[i]; }
  for (uint64_t i = tid; i < n_taxa; i += nth) n_reads[i] += n_reads2[i];
}
void launch_merge_state(uint8_t *regs, const uint8_t *regs2, unsigned long long *n_kmers, const unsigned long long *n_kmers2,
                        uint32_t n_sketch, unsigned long long *n_reads, const unsigned long long *n_reads2, uint32_t n_taxa,
                        uint8_t *dense, const uint8_t *dense2, cudaStream_t stream) {
  k_merge_state<<<device_sm_count() * 4, 256, 0, stream>>>(reinterpret_cast<uint32_t *>(regs), reinterpret_cast<const uint32_t *>(regs2),
                                             (uint64_t)n_sketch * (HLL_M / 4), n_kmers, n_kmers2, n_sketch, n_reads, n_reads2, n_taxa,
                                             dense, dense2);
}

// ------------------------------------------------------------------------------------------------------
// Cross-GPU step synchronisation without the host (database sharded by minimizer range, SURVEY.md §8(e).2).
// Flags are 64-bit counters in device memory every peer has mapped (CUDA IPC or peer access).  k_signal_peers runs
// in stream order after the work it announces: the kernel boundary has made that work's peer stores visible at
// system scope, the fence orders them before the flag stores.  k_wait_flags spins (one lane per flag) until every
// flag has reached `value`; a peer that died shows up as a timeout (error code 6), not as a hung GPU.
// ------------------------------------------------------------------------------------------------------
struct PeerFlags { unsigned long long *ptr[8]; };
__global__ void k_signal_peers(PeerFlags f, uint32_t n, uint32_t my_index, unsigned long long value) {
  if (threadIdx.x < n) {
    __threadfence_system();
    *reinterpret_cast<volatile unsigned long long *>(f.ptr[threadIdx.x] + my_index) = value;
    __threadfence_system();
  }
}
__global__ void k_wait_flags(const unsigned long long *flags, uint32_t n, unsigned long long value, unsigned long long timeout_ns,
                             uint32_t *error_flag) {
  if (threadIdx.x >= n) return;
  unsigned long long t0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  const volatile unsigned long long *f = flags + threadIdx.x;
  while (*f < value) {
    unsigned long long t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (t1 - t0 > timeout_ns) { atomicExch(error_flag, 6u); break; }
    __nanosleep(200);
  }
  __threadfence_system();
}
void launch_signal_peers(unsigned long long *const *flag_ptrs, uint32_t n, uint32_t my_index, unsigned long long value,
                         cudaStream_t stream) {
  PeerFlags f;
  for (uint32_t j = 0; j < 8; j++) f.ptr[j] = j < n ? flag_ptrs[j] : nullptr;
  k_signal_peers<<<1, 32, 0, stream>>>(f, n, my_index, value);
}
void launch_wait_flags(const unsigned long long *flags, uint32_t n, unsigned long long value, unsigned long long timeout_ns,
                       uint32_t *error_flag, cudaStream_t stream) {
  k_wait_flags<<<1, 32, 0, stream>>>(flags, n, value, timeout_ns, error_flag);
}

// Sparse-tier keys of the taxa that are still sparse, grouped by the rank that owns their CODE
// (part = hash(code) % n_parts): all keys that can ever be duplicates of each other — the same (taxon, code) seen on
// several GPUs, or the same code under two taxa of one clade — meet on one rank, so per-taxon distinct counts and
// clade unions are sums of per-rank results.  pass 0 counts (counts[part]), pass 1 scatters through cursors[part].
__device__ __forceinline__ uint32_t key_part(unsigned long long key, uint32_t n_parts) {
  return (uint32_t)((mix64((uint32_t)key) >> 33) % n_parts);
}
// Items grouped by owner part for the partitioned exports: pass 0 counts per part (counters[part]), pass 1 scatters
// through the per-part cursors counters[part], bounded by part_end.  Same-address atomics would serialise hundreds of
// millions of items on n_parts counters, so the items of a tile are counted / ranked on shared-memory counters (only real
// items touch them — most slots are empty and most records unflagged, and a per-part warp vote for every item made the
// kernel instruction bound), and only one thread per part and CTA touches the global cursor per tile.
// A source gives the item type, E items per thread and tile, P part counters, RANK_BITS of a tile rank (the part goes
// above them), the raw load of item i, the item it makes (an unoccupied one = none) and the item's owner.
constexpr int KP_E = 8;      // keys per thread and tile: four block-wide barriers per 2048 items instead of per 256
constexpr int XP_E = 4;      // pairs per thread and tile (16 B each)
struct SetKeyParts {         // the slots of the local sparse-tier set
  using Item = unsigned long long;
  using Raw = unsigned long long;
  static constexpr int E = KP_E, P = 8, RANK_BITS = 28;
  const unsigned long long *slots;
  const uint8_t *dense_flag;
  __device__ Raw load(uint64_t i) const { return __ldg(slots + i); }
  __device__ Item item(Raw k, uint64_t, int) const { return k && dense_flag[(uint32_t)(k >> 32) - 1] ? 0ull : k; }
  __device__ static uint32_t owner(Item k, uint32_t n_parts) { return key_part(k, n_parts); }
};
// the records a counted hit flagged and the kept records: pass 1 clears SEEN_BIT (the key leaves this GPU instead of
// entering its set); KEPT_BIT is dropped when the merged keys replace the set (kuq_sparse_replace)
struct RecordKeyParts {
  using Item = unsigned long long;
  using Raw = uint32_t;      // the record's high word
  static constexpr int E = KP_E, P = 8, RANK_BITS = 28;
  uint8_t *pairs;
  const uint8_t *dense_flag;
  uint32_t hi_mask;
  __device__ Raw load(uint64_t i) const { return __ldg(reinterpret_cast<const uint32_t *>(pairs + i * 12) + 1); }
  __device__ Item item(Raw hiw, uint64_t i, int pass) const {
    if (!(hiw & (SEEN_BIT | KEPT_BIT))) return 0ull;
    uint32_t *w = reinterpret_cast<uint32_t *>(pairs + i * 12);
    if (pass == 1 && (hiw & SEEN_BIT)) w[1] = hiw & ~SEEN_BIT;
    return dense_flag[w[2]] ? 0ull : record_key(w, hiw, hi_mask);
  }
  __device__ static uint32_t owner(Item k, uint32_t n_parts) { return key_part(k, n_parts); }
};
struct ExactPairParts {      // the slots of the exact k-mer set, owned by exact_owner of their k-mer
  using Item = ExactPair;
  using Raw = ExactPair;
  static constexpr int E = XP_E, P = EXACT_MAX_PARTS, RANK_BITS = 24;
  const ExactPair *slots;
  __device__ Raw load(uint64_t i) const { return slots[i]; }
  __device__ Item item(Raw pr, uint64_t, int) const { return pr; }
  __device__ static uint32_t owner(const Item &pr, uint32_t n_parts) { return exact_owner(pr.kmer1 - 1, n_parts); }
};

template <typename S>
__global__ void __launch_bounds__(256) k_parts(const S src, uint64_t lo, uint64_t hi, uint32_t n_parts, unsigned long long *counters,
                                               typename S::Item *out, const unsigned long long *part_end, uint32_t *error_flag,
                                               int pass) {
  __shared__ uint32_t s_cnt[S::P];               // pass 0: the CTA's items (far fewer than 2^32), pass 1: the tile's
  __shared__ unsigned long long s_base[S::P];
  constexpr uint32_t RANK_MASK = (1u << S::RANK_BITS) - 1;
  const uint32_t tid = threadIdx.x;
  if (tid < S::P) s_cnt[tid] = 0;
  __syncthreads();
  const uint64_t tile = (uint64_t)blockDim.x * S::E;
  for (uint64_t base = lo + (uint64_t)blockIdx.x * tile; base < hi; base += (uint64_t)gridDim.x * tile) {
    typename S::Raw raw[S::E];
    typename S::Item item[S::E];
    uint32_t where[S::E];                        // part << RANK_BITS | rank inside the tile's group of that part
    // all loads of the tile first (E independent requests per thread in flight: the scan is bandwidth work), then the
    // per-item arithmetic
#pragma unroll
    for (int j = 0; j < S::E; j++) {
      const uint64_t i = base + (uint64_t)j * blockDim.x + tid;
      raw[j] = typename S::Raw{};
      if (i < hi) raw[j] = src.load(i);
    }
#pragma unroll
    for (int j = 0; j < S::E; j++) {
      item[j] = src.item(raw[j], base + (uint64_t)j * blockDim.x + tid, pass);
      where[j] = 0;
      if (occupied(item[j])) {                   // only real items cost anything: one shared-memory atomic on the part's counter
        const uint32_t part = S::owner(item[j], n_parts);
        if (pass == 0) atomicAdd(&s_cnt[part], 1u);
        else where[j] = (part << S::RANK_BITS) | atomicAdd(&s_cnt[part], 1u);
      }
    }
    if (pass == 1) {
      __syncthreads();
      if (tid < n_parts && s_cnt[tid]) s_base[tid] = atomicAdd(counters + tid, (unsigned long long)s_cnt[tid]);
      __syncthreads();
#pragma unroll
      for (int j = 0; j < S::E; j++) {
        if (!occupied(item[j])) continue;
        const uint32_t part = where[j] >> S::RANK_BITS;
        const unsigned long long at = s_base[part] + (where[j] & RANK_MASK);
        if (at < part_end[part]) out[at] = item[j]; else atomicExch(error_flag, 7u);
      }
      __syncthreads();
      if (tid < S::P) s_cnt[tid] = 0;
      __syncthreads();
    }
  }
  if (pass == 0) {
    __syncthreads();
    if (tid < n_parts && s_cnt[tid]) atomicAdd(counters + tid, (unsigned long long)s_cnt[tid]);
  }
}
template <typename S>
void launch_parts(const S &src, uint64_t lo, uint64_t hi, uint32_t n_parts, unsigned long long *counters, typename S::Item *out,
                  const unsigned long long *part_end, uint32_t *error_flag, int pass, cudaStream_t stream) {
  if (hi <= lo) return;
  const int grid = (int)min((uint64_t)device_sm_count() * 8, (hi - lo + 256 * S::E - 1) / (256 * S::E));
  k_parts<<<grid, 256, 0, stream>>>(src, lo, hi, n_parts, counters, out, part_end, error_flag, pass);
}
void launch_keys_parts(int src, const unsigned long long *slots, uint8_t *pairs, uint64_t n_items, uint64_t key_mask,
                       const uint8_t *dense_flag, uint32_t n_parts, unsigned long long *counters, unsigned long long *out,
                       const unsigned long long *part_end, uint32_t *error_flag, int pass, cudaStream_t stream) {
  if (src == 0) launch_parts(SetKeyParts{slots, dense_flag}, 0, n_items, n_parts, counters, out, part_end, error_flag, pass, stream);
  else launch_parts(RecordKeyParts{pairs, dense_flag, (uint32_t)(key_mask >> 32)}, 0, n_items, n_parts, counters, out, part_end,
                    error_flag, pass, stream);
}
void launch_exact_parts(const ExactPair *slots, uint64_t lo, uint64_t hi, uint32_t n_parts, unsigned long long *counters,
                        ExactPair *out, const unsigned long long *part_end, uint32_t *error_flag, int pass, cudaStream_t stream) {
  launch_parts(ExactPairParts{slots}, lo, hi, n_parts, counters, out, part_end, error_flag, pass, stream);
}

}  // namespace kuq
