// kuq_kmerpack.cuh — a FASTA library staged on the device as KmerScanner reads it, shared by the k-mer set of
// build_db.sh step 1 (kuq_kmerset.cu) and count_unique's HyperLogLog sketch (kuq_countunique.cu).
//
// Sequences go into pinned batches of bases (two, so the host fills one while the device packs the other).  A batch is
// staged as 2-bit codes and a non-ACGT mask per 32 positions (k_ks_pack), sequence starts (with the end of the text)
// and the starts of the windows the scanner skips after a '\n' / '\r' (k_ks_mark).  A window is one the scanner yields
// when ks_window_ok holds; each consumer launches its own kernel over the staged blocks between stage() and next().
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <vector>

#include "kuq_buffers.cuh"

namespace kuq {

// bit of position pos[i] (relative to the batch) in mask[], i < n
__global__ void k_ks_mark(const uint64_t *pos, uint32_t n, uint32_t *mask);
// 2-bit codes and the non-ACGT mask of the 32-position blocks [0, nb]; positions at or past len are ambiguous.
// text: 16-byte aligned with 16 bytes of slack.
__global__ void __launch_bounds__(256) k_ks_pack(const char *text, uint64_t len, uint64_t nb, uint64_t *codes, uint32_t *amb);

// The window starting at position 32j + lane is valid when its k bases are ACGT, no sequence starts inside
// (32j + lane, 32j + lane + k) — packed_window's rule — and the scanner does not skip it (drop, or nullptr).
__device__ __forceinline__ bool ks_window_ok(const uint32_t *amb, const uint32_t *start, const uint32_t *drop, uint64_t j,
                                             uint32_t lane, uint32_t k) {
  const uint64_t kmask = (1ull << k) - 1, smask = (1ull << (k - 1)) - 1;
  const uint64_t amb64 = ((uint64_t)amb[j + 1] << 32) | amb[j];
  const uint64_t st64 = ((uint64_t)start[j + 1] << 32) | start[j];
  return !((amb64 >> lane) & kmask) && !((st64 >> (lane + 1)) & smask) && !(drop && ((drop[j] >> lane) & 1u));
}

// Starts of the windows KmerScanner::next_kmer (krakenutil.cpp:239-278) never yields over s[0, len) when s holds a
// '\n' or '\r': the scanner leaves such a character out of the k-mer but then loads the next base without counting it,
// and each further one of a run uncounts one more, so one window per such character is never produced.  clean = s
// without the line breaks, drop_ends = the clean positions where a skipped window ends.
void ks_scanner_skips(const char *s, uint64_t len, uint32_t k, std::vector<char> &clean, std::vector<uint64_t> &drop_ends);

// The batches.  add_* copy bases into the open batch; when it is full, `flush` (the consumer's: stage, its kernel,
// next) runs, and a sequence that did not fit continues in the next batch after its last k - 1 bases.
struct KsStager {
  uint32_t k = 0;
  uint64_t batch_cap = 0, max_seqs = 0;
  int n_sm = 0;
  std::function<int()> flush;
  HostBuf<char> h_text[2];
  HostBuf<uint64_t> h_offs[2];
  Event staged[2];
  int cur = 0;
  uint64_t fill = 0, seq_start = 0;
  uint32_t n_seqs = 0;
  std::vector<char> carry, clean;
  std::vector<uint64_t> drops, drop_ends;          // starts (in the batch) / ends (in `clean`) of windows the scanner skips
  DevBuf<char> d_text;
  DevBuf<uint64_t> d_offs, d_codes, d_drops;
  DevBuf<uint32_t> d_amb, d_start, d_drop;
  uint64_t drop_cap = 0;
  // what stage() packed: text length, blocks, and whether d_drop holds skipped windows
  uint64_t len = 0, nb = 0;
  bool has_drops = false;

  // buffers for batches of batch_cap bases and max_seqs sequences on the current device
  cudaError_t init(uint32_t k_, uint64_t batch_cap_, uint64_t max_seqs_);
  void release_device();                           // frees the device and pinned buffers (after the last flush)
  // the sequence s[0, len) as KmerScanner reads it over its whole length (kuq_kmer_set_add's sequences)
  int add_sequence(const char *s, uint64_t len);
  // one sequence given as its bases without line breaks and the clean positions where skipped windows end
  int add_clean(const char *clean_bases, uint64_t len, const std::vector<uint64_t> &ends);
  // true when the open batch cannot take another sequence
  bool full() const { return n_seqs + 1 >= max_seqs || fill == batch_cap; }
  bool empty() const { return n_seqs == 0; }
  // the open batch → codes / amb / start (/ drop) on the device, asynchronously on st
  cudaError_t stage(cudaStream_t st);
  // the other staging buffer is filled next: waits for its copy
  cudaError_t next();

 private:
  int append(const char *p, uint64_t n);
  void close_piece();
};

}  // namespace kuq
