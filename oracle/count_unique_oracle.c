/* oracle/count_unique_oracle.c — CPU restatement of the reference's count_unique (src/count_unique.cpp:51-79), the
 * HyperLogLog estimate of a FASTA library's distinct k-mers that krakenuniq-build sizes Jellyfish's hash with.
 *
 * TEST INFRASTRUCTURE ONLY: tests/test_count_unique_{cpu,gpu}.py load it (libkuq_count_unique_oracle.so, built by
 * __graft_entry__.build()) as the checker of bin/count_unique and kuq_count_unique_*; nothing under krakenuniq_b200/
 * links or calls it.  Parity status: PINNED against recorded runs of the reference's own count_unique
 * (tests/golden/reference/test_count_unique_cpu.py_*.zip).  Citations are file:line under the reference's src/.
 *
 * It stands alone beside kuq_oracle.c, whose HLL is fixed at classify's precision 12: the finalizer and the Ertl
 * estimator are restated here for any precision 4..18. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

uint64_t kuqo_count_unique(const char *in, size_t n, unsigned k, unsigned p, uint8_t *regs, uint64_t *n_observed);

/* murmurhash3_finalizer, hyperloglogplus.cpp:830-838 */
static uint64_t fmix64(uint64_t key) {
  key += 1;
  key ^= key >> 33;
  key *= 0xff51afd7ed558ccdULL;
  key ^= key >> 33;
  key *= 0xc4ceb9fe1a85ec53ULL;
  key ^= key >> 33;
  return key;
}
/* sigma(), hyperloglogplus.cpp:373-387 */
static double ertl_sigma(double x) {
  if (x == 1.0) return INFINITY;
  double prev, sigma_x = x, y = 1.0;
  do {
    prev = sigma_x;
    x *= x;
    sigma_x += x * y;
    y += y;
  } while (sigma_x != prev);
  return sigma_x;
}
/* tau(), :408-422 */
static double ertl_tau(double x) {
  if (x == 0.0 || x == 1.0) return 0.0;
  double prev, y = 1.0, tau_x = 1 - x;
  do {
    prev = tau_x;
    x = sqrt(x);
    y /= 2.0;
    tau_x -= pow(1 - x, 2) * y;
  } while (tau_x != prev);
  return tau_x / 3.0;
}
/* the estimator body of ertlCardinality(), :738-752, given the histogram C[0..q+1] of m registers */
static uint64_t ertl_from_hist(const int *C, size_t q, size_t m, uint64_t n_observed) {
  double est_denominator = m * ertl_tau(1.0 - (double)C[q + 1] / (double)m);
  for (int k = (int)q; k >= 1; --k) {
    est_denominator += C[k];
    est_denominator *= 0.5;
  }
  est_denominator += m * ertl_sigma((double)C[0] / (double)m);
  double m_sq_alpha_inf = (m / (2.0 * log(2))) * m;
  double est = m_sq_alpha_inf / est_denominator;
  return ((double)n_observed < est) ? n_observed : (uint64_t)round(est);
}
/* insert() of a dense HyperLogLogPlusMinus at precision p (hyperloglogplus.cpp:485-523) */
static void cu_insert(uint8_t *M, unsigned p, uint64_t kmer) {
  const uint64_t h = fmix64(kmer);
  const uint64_t w = h << p;
  const uint8_t rank = w ? (uint8_t)(__builtin_clzll(w) + 1) : (uint8_t)(64 - p + 1);
  if (rank > M[h >> (64 - p)]) M[h >> (64 - p)] = rank;
}
/* KmerScanner(seq, pos1, pos2) and next_kmer() until NULL (krakenutil.cpp:208-282) over one piece, every unambiguous
 * k-mer inserted; returns their number.  A call starts only while curr_pos < pos2 but reads on until k bases are loaded,
 * into the next piece, and at the end of the sequence onto std::string's '\0'; reads past that (undefined in the
 * reference) see '\0' too. */
static uint64_t cu_piece(const char *seq, size_t len, size_t pos1, size_t pos2, unsigned k, unsigned p, uint8_t *M) {
  const uint64_t kmer_mask = ~0ull >> (64 - 2 * k);
  const uint32_t mini_kmer_mask = ~0u >> (32 - k);
  size_t curr_pos = pos1;
  if (pos2 - pos1 + 1 < k) curr_pos = pos2;               /* :216-217 */
  int64_t loaded_nt = 0;
  uint64_t kmer = 0, n = 0;
  uint32_t ambig = 0;
  while (curr_pos < pos2) {
    int skip_pos = 0;
    if (loaded_nt) loaded_nt--;
    while (loaded_nt < (int64_t)k) {
      if (skip_pos) {
        skip_pos = 0;
      } else {
        loaded_nt++;
        kmer <<= 2;
        ambig <<= 1;
      }
      char c = curr_pos < len ? seq[curr_pos] : '\0';
      curr_pos++;
      switch (c) {
        case 'A': case 'a': break;
        case 'C': case 'c': kmer |= 1; break;
        case 'G': case 'g': kmer |= 2; break;
        case 'T': case 't': kmer |= 3; break;
        case '\n': case '\r':
          --loaded_nt;
          skip_pos = 1;
          continue;
        default: ambig |= 1; break;
      }
      kmer &= kmer_mask;
      ambig &= mini_kmer_mask;
    }
    if (!ambig) {                                           /* count_unique.cpp:69-71 */
      cu_insert(M, p, kmer);
      n++;
    }
  }
  return n;
}
static void cu_sequence(const char *seq, size_t len, unsigned k, unsigned p, uint8_t *M, uint64_t *n_observed) {
  for (size_t i = 0; i < len; i += 50000) {               /* SKIP_LEN, :26,62-64 */
    size_t end = i + 50000 + k - 1;
    *n_observed += cu_piece(seq, len, i, end < len ? end : len, k, p, M);
  }
}
/* count_unique over the bytes of its stdin, plain FASTA: every sequence in pieces of 50000 + k - 1 bases stepping by
 * 50000, a fresh KmerScanner per piece, every unambiguous forward k-mer into a dense HyperLogLog of 2^p registers
 * (p = 4..18), pieces merged by register max.  Returns the printed estimate (ertlCardinality at p, 0 without a valid
 * window); regs (optional) = 2^p registers, *n_observed (optional) = valid windows. */
uint64_t kuqo_count_unique(const char *in, size_t n, unsigned k, unsigned p, uint8_t *regs, uint64_t *n_observed) {
  const size_t m = (size_t)1 << p;
  uint8_t *M = (uint8_t *)calloc(m, 1);
  uint64_t n_obs = 0;
  char *seq = (char *)malloc(n + 1);
  size_t seq_len = 0;
  int open = 0;
  /* FastaReader::next_sequence (seqreader.cpp:34-79): the first line must start with '>' */
  for (size_t pos = 0, line_no = 0; pos < n || line_no == 0; line_no++) {
    const char *nl = pos < n ? (const char *)memchr(in + pos, '\n', n - pos) : NULL;
    const size_t end = nl ? (size_t)(nl - in) : n;
    const char *line = in + pos;
    const size_t ll = end - pos;
    if (ll && line[0] == '>') {
      if (open) cu_sequence(seq, seq_len, k, p, M, &n_obs);
      open = 1;
      seq_len = 0;
    } else if (line_no == 0) {
      break;                                                /* "malformed fasta file - expected header char > not found" */
    } else {
      memcpy(seq + seq_len, line, ll);
      seq_len += ll;
    }
    pos = nl ? end + 1 : n;
    if (!nl) break;
  }
  if (open) cu_sequence(seq, seq_len, k, p, M, &n_obs);
  free(seq);
  uint64_t est = 0;
  if (n_obs) {                                              /* else the main counter stays sparse and empty: 0 */
    int C[64 + 2];
    memset(C, 0, sizeof(C));
    for (size_t i = 0; i < m; i++) ++C[M[i]];
    est = ertl_from_hist(C, 64 - p, m, n_obs);
  }
  if (regs) memcpy(regs, M, m);
  if (n_observed) *n_observed = n_obs;
  free(M);
  return est;
}
