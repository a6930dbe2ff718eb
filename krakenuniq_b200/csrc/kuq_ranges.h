// How a database's minimizer bins are cut into ranges that fit a byte budget, for every tool that holds one range of
// records at a time: classify -x (prepare_chunking / upper_bound, krakendb.cpp:430-522), set_lcas and db_sort's
// per-range sorts.  Any partition gives the same results: a key lives in one bin.
#ifndef KUQ_RANGES_H
#define KUQ_RANGES_H
#include <stdint.h>

#include <utility>
#include <vector>

// Ranges [lo, hi) of the n_bins bins of `offsets` (the index's n_bins + 1 running record counts), each as long as its
// index slice ((hi - lo + 1) * 8 bytes) plus its records (rec_bytes each) plus 8 bytes fit `budget`.  Ranges without
// records are left out (:496-499).  Returns false when a single bin does not fit.
inline bool plan_ranges(const uint64_t *offsets, uint64_t n_bins, uint64_t budget, uint64_t rec_bytes,
                        std::vector<std::pair<uint64_t, uint64_t>> &ranges) {
  ranges.clear();
  uint64_t first = 0;
  while (first < n_bins) {
    auto fits = [&](uint64_t end) { return (end - first + 1) * 8 + (offsets[end] - offsets[first]) * rec_bytes + 8 <= budget; };
    if (!fits(first + 1)) return false;
    uint64_t lo = first + 1, hi = n_bins;             // largest `end` in (first, n_bins] that still fits
    while (lo < hi) {
      const uint64_t mid = lo + (hi - lo + 1) / 2;
      if (fits(mid)) lo = mid; else hi = mid - 1;
    }
    if (offsets[lo] > offsets[first]) ranges.emplace_back(first, lo);
    first = lo;
  }
  return true;
}

#endif
