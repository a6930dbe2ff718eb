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

// Databases sharded over G GPUs by minimizer range (classify with one or several -d on a node whose GPUs hold them
// only together).  Consecutive databases with equal (nt, index type) form a run: their windows have the same bins, so
// one lookup launch asks them in order.  Each run gets ONE cut of its 4^nt bins into G ranges, balanced by the run's
// summed record counts, and every database of the run is staged with the same range on GPU g: a window's whole
// in-order search inside a run happens on one GPU.  A range may be empty (cut[g] == cut[g + 1]).  With one database the
// cut points are those of the lower bound of key_ct / G * g in its index.
struct ShardDb {
  const uint64_t *offsets;   // the index's 4^nt + 1 running record counts
  uint32_t nt, idx_type;
};
struct ShardRun {
  size_t first, end;                 // databases [first, end)
  std::vector<uint64_t> cut;         // G + 1 bin boundaries: GPU g holds [cut[g], cut[g + 1])
};
inline std::vector<ShardRun> plan_shards(const std::vector<ShardDb> &dbs, int G) {
  std::vector<ShardRun> runs;
  for (size_t i = 0; i < dbs.size();) {
    ShardRun r;
    r.first = i;
    while (i < dbs.size() && dbs[i].nt == dbs[r.first].nt && dbs[i].idx_type == dbs[r.first].idx_type) i++;
    r.end = i;
    const uint64_t n_bins = 1ull << (2 * dbs[r.first].nt);
    auto sum = [&](uint64_t b) {                      // records of the run in bins [0, b)
      uint64_t s = 0;
      for (size_t d = r.first; d < r.end; d++) s += dbs[d].offsets[b];
      return s;
    };
    const uint64_t total = sum(n_bins);
    r.cut.assign(G + 1, 0);
    r.cut[G] = n_bins;
    for (int g = 1; g < G; g++) {                     // first bin b < n_bins with sum(b) >= total / G * g, else n_bins
      const uint64_t want = total / G * g;
      uint64_t lo = 0, hi = n_bins;
      while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (sum(mid) < want) lo = mid + 1; else hi = mid;
      }
      r.cut[g] = lo;
    }
    for (int g = 1; g <= G; g++) if (r.cut[g] < r.cut[g - 1]) r.cut[g] = r.cut[g - 1];
    runs.push_back(std::move(r));
  }
  return runs;
}

#endif
