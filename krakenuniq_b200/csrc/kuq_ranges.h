// How a database's minimizer bins are cut into ranges that fit a byte budget, for every tool that holds one range of
// records at a time: classify -x (prepare_chunking / upper_bound, krakendb.cpp:430-522), set_lcas and db_sort's
// per-range sorts.  Any partition gives the same results: a key lives in one bin.  Also how those ranges, and a round of
// read batches, are shared among the GPUs that stream them.
#ifndef KUQ_RANGES_H
#define KUQ_RANGES_H
#include <stdint.h>

#include <algorithm>
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

// ---- databases streamed over the G GPUs of a node (classify when the databases fit neither one card nor the cards
// together): every database keeps its plan_ranges cut, and GPU g streams a contiguous group of its ranges.

// G + 1 item indices: group g is items [first[g], first[g + 1]), contiguous and in order, balanced by weight.  Cut g lies
// at the item boundary nearest to total * g / G (never before cut g - 1), so it misses that point by at most half an
// item, and no group weighs more than total / G plus its heaviest item.  Groups may be empty (more groups than items,
// or a heavy item).
inline std::vector<size_t> split_balanced(const std::vector<uint64_t> &weight, int G) {
  typedef unsigned __int128 u128;                     // weights times G, compared with total * g
  const size_t n = weight.size();
  uint64_t total = 0;
  for (uint64_t w : weight) total += w;
  std::vector<size_t> first(G + 1, n);
  first[0] = 0;
  uint64_t before = 0;                                // weight of items [0, i)
  size_t i = 0;
  for (int g = 1; g < G; g++) {
    const u128 target = (u128)total * (unsigned)g;
    while (i < n && (u128)before * (unsigned)G < target) before += weight[i++];
    if (i > first[g - 1] && target - (u128)(before - weight[i - 1]) * (unsigned)G < (u128)before * (unsigned)G - target)
      before -= weight[--i];                          // the boundary before the last item is nearer
    first[g] = i;
  }
  return first;
}

// Ranges of one database for each of G GPUs: G + 1 indices into `ranges`, balanced by what each range copies to the
// device, its records (rec_bytes each) and its index slice, as plan_ranges counts them.  Record counts alone are not
// enough: minimizer bins of small value hold many records, so the first ranges have few bins and many records and the
// last ones the reverse, and on a database whose index outweighs its records a GPU with one range copied 3.5 times as
// long as the GPU with the other six.
inline std::vector<size_t> group_ranges(const uint64_t *offsets, const std::vector<std::pair<uint64_t, uint64_t>> &ranges, int G,
                                        uint64_t rec_bytes) {
  std::vector<uint64_t> bytes;
  for (auto &r : ranges) bytes.push_back((r.second - r.first + 1) * 8 + (offsets[r.second] - offsets[r.first]) * rec_bytes + 8);
  return split_balanced(bytes, G);
}

// Device memory a context may give one round of reads.  A device's free memory, less 2 GiB of headroom, is split evenly
// among the contexts on it (several contexts may share a card); each share is capped at the HBM budget, and the context's
// two range buffers come out of it.  A round has to fit every context, so it gets the tightest one's bytes.  With one
// context this is min(budget, free - 2 GiB) - range buffers.
inline uint64_t stream_round_bytes(const std::vector<int> &device, const std::vector<uint64_t> &free_bytes, uint64_t hbm_budget,
                                   uint64_t range_bytes) {
  uint64_t round = UINT64_MAX;
  for (size_t g = 0; g < device.size(); g++) {
    uint64_t sharing = 0;
    for (int d : device) sharing += d == device[g];
    const uint64_t fr = free_bytes[g] > (2ull << 30) ? free_bytes[g] - (2ull << 30) : 0;
    const uint64_t cap = std::min<uint64_t>(hbm_budget, fr / sharing);
    round = std::min<uint64_t>(round, cap > range_bytes ? cap - range_bytes : 0);
  }
  return round;
}

// What a round's batch takes on the device: every GPU holds its bases, offsets and (unit rule) unit ids, and its owner
// alone the 4 B per base of merged window ids.  The two add up to the one-GPU figure (5 B per base + 8 or 12 per read).
inline uint64_t batch_shared_bytes(uint64_t bases, uint64_t reads, bool unit_rule) {
  return (bases + 64) + (reads + 4) * (unit_rule ? 12 : 8) + 1024;
}
inline uint64_t batch_id_bytes(uint64_t bases) { return (bases + 64) * 4; }

// The owners of a round's batches: contiguous blocks balanced by bases (G + 1 batch indices, split_balanced), and the
// most device memory the round then takes on one GPU.
inline uint64_t round_peak_bytes(const std::vector<uint64_t> &bases, const std::vector<uint64_t> &reads, bool unit_rule, int G,
                                 std::vector<size_t> *owners = nullptr) {
  const std::vector<size_t> first = split_balanced(bases, G);
  uint64_t shared = 0, peak = 0;
  for (size_t b = 0; b < bases.size(); b++) shared += batch_shared_bytes(bases[b], reads[b], unit_rule);
  for (int g = 0; g < G; g++) {
    uint64_t ids = 0;
    for (size_t b = first[g]; b < first[g + 1]; b++) ids += batch_id_bytes(bases[b]);
    peak = std::max(peak, shared + ids);
  }
  if (owners) *owners = first;
  return peak;
}

#endif
