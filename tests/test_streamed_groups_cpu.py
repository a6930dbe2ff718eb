"""kuq_ranges.h's plan for databases streamed over several GPUs, compiled for the host: each database's ranges
(plan_ranges) grouped per GPU by the bytes they copy (group_ranges / split_balanced), the device memory a round of reads gets on
the tightest context (stream_round_bytes), and the owners of a round's batches with the round's peak bytes on one GPU
(round_peak_bytes)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "krakenuniq_b200", "csrc", "kuq_ranges.h")
GiB = 1 << 30

SHIM = r'''
#include "%s"
extern "C" int plan_and_group(const uint64_t *offsets, uint64_t n_bins, uint64_t budget, int G, uint64_t *ranges_out,
                              uint64_t *n_ranges, uint64_t *first_out) {
  std::vector<std::pair<uint64_t, uint64_t>> ranges;
  if (!plan_ranges(offsets, n_bins, budget, 12, ranges)) return -1;
  *n_ranges = ranges.size();
  for (size_t i = 0; i < ranges.size(); i++) { ranges_out[2 * i] = ranges[i].first; ranges_out[2 * i + 1] = ranges[i].second; }
  const std::vector<size_t> first = group_ranges(offsets, ranges, G, 12);
  for (int g = 0; g <= G; g++) first_out[g] = first[g];
  return 0;
}
extern "C" void split(const uint64_t *w, size_t n, int G, uint64_t *first_out) {
  const std::vector<size_t> first = split_balanced(std::vector<uint64_t>(w, w + n), G);
  for (int g = 0; g <= G; g++) first_out[g] = first[g];
}
extern "C" uint64_t round_bytes(const int *device, const uint64_t *free_b, size_t n, uint64_t budget, uint64_t range_bytes) {
  return stream_round_bytes(std::vector<int>(device, device + n), std::vector<uint64_t>(free_b, free_b + n), budget, range_bytes);
}
extern "C" uint64_t peak(const uint64_t *bases, const uint64_t *reads, size_t n, int unit_rule, int G, uint64_t *first_out) {
  std::vector<size_t> first;
  const uint64_t p = round_peak_bytes(std::vector<uint64_t>(bases, bases + n), std::vector<uint64_t>(reads, reads + n),
                                      unit_rule != 0, G, &first);
  for (int g = 0; g <= G; g++) first_out[g] = first[g];
  return p;
}
extern "C" uint64_t shared_bytes(uint64_t bases, uint64_t reads, int unit_rule) { return batch_shared_bytes(bases, reads, unit_rule); }
extern "C" uint64_t id_bytes(uint64_t bases) { return batch_id_bytes(bases); }
'''

P = ctypes.c_void_p


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("ranges")
    (d / "r.cpp").write_text(SHIM % HDR)
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", str(d / "r.cpp"), "-o", str(d / "r.so")],
                   check=True)
    L = ctypes.CDLL(str(d / "r.so"))
    L.round_bytes.restype = ctypes.c_uint64
    L.peak.restype = ctypes.c_uint64
    L.shared_bytes.restype = ctypes.c_uint64
    L.id_bytes.restype = ctypes.c_uint64
    return L


def split(lib, w, G):
    w = np.asarray(w, np.uint64)
    first = np.zeros(G + 1, np.uint64)
    lib.split(P(w.ctypes.data), ctypes.c_size_t(len(w)), G, P(first.ctypes.data))
    return first.astype(int).tolist()


def plan_and_group(lib, counts, budget, G):
    """counts: records per bin.  Returns (ranges, first)"""
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
    n_bins = len(counts)
    ranges = np.zeros(2 * n_bins + 2, np.uint64)
    n = np.zeros(1, np.uint64)
    first = np.zeros(G + 1, np.uint64)
    rc = lib.plan_and_group(P(offsets.ctypes.data), ctypes.c_uint64(n_bins), ctypes.c_uint64(budget), G, P(ranges.ctypes.data),
                            P(n.ctypes.data), P(first.ctypes.data))
    assert rc == 0
    k = int(n[0])
    return [(int(ranges[2 * i]), int(ranges[2 * i + 1])) for i in range(k)], first.astype(int).tolist(), offsets


def check_groups(first, weights, G):
    """every item in exactly one group, in order, groups contiguous, none heavier than total / G + the heaviest item"""
    n = len(weights)
    assert len(first) == G + 1 and first[0] == 0 and first[G] == n
    assert all(first[g] <= first[g + 1] for g in range(G))
    owner = [g for g in range(G) for _ in range(first[g], first[g + 1])]
    assert owner == sorted(owner) and len(owner) == n
    total, heaviest = sum(weights), max(weights, default=0)
    for g in range(G):
        assert sum(weights[first[g]:first[g + 1]]) <= total / G + heaviest, (g, first, weights)


@pytest.mark.parametrize("G", [1, 2, 3, 4, 7, 8])
def test_groups_of_planned_ranges(lib, G):
    rng = np.random.default_rng(G)
    for trial in range(20):
        counts = rng.integers(0, 50, int(rng.integers(1, 400)))
        counts[rng.random(len(counts)) < 0.3] = 0                 # empty bins, which no range keeps alone
        if counts.sum() == 0:
            counts[0] = 1
        budget = int(rng.integers(60 * 12, 3000 * 12))
        ranges, first, offsets = plan_and_group(lib, counts, budget, G)
        recs = [int(offsets[hi] - offsets[lo]) for lo, hi in ranges]
        assert all(r > 0 for r in recs)
        copied = [(hi - lo + 1) * 8 + r * 12 + 8 for (lo, hi), r in zip(ranges, recs)]
        # the ranges are plan_ranges' whatever G: the bins in order, each range within the budget
        assert all(ranges[i][1] <= ranges[i + 1][0] for i in range(len(ranges) - 1))
        for (lo, hi), r in zip(ranges, recs):
            assert (hi - lo + 1) * 8 + r * 12 + 8 <= budget
        check_groups(first, copied, G)
        if G == 1:
            assert first == [0, len(ranges)]


def test_one_gpu_is_one_group(lib):
    for w in ([5], [1, 2, 3], [0, 0, 9], [7] * 100):
        assert split(lib, w, 1) == [0, len(w)]


def test_more_gpus_than_ranges_leaves_groups_empty(lib):
    for w in ([4], [1, 1], [3, 1, 2]):
        for G in (len(w) + 1, len(w) + 3, 8):
            first = split(lib, w, G)
            check_groups(first, w, G)
            sizes = [first[g + 1] - first[g] for g in range(G)]
            assert sizes.count(0) >= G - len(w) and sum(sizes) == len(w)
    _, first, _ = plan_and_group(lib, [10, 10], 10 * 12 + 8 * 2 + 8, 3)   # one range per bin, three GPUs
    assert [first[g + 1] - first[g] for g in range(3)] == [1, 0, 1]


def test_balance_examples(lib):
    assert split(lib, [1] * 8, 2) == [0, 4, 8]
    assert split(lib, [1] * 8, 3) == [0, 3, 5, 8]
    assert split(lib, [10, 1, 1, 1, 1], 2) == [0, 1, 5]
    assert split(lib, [1, 1, 1, 1, 10], 2) == [0, 4, 5]
    assert split(lib, [], 3) == [0, 0, 0, 0]
    assert split(lib, [0, 0, 0], 2) == [0, 0, 3]
    rng = np.random.default_rng(1)
    for _ in range(200):
        w = rng.integers(0, 1000, int(rng.integers(0, 40))).tolist()
        G = int(rng.integers(1, 9))
        check_groups(split(lib, w, G), w, G)


def round_bytes(lib, devices, free, budget, range_bytes):
    d = np.asarray(devices, np.int32)
    f = np.asarray(free, np.uint64)
    return int(lib.round_bytes(P(d.ctypes.data), P(f.ctypes.data), ctypes.c_size_t(len(d)), ctypes.c_uint64(budget),
                               ctypes.c_uint64(range_bytes)))


def test_round_bytes_one_context_is_the_one_gpu_figure(lib):
    for free, budget, rb in ((80 * GiB, 60 * GiB, 30 * GiB), (40 * GiB, 60 * GiB, 10 * GiB), (GiB, 60 * GiB, 100),
                             (80 * GiB, 200000, 108000), (80 * GiB, 200000, 300000)):
        cap = min(budget, free - 2 * GiB if free > 2 * GiB else 0)
        assert round_bytes(lib, [0], [free], budget, rb) == (cap - rb if cap > rb else 0)


def test_round_bytes_contexts_sharing_a_device(lib):
    # three contexts on device 0 split its free memory: each share is (free - 2 GiB) / 3
    free = 80 * GiB
    share = (free - 2 * GiB) // 3
    assert round_bytes(lib, [0, 0, 0], [free] * 3, 60 * GiB, 10 * GiB) == share - 10 * GiB
    # a small budget stays the cap
    assert round_bytes(lib, [0, 0], [free] * 2, 200000, 100000) == 100000
    # two cards, the second with less free memory: the tightest context decides
    assert round_bytes(lib, [0, 1], [80 * GiB, 30 * GiB], 60 * GiB, 10 * GiB) == 28 * GiB - 10 * GiB
    # device 0 shared by two contexts, device 1 alone
    assert round_bytes(lib, [0, 0, 1], [80 * GiB, 80 * GiB, 80 * GiB], 60 * GiB, GiB) == 39 * GiB - GiB
    # range buffers larger than a share: no room for reads
    assert round_bytes(lib, [0, 0], [10 * GiB] * 2, 60 * GiB, 5 * GiB) == 0


def peak(lib, bases, reads, unit_rule, G):
    b = np.asarray(bases, np.uint64)
    r = np.asarray(reads, np.uint64)
    first = np.zeros(G + 1, np.uint64)
    p = lib.peak(P(b.ctypes.data), P(r.ctypes.data), ctypes.c_size_t(len(b)), int(unit_rule), G, P(first.ctypes.data))
    return int(p), first.astype(int).tolist()


def test_round_peak(lib):
    rng = np.random.default_rng(3)
    for _ in range(100):
        n = int(rng.integers(1, 12))
        bases = rng.integers(0, 100000, n).tolist()
        reads = [b // 150 + 1 for b in bases]
        unit_rule = bool(rng.integers(0, 2))
        G = int(rng.integers(1, 5))
        p, first = peak(lib, bases, reads, unit_rule, G)
        check_groups(first, bases, G)
        shared = sum(int(lib.shared_bytes(ctypes.c_uint64(b), ctypes.c_uint64(r), int(unit_rule))) for b, r in zip(bases, reads))
        want = max(shared + sum(int(lib.id_bytes(ctypes.c_uint64(bases[i]))) for i in range(first[g], first[g + 1]))
                   for g in range(G))
        assert p == want
        if G == 1:
            # one GPU: the sum of the one-GPU figure (5 B per base + 8 or 12 per read + 1 KiB per batch)
            assert p == sum((b + 64) * 5 + (r + 4) * (12 if unit_rule else 8) + 1024 for b, r in zip(bases, reads))
    # two batches of one 20 kbp unit on two GPUs: one each, and each GPU holds both batches' bases but one id buffer
    p, first = peak(lib, [20000, 20000], [134, 134], True, 2)
    assert first == [0, 1, 2]
    assert p == 2 * (20064 + 138 * 12 + 1024) + 20064 * 4
