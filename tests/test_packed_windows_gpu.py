"""The fused call computes its windows inside the lookup kernel from a 2-bit packed copy of the batch; the lookup and
resolve halves still scan into per-window scratch.  On the same stress batch both must give the same per-window codes,
calls, window counts, hit lists, HLL registers, counters and sparse-tier readouts — for k = 31 (m = 15, the kernels'
specialised arithmetic) and generic k, both index types and every HLL rule, with reads holding '\\n' / '\\r', runs of N,
lowercase bases, lengths around k, a read longer than a shared-memory stage of the scan, a batch whose first offset
is not 0 and reads starting at every position mod 32."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from krakenuniq_b200 import binding, synth  # noqa: E402
from krakenuniq_b200 import dist as kdist  # noqa: E402
from tests import util  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _view(ptr, n, dtype=torch.int32):
    if n == 0:
        return np.zeros(0, np.uint32 if dtype == torch.int32 else np.uint64)
    a = kdist.device_view(ptr, n * (4 if dtype == torch.int32 else 8), dtype, DEV).cpu().numpy()
    return a.view(np.uint32 if dtype == torch.int32 else np.uint64).copy()


def _run(path, kdb, idx, tax, bases, offs, first, hll_mode, unit):
    """classify reads [first, n) of (bases, offs) — device buffers, offsets slice starting at offs[first] — through
    the fused call or through the two halves; returns everything the run exposes"""
    n = len(offs) - 1 - first
    total = int(offs[-1])
    d_bases = torch.from_numpy(np.concatenate([bases, np.full(64, ord("N"), np.uint8)])).to(DEV)
    d_offs = torch.from_numpy(np.concatenate([offs, offs[-1:]]).astype(np.int64)).to(DEV)
    units, _, _ = synth.work_unit_ids(offs[first:] - offs[first], unit)
    d_unit = torch.from_numpy(units.astype(np.int32)).to(DEV)
    clf = binding.Classifier(device=0, n_slots=1, max_reads=1 << 14, max_bases=1 << 22, hll_mode=hll_mode,
                             work_unit_size=unit, sparse_set_slots=1 << 22)
    try:
        clf.stage_db(kdb, idx)
        clf.set_taxonomy(*tax.parent_map())
        off_ptr = d_offs.data_ptr() + 8 * first
        if path == "fused":
            clf.classify_device(0, d_bases.data_ptr(), off_ptr, n, total, d_unit.data_ptr(), flags=binding.F_WANT_CODES)
        else:
            d_codes = torch.zeros(total + 64, dtype=torch.int32, device=DEV)
            clf.lookup_device(0, d_bases.data_ptr(), off_ptr, n, total, d_codes.data_ptr())
            clf.resolve_device(0, d_bases.data_ptr(), off_ptr, n, total, d_codes.data_ptr(), d_unit.data_ptr(),
                               flags=binding.F_WANT_CODES)
        clf.sync(0)
        r = clf.device_result(0)
        out = dict(call=_view(r.d_call, n), n_windows=_view(r.d_n_windows, n))
        codes = _view(r.d_codes, total)
        out["codes"] = [codes[int(offs[first + i]):int(offs[first + i]) + int(out["n_windows"][i])] for i in range(n)]
        n_runs = int(_view(r.d_n_runs, 1, torch.int64)[0])
        runs = _view(r.d_runs, 2 * n_runs).reshape(-1, 2)
        start, count = _view(r.d_run_start, n), _view(r.d_run_count, n)
        out["runs"] = [runs[int(start[i]):int(start[i]) + int(count[i])] for i in range(n)]   # block order may differ
        clf.finish()
        out["counts"] = clf.counts()
        out["regs"] = {int(t): clf.registers(int(t)) for t in out["counts"]["taxid"]}
        members = util.clade_members(tax.rows, out["counts"]["taxid"])
        out["clades"] = {t: clf.clade(m) for t, m in sorted(members.items())}
        return out
    finally:
        clf.close()


def _same(a, b):
    assert np.array_equal(a["call"], b["call"])
    assert np.array_equal(a["n_windows"], b["n_windows"])
    for i, (x, y) in enumerate(zip(a["codes"], b["codes"])):
        assert np.array_equal(x, y), f"codes of read {i}"
    for i, (x, y) in enumerate(zip(a["runs"], b["runs"])):
        assert np.array_equal(x, y), f"hit list of read {i}"
    for key in ("taxid", "n_reads", "n_kmers", "unique", "sparse"):
        assert np.array_equal(a["counts"][key], b["counts"][key]), key
    for t, regs in a["regs"].items():
        assert np.array_equal(regs, b["regs"][t]), f"registers of taxon {t}"
    assert a["clades"] == b["clades"]


def _stress_batch(rng, genomes, k):
    g = [synth.decode(x).tobytes() for x in genomes]
    crlf = [g[0][50:200] + b"\r", g[0][50:110] + b"\r\n" + g[0][110:170] + b"\r\n", g[0][50:80] + b"\r", b"\r" * 40,
            g[3][7:7 + k] + b"\r\r\r", g[4][0:300] + b"\n" + g[4][300:600].lower(), g[2][0:k - 1] + b"\r" + g[2][k:k + 5]]
    long_read = b"".join(g[i % len(g)][s:s + 500] for i, s in enumerate(rng.integers(0, len(g[0]) - 500, 60).tolist()))
    assert len(long_read) > 24 * 1024
    edge = [b"", b"A", g[0][:k - 1], g[0][:k], g[0][:k + 1], g[1][100:400].lower(), g[1][0:60] + b"N" * 40 + g[1][60:200],
            g[2][10:130] + b"nnnn" + g[3][10:130].lower(), b"N" * 200, long_read, g[1][5:5 + k].lower() + b"N" + g[1][40:40 + k]]
    sampled, soffs = synth.sample_reads(rng, genomes, 600, 150, 0.01, 0.2, 0.2)
    seqs = [sampled[int(soffs[i]):int(soffs[i + 1])].tobytes() for i in range(len(soffs) - 1)]
    # reads of many lengths: their starts fall on every position mod 32
    seqs += [g[i % len(g)][s:s + ln] for i, (s, ln) in enumerate(zip(rng.integers(0, 2000, 400).tolist(),
                                                                     rng.integers(1, 300, 400).tolist()))]
    for s in edge + crlf[1:-1]:
        seqs.insert(int(rng.integers(0, len(seqs))), s)
    # two reads that the device never sees, then a CRLF read first and one last: the batch's first offset is not 0
    seqs = [b"ACGT" * 5, b"TTG"] + [crlf[0]] + seqs + [crlf[-1]]
    bases, offs = synth.pack_reads(seqs)
    return bases, offs, 2


@pytest.mark.parametrize("k,nt,idx_type,hll_mode,unit", [
    (31, 15, 2, binding.HLL_PRELOAD, 20000),
    (31, 15, 2, binding.HLL_CHUNKED, 500000),
    (31, 15, 2, binding.HLL_DENSE_ONLY, 500000),
    (31, 15, 1, binding.HLL_PRELOAD, 500000),        # KRAKIDX: xor_mask 0
    (21, 12, 2, binding.HLL_PRELOAD, 500000),
    (29, 9, 2, binding.HLL_CHUNKED, 500000),
])
def test_fused_call_equals_the_halves(k, nt, idx_type, hll_mode, unit):
    rng = np.random.default_rng(4000 + k + nt + idx_type + hll_mode)
    tax = synth.make_taxonomy(6)
    genomes = synth.random_genomes(rng, 6, 2500, shared_frac=0.25)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, k)
    kdb, idx = synth.build_db_images(km, tx, k, nt, idx_type)
    bases, offs, first = _stress_batch(rng, genomes, k)
    assert int(offs[first]) % 32 != 0
    assert len(set((offs[first:-1] % 32).tolist())) == 32
    fused = _run("fused", kdb, idx, tax, bases, offs, first, hll_mode, unit)
    halves = _run("halves", kdb, idx, tax, bases, offs, first, hll_mode, unit)
    assert int(fused["call"].astype(bool).sum()) > 0.5 * len(fused["call"])
    _same(fused, halves)


def test_preload_candidate_pair_equals_the_halves():
    """A (unit, taxon) pair with more than 1024 inserts is a candidate of the preload rule: its distinct codes are
    counted from the canonical k-mers of its windows, which the fused call recomputes from the packed blocks.  With
    exactly 1024 distinct codes the last insert decides (converts iff it repeats an earlier code)."""
    rng = np.random.default_rng(5)
    g = rng.integers(0, 4, 1024 + 30, dtype=np.uint8)
    tax = synth.make_taxonomy(1)
    km, tx = synth.label_kmers([g], synth.species_ids(tax), tax, 31)
    kdb, idx = synth.build_db_images(km, tx, 31, 7, 2)
    whole = synth.decode(g).tobytes()
    tiers = set()
    for reads in ([whole, whole[500:560]], [whole[:500] + b"\r\n" + whole[500:], whole[-60:]],
                  [whole[:1024 + 29], whole[-31:]]):
        bases, offs = synth.pack_reads([b"ACGT" * 5, b"TTG"] + reads)
        fused = _run("fused", kdb, idx, tax, bases, offs, 2, binding.HLL_PRELOAD, 10 ** 9)
        halves = _run("halves", kdb, idx, tax, bases, offs, 2, binding.HLL_PRELOAD, 10 ** 9)
        _same(fused, halves)
        tiers.add(tuple(fused["counts"]["sparse"].tolist()))
    assert len(tiers) >= 2          # the corner went both ways
