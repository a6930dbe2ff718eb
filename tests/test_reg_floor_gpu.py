"""The per-sketch register floor of the counting launches (hll_update skips the register load for hash ranks at or
below the smallest register of the sketch): registers and counters equal those of a context whose launches are too
small for a floor (it is 0 there, every window loads its register), once registers are well above 0, and again after
they were cleared through the state pointers between calls."""
import numpy as np
import pytest

from krakenuniq_b200 import binding, synth

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
K, L = 31, 150


def _registers(clf):
    from krakenuniq_b200 import dist
    sp = clf.state_ptrs()
    torch.cuda.synchronize()
    return dist.device_view(sp.d_regs, sp.regs_bytes, torch.uint8, "cuda:0").cpu().numpy().reshape(sp.n_sketch, 4096)


def _clear_registers(clf):
    from krakenuniq_b200 import dist
    sp = clf.state_ptrs()
    torch.cuda.synchronize()
    dist.device_view(sp.d_regs, sp.regs_bytes, torch.uint8, "cuda:0").zero_()
    torch.cuda.synchronize()


def _batches(rng, genomes, n_batches, n_reads):
    """half reads of the genomes, half random bases (misses: taxon 0's sketch fills fast)"""
    out = []
    for _ in range(n_batches):
        b, o = synth.sample_reads(rng, genomes, n_reads // 2, L, 0.01, 0.0, 0.2)
        seqs = [bytes(b[int(o[i]):int(o[i + 1])]) for i in range(len(o) - 1)]
        seqs += [bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), L)) for _ in range(n_reads - len(seqs))]
        out.append(synth.pack_reads(seqs))
    return out


def _run(clf, batches, reads_per_call):
    for bases, offs in batches:
        n = len(offs) - 1
        for a in range(0, n, reads_per_call):
            o = np.ascontiguousarray(offs[a:min(n, a + reads_per_call) + 1])
            clf.classify(bases, o)


@pytest.mark.parametrize("hll_mode", [binding.HLL_DENSE_ONLY, binding.HLL_PRELOAD])
def test_register_floor_changes_no_register(hll_mode):
    rng = np.random.default_rng(11)
    tax = synth.make_taxonomy(6)
    genomes = synth.random_genomes(rng, 6, 20000, shared_frac=0.25)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, K)
    kdb, idx = synth.build_db_images(km, tx, K, 11, 2)
    first, second = _batches(rng, genomes, 4, 3000), _batches(rng, genomes, 2, 3000)

    ctx = []
    for _ in range(2):
        c = binding.Classifier(device=0, max_reads=1 << 13, max_bases=4 << 20, sparse_set_slots=1 << 22, hll_mode=hll_mode)
        c.stage_db(kdb, idx)
        c.set_taxonomy(*tax.parent_map())
        ctx.append(c)
    big, small = ctx
    n_sketch = big.state_ptrs().n_sketch
    small_reads = max(1, (n_sketch * 4096) // L - 1)      # fewer bases per call than register bytes: floor 0
    assert small_reads * L < n_sketch * 4096 < 3000 * L
    try:
        _run(big, first[:2], 3000)
        assert _registers(big).min(axis=1)[0] >= 2           # taxon 0's floor is well above 0 for the next calls
        _run(big, first[2:], 3000)
        _run(small, first, small_reads)
        assert np.array_equal(_registers(big), _registers(small))
        for c in ctx:
            _clear_registers(c)                              # between calls, through kuq_state_ptrs_get
        _run(big, second, 3000)
        _run(small, second, small_reads)
        assert np.array_equal(_registers(big), _registers(small))
        for c in ctx:
            c.finish()
        a, b = big.counts(), small.counts()
        for key in ("taxid", "n_reads", "n_kmers"):
            assert np.array_equal(a[key], b[key]), key
    finally:
        for c in ctx:
            c.close()
