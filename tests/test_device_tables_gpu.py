"""The two device tables, the sparse-tier set and the exact k-mer set, when replacing their contents cannot allocate the
new table: the call fails with KUQ_E_NOMEM and the context keeps an empty table of the old size, which later imports
fill and count.  The failure is made deterministic with a key count no device could hold (2^40): the allocation fails
before any kernel reads the caller's buffer."""
import numpy as np
import pytest
import torch

from krakenuniq_b200 import binding, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KUQ_E_NOMEM = -8
TOO_MANY = 1 << 40


def _context(mode, slots):
    rng = np.random.default_rng(41)
    tax = synth.make_taxonomy(8)
    genomes = synth.random_genomes(rng, 8, 3000, shared_frac=0.25)
    km, tx = synth.label_kmers(genomes, synth.species_ids(tax), tax, 31)
    kdb, idx = synth.build_db_images(km, tx, 31, 6, 1)
    bases, offs = synth.sample_reads(rng, genomes, 600, 150, 0.02, 0.2, 0.2)
    clf = binding.Classifier(device=0, hll_mode=mode, sparse_set_slots=slots, max_reads=1 << 12, max_bases=1 << 20)
    clf.stage_db(kdb, idx)
    clf.set_taxonomy(*tax.parent_map())
    clf.classify(bases, offs)
    clf.finish()
    return clf


def _fails_with_nomem(call):
    with pytest.raises(binding.KuqError) as e:
        call()
    assert e.value.code == KUQ_E_NOMEM, str(e.value)


@pytest.mark.parametrize("mode", [binding.HLL_PRELOAD, binding.HLL_CHUNKED])
def test_failed_sparse_replace_keeps_an_empty_set(mode):
    clf = _context(mode, 1 << 14)
    n = clf.sparse_export()
    assert n > 0
    keys = torch.zeros(n, dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    assert clf.sparse_export(keys.data_ptr(), n) == n
    before = clf.sparse_tier_info()
    _fails_with_nomem(lambda: clf.sparse_replace(keys.data_ptr(), TOO_MANY))
    after = clf.sparse_tier_info()
    assert after["slots"] == before["slots"] and after["keys"] == 0, (before, after)
    clf.sparse_import(keys.data_ptr(), n)
    assert clf.sparse_tier_info()["keys"] == n
    assert clf.sparse_export() == n


def test_failed_exact_replace_keeps_an_empty_table():
    clf = _context(binding.HLL_EXACT, 1 << 12)
    n = clf.exact_export()
    assert n > 0
    pairs = torch.zeros((n, 2), dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    assert clf.exact_export(pairs.data_ptr(), n) == n
    before = clf.exact_info()
    _fails_with_nomem(lambda: clf.exact_replace(pairs.data_ptr(), TOO_MANY))
    after = clf.exact_info()
    assert after["slots"] == before["slots"] and after["pairs"] == 0, (before, after)
    clf.exact_import(pairs.data_ptr(), n)
    assert clf.exact_info()["pairs"] == before["pairs"] == n
    assert clf.exact_export() == n
