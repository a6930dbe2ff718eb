"""count_unique on the GPU: the drop-in's stdout against the recorded reference and the oracle on every input of
tests/count_unique.py, the C ABI's registers against the oracle's at every precision, independence from the batch size,
and one seeded library of a few hundred Mbp."""
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import binding, build
from tests import count_unique as cu

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def exe():
    build.build_dbtools()
    return build.COUNT_UNIQUE


@pytest.mark.parametrize("name", sorted(cu.CASES))
def test_drop_in_prints_what_the_reference_printed(exe, tmp_path, name):
    data, k, p = cu.CASES[name]
    want = cu.recorded(name, tmp_path)
    with open(tmp_path / "stdin", "rb") as f:
        got = subprocess.run([exe] + cu.args(k, p), stdin=f, capture_output=True, text=True)
    assert got.returncode == want.returncode == 0, got.stderr
    assert got.stdout == want.stdout == f"{cu.oracle_count_unique(cu.plain(data), k, p)[0]}\n"


def test_drop_in_reads_a_pipe(exe):
    data, k, p = cu.CASES["gzip_k21_p14"]
    got = subprocess.run(["sh", "-c", f"cat | {exe} -k {k} -p {p}"], input=data, capture_output=True)
    assert got.returncode == 0 and got.stdout == b"%d\n" % cu.oracle_count_unique(cu.plain(data), k, p)[0]


@pytest.mark.parametrize("p", range(4, 19))
def test_registers_equal_the_oracle_at_every_precision(p):
    for name, k in (("crlf_k21_p12", 21), ("long_k31_p14", 31), ("mixed_k15_p10", 15)):
        data = cu.plain(cu.CASES[name][0])
        want = cu.oracle_count_unique(data, k, p)
        est, n, regs = binding.count_unique(*cu.sequences(data), k, p)
        assert (est, n) == want[:2], name
        assert np.array_equal(regs, want[2]), name


@pytest.mark.parametrize("batch", [2 * 31 + 32, 1000, 50031, 1 << 16])
def test_result_does_not_depend_on_the_batch_size(batch):
    for name in ("crlf_k21_p12", "long_k31_p14", "lengths_k21_p12", "mixed_k1_p4"):
        data, k, p = cu.CASES[name]
        data = cu.plain(data)
        want = cu.oracle_count_unique(data, k, p)
        est, n, regs = binding.count_unique(*cu.sequences(data), k, p, batch=max(batch, 2 * k + 32))
        assert (est, n) == want[:2] and np.array_equal(regs, want[2]), (name, batch)


def test_adding_in_several_calls_equals_one_call():
    data, k, p = cu.CASES["crlf_k21_p12"]
    bases, offs = cu.sequences(data)
    c = binding.CountUnique(k, p)
    try:
        for r in range(len(offs) - 1):
            c.add(bases[int(offs[r]):int(offs[r + 1])], np.array([0, offs[r + 1] - offs[r]], np.uint64))
        est, n, regs = c.result()
        assert c.stats()["windows"] == n
    finally:
        c.close()
    want = cu.oracle_count_unique(data, k, p)
    assert (est, n) == want[:2] and np.array_equal(regs, want[2])


def test_a_library_of_hundreds_of_mbp(exe, tmp_path):
    rng = np.random.default_rng(7)
    lens = rng.integers(1 << 20, 40 << 20, 24)
    lens = (lens * (300e6 / lens.sum())).astype(np.int64)
    alphabet = np.frombuffer(b"ACGTACGTACGTACGTacgtN", np.uint8)
    bases = alphabet[rng.integers(0, len(alphabet), int(lens.sum()), dtype=np.uint8)]
    offs = np.zeros(len(lens) + 1, np.uint64)
    offs[1:] = np.cumsum(lens)
    fa = b"".join(b">s%d\n" % i + bases[int(offs[i]):int(offs[i + 1])].tobytes() + b"\n" for i in range(len(lens)))
    k, p = 31, 14
    want = cu.oracle_count_unique(fa, k, p)
    est, n, regs = binding.count_unique(bases, offs, k, p)
    assert (est, n) == want[:2] and np.array_equal(regs, want[2])
    (tmp_path / "lib.fa").write_bytes(fa)
    with open(tmp_path / "lib.fa", "rb") as f:
        got = subprocess.run([exe, "-k", str(k), "-p", str(p)], stdin=f, capture_output=True, text=True)
    assert got.returncode == 0 and got.stdout == f"{want[0]}\n"
