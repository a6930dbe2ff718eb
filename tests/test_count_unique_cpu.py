"""count_unique without a GPU: the plain-C oracle against the recorded runs of the reference's count_unique on every
input of tests/count_unique.py, and the drop-in's refusals of command lines, which come before any device is touched."""
import os
import subprocess

import pytest

from krakenuniq_b200 import build
from tests import count_unique as cu


@pytest.fixture
def reference(request):
    """the reference's recorded count_unique runs of this test, stdin included"""
    tape = cu.StdinTape(request.node.nodeid)
    yield tape
    tape.close()


@pytest.fixture(scope="module")
def exe():
    build.build_dbtools()
    return build.COUNT_UNIQUE


@pytest.mark.parametrize("name", sorted(cu.CASES))
def test_oracle_matches_reference(reference, tmp_path, name):
    data, k, p = cu.CASES[name]
    r = cu.run_reference(reference, tmp_path, name)
    assert r.returncode == 0, r.stderr
    est, n_observed, regs = cu.oracle_count_unique(cu.plain(data), k, p)
    assert r.stdout == f"{est}\n"
    assert ("malformed fasta file" in r.stderr) == (name in ("empty_k31_p14", "no_header_k21_p14", "fastq_k21_p14"))


def test_cases_cover_both_sides_of_n_observed():
    """the estimate is n_observed on one input and the Ertl estimate below it on another"""
    sides = set()
    for name in ("repeat_k5_p12", "mixed_k25_p18"):
        data, k, p = cu.CASES[name]
        est, n, _ = cu.oracle_count_unique(data, k, p)
        sides.add(est == n)
    assert sides == {True, False}


def test_crlf_piece_end_counts_a_window_twice():
    """with k = 21 the first piece of r1 ends on a '\\r': the scanner reads on into the next piece, and n_observed
    exceeds the windows of the sequence read as a whole"""
    data, k, p = cu.CASES["crlf_k21_p12"]
    bases, offs = cu.sequences(data)
    r1 = bytes(bases[int(offs[0]):int(offs[1])])
    assert r1[cu.PIECE + k - 2:cu.PIECE + k - 1] == b"\r"
    _, n_pieces, _ = cu.oracle_count_unique(b">r1\n" + r1 + b"\n", k, p)
    clean = r1.replace(b"\r", b"")
    whole = len(clean) - k + 1 - r1.count(b"\r")          # one window skipped per '\r'
    assert n_pieces > whole


@pytest.mark.parametrize("args", [["-k", "0"], ["-k", "32"], ["-t", "0"], ["-t", "100000"], ["-h"], ["-x"],
                                  ["-p", "21", "-k", "40"]])
def test_refusals_match_reference(reference, exe, tmp_path, args):
    data = b">a\n" + b"ACGT" * 20 + b"\n"
    stdin = tmp_path / "stdin"
    stdin.write_bytes(data)
    cwd = tmp_path / "run"
    cwd.mkdir()
    want = reference.run_tool("count_unique", args, cwd=cwd, stdin=stdin)
    with open(stdin, "rb") as f:
        got = subprocess.run([exe] + args, stdin=f, capture_output=True, text=True, cwd=cwd)
    assert (got.returncode, got.stdout) == (want.returncode, want.stdout)
    assert got.stdout == "" and "device" not in got.stderr
    assert got.stderr.splitlines()[-1:] == want.stderr.splitlines()[-1:]


@pytest.mark.parametrize("p", ["3", "19", "-1", "abc"])
def test_precision_outside_4_to_18_exits_ex_usage(reference, exe, tmp_path, p):
    """the reference aborts on an uncaught std::invalid_argument; the drop-in prints its message and exits 64"""
    stdin = tmp_path / "stdin"
    stdin.write_bytes(b">a\n" + b"ACGT" * 20 + b"\n")
    cwd = tmp_path / "run"
    cwd.mkdir()
    want = reference.run_tool("count_unique", ["-p", p], cwd=cwd, stdin=stdin)
    assert want.returncode < 0 and want.stdout == ""
    msg = "precision (number of register = 2^precision) must be between 4 and 18"
    assert msg in want.stderr
    with open(stdin, "rb") as f:
        got = subprocess.run([exe, "-p", p], stdin=f, capture_output=True, text=True, cwd=cwd)
    assert (got.returncode, got.stdout, got.stderr) == (64, "", msg + "\n")


def test_precision_wraps_like_uint8(exe, tmp_path):
    """the reference's constructor takes the precision as uint8_t: -p 260 is precision 4, which passes the check"""
    stdin = tmp_path / "stdin"
    stdin.write_bytes(b"")
    with open(stdin, "rb") as f:
        got = subprocess.run([exe, "-p", "260"], stdin=f, capture_output=True, text=True)
    assert got.returncode != 64


def test_no_cpu_fallback(exe, tmp_path):
    import numpy as np
    import torch
    from krakenuniq_b200 import binding
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    stdin = tmp_path / "stdin"
    stdin.write_bytes(b">a\n" + b"ACGT" * 20 + b"\n")
    with open(stdin, "rb") as f:
        r = subprocess.run([exe, "-k", "21"], stdin=f, capture_output=True, text=True)
    assert r.returncode == 69 and "no CPU path" in r.stderr and r.stdout == ""
    with pytest.raises(binding.KuqError) as e:
        binding.count_unique(np.frombuffer(b"ACGT" * 20, np.uint8), np.array([0, 80], np.uint64), 21, 14)
    assert e.value.code == -3
    assert os.path.exists(build.COUNT_UNIQUE)
