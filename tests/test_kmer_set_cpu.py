"""`kmer_set`, the drop-in for the Jellyfish 1 step of build_db.sh, without a GPU: the version line
scripts/check_for_jellyfish.sh accepts, and the refusals of command lines it cannot serve, which come before any device
is touched."""
import os
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import binding, build, synth


@pytest.fixture(scope="module")
def exe():
    build.build_dbtools()
    return build.KMER_SET


def test_version_line_is_jellyfish_1(exe):
    r = subprocess.run([exe, "--version"], capture_output=True, text=True)
    assert r.returncode == 0
    lines = r.stdout.splitlines()
    assert len(lines) == 1 and lines[0].split()[1].startswith("1.")


@pytest.mark.parametrize("args,msg", [
    (["count", "-m", "31", "-s", "1M", "-t", "4", "-o", "database"], "-C"),
    (["count", "-m", "32", "-s", "1M", "-C", "-t", "4", "-o", "database"], "1..31"),
    (["count", "-m", "0", "-s", "1M", "-C", "-o", "database"], "1..31"),
    (["count", "-m", "31", "-s", "1M", "-C", "--no-such-option", "-o", "database"], "unrecognized option"),
    (["count", "-m", "31", "-s", "1Q", "-C", "-o", "database"], "hash size"),
    (["count", "-s", "1M", "-C", "-o", "database"], "-m"),
    (["merge", "-o", "database"], "Usage"),
])
def test_usage_errors_exit_ex_usage(exe, tmp_path, args, msg):
    fa = tmp_path / "lib.fa"
    fa.write_bytes(b">a\n" + b"ACGT" * 20 + b"\n")
    r = subprocess.run([exe] + args + [str(fa)], capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 64, r.stderr
    assert msg in r.stderr
    assert "device" not in r.stderr
    assert not list(tmp_path.glob("database*"))


def test_no_input_file_is_a_usage_error(exe, tmp_path):
    r = subprocess.run([exe, "count", "-m", "21", "-C", "-o", "database"], capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 64 and "no input file" in r.stderr


def test_header_matches_synth():
    for k in (1, 8, 15, 21, 28, 31):
        assert np.array_equal(binding.kdb_header(k, 9840), synth.kdb_header(k, 9840))


def test_no_cpu_fallback(exe, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    fa = tmp_path / "lib.fa"
    fa.write_bytes(b">a\n" + b"ACGT" * 20 + b"\n")
    r = subprocess.run([exe, "count", "-m", "21", "-s", "1M", "-C", "-t", "2", "-o", "database", str(fa)],
                       capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 69 and "no CPU path" in r.stderr
    assert not list(tmp_path.glob("database*"))
    with pytest.raises(binding.KuqError) as e:
        binding.kmer_set(np.frombuffer(b"ACGT" * 20, np.uint8), np.array([0, 80], np.uint64), 21)
    assert e.value.code == -3
    assert os.path.exists(build.KMER_SET)
