"""Inputs of `count_unique` (the reference's src/count_unique.cpp and its GPU drop-in bin/count_unique) shared by the
CPU and GPU tests, the recorded reference runs on them (stdin included), the plain-C oracle's kuqo_count_unique
(oracle/count_unique_oracle.c), and FastaReader's sequences of an input for the C ABI."""
import ctypes as C
import gzip
import hashlib
import os

import numpy as np

from oracle import oracle_py
from tests import ref_replay

PIECE = 50000                                   # SKIP_LEN of count_unique.cpp


def _rand(rng, n, alphabet=b"ACGT"):
    return np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)].tobytes()


def _lines(seq, width, eol=b"\n"):
    return b"".join(seq[i:i + width] + eol for i in range(0, len(seq), width))


def _fasta(records, width=60, eol=b"\n"):
    return b"".join(b">" + name + eol + _lines(seq, width, eol) for name, seq in records)


def _mixed(rng, n):
    """upper and lower case, N runs and IUPAC codes"""
    s = bytearray(_rand(rng, n, b"ACGTACGTacgt"))
    for at in rng.integers(0, n - 40, n // 2000 + 1):
        run = int(rng.integers(1, 40))
        s[at:at + run] = b"N" * run
    for at in rng.integers(0, n, n // 500 + 1):
        s[at] = b"RYKMSWBDHVN"[int(rng.integers(0, 11))]
    return bytes(s)


def _cases():
    rng = np.random.default_rng(20261018)
    c = {}
    # multi-line records, lower case, N runs, IUPAC codes: the precision and k of the defaults and others
    mixed = _fasta([(b"a desc", _mixed(rng, 7000)), (b"b", _mixed(rng, 3000)), (b"c", _mixed(rng, 12000))], 70)
    c["mixed_k31_p14"] = (mixed, 31, 14)
    c["mixed_k15_p10"] = (mixed, 15, 10)
    c["mixed_k25_p18"] = (mixed, 25, 18)
    c["mixed_k1_p4"] = (mixed, 1, 4)
    # sequence lengths around k and around one piece (50000 + k - 1)
    k = 21
    lens = [k - 1, k, PIECE + k - 2, PIECE + k - 1, PIECE + k]
    c["lengths_k21_p12"] = (_fasta([(b"s%d" % n, _rand(rng, n)) for n in lens], 80), k, 12)
    # sequences spanning several pieces
    c["long_k31_p14"] = (_fasta([(b"l1", _rand(rng, 120000)), (b"l2", _mixed(rng, 260003))], 60), 31, 14)
    # CRLF: 60 bases + '\r' per line puts a '\r' at 61 j + 60; with k = 21 the piece [0, 50020) ends on one (50019).
    # A record with empty CRLF lines adds runs of '\r'; another width moves the '\r' around the other piece ends.
    crlf = [(b"r1", _rand(rng, 150000)), (b"r2", _mixed(rng, 103000))]
    body = _fasta(crlf, 60, b"\r\n") + b">r3\r\n" + b"".join(_rand(rng, 70) + b"\r\n" + b"\r\n" * int(rng.integers(0, 3))
                                                                  for _ in range(1500))
    c["crlf_k21_p12"] = (body, 21, 12)
    c["crlf_k31_p18"] = (_fasta([(b"w", _rand(rng, 180000))], 73, b"\r\n"), 31, 18)
    # nothing to count
    c["empty_k31_p14"] = (b"", 31, 14)
    c["no_valid_kmer_k21_p14"] = (b">a\nNNNNNNNNNNNNNNNNNNNNNNNNNNNNN\n>b\nACGTACGTAC\n>c\n>d\nACGTRYACGTACGTACGTACGTACGT\n", 21, 14)
    c["no_header_k21_p14"] = (b"ACGTACGTACGTACGTACGTACGTACGTACGT\n>a\n" + _rand(rng, 500) + b"\n", 21, 14)
    c["fastq_k21_p14"] = (b"@r1\n" + _rand(rng, 100) + b"\n+\n" + b"I" * 100 + b"\n", 21, 14)
    # each side of min(n_observed, ertl): a repeat (n_observed far above the few distinct k-mers) and a few random
    # windows (where the estimate can exceed n_observed)
    c["repeat_k5_p12"] = (b">rep\n" + b"ACGTTGCA" * 400 + b"\n", 5, 12)
    c["few_k21_p10"] = (b">few\n" + _rand(rng, 60) + b"\n>few2\n" + _rand(rng, 45), 21, 10)
    # gzip on stdin
    c["gzip_k21_p14"] = (gzip.compress(mixed, mtime=0), 21, 14)
    return c


CASES = _cases()


def plain(data: bytes) -> bytes:
    return gzip.decompress(data) if data[:2] == b"\x1f\x8b" else data


def args(k, p):
    return ["-k", str(k), "-p", str(p)]


class StdinTape(ref_replay.Tape):
    """ref_replay.Tape whose tool runs read a file as their standard input; the file's bytes count as an input of the
    recording like the tool's arguments and working directory"""

    def run_tool(self, tool, args, cwd, stdin):
        with open(stdin, "rb") as f:
            self.h.update(b"stdin" + hashlib.sha256(f.read()).hexdigest().encode())
        if not ref_replay.RECORD:
            return super().run_tool(tool, args, cwd)
        run = oracle_py.run_ref_tool

        def with_stdin(t, a, cwd=None):
            with open(stdin, "rb") as f:
                return run(t, a, cwd=cwd, stdin=f)
        oracle_py.run_ref_tool = with_stdin
        try:
            return super().run_tool(tool, args, cwd)
        finally:
            oracle_py.run_ref_tool = run


def run_reference(tape, tmp_path, name):
    """the recorded reference's count_unique on case `name` (stdin = the case's bytes)"""
    data, k, p = CASES[name]
    src = tmp_path / "stdin"
    src.write_bytes(data)
    cwd = tmp_path / "run"
    cwd.mkdir(exist_ok=True)
    return tape.run_tool("count_unique", args(k, p), cwd=cwd, stdin=src)


def recorded(name, tmp_path):
    """run_reference from the recording of the CPU test of case `name`"""
    tape = StdinTape(f"test_count_unique_cpu.py::test_oracle_matches_reference[{name}]")
    r = run_reference(tape, tmp_path, name)
    tape.close()
    return r


_L = None


def oracle_count_unique(data: bytes, k: int, p: int):
    """kuqo_count_unique over plain FASTA bytes: (estimate, n_observed, registers uint8[2^p])"""
    global _L
    if _L is None:
        _L = C.CDLL(os.path.join(os.path.dirname(oracle_py.__file__), "libkuq_count_unique_oracle.so"))
        _L.kuqo_count_unique.restype = C.c_uint64
        _L.kuqo_count_unique.argtypes = [C.c_char_p, C.c_size_t, C.c_uint, C.c_uint, C.c_void_p, C.POINTER(C.c_uint64)]
    regs = np.zeros(1 << p, np.uint8)
    n = C.c_uint64(0)
    est = _L.kuqo_count_unique(data, len(data), k, p, regs.ctypes.data, C.byref(n))
    return est, n.value, regs


def sequences(data: bytes):
    """FastaReader::next_sequence's sequences of plain FASTA bytes as (bases uint8, offsets uint64)"""
    lines = data.split(b"\n")
    if data == b"" or not lines[0].startswith(b">"):
        return np.zeros(0, np.uint8), np.zeros(1, np.uint64)
    seqs, cur = [], None
    for ln in lines:
        if ln.startswith(b">"):
            if cur is not None:
                seqs.append(b"".join(cur))
            cur = []
        else:
            cur.append(ln)
    seqs.append(b"".join(cur))
    offs = np.zeros(len(seqs) + 1, np.uint64)
    offs[1:] = np.cumsum([len(s) for s in seqs])
    return np.frombuffer(b"".join(seqs), np.uint8).copy(), offs
