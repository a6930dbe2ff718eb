"""Paired-end input for the tests: read_merger.pl's rules restated in Python, mate files derived from reads, and the
merger's run for the reference recordings.

`krakenuniq --paired A B` runs `perl read_merger.pl A B > merged.fa 2> merged.err` and then `classify merged.fa`
(scripts/krakenuniq:230-237).  `classify --paired A B` merges the mates in its ingest and has to produce what the
classify stage of that pipeline produces.  `merge()` is the rule set of scripts/read_merger.pl; it is held against the
script's recorded output by tests/test_paired_merge_cpu.py and writes the merged file of inputs no recording covers."""
from __future__ import annotations

import os
import re
import shutil
import stat

import numpy as np

from oracle import oracle_py
from tests import ref_replay

MERGER = "read_merger.sh"          # the recorded tool: the merger with the wrapper's redirections, in oracle/_ref/


def install_merger():
    """Put read_merger.pl (from the reference's scripts/, next to KUQ_REFERENCE_SRC) into oracle/_ref/ with a
    launcher that redirects like the wrapper.  Only recording needs it; replay reads the tapes."""
    if not ref_replay.RECORD:
        return
    src = os.path.join(os.environ.get("KUQ_REFERENCE_SRC", ""), os.pardir, "scripts", "read_merger.pl")
    if not os.path.exists(src):
        raise RuntimeError("recording the merger needs KUQ_REFERENCE_SRC=<krakenuniq>/src")
    os.makedirs(oracle_py.REF_DIR, exist_ok=True)
    shutil.copyfile(src, os.path.join(oracle_py.REF_DIR, "read_merger.pl"))
    launcher = os.path.join(oracle_py.REF_DIR, MERGER)
    with open(launcher, "w") as f:          # perl's warnings name the script: without its directory in the recordings
        f.write('#!/bin/sh\nd="$(dirname "$0")"\nperl "$d/read_merger.pl" "$@" > merged.fa 2> merged.err\nrc=$?\n'
                'sed -i "s|$d/||g" merged.err\nexit $rc\n')
    os.chmod(launcher, os.stat(launcher).st_mode | stat.S_IXUSR | stat.S_IXGRP | stat.S_IXOTH)


class MergeError(Exception):
    """where read_merger.pl dies; the records before it are written"""


def _lines(data: bytes):
    """Perl's <$fh>: lines with their '\\n', the last one without it if the file does not end in one"""
    out, i = [], 0
    while i < len(data):
        j = data.find(b"\n", i)
        j = len(data) if j < 0 else j + 1
        out.append(data[i:j])
        i = j
    return out


def _records(data: bytes, fasta: bool):
    """read_sequence (read_merger.pl:136-183): yields (id, seq) and raises MergeError at a malformed header"""
    lines, i = _lines(data), 0
    while i < len(lines):
        line = lines[i]
        marker = b">" if fasta else b"@"
        m = re.match(re.escape(marker) + rb"(\S+)", line)
        if not m:
            if not fasta and line == b"\n":            # a FASTQ file may end with a blank line (:165-167)
                return
            raise MergeError(("malformed fasta file" if fasta else "malformed fastq file") + f" (line = '{line.decode('latin-1')}')")
        rid = re.sub(rb"[/_.][12]$", b"", m.group(1))
        i += 1
        if fasta:                                      # every line up to the next '>' line, only '\n' removed
            seq = b""
            while i < len(lines) and not lines[i].startswith(b">"):
                seq += lines[i][:-1] if lines[i].endswith(b"\n") else lines[i]
                i += 1
        else:                                          # line 2; lines 3 and 4 skipped without a check
            seq = lines[i] if i < len(lines) else b""
            seq = seq[:-1] if seq.endswith(b"\n") else seq
            i += 3
        yield rid, seq


def merge(data1: bytes, data2: bytes, check_names: bool = False):
    """(merged FASTA bytes, warnings, error message or None) of `read_merger.pl [--check-names] A B` on the decompressed
    contents of A and B.  The format is A's first character ('>' FASTA, '@' FASTQ); B is read in A's format."""
    if not data1[:1] in (b">", b"@"):
        return b"", [], "Unknown file format"
    fasta = data1[:1] == b">"
    out, warnings = [], []
    r1, r2 = _records(data1, fasta), _records(data2, fasta)

    def take(it):
        return next(it, None)
    try:
        while (a := take(r1)) is not None:
            b = take(r2)
            if b is None:                               # :104-118: the rest of A unpaired, then ">" + "N"
                warnings.append("file 1 has more reads")
                out.append(b">" + a[0] + b"\n" + a[1] + b"\n")
                while (a := take(r1)) is not None:
                    out.append(b">" + a[0] + b"\n" + a[1] + b"\n")
                out.append(b">\nN\n")
                break
            if check_names and a[0] != b[0]:
                raise MergeError(f"mismatched mate pair names ('{a[0].decode('latin-1')}' & '{b[0].decode('latin-1')}')")
            out.append(b">" + a[0] + b"\n" + a[1] + b"N" + b[1] + b"\n")
        else:
            if (b := take(r2)) is not None:             # :119-126: the rest of B unpaired
                warnings.append("file 2 has more reads")
                out.append(b">" + b[0] + b"\n" + b[1] + b"\n")
                while (b := take(r2)) is not None:
                    out.append(b">" + b[0] + b"\n" + b[1] + b"\n")
    except MergeError as e:
        return b"".join(out), warnings, str(e)
    return b"".join(out), warnings, None


# ---- mate files from single reads ------------------------------------------------------------------------------------
_COMP = bytes.maketrans(b"ACGTNacgtn", b"TGCANtgcan")


def split_pairs(seqs, rng: np.random.Generator, mate_len: int = 0):
    """(mate 1, mate 2) of each read: mate 1 a prefix, mate 2 the reverse complement of the rest (mate_len > 0: both
    mates that long, taken from the two ends)"""
    out = []
    for s in seqs:
        if mate_len:
            a, b = s[:mate_len], s[-mate_len:]
        else:
            cut = int(rng.integers(0, len(s) + 1))
            a, b = s[:cut], s[cut:]
        out.append((a, b.translate(_COMP)[::-1]))
    return out


def fastq_bytes(records, crlf: bool = False):
    """records: (header after '@', seq)"""
    nl = b"\r\n" if crlf else b"\n"
    return b"".join(b"@" + h + nl + s + nl + b"+" + nl + b"I" * len(s) + nl for h, s in records)


def fasta_bytes(records, width: int = 0, crlf: bool = False):
    nl = b"\r\n" if crlf else b"\n"
    out = []
    for h, s in records:
        rows = [s[i:i + width] for i in range(0, len(s), width)] if width and s else [s]
        out.append(b">" + h + nl + b"".join(r + nl for r in rows))
    return b"".join(out)
