"""krakenuniq-extract-reads' rules restated in Python, and the script's run for the reference recordings.

`krakenuniq-extract-reads [-t TAXDB] [-i] [-f] [-a] [-p] TAXIDS out.kraken reads` prints the records of `reads` whose id
has a Kraken line with one of the listed taxa (or a taxon below them in TAXDB).  `classify --extract` has to write what
that pipeline writes.  `extract()` is the script's rule set; tests/test_extract_reads_cpu.py holds it against the
script's recorded output, and the GPU tests apply it to the Kraken lines and inputs of the same run."""
from __future__ import annotations

import gzip
import os
import re
import shutil
import stat

from oracle import oracle_py
from tests import ref_replay

SCRIPT = "krakenuniq-extract-reads"       # the recorded tool, in oracle/_ref/


def install_extract():
    """Put krakenuniq-extract-reads (the reference's scripts/, next to KUQ_REFERENCE_SRC) into oracle/_ref/.  Only
    recording needs it; replay reads the tapes."""
    if not ref_replay.RECORD:
        return
    scripts = os.path.join(os.environ.get("KUQ_REFERENCE_SRC", ""), os.pardir, "scripts")
    if not os.path.exists(os.path.join(scripts, SCRIPT)):
        raise RuntimeError("recording the extraction needs KUQ_REFERENCE_SRC=<krakenuniq>/src")
    os.makedirs(oracle_py.REF_DIR, exist_ok=True)
    exe = os.path.join(oracle_py.REF_DIR, SCRIPT)
    shutil.copyfile(os.path.join(scripts, SCRIPT), exe)
    os.chmod(exe, os.stat(exe).st_mode | stat.S_IXUSR | stat.S_IXGRP | stat.S_IXOTH)


def _lines(data: bytes):
    """Perl's readline: every line with its '\\n'"""
    return re.findall(rb"[^\n]*\n|[^\n]+$", data)


def _num(s):
    """Perl's numeric value of a string (leading whitespace, then digits; 0 when there are none)"""
    m = re.match(rb"\s*([+-]?\d+)", s or b"")
    return int(m.group(1)) if m else 0


def _split(line: bytes, sep: bytes):
    """Perl's split(/sep/, line): trailing empty fields removed"""
    f = line.split(sep)
    while f and not f[-1]:
        f.pop()
    return f


def selected(kraken: bytes, taxids: str, taxdb: bytes | None = None):
    """(the read ids marked for printing, the number of matched lines) (:60-127)"""
    taxon = {t: 0 for t in _split(taxids.encode(), b",")}
    if taxdb is not None:                               # -t (:63-78): a child multigraph, every row in file order
        children = {}
        for line in _lines(taxdb):
            f = _split(line, b"\t")
            if not f:
                break
            tid, parent = f[0], f[1] if len(f) > 1 else None
            if _num(tid) != _num(parent):
                children.setdefault(parent if parent is not None else b"", []).append(tid)

        def get_children(nodes):
            out = []
            for p in nodes:
                out += children.get(p, [])
                for c in children.get(p, []):
                    out += get_children([c])
            return out
        for c in get_children(list(taxon)):
            taxon[c] = 0
    print_it, total = set(), 0
    for line in _lines(kraken):
        f = line.split(b"\t")
        if len(f) < 3:
            continue
        readid, taxid = f[1], f[2].rstrip(b"\n") if len(f) == 3 else f[2]
        if taxid in taxon or b"-1" in taxon:
            print_it.add(readid)
            total += 1
    return print_it, total


def script_id(line: bytes, start: bytes) -> bytes:
    """the id a record line is looked up by (:142-150)"""
    words = line.split()
    rid = words[0] if words else b""
    if rid.startswith(start):
        rid = rid[1:]
    return re.sub(rb"[/.][12]$", b"", rid)


def extract(kraken: bytes, taxids: str, reads: bytes, reads2: bytes | None = None, taxdb: bytes | None = None,
            invert=False, fasta_out=False, fasta_in=False) -> bytes:
    """What the script prints: `reads` (and with -p `reads2`) decompressed, `kraken` the Kraken lines"""
    print_it, total = selected(kraken, taxids, taxdb)
    if total == 0:
        return b""
    fasta_out = fasta_out or fasta_in
    start = b">" if fasta_in else b"@"
    fq, fq2 = iter(_lines(reads)), iter(_lines(reads2 or b""))
    rd = lambda it: next(it, None)
    out = []
    line = rd(fq)
    while line is not None:
        if not line.startswith(start):
            line = rd(fq)
            continue
        rid = script_id(line, start)
        if (rid in print_it) != invert:
            if fasta_out:
                out += [b">" + rid + b"\n", rd(fq) or b""]
                if fasta_in:
                    if reads2 is not None:
                        raise ValueError("options a,f and p cannot be used at the same time")
                    line = rd(fq)
                    while line is not None and not line.startswith(b">"):
                        out.append(line)
                        line = rd(fq)
                    continue                              # redo LINE with the header that ended the record
                rd(fq), rd(fq)
                if reads2 is not None:
                    rd(fq2)
                    out += [b">" + rid + b"\n", rd(fq2) or b""]
                    rd(fq2), rd(fq2)
            else:
                out.append(line)
                out += [rd(fq) or b"" for _ in range(3)]
                if reads2 is not None:
                    out += [rd(fq2) or b"" for _ in range(4)]
        elif not fasta_in:
            for _ in range(3):
                rd(fq)
            if reads2 is not None:
                for _ in range(4):
                    rd(fq2)
        line = rd(fq)
    return b"".join(out)


def read_input(path) -> bytes:
    """an input file as the script reads it (`gunzip -c` for names ending in .gz)"""
    data = open(path, "rb").read()
    return gzip.decompress(data) if re.search(r".gz$", str(path)) else data
