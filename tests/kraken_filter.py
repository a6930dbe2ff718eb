"""krakenuniq-filter's rules restated in Python, and the script's run for the reference recordings.

`krakenuniq-filter --db DB --threshold T out.kraken` (scripts/krakenuniq-filter:87-146) moves each read's call up the
taxonomy of DB/taxDB until at least a fraction T of the read's unambiguous k-mers lie in the clade, and writes the
fraction as a `P=` column.  `classify --threshold T` has to write what that pipeline writes.  `filter_lines()` is the
script's rule set; tests/test_kraken_filter_cpu.py holds it against the script's recorded output, and the GPU tests
apply it to the unfiltered Kraken lines of the same run."""
from __future__ import annotations

import os
import shutil
import stat

from oracle import oracle_py
from tests import ref_replay

FILTER = "krakenuniq-filter"       # the recorded tool, in oracle/_ref/ next to its krakenlib.pm


def install_filter():
    """Put krakenuniq-filter and krakenlib.pm (the reference's scripts/, next to KUQ_REFERENCE_SRC) into oracle/_ref/.
    Only recording needs them; replay reads the tapes."""
    if not ref_replay.RECORD:
        return
    scripts = os.path.join(os.environ.get("KUQ_REFERENCE_SRC", ""), os.pardir, "scripts")
    if not os.path.exists(os.path.join(scripts, FILTER)):
        raise RuntimeError("recording the filter needs KUQ_REFERENCE_SRC=<krakenuniq>/src")
    os.makedirs(oracle_py.REF_DIR, exist_ok=True)
    for name in (FILTER, "krakenlib.pm"):
        shutil.copyfile(os.path.join(scripts, name), os.path.join(oracle_py.REF_DIR, name))
    exe = os.path.join(oracle_py.REF_DIR, FILTER)
    os.chmod(exe, os.stat(exe).st_mode | stat.S_IXUSR | stat.S_IXGRP | stat.S_IXOTH)


def taxdb_rows(data: bytes):
    """(taxid, parent) of every taxDB row in file order (load_taxonomy, :136-146)"""
    rows = []
    for line in data.splitlines():
        f = line.split(b"\t")
        if len(f) >= 2 and f[0]:
            rows.append((int(f[0]), int(f[1])))
    return rows


def parent_map(rows):
    """F: `$parent_map{$taxID} = $parentTaxID unless $parentTaxID == $taxID`, rows in file order"""
    F = {}
    for t, p in rows:
        if p != t:
            F[t] = p
    return F


def filter_line(line: bytes, F, threshold: float) -> bytes:
    """one Kraken line (without its '\\n') → the script's line (:88-133)"""
    code, seqid, called, length, hit_list = line.split(b"\t")[:5]
    counts = {}
    for h in hit_list.split():
        taxid, ct = h.split(b":")
        counts[taxid] = counts.get(taxid, 0) + int(ct)
    total_unambig, hit_sums = 0, {}
    for taxid, count in counts.items():
        if taxid == b"A":
            continue
        total_unambig += count                          # misses (0:n) and Q:n count
        if taxid.isdigit() and int(taxid) > 0:
            t = int(taxid)
            while t in F:
                hit_sums[t] = hit_sums.get(t, 0) + count
                t = F[t]
    pct, new = 0.0, int(called)
    while new in F:
        pct = hit_sums.get(new, 0) / total_unambig
        if pct >= threshold - 1e-5:
            break
        new = F[new]
    return b"%s\t%s\t%d\t%s\tP=%.3f\t%s\n" % (b"C" if new > 0 else b"U", seqid, new, length, pct, hit_list)


def filter_lines(kraken: bytes, F, threshold: float) -> bytes:
    """a whole Kraken file"""
    lines = kraken.split(b"\n")
    if lines and not lines[-1]:
        lines.pop()
    return b"".join(filter_line(l, F, threshold) for l in lines)
