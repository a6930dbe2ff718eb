"""krakenuniq-mpa-report's rules restated in Python, and the scripts' run for the reference recordings.

`krakenuniq-mpa-report --db DB [--show-zeros] [--header-line] [--intermediate-ranks] a.kraken b.kraken ...`
(scripts/krakenuniq-mpa-report) writes one MetaPhlAn-style table with a count column per Kraken file.
`classify --mpa-report` has to write that table for the Kraken lines of its run.  `mpa_table()` is the script's rule set;
tests/test_mpa_report_cpu.py holds it against the script's recorded output, and the GPU tests apply it to the Kraken
lines of the same run.  `load_taxonomy()` and `install_script()` serve krakenuniq-translate (tests/translate.py) too."""
from __future__ import annotations

import io
import json
import os
import shutil
import stat
import zipfile

from oracle import oracle_py
from tests import ref_replay

MPA = "krakenuniq-mpa-report"       # the recorded tool, in oracle/_ref/ next to its krakenlib.pm
RANK_CODES = {b"species": "S", b"genus": "G", b"family": "F", b"order": "O", b"class": "C", b"phylum": "P",
              b"superkingdom": "D", b"kingdom": "K"}


def install_script(name):
    """Put the script `name` and krakenlib.pm (the reference's scripts/, next to KUQ_REFERENCE_SRC) into oracle/_ref/.
    Only recording needs them; replay reads the tapes."""
    if not ref_replay.RECORD:
        return
    scripts = os.path.join(os.environ.get("KUQ_REFERENCE_SRC", ""), os.pardir, "scripts")
    if not os.path.exists(os.path.join(scripts, name)):
        raise RuntimeError(f"recording {name} needs KUQ_REFERENCE_SRC=<krakenuniq>/src")
    os.makedirs(oracle_py.REF_DIR, exist_ok=True)
    for f in (name, "krakenlib.pm"):
        shutil.copyfile(os.path.join(scripts, f), os.path.join(oracle_py.REF_DIR, f))
    exe = os.path.join(oracle_py.REF_DIR, name)
    os.chmod(exe, os.stat(exe).st_mode | stat.S_IXUSR | stat.S_IXGRP | stat.S_IXOTH)


def install_mpa_report():
    install_script(MPA)


def write_db(path, taxdb: bytes):
    """the --db directory the scripts take: taxDB, and empty database.kdb / .idx for krakenlib::find_db"""
    (path / "taxDB").write_bytes(taxdb)
    (path / "database.kdb").write_bytes(b"")
    (path / "database.idx").write_bytes(b"")


def taxdb_fields(data: bytes):
    """(taxid, parent, name, rank) of every row in file order, as `chomp; split(/\\t/)` gives them (None = undef)"""
    rows = []
    for line in data.split(b"\n"):
        if not line:
            continue
        f = line.split(b"\t")
        while f and f[-1] == b"":                          # split drops trailing empty fields
            f.pop()
        f += [None] * (4 - len(f))
        rows.append(tuple(f[:4]))
    return rows


def load_taxonomy(data: bytes):
    """load_taxonomy (:196-209): name and rank maps (last row wins) and the child lists (one entry per row whose parent
    differs from its taxid as a string, file order)"""
    names, ranks, children = {}, {}, {}
    for t, p, name, rank in taxdb_fields(data):
        names[t] = name
        ranks[t] = rank
        if p != t:
            children.setdefault(p, []).append(t)
    return names, ranks, children


def rank_code(rank) -> str:
    return RANK_CODES.get(rank, "-")


def kraken_lines(data: bytes):
    """the lines `while (<FILE>)` reads"""
    lines = data.split(b"\n")
    if lines and not lines[-1]:
        lines.pop()
    return lines


def taxo_counts(kraken: bytes):
    """`$taxo_counts{$fields[2]}++` over `split` of every line"""
    counts = {}
    for line in kraken_lines(kraken):
        f = line.split()
        key = f[2] if len(f) > 2 else b""
        counts[key] = counts.get(key, 0) + 1
    return counts


def mpa_table(files, taxdb: bytes, show_zeros=False, header_line=False, intermediate=False, ids=None) -> bytes:
    """the script's table over the Kraken data of each file, in order; `ids` are the header line's sample ids"""
    names, ranks, children = load_taxonomy(taxdb)
    file_data, hit = [], set()

    for kraken in files:
        counts = taxo_counts(kraken)

        def dfs_summation(node):
            for child in children.get(node, ()):
                dfs_summation(child)
                counts[node] = counts.get(node, 0) + counts.get(child, 0)
        dfs_summation(b"1")
        hit.update(k for k, v in counts.items() if v)
        file_data.append(counts)
    codes = list("DKPCOFGS") + (["X"] if intermediate else [])
    out = {c: [] for c in codes}

    def dfs_report(node, name):
        if not show_zeros and node not in hit:
            return
        code = rank_code(ranks.get(node))
        if code != "-" or intermediate:
            code = "X" if code == "-" else code
            nm = (names.get(node) or b"").replace(b"|", b"").replace(b".", b"").replace(b" ", b"_")
            name = (name + b"|" if name is not None else b"") + code.lower().encode() + b"__" + nm
            out[code].append(name + b"".join(b"\t%d" % d.get(node, 0) for d in file_data) + b"\n")
        for child in children.get(node, ()):
            dfs_report(child, name)
    dfs_report(b"1", None)
    head = b"#Sample ID\t" + b"\t".join(i.encode() for i in ids) + b"\n" if header_line else b""
    return head + b"".join(b"".join(out[c]) for c in codes)


def recorded_stdout(test_file: str, test_name: str):
    """the scripts' standard output of each run recorded for tests/<test_file>::<test_name>, in order"""
    path = os.path.join(ref_replay.DIR, f"{test_file}_{test_name}.zip")
    with zipfile.ZipFile(path) as z:
        meta = json.load(io.BytesIO(z.read("meta.json")))
    return [r["stdout"].encode() for r in meta["runs"]]
