"""krakenuniq-translate's rules restated in Python.

`krakenuniq-translate --db DB [--mpa-format] a.kraken ...` (scripts/krakenuniq-translate) prints `read id <TAB> lineage`
for every line that starts with C.  `classify --translate-out` has to write that for the Kraken lines of its run.
`translate()` is the script's rule set, including its cache: a lineage is stored under the node where its walk stopped,
so a line whose taxon has no parent entry prints the lineage last stored under that taxon.
tests/test_translate_cpu.py holds it against the script's recorded output."""
from __future__ import annotations

from tests import mpa_report

TRANSLATE = "krakenuniq-translate"


def install_translate():
    mpa_report.install_script(TRANSLATE)


def translate(kraken: bytes, taxdb: bytes, mpa_format=False) -> bytes:
    """the script's output over Kraken data (several files: their concatenation, as `<>` reads them)"""
    names, ranks, parent = {}, {}, {}
    for t, p, name, rank in mpa_report.taxdb_fields(taxdb):      # load_taxonomy (:131-144)
        names[t] = name
        ranks[t] = rank
        if int(p) != int(t):                                      # `unless $parentTaxID == $taxID`
            parent[t] = p
    known = {}
    out = []
    for line in mpa_report.kraken_lines(kraken):
        if not line.startswith(b"C"):
            continue
        f = line.split()
        seqid, taxid = f[1], f[2]
        if taxid not in known:                                    # get_taxonomy_str (:89-113)
            nodes = []
            while taxid in parent:
                if mpa_format:
                    code = mpa_report.rank_code(ranks.get(taxid))
                    if code != "-":
                        nodes.insert(0, code.lower().encode() + b"__" + names[taxid].replace(b" ", b"_"))
                else:
                    nodes.insert(0, names[taxid])
                taxid = parent[taxid]
            known[taxid] = (b"|".join(nodes) or b"root") if mpa_format else b";".join(nodes)
        out.append(seqid + b"\t" + known[taxid] + b"\n")
    return b"".join(out)
