"""krakenuniq-extract-reads' rules (tests/extract_reads.py) against the script's recorded output on crafted Kraken lines,
reads and taxonomies, the subtree expansion of the library (kuq_extract_taxa, no device needed) against the
restatement, and the argument checks of `classify --extract`, which run before any device call."""
import gzip
import subprocess

import pytest

from krakenuniq_b200 import binding, build
from tests import extract_reads


def fq(recs, nl=b"\n"):
    return b"".join(b"@%s%s%s%s+%s%s%s" % (h, nl, s, nl, nl, q, nl) for h, s, q in recs)


# ids with /1 /2 .1 .2 and suffixes that are not stripped; r4's quality line starts with '@'
FQ = fq([(b"r1 desc", b"ACGT", b"IIII"), (b"r2/1", b"AC", b"II"), (b"r3.2 x", b"GGG", b"III"), (b"r4", b"TTTT", b"@III"),
         (b"r5/3", b"CC", b"II"), (b"r6_1", b"A", b"I"), (b"r7", b"ACG", b"III")])
FA = b">r1 desc\nACGT\nGGCC\n>r2/1\nAC\n>r3\nTTTT\nAAAA\nCC\n>r4.1\nG\n>r7\nAC\nGT\n"
# the Kraken lines classify writes for these records (id = the header's first word)
KRAKEN = b"".join(b"\t".join(f) + b"\n" for f in [
    (b"C", b"r1", b"9", b"4", b"9:1"), (b"C", b"r2/1", b"9", b"2", b"9:1"), (b"C", b"r3.2", b"10", b"3", b"10:1"),
    (b"U", b"r4", b"0", b"4", b"0:1"), (b"C", b"r5/3", b"12", b"2", b"12:1"), (b"C", b"r6_1", b"13", b"1", b"13:1"),
    (b"C", b"r7", b"1", b"3", b"1:1"), (b"C", b"r3", b"10", b"10", b"10:1"), (b"U", b"r4.1", b"0", b"1", b"0:0")])
ONLY_C = b"".join(l + b"\n" for l in KRAKEN.split(b"\n") if l.startswith(b"C"))          # `classify -c`
FILTERED = KRAKEN.replace(b"\t9:1", b"\tP=0.500\t9:1")                                     # `--threshold` lines
# taxDB rows in file order: 10 has two rows (under 9 and under 1), a self-parent root, an empty line, and rows after it
TAXDB = b"1\t1\troot\tno rank\n9\t1\tn9\tgenus\n10\t9\tn10\tspecies\n10\t1\tn10\tspecies\n\n12\t10\tn12\tstrain\n13\t12\tn13\tstrain\n"
MATE1 = fq([(b"p1/1", b"ACGT", b"IIII"), (b"p2/1 x", b"GG", b"II"), (b"p3/1", b"T", b"I")])
MATE2 = fq([(b"p1/2", b"TTTT", b"JJJJ"), (b"p2/2", b"CC", b"JJ"), (b"p3/2", b"A", b"J")])
KRAKEN_PAIRED = b"C\tp1\t9\t9\t9:1\nU\tp2\t0\t5\t0:1\nC\tp3\t10\t3\t10:1\n"

CASES = {   # name: (Kraken lines, taxa, options, reads: fq | fa | crlf | gz | paired)
    "fastq": (KRAKEN, "9", [], "fq"),
    "subtree": (KRAKEN, "9", ["-t"], "fq"),
    "others_and_unclassified": (KRAKEN, "-1,0", [], "fq"),
    "unclassified": (KRAKEN, "0", [], "fq"),
    "absent": (KRAKEN, "77", [], "fq"),
    "absent_inverted": (KRAKEN, "77", ["-i"], "fq"),
    "inverted": (KRAKEN, "9,12", ["-i"], "fq"),
    "fasta_out": (KRAKEN, "9,10", ["-f"], "fq"),
    "fasta_in": (KRAKEN, "10,1", ["-a"], "fa"),
    "fasta_in_others": (KRAKEN, "-1", ["-a"], "fa"),
    "fasta_in_subtree_inverted": (KRAKEN, "10", ["-a", "-i", "-t"], "fa"),
    "crlf": (KRAKEN, "9,0", [], "crlf"),
    "crlf_fasta_out": (KRAKEN, "9,0", ["-f"], "crlf"),
    "gzip": (KRAKEN, "10,13", ["-t"], "gz"),
    "paired": (KRAKEN_PAIRED, "9,10", ["-p"], "paired"),
    "paired_fasta_out": (KRAKEN_PAIRED, "9", ["-p", "-f"], "paired"),
    "paired_inverted": (KRAKEN_PAIRED, "9", ["-p", "-i"], "paired"),
    "only_classified_unclassified": (ONLY_C, "0", [], "fq"),
    "only_classified_inverted": (ONLY_C, "9", ["-i"], "fq"),
    "filtered": (FILTERED, "9,0", [], "fq"),
}


def _universal(b: bytes) -> str:
    """the recorded stdout was read as text: '\\r\\n' and '\\r' became '\\n'"""
    return b.decode().replace("\r\n", "\n").replace("\r", "\n")


@pytest.mark.parametrize("case", sorted(CASES))
def test_extract_rules_match_krakenuniq_extract_reads(reference, tmp_path, case):
    kraken, taxa, opts, kind = CASES[case]
    (tmp_path / "in.kraken").write_bytes(kraken)
    (tmp_path / "taxDB").write_bytes(TAXDB)
    reads2 = None
    if kind == "paired":
        (tmp_path / "s_1.fq").write_bytes(MATE1)
        (tmp_path / "s_2.fq").write_bytes(MATE2)
        name, reads, reads2 = "s_%.fq", MATE1, MATE2
    elif kind == "gz":
        (tmp_path / "r.fq.gz").write_bytes(gzip.compress(FQ, mtime=0))
        name, reads = "r.fq.gz", FQ
    else:
        reads = {"fq": FQ, "fa": FA, "crlf": FQ.replace(b"\n", b"\r\n")}[kind]
        name = "r.fa" if kind == "fa" else "r.fq"
        (tmp_path / name).write_bytes(reads)
    args = [a for o in opts for a in ((o, "taxDB") if o == "-t" else (o,))] + ["--", taxa, "in.kraken", name]
    extract_reads.install_extract()
    r = reference.run_tool(extract_reads.SCRIPT, args, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    want = extract_reads.extract(kraken, taxa, reads, reads2, TAXDB if "-t" in opts else None, invert="-i" in opts,
                                 fasta_out="-f" in opts, fasta_in="-a" in opts)
    assert _universal(want) == r.stdout
    if case in ("absent", "absent_inverted", "only_classified_unclassified"):
        assert want == b""


def test_library_subtree_matches_the_restatement():
    rows = [l.split(b"\t")[:2] for l in TAXDB.split(b"\n") if l]
    taxid = [int(a) for a, _ in rows]
    parent = [int(b) for _, b in rows]
    kraken = b"".join(b"C\tx%d\t%d\t1\t1:1\n" % (t, t) for t in range(20))     # one line per taxon 0..19
    for taxa in ([9], [10], [1], [12, 9], [77], [0]):
        ids, _ = extract_reads.selected(kraken, ",".join(map(str, taxa)), TAXDB)
        got = binding.extract_taxa(taxa, binding.EXTRACT_SUBTREE, taxid, parent)
        assert sorted(int(i[1:]) for i in ids) == [t for t in got.tolist() if t < 20], taxa
    assert binding.extract_taxa([9], 0, taxid, parent).tolist() == [9]
    with pytest.raises(binding.KuqError):                             # 3 -> 4 -> 3 below 2
        binding.extract_taxa([2], binding.EXTRACT_SUBTREE, [3, 4, 3], [2, 3, 4])
    assert binding.extract_taxa([5], binding.EXTRACT_SUBTREE, [3, 4, 3], [2, 3, 4]).tolist() == [5]   # not reachable


def _classify(args, tmp_path):
    base = ["-d", "db.kdb", "-i", "db.idx"]
    return subprocess.run([build.build_classify()] + base + args, cwd=tmp_path, capture_output=True, text=True)


@pytest.mark.parametrize("args, msg", [
    (["-a", "taxDB", "--extract", "9", "reads.fq"], "--extract-out"),
    (["-a", "taxDB", "--extract-out", "x.fq", "reads.fq"], "need --extract"),
    (["-a", "taxDB", "--extract-invert", "reads.fq"], "need --extract"),
    (["--extract", "9", "--extract-out", "x.fq", "--extract-subtree", "reads.fq"], "-a"),
    (["-a", "taxDB", "--extract", "9", "--extract-out", "reads.fq", "reads.fq"], "one of the inputs"),
    (["-a", "taxDB", "-o", "o.kraken", "--extract", "9", "--extract-out", "o.kraken", "reads.fq"], "another output"),
    (["-a", "taxDB", "--extract", "9", "--extract-out", "-", "reads.fq"], "standard output"),
    (["-a", "taxDB", "--paired", "--extract", "9", "--extract-out", "x.fq", "m_1.fa", "m_2.fa"], "FASTQ mates"),
    (["-a", "cycle", "--extract", "9", "--extract-subtree", "--extract-out", "x.fq", "reads.fq"], "cycle"),
])
def test_extract_argument_checks_exit_64(tmp_path, args, msg):
    (tmp_path / "reads.fq").write_bytes(FQ)
    (tmp_path / "m_1.fa").write_bytes(b">a\nAC\n")
    (tmp_path / "m_2.fa").write_bytes(b">a\nGT\n")
    (tmp_path / "taxDB").write_bytes(TAXDB)
    (tmp_path / "cycle").write_bytes(b"1\t1\tr\tn\n9\t1\ta\tn\n20\t9\tb\tn\n21\t20\tc\tn\n20\t21\td\tn\n")
    r = _classify(args, tmp_path)
    assert r.returncode == 64 and msg in r.stderr, r.stderr
    assert not (tmp_path / "x.fq").exists()


def test_cycle_not_reachable_passes_the_checks(tmp_path):
    """a cycle below another taxon is no error: the run goes on to open the (missing) database"""
    (tmp_path / "reads.fq").write_bytes(FQ)
    (tmp_path / "cycle").write_bytes(b"1\t1\tr\tn\n9\t1\ta\tn\n20\t1\tb\tn\n21\t20\tc\tn\n20\t21\td\tn\n")
    r = _classify(["-a", "cycle", "--extract", "9", "--extract-subtree", "--extract-out", "x.fq", "reads.fq"], tmp_path)
    assert r.returncode not in (0, 64) and "cycle" not in r.stderr


@pytest.mark.parametrize("header, row, msg", [
    ("input\toutput\textract_out", "reads.fq\to.kraken\to.kraken", "both write"),
    ("input\textract_out", "reads.fq\treads.fq", "writes to one of the inputs"),
])
def test_sheet_extract_column_checks(tmp_path, header, row, msg):
    (tmp_path / "reads.fq").write_bytes(FQ)
    (tmp_path / "s.tsv").write_text(header + "\n" + row + "\n")
    r = _classify(["-a", "taxDB", "--extract", "9", "--sample-sheet", "s.tsv"], tmp_path)
    assert r.returncode == 64 and msg in r.stderr, r.stderr


def test_sheet_extract_column_needs_extract_and_the_other_way_round(tmp_path):
    (tmp_path / "reads.fq").write_bytes(FQ)
    (tmp_path / "s.tsv").write_text("input\textract_out\nreads.fq\tx.fq\n")
    r = _classify(["-a", "taxDB", "--sample-sheet", "s.tsv"], tmp_path)
    assert r.returncode == 64 and "needs --extract" in r.stderr
    (tmp_path / "t.tsv").write_text("input\toutput\nreads.fq\to.kraken\n")
    r = _classify(["-a", "taxDB", "--extract", "9", "--sample-sheet", "t.tsv"], tmp_path)
    assert r.returncode == 64 and "extract_out column" in r.stderr
    r = _classify(["-a", "taxDB", "--extract", "9", "--extract-out", "x.fq", "--sample-sheet", "s.tsv"], tmp_path)
    assert r.returncode == 64 and "column extract_out" in r.stderr
