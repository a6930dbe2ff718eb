"""`classify --extract`: the extracted file must be what krakenuniq-extract-reads (restated in tests/extract_reads.py)
prints from the same run's Kraken lines and inputs, and every other output (Kraken lines, report, -C, -U, stats) must
be the bytes of the run without --extract, in every layout.  The C ABI's extract_sel / n_extract are checked directly."""
import collections
import gzip
import os
import shutil
import subprocess

import numpy as np
import pytest

from krakenuniq_b200 import binding
from tests import extract_reads, paired, util
from tests.test_threshold_gpu import LAYOUTS, _copy, _exe, _setup, _stats, synthetic  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
G = util.GOLDEN
OUTS = ("-o", "-r", "-C", "-U")


def _run(tmp_path, tool, common, extra, tag, inputs, env):
    files = sum(([o, f"{tag}{o}"] for o in OUTS), [])
    r = subprocess.run([_exe(tool)] + common + extra + files + inputs, cwd=tmp_path, capture_output=True, text=True,
                       env=dict(os.environ, **env))
    assert r.returncode == 0, r.stderr[-2000:]
    assert "not usable" not in r.stderr
    return r


def _taxa(kraken: bytes):
    """the most frequent call and taxon 0: some lines are selected, some are not"""
    calls = collections.Counter(l.split(b"\t")[2] for l in kraken.splitlines())
    top = [t for t, _ in calls.most_common() if t != b"0"][0]
    return top.decode() + ",0"


def _compare(tmp_path, tool, dbs, flags, env, inputs, xflags=(), taxa=None, out="ext.x", mates=False):
    """runs without and with --extract; checks the extracted file and the unchanged outputs.  Returns the base Kraken
    lines and the taxa."""
    common = sum((["-d", f"{d}.kdb", "-i", f"{d}.idx"] for d in dbs), []) + ["-a", "taxDB"] + flags
    base = _run(tmp_path, tool, common, [], "base", inputs, env)
    kraken = (tmp_path / "base-o").read_bytes()
    assert kraken
    taxa = taxa or _taxa(kraken)
    ext = _run(tmp_path, tool, common, ["--extract", taxa, "--extract-out", out] + list(xflags), "ext", inputs, env)
    for o in OUTS:
        assert (tmp_path / f"ext{o}").read_bytes() == (tmp_path / f"base{o}").read_bytes(), o
    assert _stats(ext.stderr) == _stats(base.stderr)
    taxdb = (tmp_path / "taxDB").read_bytes() if "--extract-subtree" in xflags else None
    opts = dict(taxdb=taxdb, invert="--extract-invert" in xflags, fasta_out="--extract-fasta" in xflags)
    if mates:
        want = extract_reads.extract(kraken, taxa, extract_reads.read_input(tmp_path / inputs[0]),
                                     extract_reads.read_input(tmp_path / inputs[1]), **opts)
    else:
        want = b""
        for f in inputs:
            data = extract_reads.read_input(tmp_path / f)
            want += extract_reads.extract(kraken, taxa, data, fasta_in=data[:1] == b">", **opts)
    got = extract_reads.read_input(tmp_path / out)
    assert got == want
    return kraken, taxa, want


XFLAGS = [(), ("--extract-invert",), ("--extract-fasta",), ("--extract-subtree",), ("--extract-invert", "--extract-fasta")]


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_layouts(tmp_path, layout):
    tool, dbs, flags, env = LAYOUTS[layout]
    _setup(tmp_path, dbs)
    xflags = XFLAGS[list(LAYOUTS).index(layout) % len(XFLAGS)]
    _, _, want = _compare(tmp_path, tool, dbs, flags, env, ["reads.fa", "reads_crlf_60.fa", "reads_300.fq"], xflags)
    assert want


@pytest.mark.parametrize("xflags", XFLAGS[:3])
def test_paired(tmp_path, xflags):
    _setup(tmp_path)
    ids, seqs = util.read_fasta(os.path.join(G, "reads.fa"))
    pairs = paired.split_pairs(seqs, np.random.default_rng(5))
    (tmp_path / "m_1.fq").write_bytes(paired.fastq_bytes([(f"{i}/1".encode(), a) for i, (a, _) in zip(ids, pairs)]))
    (tmp_path / "m_2.fq").write_bytes(paired.fastq_bytes([(f"{i}/2".encode(), b) for i, (_, b) in zip(ids, pairs)]))
    for env in ({}, {"KUQ_SERIAL_INGEST": "1"}):
        _, _, want = _compare(tmp_path, "classify", ["database"], ["-M", "--paired"], env, ["m_1.fq", "m_2.fq"], xflags,
                              mates=True)
        assert want


def test_gzip_inputs_and_output(tmp_path):
    _setup(tmp_path)
    for f in ("reads.fa", "reads_300.fq"):
        (tmp_path / (f + ".gz")).write_bytes(gzip.compress((tmp_path / f).read_bytes()))
    _compare(tmp_path, "classify", ["database"], ["-M"], {}, ["reads.fa.gz", "reads_300.fq.gz"], out="ext.x.gz")
    assert (tmp_path / "ext.x.gz").read_bytes()[:2] == b"\x1f\x8b"


def test_nothing_matched_writes_nothing(tmp_path):
    _setup(tmp_path)
    for xflags in ((), ("--extract-invert",)):
        _compare(tmp_path, "classify", ["database"], ["-M"], {"KUQ_BATCH_READS": "50"}, ["reads_300.fq"], xflags,
                 taxa="4000000000")
        assert (tmp_path / "ext.x").read_bytes() == b""


def test_threshold_moves_reads(tmp_path):
    """extraction follows the filtered calls: some read enters or leaves the set through the filter"""
    _setup(tmp_path)
    plain, taxa, _ = _compare(tmp_path, "classify", ["database"], ["-M"], {}, ["reads.fa", "reads_300.fq"])
    filt, _, _ = _compare(tmp_path, "classify", ["database"], ["-M", "--threshold", "0.5"], {}, ["reads.fa", "reads_300.fq"],
                          taxa=taxa)
    keys = set(taxa.encode().split(b","))
    sel = lambda k: [l.split(b"\t")[2] in keys for l in k.splitlines()]
    assert sel(plain) != sel(filt)


def test_sample_sheet(tmp_path):
    """--extract applies to every row with an extract_out cell; an empty cell extracts nothing"""
    _setup(tmp_path)
    common = [_exe(), "-d", "database.kdb", "-i", "database.idx", "-a", "taxDB", "-M"]
    r = subprocess.run(common + ["-o", "probe.kraken", "reads.fa"], cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 0
    taxa = _taxa((tmp_path / "probe.kraken").read_bytes())
    sheet = tmp_path / "s.tsv"
    sheet.write_text("name\tinput\toutput\treport\textract_out\n"
                     "a\treads.fa\ta.kraken\ta.report\ta.x\n"
                     "b\treads_300.fq,reads_crlf_60.fa\tb.kraken\tb.report\t\n"
                     "c\treads_300.fq\tc.kraken\tc.report\tc.x.gz\n")
    base = tmp_path / "base.tsv"
    base.write_text("\n".join("\t".join(l.split("\t")[:4]) for l in sheet.read_text().splitlines()) + "\n")
    for s in (base, sheet):
        extra = ["--extract", taxa, "--extract-invert"] if s == sheet else []
        r = subprocess.run(common + extra + ["--sample-sheet", s.name], cwd=tmp_path, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        if s == base:                                                 # (the report is appended to: start afresh)
            keep = {row: ((tmp_path / f"{row}.kraken").read_bytes(), (tmp_path / f"{row}.report").read_bytes()) for row in "abc"}
            for row in "abc":
                (tmp_path / f"{row}.report").unlink()
    for row in "abc":
        assert ((tmp_path / f"{row}.kraken").read_bytes(), (tmp_path / f"{row}.report").read_bytes()) == keep[row]
    for row, f, out in (("a", "reads.fa", "a.x"), ("c", "reads_300.fq", "c.x.gz")):
        data = (tmp_path / f).read_bytes()
        want = extract_reads.extract(keep[row][0], taxa, data, invert=True, fasta_in=data[:1] == b">")
        assert extract_reads.read_input(tmp_path / out) == want and want
    assert not (tmp_path / "b.x").exists()


def test_synthetic_subtree(tmp_path, synthetic):
    """2400 species, reads over more than 32 taxa; the list holds genera and a family, with their subtrees"""
    _copy(synthetic[0], tmp_path)
    tax = synthetic[1]
    genera = [r[0] for r in tax.rows if r[3] == "genus"][:5]
    family = [r[0] for r in tax.rows if r[3] == "family"][2]
    taxa = ",".join(str(t) for t in genera + [family])
    for xflags in (("--extract-subtree",), ("--extract-subtree", "--extract-invert")):
        _, _, want = _compare(tmp_path, "classify", ["database"], ["-M"], {}, ["reads.fa"], xflags, taxa=taxa)
        assert want


def test_c_abi_result_arrays(tmp_path, synthetic):
    """extract_sel and n_extract from kuq_classify_batch against the restatement of the batch's calls; no arrays and no
    extra launch without kuq_set_extract, one launch per batch with it"""
    _copy(synthetic[0], tmp_path)
    tax = synthetic[1]
    kdb = np.fromfile(tmp_path / "database.kdb", np.uint8)
    idx = np.fromfile(tmp_path / "database.idx", np.uint8)
    seqs = (tmp_path / "reads.fa").read_bytes().split(b"\n")[1::2]
    bases = np.frombuffer(b"".join(seqs), np.uint8)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.uint64)
    rows = np.array([(r[0], r[1]) for r in tax.rows], np.uint32)
    genera = [int(r[0]) for r in tax.rows if r[3] == "genus"][:3]
    launches = {}
    for flags in (None, binding.EXTRACT_SUBTREE, binding.EXTRACT_SUBTREE | binding.EXTRACT_INVERT | binding.EXTRACT_CLASSIFIED_ONLY,
                  binding.EXTRACT_OTHERS | binding.EXTRACT_CLASSIFIED_ONLY):
        c = binding.Classifier(device=0, max_reads=1 << 14, max_bases=4 << 20)
        c.stage_db(kdb, idx)
        c.set_taxonomy(*tax.parent_map())
        if flags is not None:
            c.set_extract(genera, flags, rows[:, 0], rows[:, 1])
        l0 = c.launch_count()
        res = c.classify(bases, offs)
        launches[flags] = c.launch_count() - l0
        if flags is None:
            assert "extract_sel" not in res
            c.close()
            continue
        members = set(binding.extract_taxa(genera, flags, rows[:, 0], rows[:, 1]).tolist())
        call = res["call"].astype(np.int64)
        line = (call != 0) | (flags & binding.EXTRACT_CLASSIFIED_ONLY == 0)
        sel = line & ((flags & binding.EXTRACT_OTHERS != 0) | np.isin(call, list(members)))
        assert res["n_extract"] == int(sel.sum()) and 0 < sel.sum() < len(seqs)
        want = (sel ^ bool(flags & binding.EXTRACT_INVERT)).astype(np.uint8) | np.where(line, 0, 2).astype(np.uint8)
        assert np.array_equal(res["extract_sel"], want)
        c.close()
    assert all(v == launches[None] + 1 for k, v in launches.items() if k is not None)


def test_c_abi_refuses_a_reachable_cycle():
    c = binding.Classifier(device=0, max_reads=1 << 10, max_bases=1 << 20)
    c.set_taxonomy(np.array([1, 2, 3], np.uint32), np.array([0, 1, 2], np.uint32))
    with pytest.raises(binding.KuqError) as e:
        c.set_extract([2], binding.EXTRACT_SUBTREE, np.array([1, 2, 3, 2], np.uint32), np.array([1, 1, 2, 3], np.uint32))
    assert e.value.code == -10
    c.set_extract([2], 0, np.array([1, 2, 3, 2], np.uint32), np.array([1, 1, 2, 3], np.uint32))    # no subtree: no walk
    c.close()
