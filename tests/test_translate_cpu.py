"""krakenuniq-translate's rules (tests/translate.py) against the script's recorded output on the crafted taxonomy and
Kraken lines of tests/test_mpa_report_cpu.py: root-called lines before and after other lines, taxa without a row, a
walk that stops at a parent without a row, an empty read id, and the state that carries from one input file to the next."""
import pytest

from tests import mpa_report, translate
from tests.test_mpa_report_cpu import FILES, TAXDB


@pytest.mark.parametrize("flags", [[], ["--mpa-format"]], ids=["plain", "mpa_format"])
def test_translate_rules_match_krakenuniq_translate(reference, tmp_path, flags):
    mpa_report.write_db(tmp_path, TAXDB)
    for n, d in FILES.items():
        (tmp_path / n).write_bytes(d)
    translate.install_translate()
    for names in (["a.kraken"], ["b.kraken"], ["a.kraken", "b.kraken", "c.kraken"]):
        r = reference.run_tool(translate.TRANSLATE, ["--db", "."] + flags + names, cwd=tmp_path)
        assert r.returncode == 0, r.stderr
        want = translate.translate(b"".join(FILES[n] for n in names), TAXDB, bool(flags))
        assert want.decode() == r.stdout


def test_root_called_lines_take_the_last_stored_lineage():
    """the script's cache: a root-called line prints the lineage of the last walk that stopped at the root"""
    out = translate.translate(FILES["a.kraken"], TAXDB).split(b"\n")
    got = dict(l.split(b"\t") for l in out if l)
    assert got[b"root_first"] == got[b"root_again"] == b""
    assert got[b"root_after"] == got[b"root_after2"] == got[b"sp1"] == b"Bacteria;Terra|bacteria;Phylum one;Class.A;Order x;Fam ily;Genus g.;Genus g. species one"
    assert got[b"9"] == got[b"sp1"][:-len(b"Genus g. species one")] + b"length species"     # empty id: taxid = length
