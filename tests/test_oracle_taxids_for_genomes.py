"""set_lcas -a / -A (krakenuniq-build --taxids-for-sequences / --taxids-for-genomes): the oracle's restatement of the
taxonomy extension (oracle/taxids.py) and its set_lcas against the unmodified reference set_lcas (recorded runs,
tests/ref_replay.py) on build_db.sh's command line: rewritten taxDB, stdout, database and .counts, byte for byte."""
import numpy as np
import pytest

from krakenuniq_b200 import synth
from oracle.taxids import Extension
from tests import taxid_cases as tc


@pytest.mark.parametrize("case", list(tc.CASES))
def test_oracle_matches_reference(oracle, reference, tmp_path, case):
    a, A, T, E = tc.CASES[case]
    ref, pristine, r = tc.run_reference(reference, tmp_path, case)
    ext, kdb, counts = tc.expected(oracle, pristine, a, A, T, tc.MIN_LEN if E else 0)
    got_kdb, got_taxdb, got_counts = tc.outputs(ref)
    assert r.stdout == ext.stdout
    assert got_taxdb.decode() == ext.taxdb_text()
    assert np.array_equal(np.frombuffer(got_kdb, np.uint8), kdb)
    assert got_counts.decode() == counts
    assert open(ref / "database0.kdb", "rb").read() == open(pristine / "database0.kdb", "rb").read()
    assert "[starting new taxonomy IDs with 1000000001]" in r.stderr

    # what the cases hold: new taxa of both ranks, the map's stdout lines, the renamed taxa
    rows = {t: (p, n, rk) for t, p, n, rk in ext.rows()}
    new = {t: v for t, v in rows.items() if t > 1_000_000_000}
    sp = synth.species_ids(synth.Taxonomy.read(str(pristine / "taxDB")))
    lines = dict(line.split("\t") for line in r.stdout.splitlines())
    assert len(lines) == 13                                          # 14 map lines, one repeated seq id
    assert "parent taxon 4242 not in database" in r.stderr
    if A:
        asm = {n: t for t, (p, n, rk) in new.items() if rk == "assembly"}
        assert rows[asm["asm0"]][0] == sp[0] and rows[asm["GRCh38"]][0] == 9606
        assert rows[asm["s5"]][0] == sp[3]                             # the assembly named like a seq id
        assert "asm6" not in asm and "asm_dup" not in asm              # parent missing; repeated seq id
        assert rows[int(lines["hs1"])][1] == "GRCh38"                   # human: never renamed
    if a:
        assert rows[int(lines["hs1"])][2] != "sequence"                 # no sequence taxa for human / mouse
        assert int(lines["mm1"]) == 10090
        assert rows[int(lines["hs2"])][1] == "hs2 neanderthal"          # a child of 9606 is renamed
        assert rows[sp[3]][1] == f"kraken:taxid|{sp[3]}|x  extra words"   # kraken:taxid| header, blanks trimmed
        assert rows[int(lines["short1"])][1] == "short1" or not E       # too short (-E): not renamed
        if A:
            assert int(lines["s5"]) == asm["s5"]                         # the seq id finds the assembly of that name
            assert rows[int(lines["s6"])][0] == 0                        # under 'unclassified' after the failed assembly
        else:
            assert rows[int(lines["s5"])][0] == sp[4]
    if not (a and A):
        assert lines["s6"] == "0"                                        # a new taxon under 4242 fails: skipped
    if T:
        _, keys, vals = synth.parse_kdb(kdb)
        assert (32630 in vals.tolist()) == (not a)                        # -a: the contaminant lost its stickiness


def test_extension_refuses_pseudo_ids():
    rows = [(1, 1, "root", "no rank"), (1_000_000_005, 1, "x", "sequence")]
    with pytest.raises(ValueError):
        Extension(rows, ["s\t1"], True, False)
    Extension(rows, ["s\t1"], False, False)                              # no new taxa: no start id needed
