"""The device digest (sage_b200.digest_fasta, IndexedDatabase.from_fasta) against the CPU oracle's digest(): every array bit for bit,
protein lists as names in order with duplicates, semi_enzymatic; the index built from the digested table; the protein fields picked_fdr
reads on picked_cases' FASTA databases."""
import numpy as np
import pytest

import digest_cases as DC
import picked_cases as PC
import sage_b200
from oracle_digest import digest_oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(DC.CASES))
def test_digest_matches_oracle(name):
    fasta, kw = DC.CASES[name]
    dev = sage_b200.digest_fasta(fasta, **kw)
    DC.assert_table_equal(dev, digest_oracle.digest(fasta, **kw), name)


def test_long_equal_mass_run_is_sorted_exactly():
    fasta, kw = DC.CASES["long_equal_mass_run"]
    dev = sage_b200.digest_fasta(fasta, **kw)
    _, counts = np.unique(dev.peptides.mono.view(np.uint32), return_counts=True)
    assert counts.max() >= 5000


def test_empty_results():
    for fasta, kw in (DC.CASES["empty_fasta"], DC.CASES["min_above_max"], (">A\n>B\n", {})):
        dev = sage_b200.digest_fasta(fasta, **kw)
        assert len(dev.peptides) == 0 and list(dev.protein_offsets) == [0] and list(dev.peptides.seq_off) == [0]


@pytest.mark.parametrize("name", ["trypsin_missed1_static_c", "variable_mixed", "semi_missed2", "tagged_no_generate"])
def test_from_fasta_index_matches_oracle(name):
    from oracle.oracle import OracleDB
    fasta, kw = DC.CASES[name]
    db = sage_b200.IndexedDatabase.from_fasta(fasta, bucket_size=3000, **kw)
    ref = OracleDB.from_fasta(fasta if isinstance(fasta, str) else fasta.decode("latin-1"), bucket_size=3000, **kw).export()
    fp, fm, bm = db.export_index()
    assert np.array_equal(fp, ref["frag_pep"])
    assert np.array_equal(fm.view(np.uint32), ref["frag_mz"].view(np.uint32))
    assert np.array_equal(bm.view(np.uint32), ref["bucket_min"].view(np.uint32))
    assert db.digest.peptides is db.peptides


@pytest.mark.parametrize("generate_decoys", [True, False])
@pytest.mark.parametrize("seed", [3, 17])
def test_picked_fields_match_fasta_case(seed, generate_decoys):
    case = PC.fasta_case(seed, generate_decoys)
    dev = sage_b200.digest_fasta(DC.picked_fasta_text(seed, generate_decoys), generate_decoys=generate_decoys, **DC.PICKED_KW)
    assert np.array_equal(dev.n_proteins, case["n_proteins"])
    assert np.array_equal(DC._bits(dev.cterm), DC._bits(case["cterm"]))
    one = np.nonzero(case["n_proteins"] == 1)[0]
    assert [dev.names[dev.protein[i]] for i in one] == [case["proteins"][i][0] for i in one]
    assert [dev.proteins(i) for i in range(len(dev.peptides))] == case["proteins"]


def test_human_size_matches_oracle():
    fasta = DC.human_fasta()
    dev = sage_b200.digest_fasta(fasta, **DC.HUMAN_MODS)
    assert len(dev.peptides) > 4_000_000
    DC.assert_table_equal(dev, digest_oracle.digest(fasta, **DC.HUMAN_MODS), "human")
