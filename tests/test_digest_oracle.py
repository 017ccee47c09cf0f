"""The oracle's bulk digest accessors (oracle_digest) against its per-protein export (OracleDB.peptide_proteins) and table export, on the
picked_cases FASTA databases; and its digest() alone against the digest inside OracleDB.from_fasta."""
import numpy as np
import pytest

import digest_cases as DC
import picked_cases as PC
from oracle_digest import digest_oracle


@pytest.mark.parametrize("generate_decoys", [True, False])
@pytest.mark.parametrize("seed", [3, 17])
def test_bulk_accessors_match_per_protein_export(seed, generate_decoys):
    case = PC.fasta_case(seed, generate_decoys)
    db = case["db"]
    t = digest_oracle.db_table(db)
    assert [[x.decode() for x in lst] for lst in digest_oracle.protein_lists(t)] == [db.peptide_proteins(i) for i in range(db.n_peptides)]
    assert not t["semi"].any()
    e = db.export()
    for k, ek in (("seq_off", "seq_off"), ("seq", "seq"), ("decoy", "decoy"), ("missed", "missed")):
        assert np.array_equal(t[k], e[ek])
    for k, ek in (("mods", "mods"), ("nterm", "nterm"), ("cterm", "cterm"), ("mono", "pep_mono")):
        assert np.array_equal(t[k].view(np.uint32), e[ek].view(np.uint32))
    alone = digest_oracle.digest(DC.picked_fasta_text(seed, generate_decoys), generate_decoys=generate_decoys, **DC.PICKED_KW)
    for k in t:
        assert np.array_equal(alone[k], t[k]) if alone[k].dtype != np.float32 else np.array_equal(alone[k].view(np.uint32), t[k].view(np.uint32))


def test_semi_enzymatic_flags():
    fasta, kw = DC.CASES["semi_missed0"]
    t = digest_oracle.digest(fasta, **kw)
    assert t["semi"].any() and not t["semi"].all()
