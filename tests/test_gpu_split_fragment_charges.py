"""Split scoring (k_score<true> -> k_fold -> k_features -> k_rows) with three and more fragment charges per candidate. The hit emit of k_score<true>
decodes a task's ion index by the candidate's fragment-charge count (1, 2, 3, and a general division above), so precursors of charge 2 to 6 are
scored through every branch and must give the fused kernel's rows and the oracle's."""
import dataclasses

import numpy as np
import pytest

from sage_b200 import IndexedDatabase, Scorer, Tolerance, synth

from helpers import assert_features_equal, f64_exact_default, oracle_cfg, oracle_db_from_peptides, valid_rows

pytestmark = pytest.mark.gpu


def test_split_scoring_equals_fused_and_oracle_at_precursor_charges_2_to_6():
    pep = synth.make_peptides(20000, seed=11, static_c=True)
    spectra = synth.make_spectra(pep, 1500, seed=12)
    # the same precursor masses at charges 2..6 (fragment charges 1..5 searched per candidate)
    z_old = spectra.prec_charge.astype(np.float64)
    z = np.random.default_rng(13).integers(2, 7, len(spectra)).astype(spectra.prec_charge.dtype)
    mass = (spectra.prec_mz.astype(np.float64) - float(synth.PROTON)) * z_old
    spectra = dataclasses.replace(spectra, prec_charge=z, prec_mz=((mass + z * float(synth.PROTON)) / z).astype(np.float32))
    gdb = IndexedDatabase.build_from_peptides(pep)
    odb = oracle_db_from_peptides(pep)
    kw = dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), max_precursor_charge=6, report_psms=2)
    fused = Scorer(gdb, **kw)
    fused.set_option("score_split", 0)
    ff, fc = fused.score_batch(spectra)
    ff, fc = valid_rows(ff, fc, 2).copy(), fc.copy()
    assert (ff["charge"] >= 4).sum() > 100, "too few PSMs with three or more fragment charges"
    for fast in (1, 0):
        sc = Scorer(gdb, **kw)
        sc.set_option("score_fast", fast)
        f, c = sc.score_batch(spectra)
        assert np.array_equal(c, fc) and valid_rows(f, c, 2).tobytes() == ff.tobytes(), fast
    of, oc, _, _ = odb.score_batch(oracle_cfg(**kw), spectra.as_dict())
    assert assert_features_equal(f, c, of, oc, 2, what="precursor charges 2..6", f64_exact=f64_exact_default(0)) > 1000
