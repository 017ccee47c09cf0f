"""The device digest and prefilter (sage_b200.digest_fasta, prefilter_fasta) against the restatement of Sage's Rust (digest_reference) and the
CPU oracle (oracle_digest), bit for bit, on the cases of digest_edges aimed at the kernels and on every digest_cases case inside Sage's
domain. The digest's stage counts (windows after the length filter, groups, candidates, rows before the merge) are compared with the
restatement's, so a wrong intermediate count is caught even where the final table agrees."""
import numpy as np
import pytest

import digest_cases as DC
import digest_edges as E
import digest_reference as R
import sage_b200
from oracle.oracle import ScorerConfig
from oracle_digest import digest_oracle
from sage_b200 import Peptides, SageB200Error, Tolerance, synth
from test_digest_reference import OUTSIDE

pytestmark = pytest.mark.gpu

ELIMIT = -5
COUNTS = (("n_windows", "windows"), ("n_groups", "groups"), ("n_candidates", "candidates"), ("n_rows", "rows"))


def assert_device_matches(fasta, kw, what):
    dev = sage_b200.digest_fasta(fasta, **kw)
    ref, st = R.digest_table(fasta, **kw)
    DC.assert_table_equal(dev, ref, f"{what} (restatement)")
    for dk, rk in COUNTS:
        assert dev.info[dk] == st[rk], f"{what}: {dk} {dev.info[dk]}, restatement {st[rk]}"
    DC.assert_table_equal(dev, digest_oracle.digest(fasta, **kw), f"{what} (oracle)")
    return dev


@pytest.mark.parametrize("name", sorted(E.EDGES))
def test_edges(name):
    assert_device_matches(*E.EDGES[name], name)


@pytest.mark.parametrize("name", sorted(set(DC.CASES) - set(OUTSIDE)))
def test_cases_with_stage_counts(name):
    assert_device_matches(*DC.CASES[name], name)


def test_reference_panics_are_empty_tables():
    for name, (fasta, kw) in E.EDGE_PANICS.items():
        dev = sage_b200.digest_fasta(fasta, **kw)
        assert len(dev.peptides) == 0, name


def test_edge_shapes():
    fasta, kw = E.EDGES["shared_by_320_proteins"]
    assert int(sage_b200.digest_fasta(fasta, **kw).n_proteins.max()) >= 320
    fasta, kw = E.EDGES["accessions_72000"]
    dev = sage_b200.digest_fasta(fasta, **kw)
    assert len(dev.names) >= 70000 and any(not n.isascii() for n in dev.names)
    fasta, kw = E.EDGES["forms_k8_8_sites"]   # ranks run to the last combination of k = 8: eight modified residues in one row
    P = sage_b200.digest_fasta(fasta, **kw).peptides
    per_row = np.add.reduceat((np.asarray(P.mods) != 0).astype(np.int64), np.asarray(P.seq_off[:-1], np.int64))
    assert per_row.max() == 8


def test_limits():
    fasta = E.EDGES["max_len_255"][0]
    for kw in (dict(max_len=256), dict(cleave_at="", max_len=256), dict(variable_mods={"S": [79.966331]}, max_variable_mods=9)):
        with pytest.raises(SageB200Error) as e:
            sage_b200.digest_fasta(fasta, **kw)
        assert e.value.code == ELIMIT, kw


# ------------------------------------------------------------------------------------------------ the prefilter
NARROW = dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))


def _spectra(fasta, kw, n: int, seed: int):
    t = digest_oracle.digest(fasta, **kw)
    return synth.make_spectra(Peptides(t["seq_off"], t["seq"], t["mods"], t["nterm"], t["mono"], t["decoy"], t["missed"]), n, seed=seed, n_peaks=60)


def run_prefilter(fasta, kw, spectra, chunk, low_memory, cfg=NARROW, min_peaks=15, reference=True):
    dev = sage_b200.prefilter_fasta(fasta, spectra, prefilter_chunk_size=chunk, prefilter_low_memory=low_memory, min_peaks=min_peaks, **cfg, **kw)
    rcfg = {k: (v.as_tuple() if hasattr(v, "as_tuple") else v) for k, v in cfg.items()}
    what = f"chunk {chunk} low_memory {low_memory}"
    sd = spectra.as_dict()
    refs = [("oracle", digest_oracle.prefilter(fasta, sd, ScorerConfig(**rcfg), chunk_size=chunk, low_memory=low_memory, min_peaks=min_peaks, **kw))]
    if reference:
        refs.append(("restatement", R.prefilter(fasta, sd, rcfg, chunk_size=chunk, low_memory=low_memory, min_peaks=min_peaks, **kw)))
    for who, (t, info) in refs:
        DC.assert_table_equal(dev, t, f"{what} ({who})")
        assert (dev.info["chunk_size"], dev.info["n_chunks"], dev.info["plain_build"]) == (info["chunk_size"], info["n_chunks"], info["plain_build"]), who
        assert np.array_equal(dev.chunk_rows, info["rows"]) and np.array_equal(dev.chunk_kept, info["kept"]), f"{what} ({who})"
    return dev


@pytest.mark.parametrize("low_memory", [True, False])
def test_prefilter_decoy_filter_every_chunk_size(low_memory):
    spectra = _spectra(E.DECOY_FASTA, E.DECOY_KW, 160, 21)
    n = len(R.fasta_parse(E.DECOY_FASTA).targets)
    for chunk in range(1, n + 1):
        run_prefilter(E.DECOY_FASTA, E.DECOY_KW, spectra, chunk, low_memory)


def test_prefilter_report_psms_limit_and_min_peaks():
    fasta, kw = DC.CASES["trypsin_missed1_static_c"]
    spectra = _spectra(fasta, kw, 40, 22)
    run_prefilter(fasta, kw, spectra, 5, True, cfg=dict(NARROW, report_psms=63))   # report_psms + 1 = 64, the largest the scorer holds
    with pytest.raises(SageB200Error) as e:
        sage_b200.prefilter_fasta(fasta, spectra, prefilter_chunk_size=5, report_psms=64, **NARROW, **kw)
    assert e.value.code == ELIMIT
    dev = run_prefilter(fasta, kw, spectra, 5, True, min_peaks=60)   # every spectrum has exactly 60 peaks: all are scored
    assert dev.info["n_spectra"] == len(spectra) and len(dev.peptides) > 0
    dev = run_prefilter(fasta, kw, spectra, 5, True, min_peaks=61)
    assert dev.info["n_spectra"] == 0 and len(dev.peptides) == 0


def test_prefilter_kept_table_doubles():
    # The kept table starts at 1 024 rows and doubles when a chunk's rows do not fit (PfTable::reserve in sage_b200.cu): with every chunk
    # keeping at most 1 024 rows and more than 4 096 kept in all, it doubles at least twice.
    fasta, kw = DC.random_fasta(240, 41), dict(missed_cleavages=1)
    spectra = _spectra(fasta, kw, 150, 3)
    cfg = dict(precursor_tol=Tolerance.da(-25, 25), fragment_tol=Tolerance.ppm(-20, 20))
    dev = run_prefilter(fasta, kw, spectra, 15, False, cfg=cfg)
    assert dev.chunk_kept.max() <= 1024 and dev.chunk_kept.sum() > 4096, dev.chunk_kept


def test_auto_chunk_size_skips_windows_off_character_boundaries():
    expect = R.fasta_auto_chunk_size(E.MULTIBYTE, **E.MULTIBYTE_AUTO_KW)
    assert expect == digest_oracle.auto_chunk_size(E.MULTIBYTE, **E.MULTIBYTE_AUTO_KW) and 0 < expect < 20
    dev = sage_b200.prefilter_fasta(E.MULTIBYTE, _spectra(E.MULTIBYTE, dict(E.LOOSE, cleave_at="", min_len=5, max_len=12), 8, 23),
                                    prefilter_chunk_size=0, **NARROW, **E.MULTIBYTE_AUTO_KW)
    assert dev.info["chunk_size"] == expect
