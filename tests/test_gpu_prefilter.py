"""The device prefilter (sage_b200.prefilter_fasta, IndexedDatabase.from_fasta(prefilter=True)) against the oracle's restatement of
runner.rs:104-128, 161-278 (oracle_digest.prefilter): the table bit for bit with its protein lists as names, the per-chunk counts, the
automatic chunk size, the final index, the PSMs scored on it and the protein fields picked_fdr reads. Spectra come from the device digest
of the same FASTA (synth.make_spectra) plus noise, so that peptides of several chunks are selected."""
import numpy as np
import pytest

import digest_cases as DC
import sage_b200
from helpers import assert_features_equal, oracle_cfg, oracle_db_from_peptides
from oracle_digest import digest_oracle
from sage_b200 import Peptides, SageB200Error, SpectraBatch, Tolerance, synth

pytestmark = pytest.mark.gpu

EINVAL = -1
NARROW = dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))
WIDE = dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), wide_window=True, max_precursor_charge=3, report_psms=2)


def _concat(batches) -> SpectraBatch:
    off = [np.zeros(1, np.uint64)]
    base = 0
    for b in batches:
        off.append(b.peak_off[1:].astype(np.uint64) + np.uint64(base))
        base += int(b.peak_off[-1])
    cat = lambda k: np.concatenate([getattr(b, k) for b in batches])  # noqa: E731
    lv = None if all(b.level is None for b in batches) else np.concatenate([b.level if b.level is not None else np.full(len(b), 2, np.uint8) for b in batches])
    return SpectraBatch(np.concatenate(off), cat("masses"), cat("intensities"), cat("prec_mz"), cat("prec_charge"), cat("iso_lo"), cat("iso_hi"), cat("tic"),
                        level=lv)


def _noise(n: int, seed: int, peaks: int = 40) -> SpectraBatch:
    rng = np.random.default_rng(seed)
    masses = np.sort(rng.uniform(150.0, 1800.0, (n, peaks)).astype(np.float32), axis=1).ravel()
    return SpectraBatch(np.arange(n + 1, dtype=np.uint64) * peaks, masses, rng.lognormal(3.0, 1.0, n * peaks).astype(np.float32),
                        rng.uniform(400.0, 1200.0, n).astype(np.float32), np.full(n, 2, np.uint8), np.full(n, np.nan, np.float32),
                        np.full(n, np.nan, np.float32), np.full(n, 1000.0, np.float32))


def _spectra(fasta, kw, n: int, seed: int, noise: int = 16) -> SpectraBatch:
    d = sage_b200.digest_fasta(fasta, **kw)
    parts = [_noise(noise, seed + 1)] if noise else []
    if len(d.peptides) and n:
        parts.insert(0, synth.make_spectra(d.peptides, n, seed=seed, n_peaks=60))
    return _concat(parts) if parts else _noise(0, seed)


def _run(fasta, spectra, kw, chunk, low_memory, cfg=NARROW, min_peaks=15):
    dev = sage_b200.prefilter_fasta(fasta, spectra, prefilter_chunk_size=chunk, prefilter_low_memory=low_memory, min_peaks=min_peaks, **cfg, **kw)
    scfg = {k: v for k, v in cfg.items()}
    ref = digest_oracle.prefilter(fasta, spectra.as_dict(), oracle_cfg(**scfg), chunk_size=chunk, low_memory=low_memory, min_peaks=min_peaks, **kw)
    assert ref is not None
    t, info = ref
    DC.assert_table_equal(dev, t, f"chunk {chunk} low_memory {low_memory}")
    assert dev.info["chunk_size"] == info["chunk_size"] and dev.info["plain_build"] == info["plain_build"]
    assert dev.info["n_chunks"] == info["n_chunks"]
    assert np.array_equal(dev.chunk_rows, info["rows"]) and np.array_equal(dev.chunk_kept, info["kept"])
    assert dev.info["rows_kept"] == int(info["kept"].sum()) or info["plain_build"]
    return dev, t, info


def _n_proteins(fasta, kw) -> int:
    return int(sage_b200.digest_fasta(fasta, **kw).info["n_proteins"])


TABLE_CASES = ["trypsin_missed1_static_c", "variable_mixed", "semi_missed0", "tagged_no_generate", "structure", "duplicate_accessions"]


@pytest.mark.parametrize("low_memory", [True, False])
@pytest.mark.parametrize("name", TABLE_CASES)
def test_tables_match_oracle(name, low_memory):
    fasta, kw = DC.CASES[name]
    n = _n_proteins(fasta, kw)
    spectra = _spectra(fasta, kw, 96, 40 + len(name))
    for chunk in sorted({1, 2, 3, 7, max(1, n - 1), n, 0}):
        _run(fasta, spectra, kw, chunk, low_memory)


# ANMLHGFEDK (a target of P2) is Peptide::reverse of ADEFGHLMNK (a target of P1; in P3 a proline follows its K): with one protein per
# chunk, the decoy of chunk P1 survives its decoy filter and the merge joins it with P2's target into one target row. GGGGGR is in both entries
# of the repeated accession P1.
CROSS = ">P1\nMKADEFGHLMNKGGGGGR\n>P2\nMRANMLHGFEDKWWWWWR\n>P3\nMKADEFGHLMNKPEPTIDEKR\n>P1\nLLLLLLLKGGGGGR\n"


def test_cross_chunk_target_and_decoy_merge():
    kw = dict(min_len=3, peptide_min_mass=0.0)
    spectra = _spectra(CROSS, kw, 200, 7, noise=8)
    for low_memory in (True, False):
        for chunk in (1, 2, 3):
            dev, _, _ = _run(CROSS, spectra, kw, chunk, low_memory)
            if chunk == 1 and not low_memory:
                row = {dev.peptides.sequence(i): i for i in range(len(dev.peptides))}
                i = row["ANMLHGFEDK"]
                assert dev.proteins(i) == ["P1", "P2"] and dev.peptides.decoy[i] == 0
                assert dev.proteins(row["GGGGGR"]) == ["P1", "P1"]


def test_same_peptide_many_chunks_and_equal_mass_runs():
    fasta = "".join(f">P{i}\nPEPTIDEKPEPTLDEKGGGK{'AC' * i}MSTYR\n" for i in range(9))
    kw = dict(min_len=3, peptide_min_mass=0.0, variable_mods={"M": [15.9949], "S": [79.966331], "T": [79.966331]}, max_variable_mods=2)
    spectra = _spectra(fasta, kw, 200, 8)
    for chunk in (1, 2, 4):
        dev, _, _ = _run(fasta, spectra, kw, chunk, False)
        assert max(len(dev.proteins(i)) for i in range(len(dev.peptides))) >= 5
        key = dev.peptides.mono.view(np.uint32)
        assert len(np.unique(key)) < len(key)   # an equal-mass run (PEPTIDEK / PEPTLDEK) that spans chunks


def test_filtered_chunks_and_empty_results():
    fasta, kw = DC.CASES["trypsin_missed1_static_c"]
    spectra = _spectra(fasta, kw, 4, 9, noise=0)
    dev, _, _ = _run(fasta, spectra, kw, 1, True)
    assert ((dev.chunk_kept == 0) & (dev.chunk_rows > 0)).any()   # a chunk whose every peptide is filtered
    for sp in (_noise(0, 1), _noise(32, 2)):                       # no spectra; spectra that match nothing
        dev, _, _ = _run(fasta, sp, kw, 3, True)
        assert len(dev.peptides) == 0 and list(dev.protein_offsets) == [0] and dev.db.info["n_peptides"] == 0
    dev = sage_b200.prefilter_fasta("", spectra, prefilter_chunk_size=0, **NARROW)   # an empty FASTA
    assert len(dev.peptides) == 0 and dev.info["plain_build"] == 1


def test_min_peaks_and_ms1_spectra_are_not_scored():
    fasta, kw = DC.CASES["variable_mixed"]
    spectra = _spectra(fasta, kw, 64, 10)
    dev, _, _ = _run(fasta, spectra, kw, 4, True, min_peaks=61)
    assert dev.info["n_spectra"] == 0 and len(dev.peptides) == 0
    spectra.level = np.where(np.arange(len(spectra)) % 3 == 0, 1, 2).astype(np.uint8)
    dev, _, _ = _run(fasta, spectra, kw, 4, False)
    assert dev.info["n_spectra"] == int((spectra.level == 2).sum())


AUTO_CASES = [
    (DC.random_fasta(800, 21), dict(DC.HUMAN_MODS, variable_mods={"M": [15.9949], "[": [42.010565], "^Q": [-17.026549], "W": [3.0]}, max_variable_mods=5)),
    (DC.random_fasta(800, 22), dict(missed_cleavages=2, variable_mods={"M": [15.9949, 31.98, 47.97], "[": [42.010565]}, max_variable_mods=7)),
    (DC.random_fasta(300, 23), dict(semi_enzymatic=True, variable_mods={"M": [15.9949]}, max_variable_mods=4)),
    (DC.random_fasta(200, 24), dict(DC.HUMAN_MODS)),
]


@pytest.mark.parametrize("case", range(len(AUTO_CASES)))
def test_auto_chunk_size(case):
    fasta, kw = AUTO_CASES[case]
    expect = digest_oracle.auto_chunk_size(fasta, **kw)
    dev = sage_b200.prefilter_fasta(fasta, _noise(8, case), prefilter_chunk_size=0, **NARROW, **kw)
    assert dev.info["chunk_size"] == expect
    assert dev.info["plain_build"] == int(expect >= dev.info["n_proteins"])


def test_auto_chunk_size_human():
    fasta = DC.human_fasta()
    expect = digest_oracle.auto_chunk_size(fasta, **DC.HUMAN_MODS)
    dev = sage_b200.prefilter_fasta(fasta, _noise(0, 3), prefilter_chunk_size=0, **NARROW, **DC.HUMAN_MODS)
    assert dev.info["chunk_size"] == expect and dev.info["n_chunks"] > 1


def test_zero_automatic_chunk_size_is_einval():
    rng = np.random.default_rng(11)
    fasta = "".join(f">P{i}\n" + "".join(rng.choice(list(DC.AA), 1000)) + "\n" for i in range(2))
    kw = dict(cleave_at="", min_len=5, max_len=50, max_variable_mods=8,
              variable_mods={c: [float(i + 1)] for i, c in enumerate("ACDEFGHIKLMN")})
    assert digest_oracle.auto_chunk_size(fasta, **kw) == 0
    with pytest.raises(SageB200Error) as e:
        sage_b200.prefilter_fasta(fasta, _noise(4, 1), **NARROW, **kw)
    assert e.value.code == EINVAL


def _oracle_peptides(t) -> Peptides:
    return Peptides(t["seq_off"], t["seq"], t["mods"], t["nterm"], t["mono"], t["decoy"], t["missed"])


@pytest.mark.parametrize("cfg", ["narrow", "wide"])
def test_final_index_and_search_match_oracle(cfg):
    fasta, kw = DC.CASES["size_medium_mods"]
    c = NARROW if cfg == "narrow" else WIDE
    spectra = _spectra(fasta, kw, 400, 12)
    dev, t, _ = _run(fasta, spectra, kw, 150, True, cfg=c)
    assert len(dev.peptides) > 100 and dev.info["n_chunks"] > 2
    odb = oracle_db_from_peptides(_oracle_peptides(t))
    ref = odb.export()
    fp, fm, bm = dev.db.export_index()
    assert np.array_equal(fp, ref["frag_pep"])
    assert np.array_equal(fm.view(np.uint32), ref["frag_mz"].view(np.uint32))
    assert np.array_equal(bm.view(np.uint32), ref["bucket_min"].view(np.uint32))
    hp, hm, hb = sage_b200.IndexedDatabase.build_from_peptides(dev.peptides).export_index()   # the host-sourced build of the same table
    assert np.array_equal(fp, hp) and np.array_equal(fm.view(np.uint32), hm.view(np.uint32)) and np.array_equal(bm.view(np.uint32), hb.view(np.uint32))
    sc = sage_b200.Scorer(dev.db, **c)
    gf, gc = sc.score_batch(spectra)
    of, oc, _, _ = odb.score_batch(oracle_cfg(**c), spectra.as_dict())
    assert assert_features_equal(gf, gc, of, oc, c.get("report_psms", 1), what=f"prefiltered {cfg}") > 100


def test_from_fasta_prefilter_and_picked_fields():
    fasta, kw = DC.CASES["size_medium_mods"]
    spectra = _spectra(fasta, kw, 300, 13)
    db = sage_b200.IndexedDatabase.from_fasta(fasta, prefilter=True, spectra=spectra, scorer=NARROW, prefilter_chunk_size=200, **kw)
    d = db.digest
    assert d.db is db and d.peptides is db.peptides and d.info["n_chunks"] == 4
    t, _ = digest_oracle.prefilter(fasta, spectra.as_dict(), oracle_cfg(**NARROW), chunk_size=200, **kw)
    lists = digest_oracle.protein_lists(t)
    assert np.array_equal(d.n_proteins, np.diff(t["prot_off"]).astype(np.uint32))
    one = np.nonzero(d.n_proteins == 1)[0]
    assert [d.names[d.protein[i]].encode() for i in one] == [lists[i][0] for i in one]


def test_human_size_matches_oracle():
    fasta = DC.human_fasta()
    spectra = _concat([synth.make_spectra(sage_b200.digest_fasta(fasta, **DC.HUMAN_MODS).peptides, 4800, seed=14, n_peaks=80), _noise(200, 15)])
    dev, t, info = _run(fasta, spectra, DC.HUMAN_MODS, 0, True)
    assert info["n_chunks"] > 1 and len(dev.peptides) > 1000
