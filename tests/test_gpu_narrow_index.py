"""The narrow-search index copy (m/z-only runs, u16 block offsets, u16 directory cells over u32 group bases) on the edge cases of its layout.
Each case scores the same spectra three ways and requires identical rows and matched-fragment / candidate counts: the CPU oracle, the page
index in the reference's loop order (option narrow_index 0), and the narrow copy. The oracle builds its index from a peptide table only, so
the cases that upload a hand-made fragment layout (one m/z for every fragment, fragments on cell edges) compare the narrow copy with the page
index over that same layout."""
import numpy as np
import pytest

from sage_b200 import IndexedDatabase, Scorer, SpectraBatch, Tolerance, synth

from helpers import assert_features_equal, oracle_cfg, oracle_db_from_peptides, valid_rows
from narrow_directory import F, dir_cells, edges, mz_cells

pytestmark = pytest.mark.gpu

KW = dict(precursor_tol=Tolerance.ppm(-50, 50), fragment_tol=Tolerance.ppm(-20, 20), report_psms=3, min_isotope_err=-1, max_isotope_err=2)


@pytest.fixture(scope="module")
def peptides():
    pep = synth.make_peptides(20000, seed=31, static_c=True)
    return pep, synth.make_spectra(pep, 1200, seed=32)


def score(gdb, spectra, block, narrow_index, kw):
    sc = Scorer(gdb, **kw)
    sc.set_option("narrow_index", narrow_index)
    if block:
        sc.set_option("narrow_block", block)
    f, c = sc.score_batch(spectra)
    return f.copy(), c.copy(), sc.counters()


def check_paths(gdb, spectra, block, kw=KW, oracle=None):
    """narrow copy == page index (== oracle when given); returns the PSM count."""
    r = kw.get("report_psms", 1)
    pf, pc, pctr = score(gdb, spectra, block, 0, kw)
    nf, nc, nctr = score(gdb, spectra, block, 1, kw)
    assert pctr["pages"] > 0 and nctr["pages"] == 0, "the two counting paths were not the ones meant"
    assert np.array_equal(nc, pc) and valid_rows(nf, nc, r).tobytes() == valid_rows(pf, pc, r).tobytes(), block
    for k in ("matched_fragments", "candidates_scored", "psms"):
        assert nctr[k] == pctr[k], (block, k, nctr[k], pctr[k])
    if oracle is not None:
        of, oc, _, _ = oracle.score_batch(oracle_cfg(**kw), spectra.as_dict())
        assert_features_equal(nf, nc, of, oc, r, what=f"narrow copy, block {block}")
    return int(nc.sum())


def reference_layout(frag_pep, frag_mz, bucket_size):
    """database.rs:325-365 on given fragments: ascending m/z, pages of bucket_size, each page sorted by PeptideIx."""
    o = np.lexsort((frag_pep, frag_mz.view(np.uint32)))
    fp, fm = frag_pep[o], frag_mz[o]
    bucket_min = fm[::bucket_size].copy()
    for s in range(0, len(fp), bucket_size):
        q = np.argsort(fp[s:s + bucket_size], kind="stable")
        fp[s:s + bucket_size], fm[s:s + bucket_size] = fp[s:s + bucket_size][q], fm[s:s + bucket_size][q]
    return fp, fm, bucket_min


@pytest.mark.parametrize("block", [64, 8192])
def test_block_sizes_against_oracle(peptides, block):
    """64: windows over many blocks; 8192: one block holds > 65535 entries, so walk starts need the u32 group base."""
    pep, spectra = peptides
    gdb = IndexedDatabase.build_from_peptides(pep)
    fp, _, _ = gdb.export_index()
    per_block = np.bincount(fp // block)
    assert (per_block.max() > 65535) == (block == 8192)
    assert check_paths(gdb, spectra, block, oracle=oracle_db_from_peptides(pep)) > 400


def test_empty_blocks(peptides):
    """min_ion_index 6 keeps no fragment of peptides shorter than 8 residues: the lightest blocks of 64 peptides are empty."""
    pep, spectra = peptides
    gdb = IndexedDatabase.build_from_peptides(pep, min_ion_index=6)
    fp, _, _ = gdb.export_index()
    counts = np.bincount(fp // 64, minlength=(len(pep.mono) + 63) // 64)
    empty = np.nonzero(counts == 0)[0]
    assert len(empty) >= 1
    # the first 40 spectra get precursors of peptides inside empty blocks, so their windows probe those blocks
    sp = spectra.slice(0, 600)
    prec_mz = sp.prec_mz.copy()
    for i in range(40):
        p = int(empty[i % len(empty)]) * 64 + 7
        prec_mz[i] = np.float32(pep.mono[p] / sp.prec_charge[i] + 1.0072764)
    sp = SpectraBatch(sp.peak_off, sp.masses, sp.intensities, prec_mz, sp.prec_charge, sp.iso_lo, sp.iso_hi, sp.tic, sp.level, sp.rt, sp.ims)
    assert check_paths(gdb, sp, 64, oracle=oracle_db_from_peptides(pep, min_ion_index=6)) > 50


def test_cta_per_query_windows():
    """Windows of 1025..8192 peptides are counted by k_prelim_narrow (one CTA per query) through the same probe."""
    pep = synth.make_peptides(60000, seed=35, static_c=True, var_mods=(("M", 15.9949), ("STY", 79.9663)), max_variable_mods=2)
    spectra = synth.make_spectra(pep, 200, seed=36)
    m = np.sort(pep.mono.astype(np.float64))
    pm = (spectra.prec_mz.astype(np.float64) - 1.0072764) * spectra.prec_charge
    w = np.searchsorted(m, pm + 5.0) - np.searchsorted(m, pm - 5.0)
    assert (w > 1024).mean() > 0.3 and (w > 8192).mean() == 0
    kw = dict(precursor_tol=Tolerance.da(-5, 5), fragment_tol=Tolerance.ppm(-20, 20), report_psms=2)
    gdb = IndexedDatabase.build_from_peptides(pep)
    assert check_paths(gdb, spectra, 0, kw=kw, oracle=oracle_db_from_peptides(pep)) > 50


def test_degenerate_mz_range(peptides):
    """Every fragment at one m/z (no directory cells: each walk starts at its block start), peaks on that m/z and next to it."""
    pep, spectra = peptides
    gdb0 = IndexedDatabase.build_from_peptides(pep)
    fp, fm, _ = gdb0.export_index()
    mz = F(512.2734)
    fp2, fm2, bm2 = reference_layout(fp.copy(), np.full(len(fp), mz, F), 8192)
    gdb = IndexedDatabase.from_reference_layout(pep, fp2, fm2, bm2, 8192)
    sp = spectra.slice(0, 300)
    masses = sp.masses.copy()
    masses[::3] = mz
    masses[1::3] = np.nextafter(mz, F(np.inf))
    sp = SpectraBatch(sp.peak_off, per_spectrum_sort(masses, sp.peak_off), sp.intensities, sp.prec_mz, sp.prec_charge, sp.iso_lo, sp.iso_hi, sp.tic,
                      sp.level, sp.rt, sp.ims)
    kw = dict(KW, min_matched_peaks=1)
    for block in (256, 8192):
        check_paths(gdb, sp, block, kw=kw)


def per_spectrum_sort(masses, peak_off):
    out = masses.copy()
    for a, b in zip(peak_off[:-1], peak_off[1:]):
        out[int(a):int(b)] = np.sort(out[int(a):int(b)])
    return out


@pytest.mark.parametrize("block", [256, 8192])
def test_fragments_and_peaks_on_cell_edges(peptides, block):
    """Fragment m/z snapped to directory cell edges and one ulp to either side, including the first and the last cell of the range, and peaks on
    the same values with a Da tolerance whose lower bound is the peak itself (flo == edge)."""
    pep, spectra = peptides
    gdb0 = IndexedDatabase.build_from_peptides(pep)
    fp, fm, _ = gdb0.export_index()
    lo, hi = F(fm.min()), F(fm.max())
    cells = dir_cells(len(fp), (len(pep.mono) + block - 1) // block)
    base, inv_w = mz_cells(lo, hi, cells)
    e = edges(base, inv_w, np.arange(1, cells))
    cell = np.clip(np.searchsorted(e, fm), 0, len(e) - 1)
    snapped = e[cell]
    rng = np.random.default_rng(block)
    step = rng.integers(-1, 2, len(fm))
    snapped = np.where(step < 0, np.nextafter(snapped, F(-np.inf)), np.where(step > 0, np.nextafter(snapped, F(np.inf)), snapped)).astype(F)
    snapped[np.argmin(fm)], snapped[np.argmax(fm)] = lo, hi   # keep the range: the same cells as computed here
    fp2, fm2, bm2 = reference_layout(fp.copy(), snapped, 8192)
    gdb = IndexedDatabase.from_reference_layout(pep, fp2, fm2, bm2, 8192)
    sp = spectra.slice(0, 300)
    masses = sp.masses.copy()
    pick = rng.integers(0, len(snapped), len(masses))
    masses[::2] = snapped[pick[::2]]
    masses[:2] = [lo, hi]
    sp = SpectraBatch(sp.peak_off, per_spectrum_sort(masses, sp.peak_off), sp.intensities, sp.prec_mz, sp.prec_charge, sp.iso_lo, sp.iso_hi, sp.tic,
                      sp.level, sp.rt, sp.ims)
    kw = dict(KW, fragment_tol=Tolerance.da(0.0, 0.01), max_fragment_charge=1, min_matched_peaks=1)
    assert check_paths(gdb, sp, block, kw=kw) > 0
