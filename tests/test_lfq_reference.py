"""The CPU oracle of label-free quantification (oracle_lfq/) against the independent numpy restatement of lfq.rs (tests/lfq_reference.py), bit for
bit: the feature map, min_rts, the touched grids, every grid cell and every quantify output, on every edge workload of tests/lfq_cases.py and on
the synthetic workloads of tests/test_gpu_lfq.py; and peptide_isotopes in f32 against an mpmath evaluation of the same Poisson convolution."""
import numpy as np
import pytest

import lfq_cases
from lfq_reference import LfqReference, peptide_isotopes
from oracle_lfq import lfq_oracle as LO
from sage_b200.api import LfqSettings


def run_both(pep, settings, charges, features, alignments, batches):
    orc = LO.LfqOracle(pep, settings, charges, features, alignments)
    ref = LfqReference(pep, settings, charges, features, alignments)
    o_ranges, o_min = orc.export_map()
    assert ref.ranges.tobytes() == o_ranges.tobytes(), "range arrays differ"
    assert ref.min_rts.tobytes() == o_min.tobytes(), "min_rts differ"
    for b in batches:
        orc.add_ms1(b)
        ref.add_ms1(b)
    return orc, ref


def assert_same(orc, ref):
    """Touched keys, grid cells and every quantify output equal; returns the restatement's quantify."""
    ok, om = orc.export_grids()
    rk, rm = ref.export_grids()
    assert rk.tolist() == ok.tolist(), "touched grids differ"
    assert rm.tobytes() == om.tobytes(), "grid cells differ"
    o, r = orc.quantify(threads=8), ref.quantify()
    for f in ("id", "charge", "decoy", "present"):
        assert r[f].tolist() == o[f].tolist(), f
    p = o["present"]
    for f in () if not p.any() else ("rt", "spectral_angle", "score", "areas"):
        bad = np.nonzero(np.any((r[f][p] != o[f][p]).reshape(int(p.sum()), -1), axis=1))[0]
        assert len(bad) == 0, f"{f} differs in {len(bad)} grids, first {rk[p][bad[0]].tolist()}: {r[f][p][bad[0]]!r} vs {o[f][p][bad[0]]!r}"
    return r


def check_case(c):
    orc, ref = run_both(c["peptides"], c["settings"], c["charges"], c["features"], c["alignments"], c["batches"])
    q = assert_same(orc, ref)
    return ref, q


@pytest.mark.parametrize("name", lfq_cases.NAMES)
def test_restatement_matches_oracle_on_edge_workloads(name):
    c = lfq_cases.case(name)
    ref, q = check_case(c)
    n_grids, present = len(q["id"]), int(q["present"].sum())
    if name == "no_kept_feature":
        assert len(ref.ranges) == 0 and n_grids == 0
        return
    assert present > 0, "the workload traced nothing"
    if "pages" in c:
        assert len(ref.min_rts) == c["n_pages"] >= 3 and len(np.unique(ref.min_rts)) < len(ref.min_rts)   # two pages share a min_rt
    if "warps" in c:
        fwd = ~q["decoy"] & q["present"]
        want = np.array([c["warps"][f] for f in range(len(c["warps"]))])
        hit = np.all(q["warps"][fwd] == want, axis=1)   # a few grids also collect a near-isobaric neighbour's or a noise peak's signal
        assert hit.mean() >= 0.9, f"{int(hit.sum())} of {int(fwd.sum())} forward grids have warps {want.tolist()}; others {q['warps'][fwd][~hit][:3].tolist()}"
    print(f"{name}: {len(ref.ranges)} ranges, {ref.matches} matches, {n_grids} grids, {present} rows")


SEEDS = [(7, LfqSettings(combine_charge_states=True), (2, 4), 1), (7, LfqSettings(combine_charge_states=False), (2, 4), 3),
         (8, LfqSettings(combine_charge_states=False), (2, 4), 37), (11, LfqSettings(ppm_tolerance=3000.0), (2, 3), 2)]


@pytest.mark.parametrize("seed,settings,charges,splits", SEEDS)
def test_restatement_matches_oracle_on_gpu_test_seeds(seed, settings, charges, splits):
    runs = lfq_cases.seed_runs(seed)
    b = runs["batch"]
    cuts = np.linspace(0, len(b), splits + 1).astype(int)
    orc, ref = run_both(lfq_cases.peptides(), settings, charges, runs["features"], runs["alignments"], [b.slice(x, y) for x, y in zip(cuts[:-1], cuts[1:])])
    assert_same(orc, ref)


def test_restatement_matches_oracle_on_every_integration_strategy():
    runs = lfq_cases.seed_runs(13)
    pep = lfq_cases.peptides()
    for scoring in ("RetentionTime", "SpectralAngle", "Intensity", "Hybrid"):
        for integration in ("Apex", "Sum"):
            for threshold in (0.7, 0.0):
                s = LfqSettings(peak_scoring=scoring, integration=integration, spectral_angle=threshold)
                orc, ref = run_both(pep, s, (2, 3), runs["features"], runs["alignments"], [runs["batch"]])
                assert_same(orc, ref)


def test_isotopes_bit_exact_with_oracle_over_every_count():
    c, s = np.meshgrid(np.arange(3061), np.arange(256), indexing="ij")
    mine = peptide_isotopes(c, s)
    for cc in range(0, 3061, 7):
        for ss in (0, 1, 2, 17, 128, 255):
            assert mine[cc, ss].tobytes() == LO.peptide_isotopes(cc, ss).tobytes(), (cc, ss)


def test_isotopes_against_mpmath():
    """peptide_isotopes (isotopes.rs:43-50) in f32 against the exact Poisson convolution, for every carbon count 0..3060 (12 x 255 residues)
    and sulfur count 0..255.

    Error bound. Let u = 2^-24. The exact value is out[i] = cs[i] / max(cs[0..2]) with cs = c13 * (s33 * s35) and the Poisson terms
    c13[k] = e^-lc lc^k / k!, lc = 0.011 C (s33, s35 alike with 0.0076 S and 0.044 S). In f32:
      * each lambda is the f32 constant (relative error <= u) times the count, rounded: <= 2u; lambda^k then carries <= 2ku from the lambdas
        and k - 1 roundings of powi, so <= 3k - 1 <= 8u for k <= 3;
      * the factors e^-lambda are one rounded expf value shared by every term of one distribution: they cancel exactly in the ratio, and
        multiplying by them and dividing by k! adds <= 2u per term. So every c13, s33, s35 term is within 10u;
      * both convolutions add products of non-negative terms, so each cs[i] is within 10u + 10u + 10u (the three terms' errors) + 1u
        (product) + 3u (sums) + 1u (product) = 35u, taking s33 and s35 as they enter;
      * the division by the maximum adds the maximum's error and one rounding.
    Together |out - exact| <= 72u * exact; the test allows 80u = 4.8e-6 relative and reports the largest error observed."""
    import mpmath
    mpmath.mp.dps = 40
    F = [1, 1, 2, 6]

    def poisson(lam):
        e = mpmath.exp(-lam)
        return [float(e * lam ** k / F[k]) for k in range(4)]
    carbon = np.array([poisson(mpmath.mpf(c) * mpmath.mpf("0.011")) for c in range(3061)])
    s33 = np.array([poisson(mpmath.mpf(s) * mpmath.mpf("0.0076")) for s in range(256)])
    s35 = np.array([[float(mpmath.exp(-mpmath.mpf(s) * mpmath.mpf("0.044"))), 0.0, float(mpmath.mpf(s) * mpmath.mpf("0.044") * mpmath.exp(-mpmath.mpf(s) * mpmath.mpf("0.044"))), 0.0]
                    for s in range(256)])

    def conv(a, b):   # f64, error ~1e-16 relative: far below the f32 bound
        return np.stack([a[..., 0] * b[..., 0], a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0], a[..., 0] * b[..., 2] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 0]], -1)
    sul = np.concatenate([conv(s33, s35), np.zeros((256, 1))], -1)
    sul[:, 3] = s33[:, 0] * s35[:, 3] + s33[:, 1] * s35[:, 2] + s33[:, 2] * s35[:, 1] + s33[:, 3] * s35[:, 0]
    cs = conv(carbon[:, None, :], sul[None, :, :])
    exact = cs / cs.max(axis=-1, keepdims=True)
    c, s = np.meshgrid(np.arange(3061), np.arange(256), indexing="ij")
    got = peptide_isotopes(c, s).astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        rel = np.where(exact > 0, np.abs(got - exact) / exact, np.abs(got))
    worst = np.unravel_index(np.argmax(rel), rel.shape)
    u = 2.0 ** -24
    print(f"peptide_isotopes: max relative error {rel.max():.3e} = {rel.max() / u:.1f} u at (carbon, sulfur, isotope) = {tuple(int(x) for x in worst)}")
    assert rel.max() <= 80 * u
