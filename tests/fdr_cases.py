"""Edge workloads of PSM rescoring (spectrum_fdr), shared by the CPU and GPU tests. Each entry: name -> dict(rows, tol, and optionally aligned_rt,
delta_rt_model, delta_ims_model)."""
import numpy as np

from sage_b200 import Tolerance, synth


def _da_rows(n, seed):
    p = synth.make_psms(n, seed=seed)
    rng = np.random.default_rng(seed)
    p["expmass"] = (p["calcmass"] + rng.normal(0.0, 40.0, n) * (p["label"] == 1) + rng.uniform(-450, 450, n) * (p["label"] == -1)).astype(np.float32)
    return p


def cases():
    out = {}
    for n in (1, 2, 1000, 100_000, 1_000_000):
        out[f"psms_{n}"] = dict(rows=synth.make_psms(n, seed=n), tol=Tolerance.ppm(-20, 20))
    out["ppm_wide"] = dict(rows=synth.make_psms(5000, seed=11, ppm=150.0), tol=Tolerance.ppm(-150, 150))
    out["da_500"] = dict(rows=_da_rows(20_000, 12), tol=Tolerance.da(-500, 500))    # 1000 mass bins, bw x 0.1
    p = synth.make_psms(8000, seed=13)
    p["rank"], p["ims"], p["charge"] = 1, np.float32(0), 2                           # constant columns: the ridge carries the solve
    out["constant_columns"] = dict(rows=p, tol=Tolerance.ppm(-20, 20))
    p = synth.make_psms(3000, seed=14)
    p["label"] = 1
    out["no_decoys"] = dict(rows=p, tol=Tolerance.ppm(-20, 20))
    p = synth.make_psms(3000, seed=15)
    p["label"] = -1
    out["no_targets"] = dict(rows=p, tol=Tolerance.ppm(-20, 20))
    p = synth.make_psms(3000, seed=16)
    p["delta_next"][7] = np.nan                                                     # NaN coefficients: the fallback
    out["nan_delta_next"] = dict(rows=p, tol=Tolerance.ppm(-20, 20))
    p = synth.make_psms(6000, seed=17)
    p["poisson"][::5] = 1.0                                                         # ln_1p(-1) = -inf -> 3.5
    p["poisson"][1::7] = -np.inf                                                    # ln_1p(inf) = inf -> 3.5
    out["nonfinite_poisson"] = dict(rows=p, tol=Tolerance.ppm(-20, 20))
    b = synth.make_psms(500, seed=18)
    p = np.concatenate([b, b])                                                      # the same rows as decoys, then as targets, in one order:
    p["label"][:500], p["label"][500:] = -1, 1                                      # equal class means, coefficients 0, every discriminant 0,
    out["all_equal"] = dict(rows=p, tol=Tolerance.ppm(-20, 20))                     # score_step 0 and the NaN estimator bin read as bin 0
    p = synth.make_psms(150, seed=71)
    p["label"][:100], p["label"][100:] = 1, -1                                      # fallback ranking: 100 targets, then 50 decoys, so the
    p["poisson"] = -1.0                                                             # q-value of the top 100 is exactly 1/100 = 0.01f
    p["longest_y_pct"][:100] = np.linspace(0.9, 0.5, 100).astype(np.float32)
    p["longest_y_pct"][100:] = np.linspace(0.4, 0.0, 50).astype(np.float32)
    p["delta_next"][120] = np.nan                                                   # a NaN feature: Gauss::solve fails, the fallback ranks
    out["q_at_threshold"] = dict(rows=p, tol=Tolerance.ppm(-20, 20))
    p = synth.make_psms(4000, seed=19)
    q = p.copy()
    q["label"] = -q["label"]
    out["ties_mixed_labels"] = dict(rows=np.concatenate([p, q, p]), tol=Tolerance.ppm(-20, 20))   # equal f32 discriminants, both labels
    rng = np.random.default_rng(20)
    p = synth.make_psms(10_000, seed=20)
    out["given_columns"] = dict(rows=p, tol=Tolerance.ppm(-20, 20), aligned_rt=(p["rt"] * np.float32(1.01) + np.float32(0.5)).astype(np.float32),
                                delta_rt_model=rng.uniform(0.0, 1.2, 10_000).astype(np.float32),
                                delta_ims_model=rng.uniform(-0.1, 1.0, 10_000).astype(np.float32))
    out.update(edge_cases())
    return out


def _labels(p, decoy):
    p["label"] = np.where(decoy, -1, 1).astype(np.int32)
    return p


def edge_cases():
    """Class sizes, non-finite mass errors, LDA tile and KDE chunk boundaries, tolerance spans, bin-point mass errors and a -inf feature."""
    out = {}
    ppm = Tolerance.ppm(-20, 20)
    p = synth.make_psms(2000, seed=81)
    out["one_decoy"] = dict(rows=_labels(p, np.arange(2000) == 1234), tol=ppm)        # std 0: bandwidth 0, the decoy pdf is 0/0
    p = synth.make_psms(2000, seed=82)
    out["one_target"] = dict(rows=_labels(p, np.arange(2000) != 777), tol=ppm)
    p = synth.make_psms(3000, seed=83)
    p["delta_mass"][5::50] = np.nan                                                   # NaN mass errors: skipped by min / max, NaN std
    out["mass_nan_ppm"] = dict(rows=p, tol=ppm)
    p = synth.make_psms(3000, seed=84)
    p["delta_mass"][7], p["delta_mass"][8] = np.inf, -np.inf                           # min / max infinite: score_step inf, NaN bins
    out["mass_inf_ppm"] = dict(rows=p, tol=ppm)
    p = _da_rows(3000, 85)
    p["expmass"][3], p["expmass"][4], p["expmass"][5] = np.nan, np.inf, -np.inf         # the f32 difference is NaN / +-inf
    out["mass_nonfinite_da"] = dict(rows=p, tol=Tolerance.da(-500, 500))
    p = _da_rows(3000, 86)
    p["expmass"][9] = np.inf                                                           # one infinite Da error only
    out["mass_inf_da"] = dict(rows=p, tol=Tolerance.da(-500, 500))
    for n in (63, 64, 65, 129):                                                        # LDA_TILE = 64 rows per shared-memory tile
        out[f"lda_tile_{n}"] = dict(rows=_labels(synth.make_psms(n, seed=90 + n), np.arange(n) % 2 == 1), tol=ppm)
    out["lda_decoys_after_last_tile"] = dict(rows=_labels(synth.make_psms(150, seed=91), np.arange(150) >= 128), tol=ppm)
    for nd, nt in ((4096, 4097), (8192, 4096)):                                        # KDE_CHUNK = 4096 samples per chunk
        rng = np.random.default_rng(nd + nt)
        dec = np.zeros(nd + nt, bool)
        dec[rng.permutation(nd + nt)[:nd]] = True
        out[f"kde_decoys_{nd}_targets_{nt}"] = dict(rows=_labels(synth.make_psms(nd + nt, seed=nd), dec), tol=ppm)
    out["tol_fractional_span"] = dict(rows=synth.make_psms(3000, seed=92, ppm=50.0), tol=Tolerance.ppm(-50.25, 50.5))   # ceil(100.75) = 101 bins
    out["tol_negative_span"] = dict(rows=synth.make_psms(3000, seed=93, ppm=30.0), tol=Tolerance.ppm(30, -30))        # max(-60, 100): 100 bins
    p = _da_rows(3000, 94)
    p["expmass"] = (p["calcmass"] + np.random.default_rng(94).uniform(-0.5, 0.5, 3000)).astype(np.float32)
    out["tol_da_1"] = dict(rows=p, tol=Tolerance.da(-0.5, 0.5))                        # max(1, 1000): 1000 bins
    p = _da_rows(4000, 95)
    p["expmass"] = (p["calcmass"] + np.random.default_rng(95).uniform(-1000, 1000, 4000)).astype(np.float32)
    out["tol_da_2001"] = dict(rows=p, tol=Tolerance.da(-1000.4, 1000.4))               # ceil(2000.8) = 2001 bins
    p = synth.make_psms(2000, seed=96)
    p["delta_mass"] = (np.arange(2000) % 100).astype(np.float32)                       # 100 bins from 0 to 99, step exactly 1: every mass
    out["mass_on_bin_points"] = dict(rows=p, tol=ppm)                                  # error on a bin point, min_score and max_score included
    p = synth.make_psms(3000, seed=97)
    p["hyperscore"][::301] = -1.0                                                      # ln_1p(-1) = -inf: NaN scatter, the fallback
    out["hyperscore_minus_one"] = dict(rows=p, tol=ppm)
    return out


def kde_samples():
    """kde_build inputs: scores on the bin points of a 1000-bin estimator (min 0, max 499.5, step exactly 0.5) with min and max repeated; and
    one decoy among 3000 scores (std 0, bandwidth 0: the decoy pdf is 0/0 everywhere)."""
    s = np.concatenate([np.arange(1000) * 0.5, np.zeros(7), np.full(5, 499.5), np.arange(0, 1000, 3) * 0.5])
    one = np.random.default_rng(98).normal(0.0, 1.0, 3000)
    return dict(bin_points=(s, np.arange(len(s)) % 3 == 0), one_decoy=(one, np.arange(3000) == 17))
