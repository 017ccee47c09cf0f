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
    return out


def q_reference(disc, label):
    """qvalue.rs restated in numpy f32 on the given discriminants: (spectrum_q by row, passing, order)."""
    disc = np.asarray(disc, np.float32)
    b = disc.view(np.int32)
    key = b ^ ((b >> 31).astype(np.uint32) >> 1).astype(np.int32)
    order = np.argsort(-key.astype(np.int64), kind="stable")
    dec = np.cumsum(label[order] == -1).astype(np.int64)
    tar = np.arange(1, len(disc) + 1) - dec
    q = ((1 + dec).astype(np.int32).astype(np.float32) / tar.astype(np.int32).astype(np.float32)).astype(np.float32)
    qmin = np.minimum(np.minimum.accumulate(q[::-1])[::-1], np.float32(1.0))
    out = np.empty_like(qmin)
    out[order] = qmin
    return out, int((qmin <= np.float32(0.01)).sum()), order.astype(np.uint32)
