"""PSM rescoring benchmark: spectrum_fdr (runner.rs:280-291) on the device (sage_b200.spectrum_fdr) and on the CPU oracle (oracle_ml/), on
synth.make_psms rows with a Ppm tolerance, with the parity of every output row checked in the same run. Prints one JSON line.

    python tools/bench_rescore.py [--rows 1000000 --warmup 1 --repeats 5]

Stage times are the CUDA-event times the library reports (median of --repeats calls); e2e_wall_ms is the host wall clock of the call, copies
included. The KDE rates count one f64 exp per (bin, sample) pair: bins x n for the mass-error KDE (of the class sizes, summed) and 1000 x n for
the discriminant KDE. Nothing is written to disk."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle_ml import ml_oracle  # noqa: E402
from sage_b200 import Tolerance, api, synth  # noqa: E402

H100_SXM_FP64_TFLOPS = 34.0   # data sheet, non-tensor FP64 at 700 W


def gpu_name_and_power_limit():
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], text=True, timeout=30)
        name, pl = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, float(pl)
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0x0FD2)
    a = ap.parse_args()
    rows = synth.make_psms(a.rows, seed=a.seed)
    tol = Tolerance.ppm(-20, 20)
    for _ in range(a.warmup):
        api.spectrum_fdr(rows, tol)
    runs, walls = [], []
    for _ in range(a.repeats):
        t = time.perf_counter()
        runs.append(api.spectrum_fdr(rows, tol))
        walls.append((time.perf_counter() - t) * 1e3)
    dev = runs[-1]
    orc = ml_oracle.spectrum_fdr(rows, tol)
    keys = ("discriminant_score", "posterior_error", "spectrum_q", "order")
    rows_equal = int(np.logical_and.reduce([(dev[k].view(np.uint32) == orc[k].view(np.uint32)) | (np.isnan(dev[k]) & np.isnan(orc[k]) if dev[k].dtype.kind == "f" else False)
                                            for k in keys]).sum())
    parity = rows_equal == a.rows and dev["passing"] == orc["passing"] and dev["coef"].tobytes() == orc["coef"].tobytes() and dev["eps"] == orc["eps"]
    med = {s: float(np.median([r[s] for r in runs])) for s in api.FDR_STAGES}
    mass_bins = 100
    exps = {"mass_kde": mass_bins * a.rows, "discriminant_kde": 1000 * a.rows}
    rate = {k: exps[k] / (med["ms_" + k] * 1e-3) for k in exps}
    name, pl = gpu_name_and_power_limit()
    print(json.dumps(dict(
        workload=f"make_psms rows={a.rows} Ppm(-20,20)", gpu=name, power_limit_w=pl, repeats=a.repeats,
        stage_ms={k[3:]: round(v, 3) for k, v in med.items()}, e2e_wall_ms=round(float(np.median(walls)), 3),
        oracle_s=round(orc["seconds"], 3), oracle_threads=orc["threads"],
        exp_per_s={k: float("%.4g" % v) for k, v in rate.items()},
        exp_share_of_datasheet_fp64_at_20_flop_per_exp={k: round(v * 20 / (H100_SXM_FP64_TFLOPS * 1e12), 4) for k, v in rate.items()},
        parity=bool(parity), rows_equal=rows_equal, passing=dev["passing"], lda_fitted=dev["lda_fitted"], eps=dev["eps"])))
    if not parity:
        sys.exit(1)


if __name__ == "__main__":
    main()
