"""predict_rt benchmark: the runner's RT alignment and RT / mobility prediction stage (runner.rs:513-531) on the device (sage_b200.predict_rt) and
on the CPU oracle (oracle_ml/), on synth.make_rt_psms rows with mobilities, with the parity of every output checked in the same run. Prints one
JSON line.

    python tools/bench_predict_rt.py [--rows 1000000 --files 8 --warmup 1 --repeats 5]

Stage times are the CUDA-event times the library reports (median of --repeats calls; the host Gauss::solve of each model falls inside its
stage); e2e_wall_ms is the host wall clock of the call, argument checks and copies included. Nothing is written to disk."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_rescore import gpu_name_and_power_limit  # noqa: E402
from oracle_ml import ml_oracle  # noqa: E402
from sage_b200 import IndexedDatabase, api, synth  # noqa: E402

COLUMNS = ("aligned_rt", "predicted_rt", "delta_rt_model", "predicted_ims", "delta_ims_model", "spectrum_q")


def same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    w = np.uint64 if a.dtype.itemsize == 8 else np.uint32
    return (a.view(w) == b.view(w)) | (np.isnan(a) & np.isnan(b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--files", type=int, default=8)
    ap.add_argument("--peptides", type=int, default=200_000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0x5E7)
    a = ap.parse_args()
    pep = synth.make_peptides(a.peptides, seed=a.seed, static_c=True)
    rows, fid = synth.make_rt_psms(pep, a.rows, a.files, seed=a.seed, mobility=True)
    db = IndexedDatabase.build_from_peptides(pep)
    for _ in range(a.warmup):
        api.predict_rt(db, pep, rows, fid, a.files)
    runs, walls = [], []
    for _ in range(a.repeats):
        t = time.perf_counter()
        runs.append(api.predict_rt(db, pep, rows, fid, a.files))
        walls.append((time.perf_counter() - t) * 1e3)
    dev = runs[-1]
    orc = ml_oracle.predict_rt(pep, rows, fid, a.files)
    rows_equal = int(np.logical_and.reduce([same(dev[c], orc[c]) for c in COLUMNS]).sum())
    scalars = all(dev[k] == orc[k] for k in ("training_rows", "aligned_peptides", "rt_fitted", "ims_fitted", "rt_eps", "ims_eps"))
    vectors = all(same(np.atleast_1d(np.float64(dev[k])), np.atleast_1d(np.float64(orc[k]))).all() for k in ("rt_r2", "ims_r2", "rt_beta", "ims_beta"))
    align = bool(same(dev["alignments"].view(np.float32), orc["alignments"].view(np.float32)).all())
    parity = rows_equal == a.rows and scalars and vectors and align
    med = {s: float(np.median([r[s] for r in runs])) for s in api.RT_STAGES}
    name, pl = gpu_name_and_power_limit()
    print(json.dumps(dict(
        workload=f"make_rt_psms rows={a.rows} files={a.files} peptides={len(pep)} mobility", gpu=name, power_limit_w=pl, repeats=a.repeats,
        stage_ms={k[3:]: round(v, 3) for k, v in med.items()}, e2e_wall_ms=round(float(np.median(walls)), 3),
        oracle_s=round(orc["seconds"], 3), oracle_threads=orc["threads"], parity=bool(parity), rows_equal=rows_equal, alignments_equal=align,
        training_rows=dev["training_rows"], aligned_peptides=dev["aligned_peptides"], rt_r2=dev["rt_r2"], ims_r2=dev["ims_r2"],
        rt_eps=dev["rt_eps"], ims_eps=dev["ims_eps"])))
    if not parity:
        sys.exit(1)


if __name__ == "__main__":
    main()
