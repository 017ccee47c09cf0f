"""Label-free quantification benchmark: build_feature_map + quantify (lfq.rs) on the device (sage_b200.FeatureMap) and on the CPU oracle
(oracle_lfq/), on one synthetic workload (synth.make_ms1_runs), with the parity of every grid checked in the same run. Prints one JSON line.

    python tools/bench_lfq.py [--ids 30000 --files 4 --spectra 3000 --peaks 1500 --batches 4 --repeats 3]

Device times are CUDA-event times the library reports per stage (best of --repeats full runs); e2e_wall_ms is the host wall clock of
build + every add_ms1 + quantify of that run. Nothing is written to disk."""
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

from oracle_lfq import lfq_oracle as LO  # noqa: E402
from sage_b200 import FeatureMap, IndexedDatabase, LfqSettings, synth  # noqa: E402


def gpu_name_and_power_limit():
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], text=True, timeout=30)
        name, pl = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, float(pl)
    except Exception:
        return None, None


def parity(fm, orc, dev_rows, orc_rows, n_files):
    """Grid cells bit for bit; integration under DESIGN.md §9 (presence, rt, areas identical on grids without an acos near-tie;
    score and spectral_angle within 1e-12 relative)."""
    ex = fm.export(grids=True)
    r, m = orc.export_map()
    map_ok = ex["ranges"].tobytes() == r.tobytes() and ex["min_rts"].tobytes() == m.tobytes()
    ok_keys, ok_mats = orc.export_grids()
    t = ex["touched"].astype(bool)
    slots = np.unique(ex["ranges"]["peptide"])
    g = np.nonzero(t)[0]
    keys = np.stack([slots[g // 2], np.zeros_like(g), g % 2], 1).astype(np.uint32)
    grids_ok = keys.tolist() == ok_keys.tolist() and ex["grids"][t].tobytes() == ok_mats.tobytes()
    o, d = orc_rows, dev_rows
    okey = {k: i for i, k in enumerate(zip(o["id"].tolist(), o["charge"].tolist(), o["decoy"].tolist()))}
    seen = np.zeros(len(o["id"]), bool)
    near, bad = 0, 0
    for j, k in enumerate(zip(d["id"].tolist(), d["charge"].tolist(), d["decoy"].tolist())):
        i = okey.get(k)
        if i is None:
            bad += 1
            continue
        seen[i] = True
        if o["margin"][i] <= 1e-9:
            near += 1
            continue
        same = o["present"][i] and d["rt"][j] == o["rt"][i] and d["areas"][j].tobytes() == o["areas"][i].tobytes()
        for f in ("score", "spectral_angle"):
            same = same and abs(d[f][j] - o[f][i]) <= 1e-12 * abs(o[f][i])
        bad += not same
    bad += int((o["present"] & ~seen & (o["margin"] > 1e-9)).sum())
    return dict(map_identical=bool(map_ok), grids_identical=bool(grids_ok), grids_compared=int(t.sum()), rows_compared=len(d["id"]) - near,
                near_tie_grids=near, rows_mismatched=bad, ok=bool(map_ok and grids_ok and bad == 0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--peptides", type=int, default=120_000)
    ap.add_argument("--ids", type=int, default=30_000)
    ap.add_argument("--files", type=int, default=4)
    ap.add_argument("--spectra", type=int, default=3000, help="MS1 spectra per file")
    ap.add_argument("--peaks", type=int, default=1500, help="peaks per MS1 spectrum")
    ap.add_argument("--batches", type=int, default=4, help="add_ms1 calls")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--threads", type=int, default=os.cpu_count(), help="oracle integration threads")
    ap.add_argument("--seed", type=int, default=17)
    a = ap.parse_args()

    pep = synth.make_peptides(a.peptides, seed=43)
    runs = synth.make_ms1_runs(pep, n_ids=a.ids, n_files=a.files, spectra_per_file=a.spectra, peaks_per_spectrum=a.peaks, seed=a.seed)
    batch, settings, charges = runs["batch"], LfqSettings(), (2, 4)
    cuts = np.linspace(0, len(batch), a.batches + 1).astype(int)
    parts = [batch.slice(x, y) for x, y in zip(cuts[:-1], cuts[1:])]
    db = IndexedDatabase.build_from_peptides(pep, device=0)

    best = None
    for rep in range(a.repeats + 1):    # the first run warms up the context and the allocator
        t0 = time.perf_counter()
        fm = FeatureMap.build(db, pep, settings, charges, runs["features"], runs["alignments"])
        for p in parts:
            fm.add_ms1(p)
        rows = fm.quantify()
        wall = (time.perf_counter() - t0) * 1e3
        info = fm.info()
        if rep and (best is None or wall < best[0]):
            best = (wall, info, rows, fm)
        elif rep:
            del fm
    wall, info, dev_rows, fm = best

    t0 = time.perf_counter()
    orc = LO.LfqOracle(pep, settings, charges, runs["features"], runs["alignments"])
    t1 = time.perf_counter()
    orc.add_ms1(batch)
    t2 = time.perf_counter()
    orc_rows = orc.quantify(threads=a.threads)
    t3 = time.perf_counter()

    name, pl = gpu_name_and_power_limit()
    trace_s, integ_s = info["ms_trace"] / 1e3, info["ms_integrate"] / 1e3
    out = dict(
        bench="lfq", gpu=name, power_limit_w=pl,
        workload=dict(peptides=len(pep), identified=int(info["n_peptides"]), files=a.files, ms1_spectra=int(info["ms1_spectra"]), ms1_peaks=int(info["ms1_peaks"]),
                      add_ms1_calls=a.batches, ranges=int(info["n_ranges"]), pages=int(info["n_pages"]), grids=int(info["n_grids"]),
                      grids_touched=int(info["grids_touched"]), rows=len(dev_rows["id"]), settings="LfqSettings() defaults, precursor_charge (2, 4)"),
        device_ms=dict(build=round(info["ms_build"], 3), trace=round(info["ms_trace"], 3), integrate=round(info["ms_integrate"], 3),
                       download=round(info["ms_download"], 3)),
        e2e_wall_ms=round(wall, 3), repeats=a.repeats,
        ms1_peaks_per_s=info["ms1_peaks"] / trace_s if trace_s > 0 else None,
        grids_per_s=info["grids_touched"] / integ_s if integ_s > 0 else None,
        contributions=int(info["contributions"]), device_bytes=int(info["device_bytes"]),
        oracle_ms=dict(build=round((t1 - t0) * 1e3, 1), trace=round((t2 - t1) * 1e3, 1), integrate=round((t3 - t2) * 1e3, 1)),
        oracle_threads=dict(build=1, trace=1, integrate=a.threads),
        parity=parity(fm, orc, dev_rows, orc_rows, a.files),
    )
    print(json.dumps(out))


if __name__ == "__main__":
    main()
