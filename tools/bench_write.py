#!/usr/bin/env python
"""Times the device writer of Sage's result files (sage_b200_write_tsv) against the C++ oracle writer (oracle_ml/ml_oracle.cpp) on all
host threads, and checks that both produce the same bytes. Workloads (synthetic, seeded):
  results     10^6 results.sage.tsv records (43 fields; peptide, protein and protein-group strings) over a 2*10^5-peptide table
  pin         the same 10^6 rows as results.sage.pin (glibc log1p / log1pf columns, ScanNr)
  fragments   ~2*10^7 matched_fragments.sage.tsv records (10^6 rows of 20 fragments): the largest file a run with annotate_matches writes
  tmt         10^6 tmt.tsv records with 18 channels and real-looking spectrum ids: strings, CSR lookups and quoting
Prints one JSON line per workload: device stage times (CUDA events), H2D / D2H bytes, wall time of the call, oracle wall time, card
name and power limit. Usage: python tools/bench_write.py [--repeat 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle_ml import ml_oracle as M  # noqa: E402
from sage_b200 import api  # noqa: E402


def gpu_name_and_power_limit():
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], text=True, timeout=30)
        name, pl = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, float(pl)
    except Exception:
        return None, None


def fragments_workload(rng):
    n_rows, per = 1_000_000, 20
    rows = np.zeros(n_rows, api.FEATURE_DTYPE)
    rows["fragment_count"] = per
    rows["fragment_offset"] = np.arange(n_rows, dtype=np.uint32) * per
    fr = np.zeros(n_rows * per, api.FRAGMENT_DTYPE)
    fr["kind"] = rng.choice([1, 4], len(fr))
    fr["charge"] = rng.integers(1, 3, len(fr))
    fr["ordinal"] = rng.integers(2, 30, len(fr))
    fr["mz_calculated"] = (rng.random(len(fr)) * 1800 + 150).astype(np.float32)
    fr["mz_experimental"] = fr["mz_calculated"] * (1 + (rng.random(len(fr)) - 0.5) * 2e-5).astype(np.float32)
    fr["intensity"] = (rng.random(len(fr)) * 1e6).astype(np.float32)
    pid = np.arange(n_rows, dtype=np.uint64)
    dev = lambda st: api.write_fragments(rows, fr, pid, stats=st)
    ora = lambda: M.write_fragments(pid, rows["fragment_offset"], rows["fragment_count"], fr)
    return dev, ora


def rows_workload(rng, pin):
    from sage_b200 import synth
    pep = synth.make_peptides(100_000, seed=7, static_c=True)
    n_pep, n_names = len(pep), 20000
    counts = rng.integers(1, 4, n_pep)
    digest = api.DigestResult(peptides=pep, cterm=np.full(n_pep, np.nan, np.float32), semi_enzymatic=np.zeros(n_pep, np.uint8),
                              protein_offsets=np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32),
                              protein_ids=np.concatenate([np.sort(rng.integers(0, n_names, c)) for c in counts]).astype(np.uint32),
                              names=sorted("sp|P%06d|PROT_HUMAN" % i for i in range(n_names)), info={})
    n = 1_000_000
    rows = np.zeros(n, api.FEATURE_DTYPE)
    rows["peptide_idx"] = rng.integers(0, n_pep, n)
    rows["label"] = np.where(pep.decoy[rows["peptide_idx"]] != 0, -1, 1)
    rows["charge"], rows["rank"], rows["peptide_len"] = rng.integers(2, 5, n), 1, rng.integers(7, 30, n)
    for f in ("expmass", "calcmass", "rt", "delta_mass", "average_ppm", "longest_y_pct", "matched_intensity_pct", "ms2_intensity"):
        rows[f] = (rng.random(n) * 1000).astype(np.float32)
    for f in ("hyperscore", "delta_next", "delta_best"):
        rows[f] = rng.random(n) * 50
    rows["poisson"] = -rng.random(n) * 20
    cols = {k: rng.random(n).astype(np.float32) for k in ("discriminant_score", "posterior_error", "spectrum_q", "aligned_rt", "predicted_rt",
                                                             "delta_rt_model", "predicted_ims", "delta_ims_model", "peptide_q", "protein_q")}
    pid, fid, six = np.arange(n, dtype=np.uint64), (np.arange(n) % 8).astype(np.uint32), np.arange(n, dtype=np.uint32)
    files = ["run%02d.mzML" % i for i in range(8)]
    ids = ["controllerType=0 controllerNumber=1 scan=%d" % i for i in range(n)]
    if pin:
        dev = lambda st: api.write_pin(digest, rows, pid, fid, six, files, ids, fdr=cols, rt=cols, stats=st)
    else:
        dev = lambda st: api.write_results(digest, rows, pid, fid, six, files, ids, fdr=cols, rt=cols, picked=cols, stats=st)
    ora = lambda: M.write_results(digest, rows, pid, fid, six, files, ids, fdr=cols, rt=cols, picked=None if pin else cols, pin=pin)
    return dev, ora


def tmt_workload(rng):
    n = 1_000_000
    files = ["run%02d.mzML" % i for i in range(8)]
    ids = ["controllerType=0 controllerNumber=1 scan=%d" % i for i in range(n)]
    fi, si = rng.integers(0, len(files), n), np.arange(n)
    inj = (rng.random(n) * 50).astype(np.float32)
    peaks = (rng.random((n, 18)) * 1e6).astype(np.float32)
    peaks[rng.random((n, 18)) < 0.2] = 0.0
    fb, ib = [f.encode() for f in files], [s.encode() for s in ids]
    dev = lambda st: api.write_tmt(files, ids, fi, si, inj, peaks, stats=st)
    ora = lambda: M.write_tmt(fb, ib, fi, si, inj, peaks)
    return dev, ora


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--workloads", default="results,pin,fragments,tmt")
    args = ap.parse_args()
    name, pl = gpu_name_and_power_limit()
    for w in args.workloads.split(","):
        make = {"results": lambda r: rows_workload(r, False), "pin": lambda r: rows_workload(r, True), "fragments": fragments_workload,
                "tmt": tmt_workload}[w]
        dev, ora = make(np.random.default_rng(1))
        dev({})   # warm-up: module load, allocations
        best, stats, text = None, None, None
        for _ in range(args.repeat):
            st = {}
            t0 = time.perf_counter()
            text = dev(st)
            dt = time.perf_counter() - t0
            if best is None or dt < best:
                best, stats = dt, st
        t0 = time.perf_counter()
        want = ora()
        t_ora = time.perf_counter() - t0
        print(json.dumps(dict(workload=w, bytes=len(text), identical=text == want, records=stats["records"], chunks=stats["chunks"],
                              wall_s=round(best, 4), call_ms=round(stats["ms_total"], 2), ms_upload=round(stats["ms_upload"], 2),
                              ms_measure=round(stats["ms_measure"], 2), ms_scan=round(stats["ms_scan"], 2), ms_write=round(stats["ms_write"], 2),
                              ms_d2h=round(stats["ms_d2h"], 2), h2d_bytes=stats["h2d_bytes"], d2h_bytes=stats["d2h_bytes"],
                              oracle_s=round(t_ora, 3), oracle_threads=M.default_threads(), gpu=name, power_limit_w=pl)), flush=True)


if __name__ == "__main__":
    main()
