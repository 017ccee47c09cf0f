"""SpectrumProcessor::process for raw MS1 at label-free-quantification scale (synth.make_ms1_runs defaults: 4 files x 3 000 spectra x 1 500
peaks): sage_b200_process_raw and FeatureMap.add_raw_ms1 on the device against host processing (the single-thread CPU oracle) followed by
add_ms1, with peaks sorted and shuffled inside spectra, with and without mobility. Every device result is checked bit for bit against the
oracle in the same run. Prints one JSON line.

    python tools/bench_process.py [--ids 30000 --files 4 --spectra 3000 --peaks 1500 --repeats 5]

process_raw_wall_ms is the host wall clock of one call (upload, kernels, read-back; median of --repeats). Kernel times come from a separate
torch.profiler run with CUDA activities (summed per kernel, per call); bytes_per_kernel_s is the least traffic k_raw_process needs (read m/z,
intensity [, mobility], write mass, intensity, mobility) over its time, against the 3.35 TB/s data-sheet HBM3 bandwidth. lfq_*_ms are the
library's CUDA-event tracing times (ms_trace) and the host wall clock of the add calls. Nothing is written to disk."""
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

from oracle_process import process_oracle as PO  # noqa: E402
from sage_b200 import FeatureMap, IndexedDatabase, LfqSettings, Ms1Batch, SpectrumProcessor, synth  # noqa: E402

HBM3_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def gpu_name_and_power_limit():
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], text=True, timeout=30)
        name, pl = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, float(pl)
    except Exception:
        return None, None


def kernel_ms(fn):
    """Per-kernel CUDA time of one fn() call, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t:
            out[e.key[:60]] = out.get(e.key[:60], 0.0) + t / 1e3
    return out


def same(a, b):
    return np.asarray(a, np.float32).view(np.uint32).tobytes() == np.asarray(b, np.float32).view(np.uint32).tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ids", type=int, default=30000)
    ap.add_argument("--files", type=int, default=4)
    ap.add_argument("--spectra", type=int, default=3000)
    ap.add_argument("--peaks", type=int, default=1500)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    name, power = gpu_name_and_power_limit()
    if name is None:
        raise SystemExit("bench_process needs a GPU (nvidia-smi found none)")
    pep = synth.make_peptides(20000, seed=41)
    db = IndexedDatabase.build_from_peptides(pep, device=0)
    runs = synth.make_ms1_runs(pep, n_ids=a.ids, n_files=a.files, spectra_per_file=a.spectra, peaks_per_spectrum=a.peaks, mobility=True)
    settings, charges = LfqSettings(), (2, 3)
    sp = SpectrumProcessor(150, False, 0.0)
    result = dict(tool="bench_process", gpu=name, power_limit_w=power, spectra=len(runs["batch"]), peaks=int(runs["batch"].peak_off[-1]), cases=[])
    for shuffle in (False, True):
        for mobility in (False, True):
            raw = synth.ms1_to_raw(runs["batch"], shuffle=shuffle)
            if not mobility:
                raw.mobility = None
            npk = int(raw.peak_off[-1])
            t0 = time.perf_counter()
            want = PO.so_process(raw)
            oracle_ms = (time.perf_counter() - t0) * 1e3
            sp.process_raw(raw)   # warm-up
            walls = []
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                got = sp.process_raw(raw)
                walls.append((time.perf_counter() - t0) * 1e3)
            ok = (got.peak_off.tolist() == want["peak_off"].tolist() and same(got.masses, want["masses"]) and same(got.intensities, want["intensities"])
                  and same(got.mobilities, want["mobilities"]) and same(got.tic, want["tic"]))
            kms = kernel_ms(lambda: sp.process_raw(raw))
            k_proc = sum(v for k, v in kms.items() if "k_raw_process" in k)
            need = npk * (4 + 4 + (4 if mobility else 0)) + npk * 12
            processed = Ms1Batch(want["peak_off"], want["masses"], want["intensities"], raw.file_id, raw.scan_start_time,
                                 want["mobilities"] if mobility else None)

            def lfq(add, batch):
                fm = FeatureMap.build(db, pep, settings, charges, runs["features"], runs["alignments"])
                t0 = time.perf_counter()
                add(fm, batch)
                wall = (time.perf_counter() - t0) * 1e3
                return fm, wall, fm.info()["ms_trace"]
            lfq(FeatureMap.add_raw_ms1, raw)   # warm-up
            fr, raw_wall, raw_trace = lfq(FeatureMap.add_raw_ms1, raw)
            fp, proc_wall, proc_trace = lfq(FeatureMap.add_ms1, processed)
            lfq_ok = fr.export(grids=True)["grids"].tobytes() == fp.export(grids=True)["grids"].tobytes()
            result["cases"].append(dict(
                shuffled=shuffle, mobility=mobility, parity=bool(ok), lfq_parity=bool(lfq_ok),
                process_raw_wall_ms=float(np.median(walls)), process_raw_wall_ms_min=float(min(walls)),
                kernel_ms={k: round(v, 4) for k, v in sorted(kms.items(), key=lambda kv: -kv[1])[:8]},
                k_raw_process_ms=k_proc, bytes_per_kernel_s=need / (k_proc / 1e3) if k_proc else None,
                share_of_hbm_peak=need / (k_proc / 1e3) / HBM3_PEAK if k_proc else None,
                oracle_single_thread_ms=oracle_ms,
                lfq_add_raw_ms1_wall_ms=raw_wall, lfq_add_raw_ms1_trace_ms=raw_trace,
                host_process_plus_add_ms1_ms=oracle_ms + proc_wall, lfq_add_ms1_wall_ms=proc_wall, lfq_add_ms1_trace_ms=proc_trace))
    print(json.dumps(result))
    if not all(c["parity"] and c["lfq_parity"] for c in result["cases"]):
        raise SystemExit("parity failed")


if __name__ == "__main__":
    main()
