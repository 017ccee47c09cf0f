"""Reading MGF on the device against the single-thread CPU oracle of MgfReader::parse. The file is synth.make_spectra's spectra written by
synth.write_mgf (every f32 in shortest round-trip form, RTINSECONDS included), tiled --tile times. Prints one JSON line.

    python tools/bench_mgf.py [--peptides 20000 --spectra 25000 --peaks 200 --tile 4 --repeats 3]

h2d_ms and read_ms are the library's CUDA-event times of one sage_b200_mgf_create (the text's upload; the parse from bytes to the resident
spectra, including its small count read-backs); export_ms and process_ms are host wall clocks around sage_b200_mgf_export and
sage_b200_mgf_process (SpectrumProcessor(150, deisotope) on the resident spectra), which end in a stream synchronise; each is the median of
--repeats. oracle_ms is one run of the single-thread oracle on the same bytes. GB/s are file bytes over each time. Parity: the device's
export equals the oracle's on the whole file, and process equals process_raw of the exported batch. Nothing is written to disk."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle_mgf import mgf_oracle as MO  # noqa: E402
from sage_b200 import SpectrumProcessor, api, synth  # noqa: E402

FIELDS = ["peak_off", "mz", "intensity", "scan_start_time", "tic", "prec_off", "prec_mz", "prec_intensity", "prec_intensity_some", "prec_charge",
          "prec_charge_some", "iso_kind", "iso_lo", "iso_hi", "id_off", "id_bytes"]


def gpu_name_and_power_limit():
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], text=True, timeout=30)
        name, pl = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, float(pl)
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--peptides", type=int, default=20000)
    ap.add_argument("--spectra", type=int, default=25000)
    ap.add_argument("--peaks", type=int, default=200)
    ap.add_argument("--tile", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    name, power = gpu_name_and_power_limit()
    if name is None or api.device_count() == 0:
        raise SystemExit("bench_mgf needs a GPU (nvidia-smi found none)")
    pep = synth.make_peptides(a.peptides, seed=41, static_c=True)
    sp = synth.make_spectra(pep, a.spectra, seed=42, n_peaks=a.peaks)
    rt = np.random.default_rng(43).uniform(0, 7200, len(sp)).astype(np.float32)
    text = synth.write_mgf(sp, rt=rt) * a.tile
    lib = api.load_library()
    proc = SpectrumProcessor(150, True, 0.0)
    h2d, read, exp, prc = [], [], [], []
    m = None
    for r in range(a.repeats + 1):   # the first call warms up (module load, cub's algorithm choice)
        m = None
        t0 = time.perf_counter()
        m = api.read_mgf(text)
        t1 = time.perf_counter()
        b = m.process(proc)
        t2 = time.perf_counter()
        info = m.info
        n, npk, npr, nid = info["n_spectra"], info["n_peaks"], info["n_precursors"], info["id_bytes"]
        outs = [np.zeros(n + 1, np.uint64), np.zeros(npk, np.float32), np.zeros(npk, np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32),
                np.zeros(n + 1, np.uint64)] + [np.zeros(npr, dt) for dt in (np.float32, np.float32, np.uint8, np.uint8, np.uint8, np.uint8, np.float32,
                                                                            np.float32)] + [np.zeros(n + 1, np.uint64), np.zeros(nid, np.uint8)]
        t3 = time.perf_counter()
        api._check(lib.sage_b200_mgf_export(C.c_void_p(m._h), *[api._ptr(x) for x in outs]))
        t4 = time.perf_counter()
        if r:
            h2d.append(info["ms_h2d"])
            read.append(info["ms_read"])
            prc.append((t2 - t1) * 1e3)
            exp.append((t4 - t3) * 1e3)
    t0 = time.perf_counter()
    o = MO.parse(text)
    oracle_ms = (time.perf_counter() - t0) * 1e3
    parity = all(np.ascontiguousarray(getattr(m, k)).view(np.uint8).tobytes() == np.ascontiguousarray(o[k]).view(np.uint8).tobytes() for k in FIELDS)
    parity = parity and {k: m.info[k] for k in o["info"]} == o["info"]
    p = proc.process_raw(m.raw())
    process_parity = (np.array_equal(b.peak_off, p.peak_off) and np.array_equal(b.masses.view(np.uint32), p.masses.view(np.uint32))
                      and np.array_equal(b.intensities.view(np.uint32), p.intensities.view(np.uint32)) and np.array_equal(b.tic.view(np.uint32), p.tic.view(np.uint32)))
    med = lambda x: float(np.median(x))  # noqa: E731
    gbs = lambda ms: len(text) / (ms * 1e-3) / 1e9  # noqa: E731
    result = dict(tool="bench_mgf", gpu=name, power_limit_w=power, bytes=len(text), spectra=int(m.info["n_spectra"]), peaks=int(m.info["n_peaks"]),
                  lines=int(m.info["n_lines"]), h2d_ms=med(h2d), read_ms=med(read), process_ms=med(prc), export_ms=med(exp), oracle_ms=oracle_ms,
                  h2d_gb_s=gbs(med(h2d)), read_gb_s=gbs(med(read)), oracle_gb_s=gbs(oracle_ms), read_ms_all=read, h2d_ms_all=h2d,
                  peak_device_bytes=int(m.info["peak_device_bytes"]), parity=bool(parity), process_parity=bool(process_parity))
    print(json.dumps(result))
    if not (parity and process_parity):
        raise SystemExit("parity failed")


if __name__ == "__main__":
    main()
