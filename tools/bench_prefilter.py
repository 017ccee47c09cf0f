"""Prefilter benchmark: the database prefilter (runner.rs:104-128, 161-278) on the device (sage_b200.prefilter_fasta) on the seeded human-size
FASTA (tests/digest_cases.py) with synthetic spectra, next to the plain IndexedDatabase.from_fasta where that builds. Prints one JSON line
per workload and run.

    python tools/bench_prefilter.py [--workloads a,b,c] [--repeats 2] [--spectra 50000] [--no-plain]

Spectra are synth.make_spectra of the plain digest of a smaller (2 000-protein) FASTA of the same generator, so they are not drawn from
the searched table itself; their precursors and fragments still fall among its peptides' masses. Stage times are the library's (each
stage ends with its work finished). Peak HBM is what the library counts (the scorer's work buffers are not counted). Nothing is written
to disk."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import digest_cases as DC  # noqa: E402
from sage_b200 import IndexedDatabase, SageB200Error, Tolerance, digest_fasta, prefilter_fasta, synth  # noqa: E402
from sage_b200.api import PREFILTER_TIMES  # noqa: E402

STATIC_C = {"C": 57.021464}
WORKLOADS = {
    "a": ("human_mods_auto", DC.HUMAN_MODS),
    "b": ("plus_phospho_max3_auto", dict(missed_cleavages=1, static_mods=STATIC_C, max_variable_mods=3,
                                         variable_mods={"M": [15.9949], "[": [42.010565], "S": [79.966331], "T": [79.966331], "Y": [79.966331]})),
    "c": ("semi_enzymatic_auto", dict(missed_cleavages=1, static_mods=STATIC_C, semi_enzymatic=True)),
}
SCORER = dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))


def gpu_name_and_power_limit():
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], text=True, timeout=30)
        name, pl = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, float(pl)
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="a,b,c")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--spectra", type=int, default=50_000)
    ap.add_argument("--no-plain", action="store_true")
    a = ap.parse_args()
    name, power = gpu_name_and_power_limit()
    human = DC.human_fasta()
    for w in a.workloads.split(","):
        label, kw = WORKLOADS[w]
        spectra = synth.make_spectra(digest_fasta(DC.random_fasta(2000, 0x5A6E), **DC.HUMAN_MODS).peptides, a.spectra, seed=0xB202, n_peaks=150)
        for r in range(max(1, a.repeats)):
            t = time.perf_counter()
            res = prefilter_fasta(human, spectra, **SCORER, **kw)
            wall = (time.perf_counter() - t) * 1e3
            I = res.info
            rec = dict(workload=w, name=label, run=r, spectra=len(spectra), chunk_size=I["chunk_size"], chunks=I["n_chunks"], plain_build=I["plain_build"],
                       unmodified_peptides=I["unmodified_peptides"], rows_digested=I["rows_digested"], rows_kept=I["rows_kept"], peptides=I["n_peptides"],
                       fragments=I["n_fragments"], peak_hbm_bytes=I["peak_device_bytes"], held_hbm_bytes=I["device_bytes"], python_wall_ms=round(wall, 1),
                       **{k: round(I[k], 1) for k in PREFILTER_TIMES}, gpu=name, power_limit_w=power)
            del res
            if not a.no_plain and w != "b":
                t = time.perf_counter()
                try:
                    db = IndexedDatabase.from_fasta(human, **kw)
                    rec["plain_wall_ms"] = round((time.perf_counter() - t) * 1e3, 1)
                    rec["plain_peptides"], rec["plain_fragments"] = db.info["n_peptides"], db.info["n_fragments"]
                    rec["plain_peak_hbm_bytes"] = db.digest.info["peak_device_bytes"] + db.info["device_bytes"]
                    del db
                except SageB200Error as e:
                    rec["plain_wall_ms"] = f"not built: {e.message}"
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
