"""Digest benchmark: FASTA text -> peptide table (Parameters::digest, database.rs:162-258) on the device (sage_b200.digest_fasta) and the
re-upload + index build of IndexedDatabase.from_fasta, on the seeded human-size FASTA (tests/digest_cases.py), with a full parity check
against the CPU oracle's digest in the same run. Prints one JSON line per workload.

    python tools/bench_digest.py [--workloads 1,2,3,4,5] [--repeats 2] [--no-oracle]

Stage times are the CUDA-event times the library reports (best of --repeats); wall_ms is the host wall clock from FASTA text to the exported
table of that run. oracle_digest_s times oracle_digest's single-threaded C++ restatement of the digest (not Sage itself). Nothing is
written to disk."""
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
from oracle_digest import digest_oracle  # noqa: E402
from sage_b200 import IndexedDatabase, SageB200Error, digest_fasta  # noqa: E402
from sage_b200.api import DIGEST_TIMES  # noqa: E402

STATIC_C = {"C": 57.021464}
WORKLOADS = {
    1: ("tryptic_missed1_static_c", None, dict(missed_cleavages=1, static_mods=STATIC_C)),
    2: ("plus_ox_acetyl_max2", None, dict(missed_cleavages=1, static_mods=STATIC_C, variable_mods={"M": [15.9949], "[": [42.010565]}, max_variable_mods=2)),
    3: ("plus_phospho_max3", None, dict(missed_cleavages=1, static_mods=STATIC_C, max_variable_mods=3,
                                        variable_mods={"M": [15.9949], "[": [42.010565], "S": [79.966331], "T": [79.966331], "Y": [79.966331]})),
    4: ("semi_enzymatic", None, dict(missed_cleavages=1, static_mods=STATIC_C, semi_enzymatic=True)),
    5: ("nonspecific_8_12_2000_proteins", 2000, dict(cleave_at="", min_len=8, max_len=12, static_mods=STATIC_C)),
}


def gpu_name_and_power_limit():
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], text=True, timeout=30)
        name, pl = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, float(pl)
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="1,2,3,4,5")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    name, power = gpu_name_and_power_limit()
    human = DC.human_fasta()
    for w in [int(x) for x in a.workloads.split(",")]:
        label, n_prot, kw = WORKLOADS[w]
        fasta = human if n_prot is None else DC.random_fasta(n_prot, 0x5A6E)
        best, dev = None, None
        for _ in range(max(1, a.repeats)):
            t = time.perf_counter()
            d = digest_fasta(fasta, **kw)
            wall = (time.perf_counter() - t) * 1e3
            if best is None or d.info["ms_total"] < best[0].info["ms_total"]:
                best = (d, wall)
            dev = d
        d, wall = best
        t = time.perf_counter()
        try:
            db = IndexedDatabase.build_from_peptides(d.peptides, bucket_size=8192)
            index_ms, fragments = round((time.perf_counter() - t) * 1e3, 1), db.info["n_fragments"]
            del db
        except SageB200Error as e:   # the index build's own limits (e.g. 2^31 fragments) are not the digest's
            index_ms, fragments = f"not built: {e.message}", None
        rec = dict(workload=w, name=label, proteins=d.info["n_proteins"], peptides=d.info["n_peptides"], residues=d.info["n_residues"],
                   windows=d.info["n_windows"], groups=d.info["n_groups"], candidates=d.info["n_candidates"], rows=d.info["n_rows"],
                   fragments=fragments, wall_ms=round(wall, 1), export_ms=round(d.info["ms_export"], 1), reupload_index_build_ms=index_ms, peak_hbm_bytes=d.info["peak_device_bytes"], table_hbm_bytes=d.info["device_bytes"],
                   **{k: round(d.info[k], 3) for k in DIGEST_TIMES}, gpu=name, power_limit_w=power)
        if not a.no_oracle:
            t = time.perf_counter()
            ref = digest_oracle.digest(fasta, **kw)
            rec["oracle_digest_s"] = round(time.perf_counter() - t, 2)
            try:
                DC.assert_table_equal(dev, ref, label)
                rec["parity"] = "bit-exact"
            except AssertionError as e:
                rec["parity"] = f"MISMATCH: {e}"
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
