"""Times picked_fdr (picked_peptide + picked_protein) on 10^6 rows over a make_peptides table on one GPU: each stage's CUDA-event time, the
host wall clock including copies, the C++ oracle's time (oracle_ml, all host threads), and a parity check of every output against it."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import picked_cases as PC  # noqa: E402
from oracle_ml import ml_oracle  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    case = PC.synth_case(a.rows, seed=2024, n_target=a.rows // 2)
    PC.device(case)   # warm-up
    runs = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        res = PC.device(case)
        runs.append(dict(wall_ms=(time.perf_counter() - t0) * 1e3, **{k: res[k] for k in ("ms_keys", "ms_peptide", "ms_protein", "ms_total")}))
    ref = PC.oracle(case)
    cpu_s = ref["seconds"]
    parity = all(np.array_equal(res[k].view(np.uint32), ref[k].view(np.uint32)) if isinstance(ref[k], np.ndarray) else res[k] == ref[k]
                 for k in ("peptide_q", "protein_q", "peptide_passing", "protein_passing", "peptide_entries", "protein_entries"))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu, rows=a.rows, entries=res["peptide_entries"], runs=runs, oracle_s=cpu_s, oracle_threads=ml_oracle.default_threads(), parity=parity)))


if __name__ == "__main__":
    main()
