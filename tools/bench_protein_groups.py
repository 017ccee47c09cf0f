"""Times protein_groups (generate_protein_groups + picked_protein_group) on 10^6 rows of the isoform-family workload over a make_peptides
table on one GPU: each stage's CUDA-event time, the host wall clock including copies, the C++ oracle's time (oracle_ml, all host threads,
the literal cover loop), the component statistics, and a parity check of every output against the oracle."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import protein_group_cases as G  # noqa: E402
from oracle_ml import ml_oracle  # noqa: E402

STAGES = ("ms_build", "ms_cover", "ms_lookup", "ms_picked", "ms_total")
STATS = ("peptides", "proteins", "meta_peptides", "groups", "edges", "covered", "forced", "greedy_picks", "components", "largest_component", "annotated")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    case = G.family_case(a.rows, seed=2024)
    G.device(case)   # warm-up
    import sage_b200
    off, ids, names = G.name_ids(case)
    rows = G.rows_of(case)
    runs = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()   # the call alone: copies in and out included, strings not built
        r = sage_b200.protein_groups(case["peptides"], rows, case["peptide_q"], case["score"], off, ids, len(names), True, case["threshold"],
                                     case["generate_decoys"])
        runs.append(dict(wall_ms=(time.perf_counter() - t0) * 1e3, **{k: r[k] for k in STAGES}))
    res = G.device(case)
    ref = G.oracle(case)
    try:
        G.same(res, ref, "bench")
        parity = True
    except AssertionError:
        parity = False
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu, rows=a.rows, runs=runs, stats={k: res[k] for k in STATS}, entries=res["entries"], passing=res["passing"],
                          oracle_s=ref["seconds"], oracle_threads=ref["threads"], parity=parity)))


if __name__ == "__main__":
    main()
