#!/usr/bin/env python
"""A/B timing of two or more library builds in one session: runs `bench.py --no-extras --no-cpu-baseline` on one workload, alternating the
builds round by round (SAGE_B200_LIB), and prints value, score phase, card, power limit and SM clock of every run.

    python tools/ab_bench.py --lib old=sage_b200/lib/ab/old.so --lib new=sage_b200/lib/ab/new.so --rounds 3 [--workload cfg2] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, metavar="NAME=PATH")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workload", default="cfg2")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="", help="also write every run's JSON line to DIR/ab_<workload>.jsonl")
    args = ap.parse_args()
    libs = [tuple(s.split("=", 1)) for s in args.lib]
    rows = []
    for r in range(args.rounds):
        for name, path in libs:
            env = dict(os.environ, SAGE_B200_LIB=os.path.abspath(path))
            cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
                   "--workload", args.workload, "--no-extras", "--no-cpu-baseline"]
            p = subprocess.run(cmd, env=env, capture_output=True, text=True)
            line = next((ln for ln in p.stdout.splitlines() if ln.startswith("{")), None)
            if p.returncode != 0 or line is None:
                raise SystemExit(f"{name} round {r}: bench.py failed ({p.returncode})\n{p.stderr[-3000:]}")
            j = json.loads(line)
            ck = j.get("clocks", {})
            rows.append(dict(build=name, round=r, value=j["value"], score_ms=j["phases_ms_per_step"]["score"], ms_per_step=j["ms_per_step"],
                             gpu=ck.get("gpu"), power_limit_w=ck.get("power_limit_w"), sm_mhz=ck.get("sm_mhz"), reasons=ck.get("reasons")))
            print(json.dumps(rows[-1]), flush=True)
            if args.out:
                os.makedirs(args.out, exist_ok=True)
                with open(os.path.join(args.out, f"ab_{args.workload}.jsonl"), "a") as f:
                    f.write(line + "\n")
    for name, _ in libs:
        v = [x["value"] for x in rows if x["build"] == name]
        s = [x["score_ms"] for x in rows if x["build"] == name]
        print(f"{name:8s} value min {min(v):10.0f} max {max(v):10.0f}   score ms min {min(s):.4f} max {max(s):.4f}")


if __name__ == "__main__":
    main()
