#!/usr/bin/env python
"""Per-kernel CUDA times of the resident search step (torch.profiler, CUDA activities) on one workload; SAGE_B200_LIB selects the build.

    SAGE_B200_LIB=$PWD/sage_b200/lib/ab/new.so python tools/score_kernel_times.py [cfg2|cfg5] [steps]
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch   # noqa: E402
from torch.profiler import ProfilerActivity, profile   # noqa: E402

from sage_b200 import IndexedDatabase, Scorer, Tolerance, synth   # noqa: E402

wl = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
pep = synth.make_peptides(2_000_000)
spectra = synth.make_spectra(pep, 50_000 if wl == "cfg2" else 100_000, seed=0xB202, chimeric=(wl == "cfg5"))
db = IndexedDatabase.build_from_peptides(pep)
kw = dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))
if wl == "cfg5":
    kw.update(chimera=True, report_psms=5)
sc = Scorer(db, **kw)
sc.upload(spectra)
for _ in range(3):
    sc.run()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
        sc.run()
    torch.cuda.synchronize()
agg = {}
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0:
        a = agg.setdefault(e.name, [0, 0.0])
        a[0] += 1
        a[1] += e.device_time
print(f"{wl}: {torch.cuda.get_device_name(0)}, {steps} steps; kernel, launches per step, us per step")
for name, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:12]:
    print(f"  {us / steps:10.1f}  {n / steps:5.1f}  {name[:110]}")
