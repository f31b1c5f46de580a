#!/usr/bin/env python
"""K3 launch-shape sweep (cold L2, graph-timed): CTA count and tile width at the BASELINE K.   python tools/tune_reduce.py [K ...]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Ks = [int(a) for a in sys.argv[1:]] or [10000, 65536]
code = ("import sys; sys.path.insert(0, %r); import bench, torch, numpy as np\n"
        "from mppi_isaac_b200 import MPPIisaacPlanner\nfrom mppi_isaac_b200.objectives import PandaReachObjective\n"
        "p = MPPIisaacPlanner(bench.panda_cfg(10000, 'cuda:0'), PandaReachObjective(), use_cuda_graph=False)\n"
        "r = bench.k3_roofline(p, 3350.0, 'x', %r)\n"
        "print('RES', ' '.join('%%d:%%.2f' %% (e['K'], e['us']) for e in r))\n") % (ROOT, Ks)
res = {}
CASES = [{}, {"MPPIB_K3_VARIANT": "32x2", "MPPIB_K3_GRID": "264"}, {"MPPIB_K3_VARIANT": "64x1", "MPPIB_K3_GRID": "264"},
         {"MPPIB_K3_VARIANT": "32x4"}, {"MPPIB_K3_VARIANT": "32x2", "MPPIB_K3_GRID": "132"}, {"MPPIB_K3_VARIANT": "32x2", "MPPIB_K3_GRID": "396"}]
for case in CASES:
    env = dict(os.environ, **case)
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    line = [l for l in out.stdout.splitlines() if l.startswith("RES")]
    key = " ".join(f"{k[9:]}={v}" for k, v in case.items()) or "default"
    res[key] = line[0][4:] if line else out.stderr[-300:]
    print(f"{key:32s} {res[key]}", flush=True)
print(json.dumps(res))
