#!/usr/bin/env python
"""Builds rollout-kernel variants (-D knobs of rollout.cu) and times each on the bench workload (graph-captured launches).
    python tools/tune_rollout.py build      # here (nvcc, no GPU needed) -> gpurun_out/tune/libmppib_<name>.so
    python tools/tune_rollout.py run        # on the GPU box
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tune_build")
VARIANTS = {
    "base": [],
    "s2u2": ["-DROLL_UNROLL_S2=2"],
    "s2u2_s3u3": ["-DROLL_UNROLL_S2=2", "-DROLL_UNROLL_S3=3"],
    "s3u3": ["-DROLL_UNROLL_S3=3"],
    "maxreg128": ["-maxrregcount=128"],
    "s1pipe": ["-DROLL_S1_PIPE=1"],
}

if sys.argv[1] == "build":
    os.makedirs(OUT, exist_ok=True)
    csrc = os.path.join(ROOT, "mppi_isaac_b200", "csrc")
    for name, flags in VARIANTS.items():
        so = os.path.join(OUT, f"libmppib_{name}.so")
        cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
               "-diag-suppress", "177", *flags, "-o", so] + [os.path.join(csrc, f) for f in ("api.cu", "sample.cu", "rollout.cu", "reduce.cu", "cost.cu")]
        subprocess.check_call(cmd)
        print("built", so)
elif sys.argv[1] == "run":
    res = {}
    for name in VARIANTS:
        env = dict(os.environ, MPPIB_LIB=os.path.join(OUT, f"libmppib_{name}.so"))
        code = ("import sys; sys.path.insert(0, %r); import bench, torch, numpy as np\n"
                "from mppi_isaac_b200 import MPPIisaacPlanner\nfrom mppi_isaac_b200.objectives import PandaReachObjective\n"
                "p = MPPIisaacPlanner(bench.panda_cfg(10000, 'cuda:0'), PandaReachObjective(), use_cuda_graph=False)\n"
                "q0, goal = bench.synthetic_state(); p.sim.set_actor_position_by_name(goal, 'goal'); p.sim.reset_robot_state(q0, np.zeros(7))\n"
                "p.mppi.command(); m = p.mppi\n"
                "print('US', bench.graph_time_us(lambda: p.sim.rollout_all(m.actions), 10))\n") % ROOT
        out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
        us = [float(l.split()[1]) for l in out.stdout.splitlines() if l.startswith("US")]
        res[name] = us[0] if us else out.stderr[-300:]
        print(name, res[name], flush=True)
    print(json.dumps(res))
