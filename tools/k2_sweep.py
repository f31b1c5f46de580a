#!/usr/bin/env python
"""K-sweep of the K2 rollout kernel on the panda reach workload (T = 30, 2 substeps): the lanes-per-rollout mapping
(csrc/rollout_lanes.cu) against the thread-per-rollout mapping (csrc/rollout.cu, MPPIB_K2_LANES=0 MPPIB_K2_TEAM=0).  Device time per launch from
graph-captured back-to-back launches (bench.graph_time_us).  Run on the GPU box:

    python tools/k2_sweep.py [K ...] > gpurun_out/k2_sweep.md
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from mppi_isaac_b200 import MPPIisaacPlanner  # noqa: E402
from mppi_isaac_b200.objectives import PandaReachObjective  # noqa: E402

KS = [int(a) for a in sys.argv[1:]] or [1252, 2500, 5000, 10000, 20000, 40000, 65536, 131072]


def time_rollout(K, lanes):
    os.environ["MPPIB_K2_LANES"] = "1" if lanes else "0"      # read by mppib_create
    os.environ["MPPIB_K2_TEAM"] = "0"                         # (a chain is also a tree: without this the team kernel would take it)
    planner = MPPIisaacPlanner(bench.panda_cfg(K, "cuda:0"), PandaReachObjective(), use_cuda_graph=False)
    q0, goal = bench.synthetic_state()
    planner.sim.set_actor_position_by_name(goal, "goal")
    planner.sim.reset_robot_state(q0, np.zeros(7))
    planner.mppi.command()
    m = planner.mppi
    us = bench.graph_time_us(lambda: planner.sim.rollout_all(m.actions), 5)
    obs = planner.sim._obs.clone()
    del planner
    return us, obs


rows = []
print("| K | lanes (us) | thread-per-rollout (us) | lanes vs thread | rollout-steps/s (lanes) | max abs obs diff |")
print("|---|---|---|---|---|---|")
for K in KS:
    K = (K // 4) * 4
    a, oa = time_rollout(K, True)
    b, ob = time_rollout(K, False)
    diff = float((oa - ob).abs().max())
    rows.append({"K": K, "lanes_us": a, "thread_us": b, "max_abs_obs_diff": diff})
    print(f"| {K} | {a:.1f} | {b:.1f} | {b / a:.2f}x | {K * 30 / (a * 1e-6):.3e} | {diff:.2e} |", flush=True)
    torch.cuda.empty_cache()
print()
print(json.dumps(rows))
