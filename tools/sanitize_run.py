#!/usr/bin/env python
"""Small, complete pass over every kernel of libmppib.so for compute-sanitizer (tools/sanitize.sh): K1 (Gaussian and Halton-spline
library), K2 (lanes-per-rollout chain kernel, team kernel on contact scenes of small and large robots, thread-per-rollout chain / tree /
contact kernels), fused cost, K3 (warp-specialised
ring, ragged last tile), K4, shift, and whole plans (eager and CUDA-graph replay).  Sizes are
small: the sanitizer serialises the GPU.  With WORLD_SIZE > 1 (torchrun) the plans also run the peer-memory exchange."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from mppi_isaac_b200 import MPPIisaacPlanner  # noqa: E402
from mppi_isaac_b200.objectives import PandaPickObjective, PandaReachObjective, PointReachObjective, PushObjective  # noqa: E402
from scenes import boxer_cfg, panda_cfg, pick_cfg, point_cfg, push_cfg  # noqa: E402

rank = int(os.environ.get("RANK", "0"))
world = int(os.environ.get("WORLD_SIZE", "1"))
local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dev = f"cuda:{local}"
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=torch.device(dev))

CASES = [
    ("panda reach (lanes K2, Gaussian K1, warp-specialised K3, ragged tile)", lambda: panda_cfg(K=4100 * world, T=30, device=dev), PandaReachObjective, [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]),
    ("point robot (lanes K2 G=4, Halton-spline K1, savgol K4)", lambda: point_cfg(K=256 * world, T=12, device=dev), PointReachObjective, [0.1, 0.0, 0.0]),
    ("heijn push (team K2: contacts, 8 lanes per rollout, 2 coordinate slots)", lambda: push_cfg(K=128 * world, T=10, device=dev), PushObjective, [0.0, 0.0, 0.0]),
    ("boxer push (team K2: contacts, planar base tree)", lambda: boxer_cfg(K=128 * world, T=10, device=dev), lambda: PushObjective(robot="boxer", link="ee_link"), [0.0, 2.5, 0.0]),
    ("panda pick (team K2: contacts, 16-lane articulation in 2 passes, compact layout)", lambda: pick_cfg(K=64 * world, T=9, device=dev), PandaPickObjective, [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0, 0.02, 0.02]),
]
for name, mk, obj, q in CASES:
    for graph in (False, True):
        pl = MPPIisaacPlanner(mk(), obj(), use_cuda_graph=graph)
        for _ in range(3 if graph else 2):
            a = pl.compute_action(q, [0.0] * len(q))
        assert torch.isfinite(a).all(), name
        if world > 1:
            pl.mppi.invalidate_graph(); pl.mppi.close_peers()
        del pl
    if rank == 0:
        print("ok:", name, flush=True)
if world == 1:
    os.environ["MPPIB_K2_LANES"] = "0"                # a serial chain on the contact-free TEAM kernel (a chain is a tree)
    pl = MPPIisaacPlanner(panda_cfg(K=512, T=10, device=dev), PandaReachObjective(), use_cuda_graph=False)
    pl.compute_action([0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0], [0.0] * 7)
    os.environ["MPPIB_K2_TEAM"] = "0"                 # ... and on the thread-per-rollout chain kernel
    pl = MPPIisaacPlanner(panda_cfg(K=512, T=10, device=dev), PandaReachObjective(), use_cuda_graph=False)
    pl.compute_action([0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0], [0.0] * 7)
    os.environ["MPPIB_K2_TEAM"] = "0"                 # the thread-per-rollout contact kernels (chain and tree)
    for mk, obj, q in [(lambda: push_cfg(K=128, T=10, device=dev), PushObjective, [0.0, 0.0, 0.0]),
                       (lambda: pick_cfg(K=64, T=9, device=dev), PandaPickObjective, [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0, 0.02, 0.02])]:
        pl = MPPIisaacPlanner(mk(), obj(), use_cuda_graph=False)
        pl.compute_action(q, [0.0] * len(q))
        del pl
    del os.environ["MPPIB_K2_TEAM"]
    print("ok: team and thread-per-rollout chain K2, thread-per-rollout contact K2", flush=True)
torch.cuda.synchronize()
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
if rank == 0:
    print("sanitize_run done", flush=True)
