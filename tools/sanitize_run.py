#!/usr/bin/env python
"""Small, complete pass over every kernel of libmppib.so for compute-sanitizer (tools/sanitize.sh): K1 (Gaussian and Halton-spline
library), K2 (lanes-per-rollout chain kernel, team kernel on contact scenes of small and large robots, thread-per-rollout chain / tree /
contact kernels), fused cost, K3 (warp-specialised
ring, ragged last tile), K4, shift, the cov_type horizon kernels (horizon-colour K1, SYRK, its fused K4), the colored K1, the mppi_mode cem kernels (CEM K1, elite kernel with its last-CTA merge, CEM K4 and shift), the mppi_mode smooth kernels (smooth K1,
K3 with the smoothness cost and the fused smooth K4), the risk-aware K1 / K2 / K3 (n_worlds), the temperature pass of lambda_mode ess (with its
fused solve, or the split solve after an all-gather), and whole plans (eager and CUDA-graph replay).  Sizes are
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
    ("panda reach, cov_type horizon (horizon-colour K1, K3 with S_k, SYRK with the fused K4 factorisation; n = 210)",
     lambda: panda_cfg(K=1000 * world, T=30, device=dev, update_cov=True, update_lambda=True, cov_type="horizon"), PandaReachObjective,
     [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]),
    ("point robot, cov_type horizon (horizon-colour library K1, savgol K4; n = 36)",
     lambda: point_cfg(K=256 * world, T=12, device=dev, update_cov=True, cov_type="horizon"), PointReachObjective, [0.1, 0.0, 0.0]),
    ("point robot, cov_type horizon at n = 255 (ragged K against the 64-sample K1 tile and the SYRK chunks, SYRK-fused K4 with 127 KB of "
     "shared memory)", lambda: point_cfg(K=4100 * world, T=85, device=dev, update_cov=True, update_lambda=True, cov_type="horizon", filter_u=True),
     PointReachObjective, [0.1, 0.0, 0.0]),
    ("panda reach, sampling_method colored (colored K1: 32-sample tiles, ragged last tile, row pairs of an odd T)",
     lambda: panda_cfg(K=1000 * world, T=31, device=dev, sampling_method="colored"), PandaReachObjective, [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]),
    ("point robot, sampling_method colored with cov_type full (colored K1 with the live L; T*nu = 510)",
     lambda: point_cfg(K=100 * world, T=170, device=dev, sampling_method="colored", update_cov=True, cov_type="full"), PointReachObjective, [0.1, 0.0, 0.0]),
    ("panda reach, mppi_mode cem (CEM K1 with carried rows, elite kernel with a multi-pass last-CTA merge, CEM K4 fused and split; "
     "I = 2)", lambda: panda_cfg(K=20000 * world, T=12, device=dev, mppi_mode="cem", sampling_method="colored", n_elites=128,
                                 keep_elites=0.5, cem_iterations=2), PandaReachObjective, [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]),
    ("panda reach, mppi_mode smooth (smooth K1: 32-sample tiles, ragged last tile, four warps over nu = 7; smooth K3 with the fused "
     "K4)", lambda: panda_cfg(K=1000 * world, T=31, device=dev, mppi_mode="smooth", sampling_method="random", filter_u=False,
                                 smooth_weight=0.5, du_min=[-1.0], du_max=[1.0]), PandaReachObjective, [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]),
    ("heijn push, n_worlds 8 (K1 keyed by the control sample, team K2 keyed by the world, RISK K3 with the fused K4)",
     lambda: push_cfg(K=256 * world, T=10, device=dev, n_worlds=8, cvar_alpha=0.25), PushObjective, [0.0, 0.0, 0.0]),
    ("panda reach, lambda_mode ess (temperature pass: ragged last 256-sample tile, fused solve; RULE_DIST K3 / K4 with both flags off)",
     lambda: panda_cfg(K=4100 * world, T=30, device=dev, sampling_method="random", lambda_mode="ess", ess_target=0.05), PandaReachObjective,
     [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]),
    ("point robot, lambda_mode ess with cov_type full, MEAN mode (temperature pass without the noise rows)",
     lambda: point_cfg(K=300 * world, T=12, device=dev, mppi_mode="halton-spline", update_cov=True, cov_type="full", lambda_mode="ess"),
     PointReachObjective, [0.1, 0.0, 0.0]),
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
