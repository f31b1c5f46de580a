"""Cost and effect of annealed MPPI (``anneal_iterations`` / ``anneal_iter_decay`` / ``anneal_horizon_decay``) on the device.

1. K1 (mppib_sample, the Gaussian sampler) and K3 (mppib_reduce) alone, cold L2 (buffers rotated over more than twice the L2 size),
   device time from torch.profiler, without a schedule and with a registered one (N = 4), alternated round by round, at the C2 (panda
   reach, K = 10 000) and C5 (panda_pick) shapes.
2. The panda-reach plan p50 / p10 / p90 with N = 1, 2 and 4 at K = 10 000 and at the fixed rollout budget K = 10 000 / N, CUDA-graph replay
   as in production, L2 flushed before every plan, the planners alternated in blocks.
3. Closed loop: the planner against a one-env simulator (as examples/panda/world.py does) on panda reach and boxer_push for a fixed number
   of steps, N = 1 at K against N = 4 at K / 4 with decays below 1; reports the final goal distance (end effector to goal, block to goal)
   and the Objective's cost summed over the steps of the world.

Every planner here samples with ``sampling_method: random`` (annealing excludes the Halton library).  Prints the card name and its power
limit (read through NVML, nothing is changed) next to the numbers.
    python tools/anneal_bench.py [--rounds 5] [--plans 200] [--steps 150] [--out results.json]
"""
import argparse
import copy
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "examples", "panda"))

from adaptive_bench import card  # noqa: E402
from smooth_bench import _profile  # noqa: E402

CONFIGS = {"C2": "config_panda_b200", "C3": "config_boxer_push_b200", "C5": "config_panda_pick_b200"}
DECAYS = dict(anneal_iter_decay=0.6, anneal_horizon_decay=0.9)


def _shape(name):
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = load_isaacgym_config(CONFIGS[name])
    nu = int(np.asarray(cfg.mppi.noise_sigma).shape[0])
    return int(cfg.mppi.num_samples) // 64 * 64, int(cfg.mppi.horizon), nu


def _handle(K, T, nu, N):
    """A handle of the shape; with N > 0 a registered schedule of N iterations (counter at iteration 1, so that the scales are not 1)."""
    from mppi_isaac_b200.backend import CudaBackend
    from mppi_isaac_b200.model.blob import OBS_DOF_STATE, anneal_schedule, make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    from synth_mppi import nu_model
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.1 * np.eye(nu)).tolist(),
                    u_min=[-0.2], u_max=[0.2], lambda_=0.05, sample_null_action=True, filter_u=T >= 9)
    be = CudaBackend("cuda:0")
    be.create(nu_model(nu), make_params(mc, IsaacGymConfig(), nu, K, [(OBS_DOF_STATE, 0)]))
    if N > 0:
        s, r = anneal_schedule(N, DECAYS["anneal_iter_decay"], DECAYS["anneal_horizon_decay"], T)
        be._anneal_buf = torch.from_numpy(np.concatenate([[1.0], s.ravel(), r.ravel()]).astype(np.float32)).to("cuda:0")
        be.set_anneal(be._anneal_buf, N)
    return be


def kernel_profile(name, rounds):
    K, T, nu = _shape(name)
    hs = {"plain": _handle(K, T, nu, 0), "annealed_N4": _handle(K, T, nu, 4)}
    U = 0.05 * torch.ones((T, nu), device="cuda:0")
    ctr = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    out = {"config": name, "K": K, "T": T, "nu": nu}
    nbuf = max(2, int(np.ceil(2 * 50e6 / (2 * 4 * K * T * nu))) + 1)
    bufs = [(torch.empty((T, nu, K), device="cuda:0"), torch.empty((T, nu, K), device="cuda:0")) for _ in range(nbuf)]
    run = {n: (lambda h: lambda a, x: h.sample(1, 0, 0, K, U, None, a, x, ctr))(h) for n, h in hs.items()}
    out["k1"] = {"l2": f"cold: {nbuf} rotating output pairs"}
    out["k1"].update(_profile(run, {n: r"mppib_sample_kernel" for n in run}, bufs, rounds))
    parts = {n: torch.zeros(2 + T * nu, device="cuda:0") for n in hs}
    nbuf = max(2, int(np.ceil(2 * 50e6 / (4 * K * T * (nu + 1)))) + 1)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    bufs = [(torch.rand((T, K), device="cuda:0", generator=g), 0.2 * torch.randn((T, nu, K), device="cuda:0", generator=g)) for _ in range(nbuf)]
    run = {n: (lambda h, part: lambda c, x: h.reduce(c, x, U, part))(h, parts[n]) for n, h in hs.items()}
    out["k3"] = {"l2": f"cold: {nbuf} rotating input pairs"}
    out["k3"].update(_profile(run, {n: r"mppib_reduce_ws_kernel" for n in run}, bufs, rounds))
    for h in hs.values():
        h.destroy()
    return out


def _cfg(name, K=None, N=1):
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = copy.deepcopy(load_isaacgym_config(CONFIGS[name]))
    cfg.mppi.device, cfg.mppi.sampling_method = "cuda:0", "random"
    if K is not None:
        cfg.mppi.num_samples = int(K)
    if N > 1:
        cfg.mppi.anneal_iterations = N
        cfg.mppi.anneal_iter_decay, cfg.mppi.anneal_horizon_decay = DECAYS["anneal_iter_decay"], DECAYS["anneal_horizon_decay"]
    return cfg


def _objective(name):
    from mppi_isaac_b200.objectives import PandaReachObjective, PushObjective
    return PushObjective(robot="boxer", link="ee_link") if name == "C3" else PandaReachObjective()


def plan_ab(plans, block=20):
    from mppi_isaac_b200 import MPPIisaacPlanner
    spec = {"N1_K10000": (10000, 1), "N2_K10000": (10000, 2), "N4_K10000": (10000, 4), "N2_K5000": (5000, 2), "N4_K2500": (2500, 4)}
    pls = {n: MPPIisaacPlanner(_cfg("C2", K, N), _objective("C2"), use_cuda_graph=True) for n, (K, N) in spec.items()}
    for pl in pls.values():
        for _ in range(5):
            pl.mppi.command()
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda:0")
    ms = {n: [] for n in pls}
    names = list(pls)
    for b in range(max(1, plans // block)):
        for n in (names if b % 2 == 0 else names[::-1]):
            for _ in range(block):
                flush.zero_()
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); pls[n].mppi.command(); e.record(); e.synchronize()
                ms[n].append(a.elapsed_time(e))
    out = {n: {"p50_ms": statistics.median(v), "p10_ms": float(np.percentile(v, 10)), "p90_ms": float(np.percentile(v, 90)), "n": len(v),
               "K": spec[n][0], "N": spec[n][1], "graph_captured": pls[n].mppi._graph is not None} for n, v in ms.items()}
    return out


def _distance(name, world):
    if name == "C3":
        d = world.get_actor_position_by_name("block")[0, 0:2] - world.get_actor_position_by_name("goal")[0, 0:2]
        return float(torch.linalg.norm(d))
    from world import goal_distance
    return goal_distance(world)


def closed_loop(name, steps, K, N):
    """(final goal distance, summed world cost) of `steps` closed-loop steps of a planner against a one-env simulator of the config."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from world import build_world, control_step
    cfg, world = build_world(CONFIGS[name], device="cuda:0")
    planner = MPPIisaacPlanner(_cfg(name, K, N), _objective(name), use_cuda_graph=True)
    judge = _objective(name)
    total = 0.0
    for _ in range(steps):
        control_step(world, planner)
        total += float(judge.compute_cost(world).reshape(-1)[0])
    return {"K": K, "N": N, "steps": steps, "final_goal_distance": _distance(name, world), "summed_cost": total}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--plans", type=int, default=200)
    ap.add_argument("--steps", type=int, default=150)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__  # noqa: F401  (repository root on the path)
    if not torch.cuda.is_available():
        raise SystemExit("anneal_bench needs a CUDA device")
    out = {"card": card(), "kernels": [kernel_profile(n, a.rounds) for n in ("C2", "C5")], "plan": plan_ab(a.plans), "closed_loop": {}}
    for name in ("C2", "C3"):
        K = _shape(name)[0] if name == "C3" else 10000
        out["closed_loop"][name] = [closed_loop(name, a.steps, K, 1), closed_loop(name, a.steps, K // 4, 4)]
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
