"""Cost and effect of constrained MPPI (``constraint_mode: feasible_first``) on the device.

1. K3 alone, cold L2 (buffers rotated over more than twice the L2 size), device time from torch.profiler, alternated round by round: the
   feasibility-first K3 (which also streams the (T, K) violation rows) against today's K3 at the C2 (panda reach, K = 10 000) and C5
   (panda_pick) shapes, and the copy of the Objective's margins into the registered (T, K) buffer.
2. The panda-reach plan p50 / p10 / p90 at K = 10 000 with and without the mode (PandaReachKeepOutObjective, its sphere out of reach, so
   every sample is feasible), CUDA-graph replay as in production, L2 flushed before every plan, the planners alternated in blocks.
3. Closed loop: 100 steps of panda reach against a one-env simulator (examples/panda/world.py) with a keep-out sphere for the tip on the
   straight line from the start to the goal, for three ways of saying the sphere is forbidden: a penalty in the cost, an infinite cost,
   and feasible_first.  Reports the steps whose executed tip lay inside the sphere and the final goal distance.

Every planner here samples with ``sampling_method: random``.  Prints the card name and its power limit (read through NVML, nothing is
changed) next to the numbers.
    python tools/constraint_bench.py [--rounds 5] [--plans 200] [--steps 100] [--parts kernels,plan,closed_loop] [--out results.json]
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

CONFIGS = {"C2": "config_panda_b200", "C5": "config_panda_pick_b200"}
FF = "feasible_first"


def _shape(name):
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = load_isaacgym_config(CONFIGS[name])
    nu = int(np.asarray(cfg.mppi.noise_sigma).shape[0])
    return int(cfg.mppi.num_samples) // 64 * 64, int(cfg.mppi.horizon), nu


def _handle(K, T, nu, on):
    """A handle of the shape; with `on` a registered (T, K) violation buffer of margins <= 0."""
    from mppi_isaac_b200.backend import CudaBackend
    from mppi_isaac_b200.model.blob import OBS_DOF_STATE, make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    from synth_mppi import nu_model
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.1 * np.eye(nu)).tolist(),
                    u_min=[-0.2], u_max=[0.2], lambda_=0.05, sample_null_action=True, filter_u=False,
                    constraint_mode=FF if on else "none")
    be = CudaBackend("cuda:0")
    be.create(nu_model(nu), make_params(mc, IsaacGymConfig(), nu, K, [(OBS_DOF_STATE, 0)]))
    if on:
        be._viol = -torch.rand((T, K), device="cuda:0")
        be._cstate = torch.zeros(2, device="cuda:0")
        be.set_constraint(be._viol, be._cstate)
    return be


def kernel_profile(name, rounds):
    K, T, nu = _shape(name)
    hs = {"plain": _handle(K, T, nu, False), FF: _handle(K, T, nu, True)}
    U = 0.05 * torch.ones((T, nu), device="cuda:0")
    tile_rows = {"plain": T * nu + T, FF: T * nu + 2 * T}
    out = {"config": name, "K": K, "T": T, "nu": nu,
           "tile_rows": tile_rows, "tile_bytes_ratio": tile_rows[FF] / tile_rows["plain"]}
    parts = {n: torch.zeros(h.partial_row_floats(), device="cuda:0") for n, h in hs.items()}
    nbuf = max(2, int(np.ceil(2 * 50e6 / (4 * K * T * (nu + 1)))) + 1)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    bufs = [(torch.rand((T, K), device="cuda:0", generator=g), 0.2 * torch.randn((T, nu, K), device="cuda:0", generator=g)) for _ in range(nbuf)]
    run = {n: (lambda c, x, n=n: hs[n].reduce(c, x, U, parts[n])) for n in hs}
    out["k3"] = {"l2": f"cold: {nbuf} rotating input pairs (the violation rows are one buffer, re-read every launch)"}
    out["k3"].update(_profile(run, {n: r"mppib_reduce_ws_kernel" for n in run}, bufs, rounds))
    # the copy of the Objective's (T*K) margins into the registered buffer, as the batched plan does it
    src = torch.rand((T * K,), device="cuda:0")
    for _ in range(10):
        hs[FF]._viol.copy_(src.view(T, K))
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(200):
        hs[FF]._viol.copy_(src.view(T, K))
    e.record(); e.synchronize()
    out["viol_copy_us"] = a.elapsed_time(e) / 200 * 1e3
    for h in hs.values():
        h.destroy()
    return out


def _cfg(K=10000, on=False, **kw):
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = copy.deepcopy(load_isaacgym_config(CONFIGS["C2"]))
    cfg.mppi.device, cfg.mppi.sampling_method = "cuda:0", "random"
    cfg.mppi.num_samples = int(K)
    cfg.mppi.constraint_mode = FF if on else "none"
    for k, v in kw.items():
        setattr(cfg.mppi, k, v)
    return cfg


def plan_ab(plans, block=20):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachKeepOutObjective, PandaReachObjective
    far = PandaReachKeepOutObjective(centre=(10.0, 10.0, 10.0), radius=0.1)   # every sample feasible
    pls = {"plain": MPPIisaacPlanner(_cfg(), PandaReachObjective(), use_cuda_graph=True),
           FF: MPPIisaacPlanner(_cfg(on=True), far, use_cuda_graph=True)}
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
    return {n: {"p50_ms": statistics.median(v), "p10_ms": float(np.percentile(v, 10)), "p90_ms": float(np.percentile(v, 90)), "n": len(v),
                "K": 10000, "graph_captured": pls[n].mppi._graph is not None} for n, v in ms.items()}


class _Penalty:
    """The keep-out Objective with its violation in the cost: w max(g, 0) (a penalty) or +inf where g > 0."""

    def __init__(self, base, weight):
        self.base, self.weight = base, weight
        self.weights = base.weights

    def reset(self):
        pass

    def compute_cost(self, sim):
        c = self.base.compute_cost(sim)
        g = self.base.compute_constraint(sim)
        if self.weight == float("inf"):
            return torch.where(g > 0, torch.full_like(c, float("inf")), c)
        return c + self.weight * torch.clamp_min(g, 0.0)


def closed_loop(steps, K, radius_frac=0.25):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachKeepOutObjective
    from world import build_world, control_step, goal_distance
    out = {}
    for kind in ("penalty", "inf_cost", FF):
        cfg, world = build_world(CONFIGS["C2"], device="cuda:0")
        tip = world.get_actor_link_by_name("panda", "panda_ee_tip")[0, 0:3].detach().cpu().numpy().astype(np.float64)
        goal = world.get_actor_position_by_name("goal")[0, 0:3].detach().cpu().numpy().astype(np.float64)
        centre = 0.5 * (tip + goal)
        radius = radius_frac * float(np.linalg.norm(goal - tip))
        keep_out = PandaReachKeepOutObjective(centre=tuple(centre), radius=radius)
        obj = {"penalty": _Penalty(keep_out, 10.0), "inf_cost": _Penalty(keep_out, float("inf")), FF: keep_out}[kind]
        planner = MPPIisaacPlanner(_cfg(K, on=kind == FF), obj, use_cuda_graph=True)
        inside, fallback = 0, 0
        for _ in range(steps):
            control_step(world, planner)
            p = world.get_actor_link_by_name("panda", "panda_ee_tip")[0, 0:3].detach().cpu().numpy().astype(np.float64)
            inside += int(np.linalg.norm(p - centre) < radius)
            if kind == FF:
                fallback += int(planner.mppi.feasible_samples == 0)
        out[kind] = {"K": K, "steps": steps, "centre": centre.tolist(), "radius": radius, "steps_inside": inside,
                     "final_goal_distance": goal_distance(world), "plans_without_a_feasible_sample": fallback if kind == FF else None}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--plans", type=int, default=200)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--out", default=None)
    ap.add_argument("--parts", default="kernels,plan,closed_loop", help="comma-separated subset of kernels, plan, closed_loop")
    a = ap.parse_args()
    parts = set(a.parts.split(","))
    import __graft_entry__  # noqa: F401  (repository root on the path)
    if not torch.cuda.is_available():
        raise SystemExit("constraint_bench needs a CUDA device")
    out = {"card": card(), "kernels": [kernel_profile(n, a.rounds) for n in ("C2", "C5")] if "kernels" in parts else None,
           "plan": plan_ab(a.plans) if "plan" in parts else None,
           "closed_loop": closed_loop(a.steps, 10000) if "closed_loop" in parts else None}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
