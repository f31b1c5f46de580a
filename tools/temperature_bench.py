"""Cost and effect of the ESS-targeted temperature (``lambda_mode: ess``) on the device.

1. The temperature pass alone (with its fused solve), cold L2 (inputs rotated over more than twice the L2 size), device time from
   torch.profiler, next to today's K3 of the same shape, alternated round by round: C2 (panda reach, K = 10 000), C3 (boxer push,
   K = 4 000), C5 (panda pick, K = 65 536) in SIMPLE mode and a K = 500 MEAN-mode shape (the Halton-spline panda).  Reports the bytes the
   pass reads (4*T*K in MEAN mode, 4*K*T*(nu + 1) in SIMPLE mode) and the rate they imply.
2. The panda-reach plan p50 / p10 / p90 at K = 10 000 with and without the mode, CUDA-graph replay as in production, L2 flushed before every
   plan, the planners alternated in blocks.
3. Closed loop: 100 steps of panda reach (tip-to-goal distance) and of boxer push (block-to-goal distance) against a one-env simulator
   (examples/panda/world.py), with the shipped lambda_ and with lambda_mode ess at a few targets; reports the final distances and the
   range of the chosen temperatures.

Prints the card name and its power limit (read through NVML, nothing is changed) next to the numbers.
    python tools/temperature_bench.py [--rounds 5] [--plans 200] [--steps 100] [--parts kernels,plan,closed_loop] [--out results.json]
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
SHAPES = [("C2", None, "simple"), ("C3", None, "simple"), ("C5", 65536, "simple"), ("K500 MEAN/Halton", 500, "halton-spline")]


def _shape(name, K):
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = load_isaacgym_config(CONFIGS.get(name, "config_panda_b200"))
    nu = int(np.asarray(cfg.mppi.noise_sigma).shape[0])
    return int(K or cfg.mppi.num_samples) // 4 * 4, int(cfg.mppi.horizon), nu


def _handle(K, T, nu, mode, ess):
    from mppi_isaac_b200.backend import CudaBackend
    from mppi_isaac_b200.model.blob import ESS_GRID, ESS_STATE_FLOATS, OBS_DOF_STATE, ess_grid, make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    from synth_mppi import nu_model
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode=mode, sampling_method="random", noise_sigma=(0.1 * np.eye(nu)).tolist(),
                    u_min=[-0.2], u_max=[0.2], lambda_=0.05, sample_null_action=True, filter_u=False, lambda_mode="ess" if ess else "fixed")
    p = make_params(mc, IsaacGymConfig(), nu, K, [(OBS_DOF_STATE, 0)])
    be = CudaBackend("cuda:0")
    be.create(nu_model(nu), p)
    if ess:
        be._dist = torch.tensor([p.lambda_] + [0.1] * nu, dtype=torch.float32, device="cuda:0")
        be.set_distribution(be._dist)
        lam, inv = ess_grid(p.lambda_)
        st = torch.zeros(ESS_STATE_FLOATS)
        st[:ESS_GRID], st[ESS_GRID:2 * ESS_GRID] = torch.from_numpy(lam), torch.from_numpy(inv)
        be._state = st.to("cuda:0")
        be.set_temperature(be._state)
        be._row = torch.zeros(196, device="cuda:0")
    return be


def kernel_profile(name, K, mode, rounds):
    K, T, nu = _shape(name, K)
    hs = {"k3": _handle(K, T, nu, mode, False), "temperature": _handle(K, T, nu, mode, True)}
    U = 0.05 * torch.ones((T, nu), device="cuda:0")
    part = torch.zeros(hs["k3"].partial_row_floats(), device="cuda:0")
    simple = mode == "simple"
    nbytes = 4 * K * T * ((nu + 1) if simple else 1)
    nbuf = max(2, int(np.ceil(2 * 50e6 / (4 * K * T * (nu + 1)))) + 1)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    bufs = [(torch.rand((T, K), device="cuda:0", generator=g), 0.2 * torch.randn((T, nu, K), device="cuda:0", generator=g)) for _ in range(nbuf)]
    t = hs["temperature"]
    run = {"k3": lambda c, x: hs["k3"].reduce(c, x, U, part), "temperature": lambda c, x: t.temperature(c, x, U, t._row, solve=True)}
    prof = _profile(run, {"k3": r"mppib_reduce_ws_kernel", "temperature": r"mppib_temperature_kernel"}, bufs, rounds)
    for h in hs.values():
        h.destroy()
    us = prof["temperature"]["us_median"]
    return {"config": name, "K": K, "T": T, "nu": nu, "mode": mode, "l2": f"cold: {nbuf} rotating input pairs", "temperature_bytes": nbytes,
            "temperature_GBps": nbytes / (us * 1e-6) / 1e9, **prof}


def _cfg(name="C2", K=None, ess=None, **kw):
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = copy.deepcopy(load_isaacgym_config(CONFIGS[name]))
    cfg.mppi.device = "cuda:0"
    if K:
        cfg.mppi.num_samples = int(K)
    if ess is not None:
        cfg.mppi.lambda_mode, cfg.mppi.ess_target = "ess", float(ess)
    for k, v in kw.items():
        setattr(cfg.mppi, k, v)
    return cfg


def plan_ab(plans, block=20):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    pls = {"fixed": MPPIisaacPlanner(_cfg(), PandaReachObjective(), use_cuda_graph=True),
           "ess": MPPIisaacPlanner(_cfg(ess=0.05), PandaReachObjective(), use_cuda_graph=True)}
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
                "K": int(pls[n].mppi.K_total), "graph_captured": pls[n].mppi._graph is not None} for n, v in ms.items()}


def closed_loop(steps, targets=(None, 0.01, 0.05, 0.2)):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective, PushObjective
    from world import build_world, control_step, goal_distance
    out = {}
    tasks = {"panda reach": ("C2", PandaReachObjective, lambda w: goal_distance(w)),
             "boxer push": ("C3", lambda: PushObjective(robot="boxer", link="ee_link"),
                            lambda w: float(torch.linalg.norm(w.get_actor_position_by_name("block")[0, 0:2] - w.get_actor_position_by_name("goal")[0, 0:2])))}
    for task, (name, obj, dist) in tasks.items():
        for rho in targets:
            _, world = build_world(CONFIGS[name], device="cuda:0")
            planner = MPPIisaacPlanner(_cfg(name, ess=rho), obj(), use_cuda_graph=True)
            start = dist(world)
            lams = []
            for _ in range(steps):
                control_step(world, planner)
                if rho is not None:
                    lams.append(float(planner.mppi.current_lambda))
            key = f"{task}, " + ("shipped lambda_" if rho is None else f"ess_target {rho}")
            out[key] = {"K": int(planner.mppi.K_total), "steps": steps, "lambda_": float(planner.mppi.lambda_), "start_distance": start,
                        "final_distance": dist(world), "chosen_lambda_min": min(lams) if lams else None,
                        "chosen_lambda_median": statistics.median(lams) if lams else None, "chosen_lambda_max": max(lams) if lams else None}
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
        raise SystemExit("temperature_bench needs a CUDA device")
    out = {"card": card(), "kernels": [kernel_profile(n, K, m, a.rounds) for n, K, m in SHAPES] if "kernels" in parts else None,
           "plan": plan_ab(a.plans) if "plan" in parts else None,
           "closed_loop": closed_loop(a.steps) if "closed_loop" in parts else None}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
