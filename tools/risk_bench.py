"""Cost of risk-aware MPPI (``n_worlds`` / ``cvar_alpha``) on the device.

1. K3 alone (mppib_reduce), cold L2 (inputs rotated over more than twice the L2 size), device time from torch.profiler: the plain
   reduction against the RISK one (R = 8, m = 2 and m = 8) at the C2 (panda reach, K = 10 000), C3 (boxer_push) and C4 (heijn_push)
   shapes, the variants alternated round by round in one process.
2. K1 (the Gaussian K1, cold L2) with R = 8 against R = 1 at the C3 shape.
3. The C3 and C4 plan p50 / p10 / p90 with n_worlds = 1 and 8 (cvar_alpha = 0.25), CUDA-graph replay as in production, L2 flushed
   before every plan, the two planners alternated in blocks.

Prints the card name and its power limit (read through NVML, nothing is changed) next to the numbers.
    python tools/risk_bench.py [--rounds 5] [--plans 200] [--out results.json]
"""
import argparse
import copy
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from adaptive_bench import card  # noqa: E402
from smooth_bench import _profile  # noqa: E402

CONFIGS = {"C2": "config_panda_b200", "C3": "config_boxer_push_b200", "C4": "config_heijn_push_b200"}
Q = {"C3": [0.0, 2.5, 0.0], "C4": [0.0, 0.0, 0.0]}


def _shape(name):
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = load_isaacgym_config(CONFIGS[name])
    nu = int(np.asarray(cfg.mppi.noise_sigma).shape[0])
    return int(cfg.mppi.num_samples) // 8 * 8, int(cfg.mppi.horizon), nu


def _handle(K, T, nu, R=1, alpha=1.0):
    from mppi_isaac_b200.backend import CudaBackend
    from mppi_isaac_b200.model.blob import OBS_DOF_STATE, make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    from synth_mppi import nu_model
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.1 * np.eye(nu)).tolist(),
                    u_min=[-0.2], u_max=[0.2], lambda_=0.05, sample_null_action=True, n_worlds=R, cvar_alpha=alpha)
    be = CudaBackend("cuda:0")
    be.create(nu_model(nu), make_params(mc, IsaacGymConfig(), nu, K, [(OBS_DOF_STATE, 0)]))
    return be


def k3_profile(name, rounds):
    K, T, nu = _shape(name)
    hs = {"plain": _handle(K, T, nu), "risk_R8_m2": _handle(K, T, nu, 8, 0.25), "risk_R8_m8": _handle(K, T, nu, 8, 1.0)}
    U = 0.1 * torch.ones((T, nu), device="cuda:0")
    part = torch.zeros(2 + T * nu, device="cuda:0")
    bytes_in = 4 * K * T * (nu + 1)
    nbuf = max(2, int(np.ceil(2 * 50e6 / bytes_in)) + 1)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    bufs = [(torch.rand((T, K), device="cuda:0", generator=g), 0.2 * torch.randn((T, nu, K), device="cuda:0", generator=g)) for _ in range(nbuf)]
    run = {n: (lambda h: lambda c, x: h.reduce(c, x, U, part))(h) for n, h in hs.items()}
    out = {"config": name, "K": K, "T": T, "nu": nu, "l2": f"cold: {nbuf} rotating input pairs"}
    out.update(_profile(run, {n: r"mppib_reduce_ws_kernel" for n in run}, bufs, rounds))
    for h in hs.values():
        h.destroy()
    return out


def k1_profile(name, rounds):
    K, T, nu = _shape(name)
    hs = {"R1": _handle(K, T, nu), "R8": _handle(K, T, nu, 8)}
    U = torch.zeros((T, nu), device="cuda:0")
    bytes_out = 2 * 4 * K * T * nu
    nbuf = max(2, int(np.ceil(2 * 50e6 / bytes_out)) + 1)
    bufs = [(torch.empty((T, nu, K), device="cuda:0"), torch.empty((T, nu, K), device="cuda:0")) for _ in range(nbuf)]
    run = {n: (lambda h: lambda a, x: h.sample(1, 0, 0, K, U, None, a, x))(h) for n, h in hs.items()}
    out = {"config": name, "K": K, "T": T, "nu": nu, "l2": f"cold: {nbuf} rotating output pairs"}
    out.update(_profile(run, {n: r"mppib_sample_kernel" for n in run}, bufs, rounds))
    for h in hs.values():
        h.destroy()
    return out


def _planner(name, R):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PushObjective
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = copy.deepcopy(load_isaacgym_config(CONFIGS[name]))
    cfg.mppi.device = "cuda:0"
    cfg.mppi.num_samples = int(cfg.mppi.num_samples) // 8 * 8
    cfg.mppi.n_worlds, cfg.mppi.cvar_alpha = R, 0.25
    obj = PushObjective(robot="boxer", link="ee_link") if name == "C3" else PushObjective()
    pl = MPPIisaacPlanner(cfg, obj, use_cuda_graph=True)
    pl.sim.reset_robot_state(Q[name], [0.0] * 3)
    return pl


def plan_ab(name, plans, block=20):
    pls = {"n_worlds_1": _planner(name, 1), "n_worlds_8": _planner(name, 8)}
    for pl in pls.values():
        for _ in range(5):
            pl.mppi.command()
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda:0")
    ms = {n: [] for n in pls}
    for b in range(max(1, plans // block)):
        for n in (list(pls) if b % 2 == 0 else list(pls)[::-1]):
            for _ in range(block):
                flush.zero_()
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); pls[n].mppi.command(); e.record(); e.synchronize()
                ms[n].append(a.elapsed_time(e))
    out = {n: {"p50_ms": statistics.median(v), "p10_ms": float(np.percentile(v, 10)), "p90_ms": float(np.percentile(v, 90)), "n": len(v)}
           for n, v in ms.items()}
    out["config"] = name
    out["K"] = int(pls["n_worlds_1"].mppi.K_total)
    out["graph_captured"] = {n: pl.mppi._graph is not None for n, pl in pls.items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--plans", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__  # noqa: F401  (repository root on the path)
    if not torch.cuda.is_available():
        raise SystemExit("risk_bench needs a CUDA device")
    out = {"card": card(), "k3": [k3_profile(n, a.rounds) for n in ("C2", "C3", "C4")], "k1": k1_profile("C3", a.rounds),
           "plan": [plan_ab(n, a.plans) for n in ("C3", "C4")]}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
