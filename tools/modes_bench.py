"""Cost of multi-modal MPPI (``n_modes``) on the device.

1. K3 alone (mppib_reduce), cold L2 (inputs rotated over more than twice the L2 size), device time from torch.profiler: M = 1 against the
   per-mode reduction with M = 4 and 16 at the C2 (panda reach, K = 10 000) and C3 (boxer_push) shapes, alternated round by round.
2. K4 alone (mppib_finalize, one shard row) at T*nu = 210 and 512 with M = 1, 4 and 16.
3. The panda-reach plan p50 / p10 / p90 (K = 10 000) with n_modes = 1 and 4, CUDA-graph replay as in production, L2 flushed before
   every plan, the two planners alternated in blocks.

Prints the card name and its power limit (read through NVML, nothing is changed) next to the numbers.
    python tools/modes_bench.py [--rounds 5] [--plans 200] [--out results.json]
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

CONFIGS = {"C2": "config_panda_b200", "C3": "config_boxer_push_b200"}


def _shape(name):
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = load_isaacgym_config(CONFIGS[name])
    nu = int(np.asarray(cfg.mppi.noise_sigma).shape[0])
    return int(cfg.mppi.num_samples) // 64 * 64, int(cfg.mppi.horizon), nu


def _handle(K, T, nu, M=1):
    from mppi_isaac_b200.backend import CudaBackend
    from mppi_isaac_b200.model.blob import OBS_DOF_STATE, make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    from synth_mppi import nu_model
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.1 * np.eye(nu)).tolist(),
                    u_min=[-0.2], u_max=[0.2], lambda_=0.05, sample_null_action=True, filter_u=T >= 9, n_modes=M)
    be = CudaBackend("cuda:0")
    be.create(nu_model(nu), make_params(mc, IsaacGymConfig(), nu, K, [(OBS_DOF_STATE, 0)]))
    if M > 1:
        be.set_distribution(torch.cat([torch.zeros(1 + M), torch.zeros(T * nu)]).to("cuda:0"))
    return be


def k3_profile(name, rounds):
    K, T, nu = _shape(name)
    hs = {f"M{M}": _handle(K, T, nu, M) for M in (1, 4, 16)}
    Us = {n: 0.1 * torch.ones((int(n[1:]), T, nu), device="cuda:0") for n in hs}
    parts = {n: torch.zeros(h.partial_row_floats(), device="cuda:0") for n, h in hs.items()}
    bytes_in = 4 * K * T * (nu + 1)
    nbuf = max(2, int(np.ceil(2 * 50e6 / bytes_in)) + 1)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    bufs = [(torch.rand((T, K), device="cuda:0", generator=g), 0.2 * torch.randn((T, nu, K), device="cuda:0", generator=g)) for _ in range(nbuf)]
    run = {n: (lambda h, U, part: lambda c, x: h.reduce(c, x, U, part))(h, Us[n], parts[n]) for n, h in hs.items()}
    out = {"config": name, "K": K, "T": T, "nu": nu, "l2": f"cold: {nbuf} rotating input pairs"}
    out.update(_profile(run, {n: r"mppib_reduce_ws_kernel" for n in run}, bufs, rounds))
    for h in hs.values():
        h.destroy()
    return out


def k4_profile(T, nu, rounds):
    K = 4096
    hs = {f"M{M}": _handle(K, T, nu, M) for M in (1, 4, 16)}
    g = torch.Generator(device="cuda:0").manual_seed(1)
    rows = {}
    for n, h in hs.items():
        M = int(n[1:])
        r = 0.01 * torch.randn((1, M, 2 + T * nu), device="cuda:0", generator=g)
        r[..., 0], r[..., 1] = torch.rand((1, M), device="cuda:0", generator=g), 50.0
        rows[n] = r.reshape(1, -1)
    U0 = {n: 0.05 * torch.randn((int(n[1:]), T, nu), device="cuda:0", generator=g) for n in hs}
    act, st = torch.zeros(nu, device="cuda:0"), torch.zeros(2, device="cuda:0")
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda:0")
    bufs = [(flush,)]
    run = {n: (lambda h, r, U: lambda f: (f.zero_(), h.finalize(r, 1, U, act, st)))(h, rows[n], U0[n]) for n, h in hs.items()}
    out = {"T": T, "nu": nu, "T*nu": T * nu, "l2": "cold: 256 MB zeroed before every launch"}
    out.update(_profile(run, {n: r"mppib_finalize_kernel" for n in run}, bufs, rounds))
    for h in hs.values():
        h.destroy()
    return out


def _planner(M):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = copy.deepcopy(load_isaacgym_config(CONFIGS["C2"]))
    cfg.mppi.device = "cuda:0"
    cfg.mppi.n_modes = M
    return MPPIisaacPlanner(cfg, PandaReachObjective(), use_cuda_graph=True)


def plan_ab(plans, block=20):
    pls = {"n_modes_1": _planner(1), "n_modes_4": _planner(4)}
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
    out["K"] = int(pls["n_modes_1"].mppi.K_total)
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
        raise SystemExit("modes_bench needs a CUDA device")
    out = {"card": card(), "k3": [k3_profile(n, a.rounds) for n in ("C2", "C3")],
           "k4": [k4_profile(T, nu, a.rounds) for T, nu in ((30, 7), (32, 16))], "plan": plan_ab(a.plans)}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
