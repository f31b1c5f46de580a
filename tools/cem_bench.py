"""Cost of cross-entropy planning (``mppi_mode: cem``) on the device.

1. The elite kernel alone (mppib_reduce) and the fused elite + K4 launch (mppib_reduce_finalize), cold L2 (the cost / action buffers
   rotated over more than twice the L2 size), device time from torch.profiler (CUDA activities): the C2 shape (K = 10 000, T = 30,
   nu = 7) at E = 10 and E = 128, and the C5 shape (K = 65 536, T = 30, nu = 9) at E = 10.  Next to it the bytes the kernel reads.
2. The panda reach plan (config_panda_b200: K = 10 000, T = 30) with `cem` at I = 1 and I = 3 and with `colored` MPPI, plans of the
   planners alternated in blocks, L2 flushed before every plan, CUDA-graph replay as in production: p50 / p10 / p90 per plan.

Prints the card name and its power limit (read through NVML, nothing is changed) next to the numbers.
    python tools/cem_bench.py [--rounds 5] [--plans 200] [--out results.json]
"""
import argparse
import copy
import json
import os
import re
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from adaptive_bench import card  # noqa: E402

Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]


def elite_profile(K, T, nu, E, rounds):
    """Mean device time per launch of the elite kernel, split and fused with K4 (torch.profiler), inputs rotated over > 2x the L2."""
    from torch.profiler import ProfilerActivity, profile
    from mppi_isaac_b200.backend import CudaBackend, cem_row_floats, dist_floats
    from mppi_isaac_b200.model.blob import OBS_DOF_STATE, make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from synth_mppi import nu_model
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode="cem", sampling_method="colored", noise_sigma=(0.1 * np.eye(nu)).tolist(),
                    u_min=[-0.2], u_max=[0.2], lambda_=0.05, sample_null_action=True, n_elites=E)
    params = make_params(mc, IsaacGymConfig(), nu, K, [(OBS_DOF_STATE, 0)])
    be = CudaBackend("cuda:0")
    be.create(nu_model(nu), params)
    state = torch.zeros(dist_floats(params, nu)[0], device="cuda:0")
    state[2 + E:2 + E + T * nu] = 0.3
    be.set_distribution(state)
    U = torch.zeros((T, nu), device="cuda:0")
    part = torch.zeros(cem_row_floats(T, nu, E), device="cuda:0")
    act, stats = torch.zeros(nu, device="cuda:0"), torch.zeros(2, device="cuda:0")
    bytes_in = 4 * K * T * (nu + 1)
    nbuf = max(2, int(np.ceil(2 * 50e6 / bytes_in)) + 1)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    bufs = [(torch.rand((T, K), device="cuda:0", generator=g), 0.2 * torch.rand((T, nu, K), device="cuda:0", generator=g)) for _ in range(nbuf)]
    run = {"elite": lambda c, x: be.reduce(c, x, U, part),
           "elite+K4": lambda c, x: be.reduce_finalize(c, x, U, part, act, stats)}
    for f in run.values():
        f(*bufs[0])
    torch.cuda.synchronize()
    us = {n: [] for n in run}
    for r in range(rounds):
        for n in (list(run) if r % 2 == 0 else list(run)[::-1]):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for c, x in bufs:
                    run[n](c, x)
                torch.cuda.synchronize()
            tot = cnt = 0
            for ev in prof.key_averages():
                if ev.device_type == torch.autograd.DeviceType.CUDA and re.search(r"mppib_elite_kernel", ev.key):
                    tot += ev.device_time_total
                    cnt += ev.count
            us[n].append(tot / max(1, cnt))
    be.destroy()
    out = {"K": K, "T": T, "nu": nu, "E": E, "bytes_read": 4 * K * T + 4 * E * T * nu, "k3_bytes_read": bytes_in,
           "l2": f"cold: {nbuf} rotating input pairs"}
    for n, v in us.items():
        out[n] = {"us_median": statistics.median(v), "us_min": min(v), "us_max": max(v)}
    return out


def _planner(mode, iters=1):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = copy.deepcopy(load_isaacgym_config("config_panda_b200"))
    cfg.mppi.device, cfg.mppi.sampling_method = "cuda:0", "colored"
    if mode == "cem":
        cfg.mppi.mppi_mode, cfg.mppi.cem_iterations = "cem", iters
    return MPPIisaacPlanner(cfg, PandaReachObjective(), use_cuda_graph=True)


def plan_ab(plans, block=20):
    pls = {"colored": _planner("colored"), "cem_I1": _planner("cem", 1), "cem_I3": _planner("cem", 3)}
    for pl in pls.values():
        for _ in range(5):
            pl.compute_action(Q0, [0.0] * 7)
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda:0")
    ms = {n: [] for n in pls}
    for b in range(max(1, plans // block)):
        order = list(pls) if b % 2 == 0 else list(pls)[::-1]
        for n in order:
            pl = pls[n]
            for _ in range(block):
                flush.zero_()
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); pl.mppi.command(); e.record(); e.synchronize()
                ms[n].append(a.elapsed_time(e))
    out = {n: {"p50_ms": statistics.median(v), "p10_ms": float(np.percentile(v, 10)), "p90_ms": float(np.percentile(v, 90)), "n": len(v)}
           for n, v in ms.items()}
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
        raise SystemExit("cem_bench needs a CUDA device")
    out = {"card": card(),
           "elite": [elite_profile(10000, 30, 7, 10, a.rounds), elite_profile(10000, 30, 7, 128, a.rounds),
                     elite_profile(65536, 30, 9, 10, a.rounds)],
           "plan_c2": plan_ab(a.plans)}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
