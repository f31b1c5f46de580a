"""Cost of colored-noise sampling (``sampling_method: colored``) against the white Gaussian K1 (``random``) on the device.

1. K1 alone, cold L2 (the output buffers rotated over more than twice the L2 size, the two samplers alternated round by round in one
   process), device time from torch.profiler (CUDA activities): the C2 shape (K = 10 000, T = 30, nu = 7) and the C5 shape
   (K = 65 536, T = 30, nu = 9), beta = 2.  Next to it the bytes K1 has to write and the FFMA the temporal colour adds.
2. The panda reach plan (config_panda_b200: K = 10 000, T = 30) with `random` and with `colored`, plans of the two planners alternated
   in blocks, L2 flushed before every plan, CUDA-graph replay as in production: p50 / p10 / p90 of the device time per plan.

Prints the card name and its power limit (read through NVML, nothing is changed) next to the numbers.
    python tools/colored_bench.py [--rounds 5] [--plans 200] [--out results.json]
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


def k1_profile(K, T, nu, rounds, beta=2.0):
    """Mean device time per launch of the white and the colored K1 (torch.profiler), outputs rotated over > 2x the L2 size."""
    from torch.profiler import ProfilerActivity, profile
    from mppi_isaac_b200.backend import CudaBackend
    from mppi_isaac_b200.model.blob import OBS_DOF_STATE, make_params
    from mppi_isaac_b200.planner.mppi import colored_noise_chol
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from synth_mppi import nu_model
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.1 * np.eye(nu)).tolist(),
                    u_min=[-0.2], u_max=[0.2], lambda_=0.05, sample_null_action=True)
    be = CudaBackend("cuda:0")
    be.create(nu_model(nu), make_params(mc, IsaacGymConfig(), nu, K, [(OBS_DOF_STATE, 0)]))
    Lt = torch.from_numpy(colored_noise_chol(T, beta)).cuda()
    U = torch.zeros((T, nu), device="cuda:0")
    ctr = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    bytes_out = 2 * 4 * K * T * nu
    nbuf = max(2, int(np.ceil(2 * 50e6 / bytes_out)) + 1)
    bufs = [(torch.empty((T, nu, K), device="cuda:0"), torch.empty((T, nu, K), device="cuda:0")) for _ in range(nbuf)]
    run = {"random": lambda a, n: be.sample(1, 0, 0, K, U, None, a, n, ctr),
           "colored": lambda a, n: be.sample_colored(1, 0, 0, K, U, None, Lt, a, n, ctr)}
    for f in run.values():                                                    # warm-up (module load, smem attribute)
        f(*bufs[0])
    torch.cuda.synchronize()
    us = {n: [] for n in run}
    for r in range(rounds):
        for n in (list(run) if r % 2 == 0 else list(run)[::-1]):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for a, nz in bufs:
                    run[n](a, nz)
                torch.cuda.synchronize()
            tot = cnt = 0
            for ev in prof.key_averages():
                if ev.device_type == torch.autograd.DeviceType.CUDA and re.search(r"mppib_sample(_colored)?_kernel", ev.key):
                    tot += ev.device_time_total
                    cnt += ev.count
            us[n].append(tot / max(1, cnt))
    be.destroy()
    out = {"K": K, "T": T, "nu": nu, "beta": beta, "bytes_written": bytes_out, "colour_ffma": K * nu * T * (T + 1) // 2,
           "l2": f"cold: {nbuf} rotating output pairs"}
    for n, v in us.items():
        med = statistics.median(v)
        out[n] = {"us_median": med, "us_min": min(v), "us_max": max(v), "GBps_written": bytes_out / (med * 1e-6) / 1e9}
    return out


def _planner(sampling, beta=2.0, K=None):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = copy.deepcopy(load_isaacgym_config("config_panda_b200"))
    cfg.mppi.device, cfg.mppi.sampling_method, cfg.mppi.noise_beta = "cuda:0", sampling, beta
    if K is not None:
        cfg.mppi.num_samples = K
    return MPPIisaacPlanner(cfg, PandaReachObjective(), use_cuda_graph=True)


def plan_ab(plans, block=20):
    pls = {n: _planner(n) for n in ("random", "colored")}
    for pl in pls.values():
        for _ in range(5):
            pl.compute_action(Q0, [0.0] * 7)
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda:0")
    ms = {n: [] for n in pls}
    for b in range(max(1, plans // block)):
        for n in (list(pls) if b % 2 == 0 else list(pls)[::-1]):
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
        raise SystemExit("colored_bench needs a CUDA device")
    out = {"card": card(),
           "k1": [k1_profile(10000, 30, 7, a.rounds), k1_profile(65536, 30, 9, a.rounds)],
           "plan_c2": plan_ab(a.plans)}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
