"""Cost of Smooth MPPI (``mppi_mode: smooth``) on the device.

1. K1 alone, cold L2 (the output buffers rotated over more than twice the L2 size, the samplers alternated round by round in one
   process), device time from torch.profiler (CUDA activities): the smooth K1 against the white Gaussian K1 and the colored K1
   (beta = 2) at the C2 shape (K = 10 000, T = 30, nu = 7) and the C5 shape (K = 65 536, T = 30, nu = 9).
2. K3 alone (mppib_reduce), cold L2 (inputs rotated), in mode smooth (omega = 0.5) against SIMPLE at C2.
3. The panda reach plan (config_panda_b200: K = 10 000, T = 30) with `smooth` and with `simple` / `random`, plans of the two planners
   alternated in blocks, L2 flushed before every plan, CUDA-graph replay as in production: p50 / p10 / p90 of the device time per plan.

Prints the card name and its power limit (read through NVML, nothing is changed) next to the numbers.
    python tools/smooth_bench.py [--rounds 5] [--plans 200] [--out results.json]
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
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from adaptive_bench import card  # noqa: E402

Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]


def _handle(K, T, nu, mode, **kw):
    from mppi_isaac_b200.backend import CudaBackend
    from mppi_isaac_b200.model.blob import OBS_DOF_STATE, make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    from synth_mppi import nu_model
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode=mode, sampling_method="random", noise_sigma=(0.1 * np.eye(nu)).tolist(),
                    u_min=[-0.2], u_max=[0.2], lambda_=0.05, sample_null_action=True, **kw)
    be = CudaBackend("cuda:0")
    be.create(nu_model(nu), make_params(mc, IsaacGymConfig(), nu, K, [(OBS_DOF_STATE, 0)]))
    if mode == "smooth":
        be.set_smooth_state(torch.zeros(nu + T * nu, device="cuda:0"))
    return be


def _profile(run, pattern, bufs, rounds):
    """Median / min / max device time per launch of each entry of `run` (alternated), the kernels matched by pattern[name]."""
    from torch.profiler import ProfilerActivity, profile
    for f in run.values():                                                    # warm-up (module load, smem attribute)
        f(*bufs[0])
    torch.cuda.synchronize()
    us = {n: [] for n in run}
    for r in range(rounds):
        for n in (list(run) if r % 2 == 0 else list(run)[::-1]):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for b in bufs:
                    run[n](*b)
                torch.cuda.synchronize()
            tot = cnt = 0
            for ev in prof.key_averages():
                if ev.device_type == torch.autograd.DeviceType.CUDA and re.search(pattern[n], ev.key):
                    tot += ev.device_time_total
                    cnt += ev.count
            us[n].append(tot / max(1, cnt))
    return {n: {"us_median": statistics.median(v), "us_min": min(v), "us_max": max(v)} for n, v in us.items()}


def k1_profile(K, T, nu, rounds):
    from mppi_isaac_b200.planner.mppi import colored_noise_chol
    white, smooth = _handle(K, T, nu, "simple"), _handle(K, T, nu, "smooth", smooth_weight=0.5, du_min=[-1.0], du_max=[1.0])
    Lt = torch.from_numpy(colored_noise_chol(T, 2.0)).cuda()
    U = torch.zeros((T, nu), device="cuda:0")
    ctr = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    bytes_out = 2 * 4 * K * T * nu
    nbuf = max(2, int(np.ceil(2 * 50e6 / bytes_out)) + 1)
    bufs = [(torch.empty((T, nu, K), device="cuda:0"), torch.empty((T, nu, K), device="cuda:0")) for _ in range(nbuf)]
    run = {"random": lambda a, n: white.sample(1, 0, 0, K, U, None, a, n, ctr),
           "colored": lambda a, n: white.sample_colored(1, 0, 0, K, U, None, Lt, a, n, ctr),
           "smooth": lambda a, n: smooth.sample_smooth(1, 0, 0, K, U, a, n, ctr)}
    pattern = {"random": r"mppib_sample_kernel", "colored": r"mppib_sample_colored_kernel", "smooth": r"mppib_sample_smooth_kernel"}
    out = {"K": K, "T": T, "nu": nu, "beta": 2.0, "bytes_written": bytes_out, "l2": f"cold: {nbuf} rotating output pairs"}
    out.update(_profile(run, pattern, bufs, rounds))
    for n in run:
        out[n]["GBps_written"] = bytes_out / (out[n]["us_median"] * 1e-6) / 1e9
    white.destroy(); smooth.destroy()
    return out


def k3_profile(K, T, nu, rounds):
    simple, smooth = _handle(K, T, nu, "simple"), _handle(K, T, nu, "smooth", smooth_weight=0.5, du_min=[-1.0], du_max=[1.0])
    U = 0.1 * torch.ones((T, nu), device="cuda:0")
    part = torch.zeros(2 + T * nu, device="cuda:0")
    bytes_in = 4 * K * T * (nu + 1)
    nbuf = max(2, int(np.ceil(2 * 50e6 / bytes_in)) + 1)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    bufs = [(torch.rand((T, K), device="cuda:0", generator=g), 0.2 * torch.randn((T, nu, K), device="cuda:0", generator=g)) for _ in range(nbuf)]
    run = {"simple": lambda c, x: simple.reduce(c, x, U, part), "smooth": lambda c, x: smooth.reduce(c, x, U, part)}
    pattern = {n: r"mppib_reduce_ws_kernel" for n in run}
    out = {"K": K, "T": T, "nu": nu, "omega": 0.5, "bytes_read": bytes_in, "l2": f"cold: {nbuf} rotating input pairs"}
    out.update(_profile(run, pattern, bufs, rounds))
    simple.destroy(); smooth.destroy()
    return out


def _planner(mode):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    cfg = copy.deepcopy(load_isaacgym_config("config_panda_b200"))
    cfg.mppi.device = "cuda:0"
    if mode == "smooth":
        cfg.mppi.mppi_mode, cfg.mppi.filter_u = "smooth", False
        cfg.mppi.smooth_weight, cfg.mppi.du_min, cfg.mppi.du_max = 0.5, [-1.0], [1.0]
    return MPPIisaacPlanner(cfg, PandaReachObjective(), use_cuda_graph=True)


def plan_ab(plans, block=20):
    pls = {"simple_random": _planner("simple"), "smooth": _planner("smooth")}
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
        raise SystemExit("smooth_bench needs a CUDA device")
    out = {"card": card(), "k1": [k1_profile(10000, 30, 7, a.rounds), k1_profile(65536, 30, 9, a.rounds)],
           "k3_c2": k3_profile(10000, 30, 7, a.rounds), "plan_c2": plan_ab(a.plans)}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
