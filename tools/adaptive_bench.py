"""Cost of adaptive MPPI (update_cov / update_lambda) on the device.

1. K3 alone with and without the second-moment row (a registered distribution with update_cov), cold L2: inputs rotated over more
   than twice the L2 size as bench.py's roofline sweep does, both variants alternated round by round in one process.
2. The panda reach plan (config_panda_b200: K = 10 000, T = 30) with both flags on against both flags off, plans of the two planners
   alternated in blocks, L2 flushed before every plan, CUDA-graph replay as in production.

Prints the card name and its power limit (read through NVML, nothing is changed) next to the numbers.
    python tools/adaptive_bench.py [--ks 10000,65536,262144] [--rounds 5] [--plans 200]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(int((os.environ.get("CUDA_VISIBLE_DEVICES") or "0").split(",")[0] or 0))
        out["power_limit_w"] = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception as e:  # noqa: BLE001
        out["power_limit_w"] = f"unavailable ({type(e).__name__})"
    return out


def graph_time_us(fn, reps, replays=3):
    fn(); torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay(); torch.cuda.synchronize()
    best = float("inf")
    for _ in range(replays):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); g.replay(); b.record(); torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) * 1e3 / reps)
    return best


def k3_sweep(ks, rounds):
    from mppi_isaac_b200.backend import CudaBackend
    from mppi_isaac_b200.model.blob import OBS_DOF_STATE, build_scene, make_params
    from mppi_isaac_b200.utils.config_store import load_actor_cfgs, load_isaacgym_config
    cfg = load_isaacgym_config("config_panda_b200")
    sc = build_scene(load_actor_cfgs(["panda_stick", "goal"]))
    T, nu = int(cfg.mppi.horizon), sc.nu
    res = []
    for K in ks:
        bes = {}
        for name, adaptive in (("fixed", False), ("second_moment", True)):
            cfg.mppi.update_cov = cfg.mppi.update_lambda = adaptive
            p = make_params(cfg.mppi, cfg.isaacgym, nu, K, [(OBS_DOF_STATE, 0)])
            be = CudaBackend("cuda:0")
            be.create(sc.model, p)
            if adaptive:
                dist = torch.tensor([p.lambda_] + [0.1] * nu, device="cuda:0")
                be.set_distribution(dist)
                bes[name] = (be, torch.zeros(2 + 2 * T * nu, device="cuda:0"), dist)
            else:
                bes[name] = (be, torch.zeros(2 + T * nu, device="cuda:0"), None)
        bytes_alg = 4 * K * T * (nu + 1)
        nbuf = min(64, max(2, int(np.ceil(300e6 / bytes_alg))))
        xs = [torch.randn((T, nu, K), device="cuda:0") * 0.3 for _ in range(nbuf)]
        cs = [torch.rand((T, K), device="cuda:0") * 10 for _ in range(nbuf)]
        U = torch.zeros((T, nu), device="cuda:0")
        times = {n: [] for n in bes}
        for r in range(rounds):
            for n in (list(bes) if r % 2 == 0 else list(bes)[::-1]):
                be, part, _ = bes[n]
                times[n].append(graph_time_us(lambda: [be.reduce(cs[i], xs[i], U, part) for i in range(nbuf)], 2) / nbuf)
        row = {"K": K, "T": T, "nu": nu, "bytes": bytes_alg, "l2": f"cold: {nbuf} rotating input sets"}
        for n, v in times.items():
            us = statistics.median(v)
            row[n] = {"us_median": us, "us_min": min(v), "us_max": max(v), "GBps": bytes_alg / (us * 1e-6) / 1e9}
        res.append(row)
        del xs, cs
        for be, _, _ in bes.values():
            be.destroy()
    return res


def plan_ab(plans, block=20):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from mppi_isaac_b200.utils.config_store import load_isaacgym_config
    import copy
    q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
    pls = {}
    for name, on in (("flags_off", False), ("flags_on", True)):
        cfg = copy.deepcopy(load_isaacgym_config("config_panda_b200"))
        cfg.mppi.device, cfg.mppi.update_cov, cfg.mppi.update_lambda = "cuda:0", on, on
        pl = MPPIisaacPlanner(cfg, PandaReachObjective(), use_cuda_graph=True)
        for _ in range(5):
            pl.compute_action(q0, [0.0] * 7)
        pls[name] = pl
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
    out["lambda_after"] = float(pls["flags_on"].mppi.current_lambda)
    out["cov_after"] = pls["flags_on"].mppi.cov_action.cpu().tolist()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="10000,65536,262144")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--plans", type=int, default=200)
    a = ap.parse_args()
    import __graft_entry__  # noqa: F401  (repository root on the path)
    out = {"card": card(), "k3": k3_sweep([int(k) for k in a.ks.split(",")], a.rounds), "plan_c2": plan_ab(a.plans)}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
