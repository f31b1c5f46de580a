"""Cost of adaptive MPPI (update_cov / update_lambda) on the device.

1. K3 alone without and with the second-moment row (a registered distribution with update_cov), and with the covariance row of
   cov_type full, cold L2: inputs rotated over more than twice the L2 size as bench.py's roofline sweep does, the variants alternated
   round by round in one process.  Panda (T = 30, nu = 7) and omnipanda (T = 30, nu = 12).
2. The panda reach plan (config_panda_b200: K = 10 000, T = 30) with both flags off, with both flags on (diagonal rule), with both
   flags on and cov_type full, and with both flags on and cov_type horizon (n = T*nu = 210), plans of the planners alternated in
   blocks, L2 flushed before every plan, CUDA-graph replay as in production.
3. Per-kernel device times of the cov_type full and horizon plans (torch.profiler with CUDA activities, in a run of its own after
   the timed plans): K1, K3, the SYRK and K4 of the horizon rule next to the kernels of the full rule.

Prints the card name and its power limit (read through NVML, nothing is changed) next to the numbers.
    python tools/adaptive_bench.py [--ks 10000,65536,262144] [--rounds 5] [--plans 200] [--scenes panda,omnipanda]
"""
import argparse
import json
import os
import re
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


def k3_sweep(ks, rounds, actors=("panda_stick", "goal")):
    from mppi_isaac_b200.backend import CudaBackend
    from mppi_isaac_b200.model.blob import OBS_DOF_STATE, build_scene, make_params
    from mppi_isaac_b200.utils.config_store import load_actor_cfgs, load_isaacgym_config
    cfg = load_isaacgym_config("config_panda_b200")
    sc = build_scene(load_actor_cfgs(list(actors)))
    T, nu = int(cfg.mppi.horizon), sc.nu
    res = []
    for K in ks:
        bes = {}
        for name, adaptive in (("fixed", False), ("second_moment", True), ("full", True)):
            cfg.mppi.update_cov = cfg.mppi.update_lambda = adaptive
            cfg.mppi.cov_type = "full" if name == "full" else "diag"
            if np.asarray(cfg.mppi.noise_sigma).shape != (nu, nu):                # a scene other than the config's robot
                cfg.mppi.noise_sigma = (0.1 * np.eye(nu)).tolist()
            p = make_params(cfg.mppi, cfg.isaacgym, nu, K, [(OBS_DOF_STATE, 0)])
            be = CudaBackend("cuda:0")
            be.create(sc.model, p)
            if name == "full":
                L = 0.3 * np.eye(nu)
                dist = torch.tensor(np.concatenate([[p.lambda_], (L @ L.T).ravel(), L.ravel(), np.linalg.inv(L @ L.T).ravel()]),
                                    dtype=torch.float32, device="cuda:0")
                be.set_distribution(dist)
                bes[name] = (be, torch.zeros(be.partial_row_floats(), device="cuda:0"), dist)
            elif adaptive:
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
    for name, on in (("flags_off", False), ("flags_on", True), ("flags_on_full", True), ("flags_on_horizon", True)):
        cfg = copy.deepcopy(load_isaacgym_config("config_panda_b200"))
        cfg.mppi.device, cfg.mppi.update_cov, cfg.mppi.update_lambda = "cuda:0", on, on
        cfg.mppi.cov_type = {"flags_on_full": "full", "flags_on_horizon": "horizon"}.get(name, "diag")
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
    out["sigma_after_full"] = pls["flags_on_full"].mppi.cov_action.cpu().tolist()
    S_h = pls["flags_on_horizon"].mppi.cov_action.double().cpu()
    out["sigma_h_after"] = {"n": S_h.shape[0], "max_abs": float(S_h.abs().max()),
                            "max_abs_off_block_diagonal": float((S_h - torch.block_diag(*[S_h[i:i + 7, i:i + 7] for i in range(0, S_h.shape[0], 7)])).abs().max()),
                            "cond": float(torch.linalg.cond(S_h))}
    out["kernels_us"] = kernel_times({n: pls[n] for n in ("flags_on_full", "flags_on_horizon")}, flush)
    return out


def kernel_times(pls, flush, plans=50):
    """Mean device time per launch of every kernel of a plan (torch.profiler, CUDA activities), per planner."""
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for n, pl in pls.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(plans):
                flush.zero_()
                pl.mppi.command()
            torch.cuda.synchronize()
        rows = {}
        for ev in prof.key_averages():
            if ev.device_type == torch.autograd.DeviceType.CUDA and "mppib" in ev.key:
                key = ev.key.replace("(anonymous namespace)", "")
                name = re.search(r"mppib_\w+", key).group(0) + ("<" + key.split("<", 1)[1].split(">")[0] + ">" if "<" in key.split("(")[0] else "")
                r = rows.setdefault(name, {"us": 0.0, "count": 0})
                r["us"] += ev.device_time_total
                r["count"] += ev.count
        out[n] = {k: round(v["us"] / max(1, v["count"]), 2) for k, v in rows.items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="10000,65536,262144")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--plans", type=int, default=200)
    ap.add_argument("--scenes", default="panda,omnipanda")
    a = ap.parse_args()
    import __graft_entry__  # noqa: F401  (repository root on the path)
    scenes = {"panda": ("panda_stick", "goal"), "omnipanda": ("omnipanda", "goal")}
    ks = [int(k) for k in a.ks.split(",")]
    out = {"card": card(), "k3": [r for s in a.scenes.split(",") for r in k3_sweep(ks, a.rounds, scenes[s])], "plan_c2": plan_ab(a.plans)}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
