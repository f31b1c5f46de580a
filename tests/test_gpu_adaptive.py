"""-m gpu: adaptive MPPI (update_cov / update_lambda) on the device against the CPU reference of ``adaptive_oracle``: the K1 variants,
the second-moment row of K3, the distribution update of K4, and whole plans through the planner (graph, eager, fused, split)."""
import copy

import numpy as np
import pytest
import torch

import adaptive_oracle as ada
from mppi_isaac_b200.model.blob import MODE_SIMPLE
from scenes import boxer_cfg, gripper_setup, panda_cfg, panda_setup, point_setup

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]


def gpu_backend(sc, p, dist=None):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(sc.model, p)
    if dist is not None:
        be.set_distribution(dist)
    return be


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def _dist(nu, lam=0.05, seed=0):
    rng = np.random.default_rng(seed)
    return np.concatenate([[lam], rng.uniform(0.02, 0.3, nu)]).astype(np.float32)


def test_k1_diagonal_variants_match_the_reference(oracle):
    sc, p, _ = panda_setup(K=1000, T=30, update_cov=True)
    nu, T, K = sc.nu, p.T, p.K
    d = _dist(nu)
    be = gpu_backend(sc, p, dev(d))
    U = np.random.default_rng(1).uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    be.sample(11, 3, 0, K, dev(U), None, a, n)
    a_ref, n_ref = oracle.sample(sc.model, ada.dist_params(p, nu, d), 11, 3, U)
    scale = float(np.sqrt(d[1:].max()))                                     # the tolerance of the fixed-Sigma K1 test
    assert np.abs(a.cpu().numpy() - a_ref).max() <= 2e-6 * max(1.0, 6 * scale)
    assert np.abs(n.cpu().numpy() - n_ref).max() <= 2e-6 * max(1.0, 6 * scale)
    # Halton library: white on the device, scaled by sqrt(cov) per plan
    from mppi_isaac_b200.planner.mppi import halton_spline_operator, halton_table
    nk = T // 4
    B, tab = halton_spline_operator(T, nk), halton_table(nk * nu, 3)
    Z = torch.zeros((T, nu, K), device=DEV)
    be.noise_library(0, K, dev(tab, torch.int32), dev(B), nk, Z)
    Z_ref = oracle.noise_library(sc.model, ada.dist_params(p, nu, d, white=True), tab, B, nk)
    assert np.abs(Z.cpu().numpy() - Z_ref).max() <= 1e-4                    # the tolerance of the coloured library (float erfinvf)
    assert np.median(np.abs(Z.cpu().numpy() - Z_ref)) <= 1e-6
    be.sample_library(0, K, dev(U), None, Z, a, n)
    a_ref, n_ref = oracle.sample_library(sc.model, p, U, np.sqrt(d[1:])[None, :, None] * Z.cpu().numpy())
    np.testing.assert_allclose(a.cpu().numpy(), a_ref, rtol=0, atol=1e-6)
    np.testing.assert_allclose(n.cpu().numpy(), n_ref, rtol=0, atol=1e-6)


@pytest.mark.parametrize("which,K", [("panda", 10000), ("gripper", 65536), ("point", 65536), ("panda", 131072)])
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_k3_second_moment_row_matches_the_reference(oracle, which, K, mode):
    setup, T = {"gripper": (gripper_setup, 30), "point": (point_setup, 12), "panda": (panda_setup, 30)}[which]
    sc, p, _ = setup(K=K, T=T, mode=mode, update_cov=True, update_lambda=True)
    nu, NR = sc.nu, T * sc.nu
    d = _dist(nu, lam=0.3)
    be = gpu_backend(sc, p, dev(d))
    rng = np.random.default_rng(7)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    x = (rng.standard_normal((T, nu, K)) * 0.3).astype(np.float32)
    if p.mode != MODE_SIMPLE:
        x += U[:, :, None]
    cost = rng.uniform(0, 10, (T, K)).astype(np.float32)
    cost[:, K // 3] = np.nan
    partial = torch.zeros(2 + 2 * NR, device=DEV)
    for _ in range(2):
        be.reduce(dev(cost), dev(x), dev(U), partial)
    ref = ada.reduce(sc.model, p, cost, x, U, d)
    pg = partial.cpu().numpy()
    assert abs(pg[0] - ref[0]) <= 1e-5 * max(1, abs(ref[0]))
    np.testing.assert_allclose(pg[1], ref[1], rtol=5e-5)
    for sl in (slice(2, 2 + NR), slice(2 + NR, None)):
        assert np.abs(pg[sl] - ref[sl]).max() <= 1e-5 * max(1.0, np.abs(ref[sl]).max())
    # K4 on the row: U and the updated distribution
    Ud, act, st, dd = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV), dev(d)
    be.set_distribution(dd)
    be.finalize(partial.view(1, -1), 1, Ud, act, st)
    U_ref, _, _, d_ref = ada.finalize(sc.model, p, pg[None], U, d)
    np.testing.assert_allclose(Ud.cpu().numpy(), U_ref, rtol=0, atol=1e-5 * max(1.0, np.abs(U_ref).max()))
    np.testing.assert_allclose(dd.cpu().numpy(), d_ref, rtol=2e-5, atol=1e-7)


def test_flags_off_with_a_registered_distribution_is_bit_identical(oracle):
    sc, p, _ = panda_setup(K=4096, T=30, mode="simple", filter_u=True)
    nu, T, K = sc.nu, p.T, p.K
    rng = np.random.default_rng(2)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    a, n = oracle.sample(sc.model, p, 3, 0, U)
    cost = rng.uniform(0, 10, (T, K)).astype(np.float32)
    outs = []
    for d in (None, dev([p.lambda_] + [0.1] * nu)):
        be = gpu_backend(sc, p, d)
        part, Ud, act, st = torch.zeros(2 + T * nu, device=DEV), dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        be.reduce(dev(cost), dev(n), Ud, part)
        be.finalize(part.view(1, -1), 1, Ud, act, st)
        outs.append((part.cpu(), Ud.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_fused_tail_equals_split_reduce_and_finalize(oracle, mode):
    sc, p, _ = panda_setup(K=10000, T=30, mode=mode, filter_u=True, update_cov=True, update_lambda=True, eta_u_bound=50.0, eta_l_bound=5.0)
    nu, T, K = sc.nu, p.T, p.K
    rng = np.random.default_rng(4)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    d = _dist(nu, lam=0.5)
    a, n = oracle.sample(sc.model, ada.dist_params(p, nu, d), 3, 0, U)
    x = dev(n if p.mode == MODE_SIMPLE else a)
    cost = dev(rng.uniform(0, 10, (T, K)).astype(np.float32))
    res = []
    for fused in (True, False):
        dd = dev(d)
        be = gpu_backend(sc, p, dd)
        part, Ud, act, st = torch.zeros(2 + 2 * T * nu, device=DEV), dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        if fused:
            be.reduce_finalize(cost, x, Ud, part, act, st)
        else:
            be.reduce(cost, x, Ud, part)
            be.finalize(part.view(1, -1), 1, Ud, act, st)
        res.append([t.cpu() for t in (part, Ud, act, st, dd)])
        assert not torch.equal(dd.cpu(), torch.from_numpy(d))
    for u, v in zip(*res):
        assert torch.equal(u, v)


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("G", [4, 8])
def test_k4_combines_g_shard_rows_like_one(oracle, mode, G):
    """G shards through K3 (update_cov) and ONE split K4 over the G rows == the single-shard launch: the K4 combine of M2 over
    several rows, at the row stride of the long row."""
    K = 10000 if G == 4 else 10240                                            # shards stay multiples of 4
    sc, p, _ = panda_setup(K=K, T=30, mode=mode, filter_u=True, update_cov=True, update_lambda=True, eta_u_bound=50.0, eta_l_bound=5.0)
    nu, T = sc.nu, p.T
    P = 2 + 2 * T * nu
    rng = np.random.default_rng(11)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    d = _dist(nu, lam=0.5)
    a, n = oracle.sample(sc.model, ada.dist_params(p, nu, d), 5, 0, U)
    x = dev(n if p.mode == MODE_SIMPLE else a)
    cost = dev(rng.uniform(0, 10, (T, K)).astype(np.float32))
    d1 = dev(d)
    be1 = gpu_backend(sc, p, d1)
    part1, U1, act, st1 = torch.zeros(P, device=DEV), dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be1.reduce(cost, x, U1, part1)
    be1.finalize(part1.view(1, -1), 1, U1, act, st1)
    pg = copy.copy(p); pg.K = K // G
    dG = dev(d)
    beG = gpu_backend(sc, pg, dG)
    parts = torch.zeros((G, P), device=DEV)
    UG = dev(U)
    for g in range(G):
        sl = slice(g * pg.K, (g + 1) * pg.K)
        beG.reduce(cost[:, sl].contiguous(), x[:, :, sl].contiguous(), UG, parts[g])
    stG = torch.zeros(2, device=DEV)
    beG.finalize(parts, G, UG, act, stG)
    # the rows against the reference, then the combine against the single launch
    for g in range(G):
        sl = slice(g * pg.K, (g + 1) * pg.K)
        ref = ada.reduce(sc.model, pg, np.ascontiguousarray(cost[:, sl].cpu().numpy()), np.ascontiguousarray(x[:, :, sl].cpu().numpy()), U, d)
        assert np.abs(parts[g, 2:].cpu().numpy() - ref[2:]).max() <= 1e-5 * max(1.0, np.abs(ref[2:]).max())
    torch.testing.assert_close(stG, st1, rtol=2e-6, atol=0)
    torch.testing.assert_close(UG, U1, atol=2e-6, rtol=0)
    torch.testing.assert_close(dG, d1, rtol=2e-6, atol=0)
    assert not torch.equal(d1.cpu(), torch.from_numpy(d))
    U_ref, _, _, d_ref = ada.finalize(sc.model, p, parts.cpu().numpy(), U, d)
    np.testing.assert_allclose(dG.cpu().numpy(), d_ref, rtol=2e-5, atol=1e-7)


def _planners(kind, graph=True, K=1000):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective, PushObjective
    flags = dict(update_cov=True, update_lambda=True)
    if kind == "panda":
        mk, obj = (lambda d: panda_cfg(K=K, T=30, device=d, eta_u_bound=40.0, eta_l_bound=4.0, **flags)), PandaReachObjective
    else:
        mk, obj = (lambda d: boxer_cfg(K=512, T=12, device=d, eta_u_bound=40.0, eta_l_bound=4.0, **flags)), (lambda: PushObjective(robot="boxer", link="ee_link"))
    gpu = MPPIisaacPlanner(mk(DEV), obj(), use_cuda_graph=graph)
    cpu = MPPIisaacPlanner(mk("cpu"), obj(), backend=ada.AdaptiveOracleBackend(nthreads=8))
    return gpu, cpu


@pytest.mark.parametrize("kind,plans", [("panda", 20), ("boxer", 20)])
def test_planner_tracks_the_reference(kind, plans):
    gpu, cpu = _planners(kind)
    q = Q0 if kind == "panda" else [0.0, 2.5, 0.0]
    qd = [0.0] * len(q)
    # bounds a few times above the worst values measured on an H100 (panda, free-running: action 8e-6, U 1.4e-5, cov 2.2e-5 relative;
    # boxer, re-synced every plan: 5.3e-5, 7.3e-5, 1.2e-4); a wrong kappa or step size moves cov by more than 10 %
    tol, cov_rtol = (1e-4, 1e-4) if kind == "panda" else (5e-4, 5e-4)
    d0 = gpu.mppi.dist.cpu().clone()
    for it in range(plans):
        if kind == "boxer":
            # contact scenes: rollouts differ by float32 rounding that the penalty contacts amplify, and lambda = 0.01 turns that
            # into visibly different weights within a few plans; the reference therefore plans from the device's U and dist
            cpu.mppi.U.copy_(gpu.mppi.U.cpu())
            cpu.mppi.dist.copy_(gpu.mppi.dist.cpu())
        ag, ac = gpu.compute_action(q, qd), cpu.compute_action(q, qd)
        assert float((ag - ac).abs().max()) <= tol, f"plan {it}"
        np.testing.assert_allclose(gpu.mppi.U.cpu().numpy(), cpu.mppi.U.numpy(), rtol=0, atol=tol, err_msg=f"plan {it}")
        np.testing.assert_allclose(float(gpu.mppi.current_lambda), float(cpu.mppi.current_lambda), rtol=1e-5, err_msg=f"plan {it}")
        np.testing.assert_allclose(gpu.mppi.cov_action.cpu().numpy(), cpu.mppi.cov_action.numpy(), rtol=cov_rtol, atol=0, err_msg=f"plan {it}")
    assert gpu.mppi._graph is not None
    assert not torch.equal(gpu.mppi.dist.cpu(), d0)


@pytest.mark.parametrize("kind", ["panda", "boxer"])
def test_captured_graph_and_eager_plans_are_bit_identical(kind):
    """The graph reads the live distribution buffer: replaying it (never re-captured) gives the eager path's U and dist bit for bit."""
    g, _ = _planners(kind, graph=True)
    e, _ = _planners(kind, graph=False)
    q = Q0 if kind == "panda" else [0.0, 2.5, 0.0]
    d0 = g.mppi.dist.clone()
    graph = None
    for it in range(20):
        g.compute_action(q, [0.0] * len(q))
        e.compute_action(q, [0.0] * len(q))
        graph = graph or g.mppi._graph
        assert g.mppi._graph is graph, "the plan graph was re-captured"
        assert torch.equal(g.mppi.dist, e.mppi.dist) and torch.equal(g.mppi.U, e.mppi.U), f"plan {it}"
    assert e.mppi._graph is None and not torch.equal(g.mppi.dist, d0)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_peer_and_nccl_exchanges_agree_on_dist():
    """2 ranks, both flags on: the peer-memory exchange of the long [beta, eta, W, M2] row and the NCCL all-gather give the same action and
    the same dist bit for bit, and the ranks agree on dist."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    res = {}
    for exch in ("peer", "nccl"):
        env = dict(os.environ, MPPIB_EXCHANGE=exch, MPPIB_PEER_TIMEOUT_S="10")
        out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                              "--master-port", "29541", os.path.join(here, "adaptive_dist_worker.py")],
                             capture_output=True, text=True, timeout=300, env=env, cwd=os.path.dirname(here))
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
        lines = [ln.split() for ln in out.stdout.splitlines() if ln.startswith("RESULT ")]
        assert len(lines) == 2 and all(ln[1] == exch for ln in lines), out.stdout[-2000:]
        assert lines[0][3:] == lines[1][3:], "the ranks disagree on the action or on dist"
        res[exch] = lines[0][3:]
    assert res["peer"] == res["nccl"]
