"""-m gpu: adaptive MPPI with a full sampling covariance (update_cov with cov_type: full) on the device against the CPU reference of
``adaptive_full_oracle``: the full-colour K1 variants, the covariance row C of K3, the Sigma / L / Sigma^-1 update of K4, and whole
plans through the planner (graph, eager, fused, split)."""
import copy

import numpy as np
import pytest
import torch

import adaptive_full_oracle as afo
from mppi_isaac_b200.model.blob import MODE_SIMPLE, OBS_DOF_STATE, build_scene, make_params
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, load_actor_cfgs
from scenes import boxer_cfg, panda_cfg, panda_mppi, panda_setup

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]


def corr_sigma(nu, scale=0.1, seed=3):
    """A symmetric positive-definite Sigma with strong correlations, diagonal about `scale`."""
    A = np.random.default_rng(seed).normal(0, 1.0, (nu, nu))
    S = A @ A.T / nu + 0.3 * np.eye(nu)
    S = scale * S / np.mean(np.diag(S))
    return 0.5 * (S + S.T)


def gpu_backend(sc, p, dist=None):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(sc.model, p)
    if dist is not None:
        be.set_distribution(dist)
    return be


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def omni_setup(K=64, T=30, mode="simple", **kw):
    """omnipanda (nu = 12): only its control dimension matters to K1 / K3 / K4."""
    sc = build_scene(load_actor_cfgs(["omnipanda", "goal"]))
    kw.setdefault("noise_sigma", (0.1 * np.eye(sc.nu)).tolist())
    p = make_params(panda_mppi(K, T, mode, **kw), IsaacGymConfig(), sc.nu, K, [(OBS_DOF_STATE, 0)])
    return sc, p, None


def _full(setup, K, T, mode="simple", lam=0.3, **kw):
    sc, _, _ = setup(K=4, T=T)
    sig = corr_sigma(sc.nu)
    sc, p, _ = setup(K=K, T=T, mode=mode, update_cov=True, cov_type="full", noise_sigma=sig.tolist(), **kw)
    return sc, p, afo.make_dist(lam, sig)


def _rel(a, b):
    return np.abs(np.asarray(a, np.float64) - b).max() / max(1.0, np.abs(b).max())


def test_k1_full_colour_variants_match_the_reference(oracle):
    sc, p, d = _full(panda_setup, 1000, 30, lam=0.05)
    nu, T, K = sc.nu, p.T, p.K
    be = gpu_backend(sc, p, dev(d))
    U = np.random.default_rng(1).uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    be.sample(11, 3, 0, K, dev(U), None, a, n)
    a_ref, n_ref = oracle.sample(sc.model, afo.dist_params(p, nu, d), 11, 3, U)
    sigma = float(np.sqrt(np.diag(afo.unpack(d, nu)[1]).max()))
    tol = 2e-6 * max(1.0, 6 * sigma)
    assert np.abs(a.cpu().numpy() - a_ref).max() <= tol
    assert np.abs(n.cpu().numpy() - n_ref).max() <= tol
    # Halton library: white on the device, coloured by the live L on every plan
    from mppi_isaac_b200.planner.mppi import halton_spline_operator, halton_table
    nk = T // 4
    B, tab = halton_spline_operator(T, nk), halton_table(nk * nu, 3)
    Z = torch.zeros((T, nu, K), device=DEV)
    be.noise_library(0, K, dev(tab, torch.int32), dev(B), nk, Z)
    Z_ref = oracle.noise_library(sc.model, afo.dist_params(p, nu, d, white=True), tab, B, nk)
    assert np.abs(Z.cpu().numpy() - Z_ref).max() <= 1e-4                    # the tolerance of the coloured library (float erfinvf)
    be.sample_library(0, K, dev(U), None, Z, a, n)
    a_ref, n_ref = oracle.sample_library(sc.model, p, U, afo.color_library(d, nu, Z.cpu().numpy()))
    scale = max(1.0, np.abs(Z.cpu().numpy()).max() * sigma)
    assert np.abs(a.cpu().numpy() - a_ref).max() <= 2e-6 * scale
    assert np.abs(n.cpu().numpy() - n_ref).max() <= 2e-6 * scale


def _check_dist(dd, d_ref, nu, rtol=1e-5):
    """Sigma against the reference to `rtol` of its largest entry; L L^T = Sigma and Sigma^-1 Sigma = I on the device's own values."""
    _, S, L, I = afo.unpack(dd, nu)
    _, Sr, _, _ = afo.unpack(d_ref, nu)
    assert _rel(S, Sr) <= rtol
    np.testing.assert_array_equal(S, S.T)
    np.testing.assert_array_equal(I, I.T)
    np.testing.assert_array_equal(L, np.tril(L))
    S64 = S.astype(np.float64)
    assert np.abs(L.astype(np.float64) @ L.T.astype(np.float64) - S64).max() <= 2e-6 * np.abs(S64).max()
    cond = np.linalg.cond(S64)
    assert np.abs(I.astype(np.float64) @ S64 - np.eye(nu)).max() <= 1e-6 * cond
    np.testing.assert_allclose(dd[0], d_ref[0], rtol=1e-6)


@pytest.mark.parametrize("which,K", [("panda", 10000), ("panda", 65536), ("panda", 131072), ("omni", 10000), ("omni", 65536), ("omni", 131072)])
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_k3_covariance_row_and_k4_update_match_the_reference(oracle, which, K, mode):
    setup = {"panda": panda_setup, "omni": omni_setup}[which]
    sc, p, d = _full(setup, K, 30, mode=mode, update_lambda=True)
    nu, NR, T = sc.nu, 30 * sc.nu, 30
    be = gpu_backend(sc, p, dev(d))
    rng = np.random.default_rng(7)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    L = afo.unpack(d, nu)[2].astype(np.float64)
    x = np.einsum("ji,tik->tjk", L, rng.standard_normal((T, nu, K))).astype(np.float32)
    if p.mode != MODE_SIMPLE:
        x += U[:, :, None]
    cost = rng.uniform(0, 10, (T, K)).astype(np.float32)
    cost[:, K // 3] = np.nan
    partial = torch.zeros(2 + NR + nu * (nu + 1) // 2, device=DEV)
    for _ in range(2):
        be.reduce(dev(cost), dev(x), dev(U), partial)
    ref = afo.reduce(sc.model, p, cost, x, U, d)
    pg = partial.cpu().numpy()
    assert abs(pg[0] - ref[0]) <= 1e-5 * max(1, abs(ref[0]))
    np.testing.assert_allclose(pg[1], ref[1], rtol=5e-5)
    for sl in (slice(2, 2 + NR), slice(2 + NR, None)):
        assert np.abs(pg[sl] - ref[sl]).max() <= 1e-5 * max(1.0, np.abs(ref[sl]).max())
    # K4 on the row: U and Sigma, L, Sigma^-1
    Ud, act, st, dd = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV), dev(d)
    be.set_distribution(dd)
    be.finalize(partial.view(1, -1), 1, Ud, act, st)
    U_ref, _, _, d_ref = afo.finalize(sc.model, p, pg[None], U, d)
    np.testing.assert_allclose(Ud.cpu().numpy(), U_ref, rtol=0, atol=1e-5 * max(1.0, np.abs(U_ref).max()))
    assert not np.array_equal(d_ref[1:], d[1:])
    _check_dist(dd.cpu().numpy(), d_ref, nu)


@pytest.mark.parametrize("fused", [True, False])
def test_k4_indefinite_update_leaves_sigma_l_and_inverse_unchanged(fused):
    """Hand-built partials whose Sigma update is indefinite (C = -100 I): K4 keeps Sigma, L and Sigma^-1 bit for bit and still
    applies the lambda rule.  The fused tail reaches the same branch through K3 on a single dominant sample."""
    sc, p, d = _full(panda_setup, 64, 12, update_lambda=True, eta_u_bound=10.0, eta_l_bound=5.0)
    nu, T = sc.nu, p.T
    NR, P = T * nu, 2 + T * nu + nu * (nu + 1) // 2
    dd = dev(d)
    be = gpu_backend(sc, p, dd)
    Ud, act, st = torch.zeros((T, nu), device=DEV), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    if fused:
        # one valid sample (all others NaN) with x = 0 gives C = 0 and V = 0; kappa < 0 is refused, so make the previous Sigma
        # indefinite instead: (1 - s) Sigma + kappa I with Sigma = -I is negative definite
        bad = d.copy()
        bad[1:1 + nu * nu] = (-np.eye(nu)).ravel()
        dd.copy_(dev(bad))
        cost = torch.full((T, p.K), float("nan"), device=DEV)
        cost[:, 5] = 1.0
        x = torch.zeros((T, nu, p.K), device=DEV)
        be.reduce_finalize(cost, x, Ud, torch.zeros(P, device=DEV), act, st)
        out = dd.cpu().numpy()
        np.testing.assert_array_equal(out[1:], bad[1:])
    else:
        row = np.zeros(P, np.float32)
        row[1] = 2.0                                                         # eta < eta_l_bound: lambda *= 1.1
        row[2 + NR:] = afo.tril_pack(-100.0 * np.eye(nu))
        be.finalize(dev(row).view(1, -1), 1, Ud, act, st)
        out = dd.cpu().numpy()
        np.testing.assert_array_equal(out[1:], d[1:])
    assert out[0] == np.float32(d[0]) * (np.float32(1) + np.float32(0.1))


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_fused_tail_equals_split_reduce_and_finalize(oracle, mode):
    sc, p, d = _full(panda_setup, 10000, 30, mode=mode, lam=0.5, filter_u=True, update_lambda=True, eta_u_bound=50.0, eta_l_bound=5.0)
    nu, T, K = sc.nu, p.T, p.K
    rng = np.random.default_rng(4)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    a, n = oracle.sample(sc.model, afo.dist_params(p, nu, d), 3, 0, U)
    x = dev(n if p.mode == MODE_SIMPLE else a)
    cost = dev(rng.uniform(0, 10, (T, K)).astype(np.float32))
    res = []
    for fused in (True, False):
        dd = dev(d)
        be = gpu_backend(sc, p, dd)
        part, Ud, act, st = torch.zeros(2 + T * nu + nu * (nu + 1) // 2, device=DEV), dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        if fused:
            be.reduce_finalize(cost, x, Ud, part, act, st)
        else:
            be.reduce(cost, x, Ud, part)
            be.finalize(part.view(1, -1), 1, Ud, act, st)
        res.append([t.cpu() for t in (part, Ud, act, st, dd)])
        assert not torch.equal(dd.cpu()[1:], torch.from_numpy(d)[1:])
    for u, v in zip(*res):
        assert torch.equal(u, v)


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("G", [4, 8])
def test_k4_combines_g_shard_rows_like_one(oracle, mode, G):
    """G shards through K3 and ONE split K4 over the G rows == the single-shard launch: the K4 combine of C over several rows."""
    K = 10000 if G == 4 else 10240                                            # shards stay multiples of 4
    sc, p, d = _full(panda_setup, K, 30, mode=mode, lam=0.5, filter_u=True, update_lambda=True, eta_u_bound=50.0, eta_l_bound=5.0)
    nu, T = sc.nu, p.T
    P = 2 + T * nu + nu * (nu + 1) // 2
    rng = np.random.default_rng(11)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    a, n = oracle.sample(sc.model, afo.dist_params(p, nu, d), 5, 0, U)
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
    # the rows against the reference.  A shard of 1 250 or 1 280 samples puts its weight on a handful of them, so the float32
    # rounding of S (about 150 here, lambda = 0.5) moves W and C by up to 2e-5 relative (1.9e-5 measured on an H100 at G = 8,
    # SIMPLE); the 1e-5 gate of C is test_k3_covariance_row_and_k4_update_match_the_reference at K >= 10 000
    for g in range(G):
        sl = slice(g * pg.K, (g + 1) * pg.K)
        ref = afo.reduce(sc.model, pg, np.ascontiguousarray(cost[:, sl].cpu().numpy()), np.ascontiguousarray(x[:, :, sl].cpu().numpy()), U, d)
        assert np.abs(parts[g, 2:].cpu().numpy() - ref[2:]).max() <= 5e-5 * max(1.0, np.abs(ref[2:]).max())
    torch.testing.assert_close(stG, st1, rtol=2e-6, atol=0)
    torch.testing.assert_close(UG, U1, atol=2e-6, rtol=0)
    o1, oG = d1.cpu().numpy(), dG.cpu().numpy()
    n2 = nu * nu
    assert _rel(oG[1:1 + 2 * n2], o1[1:1 + 2 * n2]) <= 2e-6                 # Sigma and L
    assert _rel(oG[1 + 2 * n2:], o1[1 + 2 * n2:]) <= 2e-6 * np.linalg.cond(afo.unpack(o1, nu)[1].astype(np.float64))
    assert oG[0] == o1[0]
    U_ref, _, _, d_ref = afo.finalize(sc.model, p, parts.cpu().numpy(), U, d)
    _check_dist(oG, d_ref, nu)


def _planners(kind, graph=True, K=1000):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective, PushObjective
    if kind == "panda":
        flags = dict(update_cov=True, update_lambda=True, cov_type="full", noise_sigma=corr_sigma(7).tolist())
        mk, obj = (lambda d: panda_cfg(K=K, T=30, device=d, eta_u_bound=40.0, eta_l_bound=4.0, **flags)), PandaReachObjective
    else:
        flags = dict(update_cov=True, update_lambda=True, cov_type="full", noise_sigma=[[2.0, 1.5], [1.5, 8.0]])
        mk, obj = (lambda d: boxer_cfg(K=512, T=12, device=d, eta_u_bound=40.0, eta_l_bound=4.0, **flags)), (lambda: PushObjective(robot="boxer", link="ee_link"))
    gpu = MPPIisaacPlanner(mk(DEV), obj(), use_cuda_graph=graph)
    cpu = MPPIisaacPlanner(mk("cpu"), obj(), backend=afo.AdaptiveFullOracleBackend(nthreads=8))
    return gpu, cpu


@pytest.mark.parametrize("kind,plans", [("panda", 20), ("boxer", 20)])
def test_planner_tracks_the_reference(kind, plans):
    gpu, cpu = _planners(kind)
    q = Q0 if kind == "panda" else [0.0, 2.5, 0.0]
    qd = [0.0] * len(q)
    nu = gpu.mppi.nu
    tol, cov_rtol = (2e-4, 2e-4) if kind == "panda" else (5e-4, 5e-4)
    d0 = gpu.mppi.dist.cpu().clone()
    worst = [0.0, 0.0, 0.0]
    for it in range(plans):
        if kind == "boxer":
            # contact scenes: rollouts differ by float32 rounding that the penalty contacts amplify; the reference therefore plans
            # from the device's U and dist
            cpu.mppi.U.copy_(gpu.mppi.U.cpu())
            cpu.mppi.dist.copy_(gpu.mppi.dist.cpu())
        ag, ac = gpu.compute_action(q, qd), cpu.compute_action(q, qd)
        S_g, S_c = gpu.mppi.cov_action.cpu().numpy(), cpu.mppi.cov_action.numpy()
        assert S_g.shape == (nu, nu)
        worst = [max(worst[0], float((ag.cpu() - ac).abs().max())), max(worst[1], float(np.abs(gpu.mppi.U.cpu().numpy() - cpu.mppi.U.numpy()).max())),
                 max(worst[2], _rel(S_g, S_c))]
        assert float((ag.cpu() - ac).abs().max()) <= tol, f"plan {it}"
        np.testing.assert_allclose(gpu.mppi.U.cpu().numpy(), cpu.mppi.U.numpy(), rtol=0, atol=tol, err_msg=f"plan {it}")
        np.testing.assert_allclose(float(gpu.mppi.current_lambda), float(cpu.mppi.current_lambda), rtol=1e-5, err_msg=f"plan {it}")
        assert _rel(S_g, S_c) <= cov_rtol, f"plan {it}"
    print(f"{kind}: worst action {worst[0]:.2e}, U {worst[1]:.2e}, Sigma {worst[2]:.2e} relative")
    assert gpu.mppi._graph is not None
    assert not torch.equal(gpu.mppi.dist.cpu(), d0)


@pytest.mark.parametrize("kind", ["panda", "boxer"])
def test_captured_graph_and_eager_plans_are_bit_identical(kind):
    """The graph reads the live Sigma, L and Sigma^-1: replaying it (never re-captured) gives the eager path's U and dist bit for bit."""
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


def test_backend_checks_the_buffer_and_row_lengths():
    sc, p, d = _full(panda_setup, 64, 12)
    nu, T = sc.nu, p.T
    be = gpu_backend(sc, p)
    with pytest.raises(RuntimeError, match="cov_full"):
        be.set_distribution(torch.zeros(1 + nu, device=DEV))
    be.set_distribution(dev(d))
    cost, x, U = torch.zeros((T, p.K), device=DEV), torch.zeros((T, nu, p.K), device=DEV), torch.zeros((T, nu), device=DEV)
    with pytest.raises(RuntimeError, match="cov_full"):
        be.reduce(cost, x, U, torch.zeros(2 + 2 * T * nu, device=DEV))
    assert be.partial_row_floats() == 2 + T * nu + nu * (nu + 1) // 2


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_peer_and_nccl_exchanges_agree_on_dist():
    """2 ranks, full covariance: the peer-memory exchange of the [beta, eta, W, C] row and the NCCL all-gather give the same action and
    the same dist bit for bit, and the ranks agree on dist."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    res = {}
    for exch in ("peer", "nccl"):
        env = dict(os.environ, MPPIB_EXCHANGE=exch, MPPIB_PEER_TIMEOUT_S="10")
        out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                              "--master-port", "29543", os.path.join(here, "adaptive_full_dist_worker.py")],
                             capture_output=True, text=True, timeout=300, env=env, cwd=os.path.dirname(here))
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
        lines = [ln.split() for ln in out.stdout.splitlines() if ln.startswith("RESULT ")]
        assert len(lines) == 2 and all(ln[1] == exch for ln in lines), out.stdout[-2000:]
        assert lines[0][3:] == lines[1][3:], "the ranks disagree on the action or on dist"
        res[exch] = lines[0][3:]
    assert res["peer"] == res["nccl"]
