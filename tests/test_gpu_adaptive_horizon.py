"""-m gpu: adaptive MPPI with a covariance over the whole horizon (update_cov with cov_type: horizon) on the device against the CPU
reference of ``adaptive_horizon_oracle``: the horizon-colour K1 variants, the covariance row C of the SYRK, the Sigma_H update, shift
and factorisation of K4, and whole plans through the planner (graph, eager, fused, split)."""
import copy

import numpy as np
import pytest
import torch

import adaptive_horizon_oracle as aho
from mppi_isaac_b200.model.blob import MODE_SIMPLE, OBS_DOF_STATE, build_scene, make_params
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, load_actor_cfgs
from scenes import panda_cfg, panda_mppi, panda_setup, point_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]


def corr_sigma(nu, scale=0.1, seed=3):
    A = np.random.default_rng(seed).normal(0, 1.0, (nu, nu))
    S = A @ A.T / nu + 0.3 * np.eye(nu)
    S = scale * S / np.mean(np.diag(S))
    return 0.5 * (S + S.T)


def corr_horizon(T, sig0, tau=3.0):
    """A Sigma_H with cross-time correlations: exp(-|t - t'| / tau) (x) Sigma0 (symmetric positive definite)."""
    t = np.arange(T)
    return np.kron(np.exp(-np.abs(t[:, None] - t[None, :]) / tau), sig0)


def gpu_backend(sc, p, dist=None):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(sc.model, p)
    if dist is not None:
        be.set_distribution(dist)
    return be


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def boxer_setup(K=64, T=30, mode="simple", **kw):
    """boxer (nu = 2): only its control dimension matters to K1 / K3 / K4; T = 128 gives n = 256, T = 1 gives n = 2."""
    sc = build_scene(load_actor_cfgs(["boxer", "goal"]))
    kw.setdefault("noise_sigma", (0.1 * np.eye(sc.nu)).tolist())
    p = make_params(panda_mppi(K, T, mode, **kw), IsaacGymConfig(), sc.nu, K, [(OBS_DOF_STATE, 0)])
    return sc, p, None


def _hzn(setup, K, T, mode="simple", lam=0.3, **kw):
    sc, _, _ = setup(K=4, T=T)
    sig = corr_sigma(sc.nu)
    sc, p, _ = setup(K=K, T=T, mode=mode, update_cov=True, cov_type="horizon", noise_sigma=sig.tolist(), **kw)
    return sc, p, sig


def _rel(a, b):
    return np.abs(np.asarray(a, np.float64) - b).max() / max(1.0, np.abs(b).max())


def test_k1_horizon_colour_variants_match_the_reference(oracle):
    sc, p, sig = _hzn(panda_setup, 1000, 30, lam=0.05)
    nu, T, K = sc.nu, p.T, p.K
    n = T * nu
    d = aho.make_dist(0.05, corr_horizon(T, sig))
    be = gpu_backend(sc, p, dev(d))
    U = np.random.default_rng(1).uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    a, nz = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    be.sample(11, 3, 0, K, dev(U), None, a, nz)
    z = aho.white(sc.model, p, 11, 3, 0, K)
    a_ref, n_ref = aho.colour(p, nu, U, z, d, 0, K)
    L = aho.unpack(d, n)[2]
    tol = 2e-6 * max(1.0, 6 * float(np.abs(L).max()) * np.sqrt(n))
    assert np.abs(a.cpu().numpy() - a_ref).max() <= tol
    assert np.abs(nz.cpu().numpy() - n_ref).max() <= tol
    # Halton library: white on the device, coloured by the live L_H on every plan
    from mppi_isaac_b200.planner.mppi import halton_spline_operator, halton_table
    nk = T // 4
    B, tab = halton_spline_operator(T, nk), halton_table(nk * nu, 3)
    Z = torch.zeros((T, nu, K), device=DEV)
    be.noise_library(0, K, dev(tab, torch.int32), dev(B), nk, Z)
    pw = copy.deepcopy(p)                                                     # identity colour; the null row stays zero
    for j in range(nu):
        for i in range(nu):
            pw.sigma_chol[j * nu + i] = 1.0 if i == j else 0.0
    Z_ref = oracle.noise_library(sc.model, pw, tab, B, nk)
    assert np.abs(Z.cpu().numpy() - Z_ref).max() <= 1e-4
    be.sample_library(0, K, dev(U), None, Z, a, nz)
    a_ref, n_ref = aho.colour(p, nu, U, Z.cpu().numpy(), d, 0, K)
    scale = max(1.0, np.abs(Z.cpu().numpy()).max() * float(np.abs(L).max()) * np.sqrt(n))
    assert np.abs(a.cpu().numpy() - a_ref).max() <= 2e-6 * scale
    assert np.abs(nz.cpu().numpy() - n_ref).max() <= 2e-6 * scale


def test_k1_is_shard_invariant():
    """A sample's horizon noise depends only on its global index: two shards of 500 give the columns of one launch of 1 000 bit for bit."""
    sc, p, sig = _hzn(panda_setup, 1000, 30)
    nu, T = sc.nu, p.T
    d = dev(aho.make_dist(0.3, corr_horizon(T, sig)))
    U = dev(np.random.default_rng(2).uniform(-0.1, 0.1, (T, nu)).astype(np.float32))
    be = gpu_backend(sc, p, d)
    a1, n1 = torch.zeros((T, nu, 1000), device=DEV), torch.zeros((T, nu, 1000), device=DEV)
    be.sample(5, 2, 0, 1000, U, None, a1, n1)
    ph = copy.copy(p)
    ph.K = 500
    beh = gpu_backend(sc, ph, d)
    for g in range(2):
        a, nz = torch.zeros((T, nu, 500), device=DEV), torch.zeros((T, nu, 500), device=DEV)
        beh.sample(5, 2, 500 * g, 1000, U, None, a, nz)
        assert torch.equal(a, a1[:, :, 500 * g:500 * (g + 1)]) and torch.equal(nz, n1[:, :, 500 * g:500 * (g + 1)])


def _check_dist(dd, d_ref, n, rtol=1e-5):
    """Sigma_H against the reference to `rtol` of its largest entry; L L^T = Sigma and Sigma^-1 Sigma = I on the device's own values, to
    tolerances that grow with n and the condition number."""
    _, S, L, I = aho.unpack(dd, n)
    _, Sr, _, _ = aho.unpack(d_ref, n)
    assert _rel(S, Sr) <= rtol
    np.testing.assert_array_equal(S, S.T)
    np.testing.assert_array_equal(I, I.T)
    np.testing.assert_array_equal(L, np.tril(L))
    S64 = S.astype(np.float64)
    eps = np.finfo(np.float32).eps
    assert np.abs(L.astype(np.float64) @ L.T.astype(np.float64) - S64).max() <= 4 * n * eps * np.abs(S64).max()
    cond = np.linalg.cond(S64)
    assert np.abs(I.astype(np.float64) @ S64 - np.eye(n)).max() <= 4 * n * eps * cond
    np.testing.assert_allclose(dd[0], d_ref[0], rtol=1e-6)


SHAPES = [("boxer", 1), ("panda", 30), ("boxer", 128)]                       # n = 2, 210, 256


@pytest.mark.parametrize("which,T", SHAPES)
@pytest.mark.parametrize("K", [4, 10000, 65536])
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_c_row_and_k4_update_match_the_reference(oracle, which, T, K, mode):
    setup = {"panda": panda_setup, "boxer": boxer_setup}[which]
    sc, p, sig = _hzn(setup, K, T, mode=mode, update_lambda=True)
    nu = sc.nu
    n = T * nu
    d = aho.make_dist(0.3, corr_horizon(T, sig))
    dd = dev(d)
    be = gpu_backend(sc, p, dd)
    rng = np.random.default_rng(7)
    Ud = dev(rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32))
    be.shift(Ud)                                                              # computes g = lambda Sigma_H^-1 U for SIMPLE mode
    U = Ud.cpu().numpy()
    L = aho.unpack(d, n)[2].astype(np.float64)
    x = (L @ rng.standard_normal((n, K))).reshape(T, nu, K).astype(np.float32)
    if p.mode != MODE_SIMPLE:
        x += U[:, :, None]
    cost = rng.uniform(0, 10, (T, K)).astype(np.float32)
    if K > 4:
        cost[:, K // 3] = np.nan
    P = 2 + n + n * (n + 1) // 2
    partial = torch.zeros(P, device=DEV)
    for _ in range(2):
        be.reduce(dev(cost), dev(x), Ud, partial)
    ref = aho.reduce(sc.model, p, cost, x, U, d)
    pg = partial.cpu().numpy()
    assert abs(pg[0] - ref[0]) <= 1e-5 * max(1, abs(ref[0]))
    np.testing.assert_allclose(pg[1], ref[1], rtol=5e-5)
    # C sums a chunk of K / ksplit samples in sequence per entry (about 500 at K = 65 536 on 132 SMs with 10 tiles); its float32
    # rounding reaches 1.04e-5 relative there (n = 256, MEAN mode, H100), so the gate widens with the chunk length
    ctol = 1e-5 * max(1.0, K / 32768)
    for sl, tol in ((slice(2, 2 + n), 1e-5), (slice(2 + n, None), ctol)):
        assert np.abs(pg[sl] - ref[sl]).max() <= tol * max(1.0, np.abs(ref[sl]).max())
    # K4 on the same row: U and Sigma_H, L_H, Sigma_H^-1
    act, st = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(partial.view(1, -1), 1, Ud, act, st)
    U_ref, _, _, d_ref = aho.finalize(sc.model, p, pg[None], U, d)
    np.testing.assert_allclose(Ud.cpu().numpy(), U_ref, rtol=0, atol=1e-5 * max(1.0, np.abs(U_ref).max()))
    assert not np.array_equal(d_ref[1:], d[1:])
    _check_dist(dd.cpu().numpy(), d_ref, n)


@pytest.mark.parametrize("fused", [True, False])
def test_k4_indefinite_update_leaves_sigma_l_and_inverse_unchanged(fused):
    sc, p, sig = _hzn(panda_setup, 64, 12, update_lambda=True, eta_u_bound=10.0, eta_l_bound=5.0)
    nu, T = sc.nu, p.T
    n = T * nu
    P = 2 + n + n * (n + 1) // 2
    d = aho.initial_dist(0.3, sig, T)
    dd = dev(d)
    be = gpu_backend(sc, p, dd)
    Ud, act, st = torch.zeros((T, nu), device=DEV), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    if fused:
        # one valid sample with x = 0: C = 0 and V = 0, and a previous Sigma_H = -I makes the shifted update negative definite
        bad = d.copy()
        bad[1:1 + n * n] = (-np.eye(n)).ravel()
        dd.copy_(dev(bad))
        cost = torch.full((T, p.K), float("nan"), device=DEV)
        cost[:, 5] = 1.0
        x = torch.zeros((T, nu, p.K), device=DEV)
        be.shift(Ud)
        be.reduce_finalize(cost, x, Ud, torch.zeros(P, device=DEV), act, st)
        out = dd.cpu().numpy()
        np.testing.assert_array_equal(out[1:], bad[1:])
    else:
        row = np.zeros(P, np.float32)
        row[1] = 2.0                                                         # eta < eta_l_bound: lambda *= 1.1
        row[2 + n:] = aho.tril_pack(-100.0 * np.eye(n))
        be.finalize(dev(row).view(1, -1), 1, Ud, act, st)
        out = dd.cpu().numpy()
        np.testing.assert_array_equal(out[1:], d[1:])
    assert out[0] == np.float32(d[0]) * (np.float32(1) + np.float32(0.1))


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_fused_tail_equals_split_reduce_and_finalize(mode):
    sc, p, sig = _hzn(panda_setup, 10000, 30, mode=mode, lam=0.5, filter_u=True, update_lambda=True, eta_u_bound=50.0, eta_l_bound=5.0)
    nu, T, K = sc.nu, p.T, p.K
    n = T * nu
    d = aho.make_dist(0.5, corr_horizon(T, sig))
    rng = np.random.default_rng(4)
    U0 = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    cost = dev(rng.uniform(0, 10, (T, K)).astype(np.float32))
    res = []
    for fused in (True, False):
        dd = dev(d)
        be = gpu_backend(sc, p, dd)
        part, Ud, act, st = torch.zeros(2 + n + n * (n + 1) // 2, device=DEV), dev(U0), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        a, nz = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
        be.shift(Ud)
        be.sample(3, 0, 0, K, Ud, None, a, nz)
        x = nz if p.mode == MODE_SIMPLE else a
        if fused:
            be.reduce_finalize(cost, x, Ud, part, act, st)
        else:
            be.reduce(cost, x, Ud, part)
            be.finalize(part.view(1, -1), 1, Ud, act, st)
        res.append([t.cpu() for t in (part, Ud, act, st, dd)])
        assert not torch.equal(dd.cpu()[1:], torch.from_numpy(d)[1:])
    for u, v in zip(*res):
        assert torch.equal(u, v)


def _planners(kind, graph=True, K=1000):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    if kind == "panda":
        flags = dict(update_cov=True, update_lambda=True, cov_type="horizon", noise_sigma=corr_sigma(7).tolist())
        mk, obj = (lambda d: panda_cfg(K=K, T=30, device=d, eta_u_bound=40.0, eta_l_bound=4.0, **flags)), PandaReachObjective
    else:
        from mppi_isaac_b200.objectives import PointReachObjective
        flags = dict(update_cov=True, update_lambda=True, cov_type="horizon")
        mk, obj = (lambda d: point_cfg(K=512, T=12, device=d, eta_u_bound=40.0, eta_l_bound=4.0, **flags)), PointReachObjective
    gpu = MPPIisaacPlanner(mk(DEV), obj(), use_cuda_graph=graph)
    cpu = MPPIisaacPlanner(mk("cpu"), obj(), backend=aho.AdaptiveHorizonOracleBackend(nthreads=8))
    return gpu, cpu


@pytest.mark.parametrize("kind,plans", [("panda", 10), ("point", 10)])
def test_planner_tracks_the_reference(kind, plans):
    """Lock-step: the reference plans from the device's U and dist every plan, so float32 rounding cannot build up."""
    gpu, cpu = _planners(kind)
    q = Q0 if kind == "panda" else [0.1, 0.0, 0.0]
    qd = [0.0] * len(q)
    n = gpu.mppi.T * gpu.mppi.nu
    d0 = gpu.mppi.dist.cpu().clone()
    worst = [0.0, 0.0]
    for it in range(plans):
        cpu.mppi.U.copy_(gpu.mppi.U.cpu())
        cpu.mppi.dist.copy_(gpu.mppi.dist.cpu())
        ag, ac = gpu.compute_action(q, qd), cpu.compute_action(q, qd)
        S_g, S_c = gpu.mppi.cov_action.cpu().numpy(), cpu.mppi.cov_action.numpy()
        assert S_g.shape == (n, n)
        worst = [max(worst[0], float((ag.cpu() - ac).abs().max())), max(worst[1], _rel(S_g, S_c))]
        assert float((ag.cpu() - ac).abs().max()) <= 5e-4, f"plan {it}"
        np.testing.assert_allclose(float(gpu.mppi.current_lambda), float(cpu.mppi.current_lambda), rtol=1e-5, err_msg=f"plan {it}")
        assert _rel(S_g, S_c) <= 1e-4, f"plan {it}"
    print(f"{kind}: worst action {worst[0]:.2e}, Sigma_H {worst[1]:.2e} relative")
    assert gpu.mppi._graph is not None
    assert not torch.equal(gpu.mppi.dist.cpu(), d0)


def test_captured_graph_and_eager_plans_are_bit_identical():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    flags = dict(update_cov=True, update_lambda=True, cov_type="horizon", noise_sigma=corr_sigma(7).tolist(), eta_u_bound=40.0, eta_l_bound=4.0)
    g = MPPIisaacPlanner(panda_cfg(K=2000, T=30, device=DEV, **flags), PandaReachObjective(), use_cuda_graph=True)
    e = MPPIisaacPlanner(panda_cfg(K=2000, T=30, device=DEV, **flags), PandaReachObjective(), use_cuda_graph=False)
    d0 = g.mppi.dist.clone()
    graph = None
    for it in range(10):
        g.compute_action(Q0, [0.0] * 7)
        e.compute_action(Q0, [0.0] * 7)
        graph = graph or g.mppi._graph
        assert g.mppi._graph is graph, "the plan graph was re-captured"
        assert torch.equal(g.mppi.dist, e.mppi.dist) and torch.equal(g.mppi.U, e.mppi.U), f"plan {it}"
    assert e.mppi._graph is None and not torch.equal(g.mppi.dist, d0)


def test_backend_checks_the_buffer_and_row_lengths():
    sc, p, sig = _hzn(panda_setup, 64, 12)
    nu, T = sc.nu, p.T
    n = T * nu
    be = gpu_backend(sc, p)
    with pytest.raises(RuntimeError, match="cov_horizon"):
        be.set_distribution(torch.zeros(1 + 3 * nu * nu, device=DEV))
    be.set_distribution(dev(aho.initial_dist(0.3, sig, T)))
    cost, x, U = torch.zeros((T, p.K), device=DEV), torch.zeros((T, nu, p.K), device=DEV), torch.zeros((T, nu), device=DEV)
    with pytest.raises(RuntimeError, match="cov_horizon"):
        be.reduce(cost, x, U, torch.zeros(2 + n + nu * (nu + 1) // 2, device=DEV))
    assert be.partial_row_floats() == 2 + n + n * (n + 1) // 2


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_peer_and_nccl_exchanges_agree_on_dist():
    """2 ranks, horizon covariance: the peer-memory exchange of the [beta, eta, W, C] row and the NCCL all-gather give the same action
    and the same dist bit for bit, and the ranks agree on dist."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    res = {}
    for exch in ("peer", "nccl"):
        env = dict(os.environ, MPPIB_EXCHANGE=exch, MPPIB_PEER_TIMEOUT_S="10")
        out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                              "--master-port", "29547", os.path.join(here, "adaptive_horizon_dist_worker.py")],
                             capture_output=True, text=True, timeout=300, env=env, cwd=os.path.dirname(here))
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
        lines = [ln.split() for ln in out.stdout.splitlines() if ln.startswith("RESULT ")]
        assert len(lines) == 2 and all(ln[1] == exch for ln in lines), out.stdout[-2000:]
        assert lines[0][3:] == lines[1][3:], "the ranks disagree on the action or on dist"
        res[exch] = lines[0][3:]
    assert res["peer"] == res["nccl"]
