"""Adaptive MPPI with a covariance over the whole horizon (update_cov with cov_type: horizon) on the CPU: the rule of DESIGN.md section 2
restated in float64 torch against the reference of ``adaptive_horizon_oracle``, its agreement with the full rule, the shift at T = 1,
shard invariance of the covariance row, and the configuration errors."""
import copy

import numpy as np
import pytest
import torch

import adaptive_full_oracle as afo
import adaptive_horizon_oracle as aho
from mppi_isaac_b200.model.blob import MODE_SIMPLE
from oracle import oracle as orc
from scenes import panda_setup

NU = 7
_A = np.random.default_rng(3).normal(0, 0.15, (NU, NU))
SIG0 = (_A @ _A.T + 0.05 * np.eye(NU)).round(6)
SIG0 = 0.5 * (SIG0 + SIG0.T)


def _setup(mode, K=256, T=6, **kw):
    kw.setdefault("u_min", [-1e6])
    kw.setdefault("u_max", [1e6])
    kw.setdefault("sample_null_action", False)
    sc, p, _ = panda_setup(K=K, T=T, mode=mode, noise_sigma=SIG0.tolist(), update_cov=True, cov_type="horizon", **kw)
    return sc.model, p


def _corr_dist(lam, T):
    t = np.arange(T)
    return aho.make_dist(lam, np.kron(np.exp(-np.abs(t[:, None] - t[None, :]) / 2.0), SIG0))


def _cost(a, target):
    return ((a - target[None, :, None]) ** 2).sum(1)


def _plan(m, p, U, dist, plan, target, seed=7):
    """One reference plan from (U, dist): shift, K1, K3 row with C, K4; returns (U_shifted, U_new, stats, dist, x, row, z)."""
    nu = m.nu
    U = orc.shift(m, p, U)
    z = aho.white(m, p, seed, plan, 0, p.K)
    a, n = aho.colour(p, nu, U, z, dist, 0, p.K)
    x = n if p.mode == MODE_SIMPLE else a
    row = aho.reduce(m, p, _cost(a, target), x, U, dist)
    U2, _, stats, d2 = aho.finalize(m, p, row[None], U, dist)
    return U, U2, stats, d2, x, row, z


def _restated(p, nu, U, dist, z, target):
    """float64 torch restatement of one plan tail from the shifted U: colour, S and weights, W and C, U update, V, Sigma_H update,
    shift, Cholesky factor and inverse (no Savitzky-Golay, no bounds)."""
    T, K = p.T, p.K
    n = T * nu
    lam, Sig, _, _ = (torch.tensor(np.asarray(v, np.float64)) if i else float(v) for i, v in enumerate(aho.unpack(dist, n)))
    U = torch.tensor(np.asarray(U, np.float64)).reshape(n)
    L = torch.linalg.cholesky(Sig)
    noise = L @ torch.tensor(np.asarray(z, np.float64)).reshape(n, K)
    a = U[:, None] + noise
    simple = p.mode == MODE_SIMPLE
    x = noise if simple else a
    cost = torch.tensor(_cost(a.reshape(T, nu, K).numpy(), target))
    S = ((float(p.gamma) ** torch.arange(T, dtype=torch.float64))[:, None] * cost).sum(0)
    if simple:
        S = S + lam * (torch.linalg.inv(Sig) @ U) @ noise
    w = torch.exp(-(S - S.min()) / lam)
    eta = w.sum()
    W = x @ w
    c = torch.zeros_like(U) if simple else U
    C = ((x - c[:, None]) * w) @ (x - c[:, None]).T
    U_new = U + W / eta if simple else (1 - p.step_size_mean) * U + p.step_size_mean * W / eta
    d = U_new - U
    m1 = W / eta - c
    V = C / eta - (torch.outer(m1, d) + torch.outer(d, m1) - torch.outer(d, d))
    Sn = (1 - p.step_size_cov) * Sig + p.step_size_cov * V + p.kappa * torch.eye(n, dtype=torch.float64)
    Sp = torch.zeros_like(Sn)
    Sp[:n - nu, :n - nu] = Sn[nu:, nu:]
    Sp[n - nu:, n - nu:] = torch.tensor(aho.sigma0(p, nu).astype(np.float32).astype(np.float64))
    Lp = torch.linalg.cholesky(Sp)
    return dict(a=a.numpy(), W=W.numpy(), C=C.numpy(), eta=float(eta), U=U_new.numpy(), V=V.numpy(), S=Sp.numpy(), L=Lp.numpy(),
                I=torch.cholesky_inverse(Lp).numpy())


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_restatement_matches_reference(mode):
    m, p = _setup(mode, lambda_=0.5)
    nu, T = m.nu, p.T
    n = T * nu
    target = np.linspace(-0.4, 0.4, nu).astype(np.float32)
    U, dist = np.zeros((T, nu), np.float32), _corr_dist(0.5, T)
    for plan in range(4):
        Us, U2, stats, d2, x, row, z = _plan(m, p, U, dist, plan, target)
        r = _restated(p, nu, Us, dist, z, target)
        np.testing.assert_allclose(np.asarray(x, np.float64).reshape(n, -1) + (0 if mode == "simple" else 0),
                                   (r["a"] - (np.asarray(Us, np.float64).reshape(n, 1) if mode == "simple" else 0)), rtol=0, atol=2e-6)
        np.testing.assert_allclose(stats[1], r["eta"], rtol=1e-4)
        np.testing.assert_allclose(row[2:2 + n], r["W"], rtol=1e-4, atol=1e-6 * np.abs(r["W"]).max())
        np.testing.assert_allclose(afo.tril_unpack(row[2 + n:].astype(np.float64), n), r["C"], rtol=1e-4, atol=1e-6 * np.abs(r["C"]).max())
        np.testing.assert_allclose(U2.reshape(n), r["U"], rtol=1e-4, atol=2e-5)
        _, S32, L32, I32 = aho.unpack(d2, n)
        tol = 1e-4 * np.abs(r["S"]).max()
        np.testing.assert_allclose(S32, r["S"], rtol=1e-4, atol=tol)
        np.testing.assert_allclose(L32, r["L"], rtol=1e-4, atol=1e-4 * np.abs(r["L"]).max())
        np.testing.assert_allclose(I32, r["I"], rtol=1e-3, atol=1e-3 * np.abs(r["I"]).max())
        np.testing.assert_array_equal(S32, S32.T)
        U, dist = U2, d2


def _v_horizon(p, n, row, U_old, U_new):
    rows = np.asarray(row, np.float64)
    eta, W = rows[1], rows[2:2 + n]
    C = afo.tril_unpack(rows[2 + n:], n)
    c = 0.0 if p.mode == MODE_SIMPLE else np.asarray(U_old, np.float64).reshape(n)
    m1 = W / eta - c
    d = np.asarray(U_new, np.float64).reshape(n) - np.asarray(U_old, np.float64).reshape(n)
    return C / eta - (np.outer(m1, d) + np.outer(d, m1) - np.outer(d, d))


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_diagonal_blocks_of_v_sum_to_the_full_rule(mode):
    """sum_t of the diagonal nu x nu blocks of V_H is the full rule's V on the same samples (float64 round-off)."""
    m, p = _setup(mode, lambda_=0.5)
    nu, T, K = m.nu, p.T, p.K
    n = T * nu
    rng = np.random.default_rng(5)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    x = rng.standard_normal((T, nu, K)).astype(np.float32) * 0.3
    if mode != "simple":
        x += U[:, :, None]
    cost = rng.uniform(0, 3, (T, K)).astype(np.float32)
    d_h = aho.initial_dist(0.5, SIG0, T)
    row = aho.reduce(m, p, cost, x, U, d_h)
    U_new = rng.uniform(-0.1, 0.1, (T, nu))
    VH = _v_horizon(p, n, row, U, U_new)
    blocks = sum(VH[t * nu:(t + 1) * nu, t * nu:(t + 1) * nu] for t in range(T))
    # the full rule's V from the same weights: C_full = sum_t of the diagonal blocks of C_H, and the same m1 and d per step
    rows = np.asarray(row, np.float64)
    eta, W = rows[1], rows[2:2 + n].reshape(T, nu)
    C_full = sum(afo.tril_unpack(rows[2 + n:], n)[t * nu:(t + 1) * nu, t * nu:(t + 1) * nu] for t in range(T))
    c = 0.0 if mode == "simple" else U.astype(np.float64)
    m1, dd = W / eta - c, U_new - U
    V_full = C_full / eta - (m1.T @ dd + dd.T @ m1 - dd.T @ dd)
    np.testing.assert_allclose(blocks, V_full, rtol=1e-12, atol=1e-12 * np.abs(V_full).max())
    # and C_full itself is what the full rule's reference computes (S in SIMPLE mode from a block-diagonal Sigma_H^-1)
    d_f = afo.make_dist(0.5, SIG0)
    row_f = afo.reduce(m, p, cost, x, U, d_f)
    np.testing.assert_allclose(afo.tril_unpack(row_f[2 + n:].astype(np.float64), nu), C_full, rtol=1e-5, atol=1e-6 * np.abs(C_full).max())


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_t1_keeps_sigma0_after_every_plan(mode):
    m, p = _setup(mode, T=1, lambda_=0.5)
    nu = m.nu
    target = np.linspace(-0.4, 0.4, nu).astype(np.float32)
    U, dist = np.zeros((1, nu), np.float32), aho.make_dist(0.5, 2.0 * SIG0)
    for plan in range(3):
        _, U, stats, dist, _, _, _ = _plan(m, p, U, dist, plan, target)
        assert stats[1] > 0
        np.testing.assert_array_equal(aho.unpack(dist, nu)[1], SIG0.astype(np.float32))


def test_identity_start_colours_like_the_full_rule():
    """With Sigma_H = I_T (x) Sigma0, L_H z is the full rule's per-step L z."""
    m, p = _setup("simple", K=64, T=5)
    nu, T, K = m.nu, p.T, p.K
    U = np.random.default_rng(2).uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    z = aho.white(m, p, 3, 1, 0, K)
    a_h, n_h = aho.colour(p, nu, U, z, aho.initial_dist(0.5, SIG0, T), 0, K)
    zc = afo.color_library(afo.make_dist(0.5, SIG0), nu, z)
    a_f = U[:, :, None] + zc.astype(np.float64)
    np.testing.assert_allclose(a_h, a_f, rtol=0, atol=2e-6)
    np.testing.assert_allclose(n_h, a_h - U[:, :, None], rtol=0, atol=0)


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("G", [2, 4, 8])
def test_shard_rows_combine_to_the_single_row(mode, G):
    m, p = _setup(mode, K=512, lambda_=0.5)
    nu, T, K = m.nu, p.T, p.K
    n = T * nu
    rng = np.random.default_rng(9)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    dist = _corr_dist(0.5, T)
    z = aho.white(m, p, 4, 0, 0, K)
    a, nz = aho.colour(p, nu, U, z, dist, 0, K)
    x = nz if mode == "simple" else a
    cost = rng.uniform(0, 3, (T, K)).astype(np.float32)
    row1 = aho.reduce(m, p, cost, x, U, dist)
    pg = copy.copy(p)
    pg.K = K // G
    rows = np.stack([aho.reduce(m, pg, np.ascontiguousarray(cost[:, g * pg.K:(g + 1) * pg.K]), np.ascontiguousarray(x[:, :, g * pg.K:(g + 1) * pg.K]),
                                U, dist) for g in range(G)])
    U1, _, st1, d1 = aho.finalize(m, p, row1[None], U, dist)
    UG, _, stG, dG = aho.finalize(m, p, rows, U, dist)
    np.testing.assert_allclose(stG[1], st1[1], rtol=1e-5)
    np.testing.assert_allclose(UG, U1, rtol=0, atol=1e-6)
    np.testing.assert_allclose(dG[1:1 + 2 * n * n], d1[1:1 + 2 * n * n], rtol=0, atol=1e-5 * np.abs(d1[1:1 + n * n]).max())
    assert dG[0] == d1[0]


def test_config_errors():
    with pytest.raises(ValueError, match="T\\*nu"):
        panda_setup(K=64, T=37, noise_sigma=SIG0.tolist(), update_cov=True, cov_type="horizon")          # n = 259
    panda_setup(K=64, T=36, noise_sigma=SIG0.tolist(), update_cov=True, cov_type="horizon")              # n = 252 is accepted
    with pytest.raises(ValueError, match="update_cov"):
        panda_setup(K=64, T=6, noise_sigma=SIG0.tolist(), cov_type="horizon")
    bad = SIG0.copy()
    bad[0, 0] = -1.0
    with pytest.raises(ValueError, match="positive-definite"):
        panda_setup(K=64, T=6, noise_sigma=bad.tolist(), update_cov=True, cov_type="horizon")
    asym = SIG0.copy()
    asym[0, 1] += 0.01
    with pytest.raises(ValueError, match="positive-definite"):
        panda_setup(K=64, T=6, noise_sigma=asym.tolist(), update_cov=True, cov_type="horizon")


def test_cpu_planner_runs_the_horizon_rule():
    """The reference backend drives the planner: cov_action is the (n, n) Sigma_H, started at I_T (x) Sigma0 and adapted."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from scenes import panda_cfg
    cfg = panda_cfg(K=128, T=10, device="cpu", update_cov=True, cov_type="horizon", noise_sigma=SIG0.tolist())
    pl = MPPIisaacPlanner(cfg, PandaReachObjective(), backend=aho.AdaptiveHorizonOracleBackend())
    n = 10 * NU
    np.testing.assert_allclose(pl.mppi.cov_action.numpy(), np.kron(np.eye(10), SIG0), rtol=0, atol=1e-7)
    assert pl.mppi.partial.numel() == 2 + n + n * (n + 1) // 2
    q = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
    for _ in range(2):
        pl.compute_action(q, [0.0] * NU)
    S = pl.mppi.cov_action.numpy()
    assert S.shape == (n, n) and not np.allclose(S, np.kron(np.eye(10), SIG0))
