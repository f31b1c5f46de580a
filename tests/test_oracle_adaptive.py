"""Adaptive MPPI (update_cov / update_lambda) on the CPU: the rules of DESIGN.md section 2 restated in float64 against the
reference of ``adaptive_oracle``, known answers, shard invariance of the second-moment row, and the planner plumbing."""
import copy
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as tdist
import torch.multiprocessing as mp

import adaptive_oracle as ada
from mppi_isaac_b200.model.blob import MODE_SIMPLE
from oracle import oracle as orc
from scenes import panda_cfg, point_setup

HERE = os.path.dirname(os.path.abspath(__file__))
Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
FLAGS = {"cov": dict(update_cov=True), "lambda": dict(update_lambda=True), "both": dict(update_cov=True, update_lambda=True)}


def _setup(mode, K=256, T=12, **kw):
    kw.setdefault("u_min", [-1e6])
    kw.setdefault("u_max", [1e6])
    kw.setdefault("sample_null_action", False)
    sc, p, _ = point_setup(K=K, T=T, mode=mode, **kw)
    return sc.model, p


def _cost(a, target):
    """(T, nu, K) actions -> (T, K) cost: squared distance of every step's action to a target, which makes the weights non-trivial."""
    return ((a - target[None, :, None]) ** 2).sum(1)


def _dist0(p, nu):
    return np.array([p.lambda_] + [p.sigma_chol[j * nu + j] ** 2 for j in range(nu)], np.float32)


class Restated:
    """float64 restatement of the adaptive plan tail, independent of oracle.cpp: K3 (S, weights, W, M2) + K4 (U, cov, lambda)."""

    def __init__(self, p, nu):
        self.p, self.nu = p, nu
        self.U = torch.zeros((p.T, nu), dtype=torch.float64)
        self.lam = torch.tensor(float(p.lambda_), dtype=torch.float64)
        self.cov = torch.tensor([p.sigma_chol[j * nu + j] ** 2 for j in range(nu)], dtype=torch.float64)
        self.chol = torch.tensor(np.array(p.sigma_chol[:nu * nu]).reshape(nu, nu), dtype=torch.float64)
        self.sinv = torch.tensor(np.array(p.sigma_inv[:nu * nu]).reshape(nu, nu), dtype=torch.float64)

    def plan(self, z, target):
        p, T, nu = self.p, self.p.T, self.nu
        self.U = torch.cat([self.U[1:], torch.tensor(np.array(p.u_init[:nu]), dtype=torch.float64)[None]])
        if p.update_cov:
            noise = self.cov.sqrt()[None, :, None] * z
            sinv = torch.diag(1.0 / self.cov)
        else:
            noise = torch.einsum("ji,tik->tjk", self.chol, z)
            sinv = self.sinv
        a = self.U[:, :, None] + noise
        simple = p.mode == MODE_SIMPLE
        x = noise if simple else a
        S = (float(p.gamma) ** torch.arange(T, dtype=torch.float64))[:, None].mul(_cost(a, target)).sum(0)
        if simple:
            S = S + self.lam * torch.einsum("tj,ji,tik->k", self.U, sinv, noise)
        w = torch.exp(-(S - S.min()) / self.lam)
        eta = w.sum()
        W = (w * x).sum(-1)
        c = torch.zeros_like(self.U) if simple else self.U
        M2 = (w * (x - c[:, :, None]) ** 2).sum(-1)
        U_new = self.U + W / eta if simple else (1 - p.step_size_mean) * self.U + p.step_size_mean * W / eta
        if p.update_cov:
            d = U_new - self.U
            m1 = W / eta - c
            var = torch.clamp(M2 / eta - 2 * d * m1 + d * d, min=0.0)
            self.cov = (1 - p.step_size_cov) * self.cov + p.step_size_cov * var.mean(0) + p.kappa
        if p.update_lambda:
            if eta > p.eta_u_bound:
                self.lam = self.lam * (1 - p.lambda_mult)
            elif eta < p.eta_l_bound:
                self.lam = self.lam * (1 + p.lambda_mult)
            self.lam = torch.clamp(self.lam, 1e-3 * p.lambda_, 1e3 * p.lambda_)
        self.U = U_new
        return float(eta)


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("flags", list(FLAGS))
def test_restatement_matches_reference_over_20_plans(mode, flags):
    m, p = _setup(mode, lambda_=0.5, eta_u_bound=40.0, eta_l_bound=8.0, noise_sigma=np.diag([0.3, 0.5, 0.2]).tolist(), **FLAGS[flags])
    nu, T, K = m.nu, p.T, p.K
    target = np.array([0.4, -0.3, 0.2], np.float32)
    ref = Restated(p, nu)
    U, dist = np.zeros((T, nu), np.float32), _dist0(p, nu)
    white = ada.dist_params(p, nu, dist, white=True)
    white.lambda_ = p.lambda_
    lam_moves = 0
    for plan in range(20):
        # the restatement starts every plan from the reference's state, so float32 rounding cannot accumulate over the 20 plans
        ref.U = torch.tensor(U, dtype=torch.float64)
        ref.lam = torch.tensor(float(dist[0]), dtype=torch.float64)
        ref.cov = torch.tensor(dist[1:], dtype=torch.float64)
        U = orc.shift(m, p, U)
        dp = ada.dist_params(p, nu, dist)
        a, n = orc.sample(m, dp, 7, plan, U)
        x = n if p.mode == MODE_SIMPLE else a
        row = ada.reduce(m, p, _cost(a, target), x, U, dist)
        lam_before = dist[0]
        U, _, stats, dist = ada.finalize(m, p, row[None], U, dist)
        lam_moves += int(dist[0] != lam_before)
        # the restatement draws the same standard normals: the white draw of the same Philox counters
        zw, _ = orc.sample(m, white, 7, plan, np.zeros((T, nu), np.float32))
        if not p.update_cov:
            zw = np.linalg.solve(np.array(p.sigma_chol[:nu * nu]).reshape(nu, nu), zw.transpose(1, 0, 2).reshape(nu, -1)).reshape(nu, T, K).transpose(1, 0, 2)
        eta = ref.plan(torch.tensor(np.asarray(zw, np.float64)), torch.tensor(target, dtype=torch.float64))
        np.testing.assert_allclose(stats[1], eta, rtol=1e-3)
        np.testing.assert_allclose(U, ref.U.numpy(), rtol=1e-4, atol=2e-5)
        np.testing.assert_allclose(dist[0], float(ref.lam), rtol=1e-5)
        np.testing.assert_allclose(dist[1:], ref.cov.numpy(), rtol=1e-4, atol=1e-6)
    if p.update_lambda:
        assert lam_moves > 0
    if not p.update_cov:
        np.testing.assert_array_equal(dist[1:], _dist0(p, nu)[1:])


def test_uniform_costs_lower_lambda_by_0_9_until_the_clamp():
    m, p = _setup("halton-spline", K=64, update_lambda=True, eta_u_bound=10.0, eta_l_bound=5.0, lambda_=0.2)
    nu, T, K = m.nu, p.T, p.K
    U, dist = np.zeros((T, nu), np.float32), _dist0(p, nu)
    a, _ = orc.sample(m, p, 1, 0, U)
    lam, floor = np.float32(p.lambda_), np.float32(1e-3) * np.float32(p.lambda_)
    for _ in range(80):
        row = ada.reduce(m, p, np.ones((T, K), np.float32), a, U, dist)
        assert row[1] == K                                                   # MEAN mode adds no control cost: every weight is 1
        U, _, _, dist = ada.finalize(m, p, row[None], U, dist)
        lam = max(lam * (np.float32(1) - np.float32(0.1)), floor)
        assert dist[0] == lam
    assert dist[0] == floor


def test_one_dominant_sample_raises_lambda_by_1_1():
    m, p = _setup("halton-spline", K=64, update_lambda=True, eta_u_bound=10.0, eta_l_bound=5.0, lambda_=0.01)
    nu, T, K = m.nu, p.T, p.K
    U, dist = np.zeros((T, nu), np.float32), _dist0(p, nu)
    a, _ = orc.sample(m, p, 1, 0, U)
    cost = np.full((T, K), 10.0, np.float32)
    cost[:, 5] = 0.0
    lam = np.float32(p.lambda_)
    for _ in range(10):
        row = ada.reduce(m, p, cost, a, U, dist)
        assert abs(row[1] - 1.0) < 1e-6
        U, _, _, dist = ada.finalize(m, p, row[None], U, dist)
        lam = lam * (np.float32(1) + np.float32(0.1))
        assert dist[0] == lam


def test_simple_mode_one_dominant_sample_shrinks_cov_to_0_3_cov_plus_kappa():
    m, p = _setup("simple", K=64, update_cov=True, lambda_=0.01, noise_sigma=np.diag([0.3, 0.5, 0.2]).tolist())
    nu, T, K = m.nu, p.T, p.K
    U, dist = np.zeros((T, nu), np.float32), _dist0(p, nu)
    cov = dist[1:].astype(np.float64)
    for plan in range(5):
        a, n = orc.sample(m, ada.dist_params(p, nu, dist), 3, plan, U)
        cost = np.full((T, K), 50.0, np.float32)
        cost[:, 11] = 0.0
        U, _, _, dist = ada.finalize(m, p, ada.reduce(m, p, cost, n, U, dist)[None], U, dist)
        cov = 0.3 * cov + 0.005
        np.testing.assert_allclose(dist[1:], cov, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("G", [2, 4, 8])
def test_second_moment_row_is_shard_invariant(mode, G):
    m, p = _setup(mode, K=256, update_cov=True, update_lambda=True, lambda_=0.3)
    nu, T, K = m.nu, p.T, p.K
    rng = np.random.default_rng(5)
    U = rng.normal(0, 0.2, (T, nu)).astype(np.float32)
    dist = np.array([0.25, 0.4, 0.3, 0.6], np.float32)
    a, n = orc.sample(m, ada.dist_params(p, nu, dist), 9, 4, U)
    x = n if p.mode == MODE_SIMPLE else a
    cost = rng.uniform(0, 2, (T, K)).astype(np.float32)
    one = ada.finalize(m, p, ada.reduce(m, p, cost, x, U, dist)[None], U, dist)
    Ks = K // G
    ps = copy.deepcopy(p)
    ps.K = Ks
    rows = np.stack([ada.reduce(m, ps, np.ascontiguousarray(cost[:, g * Ks:(g + 1) * Ks]), np.ascontiguousarray(x[:, :, g * Ks:(g + 1) * Ks]), U, dist)
                     for g in range(G)])
    many = ada.finalize(m, p, rows, U, dist)
    np.testing.assert_allclose(many[0], one[0], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(many[3], one[3], rtol=1e-5, atol=1e-7)


def _planner(backend_cls, **kw):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    return MPPIisaacPlanner(panda_cfg(K=64, T=12, **kw), PandaReachObjective(), backend=backend_cls())


def test_flags_off_matches_the_fixed_distribution_path_bit_for_bit():
    from oracle.backend import OracleBackend
    a, b = _planner(OracleBackend), _planner(ada.AdaptiveOracleBackend)
    assert b.mppi.dist is None
    for _ in range(3):
        np.testing.assert_array_equal(a.compute_action(Q0, [0] * 7).numpy(), b.compute_action(Q0, [0] * 7).numpy())
    np.testing.assert_array_equal(a.mppi.U.numpy(), b.mppi.U.numpy())
    # a registered distribution with both flags off leaves the row and U unchanged
    m, p = _setup("simple")
    nu, T, K = m.nu, p.T, p.K
    U = np.full((T, nu), 0.1, np.float32)
    a_, n_ = orc.sample(m, p, 2, 0, U)
    cost = np.ones((T, K), np.float32) + a_.sum(1)
    row0, _ = orc.reduce(m, p, cost, n_, U)
    row1 = ada.reduce(m, p, cost, n_, U, _dist0(p, nu))
    np.testing.assert_array_equal(row0, row1)
    np.testing.assert_array_equal(orc.finalize(m, p, row0[None], U)[0], ada.finalize(m, p, row1[None], U, _dist0(p, nu))[0])


def test_planner_errors_rebuilds_and_resets():
    sig = np.full((7, 7), 0.01) + 0.1 * np.eye(7)
    with pytest.raises(ValueError, match="diagonal"):
        _planner(ada.AdaptiveOracleBackend, update_cov=True, noise_sigma=sig.tolist())
    from oracle.backend import OracleBackend
    with pytest.raises(ValueError, match="set_distribution"):
        _planner(OracleBackend, update_lambda=True)
    _planner(ada.AdaptiveOracleBackend, update_lambda=True, noise_sigma=sig.tolist())     # update_lambda alone takes any Sigma
    pl = _planner(ada.AdaptiveOracleBackend, update_cov=True, update_lambda=True)
    d0 = pl.mppi.dist.clone()
    np.testing.assert_allclose(pl.mppi.cov_action.numpy(), np.diag(np.asarray(pl.cfg.mppi.noise_sigma)), rtol=1e-7)
    assert float(pl.mppi.current_lambda) == np.float32(pl.cfg.mppi.lambda_) and isinstance(pl.mppi.lambda_, float)
    for _ in range(4):
        pl.compute_action(Q0, [0] * 7)
    d4 = pl.mppi.dist.clone()
    assert not torch.equal(d4, d0)
    pl._build_mppi(keep_U=True)                                              # obstacle added / add_to_env: U and dist survive
    assert torch.equal(pl.mppi.dist, d4) and pl.sim.backend.dist is pl.mppi.dist
    sig2 = (0.2 * np.eye(7)).tolist()
    pl.update_mppi_params({"noise_sigma": sig2})                             # rebuilt from the new Sigma
    np.testing.assert_allclose(pl.mppi.cov_action.numpy(), 0.2, rtol=1e-7)
    assert float(pl.mppi.current_lambda) == np.float32(pl.cfg.mppi.lambda_)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    tdist.init_process_group("gloo", rank=rank, world_size=world)
    import adaptive_oracle
    pl = _planner(adaptive_oracle.AdaptiveOracleBackend, update_cov=True, update_lambda=True)
    for _ in range(4):
        pl.compute_action(Q0, [0] * 7)
    np.save(os.path.join(out_dir, f"dist_{rank}.npy"), pl.mppi.dist.numpy())
    np.save(os.path.join(out_dir, f"U_{rank}.npy"), pl.mppi.U.numpy())
    tdist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_gloo_ranks_end_with_identical_dist(tmp_path):
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    d0, d1 = np.load(tmp_path / "dist_0.npy"), np.load(tmp_path / "dist_1.npy")
    np.testing.assert_array_equal(d0, d1)
    np.testing.assert_array_equal(np.load(tmp_path / "U_0.npy"), np.load(tmp_path / "U_1.npy"))
    single = _planner(ada.AdaptiveOracleBackend, update_cov=True, update_lambda=True)
    for _ in range(4):
        single.compute_action(Q0, [0] * 7)
    np.testing.assert_allclose(d0, single.mppi.dist.numpy(), rtol=1e-4)


def test_rebuild_with_the_flags_off_unregisters_the_distribution():
    pl = _planner(ada.AdaptiveOracleBackend, update_cov=True, update_lambda=True)
    pl.compute_action(Q0, [0] * 7)
    assert pl.sim.backend.dist is pl.mppi.dist
    pl.cfg.mppi.update_cov = pl.cfg.mppi.update_lambda = False
    pl._build_mppi()
    assert pl.mppi.dist is None and pl.sim.backend.dist is None and pl.mppi.cov_action is None
    from oracle.backend import OracleBackend
    ref = _planner(OracleBackend)
    for _ in range(2):
        np.testing.assert_array_equal(pl.compute_action(Q0, [0] * 7).numpy(), ref.compute_action(Q0, [0] * 7).numpy())
