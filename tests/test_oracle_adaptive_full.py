"""Adaptive MPPI with a full sampling covariance (update_cov with cov_type: full) on the CPU: the rule of DESIGN.md section 2 restated in
float64 against the reference of ``adaptive_full_oracle``, known answers, agreement with the diagonal rule, shard invariance of the
covariance row, and the planner plumbing."""
import copy
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as tdist
import torch.multiprocessing as mp

import adaptive_full_oracle as afo
import adaptive_oracle as ada
from mppi_isaac_b200.model.blob import MODE_SIMPLE
from oracle import oracle as orc
from scenes import panda_cfg, panda_setup

HERE = os.path.dirname(os.path.abspath(__file__))
Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
NU = 7
# a correlated 7 x 7 Sigma: joints 2, 4 and 6 of a reach move together
_A = np.random.default_rng(3).normal(0, 0.15, (NU, NU))
SIG_CORR = (_A @ _A.T + 0.05 * np.eye(NU)).round(6)
SIG_CORR = 0.5 * (SIG_CORR + SIG_CORR.T)
SIG_DIAG = np.diag([0.3, 0.5, 0.2, 0.4, 0.25, 0.35, 0.15])
STARTS = {"correlated": SIG_CORR, "diagonal": SIG_DIAG}


def _setup(mode, sigma, K=256, T=12, **kw):
    kw.setdefault("u_min", [-1e6])
    kw.setdefault("u_max", [1e6])
    kw.setdefault("sample_null_action", False)
    sc, p, _ = panda_setup(K=K, T=T, mode=mode, noise_sigma=np.asarray(sigma).tolist(), update_cov=True, cov_type="full", **kw)
    return sc.model, p


def _target(nu):
    return np.linspace(-0.4, 0.4, nu).astype(np.float32)


def _cost(a, target):
    """(T, nu, K) actions -> (T, K) cost: squared distance of every step's action to a target, which makes the weights non-trivial."""
    return ((a - target[None, :, None]) ** 2).sum(1)


class Restated:
    """float64 restatement of the full-covariance plan tail, independent of oracle.cpp: K1 (L z), K3 (S, weights, W, C) and K4 (U,
    Sigma, lambda)."""

    def __init__(self, p, nu):
        self.p, self.nu = p, nu

    def plan(self, U, lam, Sigma, z, target):
        p, T, nu = self.p, self.p.T, self.nu
        U = torch.cat([U[1:], torch.tensor(np.array(p.u_init[:nu]), dtype=torch.float64)[None]])
        L = torch.linalg.cholesky(Sigma)
        noise = torch.einsum("ji,tik->tjk", L, z)
        a = U[:, :, None] + noise
        simple = p.mode == MODE_SIMPLE
        x = noise if simple else a
        S = (float(p.gamma) ** torch.arange(T, dtype=torch.float64))[:, None].mul(_cost(a, target)).sum(0)
        if simple:
            S = S + lam * torch.einsum("tj,ji,tik->k", U, torch.linalg.inv(Sigma), noise)
        w = torch.exp(-(S - S.min()) / lam)
        eta = w.sum()
        W = (w * x).sum(-1)
        c = torch.zeros_like(U) if simple else U
        dx = x - c[:, :, None]
        C = torch.einsum("tik,tjk,k->ij", dx, dx, w)
        U_new = U + W / eta if simple else (1 - p.step_size_mean) * U + p.step_size_mean * W / eta
        d = U_new - U
        m1 = W / eta - c
        V = C / eta - (m1.T @ d + d.T @ m1 - d.T @ d)
        Sigma = (1 - p.step_size_cov) * Sigma + (p.step_size_cov / T) * V + p.kappa * torch.eye(nu, dtype=torch.float64)
        if p.update_lambda:
            if eta > p.eta_u_bound:
                lam = lam * (1 - p.lambda_mult)
            elif eta < p.eta_l_bound:
                lam = lam * (1 + p.lambda_mult)
            lam = min(max(lam, 1e-3 * p.lambda_), 1e3 * p.lambda_)
        return U_new, lam, Sigma, float(eta)


def _plan(m, p, U, dist, plan, target, seed=7):
    """One reference plan from (U, dist): shift, K1, K3 (with C), K4; returns (U, stats, dist, actions, x)."""
    nu = m.nu
    U = orc.shift(m, p, U)
    a, n = orc.sample(m, afo.dist_params(p, nu, dist), seed, plan, U)
    x = n if p.mode == MODE_SIMPLE else a
    row = afo.reduce(m, p, _cost(a, target), x, U, dist)
    U2, _, stats, d2 = afo.finalize(m, p, row[None], U, dist)
    return U, U2, stats, d2, a, x, row


@pytest.mark.parametrize("start", list(STARTS))
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_restatement_matches_reference_over_20_plans(mode, start):
    m, p = _setup(mode, STARTS[start], lambda_=0.5, update_lambda=True, eta_u_bound=40.0, eta_l_bound=8.0)
    nu, T = m.nu, p.T
    target = _target(nu)
    ref = Restated(p, nu)
    U, dist = np.zeros((T, nu), np.float32), afo.make_dist(p.lambda_, STARTS[start])
    white = afo.dist_params(p, nu, dist, white=True)
    off_diag = 0.0
    for plan in range(20):
        # the restatement starts every plan from the reference's state, so float32 rounding cannot accumulate over the 20 plans
        lam0, Sig0 = float(dist[0]), torch.tensor(afo.unpack(dist, nu)[1], dtype=torch.float64)
        U0 = torch.tensor(U, dtype=torch.float64)
        _, U, stats, dist, _, _, _ = _plan(m, p, U, dist, plan, target)
        z, _ = orc.sample(m, white, 7, plan, np.zeros((T, nu), np.float32))
        Ur, lam, Sig, eta = ref.plan(U0, lam0, Sig0, torch.tensor(np.asarray(z, np.float64)), torch.tensor(target, dtype=torch.float64))
        _, S32, L32, I32 = afo.unpack(dist, nu)
        np.testing.assert_allclose(stats[1], eta, rtol=1e-3)
        np.testing.assert_allclose(U, Ur.numpy(), rtol=1e-4, atol=2e-5)
        np.testing.assert_allclose(dist[0], lam, rtol=1e-5)
        np.testing.assert_allclose(S32, Sig.numpy(), rtol=1e-4, atol=1e-6 * np.abs(Sig.numpy()).max())
        np.testing.assert_allclose(L32, torch.linalg.cholesky(Sig).numpy(), rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(I32, torch.linalg.inv(Sig).numpy(), rtol=1e-3, atol=1e-4 * np.abs(I32).max())
        off_diag = max(off_diag, float(np.abs(S32 - np.diag(np.diag(S32))).max()))
    assert off_diag > 1e-5                                                    # the rule learns correlations from a diagonal start too


def test_simple_mode_one_dominant_sample_gives_v_zero():
    """SIMPLE mode, one sample with all the weight: m1 = d = x_k, so V = C - sum_t x x^T = 0 and Sigma <- 0.3 Sigma + 0.005 I."""
    m, p = _setup("simple", SIG_CORR, K=64, lambda_=0.01)
    nu, T, K = m.nu, p.T, p.K
    U, dist = np.zeros((T, nu), np.float32), afo.make_dist(p.lambda_, SIG_CORR)
    Sig = SIG_CORR.astype(np.float32).astype(np.float64)
    for plan in range(5):
        a, n = orc.sample(m, afo.dist_params(p, nu, dist), 3, plan, U)
        cost = np.full((T, K), 50.0, np.float32)
        cost[:, 11] = 0.0
        row = afo.reduce(m, p, cost, n, U, dist)
        assert abs(row[1] - 1.0) < 1e-6
        U, _, _, dist = afo.finalize(m, p, row[None], U, dist)
        Sig = 0.3 * Sig + 0.005 * np.eye(nu)
        np.testing.assert_allclose(afo.unpack(dist, nu)[1], Sig, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_sigma_stays_symmetric_and_l_reproduces_it(mode):
    m, p = _setup(mode, SIG_CORR, lambda_=0.3)
    nu, T = m.nu, p.T
    U, dist = np.zeros((T, nu), np.float32), afo.make_dist(p.lambda_, SIG_CORR)
    for plan in range(20):
        _, U, _, dist, _, _, _ = _plan(m, p, U, dist, plan, _target(nu))
        _, S, L, I = afo.unpack(dist, nu)
        np.testing.assert_array_equal(S, S.T)
        np.testing.assert_array_equal(I, I.T)
        np.testing.assert_array_equal(L, np.tril(L))
        LL = L.astype(np.float64) @ L.T.astype(np.float64)
        assert np.abs(LL - S).max() <= 1e-6 * np.abs(S).max()
        assert np.abs(I.astype(np.float64) @ S - np.eye(nu)).max() <= 1e-4


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_diagonal_start_matches_the_diagonal_rule(mode):
    """From a diagonal Sigma one plan of the full rule gives the diagonal rule's cov on the diagonal (its clamp at 0 is inactive),
    and off the diagonal (s/T) times the weighted cross-moments about the new mean."""
    m, p = _setup(mode, SIG_DIAG, lambda_=0.3)
    nu, T = m.nu, p.T
    pd = copy.deepcopy(p)
    pd.cov_full = 0
    rng = np.random.default_rng(2)
    U = rng.normal(0, 0.1, (T, nu)).astype(np.float32)
    dist = afo.make_dist(p.lambda_, SIG_DIAG)
    ddiag = np.concatenate([[p.lambda_], np.diag(SIG_DIAG)]).astype(np.float32)
    a, n = orc.sample(m, afo.dist_params(p, nu, dist), 5, 0, U)
    a2, n2 = orc.sample(m, ada.dist_params(pd, nu, ddiag), 5, 0, U)
    np.testing.assert_array_equal(a, a2)
    x = n if p.mode == MODE_SIMPLE else a
    cost = _cost(a, _target(nu))
    U_full, _, st, d_full = afo.finalize(m, p, afo.reduce(m, p, cost, x, U, dist)[None], U, dist)
    U_diag, _, _, d_diag = ada.finalize(m, pd, ada.reduce(m, pd, cost, x, U, ddiag)[None], U, ddiag)
    np.testing.assert_array_equal(U_full, U_diag)
    S = afo.unpack(d_full, nu)[1].astype(np.float64)
    np.testing.assert_allclose(np.diag(S), d_diag[1:], rtol=1e-5)
    # off the diagonal: (s/T) sum_t sum_k (w_k / eta) e_tki e_tkj with e = x - U_new (MEAN) or x - (U_new - U) (SIMPLE)
    w = afo.weights(p, nu, cost, x, U, dist)
    p_nf = copy.deepcopy(p)
    p_nf.filter_u = 0
    U_pre = orc.finalize(m, afo.dist_params(p_nf, nu, dist), orc.reduce(m, afo.dist_params(p, nu, dist), cost, x, U)[0][None], U)[0]
    centre = U_pre - U if p.mode == MODE_SIMPLE else U_pre
    e = np.asarray(x, np.float64) - centre.astype(np.float64)[:, :, None]
    cross = np.einsum("tik,tjk,k->ij", e, e, w / w.sum())
    off = ~np.eye(nu, dtype=bool)
    np.testing.assert_allclose(S[off], (p.step_size_cov / T) * cross[off], rtol=1e-4, atol=1e-7 * np.abs(cross).max())
    assert np.abs(S[off]).max() > 1e-5


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("G", [2, 4, 8])
def test_covariance_row_is_shard_invariant(mode, G):
    m, p = _setup(mode, SIG_CORR, K=256, update_lambda=True, lambda_=0.3)
    nu, T, K = m.nu, p.T, p.K
    rng = np.random.default_rng(5)
    U = rng.normal(0, 0.2, (T, nu)).astype(np.float32)
    dist = afo.make_dist(0.25, SIG_CORR)
    a, n = orc.sample(m, afo.dist_params(p, nu, dist), 9, 4, U)
    x = n if p.mode == MODE_SIMPLE else a
    cost = rng.uniform(0, 2, (T, K)).astype(np.float32)
    row1 = afo.reduce(m, p, cost, x, U, dist)
    one = afo.finalize(m, p, row1[None], U, dist)
    Ks = K // G
    ps = copy.deepcopy(p)
    ps.K = Ks
    rows = np.stack([afo.reduce(m, ps, np.ascontiguousarray(cost[:, g * Ks:(g + 1) * Ks]), np.ascontiguousarray(x[:, :, g * Ks:(g + 1) * Ks]), U, dist)
                     for g in range(G)])
    # the C blocks, rescaled to the common minimum like W, add up to the single-shard block
    s = np.exp(-(rows[:, 0].astype(np.float64) - rows[:, 0].min()) / float(dist[0]))
    NR = T * nu
    C = (s[:, None] * rows[:, 2 + NR:].astype(np.float64)).sum(0) * np.exp(-(rows[:, 0].min() - row1[0]) / float(dist[0]))
    np.testing.assert_allclose(C, row1[2 + NR:], rtol=1e-5, atol=1e-6 * np.abs(row1[2 + NR:]).max())
    many = afo.finalize(m, p, rows, U, dist)
    np.testing.assert_allclose(many[0], one[0], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(many[3], one[3], rtol=1e-5, atol=1e-7)


def test_indefinite_update_leaves_sigma_l_and_inverse_unchanged():
    """A hand-built row whose update is indefinite (a large negative C) keeps Sigma, L and Sigma^-1; lambda still moves."""
    m, p = _setup("simple", SIG_CORR, K=64, update_lambda=True, lambda_=0.3, eta_u_bound=10.0, eta_l_bound=5.0)
    nu, T = m.nu, p.T
    dist = afo.make_dist(0.3, SIG_CORR)
    row = np.zeros(2 + T * nu + nu * (nu + 1) // 2, np.float32)
    row[1] = 2.0                                                             # eta < eta_l_bound: lambda *= 1.1
    row[2 + T * nu:] = afo.tril_pack(-100.0 * np.eye(nu))
    U = np.zeros((T, nu), np.float32)
    _, _, _, d = afo.finalize(m, p, row[None], U, dist)
    np.testing.assert_array_equal(d[1:], dist[1:])
    assert d[0] == np.float32(0.3) * (np.float32(1) + np.float32(0.1))


def _planner(backend_cls, **kw):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    return MPPIisaacPlanner(panda_cfg(K=64, T=12, **kw), PandaReachObjective(), backend=backend_cls())


def test_config_errors():
    with pytest.raises(ValueError, match="cov_type"):
        _planner(afo.AdaptiveFullOracleBackend, update_cov=True, cov_type="banded")
    with pytest.raises(ValueError, match="needs update_cov"):
        _planner(afo.AdaptiveFullOracleBackend, cov_type="full", noise_sigma=SIG_CORR.tolist())
    with pytest.raises(ValueError, match="needs update_cov"):
        _planner(afo.AdaptiveFullOracleBackend, update_lambda=True, cov_type="full")
    with pytest.raises(ValueError, match="diagonal"):
        _planner(afo.AdaptiveFullOracleBackend, update_cov=True, noise_sigma=SIG_CORR.tolist())
    with pytest.raises(ValueError, match="diagonal"):
        _planner(afo.AdaptiveFullOracleBackend, update_cov=True, cov_type="diag", noise_sigma=SIG_CORR.tolist())
    bad = SIG_CORR.copy()
    bad[0, 1] += 0.01
    with pytest.raises(ValueError, match="symmetric positive-definite"):
        _planner(afo.AdaptiveFullOracleBackend, update_cov=True, cov_type="full", noise_sigma=bad.tolist())


def test_planner_state_rebuilds_and_resets():
    pl = _planner(afo.AdaptiveFullOracleBackend, update_cov=True, update_lambda=True, cov_type="full", noise_sigma=SIG_CORR.tolist())
    nu, T = 7, 12
    assert pl.mppi.dist.shape == (1 + 3 * nu * nu,) and pl.mppi.partial.shape == (2 + T * nu + nu * (nu + 1) // 2,)
    np.testing.assert_array_equal(pl.mppi.dist.numpy(), afo.make_dist(pl.cfg.mppi.lambda_, SIG_CORR))
    assert pl.mppi.cov_action.shape == (nu, nu)
    np.testing.assert_allclose(pl.mppi.cov_action.numpy(), SIG_CORR, rtol=1e-7)
    assert float(pl.mppi.current_lambda) == np.float32(pl.cfg.mppi.lambda_)
    d0 = pl.mppi.dist.clone()
    for _ in range(4):
        pl.compute_action(Q0, [0] * 7)
    d4 = pl.mppi.dist.clone()
    assert not torch.equal(d4, d0)
    assert pl.mppi.cov_action.data_ptr() == pl.mppi.dist.data_ptr() + 4                 # a view of the live buffer
    pl._build_mppi(keep_U=True)                                              # obstacle added / add_to_env: U and dist survive
    assert torch.equal(pl.mppi.dist, d4) and pl.sim.backend.dist is pl.mppi.dist
    sig2 = 0.2 * np.eye(7) + 0.01
    pl.update_mppi_params({"noise_sigma": sig2.tolist()})                    # rebuilt from the new Sigma
    np.testing.assert_array_equal(pl.mppi.dist.numpy(), afo.make_dist(pl.cfg.mppi.lambda_, sig2))
    # the diag rule keeps its (nu,) view
    pd = _planner(afo.AdaptiveFullOracleBackend, update_cov=True)
    assert pd.mppi.cov_action.shape == (nu,)


def test_rebuild_with_the_flags_off_unregisters_the_distribution():
    pl = _planner(afo.AdaptiveFullOracleBackend, update_cov=True, cov_type="full", noise_sigma=SIG_CORR.tolist())
    pl.compute_action(Q0, [0] * 7)
    assert pl.sim.backend.dist is pl.mppi.dist
    pl.cfg.mppi.update_cov = False
    pl.cfg.mppi.cov_type = "diag"
    pl._build_mppi()
    assert pl.mppi.dist is None and pl.sim.backend.dist is None and pl.mppi.cov_action is None


def test_full_rule_plans_track_the_restatement_through_the_planner():
    """The planner with the full rule on the oracle backend: the partial row it hands K4 carries C, and dist follows the
    reference's update of the same row."""
    pl = _planner(afo.AdaptiveFullOracleBackend, update_cov=True, cov_type="full", noise_sigma=SIG_CORR.tolist())
    be = pl.sim.backend
    seen = []
    orig = be.finalize

    def spy(partials, G, U, action_out, stats):
        seen.append((partials.clone(), U.clone(), be.dist.clone()))
        return orig(partials, G, U, action_out, stats)
    be.finalize = spy
    pl.compute_action(Q0, [0] * 7)
    be.finalize = orig
    (rows, U, d), = seen
    _, _, _, d_ref = afo.finalize(be.model, be.params, rows.numpy(), U.numpy(), d.numpy())
    np.testing.assert_array_equal(pl.mppi.dist.numpy(), d_ref)
    assert np.abs(rows.numpy()[0, 2 + 12 * 7:]).max() > 0


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    tdist.init_process_group("gloo", rank=rank, world_size=world)
    import adaptive_full_oracle
    pl = _planner(adaptive_full_oracle.AdaptiveFullOracleBackend, update_cov=True, update_lambda=True, cov_type="full",
                  noise_sigma=SIG_CORR.tolist())
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
    single = _planner(afo.AdaptiveFullOracleBackend, update_cov=True, update_lambda=True, cov_type="full", noise_sigma=SIG_CORR.tolist())
    for _ in range(4):
        single.compute_action(Q0, [0] * 7)
    np.testing.assert_allclose(d0, single.mppi.dist.numpy(), rtol=1e-4, atol=1e-6)
