"""CPU: the float64 reference of Smooth MPPI (``mppi_mode: smooth``) -- the integration's known answers, the smoothness cost, shard
merging -- the planner planning with it on the checker backend, the rate bound on the executed command, and every refusal of the mode."""
import numpy as np
import pytest
import torch

import smooth_oracle as so
from mppi_isaac_b200.model.blob import MODE_SMOOTH, make_params
from mppi_isaac_b200.utils.config_store import IsaacGymConfig
from scenes import panda_cfg, panda_mppi, panda_setup

Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
NU = 7


def _params(K=64, T=6, **kw):
    d = dict(smooth_weight=0.5, du_min=[-2.0], du_max=[2.0])
    d.update(kw)
    sc, p, _ = panda_setup(K=K, T=T, mode="smooth", **d)
    return sc, p


def test_make_params_sets_the_smooth_block():
    _, p = _params(smooth_weight=0.25, du_min=[-1.0], du_max=[1.5])
    assert p.mode == MODE_SMOOTH and p.gamma == 1.0 and abs(p.smooth_weight - 0.25) < 1e-7
    assert [p.du_min[j] for j in range(NU)] == [-1.0] * NU and [p.du_max[j] for j in range(NU)] == [1.5] * NU
    _, p = _params(du_min=None, du_max=None)
    assert p.du_min[0] == np.float32(-1e30) and p.du_max[NU - 1] == np.float32(1e30)
    _, p = _params(du_min=[-float(j + 1) for j in range(NU)])
    assert [p.du_min[j] for j in range(NU)] == [-float(j + 1) for j in range(NU)]


@pytest.mark.parametrize("kw, match", [
    (dict(smooth_weight=-0.1), "smooth_weight"), (dict(smooth_weight=float("inf")), "smooth_weight"),
    (dict(smooth_weight=float("nan")), "smooth_weight"), (dict(du_min=[1.0], du_max=[0.5]), "du_min"),
    (dict(du_min=[0.0, 1.0]), "du_min"), (dict(update_cov=True), "update_cov"), (dict(update_lambda=True), "update_cov"),
    (dict(filter_u=True), "switch filter_u off"), (dict(sampling_method="halton"), "halton"), (dict(sampling_method="colored"), "colored"),
])
def test_make_params_refuses(kw, match):
    sc, _, _ = panda_setup(K=4, T=12)
    with pytest.raises(ValueError, match=match):
        make_params(panda_mppi(64, 12, mode="smooth", **kw), IsaacGymConfig(), sc.nu, 64, [])


def test_make_params_refuses_long_horizons_and_a_non_positive_dt():
    sc, _, _ = panda_setup(K=4, T=12)
    with pytest.raises(ValueError, match="horizon"):
        make_params(panda_mppi(64, 80, mode="smooth"), IsaacGymConfig(), sc.nu, 64, [])            # T*nu = 560 > 512
    make_params(panda_mppi(64, 73, mode="smooth"), IsaacGymConfig(), sc.nu, 64, [])                # T*nu = 511
    with pytest.raises(ValueError, match="dt"):
        make_params(panda_mppi(64, 12, mode="smooth"), IsaacGymConfig(dt=0.0), sc.nu, 64, [])


def _z(sc, p, K, seed=3, plan=1):
    return so.co.white(sc.model, p, seed, plan, 0, K)


def test_no_binding_bound_integrates_the_derivative():
    """omega = 0 and no bound binding: A = a_prev + dt cumsum(U), the noise is the derivative noise L0 z."""
    sc, p = _params(K=16, T=8, du_min=None, du_max=None, u_min=[-1e3], u_max=[1e3], sample_null_action=False, smooth_weight=0.0)
    rng = np.random.default_rng(0)
    U = rng.uniform(-0.5, 0.5, (8, NU)).astype(np.float32)
    a_prev = rng.uniform(-0.1, 0.1, NU).astype(np.float32)
    st = so.make_state(p, NU, a_prev)
    rows = so.reduce(p, NU, np.zeros((8, 16), np.float32), np.zeros((8, NU, 16), np.float32), U)
    Un, act, stats, st2 = so.finalize(p, NU, rows[None], U, st)
    np.testing.assert_allclose(Un, U, rtol=0, atol=0)                     # W = 0: U' = U
    A = so.unpack(st2, 8, NU)[1]
    np.testing.assert_allclose(A, a_prev[None].astype(np.float64) + np.float32(p.dt) * np.cumsum(U.astype(np.float64), 0), rtol=0, atol=1e-6)
    np.testing.assert_array_equal(act, A[0])
    np.testing.assert_array_equal(so.unpack(st2, 8, NU)[0], A[0])
    z = _z(sc, p, 16)
    a, n = so.sample(p, NU, U, z, st, 0, 16)
    L = np.array(p.sigma_chol[:NU * NU], np.float32).reshape(NU, NU).astype(np.float64)
    np.testing.assert_allclose(n, np.einsum("ji,tik->tjk", L, z), rtol=0, atol=1e-6)
    v = U[:, :, None].astype(np.float64) + n
    np.testing.assert_allclose(a, a_prev[None, :, None] + np.float32(p.dt) * np.cumsum(v, 0), rtol=0, atol=1e-5)


def test_an_action_clamp_mid_horizon_continues_from_the_clamped_value_and_projects_U():
    sc, p = _params(K=8, T=6, du_min=None, du_max=None, u_min=[-0.2], u_max=[0.2], smooth_weight=0.0)
    dt = float(np.float32(p.dt))
    U = np.zeros((6, NU), np.float32)
    U[:, 0] = 2.0                                                          # 0.1 per step: binds at t = 2 from a_prev = 0
    U[3:, 0] = -2.0
    st = so.make_state(p, NU)
    rows = so.reduce(p, NU, np.zeros((6, 8), np.float32), np.zeros((6, NU, 8), np.float32), U)
    Un, _, _, st2 = so.finalize(p, NU, rows[None], U, st)
    A = so.unpack(st2, 6, NU)[1]
    np.testing.assert_allclose(A[:, 0], [0.1, 0.2, 0.2, 0.1, 0.0, -0.1], rtol=0, atol=1e-6)
    np.testing.assert_allclose(Un[:, 0], [2.0, 2.0, 0.0, -2.0, -2.0, -2.0], rtol=0, atol=1e-5)      # t = 2 projected to 0
    np.testing.assert_allclose(np.diff(np.concatenate([[0.0], A[:, 0]])) / dt, Un[:, 0], rtol=0, atol=1e-5)


def test_derivative_bounds_bind_in_the_sample_and_in_the_update():
    sc, p = _params(K=32, T=5, du_min=[-0.5], du_max=[0.25], u_min=[-10.0], u_max=[10.0], sample_null_action=False)
    U = np.zeros((5, NU), np.float32)
    U[:, 1] = 3.0
    z = _z(sc, p, 32)
    a, n = so.sample(p, NU, U, z, so.make_state(p, NU), 0, 32)
    v = n + U[:, :, None]
    assert v.min() >= -0.5 - 1e-7 and v.max() <= 0.25 + 1e-7
    np.testing.assert_allclose(v[:, 1], 0.25, rtol=0, atol=1e-7)
    rows = so.reduce(p, NU, np.zeros((5, 32), np.float32), np.zeros((5, NU, 32), np.float32), U)
    Un, _, _, _ = so.finalize(p, NU, rows[None], U, so.make_state(p, NU))
    np.testing.assert_allclose(Un[:, 1], 0.25, rtol=0, atol=1e-7)


def test_the_null_row_holds_the_previous_action():
    sc, p = _params(K=16, T=7, sample_null_action=True)
    a_prev = np.linspace(-0.15, 0.15, NU).astype(np.float32)
    U = np.random.default_rng(1).uniform(-1, 1, (7, NU)).astype(np.float32)
    a, n = so.sample(p, NU, U, _z(sc, p, 16), so.make_state(p, NU, a_prev), 0, 16)
    np.testing.assert_array_equal(a[:, :, 15], np.broadcast_to(a_prev, (7, NU)))
    np.testing.assert_array_equal(n[:, :, 15], -U)
    assert not np.allclose(a[:, :, 14], a_prev[None])


def test_eta_zero_keeps_U_but_still_integrates():
    sc, p = _params(K=8, T=4, u_min=[-0.2], u_max=[0.2])
    U = np.full((4, NU), 0.5, np.float32)
    rows = np.zeros((2, 2 + 4 * NU), np.float32)
    rows[:, 0] = np.inf                                                    # no valid sample in either shard
    Un, act, stats, st = so.finalize(p, NU, rows, U, so.make_state(p, NU))
    np.testing.assert_array_equal(Un, U)
    assert stats[1] == 0.0 and stats[0] == np.inf
    np.testing.assert_allclose(so.unpack(st, 4, NU)[1][:, 0], 0.5 * np.float32(p.dt) * np.arange(1, 5), rtol=1e-6)
    np.testing.assert_array_equal(act, so.unpack(st, 4, NU)[1][0])


def test_two_sample_weight_ratio_is_the_smoothness_cost():
    """Equal running costs and U = 0: S_k = omega dt^2 |v_k|^2, so w_1 / w_2 = exp(-omega dt^2 (|v_1|^2 - |v_2|^2) / lambda)."""
    sc, p = _params(K=4, T=5, smooth_weight=2.0, du_min=None, du_max=None)
    rng = np.random.default_rng(2)
    x = np.zeros((5, NU, 4), np.float32)
    x[:, :, 0] = rng.uniform(-1, 1, (5, NU))
    x[:, :, 1] = rng.uniform(-1, 1, (5, NU))
    x[:, :, 2:] = 50.0                                                     # weights ~ 0
    row = so.reduce(p, NU, np.ones((5, 4), np.float32), x, np.zeros((5, NU), np.float32))
    w = np.linalg.lstsq(x[:, :, :2].reshape(-1, 2).astype(np.float64), row[2:].astype(np.float64), rcond=None)[0]
    om, dt, lam = float(np.float32(p.smooth_weight)), float(np.float32(p.dt)), float(np.float32(p.lambda_))
    q = (x[:, :, :2].astype(np.float64) ** 2).sum((0, 1))
    np.testing.assert_allclose(w[0] / w[1], np.exp(-om * dt * dt * (q[0] - q[1]) / lam), rtol=1e-5)
    assert np.isclose(row[0], 5.0 + om * dt * dt * q.min(), rtol=1e-6)


def test_omega_zero_row_is_the_simple_row(oracle):
    """With omega = 0 the smooth K3 is SIMPLE's (gamma = 1): the oracle's row of the same inputs within float32 rounding."""
    sc, p = _params(K=64, T=6, smooth_weight=0.0)
    _, ps, _ = panda_setup(K=64, T=6, mode="simple")
    rng = np.random.default_rng(4)
    cost = rng.uniform(0, 1, (6, 64)).astype(np.float32)
    x = rng.uniform(-0.3, 0.3, (6, NU, 64)).astype(np.float32)
    U = rng.uniform(-0.1, 0.1, (6, NU)).astype(np.float32)
    ref, _ = oracle.reduce(sc.model, ps, cost, x, U)
    np.testing.assert_allclose(so.reduce(p, NU, cost, x, U), ref, rtol=2e-5, atol=1e-6)


@pytest.mark.parametrize("G", [2, 4, 8])
def test_merging_shard_rows_equals_one_shard(G):
    K, T = 256, 5
    sc, p = _params(K=K, T=T, u_min=[-0.2], u_max=[0.2], du_min=[-1.0], du_max=[1.0])
    rng = np.random.default_rng(G)
    cost = rng.uniform(0, 1, (T, K)).astype(np.float32)
    x = rng.uniform(-0.5, 0.5, (T, NU, K)).astype(np.float32)
    U = rng.uniform(-0.3, 0.3, (T, NU)).astype(np.float32)
    st = so.make_state(p, NU, rng.uniform(-0.1, 0.1, NU))
    one = so.finalize(p, NU, so.reduce(p, NU, cost, x, U)[None], U, st)
    b = np.linspace(0, K, G + 1).astype(int)
    rows = np.stack([so.reduce(p, NU, cost[:, lo:hi], x[:, :, lo:hi], U) for lo, hi in zip(b[:-1], b[1:])])
    many = so.finalize(p, NU, rows, U, st)
    for u, v in zip(one, many):
        np.testing.assert_allclose(u, v, rtol=1e-5, atol=1e-6)


def _planner(rollout_mode="auto", K=64, T=12, **kw):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    d = dict(mppi_mode="smooth", sampling_method="random", filter_u=False, smooth_weight=0.5, du_min=[-1.0], du_max=[1.0])
    d.update(kw)
    cfg = panda_cfg(K=K, T=T, device="cpu", **d)
    return MPPIisaacPlanner(cfg, PandaReachObjective(), backend=so.SmoothOracleBackend(), rollout_mode=rollout_mode, use_cuda_graph=False)


def test_planner_plans_batched_and_stepwise_alike():
    a, b = _planner("batched"), _planner("stepwise")
    m = a.mppi
    assert m.smooth and m.action_sequence.shape == (12, NU) and m.previous_action.shape == (NU,)
    np.testing.assert_array_equal(m.previous_action.numpy(), 0.0)
    for it in range(3):
        ua = a.compute_action(Q0, [0.0] * NU)
        ub = b.compute_action(Q0, [0.0] * NU)
        assert torch.isfinite(ua).all()
        np.testing.assert_allclose(ua.numpy(), ub.numpy(), rtol=0, atol=1e-5)
        np.testing.assert_array_equal(ua.numpy(), m.previous_action.numpy())
        np.testing.assert_array_equal(m.action_sequence[0].numpy(), m.previous_action.numpy())
        assert int(m.plan_ctr[0]) == it + 1
    np.testing.assert_allclose(a.mppi.U.numpy(), b.mppi.U.numpy(), rtol=0, atol=1e-4)


def test_rebuilds_keep_or_reset_the_previous_action():
    pl = _planner()
    pl.compute_action(Q0, [0.0] * NU)
    prev = pl.mppi.previous_action.clone()
    assert prev.abs().max() > 0
    pl._build_mppi(keep_U=True)                                            # a rebuilt simulator keeps the warm start
    np.testing.assert_array_equal(pl.mppi.previous_action.numpy(), prev.numpy())
    pl.update_mppi_params({"noise_sigma": (0.05 * np.eye(NU)).tolist()})  # a fresh planner, as in the reference
    np.testing.assert_array_equal(pl.mppi.previous_action.numpy(), 0.0)


def test_set_previous_action_takes_effect():
    pl = _planner(du_min=[-0.5], du_max=[0.5])
    pl.compute_action(Q0, [0.0] * NU)
    a = np.full(NU, 0.1, np.float32)
    pl.mppi.set_previous_action(a)
    np.testing.assert_array_equal(pl.mppi.previous_action.numpy(), a)
    act = pl.compute_action(Q0, [0.0] * NU).numpy()
    assert np.all(np.abs(act - a) <= 0.5 * np.float32(pl.cfg.isaacgym.dt) + 1e-6)


def test_executed_command_is_rate_bounded_over_50_plans():
    """Wide derivative noise (sigma = 2 against du_max = 0.4) and no null row, so that consecutive plans differ: every executed step
    stays within du_max dt, and some come close to it."""
    pl = _planner(K=32, T=8, du_min=[-0.4], du_max=[0.4], smooth_weight=0.0, sample_null_action=False, noise_sigma=(4.0 * np.eye(NU)).tolist())
    bound = 0.4 * float(np.float32(pl.cfg.isaacgym.dt)) * (1 + 1e-5)
    prev = np.zeros(NU, np.float32)
    jumps = []
    for _ in range(50):
        a = pl.compute_action(Q0, [0.0] * NU).numpy()
        jumps.append(np.abs(a - prev).max())
        prev = a
    assert max(jumps) <= bound and max(jumps) > 0.25 * bound, (max(jumps), bound)


def test_planner_refuses_priors_and_several_actions_per_command():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective

    class Prior:
        def compute_command(self, sim):
            return torch.zeros(NU)
    cfg = panda_cfg(K=32, T=8, device="cpu", mppi_mode="smooth", sampling_method="random", filter_u=False, use_priors=True)
    with pytest.raises(ValueError, match="prior"):
        MPPIisaacPlanner(cfg, PandaReachObjective(), prior=Prior(), backend=so.SmoothOracleBackend())
    cfg = panda_cfg(K=32, T=8, device="cpu", mppi_mode="smooth", sampling_method="random", filter_u=False, u_per_command=2)
    with pytest.raises(ValueError, match="u_per_command"):
        MPPIisaacPlanner(cfg, PandaReachObjective(), backend=so.SmoothOracleBackend())
