"""CPU: the float64 reference of annealed MPPI (``anneal_iterations`` / ``anneal_iter_decay`` / ``anneal_horizon_decay``) -- known schedule
values, every refusal, the unchanged planner at the defaults, an N-iteration plan against N hand-sequenced plain MPPI steps, the counter,
``set_noise_schedule``, the ``keep_U`` rebuild, a stepwise plan with a prior and the ``n_worlds`` keying."""
import copy

import numpy as np
import pytest
import torch

import anneal_oracle as ao
from mppi_isaac_b200.model.blob import anneal_schedule, make_params
from mppi_isaac_b200.utils.config_store import IsaacGymConfig
from scenes import point_cfg, point_mppi, point_setup

Q0, QD0 = [0.1, 0.0, 0.0], [0.0] * 3
ANNEAL = dict(anneal_iterations=3, anneal_iter_decay=0.6, anneal_horizon_decay=0.9)


def _planner(backend=None, **kw):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    kw.setdefault("filter_u", False)                                           # the point config filters U, which needs T >= 9
    return MPPIisaacPlanner(point_cfg(**kw), PointReachObjective(), backend=backend or ao.AnnealOracleBackend(), use_cuda_graph=False)


def test_known_schedule_values():
    s, r = ao.schedule(3, 0.5, 0.8, 4)
    assert s[0, 3] == 1.0 and r[0, 3] == 1.0                                   # iteration 0, far end of the horizon
    assert s[1, 0] == np.float32(0.5 * 0.8 ** 3) and s[2, 3] == np.float32(0.25) and s[2, 2] == np.float32(0.2)
    assert r[2, 3] == np.float32(16.0) and r[1, 0] == np.float32(1.0 / (0.5 * 0.8 ** 3) ** 2)
    p = _planner(K=64, T=4, anneal_iterations=3, anneal_iter_decay=0.5, anneal_horizon_decay=0.8)
    np.testing.assert_array_equal(p.mppi.noise_schedule.numpy(), s)
    np.testing.assert_array_equal(p.mppi.anneal_state.numpy(), ao.make_state(s, r))
    assert p.mppi.anneal_iterations == 3 and p.mppi.iterations == 3


@pytest.mark.parametrize("kw, msg", [
    (dict(anneal_iterations=0), "anneal_iterations"),
    (dict(anneal_iterations=17), "anneal_iterations"),
    (dict(anneal_iter_decay=0.0), "anneal_iter_decay"),
    (dict(anneal_iter_decay=1.5), "anneal_iter_decay"),
    (dict(anneal_horizon_decay=float("nan")), "anneal_horizon_decay"),
    (dict(anneal_horizon_decay=float("inf")), "anneal_horizon_decay"),
    (dict(anneal_horizon_decay=0.5, horizon=30), "2\\^-20"),
    (dict(anneal_iterations=16, anneal_iter_decay=0.3), "2\\^-20"),
    (dict(mppi_mode="cem"), "cem"),
    (dict(mppi_mode="smooth"), "smooth"),
    (dict(sampling_method="halton"), "halton"),
    (dict(update_cov=True), "update_cov"),
    (dict(update_lambda=True), "update_cov and update_lambda"),
    (dict(update_cov=True, cov_type="full"), "update_cov"),
    (dict(n_modes=2), "n_modes"),
])
def test_make_params_refusals(kw, msg):
    d = dict(anneal_iterations=2, anneal_iter_decay=0.8)
    d.update(kw)
    T = d.pop("horizon", 10)
    with pytest.raises(ValueError, match=msg):
        make_params(point_mppi(64, T, **d), IsaacGymConfig(), 3, 64, [])


def test_edge_schedules_are_accepted():
    make_params(point_mppi(64, 21, anneal_horizon_decay=0.5), IsaacGymConfig(), 3, 64, [])        # 0.5^20 = 2^-20 exactly
    make_params(point_mppi(64, 10, anneal_iterations=16), IsaacGymConfig(), 3, 64, [])            # N = 16 at unit decays


def test_library_refusals():
    sc, p, _ = point_setup(K=64, T=6)
    be = ao.AnnealOracleBackend()
    be.create(sc.model, p)
    s, r = ao.schedule(2, 0.7, 1.0, 6)
    st = torch.from_numpy(ao.make_state(s, r))
    with pytest.raises(RuntimeError, match="n_iterations"):
        be.set_anneal(st, 17)
    for bad in (dict(mode=2), dict(mode=3), dict(update_cov=1), dict(update_lambda=1), dict(n_modes=2)):
        q = copy.copy(p)
        for k, v in bad.items():
            setattr(q, k, v)
        be.set_params(q)
        with pytest.raises(RuntimeError, match="annealed MPPI excludes"):
            be.set_anneal(st, 2)
    be.set_params(p)
    be.set_anneal(st, 2)
    q = copy.copy(p)
    q.T = 7
    be.set_params(q)                                                           # T changed without a new registration
    U = torch.zeros((7, 3))
    with pytest.raises(RuntimeError, match="registered for T = 6"):
        be.shift(U)
    with pytest.raises(RuntimeError, match="registered for T = 6"):
        be.sample(0, 0, 0, 64, U, None, torch.zeros((7, 3, 64)), torch.zeros((7, 3, 64)))
    be.set_params(p)
    with pytest.raises(RuntimeError, match="noise library"):
        be.sample_library(0, 64, torch.zeros((6, 3)), None, torch.zeros((6, 3, 64)), torch.zeros((6, 3, 64)), None)


def test_defaults_register_nothing_and_keep_the_plan():
    from oracle.backend import OracleBackend
    a = _planner(OracleBackend(), K=64, T=10)
    b = _planner(K=64, T=10, anneal_iterations=1, anneal_iter_decay=1.0, anneal_horizon_decay=1.0)
    assert b.mppi.anneal_state is None and b.mppi.noise_schedule is None and b.mppi.backend.anneal is None and b.mppi.iterations == 1
    for _ in range(3):
        np.testing.assert_array_equal(a.compute_action(Q0, QD0).numpy(), b.compute_action(Q0, QD0).numpy())
    np.testing.assert_array_equal(a.mppi.U.numpy(), b.mppi.U.numpy())


def test_registered_ones_match_the_plain_planner():
    """N = 1 with a schedule of ones registered: the float64 restatement of the annealed K1 / K3 gives the plain plan."""
    from oracle.backend import OracleBackend
    a = _planner(OracleBackend(), K=64, T=10)
    b = _planner(K=64, T=10, anneal_iterations=1, anneal_iter_decay=0.5)
    b.mppi.set_noise_schedule(np.ones((1, 10)))
    np.testing.assert_array_equal(b.mppi.anneal_state.numpy()[1:], np.ones(20, np.float32))
    for _ in range(3):
        np.testing.assert_allclose(a.compute_action(Q0, QD0).numpy(), b.compute_action(Q0, QD0).numpy(), rtol=0, atol=1e-5)
    np.testing.assert_allclose(a.mppi.U.numpy(), b.mppi.U.numpy(), rtol=0, atol=1e-5)


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_n_iteration_plan_equals_hand_sequenced_plain_steps(mode):
    """With c_h = 1, iteration i is a plain MPPI step under Sigma_i = s_i^2 Sigma (noise s_i L z, Sigma_i^-1 = r_i Sigma^-1) keyed by
    plan_idx = i << 32: one annealed plan equals a shift and three such steps sequenced by hand on the plain oracle."""
    from oracle.backend import OracleBackend
    N, ci, T, K = 3, 0.6, 10, 64
    kw = dict(K=K, T=T, mppi_mode=mode, filter_u=False)
    a = _planner(anneal_iterations=N, anneal_iter_decay=ci, **kw)
    b = _planner(OracleBackend(), **kw)
    act = a.compute_action(Q0, QD0).numpy()
    m, be, sim = b.mppi, b.mppi.backend, b.sim
    sim.reset_root_state()
    sim.reset_robot_state(Q0, QD0)
    sim.save_root_state()
    p0 = be.params
    be.shift(m.U, m.plan_ctr)
    s, r = ao.schedule(N, ci, 1.0, T)
    for i in range(N):
        q = copy.deepcopy(p0)
        for e in range(9):
            q.sigma_chol[e] = float(np.float32(np.float64(p0.sigma_chol[e]) * s[i, 0]))
            q.sigma_inv[e] = float(np.float32(np.float64(p0.sigma_inv[e]) * r[i, 0]))
        be.set_params(q)
        be.sample(m.seed, i << 32, 0, K, m.U, None, m.actions, m.noise, m.plan_ctr)
        sim.rollout_all(m.actions)
        x = m.noise if mode == "simple" else m.actions
        be.reduce(m._cost_batched(), x, m.U, m.partial)
        be.finalize(m.partial.view(1, -1), 1, m.U, m._action, m.stats)
    be.set_params(p0)
    np.testing.assert_allclose(act, m._action.numpy(), rtol=0, atol=2e-5)
    np.testing.assert_allclose(a.mppi.U.numpy(), m.U.numpy(), rtol=0, atol=2e-5)
    assert float(a.mppi.anneal_state[0]) == N


def test_counter_is_reset_by_the_shift_and_advanced_by_k4():
    p = _planner(K=64, T=8, **ANNEAL)
    st = p.mppi.anneal_state
    assert float(st[0]) == 0.0
    p.compute_action(Q0, QD0)
    assert float(st[0]) == 3.0
    p.mppi.backend.shift(p.mppi.U, p.mppi.plan_ctr)
    assert float(st[0]) == 0.0
    st[0] = 7.0                                                                # past the last row: iteration N - 1 is read
    np.testing.assert_array_equal(ao.rows(st.numpy(), 3, 8)[0], p.mppi.noise_schedule.numpy()[2])


def test_set_noise_schedule_equals_a_planner_built_with_it():
    a = _planner(K=64, T=8, **ANNEAL)
    b = _planner(K=64, T=8, anneal_iterations=3, anneal_iter_decay=0.8, anneal_horizon_decay=0.95)
    a.mppi.set_noise_schedule(anneal_schedule(3, 0.8, 0.95, 8)[0])
    np.testing.assert_array_equal(a.mppi.anneal_state.numpy(), b.mppi.anneal_state.numpy())
    for _ in range(2):
        np.testing.assert_array_equal(a.compute_action(Q0, QD0).numpy(), b.compute_action(Q0, QD0).numpy())
    with pytest.raises(ValueError, match="shape"):
        a.mppi.set_noise_schedule(np.ones((2, 8)))
    with pytest.raises(ValueError, match="2\\^-20"):
        a.mppi.set_noise_schedule(np.full((3, 8), 1e-7))
    with pytest.raises(RuntimeError, match="annealed MPPI"):
        _planner(K=64, T=8).mppi.set_noise_schedule(np.ones((1, 8)))


def test_keep_u_rebuild_rebuilds_the_schedule_from_the_config():
    p = _planner(K=64, T=8, **ANNEAL)
    p.compute_action(Q0, QD0)
    ref = p.mppi.anneal_state.clone()
    p.mppi.set_noise_schedule(np.full((3, 8), 0.5))
    U = p.mppi.U.clone()
    old_be = p.mppi.backend
    p._build_mppi(keep_U=True)
    np.testing.assert_array_equal(p.mppi.U.numpy(), U.numpy())
    np.testing.assert_array_equal(p.mppi.anneal_state.numpy()[1:], ref.numpy()[1:])        # the config's schedule again
    assert p.mppi.backend.anneal is p.mppi.anneal_state and old_be is p.mppi.backend
    p.cfg.mppi.anneal_iterations, p.cfg.mppi.anneal_iter_decay, p.cfg.mppi.anneal_horizon_decay = 1, 1.0, 1.0
    p.update_mppi_params({"noise_sigma": p.cfg.mppi.noise_sigma})
    assert p.mppi.anneal_state is None and p.mppi.backend.anneal is None                      # off: NULL registered


def test_stepwise_plan_with_a_prior_iterates():
    """rollout_mode stepwise with a prior: every iteration draws, rewrites the prior row, rolls out and updates (K4 counts N)."""
    class Prior:
        def compute_command(self, sim):
            return torch.full((3,), 0.05)
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    cfg = point_cfg(K=64, T=8, use_priors=True, filter_u=False, **ANNEAL)
    p = MPPIisaacPlanner(cfg, PointReachObjective(), prior=Prior(), backend=ao.AnnealOracleBackend())
    assert p.mppi.rollout_mode == "stepwise"
    p.compute_action(Q0, QD0)
    assert float(p.mppi.anneal_state[0]) == 3.0
    np.testing.assert_array_equal(p.mppi.actions.numpy()[:, :, 64 - 2], np.full((8, 3), 0.05, np.float32))   # the last iteration's prior row
    assert np.all(np.isfinite(p.mppi.U.numpy()))


def test_n_worlds_keys_the_annealed_draw_by_control_sample():
    R, K, T = 4, 64, 6
    sc, p, _ = point_setup(K=K, T=T, n_worlds=R, cvar_alpha=0.5, **ANNEAL)
    assert p.n_worlds == R
    be = ao.AnnealOracleBackend()
    be.create(sc.model, p)
    s, r = ao.schedule(3, 0.6, 0.9, T)
    st = torch.from_numpy(ao.make_state(s, r, counter=1.0))
    be.set_anneal(st, 3)
    U = torch.from_numpy((0.1 * np.random.default_rng(3).standard_normal((T, 3))).astype(np.float32))
    a, n = torch.zeros((T, 3, K)), torch.zeros((T, 3, K))
    be.sample(9, 1 << 32, 0, K, U, None, a, n)
    pc = ao.ro.control_params(p)
    ac, _ = ao.sample(sc.model, pc, 9, 1 << 32, U.numpy(), 0, K // R, s[1])
    np.testing.assert_array_equal(a.numpy(), np.repeat(ac, R, axis=-1))
    rng = np.random.default_rng(4)
    cost = rng.random((T, K)).astype(np.float32)
    part = torch.zeros(2 + T * 3)
    be.reduce(torch.from_numpy(cost), n, U, part)
    S, lam = ao.scores(p, 3, cost, n.numpy(), U.numpy(), r[1])
    rho = ao.ro.rho(S, R, int(p.risk_tail))
    w = np.exp(-(rho - rho.min()) / lam)
    np.testing.assert_allclose(part.numpy()[:2], [rho.min(), w.sum()], rtol=1e-6)
    np.testing.assert_allclose(part.numpy()[2:], np.einsum("tjc,c->tj", n.numpy()[:, :, ::R].astype(np.float64), w).reshape(-1), rtol=1e-5, atol=1e-6)
