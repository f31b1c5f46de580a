"""CPU: the float64 reference of cross-entropy planning (``mppi_mode: cem``) -- selection, the update's known answers, carry-over,
shard merging -- the planner planning with it on the checker backend, and every refusal of the mode."""
import numpy as np
import pytest
import torch

import cem_oracle as ce
from mppi_isaac_b200.model.blob import MODE_CEM, make_params
from mppi_isaac_b200.utils.config_store import IsaacGymConfig
from scenes import panda_cfg, panda_mppi, panda_setup

Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]


def _params(K=64, T=4, E=10, **kw):
    d = dict(mppi_mode="cem", n_elites=E)
    d.update(kw)
    sc, p, _ = panda_setup(K=K, T=T, **d)
    return sc, p


def _rand_rows(params, nu, rng, K, cost):
    T = params.T
    actions = rng.uniform(-0.2, 0.2, (T, nu, K)).astype(np.float32)
    return actions, ce.elite_row(params, nu, cost, actions, 0)


def test_make_params_sets_the_cem_block():
    _, p = _params(E=10, keep_elites=0.3, elite_momentum=0.25)
    assert p.mode == MODE_CEM and p.n_elites == 10 and p.n_keep == 3 and p.elite_alpha == 0.25
    assert abs(p.gamma - 0.95) < 1e-7                                     # rollout_var_discount, as in halton-spline


def test_selection_ties_go_to_the_lower_index_and_non_finite_is_never_an_elite():
    _, p = _params(K=16, T=1, E=5)
    cost = np.array([[3, 1, 2, 1, np.nan, -np.inf, np.inf, 0, 1, 2, 5, 0, 7, 1, 9, 4]], np.float32)
    actions = np.arange(7 * 16, dtype=np.float32).reshape(1, 7, 16)
    row = ce.elite_row(p, 7, cost, actions, 0)
    idx = row[1:10:2].view(np.uint32)
    np.testing.assert_array_equal(idx, [7, 11, 1, 3, 8])
    np.testing.assert_array_equal(row[0:10:2], [0, 0, 1, 1, 1])
    np.testing.assert_array_equal(row[10:17], actions[0, :, 7])
    # with a k_offset the indices are global, the order the same
    row_off = ce.elite_row(p, 7, cost, actions, 1000)
    np.testing.assert_array_equal(row_off[1:10:2].view(np.uint32), idx + 1000)


def test_all_equal_costs_pick_the_first_samples():
    _, p = _params(K=32, T=3, E=10)
    row = ce.elite_row(p, 7, np.ones((3, 32), np.float32), np.zeros((3, 7, 32), np.float32), 0)
    np.testing.assert_array_equal(row[1:20:2].view(np.uint32), np.arange(10))


def test_fewer_than_E_finite_samples_change_nothing():
    sc, p = _params(K=16, T=2, E=10)
    cost = np.full((2, 16), np.nan, np.float32)
    cost[:, :9] = 1.0                                                      # 9 finite samples < E
    rng = np.random.default_rng(0)
    actions, row = _rand_rows(p, 7, rng, 16, cost)
    assert row[2 * 9] == np.inf and row[2 * 9 + 1:2 * 9 + 2].view(np.uint32)[0] == ce.NONE_INDEX
    st = ce.make_state(np.full(7, 0.01), 2, 7, 10)
    U = rng.uniform(-0.1, 0.1, (2, 7)).astype(np.float32)
    Un, act, stats, st2 = ce.finalize(p, 7, row[None], U, st)
    np.testing.assert_array_equal(Un, U)
    np.testing.assert_array_equal(st2, st)
    assert stats[0] == np.float32(1.95) and stats[1] == np.inf                # S = 1 + gamma * 1


@pytest.mark.parametrize("E", [1, 4, 10])
def test_update_known_answers(E):
    sc, p = _params(K=64, T=5, E=E, elite_momentum=1.0)
    rng = np.random.default_rng(E)
    cost = rng.uniform(0, 1, (5, 64)).astype(np.float32)
    actions, row = _rand_rows(p, 7, rng, 64, cost)
    st = ce.make_state(np.full(7, 0.01), 5, 7, E)
    U = rng.uniform(-0.1, 0.1, (5, 7)).astype(np.float32)
    Un, _, _, st1 = ce.finalize(p, 7, row[None], U, st)                     # alpha = 1: U and sigma unchanged
    np.testing.assert_array_equal(Un, U)
    np.testing.assert_array_equal(ce.unpack(st1, 5, 7, E)[3], ce.unpack(st, 5, 7, E)[3])
    assert ce.unpack(st1, 5, 7, E)[1] == 1.0 and ce.unpack(st1, 5, 7, E)[0] == 0.0
    p.elite_alpha = 0.0
    Un, act, stats, st2 = ce.finalize(p, 7, row[None], U, st)
    best = int(np.argmin(ce.scores(p, cost)))
    S = ce.scores(p, cost)
    pick = ce.select(S, np.arange(64), E)
    A = actions[:, :, pick].transpose(2, 0, 1).astype(np.float64)
    if E == 1:                                                             # alpha = 0, E = 1: U is the best sample's actions
        np.testing.assert_array_equal(Un, actions[:, :, best])
        np.testing.assert_array_equal(ce.unpack(st2, 5, 7, E)[3], 0.0)      # one elite: sigma = 0
    At = torch.from_numpy(A)
    np.testing.assert_allclose(Un, At.mean(0).numpy(), rtol=0, atol=1e-7)
    np.testing.assert_allclose(ce.unpack(st2, 5, 7, E)[3], At.std(0, unbiased=False).numpy(), rtol=0, atol=1e-7)
    np.testing.assert_array_equal(ce.unpack(st2, 5, 7, E)[4], A.astype(np.float32))
    np.testing.assert_array_equal(act, Un[0])
    assert stats[0] == np.float32(S[pick[0]]) and stats[1] == np.float32(S[pick[-1]])


def test_identical_elites_give_zero_sigma():
    sc, p = _params(K=16, T=3, E=4, elite_momentum=0.0)
    actions = np.repeat(np.linspace(-0.1, 0.1, 21, dtype=np.float32).reshape(3, 7, 1), 16, axis=2)
    row = ce.elite_row(p, 7, np.zeros((3, 16), np.float32), actions, 0)
    _, _, _, st = ce.finalize(p, 7, row[None], np.zeros((3, 7), np.float32), ce.make_state(np.full(7, 0.01), 3, 7, 4))
    np.testing.assert_array_equal(ce.unpack(st, 3, 7, 4)[3], 0.0)


def test_carried_rows_are_shifted_at_iteration_zero_and_unshifted_later(oracle):
    sc, p = _params(K=32, T=6, E=4, keep_elites=0.5)                      # E_keep = 2: rows 29 and 28
    assert p.n_keep == 2
    rng = np.random.default_rng(3)
    st = ce.make_state(np.full(7, 0.01), 6, 7, 4)
    _, _, _, sig, el = ce.unpack(st, 6, 7, 4)
    el[:] = rng.uniform(-0.1, 0.1, el.shape).astype(np.float32)
    st[1] = 1.0
    U = rng.uniform(-0.05, 0.05, (6, 7)).astype(np.float32)
    z = ce.co.white(sc.model, p, 5, 1, 0, 32)
    Lt = np.eye(6, dtype=np.float32)
    st[0] = 0.0
    a0, n0 = ce.sample(p, 7, U, z, Lt, st, 0, 32)
    for e in range(2):
        np.testing.assert_array_equal(a0[:, :, 29 - e], el[e])              # unshifted: the previous iteration's elites
    st[0] = 1.0
    a1, _ = ce.sample(p, 7, U, z, Lt, st, 0, 32)
    fresh = st.copy()
    fresh[1] = 0.0                                                         # no elites yet: every row an ordinary sample
    a2, _ = ce.sample(p, 7, U, z, Lt, fresh, 0, 32)
    for e in range(2):
        np.testing.assert_array_equal(a1[:5, :, 29 - e], el[e, 1:])          # shifted by one step
        np.testing.assert_array_equal(a1[5, :, 29 - e], a2[5, :, 29 - e])    # the last step is the row's own draw
    np.testing.assert_array_equal(n0, a0 - U[:, :, None])
    np.testing.assert_array_equal(np.delete(a1, [28, 29], axis=2), np.delete(a2, [28, 29], axis=2))
    assert not np.array_equal(a2[:5, :, 29], el[0, 1:])


def test_sigma_sample_restates_the_colored_sampler_on_a_diagonal_sigma():
    """With sigma = sqrt(diag(Sigma)) and no elites the CEM draw is the colored draw of the fixed diagonal Sigma."""
    sc, p = _params(K=64, T=12, E=4, noise_beta=2.0, sampling_method="colored")
    from mppi_isaac_b200.planner.mppi import colored_noise_chol
    Lt = colored_noise_chol(12, 2.0)
    z = ce.co.white(sc.model, p, 9, 2, 0, 64)
    U = np.zeros((12, 7), np.float32)
    a, _ = ce.sample(p, 7, U, z, Lt, ce.make_state(np.full(7, 0.1), 12, 7, 4), 0, 64)
    a_ref, _ = ce.co.colour(p, 7, U, z, Lt, 0, 64)
    np.testing.assert_allclose(a, a_ref, rtol=0, atol=1e-7)


@pytest.mark.parametrize("G", [2, 4, 8])
def test_merging_shard_rows_equals_one_shard(G):
    K, T, E = 256, 3, 10
    sc, p = _params(K=K, T=T, E=E)
    rng = np.random.default_rng(G)
    cost = rng.integers(0, 20, (T, K)).astype(np.float32)                 # many ties
    cost[0, rng.integers(0, K, 9)] = np.nan
    actions = rng.uniform(-0.2, 0.2, (T, 7, K)).astype(np.float32)
    one = ce.elite_row(p, 7, cost, actions, 0)
    bounds_ = np.linspace(0, K, G + 1).astype(int)
    rows = np.stack([ce.elite_row(p, 7, cost[:, a:b], actions[:, :, a:b], a) for a, b in zip(bounds_[:-1], bounds_[1:])])
    st = ce.make_state(np.full(7, 0.01), T, 7, E)
    U = np.zeros((T, 7), np.float32)
    r1 = ce.finalize(p, 7, one[None], U, st)
    rG = ce.finalize(p, 7, rows, U, st)
    for x, y in zip(r1, rG):
        np.testing.assert_array_equal(x, y)


def test_shift_resets_sigma_and_sets_the_carry_offset():
    sc, p = _params(K=16, T=4, E=2)
    st = ce.make_state(np.full(7, 0.01), 4, 7, 2)
    st[2 + 2:2 + 2 + 28] = 5.0
    U = np.arange(28, dtype=np.float32).reshape(4, 7)
    Un, st2 = ce.shift(p, 7, U, st)
    np.testing.assert_array_equal(Un[:3], U[1:])
    np.testing.assert_array_equal(ce.unpack(st2, 4, 7, 2)[3], np.float32(np.sqrt(0.1)))
    assert st2[0] == 1.0


@pytest.mark.parametrize("sampling", ["random", "colored"])
def test_planner_plans_with_cem_on_the_checker_backend(sampling):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    cfg = panda_cfg(K=64, T=12, device="cpu", mppi_mode="cem", sampling_method=sampling, n_elites=8, keep_elites=0.25, cem_iterations=2)
    pl = MPPIisaacPlanner(cfg, PandaReachObjective(), backend=ce.CemOracleBackend())
    m = pl.mppi
    assert m.cem and m.cem_iterations == 2 and m.current_lambda is None
    assert m.cov_action.shape == (12, 7) and m.elites.shape == (8, 12, 7) and m.elite_costs.shape == (8,)
    np.testing.assert_allclose(m.cov_action.numpy(), np.sqrt(0.1), rtol=1e-7)
    for it in range(3):
        a = pl.compute_action(Q0, [0.0] * 7)
        assert torch.isfinite(a).all()
        assert m.dist[1] == 1.0 and m.dist[0] == 0.0                       # elites valid, last update unshifted
        S = m.elite_costs.numpy()
        assert np.all(np.diff(S) >= 0) and m.stats[0] == S[0] and m.stats[1] == S[-1]
        assert np.all(m.cov_action.numpy() < np.sqrt(0.1) + 1e-6)
        assert int(m.plan_ctr[0]) == it + 1


def test_planner_stepwise_plans_with_cem():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    cfg = panda_cfg(K=32, T=9, device="cpu", mppi_mode="cem", sampling_method="random", n_elites=4, cem_iterations=2, filter_u=True)
    pl = MPPIisaacPlanner(cfg, PandaReachObjective(), backend=ce.CemOracleBackend(), rollout_mode="stepwise")
    a = pl.compute_action(Q0, [0.0] * 7)
    assert torch.isfinite(a).all() and pl.mppi.dist[1] == 1.0


@pytest.mark.parametrize("kw, match", [
    (dict(n_elites=0), "n_elites"), (dict(n_elites=129), "n_elites"), (dict(n_elites=60, keep_elites=0.1), "num_samples"),
    (dict(elite_momentum=-0.1), "elite_momentum"), (dict(elite_momentum=1.5), "elite_momentum"),
    (dict(keep_elites=-0.5), "keep_elites"), (dict(keep_elites=1.01), "keep_elites"), (dict(cem_iterations=0), "cem_iterations"),
    (dict(update_cov=True), "update_cov"), (dict(update_lambda=True), "update_cov"), (dict(sampling_method="halton"), "halton"),
    (dict(noise_sigma=(0.1 * np.eye(7) + 0.01).tolist()), "diagonal"),
])
def test_make_params_refuses(kw, match):
    sc, _, _ = panda_setup(K=4, T=12)
    with pytest.raises(ValueError, match=match):
        make_params(panda_mppi(64, 12, mode="cem", **kw), IsaacGymConfig(), sc.nu, 64, [])


def test_make_params_refuses_long_horizons_and_accepts_the_edges():
    sc, _, _ = panda_setup(K=4, T=12)
    with pytest.raises(ValueError, match="horizon"):
        make_params(panda_mppi(64, 80, mode="cem"), IsaacGymConfig(), sc.nu, 64, [])               # T*nu = 560 > 512
    make_params(panda_mppi(64, 73, mode="cem"), IsaacGymConfig(), sc.nu, 64, [])                   # T*nu = 511
    make_params(panda_mppi(12, 12, mode="cem", n_elites=10, keep_elites=0.0), IsaacGymConfig(), sc.nu, 12, [])   # E + 0 + 2 = K
    make_params(panda_mppi(256, 12, mode="cem", n_elites=128, keep_elites=0.9, elite_momentum=1.0), IsaacGymConfig(), sc.nu, 256, [])
