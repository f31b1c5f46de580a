"""CPU: the float64 reference of risk-aware MPPI (``n_worlds`` / ``cvar_alpha``) -- known answers of the CVaR score, a cost set where
the mean and the worst case disagree, the world mapping of K2 on a randomised contact scene, the planner planning with it on the
checker backend, and every refusal."""
import copy

import numpy as np
import pytest
import torch

import risk_oracle as ro
from mppi_isaac_b200.model.blob import make_params, risk_tail
from mppi_isaac_b200.planner.mppi import shard_samples
from mppi_isaac_b200.utils.config_store import IsaacGymConfig
from scenes import boxer_cfg, boxer_setup, panda_cfg, panda_mppi, panda_setup

INF = np.inf


def test_rho_known_answers():
    S = np.array([1.0, 4.0, 2.0, 3.0])
    assert ro.rho(S, 4, 4)[0] == 2.5                                          # alpha = 1: the mean
    assert ro.rho(S, 4, 1)[0] == 4.0                                          # alpha <= 1/R: the worst case
    assert ro.rho(S, 4, 2)[0] == 3.5                                          # the two worst
    assert ro.rho(np.array([2.0, 2.0, 2.0, 1.0]), 4, 3)[0] == 2.0             # ties
    assert ro.rho(np.array([1.0, np.nan, 0.0, 0.0]), 4, 1)[0] == INF          # one non-finite world invalidates the control
    assert ro.rho(np.array([1.0, INF, -INF, 0.0]), 4, 4)[0] == INF            # several
    np.testing.assert_array_equal(ro.rho(np.array([1.0, 2.0, 5.0, 7.0]), 2, 1), [2.0, 7.0])
    np.testing.assert_array_equal(ro.rho_f32(np.array([1.0, 2.0, 5.0, 7.0], np.float32), 2, 2), np.float32([1.5, 6.0]))


def test_risk_tail_rounds_up_in_float64():
    assert [risk_tail(8, a) for a in (1.0, 0.5, 0.25, 0.2, 0.125, 0.01)] == [8, 4, 2, 2, 1, 1]
    assert risk_tail(32, 1 / 32) == 1 and risk_tail(2, 0.75) == 2


def _row(cost, R, alpha, lam=1.0):
    _, p, _ = panda_setup(K=cost.shape[1], T=1, n_worlds=R, cvar_alpha=alpha, lambda_=lam, sample_null_action=False)
    x = np.zeros((1, 7, cost.shape[1]), np.float32)
    x[0, 0] = np.repeat(np.arange(cost.shape[1] // R, dtype=np.float32), R)    # x of control c = c
    return ro.reduce(p, 7, cost, x, np.zeros((1, 7), np.float32))


def test_mean_and_worst_case_pick_different_controls():
    """Control A has the lower mean, B the lower worst case: alpha = 1 prefers A, alpha = 1/R prefers B."""
    R = 4
    A = [0.0, 0.0, 0.0, 10.0]        # mean 2.5, worst 10
    B = [3.0, 3.0, 3.0, 3.0]         # mean 3,   worst 3
    cost = np.array([A + B], np.float32)
    r1, rw = _row(cost, R, 1.0, lam=0.01), _row(cost, R, 1.0 / R, lam=0.01)
    assert r1[0] == 2.5 and r1[2] / r1[1] < 0.01                              # beta = rho_A, the weight sits on A (x = 0)
    assert rw[0] == 3.0 and rw[2] / rw[1] > 0.99                              # beta = rho_B, the weight sits on B (x = 1)


def test_row_is_a_control_level_mppi_row():
    """With R worlds of identical cost the row equals the plain row of the Kc control samples."""
    rng = np.random.default_rng(1)
    Kc, R, T = 16, 8, 3
    _, p, _ = panda_setup(K=Kc * R, T=T, n_worlds=R, cvar_alpha=0.3)
    cost = np.repeat(rng.random((T, Kc)).astype(np.float32), R, axis=1)
    x = np.repeat((0.1 * rng.standard_normal((T, 7, Kc))).astype(np.float32), R, axis=2)
    U = (0.05 * rng.standard_normal((T, 7))).astype(np.float32)
    row = ro.reduce(p, 7, cost, x, U)
    pc = ro.control_params(p)
    pc.n_worlds, pc.risk_tail = 1, 1
    ref = ro.reduce(pc, 7, cost[:, ::R], x[:, :, ::R], U)
    np.testing.assert_allclose(row, ref, rtol=1e-6, atol=0)


def test_k2_keys_the_randomisation_by_world():
    """All controls equal on a randomised contact scene: samples k and k' end in the same state iff k % R == k' % R, and sample k is the
    plain (R = 1) rollout of sample k % R."""
    from oracle import oracle as orc
    K, T, R = 16, 4, 4
    sc, p, s0 = boxer_setup(K=K, T=T, noise=True)
    pr = copy.deepcopy(p)
    pr.n_worlds, pr.risk_tail = R, 1
    be = ro.RiskOracleBackend()
    be.create(sc.model, pr)
    a = np.zeros((T, 2, K), np.float32)
    a[:, 0] = 0.8
    NS = be.state_size()
    st = torch.zeros((NS, K))
    obs = torch.zeros((be.obs_size(), T, K))
    be.rollout(torch.from_numpy(s0), st, torch.from_numpy(a), 0, T, obs, root0=torch.from_numpy(sc.root_state0))
    o = obs.numpy()
    for k in range(K):
        for k2 in range(K):
            assert np.array_equal(o[..., k], o[..., k2]) == (k % R == k2 % R)
    p1 = copy.deepcopy(p)
    p1.K = R
    _, o1 = orc.rollout(sc.model, p1, s0, a[:, :, :R], root0=sc.root_state0)
    np.testing.assert_array_equal(o[..., :R], o1)
    np.testing.assert_array_equal(o[..., R:2 * R], o1)


def test_planner_plans_over_worlds_on_the_checker_backend():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PushObjective
    pl = MPPIisaacPlanner(boxer_cfg(K=64, T=10, n_worlds=4, cvar_alpha=0.5, sampling_method="random", mppi_mode="simple"),
                          PushObjective(robot="boxer", link="ee_link"), backend=ro.RiskOracleBackend())
    assert pl.mppi.n_worlds == 4 and pl.mppi.control_samples == 16 and pl.mppi.backend.params.risk_tail == 2
    for _ in range(2):
        a = pl.compute_action([0.0, 2.5, 0.0], [0.0] * 3)
    assert torch.isfinite(a).all()
    act = pl.mppi.actions.numpy()
    np.testing.assert_array_equal(act, np.repeat(act[:, :, ::4], 4, axis=2))     # the R rollouts of a control carry its actions
    assert (act[:, :, -4:] == 0).all()                                         # the null control is the last group


@pytest.mark.parametrize("kw, match", [
    (dict(n_worlds=3), "power of two"), (dict(n_worlds=64), "power of two"), (dict(n_worlds=0), "power of two"),
    (dict(n_worlds=4, cvar_alpha=0.0), "cvar_alpha"), (dict(n_worlds=4, cvar_alpha=1.5), "cvar_alpha"),
    (dict(n_worlds=4, cvar_alpha=float("nan")), "cvar_alpha"), (dict(n_worlds=32), "at least two control samples"),
    (dict(n_worlds=4, mppi_mode="cem"), "excludes mppi_mode cem"), (dict(n_worlds=4, mppi_mode="smooth"), "excludes mppi_mode cem and smooth"),
    (dict(n_worlds=4, update_cov=True, cov_type="horizon"), "horizon"),
])
def test_make_params_refuses(kw, match):
    sc, _, _ = panda_setup(K=4, T=6)
    with pytest.raises(ValueError, match=match):
        make_params(panda_mppi(32, 6, **kw), IsaacGymConfig(), sc.nu, 32, [])


def test_make_params_refuses_a_split_group_and_keeps_r1_unchanged():
    sc, _, _ = panda_setup(K=4, T=6)
    with pytest.raises(ValueError, match="whole groups"):
        make_params(panda_mppi(64, 6, n_worlds=8), IsaacGymConfig(), sc.nu, 28, [])
    with pytest.raises(ValueError, match="multiple"):
        make_params(panda_mppi(36, 6, n_worlds=8), IsaacGymConfig(), sc.nu, 36, [])
    p1 = make_params(panda_mppi(64, 6), IsaacGymConfig(), sc.nu, 64, [])
    p2 = make_params(panda_mppi(64, 6, n_worlds=1, cvar_alpha=0.1), IsaacGymConfig(), sc.nu, 64, [])
    assert bytes(p1) == bytes(p2) and p1.n_worlds == 0 and p1.risk_tail == 0


def test_planner_refuses_a_prior_and_an_unrandomised_scene():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective, PushObjective
    from oracle.backend import OracleBackend
    with pytest.raises(ValueError, match="identical copies"):
        MPPIisaacPlanner(panda_cfg(K=64, T=10, n_worlds=4), PandaReachObjective(), backend=OracleBackend())

    class Prior:
        def compute_command(self, sim):
            return torch.zeros(2)
    with pytest.raises(ValueError, match="prior"):
        MPPIisaacPlanner(boxer_cfg(K=64, T=10, n_worlds=4, use_priors=True), PushObjective(robot="boxer", link="ee_link"), prior=Prior(),
                         backend=ro.RiskOracleBackend())


def test_shard_samples_unit():
    assert shard_samples(64, 1, 2) == (32, 32)
    assert shard_samples(48, 0, 4, unit=8) == (16, 0) and shard_samples(48, 3, 4, unit=8) == (8, 40)
    with pytest.raises(ValueError, match="multiple of 8"):
        shard_samples(36, 0, 2, unit=8)
    with pytest.raises(ValueError, match="too small"):
        shard_samples(16, 3, 4, unit=8)
