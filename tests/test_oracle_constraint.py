"""Constrained MPPI (``constraint_mode: feasible_first``) without a GPU: the float64 row on hand-made cases (the tolerance boundary,
negative margins, NaN and +inf), all-feasible plans equal to the plain planner, violation-only plans equal to the plain planner on the
violation cost, every refusal, the traced observation plan and a stepwise plan with a prior."""
import math

import numpy as np
import pytest
import torch

import constraint_oracle as cn
from mppi_isaac_b200 import MPPIisaacPlanner
from mppi_isaac_b200.backend import shard_row_floats
from mppi_isaac_b200.model.blob import make_params
from mppi_isaac_b200.objectives import PandaReachKeepOutObjective, PandaReachObjective, PointReachObjective
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from knots_oracle import KnotsOracleBackend as OracleBackend   # the checker backend with every sampler of the plain rule
from scenes import panda_cfg, point_cfg

Q0, QD0 = [0.1, 0.0, 0.0], [0.0] * 3
FF = dict(constraint_mode="feasible_first")


def params(nu=2, T=4, K=8, **kw):
    d = dict(num_samples=K, horizon=T, mppi_mode="halton-spline", sampling_method="random", noise_sigma=np.eye(nu).tolist(), u_min=[-1.0],
             u_max=[1.0], filter_u=False, rollout_var_discount=1.0, lambda_=0.5)
    d.update(kw)
    return make_params(MPPIConfig(**d), IsaacGymConfig(), nu, K, [])


class PointKeepOut(PointReachObjective):
    """Point reach with a margin `fn(p, kg)` of the robot position p (N, 3) and the global sample index kg of each row."""

    def __init__(self, fn, **kw):
        super().__init__(**kw)
        self.fn = fn

    def compute_constraint(self, sim):
        r = sim.get_actor_link_by_name(actor_name=self.actor, link_name=self.link)
        kg = sim.k_offset + torch.arange(r.shape[0]) % sim.num_envs
        return self.fn(r[:, 0:3], kg).to(torch.float32)


class ViolationCost(PointKeepOut):
    """The violation max(g, 0) of PointKeepOut as a cost, for the plain planner."""

    def compute_cost(self, sim):
        return torch.clamp_min(self.compute_constraint(sim), 0.0)


def ring(p, kg):
    return 0.05 - torch.linalg.norm(p[:, 0:2] - torch.tensor([0.3, 0.0]), dim=1)


def _pair(obj_a, obj_b, plans=4, kw_b=None, **kw):
    a = MPPIisaacPlanner(point_cfg(**kw), obj_a, backend=OracleBackend())
    b = MPPIisaacPlanner(point_cfg(**kw, **(kw_b or {})), obj_b, backend=cn.ConstraintOracleBackend())
    out = []
    for _ in range(plans):
        out.append((a.compute_action(Q0, QD0).numpy().copy(), b.compute_action(Q0, QD0).numpy().copy()))
        np.testing.assert_allclose(b.mppi.U.numpy(), a.mppi.U.numpy(), rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.mppi.stats.numpy(), a.mppi.stats.numpy(), rtol=2e-5, atol=2e-5)
    for x, y in out:
        np.testing.assert_allclose(y, x, rtol=0, atol=2e-5)
    return a, b


# ---- the float64 row ----------------------------------------------------------------------------------------------------

def test_row_tolerance_boundary_negative_margins_and_non_finite():
    p = params(nu=1, T=2, K=6, constraint_tol=0.25, **FF)
    cost = np.array([[1.0, 2.0, 3.0, 4.0, 5.0, 6.0], [0.0] * 6])
    x = np.arange(12, dtype=np.float64).reshape(2, 1, 6) * 0.1
    U = np.zeros((2, 1))
    g = np.array([[0.25, -5.0, 0.1, np.nan, np.inf, 0.2],
                  [0.0, -1.0, 0.2, 0.0, 0.0, -0.1]])
    r = cn.row(p, 1, cost, x, U, g)
    # V = 0.25 (feasible at the boundary), 0 (negative margins count 0), 0.3, NaN, inf, 0.2: samples 0, 1 and 5 are feasible
    assert r[-2] == 3 and r[-1] == 0.0
    S = cost.sum(0)
    w = np.exp(-(S - 1.0) / 0.5) * np.array([1, 1, 0, 0, 0, 1])
    np.testing.assert_allclose(r[:2], [1.0, w.sum()])
    np.testing.assert_allclose(r[2:4], x.reshape(2, 6) @ w)
    # one ulp below the boundary: sample 0 becomes infeasible
    p.constraint_tol = float(np.nextafter(np.float32(0.25), np.float32(0)))
    assert cn.row(p, 1, cost, x, U, g)[-2] == 2


def test_row_without_a_feasible_sample_weights_the_violations_and_skips_invalid_ones():
    p = params(nu=1, T=2, K=4, constraint_lambda=2.0, **FF)
    cost = np.array([[1.0, np.nan, 3.0, 4.0], [0.0] * 4])
    x = np.ones((2, 1, 4))
    g = np.array([[1.0, 0.1, 0.5, np.nan], [1.0, 0.0, 0.0, 0.0]])
    r = cn.row(p, 1, cost, x, np.zeros((2, 1)), g)
    # valid: 0 (V = 2) and 2 (V = 0.5); 1 has a NaN cost, 3 a NaN margin
    w = np.exp(-(np.array([2.0, 0.5]) - 0.5) / 2.0)
    assert r[-2] == 0 and r[-1] == 0.5 and r[0] == 0.5
    np.testing.assert_allclose(r[1], w.sum())
    none = cn.row(p, 1, cost, x, np.zeros((2, 1)), np.full((2, 4), np.nan))
    assert none[0] == np.inf and none[1] == 0.0 and none[-1] == np.inf and none[-2] == 0


def test_merge_is_feasibility_first_and_order_free():
    p = params(**FF)
    feas = np.array([5.0, 1.0, 1.0, 2.0, 3, 0.0])
    viol = np.array([0.1, 7.0, 7.0, 7.0, 0, 0.1])
    empty = np.array([np.inf, 0.0, 0.0, 0.0, 0, np.inf])
    for rows in ([feas, viol, empty], [viol, empty, feas], [empty, feas, viol]):
        b, e, W, n, vmin = cn.merge(p, np.stack(rows))
        assert (b, e, n, vmin) == (5.0, 1.0, 3, 0.0)
        np.testing.assert_array_equal(W, [1.0, 2.0])
    b, e, W, n, vmin = cn.merge(p, np.stack([viol, empty]))
    assert (b, e, n, vmin) == (0.1, 7.0, 0, 0.1)


def test_row_floats_and_block():
    p = params(nu=3, T=5, **FF)
    assert shard_row_floats(p, 3) == 4 + 15
    assert p.constraint_mode == 1 and p.constraint_tol == 0.0 and p.constraint_lambda == np.float32(0.5)
    off = params(nu=3, T=5)
    assert shard_row_floats(off, 3) == 2 + 15
    assert (off.constraint_mode, off.constraint_tol, off.constraint_lambda) == (0, 0.0, 0.0)


# ---- planner-level ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("method", ["random", "halton", "colored"])
def test_all_feasible_plans_are_the_plain_plans(mode, method):
    kw = dict(K=128, T=12, mppi_mode=mode, sampling_method=method, sample_null_action=True, filter_u=mode == "simple")
    a, b = _pair(PointReachObjective(), PointKeepOut(lambda p, kg: -1.0 - p[:, 0].abs()), kw_b=FF, **kw)
    assert b.mppi.feasible_samples == 128 and float(b.mppi.min_violation) == 0.0
    assert a.mppi.feasible_samples is None and a.mppi.violation is None and a.mppi.min_violation is None
    assert tuple(b.mppi.violation.shape) == (12, 128)


def test_no_feasible_sample_is_the_plain_planner_on_the_violation_cost():
    """MEAN mode with gamma = 1: the fallback weights exp(-(V - b)/lambda_c), the plain planner on cost := c with lambda := lambda_c."""
    fn = lambda p, kg: 0.5 + p[:, 0] ** 2 + 0.1 * p[:, 1]   # noqa: E731
    kw = dict(K=128, T=12, mppi_mode="halton-spline", sampling_method="random", rollout_var_discount=1.0, filter_u=False)
    b2 = MPPIisaacPlanner(point_cfg(**kw, constraint_lambda=0.3, **FF), PointKeepOut(fn), backend=cn.ConstraintOracleBackend())
    a2 = MPPIisaacPlanner(point_cfg(**kw, lambda_=0.3), ViolationCost(fn), backend=OracleBackend())
    for _ in range(3):
        np.testing.assert_allclose(b2.compute_action(Q0, QD0).numpy(), a2.compute_action(Q0, QD0).numpy(), rtol=0, atol=2e-5)
        np.testing.assert_allclose(b2.mppi.U.numpy(), a2.mppi.U.numpy(), rtol=0, atol=2e-5)
        assert b2.mppi.feasible_samples == 0 and float(b2.mppi.min_violation) > 0.0
        np.testing.assert_allclose(b2.mppi.stats.numpy(), a2.mppi.stats.numpy(), rtol=1e-5)


def test_mixed_plans_move_towards_the_feasible_samples():
    """Samples whose first move goes left of x = 0.1 are infeasible: the update keeps only the others."""
    kw = dict(K=128, T=12, mppi_mode="simple", sampling_method="random", filter_u=False)
    p = MPPIisaacPlanner(point_cfg(**kw, **FF), PointKeepOut(lambda q, kg: 0.1 - q[:, 0]), backend=cn.ConstraintOracleBackend())
    p.compute_action(Q0, QD0)
    n = p.mppi.feasible_samples
    assert 0 < n < 128
    g = p.mppi.violation.numpy()
    V = np.where(g <= 0, 0.0, g).sum(0)
    assert n == int((V <= 0).sum()) and float(p.mppi.min_violation) == 0.0


def test_stepwise_plan_with_a_prior_all_feasible_is_the_plain_plan():
    class Prior:
        def compute_command(self, sim):
            return torch.tensor([0.2, -0.1, 0.0])
    kw = dict(K=64, T=10, mppi_mode="simple", sampling_method="random", use_priors=True, filter_u=False)
    a = MPPIisaacPlanner(point_cfg(**kw), PointReachObjective(), Prior(), backend=OracleBackend())
    b = MPPIisaacPlanner(point_cfg(**kw, **FF), PointKeepOut(lambda q, kg: -torch.ones(q.shape[0])), Prior(), backend=cn.ConstraintOracleBackend())
    assert a.mppi.rollout_mode == b.mppi.rollout_mode == "stepwise"
    for _ in range(3):
        np.testing.assert_allclose(b.compute_action(Q0, QD0).numpy(), a.compute_action(Q0, QD0).numpy(), rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.mppi.U.numpy(), a.mppi.U.numpy(), rtol=0, atol=2e-5)
    assert b.mppi.feasible_samples == 64


def test_stepwise_constraint_is_written_per_step():
    kw = dict(K=64, T=10, mppi_mode="simple", sampling_method="random", filter_u=False)
    p = MPPIisaacPlanner(point_cfg(**kw, **FF), PointKeepOut(ring), backend=cn.ConstraintOracleBackend(), rollout_mode="stepwise")
    q = MPPIisaacPlanner(point_cfg(**kw, **FF), PointKeepOut(ring), backend=cn.ConstraintOracleBackend(), rollout_mode="batched")
    for _ in range(2):
        np.testing.assert_allclose(p.compute_action(Q0, QD0).numpy(), q.compute_action(Q0, QD0).numpy(), rtol=0, atol=2e-5)
        np.testing.assert_allclose(p.mppi.violation.numpy(), q.mppi.violation.numpy(), rtol=0, atol=1e-6)


def test_the_constraint_is_traced_into_the_observation_plan():
    class Link7KeepOut(PandaReachObjective):
        def compute_constraint(self, sim):
            return 0.05 - sim.get_actor_link_by_name("panda", "panda_link7")[:, 2]
    cfg = panda_cfg(K=32, T=9, sampling_method="random", filter_u=False, **FF)
    p = MPPIisaacPlanner(cfg, Link7KeepOut(), backend=cn.ConstraintOracleBackend())
    plain = MPPIisaacPlanner(panda_cfg(K=32, T=9, sampling_method="random", filter_u=False), PandaReachObjective(), backend=OracleBackend())
    extra = set(p.sim._obs_items) - set(plain.sim._obs_items)
    assert len(extra) == 1
    p.compute_action([0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0], [0.0] * 7)
    assert tuple(p.mppi.violation.shape) == (9, 32)
    p.update_objective(PandaReachKeepOutObjective(centre=(0.4, 0.0, 0.6), radius=0.05))
    p.compute_action([0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0], [0.0] * 7)
    assert 0 <= p.mppi.feasible_samples <= 32


# ---- refusals -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kw, msg", [
    (dict(update_cov=True), "update_cov"),
    (dict(update_lambda=True), "update_lambda"),
    (dict(mppi_mode="cem"), "cem"),
    (dict(mppi_mode="smooth"), "smooth"),
    (dict(n_modes=2), "n_modes"),
    (dict(n_worlds=2), "n_worlds"),
    (dict(anneal_iterations=2), "annealed"),
    (dict(control_knots=3), "control_knots"),
    (dict(constraint_mode="hard"), "unknown constraint_mode"),
    (dict(constraint_tol=-1.0), "constraint_tol"),
    (dict(constraint_tol=math.inf), "constraint_tol"),
    (dict(constraint_lambda=0.0), "constraint_lambda"),
    (dict(constraint_lambda=math.nan), "constraint_lambda"),
])
def test_make_params_refuses(kw, msg):
    d = dict(FF)
    d.update(kw)
    with pytest.raises(ValueError, match=msg):
        params(nu=2, T=10, K=64, **d)


def test_objective_without_compute_constraint_is_refused():
    with pytest.raises(ValueError, match="compute_constraint"):
        MPPIisaacPlanner(point_cfg(K=64, T=10, **FF), PointReachObjective(), backend=cn.ConstraintOracleBackend())
    p = MPPIisaacPlanner(point_cfg(K=64, T=10, **FF), PointKeepOut(ring), backend=cn.ConstraintOracleBackend())
    with pytest.raises(ValueError, match="compute_constraint"):
        p.update_objective(PointReachObjective())


def test_backend_without_set_constraint_is_refused():
    with pytest.raises(ValueError, match="set_constraint"):
        MPPIisaacPlanner(point_cfg(K=64, T=10, **FF), PointKeepOut(ring), backend=OracleBackend())


def test_oracle_backend_refuses_a_mismatched_registration():
    p = MPPIisaacPlanner(point_cfg(K=64, T=10, **FF), PointKeepOut(ring), backend=cn.ConstraintOracleBackend())
    be = p.sim.backend
    viol, cstate = be.constraint[0], be.constraint[1]
    be.constraint = (viol, cstate, 9, 64)
    with pytest.raises(RuntimeError, match="registered"):
        p.compute_action(Q0, QD0)
