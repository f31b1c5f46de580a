"""CPU: the float64 reference of multi-modal MPPI (``n_modes`` / ``mode_switch_margin``) -- the parameter block and plan of n_modes = 1,
known answers of the coupling, the bandwidth and the selection, K1 per mode, planner plans on the checker backend, a point robot that
keeps modes on both sides of a bump, and every refusal."""
import numpy as np
import pytest
import torch

import modes_oracle as mo
from mppi_isaac_b200.model.blob import make_params
from mppi_isaac_b200.utils.config_store import IsaacGymConfig
from scenes import point_cfg, point_mppi, point_setup


def test_one_mode_keeps_the_parameter_block_and_the_plan():
    sc, p1, _ = point_setup(K=64, T=10)
    p2 = make_params(point_mppi(64, 10, n_modes=1, mode_switch_margin=0.0), IsaacGymConfig(), sc.nu, 64, [])
    p1b = make_params(point_mppi(64, 10), IsaacGymConfig(), sc.nu, 64, [])
    assert bytes(p1b) == bytes(p2) and p2.n_modes == 0 and p2.mode_samples == 0
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    from oracle.backend import OracleBackend
    a = MPPIisaacPlanner(point_cfg(K=64, T=10), PointReachObjective(), backend=OracleBackend())
    b = MPPIisaacPlanner(point_cfg(K=64, T=10, n_modes=1), PointReachObjective(), backend=mo.ModesOracleBackend())
    for _ in range(2):
        np.testing.assert_array_equal(a.compute_action([0.1, 0.0, 0.0], [0.0] * 3).numpy(), b.compute_action([0.1, 0.0, 0.0], [0.0] * 3).numpy())
    assert b.mppi.modes is None and b.mppi.mode_free_energy is None and b.mppi.active_mode is None


def test_far_modes_take_exactly_their_own_step():
    """Modes 0..2 close together, mode 3 far away: the median bandwidth is small, k_3j = 0, and mode 3 moves by exactly d_3."""
    rng = np.random.default_rng(0)
    T, nu = 5, 2
    U = np.zeros((4, T, nu))
    U[1, 0, 0], U[2, 1, 1] = 0.01, 0.02
    U[3] = 50.0
    d = rng.standard_normal((4, T * nu))
    Un, h = mo.couple(U, d, np.eye(nu))
    assert h > 0 and np.exp(-mo.distances(U, np.eye(nu))[3, 0] / h) == 0.0
    np.testing.assert_array_equal(Un[3], U[3].reshape(-1) + d[3])


def test_two_modes_with_no_step_repel_by_the_known_amount():
    T, nu = 4, 3
    U = np.zeros((2, T, nu))
    U[1] = 0.3
    sinv = np.diag([1.0, 2.0, 4.0])
    Un, h = mo.couple(U, np.zeros((2, T * nu)), sinv)
    D = T * 0.09 * 7.0
    assert np.isclose(h, D / np.log(3))
    k = np.exp(-D / h)                                                         # = 1/3 for M = 2
    assert np.isclose(k, 1.0 / 3.0)
    for i, j in ((0, 1), (1, 0)):
        diff = (U[i] - U[j]).reshape(-1)
        np.testing.assert_allclose(Un[i] - U[i].reshape(-1), (2.0 / h) * k * diff / (1.0 + k), rtol=1e-12, atol=0)


def test_coincident_modes_fall_back_to_the_plain_step():
    U = np.ones((3, 2, 2))
    d = np.arange(12.0).reshape(3, 4)
    Un, h = mo.couple(U, d, np.eye(2))
    assert h == 0.0
    np.testing.assert_allclose(Un, U.reshape(3, -1) + d.mean(0), rtol=1e-15)


def test_median_bandwidth_known_answers():
    D3 = np.array([[0, 1.0, 4.0], [1.0, 0, 9.0], [4.0, 9.0, 0]])
    assert mo.bandwidth(D3) == 4.0 / np.log(4)
    D4 = np.zeros((4, 4))
    for (i, j), v in zip([(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)], [6.0, 1.0, 5.0, 2.0, 4.0, 3.0]):
        D4[i, j] = D4[j, i] = v
    assert mo.bandwidth(D4) == 3.0 / np.log(5)                               # lower median of 1..6
    U = np.array([[[0.0]], [[1.0]], [[3.0]]])
    np.testing.assert_array_equal(mo.distances(U, np.eye(1)), [[0, 1, 9], [1, 0, 4], [9, 4, 0]])


def test_selection_rules():
    inf = np.inf
    assert mo.select(np.array([3.0, 1.0, 2.0]), 0, 0.0) == 1                    # lowest F
    assert mo.select(np.array([2.0, 1.0, 1.0]), 0, 0.0) == 1                    # ties: lowest index
    assert mo.select(np.array([1.5, 1.0, 2.0]), 0, 0.5) == 0                    # p kept inside the margin
    assert mo.select(np.array([1.6, 1.0, 2.0]), 0, 0.5) == 1
    assert mo.select(np.array([inf, inf]), 1, 0.0) == 1                         # every F infinite keeps p
    assert mo.select(np.array([inf, 5.0]), 0, 100.0) == 1                       # F_p = inf never stays
    sc, p, _ = point_setup(K=64, T=4, n_modes=2)
    F = mo.free_energy(p, np.array([1.0, 2.0]), np.array([0.0, 3.0]))
    assert F[0] == inf and np.isclose(F[1], 2.0 - np.float32(0.1) * np.log(3.0 / 32))


def test_k1_columns_are_the_plain_k1_of_their_mode():
    """Oracle K1 of a shard cutting mode 1: the columns of mode m equal the plain K1 with U := U_m."""
    from oracle import oracle as orc
    K, T, M = 128, 6, 4
    sc, p, _ = point_setup(K=K, T=T, n_modes=M)
    U = (0.2 * np.random.default_rng(1).standard_normal((M, T, 3))).astype(np.float32)
    be = mo.ModesOracleBackend()
    be.create(sc.model, p)
    off, Kl = 48, 64
    import copy
    q = copy.copy(p)
    q.K, q.k_offset = Kl, off
    be.set_params(q)
    a, n = torch.zeros((T, 3, Kl)), torch.zeros((T, 3, Kl))
    be.sample(5, 2, off, K, torch.from_numpy(U), None, a, n)
    modes = mo.modes_of(q, off, Kl)
    assert set(modes) == {1, 2, 3}
    for m in range(M):
        pa, pn = orc.sample(sc.model, q, 5, 2, U[m], off, K)
        cols = modes == m
        np.testing.assert_array_equal(a.numpy()[:, :, cols], pa[:, :, cols])
        np.testing.assert_array_equal(n.numpy()[:, :, cols], pn[:, :, cols])


def test_shard_rows_combine_to_the_single_shard_row():
    """Two shards whose boundary cuts mode 1 combine in K4 to what one shard gives."""
    rng = np.random.default_rng(2)
    K, T, M, nu = 128, 5, 4, 3
    sc, p, _ = point_setup(K=K, T=T, n_modes=M, filter_u=False)
    cost = rng.random((T, K)).astype(np.float32)
    x = (0.3 * rng.standard_normal((T, nu, K))).astype(np.float32)
    U = (0.2 * rng.standard_normal((M, T, nu))).astype(np.float32)
    one = mo.reduce(p, nu, cost, x, U, k_offset=0)
    two = np.stack([mo.reduce(p, nu, cost[:, :48], x[:, :, :48], U, k_offset=0), mo.reduce(p, nu, cost[:, 48:], x[:, :, 48:], U, k_offset=48)])
    assert two[1][0] == np.inf and two[1][1] == 0                               # mode 0 has no sample on the second shard
    state = np.concatenate([[0], np.full(M, np.inf), U[0].ravel()]).astype(np.float32)
    r1, r2 = mo.finalize(p, nu, one[None], U, state), mo.finalize(p, nu, two, U, state)
    for a, b in zip(r1, r2):
        np.testing.assert_allclose(a, b, rtol=2e-6, atol=2e-6)
    assert r1[3][0] == np.argmin(r1[3][1:1 + M]) or np.isinf(r1[3][1:1 + M]).all()


@pytest.mark.parametrize("mode", ["batched", "stepwise"])
def test_planner_plans_with_modes_on_the_checker_backend(mode):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    pl = MPPIisaacPlanner(point_cfg(K=128, T=10, n_modes=4, mode_switch_margin=0.5), PointReachObjective(), backend=mo.ModesOracleBackend(),
                          rollout_mode=mode)
    m = pl.mppi
    assert m.modes.shape == (4, 10, 3) and m.partial.numel() == 4 * (2 + 30)
    assert not torch.equal(m.modes[0], m.modes[1])                               # the start breaks the symmetry
    for _ in range(3):
        a = pl.compute_action([0.1, 0.0, 0.0], [0.0] * 3)
    assert torch.isfinite(a).all() and torch.isfinite(m.mode_free_energy).all()
    p = m.active_mode
    np.testing.assert_array_equal(m.mean_action.numpy(), m.modes[p].numpy())
    np.testing.assert_array_equal(a.numpy(), m.modes[p, 0].numpy())


def test_keep_u_rebuild_keeps_the_modes_and_update_params_resets_them():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    pl = MPPIisaacPlanner(point_cfg(K=128, T=10, n_modes=2), PointReachObjective(), backend=mo.ModesOracleBackend())
    pl.compute_action([0.1, 0.0, 0.0], [0.0] * 3)
    U, st = pl.mppi.modes.clone(), pl.mppi.mode_state.clone()
    pl._build_mppi(keep_U=True)
    assert torch.equal(pl.mppi.modes, U) and torch.equal(pl.mppi.mode_state, st)
    pl._build_mppi()
    assert not torch.equal(pl.mppi.modes, U) and pl.mppi.active_mode == 0


class BumpObjective:
    """Point robot from (0, 0) to a goal at (2, 0) with a Gaussian bump of cost centred between them on the start-goal line."""

    def __init__(self, height=40.0, width=0.35):
        self.height, self.width = height, width

    def reset(self):
        pass

    def compute_cost(self, sim):
        r = sim.get_actor_link_by_name(actor_name="point_robot", link_name="base_link")[:, 0:2]
        goal = torch.tensor([2.0, 0.0], dtype=r.dtype, device=r.device)
        bump = torch.tensor([1.0, 0.0], dtype=r.dtype, device=r.device)
        return torch.linalg.norm(r - goal, dim=-1) + self.height * torch.exp(-((r - bump) ** 2).sum(-1) / self.width ** 2)


def nominal_ends(pl, q):
    """y of the end of every mode's nominal rollout (the point robot integrates its velocity command: x_T = x_0 + dt sum_t u_t)."""
    dt = float(pl.cfg.isaacgym.dt)
    return q[1] + dt * pl.mppi.modes[:, :, 1].sum(1).numpy()


def test_point_robot_keeps_modes_on_both_sides_of_a_bump():
    from mppi_isaac_b200 import MPPIisaacPlanner
    pl = MPPIisaacPlanner(point_cfg(K=256, T=20, n_modes=4, seed_val=3), BumpObjective(), backend=mo.ModesOracleBackend())
    q = [0.0, 0.0, 0.0]
    for _ in range(8):
        pl.compute_action(q, [0.0] * 3)
    ends = nominal_ends(pl, q)
    assert (ends > 0.05).any() and (ends < -0.05).any(), ends


@pytest.mark.parametrize("kw, match", [
    (dict(n_modes=0), "n_modes"), (dict(n_modes=17), "n_modes"), (dict(n_modes=3), "multiple"), (dict(n_modes=8, num_samples=128), "at least 32"),
    (dict(n_modes=2, mode_switch_margin=-1.0), "margin"), (dict(n_modes=2, mode_switch_margin=float("inf")), "margin"),
    (dict(n_modes=2, mppi_mode="smooth"), "excludes mppi_mode cem and smooth"),
    (dict(n_modes=2, mppi_mode="cem", noise_sigma=np.eye(3).tolist()), "excludes mppi_mode cem"),
    (dict(n_modes=2, update_cov=True), "update_cov"), (dict(n_modes=2, update_lambda=True), "update_cov and update_lambda"),
])
def test_make_params_refuses(kw, match):
    sc, _, _ = point_setup(K=64, T=6)
    d = dict(num_samples=256)
    d.update(kw)
    K = d.pop("num_samples")
    with pytest.raises(ValueError, match=match):
        make_params(point_mppi(K, 10, **d), IsaacGymConfig(), sc.nu, K, [])


def test_make_params_refuses_worlds_and_the_planner_refuses_a_prior():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    sc, _, _ = point_setup(K=64, T=6)
    with pytest.raises(ValueError, match="n_worlds"):
        make_params(point_mppi(256, 10, n_modes=2, n_worlds=2), IsaacGymConfig(), sc.nu, 256, [])

    class Prior:
        def compute_command(self, sim):
            return torch.zeros(3)
    with pytest.raises(ValueError, match="prior"):
        MPPIisaacPlanner(point_cfg(K=128, T=10, n_modes=2, use_priors=True), PointReachObjective(), prior=Prior(), backend=mo.ModesOracleBackend())
