"""Spline MPPI (``control_knots`` / ``spline_degree``) without a GPU: the basis against scipy and its listed properties, the identity at
d = 1, P = T, the exact shift of linear sequences, the table layout, every refusal of make_params, and the unchanged parameter block at
control_knots = 0."""
import ctypes as C

import numpy as np
import pytest
from scipy.interpolate import BSpline

import knots_oracle as ko
from mppi_isaac_b200.backend import shard_row_floats, spline_table_floats
from mppi_isaac_b200.model.blob import make_params, spline_basis, spline_initial_knots, spline_knot_vector, spline_table
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig

SHAPES = [(2, 2, 1), (30, 8, 1), (30, 8, 2), (30, 8, 3), (30, 30, 1), (256, 256, 1), (64, 32, 3), (256, 4, 3), (10, 7, 2), (31, 9, 3)]


def params(nu=2, T=30, **kw):
    d = dict(num_samples=64, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=np.eye(nu).tolist(), u_min=[-1.0],
             u_max=[1.0], filter_u=False)
    d.update(kw)
    return make_params(MPPIConfig(**d), IsaacGymConfig(), nu, 64, [])


@pytest.mark.parametrize("T, P, d", SHAPES)
def test_basis_matches_scipy_and_its_properties(T, P, d):
    B, S, xi = spline_basis(T, P, d)
    u = spline_knot_vector(T, P, d)
    ref = BSpline.design_matrix(np.arange(T, dtype=np.float64), u, d).toarray()
    np.testing.assert_allclose(B, ref, rtol=0, atol=1e-13)
    assert B.shape == (T, P) and np.all(B >= 0)
    np.testing.assert_allclose(B.sum(1), 1.0, rtol=0, atol=1e-13)
    assert np.array_equal(B[0], np.eye(P)[0]) and np.array_equal(B[-1], np.eye(P)[-1])
    assert np.all(np.count_nonzero(B, axis=1) <= d + 1)
    assert xi[0] == 0.0 and xi[-1] == T - 1
    for p in range(P):
        if not np.isnan(S[p]).any():
            assert np.all(S[p] >= 0) and abs(S[p].sum() - 1.0) < 1e-13


def test_identity_at_degree_one_and_p_equal_t():
    for T in (2, 9, 30, 256):
        B, S, xi = spline_basis(T, T, 1)
        assert np.array_equal(B, np.eye(T))
        assert np.array_equal(xi, np.arange(T, dtype=np.float64))
        assert np.array_equal(S[:-1], np.eye(T)[1:]) and np.isnan(S[-1]).all()
        tab = spline_table(T, T, 1, 1)
        rows = tab[:(2 * T) * 4].reshape(2 * T, 4)
        assert np.array_equal(rows[:T, :3], np.stack([np.arange(T), np.ones(T), np.ones(T)], 1))
        assert np.array_equal(rows[T:2 * T - 1, :3], np.stack([np.arange(1, T), np.ones(T - 1), np.ones(T - 1)], 1))
        assert rows[2 * T - 1, 1] == 0.0


@pytest.mark.parametrize("T, P, d", [s for s in SHAPES if s[1] > s[2] + 0])
def test_shift_reproduces_linear_sequences(T, P, d):
    """theta_p = a + b xi_p is the spline a + b t; the shifted spline a + b (t + 1) has knots a + b (xi_p + 1), wherever a successor exists."""
    _, S, xi = spline_basis(T, P, d)
    th = 0.3 + 0.05 * xi
    for p in range(P):
        if not np.isnan(S[p]).any():
            assert abs(S[p] @ th - (0.3 + 0.05 * (xi[p] + 1.0))) < 1e-12


def test_table_layout_and_initial_knots():
    T, P, d, nu = 30, 8, 3, 2
    th = np.random.default_rng(0).standard_normal((P, nu))
    tab = spline_table(T, P, d, nu, th)
    assert tab.size == spline_table_floats(T, P, d, nu) and tab.dtype == np.float32
    B, S, _ = spline_basis(T, P, d)
    rows = tab[:(T + P) * (d + 3)].reshape(T + P, d + 3)
    for r, w in enumerate(list(B) + list(S)):
        if np.isnan(w).any():
            assert rows[r, 1] == 0
            continue
        f, n = int(rows[r, 0]), int(rows[r, 1])
        full = np.zeros(P)
        full[f:f + n] = rows[r, 2:2 + n]
        np.testing.assert_array_equal(full, w.astype(np.float32))
    np.testing.assert_array_equal(tab[-T * nu:], (B @ th).astype(np.float32).reshape(-1))
    U = np.stack([np.linspace(-1, 1, T), np.full(T, 0.25)], 1)
    k = spline_initial_knots(T, P, d, U)
    _, _, xi = spline_basis(T, P, d)
    np.testing.assert_allclose(k[:, 0], (-1 + 2 * xi / (T - 1)).astype(np.float32), atol=1e-7)
    assert np.all(k[:, 1] == np.float32(0.25))


def test_p0_block_is_todays_byte_for_byte():
    p0 = params()
    p1 = params(control_knots=0, spline_degree=3)
    assert p0.control_knots == 0 and p0.spline_degree == 0
    assert bytes(p0) == bytes(p1)
    n = C.sizeof(p0) - 8
    p2 = params(control_knots=8, spline_degree=2)
    assert bytes(p2)[:n] == bytes(p0)[:n] and (p2.control_knots, p2.spline_degree) == (8, 2)
    assert shard_row_floats(p2, 2) == 2 + 8 * 2 and shard_row_floats(p0, 2) == 2 + 30 * 2


@pytest.mark.parametrize("kw, msg", [
    (dict(control_knots=-1), "must be >= 0"),
    (dict(control_knots=8, spline_degree=0), "spline_degree"),
    (dict(control_knots=8, spline_degree=4), "spline_degree"),
    (dict(control_knots=3, spline_degree=3), "must lie in"),
    (dict(control_knots=31), "must lie in"),
    (dict(control_knots=300, horizon=300), "horizon <= 256"),
    (dict(control_knots=8, sampling_method="halton"), "sampling_method random"),
    (dict(control_knots=8, sampling_method="colored"), "sampling_method random"),
    (dict(control_knots=8, mppi_mode="cem"), "cem"),
    (dict(control_knots=8, mppi_mode="smooth"), "cem and smooth"),
    (dict(control_knots=8, update_cov=True), "update_cov"),
    (dict(control_knots=8, update_lambda=True), "update_cov and update_lambda"),
    (dict(control_knots=8, n_modes=2), "n_modes"),
    (dict(control_knots=8, n_worlds=2, cvar_alpha=0.5), "n_worlds"),
    (dict(control_knots=8, anneal_iterations=2), "annealed"),
    (dict(control_knots=8, filter_u=True), "switch filter_u off"),
])
def test_refusals(kw, msg):
    with pytest.raises(ValueError, match=msg):
        params(**kw)


def test_pxnu_limit():
    with pytest.raises(ValueError, match="control_knots \\* nu <= 512"):
        params(nu=16, T=64, control_knots=33, noise_sigma=np.eye(16).tolist())
    params(nu=16, T=64, control_knots=32, noise_sigma=np.eye(16).tolist())


def test_oracle_at_identity_is_the_plain_plan():
    """At d = 1, P = T the oracle's K4 and shift are plain MPPI's: theta' = theta + W/eta, U_exec = theta', shift by one step."""
    p = params(T=12, control_knots=12, spline_degree=1)
    rng = np.random.default_rng(1)
    th = rng.standard_normal((12, 2))
    rows = np.concatenate([[0.5, 2.0], rng.standard_normal(24)])
    th2, ue, act = ko.finalize(p, 2, rows, th)
    np.testing.assert_allclose(th2, th + rows[2:].reshape(12, 2) / 2.0, atol=1e-14)
    np.testing.assert_array_equal(ue, th2)
    np.testing.assert_array_equal(act, th2[0])
    sh = ko.shift(p, 2, th)
    np.testing.assert_array_equal(sh[:-1], th[1:])
    np.testing.assert_array_equal(sh[-1], np.array(p.u_init[:2], np.float32))


def _planner(backend, **kw):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    from scenes import point_cfg
    return MPPIisaacPlanner(point_cfg(K=128, T=10, device="cpu", sampling_method="random", filter_u=False, **kw), PointReachObjective(),
                            backend=backend)


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_identity_plans_equal_the_plain_oracle_planner(mode):
    """d = 1, P = T over five plans: the knots oracle (B = I, the shift rows move one step) plans what the plain oracle plans."""
    import anneal_oracle as ao
    a = _planner(ko.KnotsOracleBackend(), mppi_mode=mode, control_knots=10, spline_degree=1)
    b = _planner(ao.AnnealOracleBackend(), mppi_mode=mode)
    assert tuple(a.mppi.U.shape) == (10, b.mppi.nu) and a.mppi.knots is not None
    for _ in range(5):
        np.testing.assert_allclose(a.compute_action([0.1, 0.0, 0.0], [0.0] * 3).numpy(),
                                   b.compute_action([0.1, 0.0, 0.0], [0.0] * 3).numpy(), rtol=0, atol=2e-5)
        np.testing.assert_allclose(a.mppi.U.numpy(), b.mppi.U.numpy(), rtol=0, atol=2e-5)
        np.testing.assert_array_equal(a.mppi.mean_action.numpy(), a.mppi.U.numpy())


def test_spline_plans_keep_u_exec_and_the_action_consistent():
    """P = 4, d = 3: after every plan U_exec = B U, the action is the first knot, and the knot samples have their (P, nu, K) shape."""
    from mppi_isaac_b200.model.blob import spline_basis
    pl = _planner(ko.KnotsOracleBackend(), control_knots=4, spline_degree=3)
    B, _, _ = spline_basis(10, 4, 3)
    for _ in range(4):
        act = pl.compute_action([0.1, 0.0, 0.0], [0.0] * 3).numpy()
        U = pl.mppi.U.numpy().astype(np.float64)
        np.testing.assert_allclose(pl.mppi.mean_action.numpy(), B @ U, rtol=0, atol=1e-6)   # U_exec from the unrounded knots
        np.testing.assert_array_equal(act, pl.mppi.U.numpy()[0])
        assert tuple(pl.mppi.knot_samples.shape) == (4, pl.mppi.nu, 128)
