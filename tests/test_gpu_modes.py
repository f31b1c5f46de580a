"""-m gpu: multi-modal MPPI (``n_modes``) on the device: K1 columns of every mode against the plain K1 with U := U_m, bit for bit, for every
supported variant; K3's per-mode blocks against a float32 restatement of beta and the float64 reference; K4 against the reference, fused
against split, over 1 .. 8 shard rows; n_modes = 1 against a planner without the key; whole point-robot and C2-shape (panda reach,
T = 30, nu = 7, K = 2048) plans against the ``ModesOracleBackend`` pipeline, graph replay and a keep_U rebuild."""
import copy

import numpy as np
import pytest
import torch

import modes_oracle as mo
from mppi_isaac_b200.model.blob import make_params
from mppi_isaac_b200.planner.mppi import colored_noise_chol, halton_spline_operator, halton_table
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from scenes import point_cfg
from synth_mppi import nu_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 2.0 ** -24


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(DEV)


def params(nu, T, K_total, M=1, K=None, k_offset=0, **kw):
    d = dict(num_samples=K_total, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.3 * np.eye(nu) + 0.05).tolist(),
             u_min=[-0.5], u_max=[0.5], lambda_=0.05, sample_null_action=True, n_modes=M)
    d.update(kw)
    p = make_params(MPPIConfig(**d), IsaacGymConfig(), nu, K or K_total, [])
    p.k_offset = k_offset
    return p


def state_for(M, T, nu, U0=None):
    return dev(np.concatenate([[0.0], np.full(M, np.inf), np.zeros(T * nu) if U0 is None else np.ravel(U0)]))


def backend(nu, p, state=None):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(nu_model(nu), p)
    if state is not None:
        be.set_distribution(state)
    return be


def k1(variant, nu, T, p, U, k_offset, k_total, state=None):
    be = backend(nu, p, state)
    K = p.K
    a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    if variant == "random":
        be.sample(7, 3, k_offset, k_total, U, None, a, n)
    elif variant == "colored":
        be.sample_colored(7, 3, k_offset, k_total, U, None, dev(colored_noise_chol(T, 2.0)), a, n)
    else:
        nk = max(T // 4, 3)
        Z = torch.zeros((T, nu, K), device=DEV)
        be.noise_library(k_offset, k_total, torch.from_numpy(halton_table(nk * nu, 5)).to(DEV), dev(halton_spline_operator(T, nk)), nk, Z)
        be.sample_library(k_offset, k_total, U, None, Z, a, n)
    torch.cuda.synchronize()
    be.destroy()
    return a.cpu().numpy(), n.cpu().numpy()


@pytest.mark.parametrize("variant", ["random", "colored", "halton"])
@pytest.mark.parametrize("M", [2, 3, 16])
def test_k1_mode_columns_are_the_plain_k1_bit_for_bit(variant, M):
    nu, T, Kc = 5, 12, 64
    Kt = M * Kc
    Um = 0.1 * np.sin(np.arange(M * T * nu) * 0.7).reshape(M, T, nu)
    full_a, full_n = k1(variant, nu, T, params(nu, T, Kt, M), dev(Um), 0, Kt, state_for(M, T, nu))
    modes = np.arange(Kt) // Kc
    for m in range(M):
        pa, pn = k1(variant, nu, T, params(nu, T, Kt), dev(Um[m]), 0, Kt)
        np.testing.assert_array_equal(full_a[:, :, modes == m], pa[:, :, modes == m])
        np.testing.assert_array_equal(full_n[:, :, modes == m], pn[:, :, modes == m])
    assert (full_a[:, :, -1] == 0.0).all()                                   # the null row stays global K - 1, in mode M - 1
    off, Kl = Kc // 2 + 4, Kc + 8                                            # a shard whose offset and end cut modes
    sh_a, sh_n = k1(variant, nu, T, params(nu, T, Kt, M, K=Kl, k_offset=off), dev(Um), off, Kt, state_for(M, T, nu))
    np.testing.assert_array_equal(sh_a, full_a[:, :, off:off + Kl])
    np.testing.assert_array_equal(sh_n, full_n[:, :, off:off + Kl])


def test_k1_refuses_a_total_that_is_not_the_modes():
    p = params(3, 4, 128, 2)
    be = backend(3, p, state_for(2, 4, 3))
    with pytest.raises(RuntimeError, match="k_total"):
        be.sample(1, 0, 0, 256, torch.zeros((2, 4, 3), device=DEV), None, torch.zeros((4, 3, 128), device=DEV), None)
    be.destroy()


def k3_case(nu, T, Kc, M, seed, K=None, off=0, dead=None, mode="simple"):
    Kt = M * Kc
    K = K or Kt
    p = params(nu, T, Kt, M, K=K, k_offset=off, mppi_mode=mode, rollout_var_discount=0.9)
    rng = np.random.default_rng(seed)
    cost = rng.random((T, K)).astype(np.float32)
    cost[rng.integers(0, T, 3), rng.integers(0, K, 3)] = np.inf
    if dead is not None:                                                     # every sample of mode `dead` is invalid
        cols = np.nonzero(mo.modes_of(p, off, K) == dead)[0]
        cost[0, cols] = np.nan
    x = (0.2 * rng.standard_normal((T, nu, K))).astype(np.float32)
    U = (0.1 * rng.standard_normal((M, T, nu))).astype(np.float32) if T > 1 else np.zeros((M, T, nu), np.float32)
    return p, cost, x, U


def run_k3(nu, p, cost, x, U):
    M = int(p.n_modes)
    be = backend(nu, p, state_for(M, p.T, nu))
    part = torch.zeros(be.partial_row_floats(), device=DEV)
    be.reduce(dev(cost), dev(x), dev(U), part)
    torch.cuda.synchronize()
    be.destroy()
    return part.cpu().numpy()


@pytest.mark.parametrize("M, Kc, off, K", [(2, 2048, 0, None), (4, 32, 0, None), (3, 96, 16, 200), (16, 256, 0, None), (5, 64, 36, 160)])
def test_k3_beta_is_the_float32_minimum_bit_for_bit(M, Kc, off, K):
    """T = 1 and U = 0: S equals the cost exactly, so beta_m is the minimum of the mode's finite costs, bit for bit."""
    nu = 3
    p, cost, x, U = k3_case(nu, 1, Kc, M, seed=M + Kc, K=K, off=off)
    row = run_k3(nu, p, cost, x, U).reshape(M, -1)
    mo_ = mo.modes_of(p, off, cost.shape[1])
    for m in range(M):
        c = cost[0, mo_ == m]
        c = c[np.isfinite(c)]
        assert row[m, 0] == (c.min() if c.size else np.inf) and (row[m, 1] > 0) == (c.size > 0)


@pytest.mark.parametrize("T, nu, M, Kc, off, K, dead, mode", [
    (8, 3, 2, 1024, 0, None, None, "simple"),                                # RPL 4
    (30, 7, 4, 32, 0, None, None, "simple"),                                 # RPL 8, Kc = 32
    (30, 7, 3, 160, 48, 400, 1, "halton-spline"),                            # boundaries inside tiles, a dead mode, MEAN
    (32, 16, 16, 64, 0, None, 5, "simple"),                                  # RPL 16, M = 16 at T*nu = 512
    (20, 12, 5, 96, 20, 300, None, "simple"),
])
def test_k3_rows_against_float64(T, nu, M, Kc, off, K, dead, mode):
    p, cost, x, U = k3_case(nu, T, Kc, M, seed=T * M, K=K, off=off, dead=dead, mode=mode)
    row = run_k3(nu, p, cost, x, U).reshape(M, -1)
    ref = mo.reduce(p, nu, cost, x, U).reshape(M, -1)
    lam = float(np.float32(p.lambda_))
    mag = float(np.where(np.isfinite(cost), np.abs(cost), 0).sum(0).max()) + 1.0
    gb = (T + T * nu + 8) * EPS * (mag + np.abs(x).sum((0, 1)).max() * 10)
    gw = 64 * EPS * Kc + gb / lam * 2
    for m in range(M):
        if ref[m, 1] == 0:
            assert row[m, 0] == np.inf and row[m, 1] == 0 and (row[m, 2:] == 0).all()
            continue
        assert abs(float(row[m, 0]) - float(ref[m, 0])) <= gb
        np.testing.assert_allclose(row[m, 1], ref[m, 1], rtol=gw, atol=0)
        np.testing.assert_allclose(row[m, 2:], ref[m, 2:], rtol=0, atol=gw * max(1.0, float(np.abs(ref[m, 2:]).max())))
    if dead is not None:
        assert row[dead, 0] == np.inf and row[dead, 1] == 0


def k4_rows(nu, T, M, G, seed, mode="simple"):
    """G shard rows of a plan over Kc = 64 * G samples per mode, the shards cutting the modes, and the modes U."""
    Kc, rng = 64 * G, np.random.default_rng(seed)
    Kt = M * Kc
    U = (0.15 * rng.standard_normal((M, T, nu))).astype(np.float32)
    cost = rng.random((T, Kt)).astype(np.float32)
    x = (0.2 * rng.standard_normal((T, nu, Kt))).astype(np.float32)
    p = params(nu, T, Kt, M, mppi_mode=mode, filter_u=True, rollout_var_discount=0.9, mode_switch_margin=0.05)
    rows = np.stack([mo.reduce(p, nu, cost[:, g * Kt // G:(g + 1) * Kt // G], x[:, :, g * Kt // G:(g + 1) * Kt // G], U, k_offset=g * Kt // G)
                     for g in range(G)])
    return p, rows, U, cost, x


def run_k4(nu, p, rows, U, state):
    be = backend(nu, p, state)
    Ud = dev(U)
    act, st = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(dev(rows), rows.shape[0], Ud, act, st)
    torch.cuda.synchronize()
    be.destroy()
    return Ud.cpu().numpy(), act.cpu().numpy(), st.cpu().numpy(), state.cpu().numpy()


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("T, nu, M", [(10, 3, 2), (30, 7, 4), (32, 16, 16), (12, 2, 5)])
def test_k4_against_the_oracle(T, nu, M, mode):
    p, rows, U, _, _ = k4_rows(nu, T, M, 2, seed=T + M, mode=mode)
    state0 = np.concatenate([[M - 1], np.full(M, np.inf), U[M - 1].ravel()]).astype(np.float32)
    Ug, ag, sg, stg = run_k4(nu, p, rows, U, dev(state0))
    Ur, ar, sr, str_ = mo.finalize(p, nu, rows, U, state0)
    tol = 1e-5 * max(1.0, float(np.abs(U).max()))
    np.testing.assert_allclose(Ug, Ur, rtol=0, atol=tol)
    F = str_[1:1 + M].astype(np.float64)
    np.testing.assert_allclose(stg[1:1 + M], F, rtol=1e-5, atol=1e-5)
    order = np.sort(F[np.isfinite(F)])
    gap = np.inf if order.size < 2 else order[1] - order[0]
    if gap > 1e-4 * max(1.0, float(np.abs(order).max())) and abs(F[int(state0[0])] - order[0] - 0.05) > 1e-4:
        assert stg[0] == str_[0]                                            # the selection is exact away from float32 ties
        np.testing.assert_allclose(ag, ar, rtol=0, atol=tol)
        np.testing.assert_allclose(stg[1 + M:], str_[1 + M:], rtol=0, atol=tol)


@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_k4_is_rank_independent_and_fused_equals_split(G):
    """Every rank combines the same G rows: two handles give the same bits; with G = 1 the fused K3 + K4 equals K3 then K4."""
    nu, T, M = 4, 16, 4
    p, rows, U, cost, x = k4_rows(nu, T, M, G, seed=G)
    state0 = np.concatenate([[0], np.full(M, np.inf), U[0].ravel()]).astype(np.float32)
    a = run_k4(nu, p, rows, U, dev(state0))
    b = run_k4(nu, p, rows, U, dev(state0))
    for u, v in zip(a, b):
        np.testing.assert_array_equal(u, v)
    if G == 1:
        outs = []
        for fused in (True, False):
            st = dev(state0)
            be = backend(nu, p, st)
            Ud, part = dev(U), torch.zeros(be.partial_row_floats(), device=DEV)
            act, s2 = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
            if fused:
                be.reduce_finalize(dev(cost), dev(x), Ud, part, act, s2)
            else:
                be.reduce(dev(cost), dev(x), Ud, part)
                be.finalize(part.view(1, -1), 1, Ud, act, s2)
            torch.cuda.synchronize()
            outs.append([t.cpu().numpy() for t in (Ud, act, s2, st, part)])
            be.destroy()
        for u, v in zip(*outs):
            np.testing.assert_array_equal(u, v)


def test_reduce_and_finalize_refuse_without_a_mode_state():
    p = params(3, 4, 128, 2)
    be = backend(3, p)
    with pytest.raises(RuntimeError, match="mode state"):
        be.finalize(torch.zeros((1, 2 * 14), device=DEV), 1, torch.zeros((2, 4, 3), device=DEV), torch.zeros(3, device=DEV), None)
    be.destroy()


def _planner(device, graph=False, backend=None, **kw):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    extra = {} if backend is None else dict(backend=backend)
    return MPPIisaacPlanner(point_cfg(device=device, **kw), PointReachObjective(), use_cuda_graph=graph, **extra)


def test_one_mode_is_bit_identical_to_a_planner_without_the_key():
    a, b = _planner(DEV, K=1024, T=12), _planner(DEV, K=1024, T=12, n_modes=1)
    for _ in range(3):
        np.testing.assert_array_equal(a.compute_action([0.1, 0.0, 0.0], [0.0] * 3).cpu().numpy(), b.compute_action([0.1, 0.0, 0.0], [0.0] * 3).cpu().numpy())
    np.testing.assert_array_equal(a.mppi.U.cpu().numpy(), b.mppi.U.cpu().numpy())


def test_point_plans_agree_with_the_oracle_pipeline():
    gpu = _planner(DEV, K=256, T=12, n_modes=4)
    cpu = _planner("cpu", K=256, T=12, n_modes=4, backend=mo.ModesOracleBackend())
    for _ in range(2):
        ag, ac = gpu.compute_action([0.1, 0.0, 0.0], [0.0] * 3), cpu.compute_action([0.1, 0.0, 0.0], [0.0] * 3)
        assert float((ag.cpu() - ac).abs().max()) <= 2e-4
    np.testing.assert_allclose(gpu.mppi.modes.cpu().numpy(), cpu.mppi.modes.numpy(), rtol=0, atol=2e-4)
    assert gpu.mppi.active_mode == cpu.mppi.active_mode


def test_graph_replay_equals_the_eager_plan_and_keep_u_rebuild_keeps_the_modes():
    pls = [_planner(DEV, graph=g, K=2048, T=12, n_modes=4) for g in (True, False)]
    for _ in range(4):
        a, b = (pl.compute_action([0.1, 0.0, 0.0], [0.0] * 3).cpu().numpy() for pl in pls)
        np.testing.assert_array_equal(a, b)
    assert pls[0].mppi._graph is not None and pls[1].mppi._graph is None
    np.testing.assert_array_equal(pls[0].mppi.mode_state.cpu().numpy(), pls[1].mppi.mode_state.cpu().numpy())
    pl = pls[1]
    U, st = pl.mppi.modes.clone(), pl.mppi.mode_state.clone()
    pl._build_mppi(keep_U=True)
    assert torch.equal(pl.mppi.modes, U) and torch.equal(pl.mppi.mode_state, st)
    assert torch.isfinite(pl.compute_action([0.1, 0.0, 0.0], [0.0] * 3)).all()


def test_c2_shape_plans_agree_with_the_oracle_pipeline():
    """Panda reach at the C2 shape (T = 30, nu = 7: RPL 8) with M = 4 and K = 2048, so that K3 runs 16 CTAs per mode, closed loop, graph
    on, against the same planner on the ``ModesOracleBackend``."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from scenes import panda_cfg
    mk = lambda d: panda_cfg(K=2048, T=30, device=d, n_modes=4)
    gpu = MPPIisaacPlanner(mk(DEV), PandaReachObjective(), use_cuda_graph=True)
    cpu = MPPIisaacPlanner(mk("cpu"), PandaReachObjective(), backend=mo.ModesOracleBackend(nthreads=8))
    q = np.array([0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0])
    qd = np.zeros_like(q)
    lim = float(gpu.mppi.backend.params.u_max[0])
    for it in range(3):
        ag, ac = gpu.compute_action(q, qd), cpu.compute_action(q, qd)
        assert float((ag.cpu() - ac).abs().max()) <= 2e-4 * max(1.0, lim), f"plan {it}"
        assert gpu.mppi.active_mode == cpu.mppi.active_mode
        q = q + 0.05 * ac.numpy(); qd = ac.numpy()
    assert gpu.mppi._graph is not None
    np.testing.assert_allclose(gpu.mppi.modes.cpu().numpy(), cpu.mppi.modes.numpy(), rtol=0, atol=2e-4 * max(1.0, lim))
