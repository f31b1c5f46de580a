"""-m gpu: spline MPPI (``control_knots`` / ``spline_degree``) on the device: the spline K1 against float64 over the listed (T, nu, P, d)
and K, shards, the null row and the bounds; K3 and K4 (split and fused, SIMPLE and MEAN, RPL 4 / 8 / 16) and the shift against float64;
d = 1, P = T against plain MPPI bit for bit, kernel by kernel and over 20 graph-replayed point-robot plans; and the library's refusals."""
import numpy as np
import pytest
import torch

import knots_oracle as ko
from mppi_isaac_b200.model.blob import make_params, spline_table
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from scenes import point_cfg
from synth_mppi import nu_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 2.0 ** -24


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(DEV)


def params(nu, T, K, P, d=1, mode="simple", **kw):
    cfg = dict(num_samples=K, horizon=T, mppi_mode=mode, sampling_method="random", noise_sigma=(0.3 * np.eye(nu) + 0.05).tolist(),
               u_min=[-0.6], u_max=[0.6], lambda_=0.05, sample_null_action=True, rollout_var_discount=0.9, filter_u=False,
               control_knots=P, spline_degree=d)
    cfg.update(kw)
    return make_params(MPPIConfig(**cfg), IsaacGymConfig(), nu, K, [])


def backend(nu, p, theta=None):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(nu_model(nu), p)
    table = None
    if p.control_knots:
        table = dev(spline_table(p.T, p.control_knots, p.spline_degree, nu, theta))
        be.set_spline(table)
    return be, table


def spline_k1(nu, p, theta, k_offset=0, k_total=None):
    be, _ = backend(nu, p)
    K, T, P = p.K, p.T, p.control_knots
    a, x = torch.zeros((T, nu, K), device=DEV), torch.zeros((P, nu, K), device=DEV)
    be.sample_spline(7, 3, k_offset, k_total or K, dev(theta), a, x)
    torch.cuda.synchronize()
    be.destroy()
    return a.cpu().numpy(), x.cpu().numpy()


K1_SHAPES = [(2, 1, 2, 1), (30, 7, 8, 1), (30, 7, 8, 2), (30, 7, 8, 3), (30, 7, 30, 1), (256, 2, 256, 1), (64, 16, 32, 3), (256, 1, 4, 3)]


@pytest.mark.parametrize("T, nu, P, d", K1_SHAPES)
@pytest.mark.parametrize("K", [1, 31, 33, 1000, 65536])
def test_spline_k1_against_float64(T, nu, P, d, K):
    """Knots: |theta~ - ref| <= eps ((nu + 1) |L||z| + 2 |theta| + 2 |ref|) (the colour sum, the sum with theta, the rounding);
    actions: the knots' bound carried through the convex weights plus eps (d + 2) sum w |theta~| for the interpolation's sums."""
    p = params(nu, T, K, P, d)
    rng = np.random.default_rng(T + nu + P + d)
    th = (0.3 * rng.standard_normal((P, nu))).astype(np.float32)
    a, x = spline_k1(nu, p, th)
    ar, xr, tr = ko.sample(nu_model(nu), p, 7, 3, th, 0, K)
    z = np.abs(ko.co.white(nu_model(nu), ko.knot_params(p), 7, 3, 0, K).astype(np.float64))
    L = np.abs(np.array(p.sigma_chol[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu))
    kb = EPS * ((nu + 1) * np.einsum("ji,pik->pjk", L, z) + 2.0 * np.abs(th)[:, :, None] + 2.0 * np.abs(tr)) + 1e-30
    assert np.all(np.abs(x.astype(np.float64) - xr) <= 2 * kb)
    from mppi_isaac_b200.model.blob import spline_basis
    B, _, _ = spline_basis(T, P, d)
    ab = np.einsum("tp,pjk->tjk", B, kb + EPS * (d + 2) * np.abs(tr))
    assert np.all(np.abs(a.astype(np.float64) - ar) <= ab + 1e-30)
    lo, hi = np.float32(-0.6), np.float32(0.6)
    assert np.all((a >= lo) & (a <= hi))
    # the null row (global K - 1): every knot clamp(0) = 0, so every action is exactly 0
    assert np.all(a[:, :, K - 1] == 0.0) and np.all(x[:, :, K - 1] == -th)


def test_spline_k1_shards_are_bit_identical():
    T, nu, P, d, K = 30, 7, 8, 3, 1000
    th = (0.2 * np.random.default_rng(2).standard_normal((P, nu))).astype(np.float32)
    a, x = spline_k1(nu, params(nu, T, K, P, d), th)
    cut = 333
    a0, x0 = spline_k1(nu, params(nu, T, cut, P, d), th, 0, K)
    a1, x1 = spline_k1(nu, params(nu, T, K - cut, P, d), th, cut, K)
    np.testing.assert_array_equal(np.concatenate([a0, a1], -1), a)
    np.testing.assert_array_equal(np.concatenate([x0, x1], -1), x)


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_identity_knots_are_plain_k1_k3_k4_and_shift_bit_for_bit(mode):
    T, nu, K = 30, 7, 4096
    rng = np.random.default_rng(5)
    U = (0.2 * rng.standard_normal((T, nu))).astype(np.float32)
    pp = params(nu, T, K, 0, mode=mode)
    pk = params(nu, T, K, T, 1, mode=mode)
    bp, _ = backend(nu, pp)
    bk, table = backend(nu, pk, U)
    a0, n0 = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    a1, x1 = torch.zeros_like(a0), torch.zeros_like(a0)
    bp.sample(7, 3, 0, K, dev(U), None, a0, n0)
    bk.sample_spline(7, 3, 0, K, dev(U), a1, x1)
    torch.cuda.synchronize()
    assert torch.equal(a0, a1)
    assert torch.equal(x1, n0 if mode == "simple" else a0)
    cost = dev(rng.random((T, K)))
    outs = []
    for be, x in ((bp, n0 if mode == "simple" else a0), (bk, x1)):
        Ug, act, st, part = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV), torch.zeros(2 + T * nu, device=DEV)
        be.reduce_finalize(cost, x, Ug, part, act, st)
        Us, act2, st2 = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        be.reduce(cost, x, Us, part)
        be.finalize(part.view(1, -1), 1, Us, act2, st2)
        ctr = torch.zeros(1, dtype=torch.int32, device=DEV)
        be.shift(Us, ctr)
        torch.cuda.synchronize()
        outs.append([t.cpu().numpy() for t in (Ug, act, st, act2, st2, Us)])
    for u, v in zip(*outs):
        np.testing.assert_array_equal(u, v)
    np.testing.assert_array_equal(table[-T * nu:].cpu().numpy().reshape(T, nu), outs[0][0])   # U_exec = theta at B = I (the split K4's)
    bp.destroy(); bk.destroy()


@pytest.mark.parametrize("nu, T, P, d", [(2, 30, 8, 3), (7, 30, 8, 2), (7, 64, 30, 1), (16, 64, 32, 3), (1, 256, 4, 3)])
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_k3_k4_shift_against_float64(nu, T, P, d, mode):
    """The row of K3 over P*nu knot rows (RPL 4, 8, 16), K4 on both paths with U_exec and the action, then the shift."""
    K = 4096
    p = params(nu, T, K, P, d, mode=mode)
    rng = np.random.default_rng(nu * P + d)
    th = (0.2 * rng.standard_normal((P, nu))).astype(np.float32)
    cost = rng.random((T, K)).astype(np.float32)
    x = (0.2 * rng.standard_normal((P, nu, K))).astype(np.float32)
    if mode != "simple":
        x = x + th[:, :, None]
    be, table = backend(nu, p, th)
    part = torch.zeros(2 + P * nu, device=DEV)
    be.reduce(dev(cost), dev(x), dev(th), part)
    Us, act2 = dev(th), torch.zeros(nu, device=DEV)
    be.finalize(part.view(1, -1), 1, Us, act2, torch.zeros(2, device=DEV))
    torch.cuda.synchronize()
    ue_split = table[-T * nu:].cpu().numpy().reshape(T, nu).copy()
    Ug, act = dev(th), torch.zeros(nu, device=DEV)
    be.reduce_finalize(dev(cost), dev(x), Ug, torch.zeros_like(part), act, torch.zeros(2, device=DEV))
    torch.cuda.synchronize()
    ue_fused = table[-T * nu:].cpu().numpy().reshape(T, nu).copy()
    ref = ko.row(p, nu, cost, x, th)
    row = part.cpu().numpy()
    np.testing.assert_allclose(row[0], ref[0], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(row[1], ref[1], rtol=2e-4)
    np.testing.assert_allclose(row[2:], ref[2:], rtol=0, atol=2e-4 * max(1.0, float(np.abs(ref[2:]).max())))
    th2, ue, a = ko.finalize(p, nu, ref, th)
    for U_, act_, ue_ in ((Us, act2, ue_split), (Ug, act, ue_fused)):
        np.testing.assert_allclose(U_.cpu().numpy(), th2, rtol=0, atol=1e-4)
        np.testing.assert_allclose(act_.cpu().numpy(), a, rtol=0, atol=1e-4)
        np.testing.assert_allclose(ue_, ue, rtol=0, atol=1e-4)
    np.testing.assert_array_equal(act.cpu().numpy(), Ug.cpu().numpy()[0])
    np.testing.assert_array_equal(ue_fused[0], Ug.cpu().numpy()[0])           # B[0] = e_0: the first action is theta_0 exactly
    thg = Ug.cpu().numpy()
    be.shift(Ug, None)
    torch.cuda.synchronize()
    np.testing.assert_allclose(Ug.cpu().numpy(), ko.shift(p, nu, thg), rtol=0, atol=4 * EPS * (1 + np.abs(thg).max()))
    be.destroy()


def _planner(device, graph=False, **kw):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    return MPPIisaacPlanner(point_cfg(device=device, **kw), PointReachObjective(), use_cuda_graph=graph)


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_identity_knots_planner_is_the_plain_planner_over_graph_replays(mode):
    kw = dict(K=2048, T=12, sampling_method="random", mppi_mode=mode, filter_u=False)
    a = _planner(DEV, graph=True, **kw)
    b = _planner(DEV, graph=True, control_knots=12, spline_degree=1, **kw)
    assert b.mppi.knots is not None and tuple(b.mppi.knot_samples.shape) == (12, a.mppi.nu, 2048)
    q = [0.1, 0.0, 0.0]
    for _ in range(20):
        np.testing.assert_array_equal(a.compute_action(q, [0.0] * 3).numpy(), b.compute_action(q, [0.0] * 3).numpy())
        np.testing.assert_array_equal(a.mppi.U.cpu().numpy(), b.mppi.U.cpu().numpy())
        np.testing.assert_array_equal(a.mppi.stats.cpu().numpy(), b.mppi.stats.cpu().numpy())
        np.testing.assert_array_equal(b.mppi.mean_action.cpu().numpy(), b.mppi.U.cpu().numpy())
    assert a.mppi._graph is not None and b.mppi._graph is not None


def test_identity_knots_panda_reach_at_c2_is_the_plain_planner_over_graph_replays():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from scenes import panda_cfg
    kw = dict(sampling_method="random", filter_u=False)
    a = MPPIisaacPlanner(panda_cfg(K=10000, T=30, device=DEV, **kw), PandaReachObjective(), use_cuda_graph=True)
    b = MPPIisaacPlanner(panda_cfg(K=10000, T=30, device=DEV, control_knots=30, spline_degree=1, **kw), PandaReachObjective(),
                         use_cuda_graph=True)
    q, qd = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0], [0.0] * 7
    for _ in range(20):
        np.testing.assert_array_equal(a.compute_action(q, qd).numpy(), b.compute_action(q, qd).numpy())
        np.testing.assert_array_equal(a.mppi.U.cpu().numpy(), b.mppi.U.cpu().numpy())
        np.testing.assert_array_equal(a.mppi.stats.cpu().numpy(), b.mppi.stats.cpu().numpy())
    assert a.mppi._graph is not None and b.mppi._graph is not None


def test_a_block_without_knots_ignores_a_table_registered_before():
    """create with P > 0 and a table, then set_params with P = 0: every launch is the plain one, bit for bit, and the table is untouched;
    a model with another nu makes the table's launches refuse."""
    T, nu, K, P = 12, 3, 1024, 4
    rng = np.random.default_rng(9)
    U = (0.2 * rng.standard_normal((T, nu))).astype(np.float32)
    cost = dev(rng.random((T, K)))
    bk, table = backend(nu, params(nu, T, K, P, 2), U[:P])
    before = table.clone()
    bk.set_params(params(nu, T, K, 0))
    bp, _ = backend(nu, params(nu, T, K, 0))
    outs = []
    for be in (bp, bk):
        a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
        Ug, act, st = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        be.sample(7, 3, 0, K, Ug, None, a, n)
        be.reduce_finalize(cost, n, Ug, torch.zeros(2 + T * nu, device=DEV), act, st)
        part = torch.zeros(2 + T * nu, device=DEV)
        be.reduce(cost, n, Ug, part)
        be.finalize(part.view(1, -1), 1, Ug, act, st)
        be.shift(Ug, None)
        torch.cuda.synchronize()
        outs.append([t.cpu().numpy() for t in (a, n, Ug, act, st)])
    for u, v in zip(*outs):
        np.testing.assert_array_equal(u, v)
    assert torch.equal(table, before)
    bp.destroy(); bk.destroy()
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(nu_model(nu), params(nu, T, K, P, 2))
    be.set_spline(dev(spline_table(T, P, 2, nu)))
    be.set_model(nu_model(nu + 1))
    with pytest.raises(RuntimeError, match="registered for"):
        be.shift(dev(np.zeros((P, nu + 1))), None)
    be.destroy()


def test_spline_planner_plans_with_fewer_knots():
    pl = _planner(DEV, graph=True, K=2048, T=12, sampling_method="random", filter_u=False, control_knots=5, spline_degree=3)
    for _ in range(5):
        pl.compute_action([0.1, 0.0, 0.0], [0.0] * 3)
    assert tuple(pl.mppi.U.shape) == (5, pl.mppi.nu) and tuple(pl.mppi.mean_action.shape) == (12, pl.mppi.nu)
    assert torch.isfinite(pl.mppi.mean_action).all()


def test_library_refusals():
    nu, T, K, P = 3, 10, 256, 4
    p = params(nu, T, K, P, 2)
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(nu_model(nu), p)
    th, a, x, n = dev(np.zeros((P, nu))), torch.zeros((T, nu, K), device=DEV), torch.zeros((P, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    with pytest.raises(RuntimeError, match="spline table registered"):
        be.sample_spline(1, 0, 0, K, th, a, x)
    with pytest.raises(RuntimeError, match="spline table registered"):
        be.shift(th)
    be.set_spline(dev(spline_table(T, P, 2, nu)))
    be.sample_spline(1, 0, 0, K, th, a, x)
    with pytest.raises(RuntimeError, match="mppib_sample_spline"):
        be.sample(1, 0, 0, K, th, None, a, n)
    be.set_distribution(dev(np.ones(1 + nu)))
    with pytest.raises(RuntimeError, match="register no distribution"):
        be.reduce(torch.zeros((T, K), device=DEV), x, th, torch.zeros(2 + P * nu, device=DEV))
    be.set_distribution(None)
    be.set_params(params(nu, T + 2, K, P, 2))
    with pytest.raises(RuntimeError, match="registered for"):
        be.sample_spline(1, 0, 0, K, th, torch.zeros((T + 2, nu, K), device=DEV), x)
    import ctypes as C
    with pytest.raises(RuntimeError, match="does not match"):
        be._check(be.lib.mppib_set_spline(be.handle, C.c_void_p(th.data_ptr()), C.c_int32(5), C.c_int32(2)), "mppib_set_spline")
    torch.cuda.synchronize()
    be.destroy()
