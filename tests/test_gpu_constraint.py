"""-m gpu: constrained MPPI (``constraint_mode: feasible_first``) on the device: K3 + K4 (split and fused, SIMPLE and MEAN, RPL 4 / 8 /
16, K not a multiple of 32) against float64 with feasible, violation-only and mixed tiles over several CTAs and shards; all-feasible plans
equal to today's K3 / K4 bit for bit, kernel by kernel and over 20 graph-replayed point-robot plans; the library's refusals; and the
planner's accessors."""
import numpy as np
import pytest
import torch

import constraint_oracle as cn
from mppi_isaac_b200.model.blob import make_params
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from scenes import point_cfg
from synth_mppi import nu_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(DEV)


def params(nu, T, K, mode="simple", on=True, **kw):
    cfg = dict(num_samples=K, horizon=T, mppi_mode=mode, sampling_method="random", noise_sigma=(0.3 * np.eye(nu) + 0.05).tolist(),
               u_min=[-0.6], u_max=[0.6], lambda_=0.05, rollout_var_discount=0.9, filter_u=T >= 9)
    if on:
        cfg.update(constraint_mode="feasible_first", constraint_tol=0.05, constraint_lambda=0.2)
    cfg.update(kw)
    return make_params(MPPIConfig(**cfg), IsaacGymConfig(), nu, K, [])


def backend(nu, p, viol=None):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(nu_model(nu), p)
    cstate = torch.zeros(2, device=DEV)
    if viol is not None:
        be.set_constraint(viol, cstate)
    return be, cstate


def inputs(nu, T, K, mode, kind, seed):
    """cost, x, U and margins g of K samples; `kind` picks which samples are feasible: all, none, mixed (only some 32-sample tiles
    hold a feasible sample), or 'nonfinite' (mixed plus NaN / +inf margins and costs)."""
    rng = np.random.default_rng(seed)
    U = (0.2 * rng.standard_normal((T, nu))).astype(np.float32)
    cost = rng.random((T, K)).astype(np.float32)
    x = (0.2 * rng.standard_normal((T, nu, K))).astype(np.float32)
    if mode != "simple":
        x = x + U[:, :, None]
    g = (-rng.random((T, K))).astype(np.float32)
    if kind in ("none", "mixed", "nonfinite"):
        g[rng.integers(0, T, K), np.arange(K)] = (0.1 + rng.random(K)).astype(np.float32)    # every sample violates at one step
    if kind in ("mixed", "nonfinite"):
        tiles = np.arange(K) // 32
        keep = (tiles % 5 == 3) & (rng.random(K) < 0.5)                                      # a few tiles hold feasible samples
        g[:, keep] = np.minimum(g[:, keep], 0.0)
        g[0, keep & (rng.random(K) < 0.3)] = 0.05                                            # V = tol exactly: feasible
    if kind == "nonfinite":
        g[min(1, T - 1), rng.random(K) < 0.05] = np.nan
        g[min(2, T - 1), rng.random(K) < 0.05] = np.inf
        cost[0, rng.random(K) < 0.03] = np.inf
    return cost, x, U, g


def run(nu, T, K, mode, kind, seed=0, fused=True):
    p = params(nu, T, K, mode)
    cost, x, U, g = inputs(nu, T, K, mode, kind, seed)
    viol = dev(g)
    be, cstate = backend(nu, p, viol)
    part = torch.zeros(4 + T * nu, device=DEV)
    Us, act, st = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.reduce(dev(cost), dev(x), Us, part)
    be.finalize(part.view(1, -1), 1, Us, act, st)
    torch.cuda.synchronize()
    split = [t.cpu().numpy().copy() for t in (part, Us, act, st, cstate)]
    out = [split]
    if fused:
        Ug, actg, stg, partg = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV), torch.zeros_like(part)
        cstate.zero_()
        be.reduce_finalize(dev(cost), dev(x), Ug, partg, actg, stg)
        torch.cuda.synchronize()
        out.append([t.cpu().numpy().copy() for t in (partg, Ug, actg, stg, cstate)])
    be.destroy()
    return p, (cost, x, U, g), out


def nf_bits(v):
    return int(np.asarray(v, np.float32).reshape(1).view(np.int32)[0])


def check_row(row, ref):
    assert nf_bits(row[-2]) == int(ref[-2])
    np.testing.assert_allclose(row[-1], ref[-1], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(row[0], ref[0], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(row[1], ref[1], rtol=2e-4)
    np.testing.assert_allclose(row[2:-2], ref[2:-2], rtol=0, atol=2e-4 * max(1.0, float(np.abs(ref[2:-2]).max())))


SHAPES = [(1, 4, 4100), (2, 30, 4096), (7, 30, 10000), (7, 16, 2052), (16, 16, 8000), (8, 64, 4096), (1, 256, 1028), (1, 1, 100)]


@pytest.mark.parametrize("nu, T, K", SHAPES)
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("kind", ["all", "none", "mixed", "nonfinite"])
def test_k3_k4_against_float64(nu, T, K, mode, kind):
    p, (cost, x, U, g), outs = run(nu, T, K, mode, kind, seed=nu * T + K)
    ref = cn.row(p, nu, cost, x, U, g)
    Un, a, st, (n, vmin) = cn.finalize(nu_model(nu), p, ref[None], U)
    for part, U_, act, stats, cstate in outs:
        check_row(part, ref)
        np.testing.assert_allclose(U_, Un, rtol=0, atol=1e-4)
        np.testing.assert_allclose(act, a, rtol=0, atol=1e-4)
        np.testing.assert_allclose(stats, st, rtol=2e-4, atol=1e-5)
        assert nf_bits(cstate[0]) == n
        np.testing.assert_allclose(cstate[1], vmin, rtol=1e-5, atol=1e-6)
    # the fused tail writes the same row and the same update as the split K4
    for u, v in zip(outs[0], outs[1]):
        np.testing.assert_array_equal(u, v)
    if kind == "all":
        assert n == K
    if kind == "none":
        assert n == 0 and np.isfinite(outs[0][0][0])


def test_no_valid_sample_keeps_U():
    nu, T, K = 2, 12, 1024
    p = params(nu, T, K)
    cost, x, U, _ = inputs(nu, T, K, "simple", "all", 3)
    viol = dev(np.full((T, K), np.nan, np.float32))
    be, cstate = backend(nu, p, viol)
    Ug, part = dev(U), torch.zeros(4 + T * nu, device=DEV)
    be.reduce_finalize(dev(cost), dev(x), Ug, part, torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV))
    torch.cuda.synchronize()
    row = part.cpu().numpy()
    assert row[0] == np.inf and row[1] == 0.0 and nf_bits(row[-2]) == 0 and row[-1] == np.inf
    p0 = params(nu, T, K, on=False)
    be0, _ = backend(nu, p0)
    U0 = dev(U)
    be0.reduce_finalize(dev(np.full((T, K), np.nan, np.float32)), dev(x), U0, torch.zeros(2 + T * nu, device=DEV), torch.zeros(nu, device=DEV),
                        torch.zeros(2, device=DEV))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(Ug.cpu().numpy(), U0.cpu().numpy())     # the plain K4 with no valid sample
    be.destroy(); be0.destroy()


@pytest.mark.parametrize("G", [2, 3, 4])
@pytest.mark.parametrize("pattern", ["first", "last", "none", "all"])
def test_shards_with_and_without_feasible_samples(G, pattern):
    """G shard rows from separate K3 launches around one U, merged by the explicit-row K4, against the float64 merge of the float64 rows."""
    nu, T, Kl, mode = 7, 16, 2052, "simple"
    p = params(nu, T, Kl, mode)
    U = inputs(nu, T, Kl, mode, "all", 99)[2]
    rows, refs = [], []
    for g_ in range(G):
        kind = {"first": "mixed" if g_ == 0 else "none", "last": "mixed" if g_ == G - 1 else "none", "none": "none", "all": "all"}[pattern]
        cost, x, _, gm = inputs(nu, T, Kl, mode, kind, 100 + g_)
        be, _ = backend(nu, p, dev(gm))
        part = torch.zeros(4 + T * nu, device=DEV)
        be.reduce(dev(cost), dev(x), dev(U), part)
        torch.cuda.synchronize()
        rows.append(part.cpu().numpy().copy())
        refs.append(cn.row(p, nu, cost, x, U, gm))
        check_row(rows[-1], refs[-1])
        be.destroy()
    be, cstate = backend(nu, p, dev(np.zeros((T, Kl), np.float32)))
    Ug, act, st = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(dev(np.stack(rows)), G, Ug, act, st)
    torch.cuda.synchronize()
    Un, a, st_ref, (n, vmin) = cn.finalize(nu_model(nu), p, np.stack(refs), U)
    np.testing.assert_allclose(Ug.cpu().numpy(), Un, rtol=0, atol=1e-4)
    np.testing.assert_allclose(act.cpu().numpy(), a, rtol=0, atol=1e-4)
    np.testing.assert_allclose(st.cpu().numpy(), st_ref, rtol=2e-4, atol=1e-5)
    cs = cstate.cpu().numpy()
    assert nf_bits(cs[0]) == n
    np.testing.assert_allclose(cs[1], vmin, rtol=1e-5)
    assert (n > 0) == (pattern != "none")
    be.destroy()


@pytest.mark.parametrize("nu, T, K", [(1, 4, 4100), (7, 30, 10000), (16, 16, 8000), (1, 256, 1028), (3, 12, 100)])
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_all_feasible_is_todays_k3_k4_bit_for_bit(nu, T, K, mode):
    cost, x, U, g = inputs(nu, T, K, mode, "all", nu + T)
    cost[0, ::97] = np.nan                                                     # invalid samples are invalid in both
    g[:, ::5] = 0.0
    res = []
    for on in (False, True):
        p = params(nu, T, K, mode, on=on)
        be, _ = backend(nu, p, dev(g) if on else None)
        P = 4 + T * nu if on else 2 + T * nu
        part, Us, act, st = torch.zeros(P, device=DEV), dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        be.reduce(dev(cost), dev(x), Us, part)
        be.finalize(part.view(1, -1), 1, Us, act, st)
        Ug, actg, stg, partg = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV), torch.zeros(P, device=DEV)
        be.reduce_finalize(dev(cost), dev(x), Ug, partg, actg, stg)
        torch.cuda.synchronize()
        res.append([part.cpu().numpy()[:2 + T * nu]] + [t.cpu().numpy() for t in (Us, act, st, partg[:2 + T * nu], Ug, actg, stg)])
        be.destroy()
    for u, v in zip(*res):
        np.testing.assert_array_equal(u, v)


class PointKeepOut:
    def __init__(self, fn):
        from mppi_isaac_b200.objectives import PointReachObjective
        self.base = PointReachObjective()
        self.fn = fn
        self.weights = {}

    def reset(self):
        pass

    def compute_cost(self, sim):
        return self.base.compute_cost(sim)

    def compute_constraint(self, sim):
        r = sim.get_actor_link_by_name(actor_name="point_robot", link_name="base_link")
        return self.fn(r[:, 0:3])


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_all_feasible_planner_is_the_plain_planner_over_graph_replays(mode):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    kw = dict(K=2048, T=12, sampling_method="random", mppi_mode=mode, filter_u=True, device=DEV)
    a = MPPIisaacPlanner(point_cfg(**kw), PointReachObjective(), use_cuda_graph=True)
    b = MPPIisaacPlanner(point_cfg(constraint_mode="feasible_first", **kw), PointKeepOut(lambda q: -1.0 - q[:, 0].abs()), use_cuda_graph=True)
    q = [0.1, 0.0, 0.0]
    for _ in range(20):
        np.testing.assert_array_equal(a.compute_action(q, [0.0] * 3).numpy(), b.compute_action(q, [0.0] * 3).numpy())
        np.testing.assert_array_equal(a.mppi.U.cpu().numpy(), b.mppi.U.cpu().numpy())
        np.testing.assert_array_equal(a.mppi.stats.cpu().numpy(), b.mppi.stats.cpu().numpy())
        assert b.mppi.feasible_samples == 2048 and float(b.mppi.min_violation) == 0.0
    assert a.mppi._graph is not None and b.mppi._graph is not None
    assert a.mppi.feasible_samples is None and a.mppi.min_violation is None and a.mppi.violation is None


def test_planner_accessors_match_the_violation_buffer():
    from mppi_isaac_b200 import MPPIisaacPlanner
    kw = dict(K=1024, T=12, sampling_method="random", mppi_mode="simple", filter_u=False, device=DEV)
    b = MPPIisaacPlanner(point_cfg(constraint_mode="feasible_first", **kw), PointKeepOut(lambda q: 0.1 - q[:, 0]), use_cuda_graph=True)
    for _ in range(3):
        b.compute_action([0.1, 0.0, 0.0], [0.0] * 3)
        g = b.mppi.violation.cpu().numpy().astype(np.float64)
        V = np.where(g <= 0, 0.0, g).sum(0)
        assert b.mppi.feasible_samples == int((V <= 0).sum())
        np.testing.assert_allclose(float(b.mppi.min_violation), V.min(), rtol=1e-5, atol=1e-7)
        assert b.mppi.min_violation.device.type == "cuda" and b.mppi.min_violation.dim() == 0


def test_library_refusals():
    nu, T, K = 2, 12, 256
    cost, x, U, g = inputs(nu, T, K, "simple", "all", 1)
    p = params(nu, T, K)
    be, cstate = backend(nu, p)
    part = torch.zeros(4 + T * nu, device=DEV)
    with pytest.raises(RuntimeError, match="registered"):
        be.reduce(dev(cost), dev(x), dev(U), part)                           # the mode without a registration
    viol = dev(g)
    be.set_constraint(viol, cstate)
    be.reduce(dev(cost), dev(x), dev(U), part)
    p2 = params(nu, T, 2 * K)
    be.set_params(p2)
    with pytest.raises(RuntimeError, match="registered for"):
        be.reduce(dev(np.tile(cost, 2)), dev(np.tile(x, 2)), dev(U), part)   # K changed since the registration
    p3 = params(nu, T + 1, K)
    be.set_params(p3)
    with pytest.raises(RuntimeError, match="registered for"):
        be.finalize(part.view(1, -1), 1, dev(np.zeros((T + 1, nu))), torch.zeros(nu, device=DEV), None)   # T changed
    be.set_params(params(nu, T, K, on=False))
    with pytest.raises(RuntimeError, match="constraint_mode is 0"):
        be.reduce(dev(cost), dev(x), dev(U), torch.zeros(2 + T * nu, device=DEV))   # a registration without the mode
    with pytest.raises(RuntimeError, match="constraint_mode = 0"):
        be.set_constraint(viol, cstate)
    be.set_constraint(None)
    be.reduce(dev(cost), dev(x), dev(U), torch.zeros(2 + T * nu, device=DEV))
    torch.cuda.synchronize()
    be.destroy()


def test_a_horizon_without_room_for_two_ring_stages_is_refused_at_create():
    """T = 256, nu = 2: a tile of (T*nu + 2T)*32 floats leaves room for one ring stage only, so make_params and mppib_create refuse the
    block before any plan; a handle created without the mode cannot take it on through mppib_set_params either."""
    from mppi_isaac_b200.backend import CudaBackend
    nu, T, K = 2, 256, 1028
    with pytest.raises(ValueError, match="ring stages"):
        params(nu, T, K)
    p = params(nu, T, K, on=False)
    p.constraint_mode, p.constraint_tol, p.constraint_lambda = 1, 0.05, 0.2
    be = CudaBackend(DEV)
    with pytest.raises(RuntimeError, match="ring stages"):
        be.create(nu_model(nu), p)
    ok = params(nu, 216, K)                                                   # T = 216 fits two stages
    be.create(nu_model(nu), ok)
    with pytest.raises(RuntimeError, match="ring stages"):
        be.set_params(p)
    be.destroy()
