"""-m gpu: Smooth MPPI (``mppi_mode: smooth``) on the device against the float64 reference of ``smooth_oracle``: the smooth K1 (bit
identity of its noise with the Gaussian K1, the integrated actions, bounds, the null row, shards), the smoothness cost in K3 over the
RPL 4 / 8 / 16 instantiations, K4's clamp and integration, and whole plans through the planner."""
import copy

import numpy as np
import pytest
import torch

import smooth_oracle as so
from mppi_isaac_b200.model.blob import MODE_SIMPLE, make_params
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from scenes import panda_cfg
from synth_mppi import nu_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
EPS = 2.0 ** -24


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def smooth_params(nu, T, K, k_offset=0, **kw):
    d = dict(num_samples=K, horizon=T, mppi_mode="smooth", sampling_method="random", noise_sigma=(0.3 * np.eye(nu) + 0.05).tolist(),
             u_min=[-0.2], u_max=[0.2], du_min=[-1.0], du_max=[1.0], lambda_=0.05, sample_null_action=True, smooth_weight=0.5)
    d.update(kw)
    p = make_params(MPPIConfig(**d), IsaacGymConfig(), nu, K, [])
    p.k_offset = k_offset
    return p


def backend(nu, p, state):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(nu_model(nu), p)
    if state is not None:
        be.set_smooth_state(state)
    return be


def device_white(nu, p, seed, plan, K):
    """The device's own white draws z[T][nu][K] (the Gaussian K1 with identity colour, no bounds, no null row)."""
    w = copy.deepcopy(p)
    w.mode, w.sample_null_action, w.smooth_weight = MODE_SIMPLE, 0, 0.0
    for j in range(nu):
        w.u_min[j], w.u_max[j] = -3e38, 3e38
        for i in range(nu):
            w.sigma_chol[j * nu + i] = 1.0 if i == j else 0.0
    be = backend(nu, w, None)
    z = torch.zeros((p.T, nu, K), device=DEV)
    be.sample(seed, plan, 0, K, torch.zeros((p.T, nu), device=DEV), None, z, None)
    return z.cpu().numpy()


def run_k1(nu, p, U, state, seed=11, plan=3, k_offset=0, k_total=None):
    be = backend(nu, p, dev(state))
    K = p.K
    a, n = torch.zeros((p.T, nu, K), device=DEV), torch.zeros((p.T, nu, K), device=DEV)
    be.sample_smooth(seed, plan, k_offset, k_total or K, dev(U), a, n)
    return a.cpu().numpy(), n.cpu().numpy()


def k1_gate(nu, p, U, z, state):
    """|a_gpu - a64| per element: every step adds the rounding of the fmaf (eps (|a_t| + dt |v_t|)) and dt times the error of v, which is
    the colour sum over i <= j (nu + 1 roundings of |L z| terms) and u + n (one more); the clamps are 1-Lipschitz."""
    T = p.T
    L = np.abs(np.array(p.sigma_chol[:nu * nu], np.float32).reshape(nu, nu).astype(np.float64))
    Ln = np.einsum("ji,tik->tjk", L, np.abs(z.astype(np.float64)))
    dt = float(np.float32(p.dt))
    ev = (nu + 2) * EPS * (np.abs(U.astype(np.float64))[:, :, None] + Ln)
    a, _ = so.sample(p, nu, U, z, state, 0, p.K)
    vmax = np.abs(U.astype(np.float64))[:, :, None] + Ln
    step = EPS * (np.abs(a.astype(np.float64)) + dt * vmax) + dt * ev
    return 2 * np.cumsum(step, 0) + 1e-30


@pytest.mark.parametrize("nu, T, K", [(7, 30, 10000), (9, 30, 4096), (2, 256, 200), (16, 32, 100)])
def test_k1_noise_is_the_gaussian_k1s_bit_for_bit(nu, T, K):
    """Without a binding action clamp the noise is v - U with v = clamp(U + L0 z, du_min, du_max): mppib_sample with u_min / u_max :=
    du_min / du_max draws the same bits."""
    p = smooth_params(nu, T, K, u_min=[-1e30], u_max=[1e30], du_min=[-0.4], du_max=[0.5])
    rng = np.random.default_rng(T)
    U = rng.uniform(-0.3, 0.3, (T, nu)).astype(np.float32)
    st = so.make_state(p, nu, rng.uniform(-0.1, 0.1, nu))
    _, n = run_k1(nu, p, U, st)
    w = copy.deepcopy(p)
    w.mode = MODE_SIMPLE
    for j in range(nu):
        w.u_min[j], w.u_max[j] = p.du_min[j], p.du_max[j]
    be = backend(nu, w, None)
    a2, n2 = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    be.sample(11, 3, 0, K, dev(U), None, a2, n2)
    np.testing.assert_array_equal(n.view(np.uint32), n2.cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("bounds", ["free", "action", "derivative", "both"])
@pytest.mark.parametrize("nu, T, K", [(7, 30, 10000), (9, 30, 2048), (3, 128, 500)])
def test_k1_actions_match_the_float64_prefix(nu, T, K, bounds):
    kw = dict(free=dict(u_min=[-1e30], u_max=[1e30], du_min=None, du_max=None), action=dict(u_min=[-0.05], u_max=[0.08], du_min=None, du_max=None),
              derivative=dict(u_min=[-1e30], u_max=[1e30], du_min=[-0.3], du_max=[0.2]),
              both=dict(u_min=[-0.05], u_max=[0.05], du_min=[-0.6], du_max=[0.4]))[bounds]
    p = smooth_params(nu, T, K, **kw)
    rng = np.random.default_rng(K)
    U = rng.uniform(-0.4, 0.4, (T, nu)).astype(np.float32)
    st = so.make_state(p, nu, rng.uniform(-0.04, 0.04, nu))
    a, n = run_k1(nu, p, U, st)
    z = device_white(nu, p, 11, 3, K)
    a_ref, n_ref = so.sample(p, nu, U, z, st, 0, K)
    gate = k1_gate(nu, p, U, z, st)
    err = np.abs(a.astype(np.float64) - a_ref)
    print(f"SMOOTH K1 {bounds} nu{nu} T{T} K{K}: worst |a err| {err.max():.2e}, worst err/gate {(err / gate).max():.3f}")
    assert np.all(err <= gate)
    lo, hi, dlo, dhi = so.bounds(p, nu)
    assert np.all(a >= lo[None, :, None]) and np.all(a <= hi[None, :, None])
    v = n.astype(np.float64) + U[:, :, None]
    assert np.all(v >= dlo[None, :, None] - 1e-6) and np.all(v <= dhi[None, :, None] + 1e-6)
    # the applied derivative: where the action clamp did not bind it is the sampled v; everywhere, a_t - a_{t-1} = dt v_t up to the
    # rounding of the step
    prev = np.concatenate([np.broadcast_to(st[:nu, None], (1, nu, K)), a[:-1]]).astype(np.float64)
    dt = float(np.float32(p.dt))
    np.testing.assert_allclose(a - prev, dt * v, rtol=0, atol=4 * EPS * (np.abs(a).max() + dt * (np.abs(v).max() + np.abs(U).max())) + 1e-12)
    if bounds in ("action", "both"):
        assert np.mean(a == hi[None, :, None]) + np.mean(a == lo[None, :, None]) > 0.01      # the action clamp binds somewhere
    if bounds in ("derivative", "both"):
        assert np.mean(np.isclose(v, dhi[None, :, None], atol=1e-6)) > 0.01
    np.testing.assert_allclose(n, n_ref, rtol=0, atol=2 * gate.max() / dt + 1e-5)


def test_k1_null_row_holds_the_previous_action_and_shards_are_columns():
    nu, T, K = 7, 30, 1000
    p = smooth_params(nu, T, K)
    rng = np.random.default_rng(5)
    U = rng.uniform(-0.4, 0.4, (T, nu)).astype(np.float32)
    st = so.make_state(p, nu, rng.uniform(-0.1, 0.1, nu))
    a, n = run_k1(nu, p, U, st)
    np.testing.assert_array_equal(a[:, :, K - 1], np.broadcast_to(st[:nu], (T, nu)))
    np.testing.assert_array_equal(n[:, :, K - 1], -U)
    for lo, hi in ((0, 200), (200, 612), (612, 1000)):
        ps = smooth_params(nu, T, hi - lo, k_offset=lo)
        a_s, n_s = run_k1(nu, ps, U, st, k_offset=lo, k_total=K)
        np.testing.assert_array_equal(a_s, a[:, :, lo:hi])
        np.testing.assert_array_equal(n_s, n[:, :, lo:hi])


def test_k1_refusals():
    nu, T, K = 7, 12, 64
    p = smooth_params(nu, T, K)
    be = backend(nu, p, None)
    a = torch.zeros((T, nu, K), device=DEV)
    with pytest.raises(RuntimeError, match="no smooth state"):
        be.sample_smooth(1, 0, 0, K, torch.zeros((T, nu), device=DEV), a, a.clone())
    be.set_smooth_state(dev(so.make_state(p, nu)))
    with pytest.raises(RuntimeError, match="mode smooth"):
        be.sample(1, 0, 0, K, torch.zeros((T, nu), device=DEV), None, a, a.clone())
    with pytest.raises(RuntimeError, match="mode smooth"):
        be.sample_colored(1, 0, 0, K, torch.zeros((T, nu), device=DEV), None, torch.eye(T, device=DEV), a, a.clone())
    w = copy.deepcopy(p)
    w.mode = MODE_SIMPLE
    be2 = backend(nu, w, dev(so.make_state(p, nu)))
    with pytest.raises(RuntimeError, match="needs mode smooth"):
        be2.sample_smooth(1, 0, 0, K, torch.zeros((T, nu), device=DEV), a, a.clone())
    be3 = backend(nu, p, None)
    with pytest.raises(RuntimeError, match="needs its state registered"):
        be3.reduce(torch.zeros((T, K), device=DEV), a, torch.zeros((T, nu), device=DEV), torch.zeros(2 + T * nu, device=DEV))


# (T, nu) cells of the SIMPLE K3 sweep: T*nu = 128 (RPL 4), 129 / 256 (RPL 8), 258 / 259 / 512 (RPL 16)
K3_CELLS = [(32, 4), (43, 3), (16, 16), (129, 2), (37, 7), (32, 16), (30, 7)]


def k3_inputs(T, nu, K, seed):
    rng = np.random.default_rng(seed)
    cost = rng.uniform(0.0, 0.05, (T, K)).astype(np.float32)
    x = rng.normal(0.0, 0.4, (T, nu, K)).astype(np.float32)
    U = rng.uniform(-0.3, 0.3, (T, nu)).astype(np.float32)
    return cost, x, U


def k3_gates(p, nu, cost, x, U):
    """Per-sample bound E_k on |S_gpu - S64| (four FMA chains of T and T*nu terms, g = lambda Sigma^-1 U from nu + 1 roundings, the
    square terms from two roundings each, omega dt^2 from two, the final fma and adds), and the row gate: w_k carries (E_k + E_max)/lambda
    relative error and the float32 sums over K at most 256 eps relative."""
    T = p.T
    NR = T * nu
    c = np.abs(cost.astype(np.float64)).reshape(T, -1)
    xr = x.astype(np.float64).reshape(NR, -1)
    Uf = U.astype(np.float64).reshape(T, nu)
    Sinv = np.abs(np.array(p.sigma_inv[:nu * nu], np.float32).reshape(nu, nu).astype(np.float64))
    g = float(np.float32(p.lambda_)) * (np.abs(Uf) @ Sinv.T).reshape(-1)
    wq = float(np.float32(p.smooth_weight)) * float(np.float32(p.dt)) ** 2
    q = ((Uf.reshape(-1, 1) + xr) ** 2).sum(0)
    E = EPS * ((T / 4 + 4) * c.sum(0) + (NR / 4 + nu + 6) * (g @ np.abs(xr)) + (NR / 4 + 8) * wq * q)
    S = so.scores(p, nu, cost, x, U)
    E = 2 * (E + 4 * EPS * np.abs(S))
    lam = float(np.float32(p.lambda_))
    w = np.exp(-(S - S.min()) / lam)
    rel = (E + E.max()) / lam + 256 * EPS
    gate = np.concatenate([[E.max(), (w * rel).sum()], np.abs(xr) @ (w * rel)])
    return gate


def run_k3(nu, p, cost, x, U, state, fused=False):
    be = backend(nu, p, dev(state) if state is not None else None)
    part, Ud = torch.zeros(2 + p.T * nu, device=DEV), dev(U)
    act, st = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    if fused:
        be.reduce_finalize(dev(cost), dev(x), Ud, part, act, st)
    else:
        be.reduce(dev(cost), dev(x), Ud, part)
    return part.cpu().numpy(), be, Ud, act, st


@pytest.mark.parametrize("omega", [0.0, 0.5, 10.0])
@pytest.mark.parametrize("K", [36, 10000])
@pytest.mark.parametrize("T, nu", K3_CELLS)
def test_k3_row_against_float64(T, nu, K, omega):
    p = smooth_params(nu, T, K, smooth_weight=omega)
    cost, x, U = k3_inputs(T, nu, K, 7 * T + nu + K)
    st = so.make_state(p, nu)
    row = run_k3(nu, p, cost, x, U, st)[0]
    ref = so.reduce(p, nu, cost, x, U).astype(np.float64)
    gate = k3_gates(p, nu, cost, x, U)
    err = np.abs(row.astype(np.float64) - ref)
    print(f"SMOOTH K3 T{T} nu{nu} K{K} omega {omega}: worst err/gate {(err / gate).max():.3f}")
    assert np.all(err <= gate)
    if omega == 0.0:                                                      # the smooth K3 without its term is SIMPLE's, bit for bit
        w = copy.deepcopy(p)
        w.mode = MODE_SIMPLE
        row_simple = run_k3(nu, w, cost, x, U, None)[0]
        np.testing.assert_array_equal(row.view(np.uint32), row_simple.view(np.uint32))
    else:                                                                  # ... and with it the row moves beyond the gate
        w = copy.deepcopy(p)
        w.smooth_weight = 0.0
        assert np.any(np.abs(so.reduce(w, nu, cost, x, U).astype(np.float64) - ref) > gate)


def k4_check(p, nu, row, U, st, Ug, stg, act):
    """K4 on the device's rows against the oracle: U' carries 4 eps (|U| + |W/eta|) (the clamp and the projection keep it within dt^-1
    times the action's error), A accumulates eps (|A| + dt |U'|) + dt times that per step."""
    U_ref, act_ref, stats_ref, st_ref = so.finalize(p, nu, row, U, st)
    rows = np.asarray(row, np.float64).reshape(-1, 2 + p.T * nu)
    e = max(float(stats_ref[1]), 1e-30)
    dt = float(np.float32(p.dt))
    W = np.abs(rows[:, 2:]).max() / e if stats_ref[1] > 0 else 0.0
    gu = 8 * EPS * (np.abs(U).max() + W + np.abs(U_ref).max()) * max(1, rows.shape[0])
    A_ref = so.unpack(st_ref, p.T, nu)[1].astype(np.float64)
    gA = np.cumsum(2 * EPS * (np.abs(A_ref) + dt * np.abs(U_ref)) + dt * gu, 0)
    A = so.unpack(stg, p.T, nu)[1].astype(np.float64)
    assert np.all(np.abs(A - A_ref) <= gA), np.abs(A - A_ref).max()
    assert np.all(np.abs(Ug - U_ref) <= gu + gA / dt), np.abs(Ug - U_ref).max()
    np.testing.assert_array_equal(act, so.unpack(stg, p.T, nu)[1][0])
    np.testing.assert_array_equal(stg[:nu], act)


@pytest.mark.parametrize("what", ["plain", "action_bound", "derivative_bound", "eta0"])
@pytest.mark.parametrize("T, nu", [(30, 7), (43, 3), (32, 16)])
def test_k4_against_the_oracle_and_fused_equals_split(T, nu, what):
    K = 4096
    kw = dict(plain={}, action_bound=dict(u_min=[-0.01], u_max=[0.01]), derivative_bound=dict(du_min=[-0.05], du_max=[0.02]), eta0={})[what]
    p = smooth_params(nu, T, K, **kw)
    cost, x, U = k3_inputs(T, nu, K, T + nu)
    if what == "eta0":
        cost[0, :] = np.nan                                              # no valid sample: eta = 0, U kept, still integrated
    st = so.make_state(p, nu, np.random.default_rng(1).uniform(-0.01, 0.01, nu))
    out = []
    for fused in (False, True):
        stg = dev(st)
        be = backend(nu, p, stg)
        part, Ud = torch.zeros(2 + T * nu, device=DEV), dev(U)
        act, stats = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        if fused:
            be.reduce_finalize(dev(cost), dev(x), Ud, part, act, stats)
        else:
            be.reduce(dev(cost), dev(x), Ud, part)
            be.finalize(part.view(1, -1), 1, Ud, act, stats)
        out.append([t.cpu().numpy() for t in (part, Ud, act, stats, stg)])
    for a, b in zip(*out):
        np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))
    part, Ug, act, stats, stg = out[0]
    np.testing.assert_array_equal(stats, part[:2])
    if what == "eta0":
        assert stats[1] == 0.0
    k4_check(p, nu, part[None], U, st, Ug, stg, act)
    if what == "action_bound":
        assert np.any(np.abs(so.unpack(stg, T, nu)[1]) == np.float32(0.01))


@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_k4_merges_shard_rows(G):
    """K3 on G shards (global k_offset), K4 on their G rows: the oracle's merge within its gate, and padding the rows with empty shards
    (eta = 0), which every rank of a larger world would see, changes no bit of U, A and the action."""
    nu, T, K = 7, 30, 8192
    p = smooth_params(nu, T, K)
    cost, x, U = k3_inputs(T, nu, K, G)
    st = so.make_state(p, nu)
    b = np.linspace(0, K, G + 1).astype(int)
    rows = []
    for lo, hi in zip(b[:-1], b[1:]):
        ps = smooth_params(nu, T, hi - lo, k_offset=lo)
        row = run_k3(nu, ps, np.ascontiguousarray(cost[:, lo:hi]), np.ascontiguousarray(x[:, :, lo:hi]), U, st)[0]
        rows.append(row)
    rows = np.stack(rows)
    res = []
    for pad in (0, 8 - G):
        rr = np.concatenate([rows, np.tile(np.array([np.inf, 0.0] + [0.0] * (T * nu), np.float32), (pad, 1))])
        stg, Ud = dev(st), dev(U)
        be = backend(nu, p, stg)
        act, stats = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        be.finalize(dev(rr), len(rr), Ud, act, stats)
        res.append([t.cpu().numpy() for t in (Ud, act, stg)])
    for a, b2 in zip(*res):
        np.testing.assert_array_equal(a.view(np.uint32), b2.view(np.uint32))
    Ug, act, stg = res[0]
    k4_check(p, nu, rows, U, st, Ug, stg, act)


def _planners(K=256, T=30, **kw):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    d = dict(mppi_mode="smooth", sampling_method="random", filter_u=False, smooth_weight=0.5, du_min=[-1.0], du_max=[1.0])
    d.update(kw)
    gpu = MPPIisaacPlanner(panda_cfg(K=K, T=T, device=DEV, **d), PandaReachObjective(), use_cuda_graph=False)
    cpu = MPPIisaacPlanner(panda_cfg(K=K, T=T, device="cpu", **d), PandaReachObjective(), backend=so.SmoothOracleBackend())
    return gpu, cpu


def test_panda_reach_plan_agrees_with_the_oracle_pipeline():
    gpu, cpu = _planners()
    for it in range(3):
        a_gpu = gpu.compute_action(Q0, [0.0] * 7)
        a_cpu = cpu.compute_action(Q0, [0.0] * 7)
        err = (a_gpu - a_cpu).abs().max().item()
        print(f"SMOOTH plan {it}: |action_gpu - action_oracle| = {err:.2e}")
        assert err < 2e-4
        np.testing.assert_allclose(gpu.mppi.action_sequence.cpu().numpy(), cpu.mppi.action_sequence.numpy(), rtol=0, atol=5e-4)


def test_graph_replay_equals_the_eager_plan():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    d = dict(mppi_mode="smooth", sampling_method="random", filter_u=False, smooth_weight=0.5, du_min=[-1.0], du_max=[1.0])
    pls = [MPPIisaacPlanner(panda_cfg(K=10000, T=30, device=DEV, **d), PandaReachObjective(), use_cuda_graph=g) for g in (True, False)]
    for _ in range(4):
        a, b = (pl.compute_action(Q0, [0.0] * 7).numpy() for pl in pls)
        np.testing.assert_array_equal(a, b)
    assert pls[0].mppi._graph is not None and pls[1].mppi._graph is None
    np.testing.assert_array_equal(pls[0].mppi.smooth_state.cpu().numpy(), pls[1].mppi.smooth_state.cpu().numpy())
    np.testing.assert_array_equal(pls[0].mppi.U.cpu().numpy(), pls[1].mppi.U.cpu().numpy())


def test_rate_bound_holds_over_50_device_plans():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    cfg = panda_cfg(K=10000, T=30, device=DEV, mppi_mode="smooth", sampling_method="random", filter_u=False, du_min=[-0.4], du_max=[0.4],
                    sample_null_action=False, noise_sigma=(4.0 * np.eye(7)).tolist())
    pl = MPPIisaacPlanner(cfg, PandaReachObjective())
    bound = 0.4 * float(np.float32(cfg.isaacgym.dt)) * (1 + 1e-5)
    prev = np.zeros(7, np.float32)
    jumps = []
    for _ in range(50):
        a = pl.compute_action(Q0, [0.0] * 7).numpy()
        jumps.append(float(np.abs(a - prev).max()))
        prev = a
    print(f"SMOOTH rate bound: worst step {max(jumps):.4g} of du_max dt = {bound:.4g}")
    assert max(jumps) <= bound and max(jumps) > 0.25 * bound
