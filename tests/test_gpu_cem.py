"""-m gpu: cross-entropy planning (``mppi_mode: cem``) on the device against the float64 reference of ``cem_oracle``: exact elite
selection, K4, shard invariance, the CEM K1 and shift, and whole plans through the planner."""
import copy

import numpy as np
import pytest
import torch

import cem_oracle as ce
from mppi_isaac_b200.model.blob import make_params
from mppi_isaac_b200.utils.config_store import IsaacGymConfig
from mppi_isaac_b200.planner.mppi import colored_noise_chol
from scenes import panda_cfg, panda_mppi, panda_scene, pick_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
EPS = 2.0 ** -24
NU = 7


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def cem_params(K, T, E, keep=0, alpha=0.1, k_offset=0, **kw):
    """The panda parameter block in mode cem; E and keep set directly, so that shards smaller than E are accepted."""
    sc = panda_scene()
    p = make_params(panda_mppi(max(K, 256), T, mode="cem", **kw), IsaacGymConfig(), NU, K, [])
    p.n_elites, p.n_keep, p.elite_alpha, p.k_offset = E, keep, alpha, k_offset
    return sc, p


def backend(sc, p, state):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(sc.model, p)
    be.set_distribution(state)
    return be


def device_white(sc, p, seed, plan, K):
    """The device's own white draws z[T][nu][K] (the fixed-Sigma K1 with identity colour, no bounds, no null row), so that the K1
    reference differs from the kernel by its summation order alone, not by the libm of the Box-Muller transform."""
    from mppi_isaac_b200.backend import CudaBackend
    w = copy.deepcopy(p)
    w.mode, w.sample_null_action = 0, 0
    for j in range(NU):
        w.u_min[j], w.u_max[j] = -3e38, 3e38
        for i in range(NU):
            w.sigma_chol[j * NU + i] = 1.0 if i == j else 0.0
    be = CudaBackend(DEV)
    be.create(sc.model, w)
    z = torch.zeros((p.T, NU, K), device=DEV)
    be.sample(seed, plan, 0, K, torch.zeros((p.T, NU), device=DEV), None, z, None)
    return z.cpu().numpy()


def row_of(be, cost, actions):
    P = ce.row_floats(be.params.T, NU, be.params.n_elites)
    part = torch.full((P,), 7.0, device=DEV)
    be.reduce(dev(cost), dev(actions), torch.zeros((be.params.T, NU), device=DEV), part)
    return part.cpu().numpy()


def costs(kind, T, K, rng):
    if kind == "ties":
        c = rng.integers(0, 8, (T, K)).astype(np.float32)
    elif kind == "equal":
        c = np.ones((T, K), np.float32)
    else:
        c = rng.standard_normal((T, K)).astype(np.float32)
    if kind in ("ties", "nonfinite"):
        bad = rng.integers(0, K, max(1, K // 7))
        c[0, bad] = rng.choice(np.array([np.nan, np.inf, -np.inf], np.float32), bad.size)
    return c


@pytest.mark.parametrize("K", [4, 130, 10000, 65536, 262144])
@pytest.mark.parametrize("E", [1, 10, 33, 128])
@pytest.mark.parametrize("kind", ["ties", "nonfinite", "equal", "random"])
def test_selection_is_exact(K, E, kind):
    """T = 1: S is the cost itself, so the shard row must equal the NumPy lexsort's bit for bit, gathered actions included."""
    rng = np.random.default_rng(K + E)
    sc, p = cem_params(K, 1, E)
    be = backend(sc, p, dev(ce.make_state(np.full(NU, 0.1), 1, NU, E)))
    cost = costs(kind, 1, K, rng)
    actions = rng.standard_normal((1, NU, K)).astype(np.float32)
    got = row_of(be, cost, actions)
    want = ce.elite_row(p, NU, cost, actions, 0)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("T, K, E", [(30, 10000, 10), (30, 65536, 128), (7, 1000, 33)])
def test_selection_over_the_horizon_within_the_float32_bound(T, K, E):
    """T > 1: S_k is T fused multiply-adds in t order with gamma^t from exp2f (a few ulp), so |S_gpu - S| <= (T + 4) eps sum_t
    gamma^t |c|; every elite's S must lie within that of the float64 S of its index, and no non-elite may beat the E-th by more."""
    rng = np.random.default_rng(T)
    sc, p = cem_params(K, T, E)
    be = backend(sc, p, dev(ce.make_state(np.full(NU, 0.1), T, NU, E)))
    cost = rng.uniform(0, 2, (T, K)).astype(np.float32)
    actions = rng.standard_normal((T, NU, K)).astype(np.float32)
    got = row_of(be, cost, actions)
    S = ce.scores(p, cost)
    bound = (T + 4) * EPS * ((np.float64(np.float32(p.gamma)) ** np.arange(T))[:, None] * np.abs(cost.astype(np.float64))).sum(0)
    idx = got[1:2 * E:2].view(np.uint32).astype(np.int64)
    Sg = got[0:2 * E:2].astype(np.float64)
    assert np.all(np.abs(Sg - S[idx]) <= bound[idx]), np.max(np.abs(Sg - S[idx]) / bound[idx])
    assert np.all(np.diff(Sg) >= 0) and len(set(idx)) == E
    others = np.setdiff1d(np.arange(K), idx)
    assert np.all(S[others] + bound[others] >= Sg[-1] - bound[idx[-1]])
    for e, k in enumerate(idx):
        np.testing.assert_array_equal(got[2 * E + e * T * NU:2 * E + (e + 1) * T * NU], actions[:, :, k].ravel())


@pytest.mark.parametrize("E, filt", [(1, False), (10, True), (128, False)])
def test_finalize_against_the_float64_oracle(E, filt):
    """K4 on G = 3 random shard rows: m is a float32 sum of E values divided by E, s the sqrt of such a sum, so |m - m64| <= (E + 1)
    eps max|a| and |s - s64| <= sqrt((E + 3) eps) max|a - m| + ...; the gate below is (E + 4) eps max|a| on U and sqrt of that scale
    (times 4 max|a|) on sigma, applied after the momentum step.  The elites and their S are copied, so they must be exact."""
    T, K = 30, 4096
    rng = np.random.default_rng(E)
    sc, p = cem_params(K, T, E, alpha=0.3, filter_u=filt)
    st = ce.make_state(np.full(NU, 0.1), T, NU, E)
    rows = []
    for g in range(3):
        p_g = copy.deepcopy(p)
        p_g.k_offset = g * K
        cost = rng.uniform(0, 1, (T, K)).astype(np.float32)
        rows.append(ce.elite_row(p_g, NU, cost, rng.uniform(-0.2, 0.2, (T, NU, K)).astype(np.float32), g * K))
    rows = np.stack(rows)
    U0 = rng.uniform(-0.1, 0.1, (T, NU)).astype(np.float32)
    Uw, aw, sw, stw = ce.finalize(p, NU, rows, U0, st)
    d_st = dev(st)
    be = backend(sc, p, d_st)
    U, act, stats = dev(U0), torch.zeros(NU, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(dev(rows), 3, U, act, stats)
    got = d_st.cpu().numpy()
    amax = 0.2
    gate_u = (E + 4) * EPS * amax * (4 if filt else 1) + 2 * EPS * amax
    assert np.abs(U.cpu().numpy() - Uw).max() <= gate_u
    sg, sw_ = ce.unpack(got, T, NU, E)[3], ce.unpack(stw, T, NU, E)[3]
    assert np.abs(sg - sw_).max() <= 4 * amax * np.sqrt((E + 4) * EPS)
    np.testing.assert_array_equal(ce.unpack(got, T, NU, E)[4], ce.unpack(stw, T, NU, E)[4])
    np.testing.assert_array_equal(got[:2 + E], stw[:2 + E])
    np.testing.assert_array_equal(stats.cpu().numpy(), sw)
    np.testing.assert_array_equal(act.cpu().numpy(), U.cpu().numpy()[0])


@pytest.mark.parametrize("K, E", [(10000, 10), (65536, 128), (1024, 33)])
def test_shards_and_the_fused_launch_are_bit_identical(K, E):
    """Shards at k_offset splits combined by mppib_finalize give the same U, sigma, elites and stats for G in {1, 2, 4, 8}, and
    mppib_reduce_finalize gives what mppib_reduce + mppib_finalize give."""
    T = 30
    rng = np.random.default_rng(K)
    cost = rng.integers(0, 50, (T, K)).astype(np.float32)                  # ties across shards
    actions = rng.uniform(-0.2, 0.2, (T, NU, K)).astype(np.float32)
    st0 = ce.make_state(np.full(NU, 0.1), T, NU, E)
    U0 = rng.uniform(-0.1, 0.1, (T, NU)).astype(np.float32)
    out = {}
    for G in (1, 2, 4, 8):
        cuts = np.linspace(0, K // 4, G + 1).astype(int) * 4
        rows = []
        for g in range(G):
            a, b = cuts[g], cuts[g + 1]
            sc, p = cem_params(b - a, T, E, keep=E // 3, k_offset=a)
            be = backend(sc, p, dev(st0))
            rows.append(row_of(be, cost[:, a:b], actions[:, :, a:b]))
        sc, p = cem_params(K, T, E, keep=E // 3)
        st = dev(st0)
        be = backend(sc, p, st)
        U, act, stats = dev(U0), torch.zeros(NU, device=DEV), torch.zeros(2, device=DEV)
        be.finalize(dev(np.stack(rows)), G, U, act, stats)
        out[G] = (U.cpu().numpy(), st.cpu().numpy(), stats.cpu().numpy())
    for G in (2, 4, 8):
        for x, y in zip(out[1], out[G]):
            np.testing.assert_array_equal(x.view(np.uint32), y.view(np.uint32))
    sc, p = cem_params(K, T, E, keep=E // 3)
    st = dev(st0)
    be = backend(sc, p, st)
    U, act, stats = dev(U0), torch.zeros(NU, device=DEV), torch.zeros(2, device=DEV)
    part = torch.zeros(ce.row_floats(T, NU, E), device=DEV)
    be.reduce_finalize(dev(cost), dev(actions), U, part, act, stats)
    for x, y in zip(out[1], (U.cpu().numpy(), st.cpu().numpy(), stats.cpu().numpy())):
        np.testing.assert_array_equal(x.view(np.uint32), y.view(np.uint32))


def test_k1_draws_carried_rows_and_the_colored_draws_before_any_elite():
    T, K, E, keep = 30, 10000, 10, 3
    sc, p = cem_params(K, T, E, keep=keep)
    Lt = colored_noise_chol(T, 2.0)
    U0 = np.random.default_rng(1).uniform(-0.05, 0.05, (T, NU)).astype(np.float32)
    st0 = ce.make_state(np.full(NU, 0.1), T, NU, E)
    # before any elite the CEM draw on a diagonal Sigma is mppib_sample_colored's, bit for bit
    be = backend(sc, p, dev(st0))
    a_cem, n_cem = torch.zeros((T, NU, K), device=DEV), torch.zeros((T, NU, K), device=DEV)
    ctr = torch.tensor([4], dtype=torch.int32, device=DEV)
    be.sample_colored(99, 3 << 32, 0, K, dev(U0), None, dev(Lt), a_cem, n_cem, ctr)
    p_col = copy.deepcopy(p)
    p_col.mode = 0
    from mppi_isaac_b200.backend import CudaBackend
    bc = CudaBackend(DEV)
    bc.create(sc.model, p_col)
    a_col, n_col = torch.zeros_like(a_cem), torch.zeros_like(a_cem)
    bc.sample_colored(99, 3 << 32, 0, K, dev(U0), None, dev(Lt), a_col, n_col, ctr)
    assert torch.equal(a_cem, a_col) and torch.equal(n_cem, n_col)
    # against the float64 restatement with a live sigma and carried elites (shifted)
    rng = np.random.default_rng(2)
    st = st0.copy()
    _, _, _, sig, el = ce.unpack(st, T, NU, E)
    sig[:] = rng.uniform(0.01, 0.3, sig.shape).astype(np.float32)
    el[:] = rng.uniform(-0.3, 0.3, el.shape).astype(np.float32)
    st[0], st[1] = 1.0, 1.0
    be = backend(sc, p, dev(st))
    a, n = torch.zeros((T, NU, K), device=DEV), torch.zeros((T, NU, K), device=DEV)
    be.sample_colored(99, 1 << 32, 0, K, dev(U0), None, dev(Lt), a, n, ctr)
    z = device_white(sc, p, 99, (1 << 32) + 4, K)
    a_ref, _ = ce.sample(p, NU, U0, z, Lt, st, 0, K)
    a = a.cpu().numpy()
    w = np.abs(np.einsum("ts,sik->tik", np.abs(Lt.astype(np.float64)), np.abs(z.astype(np.float64))))
    # temporal sum of t + 1 FMA (t + 1) eps sigma sum|L z|, the product sigma w and the sum U + n one rounding each, the reference's
    # own rounding to float32 one more: the gate is eps ((t + 3) sigma sum|L||z| + |U| + 2 |a|)
    gate = EPS * ((np.arange(T) + 3)[:, None, None] * sig.astype(np.float64)[:, :, None] * w + np.abs(U0)[:, :, None] + 2 * np.abs(a_ref))
    assert np.all(np.abs(a - a_ref) <= gate), np.max(np.abs(a - a_ref) / gate)
    lo, hi = ce.bounds(p, NU)
    for e in range(keep):
        np.testing.assert_array_equal(a[:T - 1, :, K - 3 - e], np.clip(el[e, 1:], lo, hi))
    np.testing.assert_array_equal(n.cpu().numpy(), a - U0[:, :, None])


def test_shift_resets_sigma_sets_the_offset_and_bumps_the_counter():
    T, E = 12, 4
    sc, p = cem_params(64, T, E)
    st = ce.make_state(np.full(NU, 0.1), T, NU, E)
    st[2 + E:2 + E + T * NU] = 3.0
    d = dev(st)
    be = backend(sc, p, d)
    U = dev(np.arange(T * NU, dtype=np.float32).reshape(T, NU))
    ctr = torch.tensor([7], dtype=torch.int32, device=DEV)
    be.shift(U, ctr)
    Uw, stw = ce.shift(p, NU, np.arange(T * NU, dtype=np.float32).reshape(T, NU), st)
    np.testing.assert_array_equal(U.cpu().numpy(), Uw)
    np.testing.assert_array_equal(d.cpu().numpy(), stw)
    assert int(ctr[0]) == 8


@pytest.mark.parametrize("task", ["panda", "pick"])
def test_plan_through_planner_matches_the_oracle_pipeline(task):
    """I = 3 plans on the GPU (CUDA graph) against the checker backend in lock step (U, state and counter copied before each plan),
    with the gates of the colored plan-parity test."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaPickObjective, PandaReachObjective
    kw = dict(mppi_mode="cem", sampling_method="colored", noise_beta=2.0, cem_iterations=3, n_elites=10, keep_elites=0.3)
    if task == "panda":
        mk, obj, q, plans, rel = (lambda d: panda_cfg(K=10000, T=30, device=d, **kw)), PandaReachObjective, Q0, 2, 2e-4
    else:
        mk, obj, q, plans, rel = (lambda d: pick_cfg(K=1024, T=30, device=d, **kw)), PandaPickObjective, Q0 + [0.02, 0.02], 1, 2e-2
    gpu = MPPIisaacPlanner(mk(DEV), obj(), use_cuda_graph=True)
    cpu = MPPIisaacPlanner(mk("cpu"), obj(), backend=ce.CemOracleBackend(nthreads=8))
    lim = float(gpu.mppi.backend.params.u_max[0])
    for it in range(plans):
        cpu.mppi.U.copy_(gpu.mppi.U.cpu())
        cpu.mppi.dist.copy_(gpu.mppi.dist.cpu())
        cpu.mppi.plan_ctr.copy_(gpu.mppi.plan_ctr.cpu())
        ag, ac = gpu.compute_action(q, [0.0] * len(q)), cpu.compute_action(q, [0.0] * len(q))
        assert torch.isfinite(ag).all()
        err = float((ag.cpu() - ac).abs().max())
        print(f"CEM plan {task} {it}: |a_gpu - a_oracle| {err:.2e}, stats gpu {gpu.mppi.stats.cpu().tolist()} cpu {cpu.mppi.stats.tolist()}")
        assert err <= rel * max(1.0, lim), f"plan {it}"
    assert gpu.mppi._graph is not None


def test_graph_replay_equals_the_eager_plan_and_the_best_cost_never_rises():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    kw = dict(mppi_mode="cem", sampling_method="colored", cem_iterations=3, n_elites=10, keep_elites=0.3)
    g = MPPIisaacPlanner(panda_cfg(K=10000, T=30, device=DEV, **kw), PandaReachObjective(), use_cuda_graph=True)
    e = MPPIisaacPlanner(panda_cfg(K=10000, T=30, device=DEV, **kw), PandaReachObjective(), use_cuda_graph=False)
    for _ in range(3):
        ag, ae = g.compute_action(Q0, [0.0] * 7), e.compute_action(Q0, [0.0] * 7)
        assert torch.equal(ag, ae)
        assert torch.equal(g.mppi.U, e.mppi.U) and torch.equal(g.mppi.dist, e.mppi.dist)
    assert g.mppi._graph is not None
    # one plan iteration by iteration: a carried elite re-rolls to its own cost (no per-rollout randomisation in this scene)
    m = e.mppi                                                             # the world state of the last compute_action stays
    m.backend.shift(m.U, m.plan_ctr)
    best = []
    for i in range(3):
        m._iterate_batched(i)
        best.append(float(m.stats[0]))
    print("CEM best S per iteration", best)
    assert all(b <= a for a, b in zip(best, best[1:])), best

