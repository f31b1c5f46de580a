"""-m gpu: risk-aware MPPI (``n_worlds`` / ``cvar_alpha``) on the device: K1 is the plain K1 of the control samples repeated R times,
bit for bit, for every supported variant; K2 keys the randomisation by the world; K3's CVaR row against a float32 restatement and the
float64 reference; K4 fused against split; whole C3- and C4-shape plans against the ``RiskOracleBackend`` pipeline and graph replay."""
import copy

import numpy as np
import pytest
import torch

import risk_oracle as ro
from mppi_isaac_b200.model.blob import make_params
from mppi_isaac_b200.planner.mppi import colored_noise_chol, halton_spline_operator, halton_table
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from scenes import boxer_cfg, boxer_setup, push_cfg
from synth_mppi import nu_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 2.0 ** -24


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(DEV)


def params(nu, T, K, R=1, alpha=1.0, k_offset=0, **kw):
    d = dict(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.3 * np.eye(nu) + 0.05).tolist(),
             u_min=[-0.5], u_max=[0.5], lambda_=0.05, sample_null_action=True, n_worlds=R, cvar_alpha=alpha)
    d.update(kw)
    p = make_params(MPPIConfig(**d), IsaacGymConfig(), nu, K, [])
    p.k_offset = k_offset
    return p


def backend(nu, p, dist=None, model=None):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(model or nu_model(nu), p)
    if dist is not None:
        be.set_distribution(dist)
    return be


def dist_for(nu, kind):
    """(update_cov, cov_type) keys and the registered distribution of the diag / full adaptive paths (None: fixed Sigma)."""
    if kind == "fixed":
        return {}, None
    sig = 0.3 * np.eye(nu) + 0.05
    if kind == "diag":
        return dict(update_cov=True, noise_sigma=(0.3 * np.eye(nu)).tolist()), dev(np.concatenate([[0.05], 0.3 * np.ones(nu) + 0.01 * np.arange(nu)]))
    L = np.linalg.cholesky(sig)
    return dict(update_cov=True, cov_type="full"), dev(np.concatenate([[0.05], sig.ravel(), L.ravel(), np.linalg.inv(sig).ravel()]))


def k1(variant, nu, T, p, dist, U, k_offset, k_total):
    be = backend(nu, p, dist)
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


@pytest.mark.parametrize("variant, kind", [("random", "fixed"), ("random", "diag"), ("random", "full"), ("colored", "fixed"),
                                           ("colored", "diag"), ("halton", "fixed"), ("halton", "diag"), ("halton", "full")])
@pytest.mark.parametrize("R", [2, 8, 32])
def test_k1_is_the_repeated_plain_k1_bit_for_bit(variant, kind, R):
    nu, T, Kc = 5, 12, 96
    kw, dist = dist_for(nu, kind)
    U = dev(0.1 * np.sin(np.arange(T * nu)).reshape(T, nu))
    plain_a, plain_n = k1(variant, nu, T, params(nu, T, Kc, **kw), dist, U, 0, Kc)
    full_a, full_n = k1(variant, nu, T, params(nu, T, Kc * R, R, **kw), dist, U, 0, Kc * R)
    np.testing.assert_array_equal(full_a, np.repeat(plain_a, R, axis=-1))
    np.testing.assert_array_equal(full_n, np.repeat(plain_n, R, axis=-1))
    assert (full_a[:, :, -R:] == np.clip(0.0, -0.5, 0.5)).all()               # the null control is the last group
    off = 32 * R                                                              # a shard at k_offset != 0 is a slice of columns
    sh_a, sh_n = k1(variant, nu, T, params(nu, T, 32 * R, R, **kw), dist, U, off, Kc * R)
    np.testing.assert_array_equal(sh_a, full_a[:, :, off:off + 32 * R])
    np.testing.assert_array_equal(sh_n, full_n[:, :, off:off + 32 * R])


def test_k1_refuses_a_shard_that_splits_a_group():
    p = params(3, 4, 64, 8)
    be = backend(3, p)
    a = torch.zeros((4, 3, 64), device=DEV)
    with pytest.raises(RuntimeError, match="multiples"):
        be.sample(1, 0, 4, 128, torch.zeros((4, 3), device=DEV), None, a, None)
    be.destroy()


@pytest.mark.parametrize("team", ["0", "1"])
def test_k2_keys_the_randomisation_by_world(team, monkeypatch):
    monkeypatch.setenv("MPPIB_K2_TEAM", team)
    K, T, R = 64, 4, 8
    sc, p, s0 = boxer_setup(K=K, T=T, noise=True)
    p.n_worlds, p.risk_tail = R, 1
    a = np.zeros((T, 2, K), np.float32)
    a[:, 0] = 0.8
    outs = []
    for k_off, Kl in ((0, K), (16, K - 16)):
        q = copy.copy(p)
        q.K, q.k_offset = Kl, k_off
        be = backend(sc.nu, q, model=sc.model)
        obs = torch.zeros((be.obs_size(), T, Kl), device=DEV)
        be.rollout(dev(s0), None, dev(a[:, :, :Kl]), 0, T, obs, root0=dev(sc.root_state0))
        torch.cuda.synchronize()
        outs.append(obs.cpu().numpy())
        be.destroy()
    o = outs[0]
    for k in range(K):
        for k2 in range(k + 1, K):
            assert np.array_equal(o[..., k], o[..., k2]) == (k % R == k2 % R)
    np.testing.assert_array_equal(outs[1], o[..., 16:])                       # a k_offset shard sees the same worlds


def k3_case(nu, T, Kc, R, m, kind, seed, ninf=3):
    kw, dist = dist_for(nu, kind)
    p = params(nu, T, Kc * R, R, alpha=m / R, **kw)
    assert p.risk_tail == m
    rng = np.random.default_rng(seed)
    cost = rng.random((T, Kc * R)).astype(np.float32)
    cost[rng.integers(0, T, ninf), rng.integers(0, Kc * R, ninf)] = np.inf
    x = (0.2 * rng.standard_normal((T, nu, Kc * R))).astype(np.float32)
    U = (0.1 * rng.standard_normal((T, nu))).astype(np.float32) if T > 1 else np.zeros((T, nu), np.float32)
    return p, dist, cost, x, U


def run_k3(nu, p, dist, cost, x, U):
    be = backend(nu, p, dist)
    part = torch.zeros(be.partial_row_floats(), device=DEV)
    be.reduce(dev(cost), dev(x), dev(U), part)
    torch.cuda.synchronize()
    be.destroy()
    return part.cpu().numpy()


@pytest.mark.parametrize("R, m", [(2, 1), (2, 2), (8, 1), (8, 2), (8, 8), (32, 5), (32, 32)])
def test_k3_beta_is_the_float32_cvar_bit_for_bit(R, m):
    """T = 1 and U = 0: S equals the cost exactly, so beta = min over controls of the float32 CVaR restatement, bit for bit."""
    nu, Kc = 3, 4096 // R
    p, dist, cost, x, U = k3_case(nu, 1, Kc, R, m, "fixed", seed=R + m)
    row = run_k3(nu, p, dist, cost, x, U)
    r = ro.rho_f32(cost[0], R, m)
    assert row[0] == r[np.isfinite(r)].min()


@pytest.mark.parametrize("kind", ["fixed", "diag", "full"])
@pytest.mark.parametrize("R, m, T, nu", [(2, 1, 8, 3), (4, 3, 30, 4), (8, 2, 30, 7), (16, 16, 20, 12), (32, 4, 10, 12), (8, 8, 30, 9)])
def test_k3_row_against_float64(kind, R, m, T, nu):
    """RPL 4 / 8 / 16 (T*nu = 24 .. 270).  Gate: beta is the min of rho, whose float32 error is that of S (T + T*nu + 4 terms) and of
    the m-term tail sum: (T + T*nu + m + 8) eps sum|terms|; eta and W carry the weights' error exp'(.) |d rho| / lambda plus the float32
    sums over at most 4096 controls.  A reference that drops one tail term misses the beta gate by orders of magnitude."""
    Kc = 4096 // R
    p, dist, cost, x, U = k3_case(nu, T, Kc, R, m, kind, seed=T * R + m)
    row = run_k3(nu, p, dist, cost, x, U)
    ref = ro.reduce(p, nu, cost, x, U, None if dist is None else dist.cpu().numpy())
    lam = float(np.float32(p.lambda_)) if dist is None else float(dist[0])
    mag = float(np.where(np.isfinite(cost), np.abs(cost), 0).sum(0).max()) + 1.0
    gb = (T + T * nu + m + 8) * EPS * (mag + np.abs(x).sum((0, 1)).max() * 10)
    assert abs(float(row[0]) - float(ref[0])) <= gb
    gw = 64 * EPS * Kc + gb / lam * 2
    np.testing.assert_allclose(row[1], ref[1], rtol=gw, atol=0)
    np.testing.assert_allclose(row[2:], ref[2:], rtol=0, atol=gw * max(1.0, float(np.abs(ref[2:]).max())))
    if m > 1:                                                                 # the gate tells a reference with one tail term dropped
        pb = copy.copy(p)
        pb.risk_tail = m - 1
        assert abs(float(row[0]) - float(ro.reduce(pb, nu, cost, x, U, None if dist is None else dist.cpu().numpy())[0])) > gb


@pytest.mark.parametrize("G", [1, 2, 4])
def test_k4_fused_equals_split(G):
    nu, T, R = 4, 16, 8
    outs = []
    for fused in (True, False):
        p = params(nu, T, 1024 * R // G, R)
        be = backend(nu, p)
        rng = np.random.default_rng(G)
        U = dev((0.1 * rng.standard_normal((T, nu))).astype(np.float32))
        P = 2 + T * nu
        rows = torch.zeros((G, P), device=DEV)
        act, st = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        for g in range(G):
            cost = dev(rng.random((T, p.K)).astype(np.float32))
            x = dev((0.2 * rng.standard_normal((T, nu, p.K))).astype(np.float32))
            if fused and G == 1:
                be.reduce_finalize(cost, x, U, rows[g], act, st)
            else:
                be.reduce(cost, x, U, rows[g])
        if not (fused and G == 1):
            be.finalize(rows, G, U, act, st)
        torch.cuda.synchronize()
        outs.append((U.cpu().numpy(), act.cpu().numpy(), st.cpu().numpy()))
        be.destroy()
    for a, b in zip(*outs):
        np.testing.assert_array_equal(a, b)


def _plan_pair(mk, obj, q, plans=2):
    from mppi_isaac_b200 import MPPIisaacPlanner
    gpu = MPPIisaacPlanner(mk(DEV), obj(), use_cuda_graph=False)
    cpu = MPPIisaacPlanner(mk("cpu"), obj(), backend=ro.RiskOracleBackend())
    for _ in range(plans):
        ag, ac = gpu.compute_action(q, [0.0] * len(q)), cpu.compute_action(q, [0.0] * len(q))
    return gpu, cpu, ag, ac


@pytest.mark.parametrize("task", ["boxer", "push"])
def test_plan_agrees_with_the_oracle_pipeline(task):
    from mppi_isaac_b200.objectives import PushObjective
    if task == "boxer":
        mk, obj, q, lim = (lambda d: boxer_cfg(K=256, T=10, device=d, n_worlds=8, cvar_alpha=0.25)), \
            (lambda: PushObjective(robot="boxer", link="ee_link")), [0.0, 2.5, 0.0], 3.5
    else:
        mk, obj, q, lim = (lambda d: push_cfg(K=256, T=10, device=d, n_worlds=8, cvar_alpha=0.25)), PushObjective, [0.0, 0.0, 0.0], 1.0
    gpu, cpu, ag, ac = _plan_pair(mk, obj, q, plans=1)
    assert gpu.mppi.n_worlds == 8 and gpu.mppi.control_samples == 32
    assert torch.isfinite(ag).all() and float((ag - ac).abs().max()) <= 2e-2 * lim
    a = gpu.mppi.actions.cpu().numpy()
    np.testing.assert_array_equal(a, np.repeat(a[:, :, ::8], 8, axis=2))


def test_graph_replay_equals_the_eager_plan():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PushObjective
    pls = [MPPIisaacPlanner(push_cfg(K=2048, T=10, device=DEV, n_worlds=8, cvar_alpha=0.25), PushObjective(), use_cuda_graph=g) for g in (True, False)]
    for _ in range(4):
        a, b = (pl.compute_action([0.0, 0.0, 0.0], [0.0] * 3).numpy() for pl in pls)
        np.testing.assert_array_equal(a, b)
    assert pls[0].mppi._graph is not None and pls[1].mppi._graph is None
