"""-m gpu: annealed MPPI (``anneal_iterations``) on the device: K1 with a schedule of ones against plain K1 bit for bit (Gaussian, colored,
n_worlds), K1 with a random schedule against the float64 reference under a bound derived from its float32 operations, K3 over RPL 4 / 8 / 16
and RISK, split and fused, K4's counter and the shift's reset on both paths, whole point-robot plans with N = 1 and 3 against the
``AnnealOracleBackend`` pipeline, graph replay against eager plans, and the library's refusals."""
import copy

import numpy as np
import pytest
import torch

import anneal_oracle as ao
from mppi_isaac_b200.model.blob import make_params
from mppi_isaac_b200.planner.mppi import colored_noise_chol
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from scenes import point_cfg
from synth_mppi import nu_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 2.0 ** -24


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(DEV)


def params(nu, T, K, mode="simple", **kw):
    d = dict(num_samples=K, horizon=T, mppi_mode=mode, sampling_method="random", noise_sigma=(0.3 * np.eye(nu) + 0.05).tolist(),
             u_min=[-0.6], u_max=[0.6], lambda_=0.05, sample_null_action=True, rollout_var_discount=0.9)
    d.update(kw)
    return make_params(MPPIConfig(**d), IsaacGymConfig(), nu, K, [])


def backend(nu, p, state=None, N=1):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(nu_model(nu), p)
    if state is not None:
        be.set_anneal(state, N)
    return be


def random_schedule(N, T, seed):
    s = np.random.default_rng(seed).uniform(0.05, 1.0, (N, T))
    return s.astype(np.float32), (1.0 / (s * s)).astype(np.float32)


def k1(variant, nu, T, p, U, state=None, N=1, plan_idx=3):
    be = backend(nu, p, state, N)
    K = p.K
    a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    if variant == "colored":
        be.sample_colored(7, plan_idx, 0, K, U, None, dev(colored_noise_chol(T, 2.0)), a, n)
    else:
        be.sample(7, plan_idx, 0, K, U, None, a, n)
    torch.cuda.synchronize()
    be.destroy()
    return a.cpu().numpy(), n.cpu().numpy()


@pytest.mark.parametrize("variant, R", [("random", 1), ("colored", 1), ("random", 4), ("colored", 8)])
def test_k1_with_a_schedule_of_ones_is_plain_k1_bit_for_bit(variant, R):
    nu, T, K = 7, 30, 1024
    kw = dict(n_worlds=R, cvar_alpha=0.5) if R > 1 else {}
    p = params(nu, T, K, **kw)
    U = dev(0.1 * np.sin(np.arange(T * nu) * 0.7).reshape(T, nu))
    ref = k1(variant, nu, T, p, U)
    ones = dev(ao.make_state(np.ones((1, T)), np.ones((1, T))))
    got = k1(variant, nu, T, p, U, ones, 1)
    np.testing.assert_array_equal(got[0], ref[0])
    np.testing.assert_array_equal(got[1], ref[1])


@pytest.mark.parametrize("variant", ["random", "colored"])
@pytest.mark.parametrize("nu, T", [(1, 1), (7, 30), (16, 32), (3, 170)])
def test_k1_with_a_random_schedule_against_float64(variant, nu, T):
    """|a_gpu - a_64| <= eps (n_sum (|L| |L_b| |z|) s + 2 |u| + 2 |a|): the colour's float32 sums (n_sum = nu, + T for the temporal sum),
    the scale's rounding, the sum with U and the final rounding, each bounded by one unit of its operands' magnitude."""
    K, N = 512, 3
    p = params(nu, T, K, sampling_method=variant)
    s, r = random_schedule(N, T, nu * T)
    state = ao.make_state(s, r, counter=1.0)
    rng = np.random.default_rng(T)
    U = (0.2 * rng.standard_normal((T, nu))).astype(np.float32)
    a, n = k1(variant, nu, T, p, dev(U), dev(state), N, plan_idx=1 << 32)
    Lt = colored_noise_chol(T, 2.0) if variant == "colored" else None
    ar, nr = ao.sample(nu_model(nu), p, 7, 1 << 32, U, 0, K, s[1], Lt=Lt)
    z = np.abs(ao.co.white(nu_model(nu), p, 7, 1 << 32, 0, K).astype(np.float64))
    if Lt is not None:
        z = np.einsum("ts,sik->tik", np.abs(Lt.astype(np.float64)), z)
    L = np.abs(np.array(p.sigma_chol[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu))
    mag = np.einsum("ji,tik->tjk", L, z) * s[1].astype(np.float64)[:, None, None]
    nsum = nu + (T if Lt is not None else 0) + 1
    bound = EPS * (nsum * mag + 2.0 * np.abs(U)[:, :, None] + 2.0 * np.abs(ar)) + 1e-30
    assert np.all(np.abs(a.astype(np.float64) - ar) <= bound)
    assert np.all(np.abs(n.astype(np.float64) - nr) <= 2 * bound)


def k3_case(nu, T, K, seed, R=1, mode="simple"):
    kw = dict(n_worlds=R, cvar_alpha=0.5) if R > 1 else {}
    p = params(nu, T, K, mode=mode, **kw)
    rng = np.random.default_rng(seed)
    cost = rng.random((T, K)).astype(np.float32)
    x = (0.2 * rng.standard_normal((T, nu, K))).astype(np.float32)
    U = (0.1 * rng.standard_normal((T, nu))).astype(np.float32)
    return p, cost, x, U


@pytest.mark.parametrize("nu, T, R, mode", [(4, 30, 1, "simple"), (7, 30, 1, "simple"), (8, 60, 1, "simple"), (7, 30, 4, "simple"),
                                            (16, 32, 8, "simple"), (7, 30, 1, "halton-spline")])
def test_k3_against_float64_split_and_fused(nu, T, R, mode):
    """RPL 4 (T*nu <= 128), 8 and 16, RISK; the split row and the fused tail's U against the float64 row and K4 of the reference."""
    K, N = 4096, 3
    p, cost, x, U = k3_case(nu, T, K, nu + T + R, R, mode)
    s, r = random_schedule(N, T, 11)
    state = dev(ao.make_state(s, r, counter=2.0))
    be = backend(nu, p, state, N)
    part = torch.zeros(2 + T * nu, device=DEV)
    be.reduce(dev(cost), dev(x), dev(U), part)
    Ug, act, st = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.reduce_finalize(dev(cost), dev(x), Ug, torch.zeros(2 + T * nu, device=DEV), act, st)
    torch.cuda.synchronize()
    ref = ao.reduce(p, nu, cost, x, U, r[2])
    row = part.cpu().numpy()
    S, _ = ao.scores(p, nu, cost, x, U, r[2])
    np.testing.assert_allclose(row[0], ref[0], rtol=1e-5, atol=1e-5 * np.abs(S).max())
    np.testing.assert_allclose(row[1], ref[1], rtol=2e-4)
    np.testing.assert_allclose(row[2:], ref[2:], rtol=0, atol=2e-4 * max(1.0, float(np.abs(ref[2:]).max())))
    from oracle import oracle as orc
    Ur, ar, _ = orc.finalize(nu_model(nu), p, ref[None], U)
    np.testing.assert_allclose(Ug.cpu().numpy(), Ur, rtol=0, atol=1e-4)
    np.testing.assert_allclose(act.cpu().numpy(), ar, rtol=0, atol=1e-4)
    assert float(state[0]) == 3.0                                              # the fused tail advanced the counter, the split K3 did not
    ones = dev(ao.make_state(np.ones((1, T)), np.ones((1, T))))
    be.set_anneal(ones, 1)
    p1 = torch.zeros_like(part)
    be.reduce(dev(cost), dev(x), dev(U), p1)
    be.set_anneal(None)
    p0 = torch.zeros_like(part)
    be.reduce(dev(cost), dev(x), dev(U), p0)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(p1.cpu().numpy(), p0.cpu().numpy())        # r = 1 changes no bit of K3
    be.destroy()


def test_k4_advances_the_counter_and_the_shift_resets_it():
    nu, T, K, N = 3, 10, 256, 3
    p, cost, x, U = k3_case(nu, T, K, 5)
    state = dev(ao.make_state(*ao.schedule(N, 0.7, 0.9, T)))
    be = backend(nu, p, state, N)
    Ug, act, st, part = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV), torch.zeros(2 + T * nu, device=DEV)
    seen = []
    for _ in range(2):
        be.reduce(dev(cost), dev(x), Ug, part)
        be.finalize(part.view(1, -1), 1, Ug, act, st)                         # split K4
        seen.append(float(state[0]))
        be.reduce_finalize(dev(cost), dev(x), Ug, part, act, st)               # fused tail
        seen.append(float(state[0]))
    ctr = torch.zeros(1, dtype=torch.int32, device=DEV)
    be.shift(Ug, ctr)
    seen.append(float(state[0]))
    assert seen == [1.0, 2.0, 3.0, 4.0, 0.0] and int(ctr[0]) == 1
    be.destroy()


def _planner(device, graph=False, backend=None, **kw):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    extra = {} if backend is None else dict(backend=backend)
    return MPPIisaacPlanner(point_cfg(device=device, **kw), PointReachObjective(), use_cuda_graph=graph, **extra)


@pytest.mark.parametrize("N, method, filter_u", [(1, "random", False), (3, "random", False), (3, "colored", True), (1, "colored", True),
                                                 (3, "random", True)])
def test_point_plans_agree_with_the_oracle_pipeline(N, method, filter_u):
    kw = dict(K=1024, T=12, sampling_method=method, filter_u=filter_u, anneal_iterations=N, anneal_iter_decay=0.7, anneal_horizon_decay=0.9)
    gpu = _planner(DEV, **kw)
    cpu = _planner("cpu", backend=ao.AnnealOracleBackend(), **kw)
    q = [0.1, 0.0, 0.0]
    for _ in range(3):
        a, b = gpu.compute_action(q, [0.0] * 3).numpy(), cpu.compute_action(q, [0.0] * 3).numpy()
        np.testing.assert_allclose(a, b, rtol=0, atol=2e-4)
    np.testing.assert_allclose(gpu.mppi.U.cpu().numpy(), cpu.mppi.U.numpy(), rtol=0, atol=2e-4)
    assert float(gpu.mppi.anneal_state[0]) == N


def test_graph_replay_equals_eager_and_follows_set_noise_schedule():
    kw = dict(K=2048, T=12, sampling_method="random", anneal_iterations=3, anneal_iter_decay=0.7, anneal_horizon_decay=0.9)
    pls = [_planner(DEV, graph=g, **kw) for g in (True, False)]
    q = [0.1, 0.0, 0.0]
    for it in range(4):
        if it == 2:
            for pl in pls:
                pl.mppi.set_noise_schedule(np.full((3, 12), 0.4))
        acts = [pl.compute_action(q, [0.0] * 3).numpy() for pl in pls]
        np.testing.assert_array_equal(acts[0], acts[1])
    assert pls[0].mppi._graph is not None and pls[1].mppi._graph is None
    np.testing.assert_array_equal(pls[0].mppi.U.cpu().numpy(), pls[1].mppi.U.cpu().numpy())
    np.testing.assert_array_equal(pls[0].mppi.anneal_state.cpu().numpy(), pls[1].mppi.anneal_state.cpu().numpy())


def test_defaults_are_bit_identical_to_a_planner_without_the_keys():
    a = _planner(DEV, K=1024, T=12, sampling_method="random")
    b = _planner(DEV, K=1024, T=12, sampling_method="random", anneal_iterations=1, anneal_iter_decay=1.0, anneal_horizon_decay=1.0)
    assert b.mppi.anneal_state is None
    for _ in range(3):
        np.testing.assert_array_equal(a.compute_action([0.1, 0.0, 0.0], [0.0] * 3).numpy(), b.compute_action([0.1, 0.0, 0.0], [0.0] * 3).numpy())


def test_library_refusals():
    nu, T, K = 3, 10, 256
    p = params(nu, T, K, noise_sigma=(0.3 * np.eye(nu)).tolist())              # diagonal, so that a cem block is valid
    state = dev(ao.make_state(*ao.schedule(2, 0.7, 1.0, T)))
    be = backend(nu, p)
    with pytest.raises(RuntimeError, match="n_iterations"):
        be.set_anneal(dev(ao.make_state(*ao.schedule(17, 1.0, 1.0, T))), 17)
    for bad in (dict(mode=2, n_elites=1), dict(mode=3), dict(update_cov=1), dict(update_lambda=1)):
        q = copy.copy(p)
        for k, v in bad.items():
            setattr(q, k, v)
        be.set_params(q)
        with pytest.raises(RuntimeError, match="annealed MPPI excludes"):
            be.set_anneal(state, 2)
    be.set_params(p)
    be.set_anneal(state, 2)
    U, a = torch.zeros((T + 1, nu), device=DEV), torch.zeros((T + 1, nu, K), device=DEV)
    q = copy.copy(p)
    q.T = T + 1
    be.set_params(q)                                                           # T changed without a new registration
    with pytest.raises(RuntimeError, match="registered for T"):
        be.sample(1, 0, 0, K, U, None, a, None)
    with pytest.raises(RuntimeError, match="registered for T"):
        be.shift(U)
    be.set_params(p)
    q = copy.copy(p)
    q.mode, q.n_elites = 2, 1                                                  # cem after registration: refused at launch
    be.set_params(q)
    with pytest.raises(RuntimeError, match="excludes mode cem"):
        be.sample(1, 0, 0, K, U[:T], None, a[:T], None)
    be.set_params(p)
    Z = torch.zeros((T, nu, K), device=DEV)
    with pytest.raises(RuntimeError, match="noise library"):
        be.sample_library(0, K, U[:T], None, Z, a[:T], None)
    be.destroy()
