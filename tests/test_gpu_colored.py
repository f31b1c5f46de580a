"""-m gpu: colored-noise K1 (``mppib_sample_colored``, ``sampling_method: colored``) against the float64 restatement of
``colored_oracle`` on the generated cases of ``synth_mppi``, its bit-identity with the white K1 at beta = 0, shards, rows, clamps,
counters, the adaptive colours, the statistics of its own output, and whole plans through the planner.

The per-element gate of ``k1_gate`` is derived from the two float32 summation orders of the kernel, and every gated case must miss it
against a reference that drops one term of the temporal sum."""
import copy

import numpy as np
import pytest
import torch

import colored_oracle as co
from mppi_isaac_b200.planner.mppi import colored_noise_chol, colored_noise_cov
from scenes import panda_cfg, pick_cfg
from synth_mppi import EPS, make_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
SEED, PLAN0, CTR = 0x1_2345_6789, 2 ** 32 - 3, 5                              # seed and plan index >= 2^32, the plan through plan_ctr

SHAPES = [(1, 1), (12, 9), (30, 7), (30, 9), (64, 8), (256, 2), (32, 16)]
KS = [4, 63, 64, 65, 10000]
BETAS = [0.0, 1.0, 2.0, 2.5]


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def backend(case, params=None, dist=None):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(case.model, params or case.params)
    if dist is not None:
        be.set_distribution(dist)
    return be


def white_params(p, nu):
    """Identity colour, no bounds, no null row: K1 then stores the white draws z themselves (1 * z + 0 summed exactly)."""
    w = copy.deepcopy(p)
    w.sample_null_action = 0
    for j in range(nu):
        w.u_min[j], w.u_max[j] = -3e38, 3e38
        for i in range(nu):
            w.sigma_chol[j * nu + i] = 1.0 if i == j else 0.0
    return w


def device_white(case, seed=SEED, plan=PLAN0 + CTR, k_offset=0, k_total=None):
    """The device's own white draws z[T][nu][K] of the counters (global sample, t, block)."""
    T, nu, K = case.T, case.nu, case.K
    be = backend(case, white_params(case.params, nu))
    z = torch.zeros((T, nu, K), device=DEV)
    be.sample(seed, plan, k_offset, k_total or K, torch.zeros((T, nu), device=DEV), None, z, None)
    return z.cpu().numpy()


def k1_gate(Lt, L0, z, U, a_ref):
    """Per-element bound on |a_kernel - a_ref| against the float32-rounded float64 reference on the same white draws z.  Row t of the
    temporal sum adds t + 1 products in order, so |dw[t][i]| <= eps (t + 2) sum_t' |L_b[t][t'] z[t'][i]|; the control sum adds j + 1
    products of the rounded w, |dn[t][j]| <= eps (j + 2) sum_i |L0[j][i] w[t][i]| + sum_i |L0[j][i]| |dw[t][i]|; then U + n is rounded
    (eps (|U| + |a|)).  Clamping is monotone and adds nothing."""
    T, nu = U.shape
    Lb, L0 = np.abs(np.asarray(Lt, np.float64)), np.abs(np.asarray(L0, np.float64))
    az = np.abs(np.asarray(z, np.float64))
    sw = np.einsum("ts,sik->tik", Lb, az, optimize=True)                                # bounds |w| too
    dw = EPS * (np.arange(T, dtype=np.float64) + 2)[:, None, None] * sw
    dn = EPS * (np.arange(nu, dtype=np.float64) + 2)[None, :, None] * np.einsum("ji,tik->tjk", L0, sw, optimize=True) + np.einsum("ji,tik->tjk", L0, dw, optimize=True)
    return dn + EPS * (np.abs(U.astype(np.float64))[:, :, None] + np.abs(np.asarray(a_ref, np.float64)))


def drop_one_term(Lt, beta):
    """L_b without one temporal term: the first column of the last row (the wrap-around correlation) when it is non-zero, else the
    diagonal of the last row."""
    bad = np.array(Lt, np.float32)
    T = bad.shape[0]
    if T > 1 and beta > 0:
        bad[T - 1, 0] = 0.0
    else:
        bad[T - 1, T - 1] = 0.0
    return bad


def _check_case(case, beta, kind_dist=None, tag=""):
    T, nu, K, p = case.T, case.nu, case.K, case.params
    rng = np.random.default_rng(T * 31 + nu + K)
    Lt = colored_noise_chol(T, beta)
    dist = case.dist if kind_dist is None else kind_dist
    be = backend(case, dist=None if dist is None else dev(dist))
    U = rng.uniform(-0.05, 0.05, (T, nu)).astype(np.float32)
    prior = rng.uniform(-2, 2, (T, nu)).astype(np.float32)
    a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    be.sample_colored(SEED, PLAN0, 0, K, dev(U), dev(prior), dev(Lt), a, n, torch.tensor([CTR], dtype=torch.int32, device=DEV))
    ag, ng = a.cpu().numpy(), n.cpu().numpy()
    z = device_white(case)
    a_ref, n_ref = co.colour(p, nu, U, z, Lt, 0, K, prior, dist)
    L0 = co.control_chol(p, nu, dist)
    gate = k1_gate(Lt, L0, z, U, a_ref)
    body = slice(0, K - 2)
    ea = float((np.abs(ag - a_ref) - gate)[:, :, body].max(initial=-1.0))
    en = float((np.abs(ng - n_ref) - gate - EPS * np.abs(n_ref))[:, :, body].max(initial=-1.0))
    print(f"COLORED {tag} T{T}nu{nu}K{K}b{beta:g} worst |a - ref| {np.abs(ag - a_ref)[:, :, body].max(initial=0):.2e} "
          f"gate min {gate[:, :, body].min(initial=0):.2e}")
    assert ea <= 0 and en <= 0
    np.testing.assert_array_equal(ag[:, :, K - 1], 0.0)                     # null row: clamp(0) = 0 inside these bounds
    np.testing.assert_array_equal(ag[:, :, K - 2], prior)                   # prior row, not clamped
    np.testing.assert_array_equal(ng[:, :, K - 2], (prior - U).astype(np.float32))
    # a reference without one temporal term misses the gate
    a_bad, _ = co.colour(p, nu, U, z, drop_one_term(Lt, beta), 0, K, prior, dist)
    assert float((np.abs(ag - a_bad) - gate)[:, :, body].max(initial=-1.0)) > 0 or K <= 2
    # the oracle's own white draws agree with the device's (the anchor of the restatement)
    z_orc = co.white(case.model, p, SEED, PLAN0 + CTR, 0, K)
    assert np.abs(z_orc - z).max() <= 1e-5 * max(1.0, np.abs(z).max())
    return be, U, prior, Lt, ag, ng


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("T,nu", SHAPES)
def test_k1_matches_float64(T, nu, K, beta):
    _check_case(make_case(T, nu, K), beta, tag="W")


@pytest.mark.parametrize("kind", ["M2", "C"])
@pytest.mark.parametrize("T,nu,K", [(12, 9, 65), (30, 7, 10000), (256, 2, 1000), (32, 16, 63)])
def test_k1_adaptive_colours_match_float64(kind, T, nu, K):
    """update_cov: the live sqrt(cov) (diag) or the live L (cov_type full) of the registered distribution."""
    case = make_case(T, nu, K, kind=kind)
    _check_case(case, 2.0, tag=kind)


@pytest.mark.parametrize("kind", ["W", "M2", "C"])
@pytest.mark.parametrize("T,nu,K", [(1, 1, 4), (12, 9, 65), (30, 7, 10000), (31, 9, 1000), (256, 2, 1000), (32, 16, 63)])
def test_beta_zero_is_bit_identical_to_the_white_k1(kind, T, nu, K):
    case = make_case(T, nu, K, kind=kind, u_min=[-0.1], u_max=[0.15])
    be = backend(case, dist=None if case.dist is None else dev(case.dist))
    rng = np.random.default_rng(5)
    U, prior = dev(rng.uniform(-0.05, 0.05, (T, nu))), dev(rng.uniform(-2, 2, (T, nu)))
    ctr = torch.tensor([CTR], dtype=torch.int32, device=DEV)
    out = []
    for colored in (False, True):
        a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
        if colored:
            be.sample_colored(SEED, PLAN0, 0, K, U, prior, dev(colored_noise_chol(T, 0.0)), a, n, ctr)
        else:
            be.sample(SEED, PLAN0, 0, K, U, prior, a, n, ctr)
        out.append((a, n))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


@pytest.mark.parametrize("T,nu,K", [(30, 9, 1000), (256, 2, 130), (12, 9, 65)])
def test_shards_are_bit_identical_to_one_launch(T, nu, K):
    case = make_case(T, nu, K)
    Lt = dev(colored_noise_chol(T, 2.0))
    U = dev(np.random.default_rng(2).uniform(-0.05, 0.05, (T, nu)))
    a1 = torch.zeros((T, nu, K), device=DEV)
    backend(case).sample_colored(SEED, PLAN0 + CTR, 0, K, U, None, Lt, a1, None)
    k1 = K // 3 + 1
    for off, kk in ((0, k1), (k1, K - k1)):
        pp = copy.copy(case.params)
        pp.K = kk
        a = torch.zeros((T, nu, kk), device=DEV)
        backend(case, pp).sample_colored(SEED, PLAN0 + CTR, off, K, U, None, Lt, a, None)
        assert torch.equal(a, a1[:, :, off:off + kk])


def test_binding_clamps_null_and_prior_rows():
    T, nu, K = 30, 9, 10000
    lo = [-0.05 if j % 3 == 0 else -1e3 for j in range(nu)]
    hi = [0.03 if j % 3 == 0 else 1e3 for j in range(nu)]
    case = make_case(T, nu, K, u_min=lo, u_max=hi, u_init=0.01)
    be, U, prior, Lt, ag, ng = _check_case(case, 2.5, tag="clamp")
    tight = np.arange(nu) % 3 == 0
    body = ag[:, :, :-2]
    assert np.all(body >= np.asarray(lo, np.float32)[None, :, None]) and np.all(body <= np.asarray(hi, np.float32)[None, :, None])
    at = (body[:, tight] == np.asarray(hi, np.float32)[tight][None, :, None]).mean()
    assert 0.05 < at < 0.95                                                  # the clamp binds on part of the samples
    np.testing.assert_array_equal(ng[:, :, :-2], (body - U[:, :, None]).astype(np.float32))


def test_plan_counter_moves_the_stream():
    """The plan index is plan_idx + *plan_ctr on the device: the same plan reached either way draws the same noise, another does not."""
    case = make_case(30, 7, 1000)
    be = backend(case)
    Lt, U = dev(colored_noise_chol(30, 2.0)), torch.zeros((30, 7), device=DEV)
    outs = []
    for plan, ctr in ((PLAN0 + CTR, None), (PLAN0, CTR), (PLAN0, CTR + 1)):
        a = torch.zeros((30, 7, 1000), device=DEV)
        be.sample_colored(SEED, plan, 0, 1000, U, None, Lt, a, None, None if ctr is None else torch.tensor([ctr], dtype=torch.int32, device=DEV))
        outs.append(a)
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[1], outs[2])


@pytest.mark.parametrize("beta", [1.0, 2.0, 2.5])
def test_empirical_temporal_correlation_of_the_kernel_output(beta):
    """K = 65 536 unclamped samples: per control dimension the correlation of noise[t][j] and noise[t'][j] over the samples is
    Sigma_b[t][t'] (Cov(noise) = Sigma_b (x) Sigma0).  Standard error <= 1 / sqrt(K) = 3.9e-3; the gate is 6 of those."""
    T, nu, K = 30, 7, 65536
    case = make_case(T, nu, K)
    be = backend(case)
    a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    be.sample_colored(SEED, 1, 0, K, torch.zeros((T, nu), device=DEV), None, dev(colored_noise_chol(T, beta)), a, n, None)
    x = n[:, :, :-1].double()                                                # the null row excluded
    S = colored_noise_cov(T, beta)
    worst = 0.0
    for j in range(nu):
        R = torch.corrcoef(x[:, j]).cpu().numpy()
        worst = max(worst, float(np.abs(R - S).max()))
    print(f"COLORED stats beta {beta}: worst |R - Sigma_b| {worst:.2e}")
    assert worst <= 6.0 / np.sqrt(K)
    assert np.abs(S - np.eye(T)).max() > 6.0 / np.sqrt(K)                  # white noise would miss it


def test_backend_refusals():
    from mppi_isaac_b200.backend import CudaBackend
    case = make_case(12, 7, 64)
    be = backend(case)
    a = torch.zeros((12, 7, 64), device=DEV)
    with pytest.raises(RuntimeError, match="Lt"):
        be.sample_colored(0, 0, 0, 64, torch.zeros((12, 7), device=DEV), None, dev(np.eye(13)), a, None)
    with pytest.raises(RuntimeError, match="noise"):
        be.sample_colored(0, 0, 0, 64, torch.zeros((12, 7), device=DEV), None, dev(np.eye(12)), a, torch.zeros(1, device=DEV))
    hz = make_case(12, 7, 64, kind="H")
    beh = CudaBackend(DEV)
    beh.create(hz.model, hz.params)
    with pytest.raises(RuntimeError, match="cov_horizon"):
        beh.sample_colored(0, 0, 0, 64, torch.zeros((12, 7), device=DEV), None, dev(np.eye(12)), a, None)


def test_captured_graph_draws_fresh_noise_and_equals_eager():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    kw = dict(sampling_method="colored", noise_beta=2.0)
    g = MPPIisaacPlanner(panda_cfg(K=2000, T=30, device=DEV, **kw), PandaReachObjective(), use_cuda_graph=True)
    e = MPPIisaacPlanner(panda_cfg(K=2000, T=30, device=DEV, **kw), PandaReachObjective(), use_cuda_graph=False)
    graph, prev = None, None
    for it in range(5):
        g.compute_action(Q0, [0.0] * 7)
        e.compute_action(Q0, [0.0] * 7)
        graph = graph or g.mppi._graph
        assert graph is not None and g.mppi._graph is graph, "the plan graph was re-captured"
        assert torch.equal(g.mppi.noise, e.mppi.noise) and torch.equal(g.mppi.U, e.mppi.U), f"plan {it}"
        assert prev is None or not torch.equal(prev, g.mppi.noise), "a replay drew the previous plan's noise"
        prev = g.mppi.noise.clone()


@pytest.mark.parametrize("task", ["panda", "pick"])
def test_plan_through_planner_matches_the_oracle_pipeline(task):
    """MPPIisaacPlanner with colored noise on the GPU (CUDA graph) against the same planner on the checker backend fed the same colored
    noise: panda reach at K = 10 000, T = 30 (lock-step U, the gate of the white plan-parity test) and the C5 shape (T = 30, nu = 9)
    at K = 1 024 (the gate of the contact plan-parity test)."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaPickObjective, PandaReachObjective
    kw = dict(sampling_method="colored", noise_beta=2.0)
    if task == "panda":
        mk, obj, q, plans, rel = (lambda d: panda_cfg(K=10000, T=30, device=d, **kw)), PandaReachObjective, Q0, 2, 2e-4
    else:
        mk, obj, q, plans, rel = (lambda d: pick_cfg(K=1024, T=30, device=d, **kw)), PandaPickObjective, Q0 + [0.02, 0.02], 1, 2e-2
    gpu = MPPIisaacPlanner(mk(DEV), obj(), use_cuda_graph=True)
    cpu = MPPIisaacPlanner(mk("cpu"), obj(), backend=co.ColoredOracleBackend(nthreads=8))
    lim = float(gpu.mppi.backend.params.u_max[0])
    for it in range(plans):
        cpu.mppi.U.copy_(gpu.mppi.U.cpu())
        cpu.mppi.plan_ctr.copy_(gpu.mppi.plan_ctr.cpu())
        ag, ac = gpu.compute_action(q, [0.0] * len(q)), cpu.compute_action(q, [0.0] * len(q))
        assert torch.isfinite(ag).all()
        err = float((ag.cpu() - ac).abs().max())
        print(f"COLORED plan {task} {it}: |a_gpu - a_oracle| {err:.2e}")
        assert err <= rel * max(1.0, lim), f"plan {it}"
    assert gpu.mppi._graph is not None
