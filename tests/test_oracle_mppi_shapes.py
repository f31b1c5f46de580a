"""Pins the K1 / K3 / K4 references at the shapes of the generated sweep (``synth_mppi``): nu = 16, T = 32 and T = 256 against the
float64 torch restatement of ``test_oracle_mppi``, the adaptive references against the same restatement, gamma = 0, the refused
gammas, the K3 layout restatement, and the float32 error bound the GPU sweep gates on; for the horizon row kind "H", the restatement
against ``adaptive_horizon_oracle``, float32 restatements of the SYRK and K1 orders inside their gates, the SYRK split and the host's
refusals."""
import math

import numpy as np
import pytest
import torch

import adaptive_full_oracle as afo
import adaptive_horizon_oracle as aho
import adaptive_oracle as ada
from synth_mppi import (NUM_SMS, SMEM_CAP, WS_NCONS, _ws_bytes, hz_C, hz_id, hz_k1_f32, hz_k1_gate, k3_dS, k3_gate, k3_inputs, k3_restate,
                        k3_S32, last4_K, make_case, nu_model, row_excess, syrk_split, ws_layout, ws_stages)
from test_oracle_mppi import _torch_update

SHAPES = [(32, 16), (256, 2), (256, 1)]


def _update_case(oracle, case, seed):
    nu, T = case.nu, case.T
    rng = np.random.default_rng(seed)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    pf = case.params if case.kind == "W" else (ada if case.kind == "M2" else afo).dist_params(case.params, nu, case.dist)
    a, n = oracle.sample(case.model, pf, seed, 0, U)
    cost = rng.uniform(0, 10.0 / T, (T, case.K)).astype(np.float32)
    return pf, U, a, n, cost


@pytest.mark.parametrize("T,nu", SHAPES)
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_reduce_finalize_match_torch_at_sweep_shapes(oracle, T, nu, mode):
    case = make_case(T, nu, 512, mode=mode, lam=0.5)
    pf, U, a, n, cost = _update_case(oracle, case, 1)
    x = n if case.simple else a
    partial, S = oracle.reduce(case.model, case.params, cost, x, U)
    Un, act, stats = oracle.finalize(case.model, case.params, partial[None], U)
    U_ref, S_ref = _torch_update(case.params, nu, cost, n, a, U)
    np.testing.assert_allclose(S, S_ref, rtol=1e-6, atol=1e-5)
    np.testing.assert_allclose(Un, U_ref, rtol=0, atol=2e-7)
    np.testing.assert_array_equal(act, Un[0])
    assert abs(stats[0] - S_ref.min()) < 1e-5


@pytest.mark.parametrize("T,nu", SHAPES)
@pytest.mark.parametrize("kind", ["M2", "C"])
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_adaptive_references_match_torch_at_sweep_shapes(oracle, T, nu, kind, mode):
    """The U update of the adaptive references is the fixed-distribution rule with the live lambda and Sigma^-1."""
    case = make_case(T, nu, 512, mode=mode, lam=0.5, kind=kind)
    pf, U, a, n, cost = _update_case(oracle, case, 2)
    x = n if case.simple else a
    mod = ada if kind == "M2" else afo
    row = mod.reduce(case.model, case.params, cost, x, U, case.dist)
    Un, _, _, _ = mod.finalize(case.model, case.params, row[None], U, case.dist)
    U_ref, _ = _torch_update(pf, nu, cost, n, a, U)
    np.testing.assert_allclose(Un, U_ref, rtol=0, atol=2e-7)


@pytest.mark.parametrize("kind", ["W", "M2", "C"])
@pytest.mark.parametrize("T,nu,mode", [(32, 16, "simple"), (9, 14, "halton-spline"), (129, 2, "halton-spline"), (1, 1, "simple")])
def test_sweep_restatement_matches_the_references(oracle, T, nu, mode, kind):
    """The float64 numpy row the sweep derives its gates and its drop-the-tail check from == the references it compares with."""
    case = make_case(T, nu, 1000, mode=mode, kind=kind, gamma=0.95)
    cost, x, U = k3_inputs(case, seed=3)
    cost[:, 5] = np.nan
    _, _, row = k3_restate(case, cost, x, U)
    if kind == "W":
        ref = oracle.reduce(case.model, case.params, cost, x, U)[0]
    else:
        ref = (ada if kind == "M2" else afo).reduce(case.model, case.params, cost, x, U, case.dist)
    np.testing.assert_allclose(row, ref, rtol=2e-6, atol=1e-30)


def test_gamma_zero_scores_the_first_step(oracle):
    case = make_case(30, 4, 256, mode="halton-spline", gamma=0.0)
    cost, x, U = k3_inputs(case, seed=4)
    cost[3, 9] = np.inf                                                       # 0 * inf: a diverged later step still rejects the sample
    _, S = oracle.reduce(case.model, case.params, cost, x, U)
    want = cost[0].copy()
    want[9] = np.nan
    np.testing.assert_array_equal(S, want)
    S64, _, _ = k3_restate(case, cost, x, U)
    np.testing.assert_array_equal(S64.astype(np.float32), want)
    np.testing.assert_array_equal(k3_S32(case, cost, x, U), want)             # the kernel's gamma^0 = 1, gamma^t = 0


@pytest.mark.parametrize("gamma", [-0.5, -1e-30, float("nan"), float("inf"), -float("inf")])
def test_make_params_refuses_a_negative_or_non_finite_gamma(gamma):
    with pytest.raises(ValueError, match="rollout_var_discount"):
        make_case(12, 2, 64, mode="halton-spline", gamma=gamma)
    make_case(12, 2, 64, mode="simple", gamma=gamma)                          # SIMPLE mode has no discount: gamma = 1


def test_k3_layout_restatement():
    """Consumer warps of the shapes the sweep uses for each count, and the refused shapes.  The second-moment row at T = 256, nu = 2
    leaves room for two stages only next to their two consumers' partials; mode smooth's U region costs the ring a stage at 186 x 2."""
    assert [ws_layout(T, nu, "W")[1] for T, nu in [(1, 1), (125, 1), (146, 1), (174, 1), (216, 1), (187, 2)]] == [7, 6, 5, 4, 3, 2]
    assert ws_layout(256, 2, "M2") == (16, 2, 2, 256) and ws_stages(256, 2, "M2") == 2 and ws_layout(256, 2, "C") is not None
    assert _ws_bytes(256, 2, 2, "M2", WS_NCONS) > SMEM_CAP >= _ws_bytes(256, 2, 2, "M2")
    assert ws_layout(186, 2, "W")[1:3] == (3, 3) and ws_layout(186, 2, "W", smooth=True)[1:3] == (2, 2)
    assert ws_layout(257, 1, "W") is None and ws_layout(57, 9, "W") is None
    assert [ws_layout(T, nu, "W")[3] for T, nu in [(37, 7), (251, 2), (129, 2), (32, 16)]] == [37, 251, 129, 256]
    assert [ws_layout(T, nu, k)[0] for T, nu, k in [(32, 4, "W"), (43, 3, "M2"), (16, 16, "C"), (129, 2, "C"), (32, 16, "C")]] == [4, 8, 8, 16, 16]


@pytest.mark.parametrize("T,nu,mode,gamma", [(32, 16, "simple", 1.0), (256, 2, "simple", 1.0), (256, 1, "halton-spline", 1.05), (256, 2, "halton-spline", 0.5),
                                             (37, 7, "halton-spline", 0.95), (1, 1, "simple", 1.0), (20, 13, "halton-spline", 0.0)])
@pytest.mark.parametrize("kind", ["W", "M2", "C"])
def test_gate_bounds_a_float32_restatement_of_S(T, nu, mode, gamma, kind):
    """|S_float32 - S| <= dS on the generated inputs, and dS stays far below lambda there (so the gate tests the weights)."""
    case = make_case(T, nu, 2000, mode=mode, gamma=gamma, kind=kind)
    cost, x, U = k3_inputs(case, seed=5)
    S64, _, _ = k3_restate(case, cost, x, U)
    S32 = k3_S32(case, cost, x, U).astype(np.float64)
    dS = k3_dS(case, cost, x, U)
    err = np.abs(S32 - S64)
    assert np.all(err <= dS), (err / dS).max()
    assert dS.max() / case.lam < 2e-3
    assert np.ptp(S64) > case.lam                                              # the weights are spread, not collapsed onto the argmin


# ------------------------------------------------------------------------------------------------------------------------------ cov_type horizon
@pytest.mark.parametrize("T,nu,mode,sigma_h", [(1, 1, "simple", "iid"), (13, 5, "halton-spline", "corr"), (16, 16, "simple", 1e3),
                                               (256, 1, "halton-spline", 1e5)])
def test_hz_restatement_matches_the_reference(T, nu, mode, sigma_h):
    """The float64 row of kind H (n = 1, 65, 256) == adaptive_horizon_oracle.reduce, rounded; Sigma_H has the asked-for condition number."""
    case = make_case(T, nu, 1000, mode=mode, kind="H", gamma=0.95, sigma_h=sigma_h)
    n = case.n
    assert case.chol().shape == case.sinv().shape == (n, n) and case.row_floats() == 2 + n + n * (n + 1) // 2
    if not isinstance(sigma_h, str) and n > 1:
        assert abs(np.linalg.cond(aho.unpack(case.dist, n)[1].astype(np.float64)) / sigma_h - 1) < 0.05
    cost, x, U = k3_inputs(case, seed=3)
    cost[:, 5] = np.nan
    assert not U[-1].any()                                                    # u_init: U is what mppib_shift leaves
    _, _, row = k3_restate(case, cost, x, U)
    ref = aho.reduce(case.model, case.params, cost, x, U, case.dist)
    np.testing.assert_allclose(row, ref, rtol=2e-6, atol=1e-30)


def _syrk_f32(case, S32, beta, x, U, sms=NUM_SMS):
    """float32 restatement of the SYRK: w_k = expf(-(S_k - beta) / lambda) from float32 S, per-entry FFMA over each chunk in sample
    order, then the chunk sums folded in split order."""
    f = np.float32
    n, K = case.n, case.K
    _, ksplit, kchunk = syrk_split(n, K, sms)
    inv = f(1) / f(case.lam)
    with np.errstate(over="ignore", invalid="ignore"):
        w = np.where(np.isfinite(S32), np.exp(-((S32 - f(beta)).astype(f) * inv).astype(f)).astype(f), f(0))
    d = np.asarray(x, f).reshape(n, K)
    if not case.simple:
        d = (d - np.asarray(U, f).reshape(n, 1)).astype(f)
    a = (w[None] * d).astype(f)
    C = np.zeros((n, n), f)
    for s in range(ksplit):
        acc = np.zeros((n, n), f)
        for k in range(s * kchunk, min(K, (s + 1) * kchunk)):
            acc = (acc.astype(np.float64) + np.outer(a[:, k].astype(np.float64), d[:, k].astype(np.float64))).astype(f)   # fmaf
        C = (C + acc).astype(f)
    return C[np.tril_indices(n)]


@pytest.mark.parametrize("T,nu,mode,K", [(13, 5, "halton-spline", None), (8, 8, "simple", 36), (43, 3, "halton-spline", 4228)])
def test_hz_c_gate_bounds_a_float32_syrk(T, nu, mode, K):
    """The C gate holds a float32 restatement of the SYRK's order with margin, and the reference without any one split's samples
    (C - C_s) misses it."""
    n = T * nu
    K = K or last4_K(n)
    case = make_case(T, nu, K, mode=mode, kind="H", gamma=0.95)
    cost, x, U = k3_inputs(case, seed=11)
    S, w, row = k3_restate(case, cost, x, U)
    gate = k3_gate(case, cost, x, U, S, w)[2 + n:]
    S32 = k3_S32(case, cost, x, U)
    C32 = _syrk_f32(case, S32, S32[np.isfinite(S32)].min(), x, U)
    exc, err = row_excess(C32, row[2 + n:], gate)
    ratio = (np.abs(C32 - row[2 + n:]) / gate).max()
    assert exc <= 0 and ratio < 0.5, ratio
    _, ksplit, kchunk = syrk_split(n, K)
    assert ksplit > 1
    for s in range(ksplit):
        alt = row[2 + n:] - hz_C(case, x, U, w, s * kchunk, min(K, (s + 1) * kchunk))
        assert row_excess(C32, alt, gate)[0] > 0, s


@pytest.mark.parametrize("T,nu", [(13, 5), (16, 16), (256, 1)])
def test_hz_k1_gate_bounds_a_float32_colouring(T, nu):
    case = make_case(T, nu, 64, kind="H", sigma_h="corr")
    n, L = case.n, case.chol()
    rng = np.random.default_rng(n)
    z = rng.standard_normal((n, 64)).astype(np.float32)
    U = rng.uniform(-0.1, 0.1, n).astype(np.float32)
    a64 = U.astype(np.float64)[:, None] + L.astype(np.float64) @ z.astype(np.float64)
    a_ref = a64.astype(np.float32)
    gate = hz_k1_gate(L, z, U, a_ref)
    err = np.abs(hz_k1_f32(L, z, U).astype(np.float64) - a_ref)
    assert np.all(err <= gate) and (err / gate).max() < 0.5
    miss = np.abs(hz_k1_f32(L, z, U) - (a64 - np.diag(L).astype(np.float64)[:, None] * z)) > gate
    assert miss.any(axis=1).all()                                             # every row tells its diagonal term apart


def test_hz_syrk_split_and_layout_restatement():
    """The SYRK split on 132 SMs (1 tile x up to 132 splits for n <= 64, 3 x 44, 6 x 22, 10 x 13), chunks a multiple of 32 with a last
    chunk of 4 samples at last4_K; the horizon K3 sized with the M2 layout, which runs fewer ring stages and consumer warps than the W
    layout the kernel addresses at 42 shapes with n <= 256."""
    for n, ks in [(1, 128), (64, 128), (65, 44), (128, 44), (129, 22), (192, 22), (193, 13), (256, 13)]:
        nt = {128: 1, 44: 3, 22: 6, 13: 10}[ks]
        assert syrk_split(n, 65536) == (nt, ks, 32 * math.ceil(65536 / (32 * ks)) if ks != 128 else 512)
        K = last4_K(n)
        nt_, ksplit, kchunk = syrk_split(n, K)
        assert kchunk % 32 == 0 and K - (ksplit - 1) * kchunk == 4 and nt_ * ksplit <= NUM_SMS
    assert syrk_split(64, 36) == (1, 2, 32)
    assert hz_id(43, 3, 4228, "g0.95") == "hz-RPL8-T43nu3-ncons7-t6x19-K4228-g0.95"
    assert hz_id(210, 1, 36, "simple") == "hz-RPL8-T210nu1-ncons3-t10x2-K36-simple"
    fewer = [(T, nu) for T in range(1, 257) for nu in range(1, 17) if T * nu <= 256 and ws_layout(T, nu, "H") != ws_layout(T, nu, "W")]
    assert len(fewer) == 42 and (210, 1) in fewer and (96, 2) in fewer
    assert ws_layout(210, 1, "W")[1:3] == (4, 4) and ws_layout(210, 1, "H")[1:3] == (3, 3)
    assert ws_layout(257, 1, "H") is None


def test_hz_make_params_refuses_n_257():
    with pytest.raises(ValueError, match="T\\*nu <= 256"):
        make_case(257, 1, 64, kind="H")


class _RecordingLib:
    """Stands in for libmppib.so: records every call (there must be none after a refusal)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*a):
            self.calls.append(name)
            return 0
        return call


@pytest.mark.parametrize("rule", ["horizon", "full", "diag"])
def test_backend_refuses_a_change_the_registered_distribution_does_not_fit(rule):
    """set_params / set_model refuse, before the library sees them, a (T, nu) whose distribution length (1 + 3 n^2, 1 + 3 nu^2,
    1 + nu) no longer matches the registered buffer; a set_model that keeps nu goes through."""
    from mppi_isaac_b200.backend import CudaBackend, dist_floats
    kind = {"horizon": "H", "full": "C", "diag": "M2"}[rule]
    case = make_case(12, 3, 64, kind=kind)
    be = object.__new__(CudaBackend)
    be.lib, be.handle, be.model, be.params, be._dist_keepalive = _RecordingLib(), None, case.model, case.params, None
    be.set_distribution(torch.zeros(len(case.dist)))
    assert dist_floats(case.params, 3)[0] == len(case.dist) == {"horizon": 1 + 3 * 36 ** 2, "full": 28, "diag": 4}[rule]
    with pytest.raises(RuntimeError, match="mppib_set_distribution"):
        be.set_distribution(torch.zeros(len(case.dist) + 1))
    be.lib.calls.clear()
    p13 = make_case(13, 3, 64, kind=kind).params
    if rule == "horizon":
        with pytest.raises(RuntimeError, match="mppib_set_params: the registered distribution holds 3889 floats"):
            be.set_params(p13)
    else:
        be.set_params(p13)                                                     # the length of these rules does not depend on T
        be.set_params(case.params)
    be.lib.calls.clear()
    with pytest.raises(RuntimeError, match="mppib_set_model"):
        be.set_model(nu_model(4))
    assert be.lib.calls == [] and be.params is case.params and be.model is case.model
    be.set_model(nu_model(3))
    assert be.lib.calls == ["mppib_set_model"]
