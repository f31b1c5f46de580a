"""Pins the K1 / K3 / K4 references at the shapes of the generated sweep (``synth_mppi``): nu = 16, T = 32 and T = 256 against the
float64 torch restatement of ``test_oracle_mppi``, the adaptive references against the same restatement, gamma = 0, the refused
gammas, the K3 layout restatement, and the float32 error bound the GPU sweep gates on."""
import numpy as np
import pytest

import adaptive_full_oracle as afo
import adaptive_oracle as ada
from synth_mppi import k3_dS, k3_inputs, k3_restate, k3_S32, make_case, ws_layout
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
    """Consumer warps of the shapes the sweep uses for each count, and the refused shapes."""
    assert [ws_layout(T, nu, "W")[1] for T, nu in [(1, 1), (125, 1), (146, 1), (174, 1), (216, 1), (187, 2)]] == [7, 6, 5, 4, 3, 2]
    assert ws_layout(256, 2, "M2") is None and ws_layout(256, 2, "C") is not None
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
