"""CPU: the temporal covariance of colored-noise sampling (``sampling_method: colored``) against the FFT recipe it restates, the
config refusals, and the planner planning with colored noise on the checker backend."""
import math

import numpy as np
import pytest
import torch

import colored_oracle as co
from mppi_isaac_b200.model.blob import make_params
from mppi_isaac_b200.planner.mppi import colored_noise_chol, colored_noise_cov
from mppi_isaac_b200.utils.config_store import IsaacGymConfig
from scenes import panda_cfg, panda_mppi, panda_setup

TS = [1, 2, 12, 30, 31, 256]
BETAS = [0.0, 1.0, 2.0, 2.5, 3.0]


@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("beta", BETAS)
def test_covariance_is_circulant_unit_diagonal_and_positive_definite(T, beta):
    S = colored_noise_cov(T, beta)
    assert S.shape == (T, T) and S.dtype == np.float64
    np.testing.assert_array_equal(np.diag(S), 1.0)
    np.testing.assert_array_equal(S, S.T)
    for t in range(T):                                                      # circulant: each row the previous one shifted by one
        np.testing.assert_array_equal(S[t], np.roll(S[0], t))
    assert np.linalg.eigvalsh(S).min() > 0
    L = colored_noise_chol(T, beta)
    assert L.dtype == np.float32 and np.all(np.isfinite(L))
    np.testing.assert_array_equal(L, np.tril(L))
    if beta == 0.0:
        np.testing.assert_array_equal(S, np.eye(T))                         # exactly I: colored at beta = 0 is the white draw bit for bit
        np.testing.assert_array_equal(L, np.eye(T, dtype=np.float32))


@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("beta", BETAS)
def test_covariance_equals_the_fft_recipe(T, beta):
    """The formula against the exact covariance of the linear FFT recipe (to round-off) and against the empirical correlation of
    2e5 draws of it.  The draws are unit-variance Gaussians after normalisation, so an empirical correlation has standard error
    (1 - rho^2) / sqrt(N) <= 1 / sqrt(N) = 2.2e-3; the gate is 6 of those (about 1e-9 per entry of a correct formula)."""
    S = colored_noise_cov(T, beta)
    np.testing.assert_allclose(co.recipe_cov(T, beta), S, rtol=0, atol=1e-12)
    N, chunk = 200_000, 20_000
    rng = np.random.default_rng(1000 * T + int(10 * beta))
    M = np.zeros((T, T))
    for _ in range(N // chunk):
        y = co.fft_recipe(T, beta, chunk, rng)
        M += y.T @ y
    d = np.sqrt(np.diag(M))
    R = M / np.outer(d, d)
    err = np.abs(R - S).max()
    assert err <= 6.0 / math.sqrt(N), f"T={T} beta={beta}: |R - Sigma_b| = {err:.2e}"
    if T >= 12 and beta >= 1.0:                                             # a white model must miss the same gate
        assert np.abs(R - np.eye(T)).max() > 6.0 / math.sqrt(N)


def test_larger_beta_gives_smoother_sequences():
    T = 30
    rho1 = [colored_noise_cov(T, b)[0, 1] for b in BETAS]
    assert rho1[0] == 0.0 and all(b > a for a, b in zip(rho1, rho1[1:]))


@pytest.mark.parametrize("beta", [-0.5, float("nan"), float("inf"), float("-inf")])
def test_make_params_refuses_a_bad_beta(beta):
    sc, _, _ = panda_setup(K=4, T=12)
    with pytest.raises(ValueError, match="noise_beta"):
        make_params(panda_mppi(64, 12, sampling_method="colored", noise_beta=beta), IsaacGymConfig(), sc.nu, 64, [])


def test_make_params_refuses_colored_with_cov_type_horizon():
    sc, _, _ = panda_setup(K=4, T=12)
    with pytest.raises(ValueError, match="horizon"):
        make_params(panda_mppi(64, 12, sampling_method="colored", update_cov=True, cov_type="horizon"), IsaacGymConfig(), sc.nu, 64, [])
    for cov_type in ("diag", "full"):                                     # the other update rules combine with colored noise
        make_params(panda_mppi(64, 12, sampling_method="colored", update_cov=True, cov_type=cov_type), IsaacGymConfig(), sc.nu, 64, [])
    make_params(panda_mppi(64, 12, sampling_method="colored", noise_beta=0.0), IsaacGymConfig(), sc.nu, 64, [])


def test_colour_restatement_at_beta_zero_is_the_white_sampler(oracle):
    """With L_b = I the reference is the fixed-distribution oracle sampler (same draws, colour, clamp, null and prior rows)."""
    sc, p, _ = panda_setup(K=64, T=12)
    U = np.random.default_rng(0).uniform(-0.1, 0.1, (12, 7)).astype(np.float32)
    prior = np.full((12, 7), 0.05, np.float32)
    z = co.white(sc.model, p, 7, 3, 0, 64)
    a, n = co.colour(p, 7, U, z, colored_noise_chol(12, 0.0), 0, 64, prior)
    a_ref, n_ref = oracle.sample(sc.model, p, 7, 3, U, 0, 64, prior)
    assert np.abs(a - a_ref).max() <= 1e-6 and np.abs(n - n_ref).max() <= 1e-6
    np.testing.assert_array_equal(a[:, :, 63], 0.0)
    np.testing.assert_array_equal(a[:, :, 62], prior)


@pytest.mark.parametrize("flags", [{}, dict(update_cov=True, update_lambda=True), dict(update_cov=True, cov_type="full")])
def test_planner_plans_with_colored_noise_on_the_checker_backend(flags):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    cfg = panda_cfg(K=64, T=12, device="cpu", sampling_method="colored", noise_beta=2.0, **flags)
    pl = MPPIisaacPlanner(cfg, PandaReachObjective(), backend=co.ColoredOracleBackend())
    m = pl.mppi
    assert m.use_colored and not m.use_library
    np.testing.assert_array_equal(m._noise_Lt.numpy(), colored_noise_chol(12, 2.0))
    q = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
    seen = []
    for _ in range(3):
        a = pl.compute_action(q, [0.0] * 7)
        assert torch.isfinite(a).all()
        seen.append(m.noise.clone())
    assert not torch.equal(seen[0], seen[1])                                # fresh noise on every plan
    body = m.noise[:, :, :-1].numpy().astype(np.float64)                    # the null row excluded
    lag1 = np.mean([np.corrcoef(body[:-1, j].ravel(), body[1:, j].ravel())[0, 1] for j in range(7)])
    assert lag1 > 0.5                                                      # neighbouring steps of a sample are correlated
    pl.update_mppi_params({"noise_sigma": (0.05 * np.eye(7)).tolist()})    # a rebuild builds L_b again
    assert pl.mppi.use_colored and pl.mppi._noise_Lt is not None and pl.mppi._noise_Lt.shape == (12, 12)
    pl.compute_action(q, [0.0] * 7)


def test_planner_rejects_colored_with_horizon_and_builds_for_a_new_beta():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    with pytest.raises(ValueError, match="horizon"):
        MPPIisaacPlanner(panda_cfg(K=64, T=12, device="cpu", sampling_method="colored", update_cov=True, cov_type="horizon"), PandaReachObjective(),
                         backend=co.ColoredOracleBackend())
    pl = MPPIisaacPlanner(panda_cfg(K=64, T=9, device="cpu", sampling_method="colored", noise_beta=0.0), PandaReachObjective(),
                          backend=co.ColoredOracleBackend())
    np.testing.assert_array_equal(pl.mppi._noise_Lt.numpy(), np.eye(9, dtype=np.float32))
