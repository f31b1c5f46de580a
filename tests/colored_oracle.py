"""CPU reference of colored-noise sampling (``sampling_method: colored``, DESIGN.md section 2) for the tests.

The temporal covariance Sigma_b of power-law noise comes from ``planner.mppi.colored_noise_cov``; here it is restated from the FFT
recipe of ``powerlaw_psd_gaussian`` (iCEM), both as random draws and as the exact covariance of that linear recipe.  K1's colored
draw is restated in float64 from the white Philox draws of the fixed-distribution oracle: w[t] = sum_{t' <= t} L_b[t][t'] z[t'],
then the control-space colour (the fixed L0, or the live diagonal / full one of a registered distribution), the clamp and the null /
prior rows.  ``ColoredOracleBackend`` puts it behind the backend interface, so the CPU suite can drive the planner end to end.
"""
import numpy as np
import torch

import adaptive_full_oracle as afo
import adaptive_horizon_oracle as aho
from oracle.backend import _np


def _recipe_scales(T, beta):
    """Per-frequency standard deviations of the recipe, s_m = max(f_m, 1/T)^(-beta/2), f_m = m / T (the fmin = 1/T clip)."""
    f = np.fft.rfftfreq(T)
    return np.maximum(f, 1.0 / T) ** (-beta / 2.0)


def fft_recipe(T, beta, N, rng):
    """N draws (N, T) of the powerlaw_psd_gaussian recipe restated in NumPy (without its final scalar normalisation): real and
    imaginary parts N(0, s_m^2), the imaginary parts of DC and (T even) Nyquist zero and their real parts scaled by sqrt(2), irfft."""
    s = _recipe_scales(T, beta)
    sr = rng.standard_normal((N, s.size)) * s
    si = rng.standard_normal((N, s.size)) * s
    if T % 2 == 0:
        si[:, -1] = 0.0
        sr[:, -1] *= np.sqrt(2.0)
    si[:, 0] = 0.0
    sr[:, 0] *= np.sqrt(2.0)
    return np.fft.irfft(sr + 1j * si, n=T, axis=-1)


def recipe_cov(T, beta):
    """The exact covariance of ``fft_recipe`` normalised to unit diagonal: the recipe is linear in its Gaussian inputs g, y = A g, so
    Cov = A A^T with the columns of A the recipe applied to unit inputs."""
    s = _recipe_scales(T, beta)
    cols = []
    for m in range(s.size):
        edge = m == 0 or (T % 2 == 0 and m == s.size - 1)
        e = np.zeros(s.size, complex)
        e[m] = s[m] * (np.sqrt(2.0) if edge else 1.0)
        cols.append(np.fft.irfft(e, n=T))
        if not edge:
            e[m] = 1j * s[m]
            cols.append(np.fft.irfft(e, n=T))
    A = np.stack(cols, axis=1)
    C = A @ A.T
    d = np.sqrt(np.diag(C))
    return C / np.outer(d, d)


def white(model, params, seed, plan, k_offset, k_total):
    """The white Philox draws z[T][nu][K] of K1 (the oracle sampler with identity colour, U = 0, no bounds, no null row)."""
    return aho.white(model, params, seed, plan, k_offset, k_total)


def control_chol(params, nu, dist=None):
    """The float32 control-space factor K1 colours with: L0 = chol(Sigma); with update_cov and a registered distribution the live
    diag(sqrtf(cov)) or, cov_full, the live L."""
    if dist is not None and params.update_cov:
        d = np.asarray(dist, np.float32)
        if params.cov_full:
            return afo.unpack(d, nu)[2]
        return np.diag(np.sqrt(d[1:1 + nu]))
    return np.array(params.sigma_chol[:nu * nu], np.float32).reshape(nu, nu)


def colour(params, nu, U, z, Lt, k_offset, k_total, prior_row=None, dist=None, clamp=True):
    """(actions, noise) [T][nu][K] float32 of colored K1 from the white draws z, computed in float64: noise = L (L_b z) over
    (control, time), a = clamp(U + noise) with the null row (global k_total - 1) and the prior row (k_total - 2), noise := a - U."""
    T, K = params.T, np.asarray(z).shape[-1]
    L = control_chol(params, nu, dist).astype(np.float64)
    w = np.einsum("ts,sik->tik", np.asarray(Lt, np.float32).astype(np.float64), np.asarray(z, np.float64), optimize=True)
    n = np.einsum("ji,tik->tjk", L, w, optimize=True)
    Uf = np.asarray(U, np.float32).reshape(T, nu)
    a = Uf.astype(np.float64)[:, :, None] + n
    kg = k_offset + np.arange(K)
    if params.sample_null_action:
        a[:, :, kg == k_total - 1] = 0.0
    if clamp:
        lo = np.array([params.u_min[j] for j in range(nu)], np.float32).astype(np.float64)[None, :, None]
        hi = np.array([params.u_max[j] for j in range(nu)], np.float32).astype(np.float64)[None, :, None]
        a = np.minimum(np.maximum(a, lo), hi)
    a = a.astype(np.float32)
    if prior_row is not None:
        a[:, :, kg == k_total - 2] = np.asarray(prior_row, np.float32).reshape(T, nu, 1)
    return a, a - Uf[:, :, None]


class ColoredOracleBackend(afo.AdaptiveFullOracleBackend):
    """The adaptive oracle backend (fixed, diagonal and full Sigma) with colored K1."""

    def sample_colored(self, seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr=None):
        plan = plan_idx + (int(plan_ctr[0]) if plan_ctr is not None else 0)
        z = white(self.model, self.params, seed, plan, k_offset, k_total)
        a, n = colour(self.params, self.model.nu, _np(U), z, _np(Lt), k_offset, k_total, _np(prior_row),
                      _np(self.dist) if self._cov() else None)
        actions.copy_(torch.from_numpy(a))
        if noise is not None:
            noise.copy_(torch.from_numpy(n))
