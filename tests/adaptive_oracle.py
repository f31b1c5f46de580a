"""CPU reference of adaptive MPPI (``update_cov`` / ``update_lambda``, DESIGN.md section 2) for the tests.

It composes the fixed-distribution oracle (``oracle/``) with the adaptive rules: the live distribution ``dist = (lambda, cov[nu])``
is turned into a parameter block (lambda, and with ``update_cov`` Sigma = diag(cov)) for the oracle's K1 / K3 / K4, the
second-moment row and the distribution update are computed here in float64.  ``AdaptiveOracleBackend`` puts it behind the
backend interface, so the CPU suite can drive the adaptive planner end to end.
"""
import copy

import numpy as np
import torch

from mppi_isaac_b200.model.blob import MODE_SIMPLE
from oracle import oracle as orc
from oracle.backend import OracleBackend, _np


def dist_params(params, nu, dist, white=False):
    """The fixed-distribution parameter block equivalent to the live `dist` (white: identity colour for the noise library)."""
    p = copy.deepcopy(params)
    d = np.asarray(dist, np.float32)
    p.lambda_ = float(d[0])
    if params.update_cov:
        cov = d[1:1 + nu]
        for j in range(nu):
            for i in range(nu):
                p.sigma_chol[j * nu + i] = (1.0 if white else float(np.sqrt(cov[j]))) if i == j else 0.0
                p.sigma_inv[j * nu + i] = float(np.float32(1.0) / cov[j]) if i == j else 0.0
    return p


def reduce(model, params, cost, x, U, dist):
    """K3 with the live distribution: (beta, eta, W) from the oracle, + M2 = sum_k w_k (x - c)^2 (float64) with update_cov."""
    nu, T, K = model.nu, params.T, params.K
    p = dist_params(params, nu, dist)
    row, _ = orc.reduce(model, p, cost, x, U)
    if not params.update_cov:
        return row
    cost = np.asarray(cost, np.float64).reshape(T, K)
    xr = np.asarray(x, np.float64).reshape(T * nu, K)
    Uf = np.asarray(U, np.float64).reshape(T * nu)
    S = ((float(params.gamma) ** np.arange(T))[:, None] * cost).sum(0)
    if params.mode == MODE_SIMPLE:
        cov = np.asarray(dist, np.float64)[1:1 + nu]
        g = float(p.lambda_) * (Uf / np.tile(cov, T))
        S = S + g @ xr
    ok = np.isfinite(S)
    beta = S[ok].min() if ok.any() else np.inf
    w = np.where(ok, np.exp(-(np.where(ok, S, beta) - beta) / float(p.lambda_)), 0.0)
    c = 0.0 if params.mode == MODE_SIMPLE else Uf[:, None]
    M2 = ((xr - c) ** 2 * w[None, :]).sum(1)
    return np.concatenate([row, M2.astype(np.float32)])


def finalize(model, params, partials, U, dist):
    """K4 with the live distribution: U update by the oracle, then the cov / lambda rules; returns (U, action, stats, dist)."""
    nu, T = model.nu, params.T
    NR = T * nu
    partials = np.asarray(partials, np.float32).reshape(-1, 2 + NR * (2 if params.update_cov else 1))
    d = np.asarray(dist, np.float32).copy()
    p = dist_params(params, nu, d)
    U_old = np.asarray(U, np.float32).reshape(T, nu).copy()
    Un, act, stats = orc.finalize(model, p, partials[:, :2 + NR], U_old)
    e = float(stats[1])
    if not e > 0:
        return Un, act, stats, d
    if params.update_cov:
        p_nf = copy.deepcopy(p)
        p_nf.filter_u = 0
        U_pre, _, _ = orc.finalize(model, p_nf, partials[:, :2 + NR], U_old)        # the mean update before Savitzky-Golay
        rows = partials.astype(np.float64)
        valid = rows[:, 1] > 0
        b = rows[valid, 0].min()
        s = np.where(valid, np.exp(-(np.where(valid, rows[:, 0], b) - b) / float(d[0])), 0.0)
        eta = (s * rows[:, 1]).sum()
        W = (s[:, None] * rows[:, 2:2 + NR]).sum(0)
        M2 = (s[:, None] * rows[:, 2 + NR:]).sum(0)
        c = 0.0 if params.mode == MODE_SIMPLE else U_old.reshape(-1).astype(np.float64)
        m1 = W / eta - c
        dd = U_pre.reshape(-1).astype(np.float64) - U_old.reshape(-1)
        var = np.maximum(M2 / eta - 2 * dd * m1 + dd * dd, 0.0).reshape(T, nu)
        upd = var.mean(0)
        cov = d[1:1 + nu].astype(np.float64)
        d[1:1 + nu] = ((1 - params.step_size_cov) * cov + params.step_size_cov * upd + params.kappa).astype(np.float32)
    if params.update_lambda:
        lam, f32 = d[0], np.float32
        if e > params.eta_u_bound:
            lam = lam * (f32(1) - f32(params.lambda_mult))
        elif e < params.eta_l_bound:
            lam = lam * (f32(1) + f32(params.lambda_mult))
        lam0 = f32(params.lambda_)
        d[0] = min(max(lam, f32(1e-3) * lam0), f32(1e3) * lam0)
    return Un, act, stats, d


class AdaptiveOracleBackend(OracleBackend):
    """OracleBackend + a registered distribution (a CPU tensor, updated in place like the device buffer of the CUDA backend)."""

    name = "oracle"

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.dist = None

    def set_distribution(self, dist):
        self.dist = dist

    def _p(self, white=False):
        return dist_params(self.params, self.model.nu, _np(self.dist), white)

    def _cov(self):
        return self.dist is not None and bool(self.params.update_cov)

    def sample(self, seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr=None):
        if not self._cov():
            return super().sample(seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr)
        plan = plan_idx + (int(plan_ctr[0]) if plan_ctr is not None else 0)
        a, n = orc.sample(self.model, self._p(), seed, plan, _np(U), k_offset, k_total, _np(prior_row), self.nthreads)
        actions.copy_(torch.from_numpy(a))
        if noise is not None:
            noise.copy_(torch.from_numpy(n))

    def noise_library(self, k_offset, k_total, halton_tab, B, n_knots, Z):
        if not self._cov():
            return super().noise_library(k_offset, k_total, halton_tab, B, n_knots, Z)
        Z.copy_(torch.from_numpy(orc.noise_library(self.model, self._p(white=True), _np(halton_tab), _np(B), n_knots, k_offset, k_total)))

    def sample_library(self, k_offset, k_total, U, prior_row, Z, actions, noise):
        if not self._cov():
            return super().sample_library(k_offset, k_total, U, prior_row, Z, actions, noise)
        nu = self.model.nu
        Zs = np.sqrt(_np(self.dist)[1:1 + nu].astype(np.float32))[None, :, None] * _np(Z)
        a, n = orc.sample_library(self.model, self.params, _np(U), Zs, k_offset, k_total, _np(prior_row))
        actions.copy_(torch.from_numpy(a))
        if noise is not None:
            noise.copy_(torch.from_numpy(n))

    def reduce(self, cost, x, U, partial):
        if self.dist is None:
            return super().reduce(cost, x, U, partial)
        partial.copy_(torch.from_numpy(reduce(self.model, self.params, _np(cost.contiguous()), _np(x), _np(U), _np(self.dist))))

    def finalize(self, partials, G, U, action_out, stats):
        if self.dist is None:
            return super().finalize(partials, G, U, action_out, stats)
        Un, act, st, d = finalize(self.model, self.params, _np(partials.contiguous())[:G], _np(U), _np(self.dist))
        U.copy_(torch.from_numpy(Un))
        action_out.copy_(torch.from_numpy(act))
        if stats is not None:
            stats.copy_(torch.from_numpy(st))
        self.dist.copy_(torch.from_numpy(d))
