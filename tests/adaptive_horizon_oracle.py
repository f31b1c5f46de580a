"""CPU reference of adaptive MPPI with a covariance over the whole horizon (``update_cov`` with ``cov_type: horizon``, DESIGN.md
section 2).

With n = T*nu and vectors over the horizon ordered (t, j) like ``U[T][nu]``, the live distribution is
``dist = (lambda, Sigma_H[n][n], L_H[n][n], Sigma_H^-1[n][n])`` (row-major, L_H the lower Cholesky factor), started at
``Sigma_H = I_T (x) Sigma0``.  The white draws come from the fixed-distribution oracle (``oracle/``) with identity colour, U = 0 and
no bounds; the colouring, clamping, the shard row, the update, the shift and the factorisation are computed here in float64.
``AdaptiveHorizonOracleBackend`` puts it behind the backend interface, so the CPU suite can drive the planner end to end.
"""
import copy

import numpy as np
import torch

import adaptive_oracle as ada
from adaptive_full_oracle import tril_pack, tril_unpack
from mppi_isaac_b200.model.blob import MODE_SIMPLE
from oracle import oracle as orc
from oracle.backend import _np


def sigma0(params, nu):
    return np.array([params.sigma0[i] for i in range(nu * nu)], np.float64).reshape(nu, nu)


def make_dist(lam, sigma_h):
    """(lambda, Sigma_H, L_H, Sigma_H^-1) from lambda and Sigma_H, computed in float64 and rounded to float32 (as the planner)."""
    s = np.asarray(sigma_h, np.float64)
    L = np.linalg.cholesky(s)
    return np.concatenate([[lam], s.ravel(), L.ravel(), np.linalg.inv(s).ravel()]).astype(np.float32)


def initial_dist(lam, sig0, T):
    return make_dist(lam, np.kron(np.eye(T), np.asarray(sig0, np.float64)))


def unpack(dist, n):
    d = np.asarray(dist)
    n2 = n * n
    return d[0], d[1:1 + n2].reshape(n, n), d[1 + n2:1 + 2 * n2].reshape(n, n), d[1 + 2 * n2:1 + 3 * n2].reshape(n, n)


def _white_params(params, nu):
    p = copy.deepcopy(params)
    p.sample_null_action = 0
    for j in range(nu):
        p.u_min[j], p.u_max[j] = -1e30, 1e30
        for i in range(nu):
            p.sigma_chol[j * nu + i] = 1.0 if i == j else 0.0
    return p


def white(model, params, seed, plan, k_offset, k_total):
    """The white Philox draws z[T][nu][K] of K1: the oracle sampler with identity colour, U = 0 and no bounds."""
    nu, T = model.nu, params.T
    a, _ = orc.sample(model, _white_params(params, nu), seed, plan, np.zeros((T, nu), np.float32), k_offset, k_total)
    return a


def colour(params, nu, U, z, dist, k_offset, k_total, prior_row=None):
    """a = clamp(U + L_H z) with the null and prior rows, noise = a - U (float64 arithmetic, float32 results)."""
    T, K = params.T, params.K
    n = T * nu
    _, _, L, _ = unpack(np.asarray(dist, np.float32), n)
    Uf = np.asarray(U, np.float32).reshape(n)
    nz = L.astype(np.float64) @ np.asarray(z, np.float64).reshape(n, K)
    a = Uf.astype(np.float64)[:, None] + nz
    kg = k_offset + np.arange(K)
    if params.sample_null_action:
        a[:, kg == k_total - 1] = 0.0
    lo = np.tile([params.u_min[j] for j in range(nu)], T)[:, None]
    hi = np.tile([params.u_max[j] for j in range(nu)], T)[:, None]
    a = np.minimum(np.maximum(a, lo), hi).astype(np.float32)
    if prior_row is not None:
        a[:, kg == k_total - 2] = np.asarray(prior_row, np.float32).reshape(n, 1)
    noise = a - Uf[:, None]
    return a.reshape(T, nu, K), noise.reshape(T, nu, K)


def scores(params, nu, cost, x, U, dist):
    """S_k of K3 in float64: sum_t gamma^t cost[t][k] (+ g^T x_k, g = lambda Sigma_H^-1 U, in SIMPLE mode)."""
    T, K = params.T, params.K
    n = T * nu
    lam, _, _, Sinv = unpack(np.asarray(dist, np.float64), n)
    S = ((float(params.gamma) ** np.arange(T))[:, None] * np.asarray(cost, np.float64).reshape(T, K)).sum(0)
    if params.mode == MODE_SIMPLE:
        g = lam * (Sinv @ np.asarray(U, np.float64).reshape(n))
        S = S + g @ np.asarray(x, np.float64).reshape(n, K)
    return S


def reduce(model, params, cost, x, U, dist):
    """The shard row (beta, eta, W[n], C[n(n+1)/2]) in float64, rounded: w_k = exp(-(S_k - beta)/lambda) (0 for a non-finite S_k),
    C = sum_k w_k (x_k - c)(x_k - c)^T with c = U (MEAN) or 0 (SIMPLE), packed as its lower triangle."""
    nu, T, K = model.nu, params.T, params.K
    n = T * nu
    lam = float(np.asarray(dist, np.float32)[0])
    S = scores(params, nu, cost, x, U, dist)
    ok = np.isfinite(S)
    beta = S[ok].min() if ok.any() else np.inf
    w = np.where(ok, np.exp(-(np.where(ok, S, beta) - beta) / lam), 0.0)
    xr = np.asarray(x, np.float64).reshape(n, K)
    W = xr @ w
    c = 0.0 if params.mode == MODE_SIMPLE else np.asarray(U, np.float64).reshape(n, 1)
    dx = xr - c
    C = (dx * w[None, :]) @ dx.T
    return np.concatenate([[beta if ok.any() else np.inf, w.sum()], W, tril_pack(C)]).astype(np.float32)


def shift_cov(Sn, sig0):
    """Sigma'[a][b] = Sn[a + nu][b + nu] for a, b < n - nu; the last block row and column are 0 but the last diagonal block, Sigma0."""
    nu = sig0.shape[0]
    n = Sn.shape[0]
    Sp = np.zeros_like(Sn)
    Sp[:n - nu, :n - nu] = Sn[nu:, nu:]
    Sp[n - nu:, n - nu:] = sig0
    return Sp


def factor(Sp):
    """(ok, L, Sigma^-1) of a symmetric Sigma' in float64; ok is False when a pivot is not finite and positive."""
    try:
        L = np.linalg.cholesky(Sp)
    except np.linalg.LinAlgError:
        return False, None, None
    if not (np.all(np.isfinite(L)) and np.all(np.diag(L) > 0)):
        return False, None, None
    Li = np.linalg.inv(L)
    I = Li.T @ Li
    return True, L, np.tril(I) + np.tril(I, -1).T


def finalize(model, params, partials, U, dist):
    """K4 with the live distribution: U update by the oracle, then the Sigma_H update, the shift, L_H and Sigma_H^-1, and the lambda
    rule; returns (U, action, stats, dist).  A shifted Sigma_H that is not positive definite leaves the three unchanged."""
    nu, T = model.nu, params.T
    n = T * nu
    partials = np.asarray(partials, np.float32).reshape(-1, 2 + n + n * (n + 1) // 2)
    d = np.asarray(dist, np.float32).copy()
    p = copy.deepcopy(params)
    p.lambda_ = float(d[0])
    U_old = np.asarray(U, np.float32).reshape(T, nu).copy()
    Un, act, stats = orc.finalize(model, p, partials[:, :2 + n], U_old)
    e = float(stats[1])
    if not e > 0:
        return Un, act, stats, d
    p_nf = copy.deepcopy(p)
    p_nf.filter_u = 0
    U_pre, _, _ = orc.finalize(model, p_nf, partials[:, :2 + n], U_old)            # the mean update before Savitzky-Golay
    rows = partials.astype(np.float64)
    valid = rows[:, 1] > 0
    b = rows[valid, 0].min()
    s = np.where(valid, np.exp(-(np.where(valid, rows[:, 0], b) - b) / float(d[0])), 0.0)
    eta = (s * rows[:, 1]).sum()
    W = (s[:, None] * rows[:, 2:2 + n]).sum(0)
    C = tril_unpack((s[:, None] * rows[:, 2 + n:]).sum(0), n)
    c = 0.0 if params.mode == MODE_SIMPLE else U_old.reshape(n).astype(np.float64)
    m1 = W / eta - c
    dd = U_pre.reshape(n).astype(np.float64) - U_old.reshape(n)
    V = C / eta - (np.outer(m1, dd) + np.outer(dd, m1) - np.outer(dd, dd))
    _, Sig, _, _ = unpack(d, n)
    sc = float(params.step_size_cov)
    Sn = (1 - sc) * Sig.astype(np.float64) + sc * V + float(params.kappa) * np.eye(n)
    Sn = np.tril(Sn) + np.tril(Sn, -1).T
    Sp = shift_cov(Sn, sigma0(params, nu).astype(np.float32).astype(np.float64))
    ok, L, Si = factor(Sp)
    if ok:
        n2 = n * n
        d[1:1 + n2] = Sp.ravel().astype(np.float32)
        d[1 + n2:1 + 2 * n2] = L.ravel().astype(np.float32)
        d[1 + 2 * n2:1 + 3 * n2] = Si.ravel().astype(np.float32)
    if params.update_lambda:
        lam, f32 = d[0], np.float32
        if e > params.eta_u_bound:
            lam = lam * (f32(1) - f32(params.lambda_mult))
        elif e < params.eta_l_bound:
            lam = lam * (f32(1) + f32(params.lambda_mult))
        lam0 = f32(params.lambda_)
        d[0] = min(max(lam, f32(1e-3) * lam0), f32(1e3) * lam0)
    return Un, act, stats, d


class AdaptiveHorizonOracleBackend(ada.AdaptiveOracleBackend):
    """The adaptive oracle backend, which also runs the horizon rule when the parameter block has cov_horizon."""

    def _hzn(self):
        return self._cov() and bool(self.params.cov_horizon)

    def sample(self, seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr=None):
        if not self._hzn():
            return super().sample(seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr)
        plan = plan_idx + (int(plan_ctr[0]) if plan_ctr is not None else 0)
        z = white(self.model, self.params, seed, plan, k_offset, k_total)
        a, n = colour(self.params, self.model.nu, _np(U), z, _np(self.dist), k_offset, k_total, _np(prior_row))
        actions.copy_(torch.from_numpy(a))
        if noise is not None:
            noise.copy_(torch.from_numpy(n))

    def sample_library(self, k_offset, k_total, U, prior_row, Z, actions, noise):
        if not self._hzn():
            return super().sample_library(k_offset, k_total, U, prior_row, Z, actions, noise)
        a, n = colour(self.params, self.model.nu, _np(U), _np(Z), _np(self.dist), k_offset, k_total, _np(prior_row))
        actions.copy_(torch.from_numpy(a))
        if noise is not None:
            noise.copy_(torch.from_numpy(n))

    def reduce(self, cost, x, U, partial):
        if not self._hzn():
            return super().reduce(cost, x, U, partial)
        partial.copy_(torch.from_numpy(reduce(self.model, self.params, _np(cost.contiguous()), _np(x), _np(U), _np(self.dist))))

    def finalize(self, partials, G, U, action_out, stats):
        if not self._hzn():
            return super().finalize(partials, G, U, action_out, stats)
        Un, act, st, d = finalize(self.model, self.params, _np(partials.contiguous())[:G], _np(U), _np(self.dist))
        U.copy_(torch.from_numpy(Un))
        action_out.copy_(torch.from_numpy(act))
        if stats is not None:
            stats.copy_(torch.from_numpy(st))
        self.dist.copy_(torch.from_numpy(d))
