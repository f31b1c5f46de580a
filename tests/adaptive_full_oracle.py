"""CPU reference of adaptive MPPI with a full sampling covariance (``update_cov`` with ``cov_type: full``, DESIGN.md section 2).

The live distribution is ``dist = (lambda, Sigma[nu][nu], L[nu][nu], Sigma^-1[nu][nu])`` (row-major, L the lower Cholesky factor).
The fixed-distribution oracle (``oracle/``) runs K1 / K3 / K4 with the live L and Sigma^-1 substituted into ``sigma_chol`` /
``sigma_inv``; the covariance row C of K3 and the update of Sigma, L and Sigma^-1 are computed here in float64.
``AdaptiveFullOracleBackend`` puts it behind the backend interface, so the CPU suite can drive the planner end to end.
"""
import copy

import numpy as np
import torch

import adaptive_oracle as ada
from mppi_isaac_b200.model.blob import MODE_SIMPLE
from oracle import oracle as orc
from oracle.backend import _np


def make_dist(lam, sigma):
    """(lambda, Sigma, L, Sigma^-1) from lambda and Sigma, computed in float64 and rounded to float32 (as the planner builds it)."""
    s = np.asarray(sigma, np.float64)
    L = np.linalg.cholesky(s)
    return np.concatenate([[lam], s.ravel(), L.ravel(), np.linalg.inv(s).ravel()]).astype(np.float32)


def unpack(dist, nu):
    d = np.asarray(dist)
    n2 = nu * nu
    return d[0], d[1:1 + n2].reshape(nu, nu), d[1 + n2:1 + 2 * n2].reshape(nu, nu), d[1 + 2 * n2:1 + 3 * n2].reshape(nu, nu)


def tril_pack(M):
    """Lower triangle (i >= j), row-major: the layout of C in the shard row."""
    i, j = np.tril_indices(M.shape[0])
    return M[i, j]


def tril_unpack(c, nu):
    M = np.zeros((nu, nu), np.float64)
    i, j = np.tril_indices(nu)
    M[i, j] = c
    M[j, i] = c
    return M


def dist_params(params, nu, dist, white=False):
    """The fixed-distribution parameter block equivalent to the live `dist` (white: identity colour for the noise library)."""
    p = copy.deepcopy(params)
    lam, _, L, Sinv = unpack(np.asarray(dist, np.float32), nu)
    p.lambda_ = float(lam)
    for j in range(nu):
        for i in range(nu):
            p.sigma_chol[j * nu + i] = (1.0 if i == j else 0.0) if white else float(L[j, i])
            p.sigma_inv[j * nu + i] = float(Sinv[j, i])
    return p


def color_library(dist, nu, Z):
    """The white library Z[T][nu][K] coloured by the live L: Zs[t][:, k] = L Z[t][:, k]."""
    _, _, L, _ = unpack(np.asarray(dist, np.float32), nu)
    return np.einsum("ji,tik->tjk", L.astype(np.float64), np.asarray(Z, np.float64)).astype(np.float32)


def weights(params, nu, cost, x, U, dist):
    """float64 weights of K3 with the live temperature and, in SIMPLE mode, the live Sigma^-1."""
    T, K = params.T, params.K
    lam, _, _, Sinv = unpack(np.asarray(dist, np.float64), nu)
    cost = np.asarray(cost, np.float64).reshape(T, K)
    xr = np.asarray(x, np.float64).reshape(T, nu, K)
    Uf = np.asarray(U, np.float64).reshape(T, nu)
    S = ((float(params.gamma) ** np.arange(T))[:, None] * cost).sum(0)
    if params.mode == MODE_SIMPLE:
        S = S + lam * np.einsum("tj,ij,tik->k", Uf, Sinv, xr)
    ok = np.isfinite(S)
    beta = S[ok].min() if ok.any() else np.inf
    return np.where(ok, np.exp(-(np.where(ok, S, beta) - beta) / lam), 0.0)


def reduce(model, params, cost, x, U, dist):
    """K3 with the live distribution: (beta, eta, W) from the oracle, + C = sum_t sum_k w_k (x_tk - c_t)(x_tk - c_t)^T (float64),
    packed as its lower triangle."""
    nu, T, K = model.nu, params.T, params.K
    row, _ = orc.reduce(model, dist_params(params, nu, dist), cost, x, U)
    w = weights(params, nu, cost, x, U, dist)
    xr = np.asarray(x, np.float64).reshape(T, nu, K)
    c = 0.0 if params.mode == MODE_SIMPLE else np.asarray(U, np.float64).reshape(T, nu)[:, :, None]
    dx = xr - c
    C = np.einsum("tik,tjk,k->ij", dx, dx, w)
    return np.concatenate([row, tril_pack(C).astype(np.float32)])


def finalize(model, params, partials, U, dist):
    """K4 with the live distribution: U update by the oracle, then the Sigma / L / Sigma^-1 update and the lambda rule; returns
    (U, action, stats, dist).  A Sigma update that is not positive definite leaves Sigma, L and Sigma^-1 unchanged."""
    nu, T = model.nu, params.T
    NR, npairs = T * nu, nu * (nu + 1) // 2
    partials = np.asarray(partials, np.float32).reshape(-1, 2 + NR + npairs)
    d = np.asarray(dist, np.float32).copy()
    p = dist_params(params, nu, d)
    U_old = np.asarray(U, np.float32).reshape(T, nu).copy()
    Un, act, stats = orc.finalize(model, p, partials[:, :2 + NR], U_old)
    e = float(stats[1])
    if not e > 0:
        return Un, act, stats, d
    p_nf = copy.deepcopy(p)
    p_nf.filter_u = 0
    U_pre, _, _ = orc.finalize(model, p_nf, partials[:, :2 + NR], U_old)            # the mean update before Savitzky-Golay
    rows = partials.astype(np.float64)
    valid = rows[:, 1] > 0
    b = rows[valid, 0].min()
    s = np.where(valid, np.exp(-(np.where(valid, rows[:, 0], b) - b) / float(d[0])), 0.0)
    eta = (s * rows[:, 1]).sum()
    W = (s[:, None] * rows[:, 2:2 + NR]).sum(0).reshape(T, nu)
    C = tril_unpack((s[:, None] * rows[:, 2 + NR:]).sum(0), nu)
    c = 0.0 if params.mode == MODE_SIMPLE else U_old.astype(np.float64)
    m1 = W / eta - c
    dd = U_pre.astype(np.float64) - U_old
    V = C / eta - (np.einsum("ti,tj->ij", m1, dd) + np.einsum("ti,tj->ij", dd, m1) - np.einsum("ti,tj->ij", dd, dd))
    _, Sig, _, _ = unpack(d, nu)
    sc = float(params.step_size_cov)
    Sn = (1 - sc) * Sig.astype(np.float64) + (sc / T) * V + float(params.kappa) * np.eye(nu)
    Sn = np.tril(Sn) + np.tril(Sn, -1).T                                             # the lower triangle in both halves
    try:
        L = np.linalg.cholesky(Sn)
        ok = bool(np.all(np.isfinite(L)) and np.all(np.diag(L) > 0))
    except np.linalg.LinAlgError:
        ok = False
    if ok:
        n2 = nu * nu
        d[1:1 + n2] = Sn.ravel().astype(np.float32)
        d[1 + n2:1 + 2 * n2] = L.ravel().astype(np.float32)
        Li = np.linalg.inv(L)
        I = Li.T @ Li                                                           # Sigma^-1 = L^-T L^-1, lower triangle in both halves
        d[1 + 2 * n2:1 + 3 * n2] = (np.tril(I) + np.tril(I, -1).T).ravel().astype(np.float32)
    if params.update_lambda:
        lam, f32 = d[0], np.float32
        if e > params.eta_u_bound:
            lam = lam * (f32(1) - f32(params.lambda_mult))
        elif e < params.eta_l_bound:
            lam = lam * (f32(1) + f32(params.lambda_mult))
        lam0 = f32(params.lambda_)
        d[0] = min(max(lam, f32(1e-3) * lam0), f32(1e3) * lam0)
    return Un, act, stats, d


class AdaptiveFullOracleBackend(ada.AdaptiveOracleBackend):
    """The adaptive oracle backend, which also runs the full-covariance rule when the parameter block has cov_full."""

    def _full(self):
        return self._cov() and bool(self.params.cov_full)

    def _p(self, white=False):
        if not self._full():
            return super()._p(white)
        return dist_params(self.params, self.model.nu, _np(self.dist), white)

    def sample_library(self, k_offset, k_total, U, prior_row, Z, actions, noise):
        if not self._full():
            return super().sample_library(k_offset, k_total, U, prior_row, Z, actions, noise)
        Zs = color_library(_np(self.dist), self.model.nu, _np(Z))
        a, n = orc.sample_library(self.model, self.params, _np(U), Zs, k_offset, k_total, _np(prior_row))
        actions.copy_(torch.from_numpy(a))
        if noise is not None:
            noise.copy_(torch.from_numpy(n))

    def reduce(self, cost, x, U, partial):
        if not self._full():
            return super().reduce(cost, x, U, partial)
        partial.copy_(torch.from_numpy(reduce(self.model, self.params, _np(cost.contiguous()), _np(x), _np(U), _np(self.dist))))

    def finalize(self, partials, G, U, action_out, stats):
        if not self._full():
            return super().finalize(partials, G, U, action_out, stats)
        Un, act, st, d = finalize(self.model, self.params, _np(partials.contiguous())[:G], _np(U), _np(self.dist))
        U.copy_(torch.from_numpy(Un))
        action_out.copy_(torch.from_numpy(act))
        if stats is not None:
            stats.copy_(torch.from_numpy(st))
        self.dist.copy_(torch.from_numpy(d))
