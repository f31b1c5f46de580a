"""CPU reference of multi-modal MPPI (``n_modes`` / ``mode_switch_margin``, DESIGN.md section 2) for the tests.

Global sample kg belongs to mode kg // Kc.  K1 of mode m is the oracle's own K1 with U := U_m on the columns of mode m.  K3 writes one
block (beta_m, eta_m, W_m) per mode over the shard's samples of that mode, in float64 rounded to float32.  K4 combines the blocks of every
mode as today's K4 combines rows, forms the own steps d_m and free energies F_m, couples the modes by the Stein-variational step with the
median bandwidth, applies Savitzky-Golay and the clamp, and selects the executed mode, all in float64.  ``ModesOracleBackend`` puts it
behind the backend interface, so the CPU suite can drive the planner end to end.
"""
import numpy as np
import torch

import colored_oracle as co
import risk_oracle as ro
from mppi_isaac_b200.model.blob import MODE_SIMPLE
from oracle.backend import _np

SG_MID = np.array([-21.0, 14.0, 39.0, 54.0, 59.0, 54.0, 39.0, 14.0, -21.0]) / 231.0
SG_EDGE = np.array([[763.0, 441.0, 189.0, 7.0, -105.0, -147.0, -119.0, -21.0, 147.0],
                    [441.0, 322.0, 220.5, 136.5, 70.0, 21.0, -10.5, -24.5, -21.0],
                    [189.0, 220.5, 232.0, 223.5, 195.0, 146.5, 78.0, -10.5, -119.0],
                    [7.0, 136.5, 223.5, 268.0, 270.0, 229.5, 146.5, 21.0, -147.0]]) / 1155.0


def f32(v):
    return float(np.float32(v))


def modes_of(params, k_offset, K):
    """(K,) mode of every local sample of a shard [k_offset, k_offset + K)."""
    return (int(k_offset) + np.arange(int(K))) // int(params.mode_samples)


def sample(call, params, U, k_offset, K, outs):
    """Run `call(U_m, *outs_m)` once per mode on full-size buffers and keep the columns of mode m (the counters are global)."""
    M = int(params.n_modes)
    mo = modes_of(params, k_offset, K)
    for m in range(M):
        cols = np.nonzero(mo == m)[0]
        if cols.size == 0:
            continue
        tmp = [None if o is None else torch.zeros_like(o) for o in outs]
        call(U[m].contiguous(), *tmp)
        for o, t in zip(outs, tmp):
            if o is not None:
                o[..., cols] = t[..., cols]


def reduce(params, nu, cost, x, U, k_offset=None):
    """The shard row [M][2 + T*nu] in float64, rounded to float32: block m = (beta_m, eta_m, W_m) over the shard's samples of mode m
    (S with g_m = lambda Sigma^-1 U_m in SIMPLE mode); (+inf, 0, 0) for a mode without a valid sample."""
    T, M = int(params.T), int(params.n_modes)
    cost = np.asarray(cost, np.float64).reshape(T, -1)
    K = cost.shape[1]
    x = np.asarray(x, np.float64).reshape(T, nu, K)
    mo = modes_of(params, params.k_offset if k_offset is None else k_offset, K)
    U = np.asarray(U, np.float32).reshape(M, T, nu)
    rows = []
    for m in range(M):
        cols = np.nonzero(mo == m)[0]
        row = np.zeros(2 + T * nu)
        row[0] = np.inf
        if cols.size:
            S, lam = ro.scores(params, nu, cost[:, cols], x[:, :, cols], U[m])
            ok = np.isfinite(S)
            if ok.any():
                beta = S[ok].min()
                w = np.where(ok, np.exp(-(np.where(ok, S, beta) - beta) / lam), 0.0)
                row[0], row[1] = beta, w.sum()
                row[2:] = np.einsum("tjk,k->tj", x[:, :, cols], w).reshape(-1)
        rows.append(row)
    return np.concatenate(rows).astype(np.float32)


def combine(params, nu, partials):
    """(beta, eta, W) (M,), (M,), (M, T*nu) of every mode from G shard rows, float64."""
    T, M = int(params.T), int(params.n_modes)
    P1 = 2 + T * nu
    r = np.asarray(partials, np.float64).reshape(-1, M, P1)
    lam = f32(params.lambda_)
    beta, eta, W = np.full(M, np.inf), np.zeros(M), np.zeros((M, T * nu))
    for m in range(M):
        ok = r[:, m, 1] > 0
        if not ok.any():
            continue
        b = r[ok, m, 0].min()
        s = np.where(ok, np.exp(-(np.where(ok, r[:, m, 0], b) - b) / lam), 0.0)
        beta[m], eta[m], W[m] = b, (s * r[:, m, 1]).sum(), s @ r[:, m, 2:]
    return beta, eta, W


def own_steps(params, U, eta, W):
    """d_m: W_m / eta_m (SIMPLE) or 0.02 U_m + 0.98 W_m / eta_m - U_m (MEAN); 0 where eta_m = 0."""
    M = U.shape[0]
    Uf = U.reshape(M, -1)
    d = np.zeros_like(Uf)
    for m in range(M):
        if eta[m] > 0:
            wm = W[m] / eta[m]
            s = f32(params.step_size_mean)
            d[m] = wm if params.mode == MODE_SIMPLE else (1.0 - s) * Uf[m] + s * wm - Uf[m]
    return d


def free_energy(params, beta, eta):
    """F_m = beta_m - lambda ln(eta_m / Kc), +inf where eta_m = 0."""
    lam, Kc = f32(params.lambda_), int(params.mode_samples)
    with np.errstate(divide="ignore"):
        return np.where(eta > 0, beta - lam * np.log(np.where(eta > 0, eta, 1.0) / Kc), np.inf)


def distances(U, sinv):
    """D[i][j] = sum_t (U_i,t - U_j,t)^T Sigma^-1 (U_i,t - U_j,t)."""
    dU = U[:, None] - U[None, :]
    return np.einsum("ijta,ab,ijtb->ij", dU, sinv, dU)


def bandwidth(D):
    """h = lower median of {D_ij : i < j} / ln(M + 1)."""
    M = D.shape[0]
    v = np.sort(D[np.triu_indices(M, 1)])
    return v[(v.size - 1) // 2] / np.log(M + 1)


def couple(U, d, sinv, h=None):
    """The Stein-variational step: U_i + (sum_j k_ij d_j + (2/h) sum_j k_ij (U_i - U_j)) / sum_j k_ij with k_ij = exp(-D_ij / h);
    k = 1 and no repulsion when h is 0 or not finite.  U (M, T, nu), d (M, T*nu); returns (M, T*nu) and h."""
    M = U.shape[0]
    Uf = U.reshape(M, -1)
    if h is None:
        h = bandwidth(distances(U, sinv))
    if h > 0 and np.isfinite(h):
        k = np.exp(-distances(U, sinv) / h)
        rep = (2.0 / h) * (k.sum(1)[:, None] * Uf - k @ Uf)
    else:
        k, rep = np.ones((M, M)), 0.0
    return Uf + (k @ d + rep) / k.sum(1)[:, None], h


def savgol(u, T, nu):
    """Savitzky-Golay window 9, order 2, 'interp' edges of one (T*nu,) sequence, float64."""
    u = u.reshape(T, nu)
    out = np.empty_like(u)
    for t in range(T):
        if t < 4:
            out[t] = SG_EDGE[t] @ u[:9]
        elif t >= T - 4:
            out[t] = SG_EDGE[T - 1 - t] @ u[::-1][:9]
        else:
            out[t] = SG_MID @ u[t - 4:t + 5]
    return out.reshape(-1)


def select(F, p, margin):
    """The executed mode: a* = argmin F (lowest index on ties); keep p while F_p <= F_a* + margin; all F infinite keeps p."""
    a = int(np.argmin(F))
    if not np.isfinite(F[a]):
        return int(p)
    return int(p) if F[int(p)] <= F[a] + margin else a


def finalize(params, nu, partials, U, state, h=None):
    """K4: (U_new (M, T, nu) float32, action (nu,), stats (2,), state) from G shard rows, U (M, T, nu) and the mode state."""
    T, M = int(params.T), int(params.n_modes)
    U = np.asarray(U, np.float32).astype(np.float64).reshape(M, T, nu)
    beta, eta, W = combine(params, nu, partials)
    d = own_steps(params, U, eta, W)
    F = free_energy(params, beta, eta)
    sinv = np.array(params.sigma_inv[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu)
    Un, _ = couple(U, d, sinv, h)
    lo = np.tile(np.array(params.u_min[:nu], np.float32), T).astype(np.float64)
    hi = np.tile(np.array(params.u_max[:nu], np.float32), T).astype(np.float64)
    out = np.stack([np.clip(savgol(Un[m], T, nu) if params.filter_u else Un[m], lo, hi) for m in range(M)]).astype(np.float32)
    state = np.asarray(state, np.float32)
    p = select(F, int(state[0]), f32(params.mode_margin))
    st = np.concatenate([[p], F, out[p]]).astype(np.float32)
    return out.reshape(M, T, nu), out[p, :nu].copy(), np.array([beta[p], eta[p]], np.float32), st


def shift(params, nu, U):
    """Every mode shifts by one step; u_init is appended."""
    U = np.asarray(U, np.float32).copy()
    U[:, :-1] = U[:, 1:]
    U[:, -1] = np.array(params.u_init[:nu], np.float32)
    return U


class ModesOracleBackend(co.ColoredOracleBackend):
    """The colored oracle backend with the multi-modal K1, K3, K4 and shift of a parameter block with n_modes > 1."""

    def _M(self):
        return int(self.params.n_modes) if self.params is not None and self.params.n_modes > 1 else 1

    def _Um(self, U):
        return U.reshape(self._M(), self.params.T, self.model.nu)

    def sample(self, seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr=None):
        if self._M() == 1:
            return super().sample(seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr)
        sample(lambda Um, a, n: super(ModesOracleBackend, self).sample(seed, plan_idx, k_offset, k_total, Um, prior_row, a, n, plan_ctr),
               self.params, self._Um(U), k_offset, self.params.K, [actions, noise])

    def sample_colored(self, seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr=None):
        if self._M() == 1:
            return super().sample_colored(seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr)
        sample(lambda Um, a, n: super(ModesOracleBackend, self).sample_colored(seed, plan_idx, k_offset, k_total, Um, prior_row, Lt, a, n, plan_ctr),
               self.params, self._Um(U), k_offset, self.params.K, [actions, noise])

    def sample_library(self, k_offset, k_total, U, prior_row, Z, actions, noise):
        if self._M() == 1:
            return super().sample_library(k_offset, k_total, U, prior_row, Z, actions, noise)
        sample(lambda Um, a, n: super(ModesOracleBackend, self).sample_library(k_offset, k_total, Um, prior_row, Z, a, n),
               self.params, self._Um(U), k_offset, self.params.K, [actions, noise])

    def reduce(self, cost, x, U, partial):
        if self._M() == 1:
            return super().reduce(cost, x, U, partial)
        partial.copy_(torch.from_numpy(reduce(self.params, self.model.nu, _np(cost.contiguous()), _np(x), _np(U))))

    def finalize(self, partials, G, U, action_out, stats):
        if self._M() == 1:
            return super().finalize(partials, G, U, action_out, stats)
        Un, act, st, state = finalize(self.params, self.model.nu, _np(partials.contiguous())[:G], _np(U), _np(self.dist))
        U.copy_(torch.from_numpy(Un).reshape(U.shape))
        action_out.copy_(torch.from_numpy(act))
        if stats is not None:
            stats.copy_(torch.from_numpy(st))
        self.dist.copy_(torch.from_numpy(state))

    def shift(self, U, plan_ctr=None):
        if self._M() == 1:
            return super().shift(U, plan_ctr)
        U.copy_(torch.from_numpy(shift(self.params, self.model.nu, _np(U))))
        if plan_ctr is not None:
            plan_ctr += 1
