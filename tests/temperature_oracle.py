"""CPU reference of the ESS-targeted temperature (``lambda_mode: ess``, DESIGN.md section 2) for the tests.

A float64 restatement of the pass (per-sample C_k and q_k, the shifted sums of every grid temperature), of the combine over ranks and of
the rule.  ``TemperatureOracleBackend`` is the adaptive checker backend (``adaptive_oracle``) plus a registered temperature state: the
temperature of each plan is chosen here and written into dist[0], and the oracle's K3 / K4 then run with it substituted for lambda_.
``TemperatureFullOracleBackend`` composes it with ``cov_type: full`` in the same way.
"""
import numpy as np
import torch

import adaptive_full_oracle as adf
import adaptive_oracle as ada
from mppi_isaac_b200.model.blob import ESS_GRID, ESS_ROW_FLOATS, MODE_SIMPLE
from oracle.backend import _np


def sigma_inv(params, nu, dist):
    """(nu, nu) float64 Sigma^-1 of K3's control cost: the fixed one, diag(1/cov) with update_cov, the full one with cov_full."""
    if dist is not None and params.update_cov and params.cov_full:
        return adf.unpack(np.asarray(dist, np.float32), nu)[3].astype(np.float64)
    if dist is not None and params.update_cov:
        cov = np.asarray(dist, np.float32)[1:1 + nu]
        return np.diag((np.float32(1.0) / cov).astype(np.float64))
    return np.array(params.sigma_inv[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu)


def scores(params, nu, cost, x, U, dist=None):
    """(C_k, q_k) in float64: S_k(lambda) = C_k + lambda q_k is K3's S; q = 0 in MEAN mode."""
    T = int(params.T)
    cost = np.asarray(cost, np.float64).reshape(T, -1)
    C = (float(params.gamma) ** np.arange(T)) @ cost
    if params.mode != MODE_SIMPLE:
        return C, np.zeros_like(C)
    h = np.asarray(U, np.float64).reshape(T, nu) @ sigma_inv(params, nu, dist).T      # (Sigma^-1 U_t) per step
    q = h.reshape(-1) @ np.asarray(x, np.float64).reshape(T * nu, -1)
    return C, q


def shard_row(params, nu, cost, x, U, inv, dist=None):
    """(n_valid, m[65], s1[65], s2[65]) of one shard in float64; inv = the 1/lambda_j of the state."""
    C, q = scores(params, nu, cost, x, U, dist)
    with np.errstate(invalid="ignore", over="ignore"):
        ok = np.isfinite(C) & np.isfinite(q)
    inv = np.asarray(inv, np.float64)
    if not ok.any():
        return 0, np.full(ESS_GRID, np.inf), np.zeros(ESS_GRID), np.zeros(ESS_GRID)
    a = C[ok][None, :] * inv[:, None] + q[ok][None, :]
    m = a.min(1)
    e = np.exp(-(a - m[:, None]))
    return int(ok.sum()), m, e.sum(1), (e * e).sum(1)


def combine(rows):
    """(N, ESS[65]) of the shard rows of every rank."""
    N = sum(r[0] for r in rows)
    if N == 0:
        return 0, np.zeros(ESS_GRID)
    m = np.min([r[1] for r in rows], axis=0)
    s1 = sum(np.where(np.isfinite(r[1]), r[2] * np.exp(-(r[1] - m)), 0.0) for r in rows)
    s2 = sum(np.where(np.isfinite(r[1]), r[3] * np.exp(-2.0 * (r[1] - m)), 0.0) for r in rows)
    return N, s1 * s1 / s2


def rule(ess, N, rho, lam, prev):
    """The chosen temperature (float64) from the curve ESS_j over the grid lam_j; prev is kept when N = 0."""
    if N == 0:
        return float(prev)
    tau = rho * N
    hit = np.nonzero(np.asarray(ess) >= tau)[0]
    if hit.size == 0:
        return float(lam[-1])
    j = int(hit[0])
    if j == 0:
        return float(lam[0])
    theta = (np.log(tau) - np.log(ess[j - 1])) / (np.log(ess[j]) - np.log(ess[j - 1]))
    return float(lam[j - 1]) * 2.0 ** (theta / 4.0)


def ess_at(C, q, lam):
    """The Kish ESS of the softmax weights of S = C + lam q over the valid samples, in float64."""
    ok = np.isfinite(C) & np.isfinite(q)
    S = C[ok] + lam * q[ok]
    w = np.exp(-(S - S.min()) / lam)
    return w.sum() ** 2 / (w * w).sum()


def to_f32(row):
    """The device layout of a float64 row: (n_valid as int32 bits, (m_j, s1_j, s2_j)[65]) in float32."""
    n, m, s1, s2 = row
    out = np.empty(ESS_ROW_FLOATS, np.float32)
    out[0:1] = np.array([n], np.int32).view(np.float32)
    out[1:].reshape(ESS_GRID, 3)[:] = np.stack([m, s1, s2], 1)
    return out


def from_f32(r):
    r = np.asarray(r, np.float32)
    t = r[1:].reshape(ESS_GRID, 3).astype(np.float64)
    return int(r[0:1].view(np.int32)[0]), t[:, 0], t[:, 1], t[:, 2]


class TemperatureMixin:
    """The temperature entries of the backend interface over a registered state (a CPU tensor written in place like the device one)."""

    temp = None

    def set_temperature(self, state):
        self.temp = state

    def _grid(self):
        t = _np(self.temp)
        return t[:ESS_GRID].astype(np.float64), t[ESS_GRID:2 * ESS_GRID]

    def temperature(self, cost, x, U, row, solve=True):
        if self.temp is None or self.dist is None or not self.params.lambda_ess:
            raise RuntimeError("mppib_temperature: lambda_mode ess needs a distribution and a temperature state registered")
        _, inv = self._grid()
        r = shard_row(self.params, self.model.nu, _np(cost.contiguous()), None if x is None else _np(x), _np(U), inv, _np(self.dist))
        row.copy_(torch.from_numpy(to_f32(r)))
        if solve:
            self._solve([r])

    def temperature_solve(self, rows, G):
        self._solve([from_f32(_np(rows[g])) for g in range(G)])

    def _solve(self, rows):
        lam, _ = self._grid()
        N, ess = combine(rows)
        chosen = np.float32(rule(ess, N, float(np.float32(self.params.ess_target)), lam, self.dist[0].item()))
        self.dist[0] = float(chosen)
        t = self.temp
        t[2 * ESS_GRID:2 * ESS_GRID + 1] = torch.from_numpy(np.array([N], np.int32).view(np.float32))
        t[2 * ESS_GRID + 1] = float(chosen)
        t[2 * ESS_GRID + 2:] = torch.from_numpy(ess.astype(np.float32))

    def _require(self, who):
        if self.params.lambda_ess and (self.temp is None or self.dist is None):
            raise RuntimeError(f"{who}: lambda_mode ess needs a distribution and a temperature state registered")

    def reduce(self, cost, x, U, partial):
        self._require("mppib_reduce")
        return super().reduce(cost, x, U, partial)

    def finalize(self, partials, G, U, action_out, stats):
        self._require("mppib_finalize")
        return super().finalize(partials, G, U, action_out, stats)


class TemperatureOracleBackend(TemperatureMixin, ada.AdaptiveOracleBackend):
    """The adaptive checker backend with the temperature of every plan chosen by the rule (fixed or diagonal Sigma)."""


class TemperatureFullOracleBackend(TemperatureMixin, adf.AdaptiveFullOracleBackend):
    """The same over the full-covariance checker backend (update_cov with cov_type: full)."""
