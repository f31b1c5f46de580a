"""CPU reference of annealed MPPI (``anneal_iterations`` / ``anneal_iter_decay`` / ``anneal_horizon_decay``, DESIGN.md section 2) for the
tests.

The schedule is s[i][t] = c_i^i c_h^(T-1-t) and r = 1 / s^2, each from float64 rounded once to float32, in the buffer (counter, s[N][T],
r[N][T]); iteration i reads row min(counter, N - 1).  K1 is the white Philox draw of the fixed-distribution oracle, coloured over the
horizon (colored sampling) and over the controls in float64, scaled by s[i][t], clamped, with the null and prior rows; with n_worlds > 1
it is drawn per control sample and repeated R times along k.  K3 scores S_k = sum_t gamma^t c + lambda sum_t r[i][t] U_t^T Sigma^-1 x_t
(SIMPLE mode) in float64, then the row of plain MPPI or, with n_worlds > 1, of the CVaR scores.  K4 is the oracle's K4 followed by
counter += 1, the shift the oracle's shift followed by counter := 0.  ``AnnealOracleBackend`` puts it behind the backend interface, so the
CPU suite can drive the planner end to end.
"""
import numpy as np
import torch

import colored_oracle as co
import risk_oracle as ro
from mppi_isaac_b200.model.blob import MAX_ANNEAL, MODE_SIMPLE, anneal_schedule, mode_refusal
from oracle.backend import _np


def schedule(N, ci, ch, T):
    """(s, r) float32 (N, T): the float64 schedule, each rounded once."""
    s, r = anneal_schedule(N, ci, ch, T)
    return s.astype(np.float32), r.astype(np.float32)


def make_state(s, r, counter=0.0):
    """The buffer (counter, s[N][T], r[N][T]) as float32."""
    return np.concatenate([[counter], np.asarray(s, np.float32).reshape(-1), np.asarray(r, np.float32).reshape(-1)]).astype(np.float32)


def rows(state, N, T):
    """(s row, r row) float32 (T,) of the iteration the counter selects: min(counter, N - 1)."""
    st = np.asarray(state, np.float32)
    i = min(max(int(st[0]), 0), N - 1)
    return st[1 + i * T:1 + (i + 1) * T], st[1 + (N + i) * T:1 + (N + i + 1) * T]


def sample(model, params, seed, plan, U, k_offset, k_total, s_row, prior_row=None, Lt=None):
    """(actions, noise) [T][nu][K] float32 of annealed K1 in float64: w = L_b z (colored) or z, noise = s[t] (L0 w), a = clamp(U + noise)
    with the null row (global k_total - 1) and the prior row (k_total - 2), noise := a - U."""
    T, nu = int(params.T), int(model.nu)
    z = co.white(model, params, seed, plan, k_offset, k_total).astype(np.float64)
    if Lt is not None:
        z = np.einsum("ts,sik->tik", np.asarray(Lt, np.float32).astype(np.float64), z, optimize=True)
    L = np.array(params.sigma_chol[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu)
    n = np.einsum("ji,tik->tjk", L, z, optimize=True) * np.asarray(s_row, np.float32).astype(np.float64)[:, None, None]
    Uf = np.asarray(U, np.float32).reshape(T, nu)
    a = Uf.astype(np.float64)[:, :, None] + n
    kg = int(k_offset) + np.arange(a.shape[-1])
    if params.sample_null_action:
        a[:, :, kg == k_total - 1] = 0.0
    lo = np.array(params.u_min[:nu], np.float32).astype(np.float64)[None, :, None]
    hi = np.array(params.u_max[:nu], np.float32).astype(np.float64)[None, :, None]
    a = np.minimum(np.maximum(a, lo), hi).astype(np.float32)
    if prior_row is not None:
        a[:, :, kg == k_total - 2] = np.asarray(prior_row, np.float32).reshape(T, nu, 1)
    return a, a - Uf[:, :, None]


def scores(params, nu, cost, x, U, r_row):
    """S_k in float64: sum_t gamma^t c[t][k] + (SIMPLE mode) lambda sum_t r[t] U_t^T Sigma^-1 x_t,k."""
    T = int(params.T)
    c = np.asarray(cost, np.float64).reshape(T, -1)
    K = c.shape[1]
    S = ((float(np.float32(params.gamma)) ** np.arange(T))[:, None] * c).sum(0)
    lam = float(np.float32(params.lambda_))
    if params.mode == MODE_SIMPLE:
        Sinv = np.array(params.sigma_inv[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu)
        Uf = np.asarray(U, np.float32).astype(np.float64).reshape(T, nu) * np.asarray(r_row, np.float32).astype(np.float64)[:, None]
        S = S + lam * np.einsum("tj,ij,tik->k", Uf, Sinv, np.asarray(x, np.float64).reshape(T, nu, K))
    return S, lam


def reduce(params, nu, cost, x, U, r_row):
    """The shard row (beta, eta, W) in float64, rounded to float32; with n_worlds > 1 over the CVaR scores of the control samples."""
    T = int(params.T)
    S, lam = scores(params, nu, cost, x, U, r_row)
    xr = np.asarray(x, np.float64).reshape(T, nu, -1)
    R = int(params.n_worlds)
    if R > 1:
        S, xr = ro.rho(S, R, int(params.risk_tail)), xr[:, :, ::R]
    ok = np.isfinite(S)
    beta = S[ok].min() if ok.any() else np.inf
    w = np.where(ok, np.exp(-(np.where(ok, S, beta) - beta) / lam), 0.0)
    return np.concatenate([[beta, w.sum()], np.einsum("tjk,k->tj", xr, w).reshape(-1)]).astype(np.float32)


def refusal(params, nu):
    """The library's refusal of a parameter block while a schedule is registered, or None."""
    return mode_refusal(params, nu, anneal=True)


class AnnealOracleBackend(ro.RiskOracleBackend):
    """The colored / risk oracle backend with the annealed K1, K3, K4 and shift of a registered schedule, and the library's refusals."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.anneal, self.anneal_n, self.anneal_T = None, 0, 0

    def set_anneal(self, state, n_iterations=0):
        if state is None:
            self.anneal, self.anneal_n, self.anneal_T = None, 0, 0
            return
        if not 1 <= int(n_iterations) <= MAX_ANNEAL:
            raise RuntimeError(f"mppib_set_anneal: n_iterations = {n_iterations} out of range [1, {MAX_ANNEAL}]")
        if state.numel() != 1 + 2 * int(n_iterations) * int(self.params.T):
            raise RuntimeError("mppib_set_anneal: the buffer does not hold 1 + 2*N*T floats")
        why = refusal(self.params, self.model.nu)
        if why:
            raise RuntimeError(f"mppib_set_anneal: {why}")
        self.anneal, self.anneal_n, self.anneal_T = state, int(n_iterations), int(self.params.T)

    def _check(self, who):
        if self.anneal is None:
            return False
        if int(self.params.T) != self.anneal_T:
            raise RuntimeError(f"{who}: the annealing schedule was registered for T = {self.anneal_T}, the parameter block has T = {self.params.T}")
        why = refusal(self.params, self.model.nu)
        if why:
            raise RuntimeError(f"{who}: {why}")
        return True

    def _rows(self):
        return rows(_np(self.anneal), self.anneal_n, self.anneal_T)

    def _sample(self, seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr):
        def one(ko, kt, a_out, n_out):
            plan = plan_idx + (int(plan_ctr[0]) if plan_ctr is not None else 0)
            a, n = sample(self.model, self.params, seed, plan, _np(U), ko, kt, self._rows()[0], _np(prior_row), Lt)
            a_out.copy_(torch.from_numpy(a))
            if n_out is not None:
                n_out.copy_(torch.from_numpy(n))
        if self._R() > 1:
            self._grouped(one, k_offset, k_total, [actions, noise])
        else:
            one(k_offset, k_total, actions, noise)

    def sample(self, seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr=None):
        if not self._check("mppib_sample"):
            return super().sample(seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr)
        self._sample(seed, plan_idx, k_offset, k_total, U, prior_row, None, actions, noise, plan_ctr)

    def sample_colored(self, seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr=None):
        if not self._check("mppib_sample_colored"):
            return super().sample_colored(seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr)
        self._sample(seed, plan_idx, k_offset, k_total, U, prior_row, _np(Lt), actions, noise, plan_ctr)

    def noise_library(self, k_offset, k_total, halton_tab, B, n_knots, Z):
        if self.anneal is not None:
            raise RuntimeError("mppib_noise_library: annealed MPPI excludes the noise library")
        return super().noise_library(k_offset, k_total, halton_tab, B, n_knots, Z)

    def sample_library(self, k_offset, k_total, U, prior_row, Z, actions, noise):
        if self.anneal is not None:
            raise RuntimeError("mppib_sample_library: annealed MPPI excludes the noise library")
        return super().sample_library(k_offset, k_total, U, prior_row, Z, actions, noise)

    def reduce(self, cost, x, U, partial):
        if not self._check("mppib_reduce"):
            return super().reduce(cost, x, U, partial)
        partial.copy_(torch.from_numpy(reduce(self.params, self.model.nu, _np(cost.contiguous()), _np(x), _np(U), self._rows()[1])))

    def finalize(self, partials, G, U, action_out, stats):
        on = self._check("mppib_finalize")
        super().finalize(partials, G, U, action_out, stats)
        if on:
            self.anneal[0] += 1.0

    def shift(self, U, plan_ctr=None):
        on = self._check("mppib_shift")
        super().shift(U, plan_ctr)
        if on:
            self.anneal[0] = 0.0
