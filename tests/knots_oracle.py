"""CPU reference of spline MPPI (``control_knots`` / ``spline_degree``, DESIGN.md section 2) for the tests.

The basis B[T][P] and the shift map come from ``blob.spline_basis`` (checked against scipy in test_oracle_knots.py).  K1 is the white Philox
draw of the fixed-distribution oracle with the knot p in the t slot, coloured by L0 in float64, clamped (the null row takes clamp(0)), and
the actions are clamp(B theta~) (the clamp only absorbs the rounding of float32 weights).  K3 scores S_k = sum_t gamma^t c[t][k] + (SIMPLE mode) lambda sum_p theta_p^T Sigma^-1 x_p,k over the P knot rows
and forms the row (beta, eta, W[P*nu]).  K4 is the plain update of theta, U_exec = B theta, action = theta_0; the shift applies the shift
map (rows without a successor take u_init).  ``KnotsOracleBackend`` puts it behind the backend interface, so the CPU suite can drive the
planner end to end.
"""
import copy

import numpy as np
import torch

import anneal_oracle as ao
import colored_oracle as co
from mppi_isaac_b200.backend import spline_table_floats
from mppi_isaac_b200.model.blob import MODE_SIMPLE, spline_basis
from oracle.backend import _np


def knot_params(params):
    """A copy of the block with T := P: the white draws of the knots are the fixed-Sigma draws of a P-step horizon."""
    q = copy.copy(params)
    q.T = int(params.control_knots)
    return q


def sample(model, params, seed, plan, theta, k_offset, k_total):
    """(actions [T][nu][K], xk [P][nu][K], theta~ [P][nu][K]) float64 of spline K1."""
    T, P, d, nu = int(params.T), int(params.control_knots), int(params.spline_degree), int(model.nu)
    z = co.white(model, knot_params(params), seed, plan, k_offset, k_total).astype(np.float64)
    L = np.array(params.sigma_chol[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu)
    th = np.asarray(theta, np.float32).astype(np.float64).reshape(P, nu)
    a = th[:, :, None] + np.einsum("ji,pik->pjk", L, z)
    kg = int(k_offset) + np.arange(a.shape[-1])
    if params.sample_null_action:
        a[:, :, kg == k_total - 1] = 0.0
    lo = np.array(params.u_min[:nu], np.float32).astype(np.float64)[None, :, None]
    hi = np.array(params.u_max[:nu], np.float32).astype(np.float64)[None, :, None]
    a = np.minimum(np.maximum(a, lo), hi)
    B, _, _ = spline_basis(T, P, d)
    xk = a if params.mode != MODE_SIMPLE else a - th[:, :, None]
    return np.minimum(np.maximum(np.einsum("tp,pjk->tjk", B, a), lo), hi), xk, a


def row(params, nu, cost, xk, theta):
    """The shard row (beta, eta, W[P*nu]) in float64."""
    T, P = int(params.T), int(params.control_knots)
    c = np.asarray(cost, np.float64).reshape(T, -1)
    K = c.shape[1]
    S = ((float(np.float32(params.gamma)) ** np.arange(T))[:, None] * c).sum(0)
    lam = float(np.float32(params.lambda_))
    x = np.asarray(xk, np.float64).reshape(P, nu, K)
    if params.mode == MODE_SIMPLE:
        Sinv = np.array(params.sigma_inv[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu)
        S = S + lam * np.einsum("pj,ij,pik->k", np.asarray(theta, np.float64).reshape(P, nu), Sinv, x)
    b = S.min()
    w = np.exp(-(S - b) / lam)
    return np.concatenate([[b, w.sum()], (x * w).sum(-1).reshape(-1)])


def finalize(params, nu, rows, theta):
    """(theta', U_exec [T][nu], action [nu]) of K4 from the G rows, in float64."""
    T, P, d = int(params.T), int(params.control_knots), int(params.spline_degree)
    rows = np.atleast_2d(np.asarray(rows, np.float64))
    lam = float(np.float32(params.lambda_))
    b = rows[:, 0].min()
    sc = np.exp(-(rows[:, 0] - b) / lam)
    e = (sc * rows[:, 1]).sum()
    W = (sc[:, None] * rows[:, 2:2 + P * nu]).sum(0).reshape(P, nu) / e
    th = np.asarray(theta, np.float64).reshape(P, nu)
    if params.mode == MODE_SIMPLE:
        th2 = th + W
    else:
        a = float(np.float32(params.step_size_mean))
        th2 = (1.0 - a) * th + a * W
    B, _, _ = spline_basis(T, P, d)
    return th2, B @ th2, th2[0]


def shift(params, nu, theta):
    """theta' of the shift: row p = sum_q N_q(xi_p + 1) theta_q, or u_init where xi_p + 1 > T - 1."""
    T, P, d = int(params.T), int(params.control_knots), int(params.spline_degree)
    _, Sm, _ = spline_basis(T, P, d)
    th = np.asarray(theta, np.float64).reshape(P, nu)
    out = np.empty_like(th)
    for p in range(P):
        out[p] = np.array(params.u_init[:nu], np.float32) if np.isnan(Sm[p]).any() else Sm[p] @ th
    return out


class KnotsOracleBackend(ao.AnnealOracleBackend):
    """The oracle backend with spline MPPI's K1, K3, K4 and shift while the block has control_knots > 0, each in float64 rounded once to
    float32, and the library's table refusals; every other block runs the parent's kernels."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.spline = None

    def _P(self):
        return int(self.params.control_knots) if self.params is not None else 0

    def set_spline(self, table):
        if table is not None:
            P, d = self._P(), int(self.params.spline_degree)
            if P == 0 or table.numel() != spline_table_floats(self.params.T, P, d, self.model.nu):
                raise RuntimeError("mppib_set_spline: the table does not fit the parameter block")
        self.spline = None if table is None else (table, int(self.params.T), self._P(), int(self.params.spline_degree), int(self.model.nu))

    def _table(self, who):
        if self._P() == 0:
            return None
        key = (int(self.params.T), self._P(), int(self.params.spline_degree), int(self.model.nu))
        if self.spline is None or self.spline[1:] != key:
            raise RuntimeError(f"{who}: control_knots = {self._P()} needs a spline table registered for (T, P, d, nu) = {key}")
        return self.spline[0]

    def sample(self, seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr=None):
        if self._P():
            raise RuntimeError("mppib_sample: control_knots > 0 samples through mppib_sample_spline")
        return super().sample(seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr)

    def sample_spline(self, seed, plan_idx, k_offset, k_total, U, actions, xk, plan_ctr=None):
        self._table("mppib_sample_spline")
        plan = plan_idx + (int(plan_ctr[0]) if plan_ctr is not None else 0)
        a, x, _ = sample(self.model, self.params, seed, plan, _np(U), k_offset, k_total)
        actions.copy_(torch.from_numpy(a.astype(np.float32)))
        xk.copy_(torch.from_numpy(x.astype(np.float32)))

    def reduce(self, cost, x, U, partial):
        if self._table("mppib_reduce") is None:
            return super().reduce(cost, x, U, partial)
        partial.copy_(torch.from_numpy(row(self.params, self.model.nu, _np(cost.contiguous()), _np(x), _np(U)).astype(np.float32)))

    def finalize(self, partials, G, U, action_out, stats):
        table = self._table("mppib_finalize")
        if table is None:
            return super().finalize(partials, G, U, action_out, stats)
        nu, T = int(self.model.nu), int(self.params.T)
        rows = _np(partials.contiguous())[:G].astype(np.float64)
        th, ue, a = finalize(self.params, nu, rows, _np(U))
        U.copy_(torch.from_numpy(th.astype(np.float32)))
        action_out.copy_(torch.from_numpy(a.astype(np.float32)))
        table[-T * nu:].copy_(torch.from_numpy(ue.astype(np.float32).reshape(-1)))
        if stats is not None:
            lam = float(np.float32(self.params.lambda_))
            b = rows[:, 0].min()
            stats.copy_(torch.tensor([b, (np.exp(-(rows[:, 0] - b) / lam) * rows[:, 1]).sum()], dtype=torch.float32))

    def shift(self, U, plan_ctr=None):
        if self._table("mppib_shift") is None:
            return super().shift(U, plan_ctr)
        U.copy_(torch.from_numpy(shift(self.params, self.model.nu, _np(U)).astype(np.float32)))
        if plan_ctr is not None:
            plan_ctr += 1
