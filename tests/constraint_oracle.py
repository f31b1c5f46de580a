"""CPU reference of constrained MPPI (``constraint_mode: feasible_first``, DESIGN.md section 2) for the tests.

K3 scores S_k as the plain oracle does (sum_t gamma^t c[t][k], + lambda sum_t U_t^T Sigma^-1 x_t,k in SIMPLE mode), forms the per-step
violations c = max(g, 0) (NaN stays NaN) and V_k = sum_t c[t][k]; a sample is valid when S_k and V_k are finite and feasible when also
V_k <= tol.  With a feasible sample the row weights the feasible samples by exp(-(S - b)/lambda), otherwise the valid ones by
exp(-(V - b)/lambda_c); it is (beta, eta, W[T*nu], n_feasible, min V).  K4 merges the G rows feasibility-first into one plain row and hands
it to the plain oracle's K4, whose update, Savitzky-Golay, clamp and action are unchanged.  Everything is float64; the float32 row stores
n_feasible as int32 bits, as the library does.  ``ConstraintOracleBackend`` puts it behind the checker backend's interface (on top of
the other modes' oracle backends), so the CPU suite drives the planner end to end.
"""
import numpy as np
import torch

import knots_oracle as ko
from mppi_isaac_b200.model.blob import MODE_SIMPLE
from oracle import oracle as orc
from oracle.backend import _np


def scores(params, nu, cost, x, U):
    """S_k of today's K3 in float64."""
    T = int(params.T)
    c = np.asarray(cost, np.float64).reshape(T, -1)
    S = ((float(np.float32(params.gamma)) ** np.arange(T))[:, None] * c).sum(0)
    if params.mode == MODE_SIMPLE:
        lam = float(np.float32(params.lambda_))
        Sinv = np.array(params.sigma_inv[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu)
        xx = np.asarray(x, np.float64).reshape(T, nu, -1)
        S = S + lam * np.einsum("tj,ij,tik->k", np.asarray(U, np.float64).reshape(T, nu), Sinv, xx)
    return S


def violations(g):
    """V_k = sum_t c[t][k], c = g where g > 0 and 0 where g <= 0 (NaN stays NaN)."""
    g = np.asarray(g, np.float64)
    with np.errstate(invalid="ignore"):
        c = np.where(g <= 0.0, 0.0, g)
    return c.sum(0)


def row(params, nu, cost, x, U, g):
    """The shard row (beta, eta, W[T*nu], n_feasible, min V) in float64 (n_feasible as a count)."""
    T = int(params.T)
    S = scores(params, nu, cost, x, U)
    V = violations(np.asarray(g, np.float64).reshape(T, -1))
    ok = np.isfinite(S) & np.isfinite(V)
    feas = ok & (V <= float(np.float32(params.constraint_tol)))
    xx = np.asarray(x, np.float64).reshape(T * nu, -1)
    out = np.zeros(4 + T * nu)
    out[0] = np.inf
    if feas.any():
        key, mask, lam = S, feas, float(np.float32(params.lambda_))
    else:
        key, mask, lam = V, ok, float(np.float32(params.constraint_lambda))
    if mask.any():
        b = key[mask].min()
        w = np.where(mask, np.exp(-(np.where(mask, key, b) - b) / lam), 0.0)
        out[0], out[1], out[2:2 + T * nu] = b, w.sum(), xx @ w
    out[-2] = feas.sum()
    out[-1] = V[ok].min() if ok.any() else np.inf
    return out


def merge(params, rows):
    """(beta, eta, W, n_feasible, min V) of G rows merged feasibility-first."""
    rows = np.atleast_2d(np.asarray(rows, np.float64))
    nf, n_all = rows[:, -2], rows[:, -2].sum()
    match = ((nf > 0) == (n_all > 0)) & (rows[:, 1] > 0)
    lam = float(np.float32(params.lambda_ if n_all > 0 else params.constraint_lambda))
    b = rows[match, 0].min() if match.any() else np.inf
    sc = np.where(match, np.exp(-(np.where(match, rows[:, 0], b) - b) / lam), 0.0)
    return b, (sc * rows[:, 1]).sum(), (sc[:, None] * rows[:, 2:-2]).sum(0), int(n_all), rows[:, -1].min()


def finalize(model, params, rows, U):
    """(U', action, stats, (n_feasible, min V)) of K4: the merged row through the plain oracle's K4."""
    b, e, W, n, vmin = merge(params, rows)
    plain = np.concatenate([[b, e], W]).astype(np.float32)
    Un, act, st = orc.finalize(model, params, plain[None], U)
    return Un, act, st, (n, vmin)


def to_f32(r):
    """The float32 row of the library: n_feasible as int32 bits."""
    out = np.asarray(r, np.float64).astype(np.float32)
    out[-2:-1].view(np.int32)[0] = int(r[-2])
    return out


def from_f32(rows):
    """float64 rows with n_feasible read back from its int32 bits."""
    rows = np.atleast_2d(np.asarray(rows, np.float32))
    out = rows.astype(np.float64)
    out[:, -2] = np.ascontiguousarray(rows[:, -2]).view(np.int32)
    return out


class ConstraintOracleBackend(ko.KnotsOracleBackend):
    """The checker backend with constrained MPPI's K3 and K4 while the block has constraint_mode = 1, in float64, and the library's
    refusals of the registration; every other block runs the parent's kernels."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.constraint = None

    def set_constraint(self, viol, cstate=None):
        if viol is not None:
            if not self.params.constraint_mode:
                raise RuntimeError("mppib_set_constraint: the parameter block has constraint_mode = 0")
            if viol.numel() != int(self.params.T) * int(self.params.K) or cstate is None or cstate.numel() != 2:
                raise RuntimeError("mppib_set_constraint: the buffers do not fit the parameter block")
        self.constraint = None if viol is None else (viol, cstate, int(self.params.T), int(self.params.K))

    def _registered(self, who):
        if not self.params.constraint_mode:
            if self.constraint is not None:
                raise RuntimeError(f"{who}: a constraint buffer is registered but constraint_mode is 0")
            return None
        if self.constraint is None or self.constraint[2:] != (int(self.params.T), int(self.params.K)):
            raise RuntimeError(f"{who}: constraint_mode needs a violation buffer registered for (T, K) = ({self.params.T}, {self.params.K})")
        return self.constraint

    def reduce(self, cost, x, U, partial):
        reg = self._registered("mppib_reduce")
        if reg is None:
            return super().reduce(cost, x, U, partial)
        r = row(self.params, int(self.model.nu), _np(cost.contiguous()), _np(x), _np(U), _np(reg[0]))
        partial.copy_(torch.from_numpy(to_f32(r)))

    def finalize(self, partials, G, U, action_out, stats):
        reg = self._registered("mppib_finalize")
        if reg is None:
            return super().finalize(partials, G, U, action_out, stats)
        Un, act, st, (n, vmin) = finalize(self.model, self.params, from_f32(_np(partials.contiguous())[:G]), _np(U))
        U.copy_(torch.from_numpy(Un))
        action_out.copy_(torch.from_numpy(act))
        if stats is not None:
            stats.copy_(torch.from_numpy(st))
        cs = np.array([0.0, vmin], np.float32)
        cs[0:1].view(np.int32)[0] = n
        reg[1].copy_(torch.from_numpy(cs))
