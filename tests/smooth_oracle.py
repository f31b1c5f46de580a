"""CPU reference of Smooth MPPI (``mppi_mode: smooth``, DESIGN.md section 2) for the tests.

Float64 NumPy restatement of the smooth kernels.  K1 colours the white Philox draws of the fixed-distribution oracle by L0, clamps
the derivative v to [du_min, du_max] and integrates it from the last executed action a_prev, clamping every action to [u_min, u_max];
the noise is the derivative actually applied minus U.  K3 scores S_k = sum_t c + lambda U^T Sigma^-1 x + omega dt^2 sum_r (U_r + x_r)^2
and forms SIMPLE's shard row.  K4 merges the rows, moves the derivative mean, clamps it and integrates it into the planned actions A.
The shift moves U by one step.  ``SmoothOracleBackend`` puts it behind the backend interface, so the CPU suite can drive the planner end
to end.
"""
import numpy as np
import torch

import colored_oracle as co
from mppi_isaac_b200.model.blob import MODE_SMOOTH
from oracle.backend import OracleBackend, _np


def state_floats(T, nu):
    return nu + T * nu


def bounds(params, nu):
    """(u_min, u_max, du_min, du_max) float32 arrays of the parameter block."""
    f = lambda name: np.array([getattr(params, name)[j] for j in range(nu)], np.float32)
    return f("u_min"), f("u_max"), f("du_min"), f("du_max")


def make_state(params, nu, a_prev=None):
    """The state a planner starts from: a_prev = clamp(0, u_min, u_max) (or the given one), A = a_prev at every step."""
    lo, hi, _, _ = bounds(params, nu)
    a0 = np.minimum(np.maximum(np.zeros(nu, np.float32), lo), hi) if a_prev is None else np.asarray(a_prev, np.float32)
    return np.tile(a0, params.T + 1).astype(np.float32)


def unpack(state, T, nu):
    """(a_prev[nu], A[T][nu]) views of a smooth state."""
    s = np.asarray(state)
    return s[:nu], s[nu:nu + T * nu].reshape(T, nu)


def integrate(params, nu, v, a_prev):
    """a_t = clamp(a_{t-1} + dt v_t, u_min, u_max) from a_prev in float64, v (T, nu, ...) float64; returns (a, applied derivative):
    where the action clamp binds, the applied derivative is (a_t - a_{t-1}) / dt."""
    lo, hi, _, _ = bounds(params, nu)
    dt = float(np.float32(params.dt))
    ext = (slice(None),) + (None,) * (v.ndim - 2)
    lo, hi = lo.astype(np.float64)[ext], hi.astype(np.float64)[ext]
    a = np.broadcast_to(np.asarray(a_prev, np.float32).astype(np.float64)[ext], v.shape[1:]).copy()
    out, applied = np.empty_like(v), np.empty_like(v)
    for t in range(v.shape[0]):
        ah = a + dt * v[t]
        an = np.minimum(np.maximum(ah, lo), hi)
        applied[t] = np.where(an != ah, (an - a) / dt, v[t])
        out[t] = an
        a = an
    return out, applied


def sample(params, nu, U, z, state, k_offset, k_total):
    """(actions, noise) [T][nu][K] float32 of the smooth K1 from the white draws z: v = clamp(U + L0 z, du_min, du_max) (0 on the null
    row), the actions integrated from a_prev, noise = applied derivative - U."""
    T, K = params.T, np.asarray(z).shape[-1]
    L = np.array(params.sigma_chol[:nu * nu], np.float32).reshape(nu, nu).astype(np.float64)
    n = np.einsum("ji,tik->tjk", L, np.asarray(z, np.float64), optimize=True)
    Uf = np.asarray(U, np.float32).reshape(T, nu).astype(np.float64)
    _, _, dlo, dhi = bounds(params, nu)
    v = np.minimum(np.maximum(Uf[:, :, None] + n, dlo.astype(np.float64)[None, :, None]), dhi.astype(np.float64)[None, :, None])
    kg = k_offset + np.arange(K)
    if params.sample_null_action:
        v[:, :, kg == k_total - 1] = 0.0
    a, applied = integrate(params, nu, v, unpack(state, T, nu)[0])
    return a.astype(np.float32), (applied - Uf[:, :, None]).astype(np.float32)


def scores(params, nu, cost, x, U):
    """S_k in float64: sum_t c[t][k] + lambda U^T Sigma^-1 x_k + omega dt^2 sum_r (U_r + x_rk)^2 (gamma = 1)."""
    T = params.T
    c = np.asarray(cost, np.float64).reshape(T, -1)
    xr = np.asarray(x, np.float64).reshape(T * nu, -1)
    Uf = np.asarray(U, np.float32).astype(np.float64).reshape(T, nu)
    Sinv = np.array(params.sigma_inv[:nu * nu], np.float32).reshape(nu, nu).astype(np.float64)
    g = float(np.float32(params.lambda_)) * (Uf @ Sinv.T).reshape(-1)
    w = float(np.float32(params.smooth_weight)) * float(np.float32(params.dt)) ** 2
    return c.sum(0) + g @ xr + w * ((Uf.reshape(-1, 1) + xr) ** 2).sum(0)


def reduce(params, nu, cost, x, U):
    """SIMPLE's shard row (beta, eta, W[T*nu]) of the smooth S, float64 rounded to float32; w_k = 0 for a non-finite S_k."""
    lam = float(np.float32(params.lambda_))
    S = scores(params, nu, cost, x, U)
    ok = np.isfinite(S)
    beta = S[ok].min() if ok.any() else np.inf
    w = np.where(ok, np.exp(-(np.where(ok, S, beta) - beta) / lam), 0.0)
    W = np.asarray(x, np.float64).reshape(params.T * nu, -1) @ w
    return np.concatenate([[beta, w.sum()], W]).astype(np.float32)


def finalize(params, nu, rows, U, state):
    """K4: merge the rows, U' = U + W/eta (U with eta = 0), clamped to the derivative bounds, integrated from a_prev into A, U'
    projected where the action clamp bound; returns (U', action = A_0, stats, state with a_prev = A_0)."""
    T, NR = params.T, params.T * nu
    rows = np.asarray(rows, np.float32).reshape(-1, 2 + NR).astype(np.float64)
    lam = float(np.float32(params.lambda_))
    valid = rows[:, 1] > 0
    b = rows[valid, 0].min() if valid.any() else np.inf
    s = np.where(valid, np.exp(-(np.where(valid, rows[:, 0], b) - b) / lam), 0.0) if valid.any() else np.zeros(len(rows))
    eta = (s * rows[:, 1]).sum()
    W = (s[:, None] * rows[:, 2:]).sum(0)
    Uo = np.asarray(U, np.float32).reshape(NR).astype(np.float64)
    Un = Uo + (W / eta if eta > 0 else 0.0)
    _, _, dlo, dhi = bounds(params, nu)
    v = np.minimum(np.maximum(Un.reshape(T, nu), dlo.astype(np.float64)), dhi.astype(np.float64))
    st = np.asarray(state, np.float32).copy()
    A, applied = integrate(params, nu, v, unpack(st, T, nu)[0])
    st[nu:] = A.reshape(-1).astype(np.float32)
    st[:nu] = st[nu:2 * nu]
    return applied.astype(np.float32), st[:nu].copy(), np.array([b, eta], np.float32), st


def shift(params, nu, U):
    """U[t] <- U[t + 1], U[T - 1] <- u_init (a derivative: 0 holds the last action)."""
    Uf = np.asarray(U, np.float32).reshape(params.T, nu)
    return np.concatenate([Uf[1:], np.array([params.u_init[j] for j in range(nu)], np.float32)[None]])


class SmoothOracleBackend(OracleBackend):
    """The oracle backend with the smooth kernels and a registered smooth state (a CPU tensor, updated in place like the device
    buffer of the CUDA backend)."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.smooth = None

    def _on(self):
        return int(self.params.mode) == MODE_SMOOTH

    def set_smooth_state(self, state):
        self.smooth = state

    def sample_smooth(self, seed, plan_idx, k_offset, k_total, U, actions, noise, plan_ctr=None):
        plan = plan_idx + (int(plan_ctr[0]) if plan_ctr is not None else 0)
        z = co.white(self.model, self.params, seed, plan, k_offset, k_total)
        a, n = sample(self.params, self.model.nu, _np(U), z, _np(self.smooth), k_offset, k_total)
        actions.copy_(torch.from_numpy(a))
        if noise is not None:
            noise.copy_(torch.from_numpy(n))

    def reduce(self, cost, x, U, partial):
        if not self._on():
            return super().reduce(cost, x, U, partial)
        partial.copy_(torch.from_numpy(reduce(self.params, self.model.nu, _np(cost.contiguous()), _np(x), _np(U))))

    def finalize(self, partials, G, U, action_out, stats):
        if not self._on():
            return super().finalize(partials, G, U, action_out, stats)
        Un, act, st, s = finalize(self.params, self.model.nu, _np(partials.contiguous())[:G], _np(U), _np(self.smooth))
        U.copy_(torch.from_numpy(Un.reshape(U.shape)))
        action_out.copy_(torch.from_numpy(act))
        if stats is not None:
            stats.copy_(torch.from_numpy(st))
        self.smooth.copy_(torch.from_numpy(s))

    def shift(self, U, plan_ctr=None):
        if not self._on():
            return super().shift(U, plan_ctr)
        U.copy_(torch.from_numpy(shift(self.params, self.model.nu, _np(U))))
        if plan_ctr is not None:
            plan_ctr += 1
