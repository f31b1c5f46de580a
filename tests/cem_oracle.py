"""CPU reference of cross-entropy planning (``mppi_mode: cem``, iCEM, DESIGN.md section 2) for the tests.

Float64 NumPy restatement of the four CEM kernels: K1 colours the white Philox draws of the fixed-distribution oracle over time by
L_b and per step by sigma, clamps them and writes the carried elites into rows K_total - 3 - e; the elite kernel scores every sample
with S_k = sum_t gamma^t c[t][k] and keeps the E smallest (S, global index) keys of its shard; K4 merges the shard rows, moves U and
sigma towards the elites' mean and standard deviation and stores the elites; the shift moves U by one step and resets sigma.
``CemOracleBackend`` puts it behind the backend interface, so the CPU suite can drive the planner end to end.
"""
import numpy as np
import torch
from scipy.signal import savgol_filter

import colored_oracle as co
from mppi_isaac_b200.model.blob import MODE_CEM
from oracle.backend import _np

NONE_INDEX = 0xFFFFFFFF


def row_floats(T, nu, E):
    return (2 * E + E * T * nu + 3) & ~3


def state_floats(T, nu, E):
    return 2 + E + T * nu + E * T * nu


def unpack(state, T, nu, E):
    """(carry offset, elites valid, S_elite[E], sigma[T][nu], elites[E][T][nu]) views of a CEM state."""
    s = np.asarray(state)
    n = T * nu
    return s[0], s[1], s[2:2 + E], s[2 + E:2 + E + n].reshape(T, nu), s[2 + E + n:2 + E + n + E * n].reshape(E, T, nu)


def make_state(sigma_diag, T, nu, E):
    """The state the planner starts from: sigma = sqrt(diag(Sigma)) at every step, no elites."""
    st = np.zeros(state_floats(T, nu, E), np.float32)
    st[2 + E:2 + E + T * nu] = np.tile(np.sqrt(np.asarray(sigma_diag, np.float64)), T).astype(np.float32)
    return st


def bounds(params, nu):
    lo = np.array([params.u_min[j] for j in range(nu)], np.float32)
    hi = np.array([params.u_max[j] for j in range(nu)], np.float32)
    return lo, hi


def sample(params, nu, U, z, Lt, state, k_offset, k_total, prior_row=None):
    """(actions, noise) [T][nu][K] float32 of the CEM K1 from the white draws z: a = clamp(U + sigma (.) (L_b z)) in float64, the
    null and prior rows, and the carried rows k_total - 3 - e (e < n_keep) = clamp(elites[e][t + off]) once the elites are valid."""
    T, K, E = params.T, np.asarray(z).shape[-1], params.n_elites
    off, valid, _, sig, el = unpack(np.asarray(state, np.float32), T, nu, E)
    w = np.einsum("ts,sik->tik", np.asarray(Lt, np.float32).astype(np.float64), np.asarray(z, np.float64), optimize=True)
    Uf = np.asarray(U, np.float32).reshape(T, nu)
    a = Uf.astype(np.float64)[:, :, None] + sig.astype(np.float64)[:, :, None] * w
    kg = k_offset + np.arange(K)
    if params.sample_null_action:
        a[:, :, kg == k_total - 1] = 0.0
    lo, hi = bounds(params, nu)
    a = np.minimum(np.maximum(a, lo.astype(np.float64)[None, :, None]), hi.astype(np.float64)[None, :, None]).astype(np.float32)
    if valid:
        o = int(off)
        for e in range(params.n_keep):
            col = k_total - 3 - e - k_offset
            if 0 <= col < K:
                for t in range(T - o):
                    a[t, :, col] = np.minimum(np.maximum(el[e, t + o], lo), hi)
    if prior_row is not None:
        a[:, :, kg == k_total - 2] = np.asarray(prior_row, np.float32).reshape(T, nu, 1)
    return a, a - Uf[:, :, None]


def scores(params, cost):
    """S_k = sum_t gamma^t c[t][k] in float64, gamma the float32 of the parameter block."""
    c = np.asarray(cost, np.float64).reshape(params.T, -1)
    return ((np.float64(np.float32(params.gamma)) ** np.arange(params.T))[:, None] * c).sum(0)


def select(S, index, E):
    """Positions of the E smallest (S, index) keys among the finite S, best first (fewer if fewer are finite)."""
    S = np.asarray(S, np.float64)
    ok = np.flatnonzero(np.isfinite(S))
    order = ok[np.lexsort((np.asarray(index)[ok], S[ok]))]
    return order[:E]


def elite_row(params, nu, cost, actions, k_offset, S=None):
    """The shard row of the elite kernel: (S, index bits)[E], actions[E][T][nu] of the shard's E best samples; missing entries
    (+inf, 0xFFFFFFFF, 0).  S defaults to ``scores``; a caller may pass the device's own float32 S to check selection alone."""
    T, E = params.T, params.n_elites
    a = np.asarray(actions, np.float32).reshape(T * nu, -1)
    K = a.shape[1]
    S = scores(params, cost) if S is None else np.asarray(S, np.float64)
    kg = k_offset + np.arange(K, dtype=np.int64)
    pick = select(S, kg, E)
    row = np.zeros(row_floats(T, nu, E), np.float32)
    head = row[:2 * E]
    head[0::2] = np.inf
    head[1::2] = np.array([NONE_INDEX], np.uint32).view(np.float32)[0]
    for e, k in enumerate(pick):
        head[2 * e] = np.float32(S[k])
        head[2 * e + 1] = np.array([kg[k]], np.uint32).view(np.float32)[0]
        row[2 * E + e * T * nu:2 * E + (e + 1) * T * nu] = a[:, k]
    return row


def merge(rows, E):
    """(g, e) of the global elites among G shard rows in the order of their sample ranges, best first: key (S, g, e)."""
    rows = np.asarray(rows, np.float32)
    G = rows.shape[0]
    S = rows[:, 0:2 * E:2].astype(np.float64)
    idx = rows[:, 1:2 * E:2].copy().view(np.uint32)
    g, e = np.meshgrid(np.arange(G), np.arange(E), indexing="ij")
    ok = np.isfinite(S) & (idx != NONE_INDEX)
    order = np.lexsort((e[ok], g[ok], S[ok]))[:E]
    return list(zip(g[ok][order], e[ok][order]))


def savgol_clamp(params, nu, U):
    lo, hi = bounds(params, nu)
    if not params.filter_u:
        return U
    return np.minimum(np.maximum(savgol_filter(U, 9, 2, axis=0, mode="interp"), lo.astype(np.float64)), hi.astype(np.float64))


def finalize(params, nu, rows, U, state):
    """K4: merge, then with E finite elites m, s (population std) over them in float64, U <- (1 - a) m + a U, sigma <- (1 - a) s
    + a sigma, elites and S stored, carry offset 0; otherwise U, sigma, the elites and the offset stay.  Then Savitzky-Golay (with
    filter_u) and clamp, first action; stats = (S_best, S_E).  Returns (U, action, stats, state)."""
    T, E, NR = params.T, params.n_elites, params.T * nu
    rows = np.asarray(rows, np.float32).reshape(-1, row_floats(T, nu, E))
    st = np.asarray(state, np.float32).copy()
    Uo = np.asarray(U, np.float32).reshape(T, nu).astype(np.float64)
    win = merge(rows, E)
    Sw = [float(rows[g, 2 * e]) for g, e in win]
    stats = np.array([Sw[0] if Sw else np.inf, Sw[E - 1] if len(win) == E else np.inf], np.float32)
    Un = Uo
    if len(win) == E:
        A = np.stack([rows[g, 2 * E + e * NR:2 * E + (e + 1) * NR] for g, e in win]).astype(np.float64).reshape(E, T, nu)
        m = A.mean(0)
        s = np.sqrt(((A - m) ** 2).mean(0))
        al = float(np.float32(params.elite_alpha))
        _, _, _, sig, el = unpack(st, T, nu, E)
        Un = (1 - al) * m + al * Uo
        sig[:] = ((1 - al) * s + al * sig.astype(np.float64)).astype(np.float32)
        el[:] = A.astype(np.float32)
        st[2:2 + E] = np.array(Sw, np.float32)
        st[0], st[1] = 0.0, 1.0
    Uf = savgol_clamp(params, nu, Un).astype(np.float32)
    return Uf, Uf[0].copy(), stats, st


def shift(params, nu, U, state):
    """U[t] <- U[t + 1], U[T - 1] <- u_init; sigma <- sigma0 = the diagonal of sigma_chol at every step; carry offset 1."""
    T, E = params.T, params.n_elites
    Uf = np.asarray(U, np.float32).reshape(T, nu)
    Un = np.concatenate([Uf[1:], np.array([params.u_init[j] for j in range(nu)], np.float32)[None]])
    st = np.asarray(state, np.float32).copy()
    _, _, _, sig, _ = unpack(st, T, nu, E)
    sig[:] = np.array([params.sigma_chol[j * nu + j] for j in range(nu)], np.float32)[None]
    st[0] = 1.0
    return Un, st


class CemOracleBackend(co.ColoredOracleBackend):
    """The colored oracle backend, which runs the CEM kernels when the parameter block has mode MODE_CEM."""

    def _cem(self):
        return int(self.params.mode) == MODE_CEM

    def sample_colored(self, seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr=None):
        if not self._cem():
            return super().sample_colored(seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr)
        plan = plan_idx + (int(plan_ctr[0]) if plan_ctr is not None else 0)
        z = co.white(self.model, self.params, seed, plan, k_offset, k_total)
        a, n = sample(self.params, self.model.nu, _np(U), z, _np(Lt), _np(self.dist), k_offset, k_total, _np(prior_row))
        actions.copy_(torch.from_numpy(a))
        if noise is not None:
            noise.copy_(torch.from_numpy(n))

    def reduce(self, cost, x, U, partial):
        if not self._cem():
            return super().reduce(cost, x, U, partial)
        partial.copy_(torch.from_numpy(elite_row(self.params, self.model.nu, _np(cost.contiguous()), _np(x), int(self.params.k_offset))))

    def finalize(self, partials, G, U, action_out, stats):
        if not self._cem():
            return super().finalize(partials, G, U, action_out, stats)
        Un, act, st, d = finalize(self.params, self.model.nu, _np(partials.contiguous()).reshape(G, -1), _np(U), _np(self.dist))
        U.copy_(torch.from_numpy(Un))
        action_out.copy_(torch.from_numpy(act))
        if stats is not None:
            stats.copy_(torch.from_numpy(st))
        self.dist.copy_(torch.from_numpy(d))

    def shift(self, U, plan_ctr=None):
        if not self._cem():
            return super().shift(U, plan_ctr)
        Un, st = shift(self.params, self.model.nu, _np(U), _np(self.dist))
        U.copy_(torch.from_numpy(Un))
        self.dist.copy_(torch.from_numpy(st))
        if plan_ctr is not None:
            plan_ctr += 1
