"""CPU reference of risk-aware MPPI (``n_worlds`` / ``cvar_alpha``, DESIGN.md section 2) for the tests.

Global rollout kg = c R + r runs control sample c in world r.  K1 is the fixed-distribution (or adaptive, colored, Halton) draw of the
Kc = K_total / R control samples, repeated R times along k.  K2 keys the per-rollout randomisation of sample kg by its world r: the
oracle rollout of sample kg is the oracle's own rollout of a one-sample shard at k_offset = r.  K3 scores every sample in float64,
sets a non-finite score to +inf, and scores control c by rho_c = the mean of the m largest scores of its R rollouts; the shard row is
the row of a Kc-sample MPPI over the rho_c with x taken from the group's first rollout.  K4 is unchanged.  ``RiskOracleBackend``
puts it behind the backend interface, so the CPU suite can drive the planner end to end.
"""
import copy
import ctypes as C

import numpy as np
import torch

import adaptive_full_oracle as afo
import colored_oracle as co
from mppi_isaac_b200.model.blob import MODE_SIMPLE
from oracle import oracle as orc
from oracle.backend import _np


def rho(S, R, m):
    """(Kc,) float64 CVaR scores of the groups of R consecutive entries of S: +inf for a non-finite entry, then the mean of the m
    largest of the group (so a group with an invalid world scores +inf)."""
    S = np.where(np.isfinite(S), np.asarray(S, np.float64), np.inf).reshape(-1, R)
    top = -np.sort(-S, axis=1)[:, :m]
    with np.errstate(invalid="ignore"):
        return top.sum(1) / m


def rho_f32(S, R, m):
    """rho in float32 exactly as K3 forms it: the sorted group summed left to right in float32, one float32 division."""
    S = np.where(np.isfinite(S), np.asarray(S, np.float32), np.float32(np.inf)).reshape(-1, R)
    top = -np.sort(-S, axis=1)[:, :m]
    acc = top[:, 0].copy()
    for i in range(1, m):
        acc = (acc + top[:, i]).astype(np.float32)
    return (acc / np.float32(m)).astype(np.float32)


def scores(params, nu, cost, x, U, dist=None):
    """S_k in float64: sum_t gamma^t c[t][k] (+ lambda U^T Sigma^-1 x_k in SIMPLE mode, with the live lambda / Sigma^-1 of `dist`)."""
    T = params.T
    c = np.asarray(cost, np.float64).reshape(T, -1)
    K = c.shape[1]
    S = ((float(np.float32(params.gamma)) ** np.arange(T))[:, None] * c).sum(0)
    lam = float(np.float32(params.lambda_))
    Sinv = np.array(params.sigma_inv[:nu * nu], np.float32).reshape(nu, nu).astype(np.float64)
    if dist is not None:
        d = np.asarray(dist, np.float64)
        lam = d[0]
        if params.update_cov and params.cov_full:
            Sinv = afo.unpack(d, nu)[3]
        elif params.update_cov:
            Sinv = np.diag(1.0 / d[1:1 + nu].astype(np.float32).astype(np.float64))
    if params.mode == MODE_SIMPLE:
        Uf = np.asarray(U, np.float32).astype(np.float64).reshape(T, nu)
        S = S + lam * np.einsum("tj,ij,tik->k", Uf, Sinv, np.asarray(x, np.float64).reshape(T, nu, K))
    return S, lam


def reduce(params, nu, cost, x, U, dist=None):
    """The control-level shard row in float64, rounded to float32: (beta, eta, W) over rho_c with w_c = exp(-(rho_c - beta)/lambda)
    and x of the group's first rollout, + M2 (update_cov, diagonal) or the packed C (cov_full) when a distribution is registered."""
    T, R, m = params.T, int(params.n_worlds), int(params.risk_tail)
    S, lam = scores(params, nu, cost, x, U, dist)
    r = rho(S, R, m)
    ok = np.isfinite(r)
    beta = r[ok].min() if ok.any() else np.inf
    w = np.where(ok, np.exp(-(np.where(ok, r, beta) - beta) / lam), 0.0)
    xc = np.asarray(x, np.float64).reshape(T, nu, -1)[:, :, ::R]
    row = [np.array([beta, w.sum()]), np.einsum("tjc,c->tj", xc, w).reshape(-1)]
    if dist is not None and params.update_cov:
        cen = 0.0 if params.mode == MODE_SIMPLE else np.asarray(U, np.float32).astype(np.float64).reshape(T, nu)[:, :, None]
        dx = xc - cen
        if params.cov_full:
            row.append(afo.tril_pack(np.einsum("tic,tjc,c->ij", dx, dx, w)))
        else:
            row.append(np.einsum("tjc,c->tj", dx * dx, w).reshape(-1))
    return np.concatenate(row).astype(np.float32)


def control_params(params):
    """The parameter block of the Kc = K / R control samples a risk-mode shard holds (risk mode off)."""
    p = copy.deepcopy(params)
    p.K, p.n_worlds, p.risk_tail = params.K // params.n_worlds, 0, 0
    return p


class RiskOracleBackend(co.ColoredOracleBackend):
    """The colored / adaptive oracle backend with the risk-aware K1, K2 and K3 of a parameter block with n_worlds > 1."""

    def _R(self):
        return int(self.params.n_worlds) if self.params is not None and self.params.n_worlds > 1 else 1

    def _grouped(self, call, k_offset, k_total, outs, ins=()):
        """Run `call(k_offset_c, k_total_c, *ins_c, *outs_c)` on the control samples, then repeat every output R times along k."""
        R = self._R()
        full, self.params = self.params, control_params(self.params)
        try:
            oc = [None if o is None else torch.zeros(o.shape[:-1] + (o.shape[-1] // R,), dtype=o.dtype) for o in outs]
            call(k_offset // R, k_total // R, *[t[..., ::R].contiguous() for t in ins], *oc)
        finally:
            self.params = full
        for o, c in zip(outs, oc):
            if o is not None:
                o.copy_(torch.repeat_interleave(c, R, dim=-1))

    def sample(self, seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr=None):
        if self._R() == 1:
            return super().sample(seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr)
        self._grouped(lambda ko, kt, a, n: super(RiskOracleBackend, self).sample(seed, plan_idx, ko, kt, U, prior_row, a, n, plan_ctr),
                      k_offset, k_total, [actions, noise])

    def sample_colored(self, seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr=None):
        if self._R() == 1:
            return super().sample_colored(seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr)
        self._grouped(lambda ko, kt, a, n: super(RiskOracleBackend, self).sample_colored(seed, plan_idx, ko, kt, U, prior_row, Lt, a, n, plan_ctr),
                      k_offset, k_total, [actions, noise])

    def noise_library(self, k_offset, k_total, halton_tab, B, n_knots, Z):
        if self._R() == 1:
            return super().noise_library(k_offset, k_total, halton_tab, B, n_knots, Z)
        self._grouped(lambda ko, kt, z: super(RiskOracleBackend, self).noise_library(ko, kt, halton_tab, B, n_knots, z), k_offset, k_total, [Z])

    def sample_library(self, k_offset, k_total, U, prior_row, Z, actions, noise):
        if self._R() == 1:
            return super().sample_library(k_offset, k_total, U, prior_row, Z, actions, noise)
        self._grouped(lambda ko, kt, z, a, n: super(RiskOracleBackend, self).sample_library(ko, kt, U, prior_row, z, a, n),
                      k_offset, k_total, [actions, noise], ins=[Z])

    def rollout(self, state0, state, actions, t0, nsteps, obs, act_t0=0, root0=None):
        R = self._R()
        if R == 1:
            return super().rollout(state0, state, actions, t0, nsteps, obs, act_t0, root0)
        T, K, nu = self.params.T, self.params.K, self.model.nu
        src = _np(actions).reshape(-1, nu, K)
        a = np.zeros((T, nu, K), np.float32)
        a[act_t0:act_t0 + src.shape[0]] = src
        st, o = _np(state), _np(obs)
        s0 = None if state0 is None else np.ascontiguousarray(_np(state0), np.float32)
        r0 = None if root0 is None else np.ascontiguousarray(_np(root0), np.float32)
        f = lambda v: None if v is None else v.ctypes.data_as(C.POINTER(C.c_float))
        p1 = copy.deepcopy(self.params)
        p1.K, p1.n_worlds, p1.risk_tail = 1, 0, 0
        for k in range(K):
            p1.k_offset = (int(self.params.k_offset) + k) % R                 # the world of global rollout k_offset + k
            ak = np.ascontiguousarray(a[:, :, k:k + 1])
            sk = None if st is None else np.ascontiguousarray(st[:, k:k + 1])
            ok = None if o is None else np.zeros(o.shape[:-1] + (1,), np.float32)
            orc.lib().oracle_rollout(C.byref(self.model), C.byref(p1), f(s0), f(r0), f(sk), f(ak), C.c_int32(t0), C.c_int32(nsteps), f(ok),
                                     C.c_int32(int(self.use_double)), C.c_int32(1))
            if sk is not None:
                st[:, k] = sk[:, 0]
            if ok is not None:
                o[..., k] = ok[..., 0]

    def reduce(self, cost, x, U, partial):
        if self._R() == 1:
            return super().reduce(cost, x, U, partial)
        d = _np(self.dist) if self.dist is not None else None
        partial.copy_(torch.from_numpy(reduce(self.params, self.model.nu, _np(cost.contiguous()), _np(x), _np(U), d)))
