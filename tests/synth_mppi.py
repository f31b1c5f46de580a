"""Generated sampling / reduction / update cases at any accepted (T, nu, K), and the float32 error bounds of K3 that the tests gate on.

K1, K3, K4 and the shift read nothing of the model but ``nu``, so every case runs on the point robot's model with ``nu`` set and both
command maps of every joint pointing at input 0 (no dynamics run).  ``make_case`` builds the parameter block through ``make_params``
and, for the adaptive row kinds, the live distribution:

* ``W``  -- fixed Sigma (``sigma_chol`` / ``sigma_inv``), shard row ``[beta, eta, W[T*nu]]``;
* ``M2`` -- ``update_cov`` with a diagonal Sigma, ``dist = [lambda, cov[nu]]``, row ``+ M2[T*nu]``;
* ``C``  -- ``update_cov`` with ``cov_type: full``, ``dist = [lambda, Sigma, L, Sigma^-1]``, row ``+ C[nu(nu+1)/2]``.

``ws_layout`` restates the shared-memory plan of the warp-specialised K3 (``WsLayout`` and the ring-depth rule of
``launch_reduce_ws_t`` in ``csrc/reduce.cu``), so a case id can name the instantiation and the consumer-warp count that run.

The K3 gate (``k3_gate``) bounds the float32 error of the kernel per case instead of using a constant tolerance:
  dS_k <= eps * [(n/4 + 6 + 2 ln2 |log2 gamma| T) * sum_t |gamma^t c_tk| + (n/4 + nu + 6) * sum_r |x_rk| |lambda Sigma^-1|_r |U|]
(n = the terms of the four accumulation chains of phase A, the gamma^t and g = lambda Sigma^-1 U rounding folded in), which moves a
weight at most to exp(-(S_k - b -/+ (dS_k + db)) / lambda); the weighted sums then carry that spread per sample plus the rounding of
their own accumulation (``rho``, a few eps per merge step).  eps is float32's machine epsilon (twice the unit roundoff).
"""
import copy
import functools
import math
from dataclasses import dataclass

import numpy as np

from mppi_isaac_b200.model.blob import MODE_SIMPLE, OBS_DOF_STATE, OBS_LINK_STATE, make_params
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig

EPS = float(np.finfo(np.float32).eps)
NUM_SMS = 132                  # H100 SXM: the K just under / over one tile per SM and the ring-wrap K are sized for it
KINDS = ("W", "M2", "C")

# ---------------------------------------------------------------------------------------------------------------- K3 layout
WS_W, WS_NCONS, MAX_GRID, SMEM_CAP = 32, 7, 512, 224 * 1024


def row_floats(T, nu, kind):
    NR = T * nu
    return 2 + NR + (NR if kind == "M2" else nu * (nu + 1) // 2 if kind == "C" else 0)


def _ws_bytes(T, nu, nstage, kind):
    NR = T * nu
    P4 = (row_floats(T, nu, kind) + 3) & ~3
    ring, fold = nstage * (NR + T) * WS_W, MAX_GRID + 4 * P4
    g = max(ring, fold)
    if kind == "C":
        g = max(g, NR + 1 + 2 * NR + nu * (nu + 1) // 2 + 3 * nu * nu)
    gp = g + ((NR + 3) & ~3)
    wk = gp + ((T + 3) & ~3)
    misc = wk + 8 * WS_W + WS_NCONS * P4
    bar = ((misc + 8) * 4 + 15) & ~15
    return bar + 2 * 8 * nstage + 128


def ws_stages(T, nu, kind):
    ns = 8
    while ns > 1 and _ws_bytes(T, nu, ns, kind) > SMEM_CAP:
        ns -= 1
    return ns


def ws_layout(T, nu, kind):
    """(rows of W per lane, consumer warps, ring stages, rows per x TMA box) of the K3 launch, or None if the shape is refused."""
    NR = T * nu
    if NR > 512 or T > 256 or ws_stages(T, nu, "W") < 2 or ws_stages(T, nu, kind) < 2:
        return None
    ns = ws_stages(T, nu, kind)
    ncons = min(ns, WS_NCONS)
    xbox = min(NR, 256)
    while NR % xbox:
        xbox -= 1
    return (4 if NR <= 128 else 8 if NR <= 256 else 16), ncons, ncons * (ns // ncons), xbox


def wrap_K(T, nu, kind, sms=NUM_SMS):
    """A ragged K (multiple of 4) whose every CTA streams more than three full rings of tiles."""
    _, _, nstage, _ = ws_layout(T, nu, kind)
    return WS_W * sms * (3 * nstage + 1) - 12


# ---------------------------------------------------------------------------------------------------------------- cases
def corr_sigma(nu, scale=0.1, seed=3):
    """A symmetric positive-definite Sigma with real correlations, diagonal about `scale`."""
    A = np.random.default_rng(seed).normal(0, 1.0, (nu, nu))
    S = A @ A.T / nu + 0.3 * np.eye(nu)
    S = scale * S / np.mean(np.diag(S))
    return 0.5 * (S + S.T)


@functools.lru_cache(maxsize=1)
def _point_scene():
    from scenes import point_scene
    return point_scene()


def nu_model(nu):
    """The point robot's model driven through `nu` inputs; every command map points at input 0."""
    sc = _point_scene()
    m = copy.deepcopy(sc.model)
    m.nu = nu
    for i in range(m.nb):
        m.cmd_i0[i] = m.cmd_i1[i] = 0
    return m


@dataclass
class Case:
    model: object
    params: object
    T: int
    nu: int
    K: int
    kind: str
    sigma: np.ndarray                 # the live Sigma (float64)
    dist: np.ndarray = None           # float32 dist buffer of the adaptive kinds

    @property
    def simple(self):
        return self.params.mode == MODE_SIMPLE

    @property
    def lam(self):
        return float(self.dist[0]) if self.dist is not None else float(self.params.lambda_)

    def chol(self):
        """The float32 lower factor K1 colours with."""
        nu = self.nu
        if self.kind == "M2":
            return np.diag(np.sqrt(self.dist[1:1 + nu].astype(np.float32)))
        if self.kind == "C":
            return self.dist[1 + nu * nu:1 + 2 * nu * nu].reshape(nu, nu)
        return np.array(self.params.sigma_chol[:nu * nu], np.float32).reshape(nu, nu)

    def sinv(self):
        """The float32 Sigma^-1 K3 weights the SIMPLE-mode perturbation cost with."""
        nu = self.nu
        if self.kind == "M2":
            return np.diag(np.float32(1) / self.dist[1:1 + nu].astype(np.float32))
        if self.kind == "C":
            return self.dist[1 + 2 * nu * nu:].reshape(nu, nu)
        return np.array(self.params.sigma_inv[:nu * nu], np.float32).reshape(nu, nu)

    def row_floats(self):
        return row_floats(self.T, self.nu, self.kind)


def make_case(T, nu, K, mode="simple", gamma=0.95, lam=0.5, kind="W", sigma=None, filter_u=False, update_lambda=False, u_min=None, u_max=None,
              u_init=None, seed=3, **kw):
    """(model, params[, dist]) of one generated case through make_params.  `gamma` is used in MEAN mode ("halton-spline")."""
    sig = corr_sigma(nu, seed=seed) if sigma is None else np.asarray(sigma, np.float64)
    if kind == "M2":
        sig = np.diag(np.diag(sig))
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode=mode, sampling_method="random", noise_sigma=sig.tolist(), lambda_=lam, sample_null_action=True,
                    rollout_var_discount=gamma, filter_u=filter_u, update_cov=kind != "W", cov_type="full" if kind == "C" else "diag",
                    update_lambda=update_lambda, u_min=u_min if u_min is not None else [-1e3], u_max=u_max if u_max is not None else [1e3],
                    u_init=u_init if u_init is not None else 0.0, **kw)
    m = nu_model(nu)
    p = make_params(mc, IsaacGymConfig(), nu, K, [(OBS_LINK_STATE, 0), (OBS_DOF_STATE, 0)])
    dist = None
    if kind == "M2":
        dist = np.concatenate([[lam], np.diag(sig)]).astype(np.float32)
    elif kind == "C":
        import adaptive_full_oracle as afo
        dist = afo.make_dist(lam, sig)
    return Case(m, p, T, nu, K, kind, sig, dist)


def mode_tag(case):
    return "simple" if case.simple else f"g{float(case.params.gamma):g}"


def k3_id(T, nu, K, kind, tag):
    rpl, ncons, _, _ = ws_layout(T, nu, kind)
    return f"k3-RPL{rpl}-{kind}-T{T}nu{nu}-ncons{ncons}-K{K}-{tag}"


def k3_inputs(case, seed=0, spread=4.0, favour_tail=True):
    """cost [T][K], x [T][nu][K] and U [T][nu] (float32) of a K3 case.

    S_k spans about `spread` * lambda over the samples and sum_t |gamma^t c_tk| stays a few lambda, so the float32 error of S
    stays far below lambda (the gate then tests the weights, not only the argmin).  With `favour_tail` the samples of the last
    (ragged) tile get S lower by 2 lambda: they carry a share of the weight that a kernel dropping them cannot hide."""
    T, nu, K, lam = case.T, case.nu, case.K, case.lam
    rng = np.random.default_rng(seed)
    L = case.chol().astype(np.float64)
    NR = T * nu
    if case.simple:
        U = np.einsum("ij,tj->ti", L, rng.normal(0, 0.5 / math.sqrt(NR), (T, nu)))      # |L^-1 U| ~ 0.5: g.x ~ lambda / 2
    else:
        U = rng.normal(0, 0.1, (T, nu))
    U = U.astype(np.float32)
    noise = np.einsum("ij,tjk->tik", L, rng.standard_normal((T, nu, K))).astype(np.float32)
    x = noise if case.simple else (U[:, :, None] + noise).astype(np.float32)
    g = 1.0 if case.simple else float(case.params.gamma)
    Gam = sum(abs(g) ** t for t in range(T)) if g != 0 else 1.0
    v = rng.uniform(0, 1, K)[None, :] + 0.3 * rng.uniform(0, 1, (T, K))
    cost = (lam * spread / (1.3 * Gam)) * v
    if favour_tail:
        cost[0, WS_W * ((K - 1) // WS_W):] -= 2.0 * lam
    return np.ascontiguousarray(cost, np.float32), np.ascontiguousarray(x), U


# ---------------------------------------------------------------------------------------------------------------- K3 restatements
def _gammas(case):
    g = 1.0 if case.simple else float(case.params.gamma)
    return np.array([1.0] + [g ** t for t in range(1, case.T)])


def k3_restate(case, cost, x, U, keep=None):
    """float64 K3 of the case: S[K], w[K] and the shard row of its kind.  `keep`: mask of the samples that take part."""
    T, nu, K, lam = case.T, case.nu, case.K, case.lam
    c64 = np.asarray(cost, np.float64).reshape(T, K)
    x64 = np.asarray(x, np.float64).reshape(T * nu, K)
    U64 = np.asarray(U, np.float64).reshape(T, nu)
    with np.errstate(invalid="ignore"):
        S = (_gammas(case)[:, None] * c64).sum(0)
    if case.simple:
        g = lam * (U64 @ case.sinv().astype(np.float64).T).reshape(-1)       # g_r = lambda sum_j Sinv_ij U_tj
        S = S + g @ x64
    ok = np.isfinite(S) if keep is None else np.isfinite(S) & keep
    b = S[ok].min() if ok.any() else np.inf
    w = np.where(ok, np.exp(-(np.where(ok, S, b) - b) / lam), 0.0)
    row = [np.array([b, w.sum()]), x64 @ w]
    c = 0.0 if case.simple else U64.reshape(-1, 1)
    if case.kind == "M2":
        row.append(((x64 - c) ** 2) @ w)
    elif case.kind == "C":
        d = (x64 - c).reshape(T, nu, K).transpose(1, 0, 2).reshape(nu, T * K)
        C = (d * np.tile(w, T)[None]) @ d.T
        i, j = np.tril_indices(nu)
        row.append(C[i, j])
    return S, w, np.concatenate(row)


def k3_S32(case, cost, x, U):
    """float32 restatement of phase A of the kernel: gamma^t = exp2(log2(gamma) t) (1 at t = 0), g = lambda Sigma^-1 U, and S_k as
    four interleaved accumulation chains, (a0 + a1) + (a2 + a3)."""
    f = np.float32
    T, nu, K = case.T, case.nu, case.K
    NR = T * nu
    gam = f(1.0) if case.simple else f(case.params.gamma)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        lg = np.log2(gam)
        gp = np.array([f(1)] + [np.exp2(f(lg * f(t))) for t in range(1, T)], f)
    terms = [(gp[t], cost[t]) for t in range(T)]
    T4 = (T + 3) & ~3
    terms += [(f(0), cost[T - 1])] * (T4 - T)
    if case.simple:
        si, Uf = case.sinv().astype(f), np.asarray(U, f).reshape(T, nu)
        g = np.zeros(NR, f)
        for t in range(T):
            for i in range(nu):
                acc = f(0)
                for j in range(nu):
                    acc = f(acc + f(si[i, j] * Uf[t, j]))
                g[t * nu + i] = f(acc * f(case.lam))
        xr = np.asarray(x, f).reshape(NR, K)
        terms += [(g[r], xr[r]) for r in range(NR)]
        terms += [(f(0), xr[NR - 1])] * (((NR + 3) & ~3) - NR)
    a = [np.zeros(K, f) for _ in range(4)]
    with np.errstate(invalid="ignore", over="ignore"):
        for n, (gv, col) in enumerate(terms):
            a[n % 4] = (a[n % 4] + gv * col).astype(f)
        return ((a[0] + a[1]) + (a[2] + a[3])).astype(f)


def k3_dS(case, cost, x, U):
    """Per-sample bound on |S_kernel - S| (float32 kernel against the float64 restatement)."""
    T, nu, K, lam = case.T, case.nu, case.K, case.lam
    NR = T * nu
    gam = 1.0 if case.simple else float(case.params.gamma)
    lg = abs(math.log2(gam)) if gam > 0 else 0.0
    gamma_t = np.abs(_gammas(case))
    with np.errstate(invalid="ignore"):
        A = (gamma_t[:, None] * np.abs(np.asarray(cost, np.float64))).sum(0)
    n = (T + 3) // 4 * 4 + ((NR + 3) // 4 * 4 if case.simple else 0)          # terms of the four chains
    dS = (n / 4 + 6 + 2 * math.log(2) * lg * T) * A
    if case.simple:
        gabs = lam * (np.abs(np.asarray(U, np.float64)) @ np.abs(case.sinv().astype(np.float64)).T).reshape(-1)
        dS = dS + (n / 4 + nu + 6) * (gabs @ np.abs(np.asarray(x, np.float64).reshape(NR, K)))
    return EPS * dS


def k3_gate(case, cost, x, U, S, w):
    """Element-wise bound on |row_kernel - row_reference| for the case's row kind (S, w: of ``k3_restate``)."""
    T, nu, K, lam = case.T, case.nu, case.K, case.lam
    NR = T * nu
    _, ncons, _, _ = ws_layout(T, nu, case.kind)
    ntiles = (K + WS_W - 1) // WS_W
    grid = min(ntiles, NUM_SMS)
    per_cta = -(-ntiles // grid)
    per_warp = -(-per_cta // ncons)
    rho = EPS * (64 + 3 * per_warp + grid / 4)
    ok = w > 0
    dS = k3_dS(case, cost, x, U)
    db = dS[ok].max() if ok.any() else 0.0
    b = S[ok].min() if ok.any() else np.inf
    with np.errstate(over="ignore", invalid="ignore"):
        w_hi = np.where(ok, np.exp(np.minimum(-(np.where(ok, S, b) - b - dS - db) / lam, 700.0)), 0.0)
    dw = (w_hi - w) + w * rho                                                  # |w_kernel - w| per sample, in the reference's scale
    x64 = np.asarray(x, np.float64).reshape(NR, K)
    gate = [np.array([db + EPS * abs(b) if ok.any() else 0.0, dw.sum() + EPS * w.sum()]), np.abs(x64) @ dw + EPS * np.abs(x64 @ w)]
    c = 0.0 if case.simple else np.asarray(U, np.float64).reshape(-1, 1)
    if case.kind == "M2":
        d2 = (x64 - c) ** 2
        gate.append(d2 @ (dw + 4 * EPS * w) + EPS * (d2 @ w))
    elif case.kind == "C":
        d = np.abs(x64 - c).reshape(T, nu, K).transpose(1, 0, 2).reshape(nu, T * K)
        M = (d * np.tile(dw + (T + 8) * EPS * w, T)[None]) @ d.T + EPS * ((d * np.tile(w, T)[None]) @ d.T)
        i, j = np.tril_indices(nu)
        gate.append(M[i, j])
    return np.concatenate(gate)


def drop_tail_mask(K):
    """The samples of every tile but the last (ragged) one: a reference computed without them must miss the gate."""
    keep = np.ones(K, bool)
    keep[WS_W * ((K - 1) // WS_W):] = False
    return keep


def row_excess(got, ref, gate):
    """max(|got - ref| - gate) over the row, with inf == inf counted as equal; > 0 means outside the gate."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    same = (got == ref)
    err = np.where(same, 0.0, np.abs(got - ref))
    err = np.where(np.isnan(err), np.inf, err)
    return float((err - gate).max()), float(err.max())
