"""Generated sampling / reduction / update cases at any accepted (T, nu, K), and the float32 error bounds of K3 that the tests gate on.

K1, K3, K4 and the shift read nothing of the model but ``nu``, so every case runs on the point robot's model with ``nu`` set and both
command maps of every joint pointing at input 0 (no dynamics run).  ``make_case`` builds the parameter block through ``make_params``
and, for the adaptive row kinds, the live distribution:

* ``W``  -- fixed Sigma (``sigma_chol`` / ``sigma_inv``), shard row ``[beta, eta, W[T*nu]]``;
* ``M2`` -- ``update_cov`` with a diagonal Sigma, ``dist = [lambda, cov[nu]]``, row ``+ M2[T*nu]``;
* ``C``  -- ``update_cov`` with ``cov_type: full``, ``dist = [lambda, Sigma, L, Sigma^-1]``, row ``+ C[nu(nu+1)/2]``;
* ``H``  -- ``update_cov`` with ``cov_type: horizon``, ``dist = [lambda, Sigma_H, L_H, Sigma_H^-1]`` (n = T*nu), row ``+ C[n(n+1)/2]``
  over the whole horizon (the SYRK after K3 appends it).

``ws_layout`` restates the shared-memory plan of the warp-specialised K3 (``WsLayout`` and the ring-depth rule of
``launch_reduce_ws_t`` in ``csrc/reduce.cu``), so a case id can name the instantiation and the consumer-warp count that run.  For
``H`` the host sizes the ring with the M2 layout while the kernel addresses the (smaller) W layout, and the restatement follows the
host.  With ``modes`` = M > 1 it follows the MODES launch, whose ring region also holds the fused K4 (``modes_fin_floats``), and
``modes_grid`` restates that launch's (gx, M) grid.  ``syrk_split`` restates the split of the SYRK over lower-triangle 64 x 64 tiles and K-chunks.

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
SMEM_OPTIN, MAX_NU = 227 * 1024, 16    # the H100's opt-in shared memory per CTA; MPPIB_MAX_NU


def row_floats(T, nu, kind, Tc=None, feasible=False):
    """Floats of the shard row (``shard_row_floats``): Tc control rows (default T; knots: P); `feasible`: the FEASIBLE row
    (beta, eta, W[Tc*nu], n_feasible, min V)."""
    NR = (T if Tc is None else Tc) * nu
    if feasible:
        return 4 + NR
    return 2 + NR + (NR if kind == "M2" else nu * (nu + 1) // 2 if kind == "C" else NR * (NR + 1) // 2 if kind == "H" else 0)


def modes_fin_floats(NR, M, G):
    """Shared floats ``modes_rows`` (the K4 of n_modes = M > 1) needs with G shard rows: d, Sigma^-1 U / the coupled U and U [M*NR]
    each, Sigma^-1 [16 x 16], the G scales of every mode, (beta, eta, F, sum_j k_ij) [M], D and k [M][M], 4 floats."""
    return 3 * M * NR + MAX_NU * MAX_NU + M * G + 4 * M + 2 * M * M + 4


def _ws_bytes(T, nu, nstage, kind, nparts=None, smooth=False, modes=1, Tc=None, feasible=False):
    """Bytes of ``WsLayout``: nparts warp partials (default one per consumer, min(nstage, 7)); smooth adds the [NR4] U region; with
    modes = M > 1 the ring region holds at least modes_fin_floats(NR, M, 1), where the fused K4 runs ``modes_rows``.  A tile holds
    NR = Tc*nu control rows and T cost rows, and with `feasible` T violation rows more."""
    NR = (T if Tc is None else Tc) * nu
    P4 = (row_floats(T, nu, kind, Tc, feasible) + 3) & ~3
    ring, fold = nstage * (NR + (2 * T if feasible else T)) * WS_W, MAX_GRID + 4 * P4
    g = max(ring, fold)
    if kind == "C":
        g = max(g, NR + 1 + 2 * NR + nu * (nu + 1) // 2 + 3 * nu * nu)
    if modes > 1:
        g = max(g, modes_fin_floats(NR, modes, 1))
    gp = g + ((NR + 3) & ~3)
    wk = gp + ((T + 3) & ~3)
    misc = wk + 8 * WS_W + (min(nstage, WS_NCONS) if nparts is None else nparts) * P4
    us = misc + 8
    bar = ((us + (((NR + 3) & ~3) if smooth else 0)) * 4 + 15) & ~15
    return bar + 2 * 8 * nstage + 128


def ws_stages(T, nu, kind, smooth=False, Tc=None, feasible=False):
    """The ring depth rule of ``reduce_ws_stages``: the deepest ring next to seven warp partials, else two stages next to two."""
    ns = 8
    while ns > 1 and _ws_bytes(T, nu, ns, kind, WS_NCONS, smooth, Tc=Tc, feasible=feasible) > SMEM_CAP:
        ns -= 1
    if ns < 2 and _ws_bytes(T, nu, 2, kind, None, smooth, Tc=Tc, feasible=feasible) <= SMEM_CAP:
        ns = 2
    return ns


def ws_layout(T, nu, kind, smooth=False, modes=1, Tc=None, feasible=False):
    """(rows of W per lane, consumer warps, ring stages, rows per x TMA box) of the K3 launch, or None if the shape is refused.
    `smooth`: the layout of mode smooth (row W, plus the U region of the smoothness cost).  `modes` = M > 1: the MODES launch (row W
    per mode): the ring depth is chosen without the modes_rows floor, and the launch, floor included, must fit the opt-in limit.
    `Tc`: the control rows (knots: P; default T).  `feasible`: the FEASIBLE launch of constraint_mode (row W, T violation rows more
    per tile, the row 4 + T*nu)."""
    Tc = T if Tc is None else Tc
    NR = Tc * nu
    if kind == "H":
        if NR > HZ_MAX_N:
            return None
        kind = "M2"                    # the host sizes the horizon K3 (row W only) with the update_cov rule's M2 layout
    if NR > 512 or T > 256 or ws_stages(T, nu, "W", Tc=Tc) < 2 or ws_stages(T, nu, kind, smooth, Tc, feasible) < 2:
        return None
    ns = ws_stages(T, nu, kind, smooth, Tc, feasible)
    ncons = min(ns, WS_NCONS)
    nstage = ncons * (ns // ncons)
    if modes > 1 and _ws_bytes(T, nu, nstage, kind, None, smooth, modes, Tc, feasible) > SMEM_OPTIN:
        return None
    xbox = min(NR, 256)
    while NR % xbox:
        xbox -= 1
    return (4 if NR <= 128 else 8 if NR <= 256 else 16), ncons, nstage, xbox


def mode_range(K, k_offset, Kc, m):
    """[lo, hi) local samples of mode m in the shard [k_offset, k_offset + K) (lo >= hi: none), as the MODES K3 CTA restates it."""
    return max(0, m * Kc - k_offset), min(K, (m + 1) * Kc - k_offset)


def mode_tiles(K, k_offset, Kc, m):
    """32-sample tiles the MODES K3 walks for mode m: from the tile of its first local sample to that of its last (0 without one)."""
    lo, hi = mode_range(K, k_offset, Kc, m)
    return (hi + WS_W - 1) // WS_W - lo // WS_W if hi > lo else 0


def modes_grid(K, k_offset, Kc, M, sms=NUM_SMS):
    """gx of the MODES K3 grid (gx, M) (``launch_reduce_ws_t``): about one CTA per SM over all modes, no more than the tiles of the
    largest mode's local range, at least 1."""
    tmax = max(mode_tiles(K, k_offset, Kc, m) for m in range(M))
    return max(1, min(tmax, sms // M))


def wrap_K(T, nu, kind, sms=NUM_SMS, smooth=False, Tc=None, feasible=False):
    """A ragged K (multiple of 4) whose every CTA streams more than three full rings of tiles."""
    _, _, nstage, _ = ws_layout(T, nu, kind, smooth, Tc=Tc, feasible=feasible)
    return WS_W * sms * (3 * nstage + 1) - 12


# ---------------------------------------------------------------------------------------------------------------- SYRK split
HZ_MAX_N, HZ_TILE, HZ_KB = 256, 64, 32


def syrk_split(n, K, sms=NUM_SMS):
    """(ntiles, ksplit, kchunk) of the SYRK (``syrk_split`` in csrc/reduce.cu): about one CTA per SM over the lower-triangle 64 x 64
    tiles of C, chunks rounded up to a multiple of 32 samples; the last chunk holds what is left (4 samples at least)."""
    nb = (n + HZ_TILE - 1) // HZ_TILE
    ntiles = nb * (nb + 1) // 2
    ks = max(sms // ntiles, 1)
    kc = -(-K // ks)
    kc = -(-kc // HZ_KB) * HZ_KB
    return ntiles, -(-K // kc), kc


def last4_K(n, sms=NUM_SMS):
    """A K that splits into as many chunks as large K does, the last of them holding only 4 samples."""
    _, ks0, _ = syrk_split(n, 1 << 20, sms)                                     # the split count at large K
    for kc in range(HZ_KB, 1 << 16, HZ_KB):
        for ks in range(ks0, 1, -1):
            K = kc * (ks - 1) + 4
            if syrk_split(n, K, sms)[1:] == (ks, kc):
                return K
    raise ValueError(n)


def hz_id(T, nu, K, tag, sms=NUM_SMS):
    rpl, ncons, _, _ = ws_layout(T, nu, "H")
    ntiles, ksplit, _ = syrk_split(T * nu, K, sms)
    return f"hz-RPL{rpl}-T{T}nu{nu}-ncons{ncons}-t{ntiles}x{ksplit}-K{K}-{tag}"


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

    @property
    def n(self):
        return self.T * self.nu

    @property
    def Tc(self):
        """The control rows of x and U: the knots P with control_knots > 0, else T."""
        return int(self.params.control_knots) or self.T

    def chol(self):
        """The float32 lower factor K1 colours with (n x n for H)."""
        nu, n = self.nu, self.n
        if self.kind == "H":
            return self.dist[1 + n * n:1 + 2 * n * n].reshape(n, n)
        if self.kind == "M2":
            return np.diag(np.sqrt(self.dist[1:1 + nu].astype(np.float32)))
        if self.kind == "C":
            return self.dist[1 + nu * nu:1 + 2 * nu * nu].reshape(nu, nu)
        return np.array(self.params.sigma_chol[:nu * nu], np.float32).reshape(nu, nu)

    def sinv(self):
        """The float32 Sigma^-1 K3 weights the SIMPLE-mode perturbation cost with (n x n Sigma_H^-1 for H)."""
        nu, n = self.nu, self.n
        if self.kind == "H":
            return self.dist[1 + 2 * n * n:].reshape(n, n)
        if self.kind == "M2":
            return np.diag(np.float32(1) / self.dist[1:1 + nu].astype(np.float32))
        if self.kind == "C":
            return self.dist[1 + 2 * nu * nu:].reshape(nu, nu)
        return np.array(self.params.sigma_inv[:nu * nu], np.float32).reshape(nu, nu)

    def row_floats(self):
        return row_floats(self.T, self.nu, self.kind)


def horizon_sigma(T, sig0, sigma_h="iid", tau=3.0):
    """Sigma_H of an H case: "iid" I_T (x) Sigma0; "corr" exp(-|t - t'| / tau) (x) Sigma0; a number c: the correlated one with its
    eigenvalues spread geometrically (order and eigenvectors kept) to condition number c."""
    sig0 = np.asarray(sig0, np.float64)
    if sigma_h == "iid":
        return np.kron(np.eye(T), sig0)
    t = np.arange(T)
    S = np.kron(np.exp(-np.abs(t[:, None] - t[None, :]) / tau), sig0)
    if sigma_h == "corr":
        return S
    w, V = np.linalg.eigh(S)
    if len(w) > 1:
        pw = math.log(float(sigma_h)) / math.log(w[-1] / w[0])
        w = w[-1] * (w / w[-1]) ** pw
    S = (V * w) @ V.T
    return 0.5 * (S + S.T)


def make_case(T, nu, K, mode="simple", gamma=0.95, lam=0.5, kind="W", sigma=None, filter_u=False, update_lambda=False, u_min=None, u_max=None,
              u_init=None, seed=3, sigma_h="corr", **kw):
    """(model, params[, dist]) of one generated case through make_params.  `gamma` is used in MEAN mode ("halton-spline"); `sigma_h`
    chooses Sigma_H of an H case (``horizon_sigma``)."""
    sig = corr_sigma(nu, seed=seed) if sigma is None else np.asarray(sigma, np.float64)
    if kind == "M2":
        sig = np.diag(np.diag(sig))
    cov_type = {"C": "full", "H": "horizon"}.get(kind, "diag")
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode=mode, sampling_method="random", noise_sigma=sig.tolist(), lambda_=lam, sample_null_action=True,
                    rollout_var_discount=gamma, filter_u=filter_u, update_cov=kind != "W", cov_type=cov_type,
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
    elif kind == "H":
        import adaptive_horizon_oracle as aho
        dist = aho.make_dist(lam, horizon_sigma(T, sig, sigma_h))
    return Case(m, p, T, nu, K, kind, sig, dist)


def mode_tag(case):
    return "simple" if case.simple else f"g{float(case.params.gamma):g}"


def k3_id(T, nu, K, kind, tag):
    rpl, ncons, _, _ = ws_layout(T, nu, kind)
    return f"k3-RPL{rpl}-{kind}-T{T}nu{nu}-ncons{ncons}-K{K}-{tag}"


def k3_inputs(case, seed=0, spread=4.0, favour_tail=True):
    """cost [T][K], x [Tc][nu][K] and U [Tc][nu] (float32) of a K3 case (Tc: the control rows, ``Case.Tc``).

    S_k spans about `spread` * lambda over the samples and sum_t |gamma^t c_tk| stays a few lambda, so the float32 error of S
    stays far below lambda (the gate then tests the weights, not only the argmin).  With `favour_tail` the samples of the last
    (ragged) tile get S lower by 2 lambda: they carry a share of the weight that a kernel dropping them cannot hide.
    For H the noise is coloured by L_H over the whole horizon, and the last step of U is u_init = 0: U is what mppib_shift leaves
    (``shifted_from``), which is where the device computes the SIMPLE-mode g = lambda Sigma_H^-1 U."""
    T, Tc, nu, K, lam = case.T, case.Tc, case.nu, case.K, case.lam
    rng = np.random.default_rng(seed)
    L = case.chol().astype(np.float64)
    NR = Tc * nu
    if case.kind == "H":
        if case.simple:
            U = (L @ rng.normal(0, 0.5 / math.sqrt(NR), NR)).reshape(T, nu)
        else:
            U = rng.normal(0, 0.1, (T, nu))
        U[-1] = 0.0
    elif case.simple:
        U = np.einsum("ij,tj->ti", L, rng.normal(0, 0.5 / math.sqrt(NR), (Tc, nu)))     # |L^-1 U| ~ 0.5: g.x ~ lambda / 2
    else:
        U = rng.normal(0, 0.1, (Tc, nu))
    U = U.astype(np.float32)
    if case.kind == "H":
        noise = (L @ rng.standard_normal((NR, K))).reshape(T, nu, K).astype(np.float32)
    else:
        noise = np.einsum("ij,tjk->tik", L, rng.standard_normal((Tc, nu, K))).astype(np.float32)
    x = noise if case.simple else (U[:, :, None] + noise).astype(np.float32)
    g = 1.0 if case.simple else float(case.params.gamma)
    Gam = sum(abs(g) ** t for t in range(T)) if g != 0 else 1.0
    v = rng.uniform(0, 1, K)[None, :] + 0.3 * rng.uniform(0, 1, (T, K))
    cost = (lam * spread / (1.3 * Gam)) * v
    if favour_tail:
        cost[0, WS_W * ((K - 1) // WS_W):] -= 2.0 * lam
    return np.ascontiguousarray(cost, np.float32), np.ascontiguousarray(x), U


def shifted_from(U, seed=0):
    """A U_prev whose mppib_shift is U (the last step of U must be u_init): U_prev[t + 1] = U[t], U_prev[0] arbitrary."""
    Up = np.empty_like(U)
    Up[1:] = U[:-1]
    Up[0] = np.random.default_rng(seed).uniform(-1, 1, U.shape[1])
    return Up


# ---------------------------------------------------------------------------------------------------------------- K3 restatements
def _gammas(case):
    g = 1.0 if case.simple else float(case.params.gamma)
    return np.array([1.0] + [g ** t for t in range(1, case.T)])


def k3_restate(case, cost, x, U, keep=None):
    """float64 K3 of the case: S[K], w[K] and the shard row of its kind.  `keep`: mask of the samples that take part."""
    T, Tc, nu, K, lam = case.T, case.Tc, case.nu, case.K, case.lam
    c64 = np.asarray(cost, np.float64).reshape(T, K)
    x64 = np.asarray(x, np.float64).reshape(Tc * nu, K)
    U64 = np.asarray(U, np.float64).reshape(Tc, nu)
    with np.errstate(invalid="ignore"):
        S = (_gammas(case)[:, None] * c64).sum(0)
    if case.simple:
        if case.kind == "H":
            g = lam * (case.sinv().astype(np.float64) @ U64.reshape(-1))      # g = lambda Sigma_H^-1 U over the horizon
        else:
            g = lam * (U64 @ case.sinv().astype(np.float64).T).reshape(-1)   # g_r = lambda sum_j Sinv_ij U_tj
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
    elif case.kind == "H":
        row.append(hz_C(case, x, U, w))
    return S, w, np.concatenate(row)


def hz_C(case, x, U, w, k0=0, k1=None):
    """Packed lower triangle of C = sum_k w_k (x_k - c)(x_k - c)^T over the samples [k0, k1) (float64; c = U in MEAN mode, else 0)."""
    n, K = case.n, case.K
    k1 = K if k1 is None else k1
    d = np.asarray(x, np.float64).reshape(n, K)[:, k0:k1]
    if not case.simple:
        d = d - np.asarray(U, np.float64).reshape(n, 1)
    C = (d * w[None, k0:k1]) @ d.T
    return C[np.tril_indices(n)]


def k3_S32(case, cost, x, U):
    """float32 restatement of phase A of the kernel: gamma^t = exp2(log2(gamma) t) (1 at t = 0), g = lambda Sigma^-1 U, and S_k as
    four interleaved accumulation chains, (a0 + a1) + (a2 + a3), over the T cost terms and then the Tc*nu control terms."""
    f = np.float32
    T, Tc, nu, K = case.T, case.Tc, case.nu, case.K
    NR = Tc * nu
    gam = f(1.0) if case.simple else f(case.params.gamma)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        lg = np.log2(gam)
        gp = np.array([f(1)] + [np.exp2(f(lg * f(t))) for t in range(1, T)], f)
    terms = [(gp[t], cost[t]) for t in range(T)]
    T4 = (T + 3) & ~3
    terms += [(f(0), cost[T - 1])] * (T4 - T)
    if case.simple and case.kind == "H":
        si, Uf = case.sinv().astype(f), np.asarray(U, f).reshape(NR)
        acc = np.zeros(NR, f)
        for c in range(NR):                                                     # mppib_shift: a row per thread, columns in order
            acc = (acc + si[:, c] * Uf[c]).astype(f)
        g = (acc * f(case.lam)).astype(f)
        xr = np.asarray(x, f).reshape(NR, K)
        terms += [(g[r], xr[r]) for r in range(NR)]
        terms += [(f(0), xr[NR - 1])] * (((NR + 3) & ~3) - NR)
    elif case.simple:
        si, Uf = case.sinv().astype(f), np.asarray(U, f).reshape(Tc, nu)
        g = np.zeros(NR, f)
        for t in range(Tc):
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
    """Per-sample bound on |S_kernel - S| (float32 kernel against the float64 restatement): T cost terms, Tc*nu control terms."""
    T, nu, K, lam = case.T, case.nu, case.K, case.lam
    NR = case.Tc * nu
    gam = 1.0 if case.simple else float(case.params.gamma)
    lg = abs(math.log2(gam)) if gam > 0 else 0.0
    gamma_t = np.abs(_gammas(case))
    with np.errstate(invalid="ignore"):
        A = (gamma_t[:, None] * np.abs(np.asarray(cost, np.float64))).sum(0)
    n = (T + 3) // 4 * 4 + ((NR + 3) // 4 * 4 if case.simple else 0)          # terms of the four chains
    dS = (n / 4 + 6 + 2 * math.log(2) * lg * T) * A
    if case.simple:
        if case.kind == "H":                                                    # g sums n terms (mppib_shift), not nu
            gabs, inner = lam * (np.abs(case.sinv().astype(np.float64)) @ np.abs(np.asarray(U, np.float64)).reshape(-1)), NR
        else:
            gabs, inner = lam * (np.abs(np.asarray(U, np.float64)) @ np.abs(case.sinv().astype(np.float64)).T).reshape(-1), nu
        dS = dS + (n / 4 + inner + 6) * (gabs @ np.abs(np.asarray(x, np.float64).reshape(NR, K)))
    return EPS * dS


def v_dS(g):
    """Per-sample bound on the float32 error of V_k = sum_t max(g_tk, 0) summed in t order (constraint_mode's K3):
    (T + 2) eps sum_t max(g_tk, 0)."""
    g = np.asarray(g, np.float64)
    with np.errstate(invalid="ignore"):
        return (g.shape[0] + 2) * EPS * np.where(g > 0, g, 0.0).sum(0)


def k3_gate(case, cost, x, U, S, w, sms=NUM_SMS):
    """Element-wise bound on |row_kernel - row_reference| for the case's row kind (S, w: of ``k3_restate``; sms: of the device).

    The C of H (the SYRK) recomputes every weight from K3's float32 S_k and beta = row[0] with one expf, so a weight carries the
    spread of S and beta (w_hi - w) plus a few roundings; each entry is then a sample-ordered FFMA sum over a chunk of kchunk
    samples and a fold of ksplit chunk sums:  |dC_ij| <= sum_k |dx_ik| |dx_jk| (dw_k + (kchunk + ksplit + 4) eps w_k)."""
    T, nu, K, lam = case.T, case.nu, case.K, case.lam
    NR = case.Tc * nu
    _, ncons, _, _ = ws_layout(T, nu, case.kind, Tc=case.Tc)
    ntiles = (K + WS_W - 1) // WS_W
    grid = min(ntiles, sms)
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
    elif case.kind == "H":
        _, ksplit, kchunk = syrk_split(NR, K, sms)
        d = np.abs(x64 - c)
        gate.append((((d * ((w_hi - w) + (kchunk + ksplit + 4) * EPS * w)[None]) @ d.T))[np.tril_indices(NR)])
    return np.concatenate(gate)


def hz_k1_gate(L, z, U, a_ref):
    """Per-element bound on |a_kernel - a_ref| of the horizon K1 against the float32-rounded float64 colouring of the device's own white
    draws z [n][K]: row r sums r + 1 products in column order, so |da_r| <= eps ((r + 2) sum_{c<=r} |L_rc z_c| + |U_r|) + eps |a_ref|.
    Clamping is monotone and adds nothing."""
    n = L.shape[0]
    Lz = np.abs(np.asarray(L, np.float64)) @ np.abs(np.asarray(z, np.float64).reshape(n, -1))
    r = np.arange(n, dtype=np.float64)[:, None]
    return EPS * ((r + 2) * Lz + np.abs(np.asarray(U, np.float64)).reshape(n, 1) + np.abs(np.asarray(a_ref, np.float64)).reshape(n, -1))


def hz_k1_f32(L, z, U):
    """float32 restatement of the horizon K1 before clamping: U_r + sum_c L_rc z_c accumulated in column order from c = 0."""
    f = np.float32
    n = L.shape[0]
    Lf, zf = np.asarray(L, f), np.asarray(z, f).reshape(n, -1)
    acc = np.zeros_like(zf)
    for c in range(n):
        acc = (acc + Lf[:, c:c + 1] * zf[c:c + 1]).astype(f)
    return (np.asarray(U, f).reshape(n, 1) + acc).astype(f)


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
