"""-m gpu: the kernels of multi-modal MPPI (``n_modes``) and annealed MPPI (``anneal_iterations``) over every template instantiation and
the accepted (T, nu, K, n_modes, anneal_iterations) range, against the float64 references ``modes_oracle`` and ``anneal_oracle``, on the
generated cases of ``synth_mppi`` (the point robot's model with nu set; no dynamics run).

* modes K1: every sampling entry admitted with n_modes > 1 (Philox Gaussian, colored, Halton library) equals the plain K1 with U := U_m
  on the columns of mode m, bit for bit, also on shards that cut modes and tiles;
* modes K3: every mode's block (beta, eta, W) within ``_row_gate`` over that mode's samples, on (gx, M) grids from gx = 1 to
  num_sms / M, ring-wrapping K, shards that cut modes or hold no sample of some, +inf / NaN costs and dead modes; fused equals split;
* modes K4 (``modes_rows``): U, F and the executed mode against ``modes_oracle.finalize`` within a bound that carries the float32
  rounding of the combined rows, D, the bandwidth h and the kernel k through the coupled step and Savitzky-Golay;
* modes shift against ``modes_oracle.shift`` bit for bit;
* annealed K1 against ``anneal_oracle.sample`` within the bound of ``test_gpu_anneal``, and K3 (RPL 4 / 8 / 16, RISK) within
  ``_row_gate`` with g scaled by the schedule's r; split and fused, the counter advanced by the fused tail only;
* an annealed panda-reach plan at T = 30, nu = 7, K = 2048 against ``AnnealOracleBackend``.

Each gate has a negative control, a deliberately wrong reference that must miss it.  Each sweep case prints a ``MODES <id> worst ...
gate ...`` line (shown with -s)."""
import copy
import dataclasses
import math

import numpy as np
import pytest
import torch

import anneal_oracle as ao
import modes_oracle as mo
import risk_oracle as ro
from mppi_isaac_b200.model.blob import ANNEAL_MIN_SCALE, MODE_SIMPLE, make_params
from mppi_isaac_b200.planner.mppi import colored_noise_chol, halton_spline_operator, halton_table
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from synth_mppi import (EPS, NUM_SMS, WS_W, k3_dS, k3_inputs, make_case, mode_range, mode_tiles, modes_grid, nu_model, row_excess, wrap_K,
                        ws_layout)
from test_gpu_mode_shapes import _line, _risk_Ks, _row_gate

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED, PLAN = 0x1_2345_6789, 2 ** 32 + 7
MAX_PEERS = 16                                                                 # MPPIB_MAX_PEERS


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def f32(v):
    return float(np.float32(v))


def backend(nu, p, state=None, anneal=None, N=1):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(nu_model(nu), p)
    if state is not None:
        be.set_distribution(state)
    if anneal is not None:
        be.set_anneal(anneal, N)
    return be


def mparams(nu, T, K_total, M=1, K=None, k_offset=0, **kw):
    """A parameter block of n_modes = M over K_total samples (Kc = K_total / M per mode), for the shard [k_offset, k_offset + K)."""
    d = dict(num_samples=K_total, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.3 * np.eye(nu) + 0.05).tolist(),
             u_min=[-1.0], u_max=[1.0], lambda_=0.5, sample_null_action=True, n_modes=M)
    d.update(kw)
    p = make_params(MPPIConfig(**d), IsaacGymConfig(), nu, K_total, [])
    p.K, p.k_offset = K or K_total, k_offset
    return p


def mode_state(M, T, nu, active=0, U_exec=None):
    """The mode state (active mode, F[M], U_exec[T][nu])."""
    return np.concatenate([[active], np.full(M, np.inf), np.zeros(T * nu) if U_exec is None else np.ravel(U_exec)]).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------------------ modes K1
K1_NU = [1, 2, 5, 13, 16]
K1_M = [2, 3, 7, 16]
K1_KC = [32, 33, 100, 1000]


def _modes_k1_cases():
    """(nu, T) cells at T = 1, 9 and the largest accepted T (T*nu = 512 at nu = 2 and 16); every (M, Kc) pair over each 16 cases."""
    out, i = [], 0
    for nu in K1_NU:
        for T in sorted({1, 9, min(512 // nu, 256)}):
            for variant in ("random", "colored", "halton"):
                M, Kc = K1_M[i % 4], K1_KC[(i + i // 4) % 4]
                i += 1
                out.append(pytest.param(variant, T, nu, M, Kc, id=f"modes-k1-{variant}-T{T}nu{nu}-M{M}-Kc{Kc}"))
    return out


def k1_run(be, variant, T, nu, K, k_offset, k_total, U):
    """K1 of `variant` on the handle's parameter block: (actions, noise) [T][nu][K] of the shard [k_offset, k_offset + K)."""
    a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    if variant == "random":
        be.sample(SEED, PLAN, k_offset, k_total, U, None, a, n)
    elif variant == "colored":
        be.sample_colored(SEED, PLAN, k_offset, k_total, U, None, dev(colored_noise_chol(T, 2.0)), a, n)
    else:
        nk = min(max(T // 4, 3), 32)                                           # the library takes at most 32 knots
        Z = torch.zeros((T, nu, K), device=DEV)
        be.noise_library(k_offset, k_total, torch.from_numpy(halton_table(nk * nu, 5)).to(DEV), dev(halton_spline_operator(T, nk)), nk, Z)
        be.sample_library(k_offset, k_total, U, None, Z, a, n)
    torch.cuda.synchronize()
    return a.cpu().numpy(), n.cpu().numpy()


@pytest.mark.parametrize("variant,T,nu,M,Kc", _modes_k1_cases())
def test_modes_k1_sweep(variant, T, nu, M, Kc):
    """Columns of mode m = the plain K1 with U := U_m over [m Kc, (m + 1) Kc) (the counters are global samples), bit for bit, actions
    and noise; the null row stays global K - 1; shards whose offset and end fall inside a mode and a 32-sample tile equal the full launch.
    Negative control: the first and last column of every mode against the plain K1 with U_{m-1} and U_{m+1} differ (action or noise)."""
    Kt = M * Kc
    rng = np.random.default_rng(T * 131 + nu * 17 + M + Kc)
    Um = rng.uniform(-0.3, 0.3, (M, T, nu)).astype(np.float32)
    be = backend(nu, mparams(nu, T, Kt, M), dev(mode_state(M, T, nu)))
    full_a, full_n = k1_run(be, variant, T, nu, Kt, 0, Kt, dev(Um))
    pl = backend(nu, mparams(nu, T, Kt))
    same_neighbour = 0
    for m in range(M):
        q = copy.copy(pl.params)
        q.K, q.k_offset = Kc, m * Kc
        pl.set_params(q)
        cols = slice(m * Kc, (m + 1) * Kc)
        a, n = k1_run(pl, variant, T, nu, Kc, m * Kc, Kt, dev(Um[m]))
        np.testing.assert_array_equal(full_a[:, :, cols].view(np.uint32), a.view(np.uint32), err_msg=f"mode {m} actions")
        np.testing.assert_array_equal(full_n[:, :, cols].view(np.uint32), n.view(np.uint32), err_msg=f"mode {m} noise")
        for nb, col in (((m - 1) % M, 0), ((m + 1) % M, Kc - 1)):              # the neighbour across each boundary
            a2, n2 = k1_run(pl, variant, T, nu, Kc, m * Kc, Kt, dev(Um[nb]))
            kg = m * Kc + col
            same_neighbour += np.array_equal(full_a[:, :, kg], a2[:, :, col]) and np.array_equal(full_n[:, :, kg], n2[:, :, col])
    assert (full_a[:, :, Kt - 1] == 0.0).all() and (full_a[:, :, Kt - 2] != 0.0).any()   # the null row is global K - 1 only
    print(f"MODES modes-k1-{variant}-T{T}nu{nu}-M{M}-Kc{Kc} worst 0 gate 0 (bit for bit), "
          f"{2 * M - same_neighbour} of {2 * M} boundary columns tell U_m from its neighbour")
    assert same_neighbour == 0
    for off, Kl in ((Kc // 2 + 5, Kc + 7), (Kt - Kc - 3, Kc + 3)):             # cut inside mode 0 / 1 and tiles; the last mode and the null row
        sh = backend(nu, mparams(nu, T, Kt, M, K=Kl, k_offset=off), dev(mode_state(M, T, nu)))
        sa, sn = k1_run(sh, variant, T, nu, Kl, off, Kt, dev(Um))
        np.testing.assert_array_equal(sa.view(np.uint32), full_a[:, :, off:off + Kl].view(np.uint32))
        np.testing.assert_array_equal(sn.view(np.uint32), full_n[:, :, off:off + Kl].view(np.uint32))
        sh.destroy()
    be.destroy()
    pl.destroy()


# ------------------------------------------------------------------------------------------------------------------------------ modes K3
def _wrap_kc(T, nu, M):
    """Kc whose every CTA of the num_sms / M per mode streams more than three full rings."""
    return wrap_K(T, nu, "W", sms=NUM_SMS // M)


# T, nu, M, Kc, k_offset, K (None: the whole plan), mode, dead mode, what the case is for
MODES_K3 = [
    (8, 3, 2, 32, 0, None, "simple", None, "minKc"),
    (8, 3, 2, _wrap_kc(8, 3, 2), 0, None, "halton-spline", None, "wrap"),
    (8, 3, 16, 33, 0, None, "simple", 3, "odd"),
    (1, 1, 5, 96, 48, 96, "simple", None, "nolocal"),                          # modes 2 .. 4 have no local sample
    (8, 3, 5, 32, 27, 100, "halton-spline", None, "onetile"),                  # mode 0: five samples in one partial tile; mode 4: none
    (30, 7, 2, 2112, 0, None, "simple", None, "gxsms"),
    (30, 7, 16, 32, 0, None, "simple", 5, "minKc"),
    (43, 3, 5, 1001, 500, 3000, "halton-spline", 2, "cut"),
    (43, 3, 16, _wrap_kc(43, 3, 16), 0, None, "simple", None, "wrap"),
    (32, 16, 16, 256, 0, None, "simple", 7, "gxsms"),                          # the fused K4 at M = 16, T*nu = 512
    (256, 2, 16, 33, 0, None, "halton-spline", None, "odd"),
    (32, 16, 2, 32, 20, 40, "simple", None, "cut"),
    (20, 13, 5, 99, 150, 260, "simple", 1, "cut"),                             # mode 0 has no local sample, 1 and 4 are cut
    (32, 16, 16, _wrap_kc(32, 16, 16), 0, None, "halton-spline", None, "wrap"),
]


def _modes_k3_id(T, nu, M, Kc, off, K, mode, dead, what):
    K = K or M * Kc
    rpl, ncons, nstage, _ = ws_layout(T, nu, "W", modes=M)
    gx = modes_grid(K, off, Kc, M)
    tag = "simple" if mode == "simple" else "mean"
    return f"modes-k3-RPL{rpl}-T{T}nu{nu}-ncons{ncons}s{nstage}-M{M}-Kc{Kc}-gx{gx}-off{off}K{K}-{what}-{tag}" + ("" if dead is None else f"-dead{dead}")


def modes_k3_case(T, nu, M, Kc, off, K, mode, dead, seed):
    """(case, cost, x, U[M][T][nu]) of a shard: the k3_inputs construction per mode (a U_m of its own; MEAN mode x = U_m + noise), the
    first and the last local sample of every mode favoured by 2 lambda, a few +inf and one NaN cost, and NaN on every sample of `dead`."""
    K = K or M * Kc
    case = make_case(T, nu, M * Kc, mode=mode, n_modes=M, mode_switch_margin=0.05)
    p = copy.copy(case.params)
    p.K, p.k_offset = K, off
    case = dataclasses.replace(case, params=p, K=K)
    cost, noise, U0 = k3_inputs(case, seed=seed, favour_tail=False)
    if not case.simple:
        noise = noise - U0[:, :, None]                                         # MEAN mode: k3_inputs returns x = U + noise
    rng = np.random.default_rng(seed + 1)
    L = case.chol().astype(np.float64)
    NR = T * nu
    if case.simple:
        U = np.einsum("ij,mtj->mti", L, rng.normal(0, 0.5 / math.sqrt(NR), (M, T, nu)))
    else:
        U = rng.normal(0, 0.1, (M, T, nu))
    U = U.astype(np.float32)
    modes = mo.modes_of(p, off, K)
    x = noise if case.simple else (np.transpose(U[modes], (1, 2, 0)) + noise).astype(np.float32)
    for m in range(M):
        lo, hi = mode_range(K, off, Kc, m)
        if hi > lo:
            cost[0, lo] -= 2.0 * case.lam
            cost[0, hi - 1] -= 2.0 * case.lam
    cost[rng.integers(0, T, 3), rng.integers(0, K, 3)] = np.inf
    cost[rng.integers(0, T), rng.integers(0, K)] = np.nan
    if dead is not None:
        cost[0, modes == dead] = np.nan
    return case, np.ascontiguousarray(cost), np.ascontiguousarray(x), U


def modes_k3_restate(case, cost, x, U, keep=None):
    """float64 K3 per mode: the row [M][2 + T*nu] and, per mode, (local columns, S, w, beta, x rows)."""
    p, T, nu = case.params, case.T, case.nu
    M, NR = int(p.n_modes), T * nu
    modes = mo.modes_of(p, p.k_offset, case.K)
    row, parts = [], []
    for m in range(M):
        cols = np.flatnonzero(modes == m)
        xr = np.asarray(x, np.float64)[:, :, cols].reshape(NR, -1)
        if cols.size:
            with np.errstate(invalid="ignore"):
                S, lam = ro.scores(p, nu, cost[:, cols], x[:, :, cols], U[m])
        else:
            S, lam = np.zeros(0), case.lam
        ok = np.isfinite(S) if keep is None else np.isfinite(S) & keep[cols]
        b = S[ok].min() if ok.any() else np.inf
        w = np.where(ok, np.exp(-(np.where(ok, S, b) - b) / lam), 0.0)
        row.append(np.concatenate([[b, w.sum()], xr @ w]))
        parts.append((cols, S, w, b, xr))
    return np.concatenate(row), parts


def modes_k3_gate(case, cost, x, U, parts):
    """_row_gate of every mode's block over its own samples: its S within k3_dS of the float64 S (g = lambda Sigma^-1 U_m), the weighted
    sums over the mode's tiles on the gx CTAs of its row of the grid."""
    p = case.params
    M, Kc, off = int(p.n_modes), int(p.mode_samples), int(p.k_offset)
    _, ncons, _, _ = ws_layout(case.T, case.nu, "W", modes=M)
    gx = modes_grid(case.K, off, Kc, M)
    gate = []
    for m, (cols, S, w, b, xr) in enumerate(parts):
        if not cols.size:
            gate.append(np.zeros(2 + case.T * case.nu))
            continue
        sub = dataclasses.replace(case, K=cols.size)
        with np.errstate(invalid="ignore"):
            dS = k3_dS(sub, cost[:, cols], x[:, :, cols], U[m])
        g, _, _ = _row_gate(S, dS, w, b, xr, case.lam, WS_W * mode_tiles(case.K, off, Kc, m), ncons, sms=gx)
        gate.append(g)
    return np.concatenate(gate)


def drop_ends_mask(case):
    """Every local sample but the first and the last of each mode's local range."""
    p = case.params
    keep = np.ones(case.K, bool)
    for m in range(int(p.n_modes)):
        lo, hi = mode_range(case.K, int(p.k_offset), int(p.mode_samples), m)
        if hi > lo:
            keep[lo] = keep[hi - 1] = False
    return keep


def run_modes_k3(case, cost, x, U, state, fused):
    """K3 (split) or K3 + K4 (fused) of the case: (row, U, action, stats, mode state)."""
    nu, M = case.nu, int(case.params.n_modes)
    st = dev(state)
    be = backend(nu, case.params, st)
    part = torch.zeros(be.partial_row_floats(), device=DEV)
    Ud, act, stats = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    if fused:
        be.reduce_finalize(dev(cost), dev(x), Ud, part, act, stats)
    else:
        be.reduce(dev(cost), dev(x), Ud, part)
        be.finalize(part.view(1, -1), 1, Ud, act, stats)
    torch.cuda.synchronize()
    out = [t.cpu().numpy() for t in (part, Ud, act, stats, st)]
    be.destroy()
    assert out[0].size == M * (2 + case.T * nu)
    return out


@pytest.mark.parametrize("T,nu,M,Kc,off,K,mode,dead,what", [pytest.param(*c, id=_modes_k3_id(*c)) for c in MODES_K3])
def test_modes_k3_sweep(T, nu, M, Kc, off, K, mode, dead, what):
    """The MODES K3 row against the float64 blocks within the per-mode _row_gate; the reference without the first and the last local
    sample of every mode must miss it.  The fused K3 + K4 writes the split row and the split K4's U, action, stats and state, bit for
    bit, and that K4 agrees with modes_oracle.finalize of the row (check_modes_k4)."""
    case, cost, x, U = modes_k3_case(T, nu, M, Kc, off, K, mode, dead, seed=T * 7 + nu + M + Kc)
    ref, parts = modes_k3_restate(case, cost, x, U)
    gate = modes_k3_gate(case, cost, x, U, parts)
    state = mode_state(M, T, nu, M // 2, U[M // 2])
    split = run_modes_k3(case, cost, x, U, state, fused=False)
    fused = run_modes_k3(case, cost, x, U, state, fused=True)
    row = split[0]
    label = _modes_k3_id(T, nu, M, Kc, off, K, mode, dead, what)
    exc, line = _line(label, row, ref, gate)
    alt, _ = modes_k3_restate(case, cost, x, U, keep=drop_ends_mask(case))
    exc_alt, _ = row_excess(row, alt, gate)
    line += f", the reference without the first and last sample of every mode misses it by {exc_alt:.2e}"
    print(line)
    assert exc <= 0, line
    assert exc_alt > 0, line + ": the gate cannot tell the mode ends apart"
    blocks = row.reshape(M, -1)
    for m, (cols, S, w, b, xr) in enumerate(parts):                           # a mode without a valid local sample: (+inf, 0, 0)
        if not (w > 0).any():
            assert blocks[m, 0] == np.inf and blocks[m, 1] == 0 and (blocks[m, 2:] == 0).all(), f"mode {m}"
    if dead is not None:
        assert blocks[dead, 0] == np.inf and blocks[dead, 1] == 0
    for a, b_ in zip(split, fused):
        np.testing.assert_array_equal(a.view(np.uint32), b_.view(np.uint32))
    check_modes_k4(label, case.params, nu, row.reshape(1, -1), U, state, split[1:], require_decided=False)


# ------------------------------------------------------------------------------------------------------------------------------ modes K4
def sg_matrix(T):
    """The Savitzky-Golay filter of modes_oracle.savgol as a T x T matrix (T >= 9)."""
    S = np.zeros((T, T))
    for t in range(T):
        if t < 4:
            S[t, :9] = mo.SG_EDGE[t]
        elif t >= T - 4:
            S[t, T - 1 - np.arange(9)] = mo.SG_EDGE[T - 1 - t]
        else:
            S[t, t - 4:t + 5] = mo.SG_MID
    return S


def _filter_clip(p, nu, Un):
    T = int(p.T)
    lo = np.tile(np.array(p.u_min[:nu], np.float32), T).astype(np.float64)
    hi = np.tile(np.array(p.u_max[:nu], np.float32), T).astype(np.float64)
    return np.stack([np.clip(mo.savgol(u, T, nu) if p.filter_u else u, lo, hi) for u in Un])


def uncoupled(p, nu, rows, U):
    """A wrong K4: every mode takes its own step (k = I, no repulsion)."""
    M, NR = int(p.n_modes), int(p.T) * nu
    beta, eta, W = mo.combine(p, nu, rows)
    Uf = np.asarray(U, np.float32).astype(np.float64).reshape(M, int(p.T), nu)
    return _filter_clip(p, nu, Uf.reshape(M, NR) + mo.own_steps(p, Uf, eta, W)).reshape(U.shape)


def modes_k4_gate(p, nu, rows, U):
    """Element-wise bound on |U_kernel - U_oracle| of modes_rows, and (F, dF) of the free energies.

    Combining G rows: a scale exp(-(b_g - b) / lambda) carries eps (3 + (b_g - b) / lambda); eta and W add G roundings, so d_m is within
    rel_m sum_g s_g |W_g| / eta of W / eta (MEAN: the step_size_mean blend adds 4 eps).  V = Sigma^-1 U per step carries (nu + 1) eps
    |Sigma^-1| |U|, D_ij = sum_r dU_r dV_r (lane-strided, then a butterfly) (NR/32 + 8) eps sum |dU dV| plus |dU| dV.  The lower median
    moves at most max dD, so h within dh = max dD / ln(M + 1) + 3 eps h; k_ij = exp(-D_ij / h) within k (exp(dD/h + (D/h)(dh/h + 2 eps)
    + 2 eps) - 1).  The coupled step then carries these through its sums over j (M roundings each), the 2/h factor and the division by
    sum_j k_ij; Savitzky-Golay adds |SG| of that and 10 eps |SG| |u|, the clamp nothing, the float32 result eps |U|."""
    T, M = int(p.T), int(p.n_modes)
    NR, G = T * nu, rows.shape[0]
    lam, Kc = f32(p.lambda_), int(p.mode_samples)
    r = np.asarray(rows, np.float64).reshape(G, M, 2 + NR)
    Uf = np.asarray(U, np.float32).astype(np.float64).reshape(M, NR)
    beta, eta, W = mo.combine(p, nu, rows)
    ok = r[:, :, 1] > 0
    with np.errstate(invalid="ignore"):
        arg = np.where(ok, (r[:, :, 0] - np.where(np.isfinite(beta), beta, 0.0)[None]) / lam, 0.0)
    s = np.where(ok, np.exp(-arg), 0.0)
    rel = EPS * (G + 4 + arg.max(0))
    live = eta > 0
    A = np.einsum("gm,gmr->mr", s, np.abs(r[:, :, 2:])) / np.where(live, eta, 1.0)[:, None]
    d = mo.own_steps(p, Uf.reshape(M, T, nu), eta, W)
    dd = 2 * rel[:, None] * A + EPS * A
    if p.mode != MODE_SIMPLE:
        sm = f32(p.step_size_mean)
        dd = sm * dd + 4 * EPS * (np.abs(Uf) + sm * A)
    dd = np.where(live[:, None], dd, 0.0)
    F = mo.free_energy(p, beta, eta)
    with np.errstate(divide="ignore", invalid="ignore"):
        lnr = np.abs(np.log(np.where(live, eta, 1.0) / Kc))
        dF = np.where(live, lam * (2 * rel + 3 * EPS) + 3 * EPS * lam * lnr + 2 * EPS * np.abs(np.where(live, F, 0.0)), 0.0)
    sinv = np.array(p.sigma_inv[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu)
    U3 = Uf.reshape(M, T, nu)
    V = np.einsum("ab,mtb->mta", sinv, U3).reshape(M, NR)
    dV = (nu + 1) * EPS * np.einsum("ab,mtb->mta", np.abs(sinv), np.abs(U3)).reshape(M, NR)
    dU, dW = Uf[:, None] - Uf[None], V[:, None] - V[None]
    D = (dU * dW).sum(-1)
    dD = EPS * (NR / 32 + 10) * np.abs(dU * dW).sum(-1) + (np.abs(dU) * (dV[:, None] + dV[None])).sum(-1)
    np.fill_diagonal(D, 0.0)
    np.fill_diagonal(dD, 0.0)
    h = mo.bandwidth(D)
    if h > 0 and np.isfinite(h):
        dh = dD.max() / math.log(M + 1) + 3 * EPS * h
        assert dh < 0.25 * h, f"the bandwidth {h:.3e} is not resolved in float32 (within {dh:.2e})"
        k = np.exp(-D / h)
        dk = k * np.expm1(dD / h + (D / h) * (dh / h + 2 * EPS) + 2 * EPS)
        c2, dc2 = 2.0 / h, (2.0 / h) * (dh / (h - dh) + 2 * EPS)
    else:
        k, dk, c2, dc2 = np.ones((M, M)), np.zeros((M, M)), 0.0, 0.0
    ks = k.sum(1)
    dks = dk.sum(1) + M * EPS * ks
    absa1 = k @ np.abs(d)
    da1 = dk @ np.abs(d) + k @ dd + (M + 1) * EPS * absa1
    a2 = np.einsum("ij,ijr->ir", k, dU)
    absa2 = np.einsum("ij,ijr->ir", k, np.abs(dU))
    da2 = np.einsum("ij,ijr->ir", dk, np.abs(dU)) + (M + 2) * EPS * absa2
    num = k @ d + c2 * a2
    dnum = da1 + c2 * da2 + dc2 * absa2 + 2 * EPS * (absa1 + c2 * absa2)
    q = num / ks[:, None]
    un = Uf + q
    dun = (dnum + np.abs(q) * dks[:, None]) / ks[:, None] + EPS * (np.abs(q) + np.abs(un))
    if p.filter_u:
        S = np.abs(sg_matrix(T))
        dun = np.stack([(S @ dun[m].reshape(T, nu) + 10 * EPS * (S @ np.abs(un[m]).reshape(T, nu))).reshape(-1) for m in range(M)])
    out = _filter_clip(p, nu, un)
    return (dun + EPS * np.abs(out) + 1e-30).reshape(M, T, nu), F, dF


def selection_decided(F, dF, prev, margin):
    """True when float32 errors within dF cannot change the executed mode: the argmin is separated from every other F, and F_prev from
    F_a + margin."""
    fin = np.isfinite(F)
    if not fin.any():
        return True
    a = int(np.argmin(F))
    for j in np.flatnonzero(fin):
        if j != a and F[j] - F[a] <= dF[j] + dF[a]:
            return False
    if fin[prev] and prev != a:
        return abs(F[prev] - F[a] - margin) > dF[prev] + dF[a] + 2 * EPS * (abs(F[a]) + margin)
    return True


def run_k4(nu, p, rows, U, state):
    st = dev(state)
    be = backend(nu, p, st)
    Ud, act, stats = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(dev(rows), rows.shape[0], Ud, act, stats)
    torch.cuda.synchronize()
    out = [t.cpu().numpy() for t in (Ud, act, stats, st)]
    be.destroy()
    return out


def check_modes_k4(label, p, nu, rows, U, state0, got, require_decided=True):
    """got = (U, action, stats, state) of the device K4 on `rows` against modes_oracle.finalize within modes_k4_gate; the uncoupled K4
    must miss the gate.  Where the selection is decided (always with require_decided), the executed mode equals the oracle's; the state's
    U_exec and the action are the executed mode's U bit for bit, stats = (beta, eta) of that mode."""
    Ug, ag, sg, stg = got
    M, T = int(p.n_modes), int(p.T)
    Ur, _, _, st_r = mo.finalize(p, nu, rows, U, state0)
    gate, F, dF = modes_k4_gate(p, nu, rows, U)
    err = np.abs(Ug.astype(np.float64) - Ur)
    exc = float((err - gate).max())
    miss = float((np.abs(Ug.astype(np.float64) - uncoupled(p, nu, rows, U)) - gate).max())
    Fg = stg[1:1 + M].astype(np.float64)
    fin = np.isfinite(F)
    decided = selection_decided(F, dF, int(state0[0]), f32(p.mode_margin))
    print(f"MODES {label}-k4 worst |dU| {err.max():.2e} worst dU/gate {(err / gate).max():.3f} worst |dF| "
          f"{np.abs(Fg - F)[fin].max(initial=0):.2e} gate {dF[fin].max(initial=0):.2e}, the uncoupled reference misses by {miss:.2e}, "
          f"mode {int(stg[0])} (oracle {int(st_r[0])}{'' if decided else ', within float32 error of a tie'})")
    assert exc <= 0
    assert miss > 0, "the gate cannot tell the coupled step from the uncoupled one"
    np.testing.assert_array_equal(np.isfinite(Fg), fin)
    assert np.all(np.abs(Fg - F)[fin] <= dF[fin])
    assert decided or not require_decided, "the case is not decided away from float32 ties"
    if decided:
        assert stg[0] == st_r[0]
    pe = int(stg[0])
    np.testing.assert_array_equal(stg[1 + M:].view(np.uint32), Ug[pe].ravel().view(np.uint32))
    np.testing.assert_array_equal(ag.view(np.uint32), Ug[pe, 0].view(np.uint32))
    beta, eta, _ = mo.combine(p, nu, rows)
    assert sg[0] == np.float32(beta[pe]) and abs(float(sg[1]) - eta[pe]) <= (rows.shape[0] + 8) * EPS * eta[pe] * 4


def shard_rows(p, nu, T, M, G, rng):
    """G shard rows of mo.reduce over generated cost / x, the shards cutting the modes."""
    Kt = M * int(p.mode_samples)
    cost = rng.random((T, Kt)).astype(np.float32)
    x = (0.2 * rng.standard_normal((T, nu, Kt))).astype(np.float32)
    U = (0.15 * rng.standard_normal((M, T, nu))).astype(np.float32)
    cuts = [g * Kt // G for g in range(G + 1)]
    rows = np.stack([mo.reduce(p, nu, cost[:, a:b], x[:, :, a:b], U, k_offset=a) for a, b in zip(cuts[:-1], cuts[1:])])
    return rows, U


def crafted_rows(p, nu, G, b, e, rng):
    """Rows [G][M][2 + T*nu] with beta = b, eta = e (G, M) and W = eta times a random mean; eta = 0 gives (+inf, 0, 0)."""
    M, NR = int(p.n_modes), int(p.T) * nu
    rows = np.zeros((G, M, 2 + NR), np.float32)
    rows[:, :, 0] = np.where(e > 0, b, np.inf)
    rows[:, :, 1] = e
    rows[:, :, 2:] = e[:, :, None] * rng.normal(0.0, 0.2, (G, M, NR))
    return rows.reshape(G, -1)


# label: T, nu, M, G, mode, filter_u, how the rows and U are built
MODES_K4 = [
    ("T9-filter", 9, 3, 3, 2, "simple", True, "shards"),
    ("T10-filter", 10, 2, 2, 8, "halton-spline", True, "shards"),
    ("G1", 1, 7, 2, 1, "simple", False, "shards"),
    ("M16-G16", 32, 16, 16, MAX_PEERS, "simple", False, "shards"),             # the largest modes_fin_floats
    ("M16-G1-filter", 32, 16, 16, 1, "halton-spline", True, "shards"),
    ("M16-T256", 256, 2, 16, 2, "simple", True, "shards"),
    ("M3-G16", 12, 5, 3, MAX_PEERS, "simple", False, "shards"),
    ("coincident", 12, 3, 4, 2, "simple", True, "coincident"),                 # every D = 0: h = 0, k = 1
    ("coincident-majority", 16, 2, 5, 1, "simple", False, "clamped"),          # four modes at u_max: 6 of 10 pairs at D = 0
    ("ties", 10, 2, 5, 2, "simple", True, "ties"),                             # sorted D: a tie at 3, 4 ends at the lower median
    ("dead-executed", 9, 3, 3, 2, "halton-spline", True, "dead"),
    ("margin-inside", 12, 3, 3, 1, "simple", False, "inside"),                 # F_prev - F_a = margin (1 - 1e-3): kept
    ("margin-outside", 12, 3, 3, 1, "simple", False, "outside"),               # F_prev - F_a = margin (1 + 1e-3): switched
    ("margin-met", 12, 3, 3, 1, "simple", False, "met"),                       # F_prev = F_a + margin exactly in float32: kept
    ("margin-missed", 12, 3, 3, 1, "simple", False, "missed"),                 # F_prev one float32 step above it: switched
]
MARGIN_EXACT = 0.0625                                                          # F_a = 1, F_prev = 1.0625: every value exact in float32
TIES_C = [0, 1, 2, 3, 7]                                                       # |c_i - c_j|^2 sorted: 1 1 1 4 4 | 9 16 25 36 49


def modes_k4_inputs(T, nu, M, G, mode, filt, how, seed):
    rng = np.random.default_rng(seed)
    Kc = 64 * G
    kw = dict(noise_sigma=(0.25 * np.eye(nu)).tolist()) if how == "ties" else {}             # Sigma^-1 = 4 I, exact
    p = mparams(nu, T, M * Kc, M, mppi_mode=mode, filter_u=filt, rollout_var_discount=0.9, u_min=[-0.5], u_max=[0.5],
                mode_switch_margin=MARGIN_EXACT if how in ("met", "missed") else 0.05, **kw)
    prev = M - 1
    if how == "shards":
        rows, U = shard_rows(p, nu, T, M, G, rng)
        return p, rows, U, mode_state(M, T, nu, prev, U[prev])
    b = rng.uniform(0.0, 2.0, (G, M)).astype(np.float32)
    e = rng.uniform(0.2, 1.0, (G, M)).astype(np.float32) * Kc / G
    U = (0.15 * rng.standard_normal((M, T, nu))).astype(np.float32)
    if how == "coincident":
        U[:] = U[0]
    elif how == "clamped":
        U[:4] = 0.5
    elif how == "ties":                                                        # U_m = c_m / 16 at (t, j) = (0, 0): D_ij = (c_i - c_j)^2 / 64 exactly
        U[:] = 0.0
        U[:, 0, 0] = np.array(TIES_C, np.float32) / 16
    elif how == "dead":
        prev = 1
        e[:, 1] = 0.0
    elif how in ("inside", "outside"):                                         # eta = Kc: F = beta exactly (logf(1) = 0)
        prev = 2
        e[:] = Kc
        b[0] = [1.0, 2.0, 1.0 + 0.05 * (1 - 1e-3 if how == "inside" else 1 + 1e-3)]
    elif how in ("met", "missed"):                                             # F_prev - F_a = margin exactly, or one float32 step more
        prev = 2
        e[:] = Kc
        top = np.float32(1.0 + MARGIN_EXACT)
        b[0] = [1.0, 2.0, top if how == "met" else np.nextafter(top, np.float32(np.inf))]
    return p, crafted_rows(p, nu, G, b, e, rng), U, mode_state(M, T, nu, prev, U[prev])


@pytest.mark.parametrize("label,T,nu,M,G,mode,filt,how", [pytest.param(*c, id=f"modes-k4-{c[0]}-T{c[1]}nu{c[2]}-M{c[3]}-G{c[4]}") for c in MODES_K4])
def test_modes_k4_against_float64(label, T, nu, M, G, mode, filt, how):
    p, rows, U, state0 = modes_k4_inputs(T, nu, M, G, mode, filt, how, seed=T * M + G)
    """modes_rows against modes_oracle.finalize within modes_k4_gate (check_modes_k4), and per construction: h = 0 for coincident modes;
    the lower median where a tie ends at it (a reference with the upper median misses the gate); a dead executed mode is left; the margin
    met exactly keeps the executed mode, one float32 step more switches it."""
    p, rows, U, state0 = modes_k4_inputs(T, nu, M, G, mode, filt, how, seed=T * M + G)
    got = run_k4(nu, p, rows, U, state0)
    exact_tie = how in ("met", "missed")                                       # decided by the float32 comparison itself, not away from it
    check_modes_k4(f"modes-k4-{label}-T{T}nu{nu}-M{M}-G{G}", p, nu, rows, U, state0, got, require_decided=not exact_tie)
    Ur, _, _, st_r = mo.finalize(p, nu, rows, U, state0)
    Fg = got[3][1:1 + M]
    if how in ("coincident", "clamped"):
        assert mo.bandwidth(mo.distances(U.astype(np.float64), np.eye(nu))) == 0.0
    if how == "dead":
        assert st_r[0] != 1 and np.isinf(got[3][2])                            # the dead executed mode is left
    if how == "ties":
        sinv = np.array(p.sigma_inv[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu)
        v = np.sort(mo.distances(U.astype(np.float64), sinv)[np.triu_indices(M, 1)])
        lo = (v.size - 1) // 2
        assert v[lo - 1] == v[lo] < v[lo + 1]
        gate, _, _ = modes_k4_gate(p, nu, rows, U)
        U_up = mo.finalize(p, nu, rows, U, state0, h=v[lo + 1] / math.log(M + 1))[0]
        miss = float((np.abs(got[0].astype(np.float64) - U_up) - gate).max())
        print(f"MODES modes-k4-{label} the reference with the upper median misses the gate by {miss:.2e}")
        assert miss > 0
    if how in ("inside", "met"):
        assert got[3][0] == st_r[0] == 2
    if how in ("outside", "missed"):
        assert got[3][0] == st_r[0] == 0
    if exact_tie:                                                              # F = beta bit for bit, so the tie is the kernel's own
        np.testing.assert_array_equal(Fg, rows.reshape(M, -1)[:, 0])
        assert (Fg[2] == np.float32(Fg[0] + np.float32(MARGIN_EXACT))) == (how == "met")


# ------------------------------------------------------------------------------------------------------------------------------ modes shift
@pytest.mark.parametrize("T,nu", [(1, 1), (12, 3), (32, 16)])
@pytest.mark.parametrize("M", [2, 16])
def test_modes_shift(M, T, nu):
    p = mparams(nu, T, M * 32, M, u_init=np.linspace(-0.2, 0.3, nu).tolist())
    rng = np.random.default_rng(M + T)
    U0 = rng.uniform(-1, 1, (M, T, nu)).astype(np.float32)
    U, ctr = dev(U0), torch.tensor([7], dtype=torch.int32, device=DEV)
    be = backend(nu, p, dev(mode_state(M, T, nu)))
    be.shift(U, ctr)
    torch.cuda.synchronize()
    want = mo.shift(p, nu, U0)
    np.testing.assert_array_equal(U.cpu().numpy().view(np.uint32), want.view(np.uint32))
    assert int(ctr[0]) == 8
    assert not np.array_equal(want, U0)
    be.destroy()


# ------------------------------------------------------------------------------------------------------------------------------ anneal K1
AK1_CELLS = [(1, 1), (7, 30), (16, 32), (2, 256)]                              # (nu, T): T*nu = 512 at (16, 32) and (2, 256), T = 256


def _anneal_k1_cases():
    out, i = [], 0
    for nu, T in AK1_CELLS:
        for variant in ("random", "colored"):
            for ctr in ("first", "last", "past"):
                N, R = [2, 16][i % 2], [1, 2, 32][i % 3]
                i += 1
                out.append(pytest.param(variant, T, nu, N, ctr, R, id=f"anneal-k1-{variant}-T{T}nu{nu}-N{N}-{ctr}-R{R}"))
    return out


def anneal_schedule_with_floor(N, T, row, seed):
    """(s, r) float32 (N, T): s uniform in [0.5, 1], except s[row][t0] = 2^-20 (r = 2^40), the smallest scale accepted."""
    rng = np.random.default_rng(seed)
    s = rng.uniform(0.5, 1.0, (N, T))
    t0 = int(rng.integers(T))
    s[row, t0] = ANNEAL_MIN_SCALE
    s = s.astype(np.float32)
    r = (1.0 / (s.astype(np.float64) ** 2)).astype(np.float32)
    assert r[row, t0] == 2.0 ** 40
    return s, r, t0


def anneal_k1_reference(p, nu, T, K, R, U, s_row, Lt):
    """(actions, noise, |colour| magnitude) of ao.sample; with n_worlds = R on the control samples, repeated R times along k."""
    cp = ro.control_params(p) if R > 1 else p
    model = nu_model(nu)
    a, n = ao.sample(model, cp, SEED, PLAN, U, 0, K // R, s_row, Lt=Lt)
    z = np.abs(ao.co.white(model, cp, SEED, PLAN, 0, K // R).astype(np.float64))
    if Lt is not None:
        z = np.einsum("ts,sik->tik", np.abs(Lt.astype(np.float64)), z)
    L = np.abs(np.array(p.sigma_chol[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu))
    mag = np.einsum("ji,tik->tjk", L, z) * np.asarray(s_row, np.float64)[:, None, None]
    rep = lambda v: np.repeat(v, R, axis=-1)
    return rep(a), rep(n), rep(mag)


@pytest.mark.parametrize("variant,T,nu,N,ctr,R", _anneal_k1_cases())
def test_anneal_k1_sweep(variant, T, nu, N, ctr, R):
    """K1 with the row min(counter, N - 1) of a schedule holding 2^-20, keyed by the control sample with n_worlds = R, against the
    float64 reference within the bound of test_gpu_anneal (colour sums, scale, the sum with U and the final rounding); the reference
    with the neighbouring schedule row must miss it."""
    K = 1024
    counter = {"first": 0, "last": N - 1, "past": N + 3}[ctr]
    row = min(counter, N - 1)
    kw = dict(n_worlds=R, cvar_alpha=0.5) if R > 1 else {}
    p = mparams(nu, T, K, sampling_method=variant, u_min=[-0.6], u_max=[0.6], **kw)
    s, r, t0 = anneal_schedule_with_floor(N, T, row, seed=T * nu + N + R)
    rng = np.random.default_rng(T + nu)
    U = (0.2 * rng.standard_normal((T, nu))).astype(np.float32)
    Lt = colored_noise_chol(T, 2.0) if variant == "colored" else None
    state = dev(ao.make_state(s, r, counter=float(counter)))
    be = backend(nu, p, anneal=state, N=N)
    a, n = k1_run(be, variant, T, nu, K, 0, K, dev(U))
    be.destroy()
    ar, nr, mag = anneal_k1_reference(p, nu, T, K, R, U, s[row], Lt)
    nsum = nu + (T if Lt is not None else 0) + 1
    bound = EPS * (nsum * mag + 2.0 * np.abs(U)[:, :, None] + 2.0 * np.abs(ar)) + 1e-30
    err = np.abs(a.astype(np.float64) - ar)
    nb = row - 1 if row > 0 else row + 1
    a_bad, _, _ = anneal_k1_reference(p, nu, T, K, R, U, s[nb], Lt)
    miss = float((np.abs(a.astype(np.float64) - a_bad) - bound).max())
    print(f"MODES anneal-k1-{variant}-T{T}nu{nu}-N{N}-ctr{counter}-R{R}-K{K} worst {err.max():.2e} worst err/gate {(err / bound).max():.3f}, "
          f"the reference with row {nb} misses it by {miss:.2e}")
    assert np.all(err <= bound)
    assert np.all(np.abs(n.astype(np.float64) - nr) <= 2 * bound)
    assert miss > 0
    assert float(state[0]) == counter                                          # K1 reads the counter, it does not move it
    if R > 1:
        np.testing.assert_array_equal(a.reshape(T, nu, -1, R), np.broadcast_to(a[:, :, ::R, None], (T, nu, K // R, R)))


# ------------------------------------------------------------------------------------------------------------------------------ anneal K3
AK3_CELLS = [(30, 4), (30, 7), (32, 16)]                                        # RPL 4, 8, 16
AK3_R = [2, 8, 32]


def _anneal_k3_cases():
    out, i = [], 0
    for T, nu in AK3_CELLS:
        for name_i in range(4):                                                # ragged, sms-, sms+, wrap
            R = AK3_R[i % 3]
            m = [1, R // 2, R][(i // 3) % 3]
            mode = ["simple", "halton-spline"][i % 2]
            ctr = (i + i // 3) % 3                                             # every (R, row) and (m, row) pair over 9 cases
            i += 1
            name, K = _risk_Ks(T, nu, "fixed", R)[1 + name_i]
            rpl, ncons, nstage, _ = ws_layout(T, nu, "W")
            out.append(pytest.param(T, nu, K, R, m, mode, ctr,
                                    id=f"anneal-k3-RPL{rpl}-T{T}nu{nu}-ncons{ncons}-R{R}m{m}-{name}K{K}-ctr{ctr}-{'simple' if mode == 'simple' else 'mean'}"))
        name, K = _risk_Ks(T, nu, "fixed", 1)[4]
        rpl, ncons, _, _ = ws_layout(T, nu, "W")
        out.append(pytest.param(T, nu, K, 1, 1, "simple", 2, id=f"anneal-k3-RPL{rpl}-T{T}nu{nu}-ncons{ncons}-R1-{name}K{K}-ctr2-simple"))
    return out


def anneal_k3_case(T, nu, K, R, m, mode, seed):
    kw = dict(n_worlds=R, cvar_alpha=m / R) if R > 1 else {}
    case = make_case(T, nu, K, mode=mode, **kw)
    cost, x, U = k3_inputs(case, seed=seed)
    rng = np.random.default_rng(seed)
    if R > 1 and K // R >= 4:                                                  # +inf: one rollout of one group, the m worst worlds of another
        g1, g2 = rng.choice(K // R - 2, 2, replace=False)
        cost[rng.integers(T), g1 * R + rng.integers(R)] = np.inf
        cost[0, g2 * R + R - m:g2 * R + R] = np.inf
    return case, cost, x, U


def anneal_restate(case, cost, x, U, r_row, params=None):
    """float64 annealed K3 (ao.scores, then the CVaR score with n_worlds > 1): (S per rollout, score, w, beta, x columns, row)."""
    p = params or case.params
    T, nu, R = case.T, case.nu, int(case.params.n_worlds)
    with np.errstate(invalid="ignore"):
        S, lam = ao.scores(p, nu, cost, x, U, r_row)
    xr = np.asarray(x, np.float64).reshape(T * nu, -1)
    sc = S
    if R > 1:
        sc, xr = ro.rho(S, R, int(case.params.risk_tail)), xr[:, ::R]
    ok = np.isfinite(sc)
    b = sc[ok].min() if ok.any() else np.inf
    w = np.where(ok, np.exp(-(np.where(ok, sc, b) - b) / lam), 0.0)
    return S, sc, w, b, xr, np.concatenate([[b, w.sum()], xr @ w])


def anneal_gate(case, cost, x, U, r_row, S, sc, w, b, xr):
    """_row_gate with k3_dS of g = lambda r[t] Sigma^-1 U (U scaled by r, plus the rounding of the r product), and under RISK the CVaR
    score's m-term tail sum (risk_gate of test_gpu_mode_shapes)."""
    T, nu, K, lam = case.T, case.nu, case.K, case.lam
    R, m = int(case.params.n_worlds), int(case.params.risk_tail)
    Ur = np.asarray(U, np.float64) * (np.asarray(r_row, np.float64)[:, None] if case.simple else 1.0)
    with np.errstate(invalid="ignore"):
        dS = k3_dS(case, cost, x, Ur)
        if case.simple:
            gabs = lam * (np.abs(Ur) @ np.abs(case.sinv().astype(np.float64)).T).reshape(-1)
            dS = dS + EPS * (gabs @ np.abs(np.asarray(x, np.float64).reshape(T * nu, K)))
    _, ncons, _, _ = ws_layout(T, nu, "W")
    if R > 1:
        Sg = np.where(np.isfinite(S), S, np.inf).reshape(-1, R)
        top = np.abs(-np.sort(-Sg, axis=1)[:, :m])
        with np.errstate(invalid="ignore"):
            dS = dS.reshape(-1, R).max(1) + (m + 2) * EPS * np.where(np.isfinite(top), top, 0).mean(1)
    return _row_gate(sc, dS, w, b, xr, lam, K, ncons)[0]


@pytest.mark.parametrize("T,nu,K,R,m,mode,ctr", _anneal_k3_cases())
def test_anneal_k3_sweep(T, nu, K, R, m, mode, ctr):
    """The annealed K3 row (schedule row `ctr` of N = 3, with r = 2^40 at one step, where U is 2^-40 times its size) against the float64
    row within its gate; negative control: the reference with the neighbouring r row (SIMPLE) misses it.  MEAN mode (halton-spline)
    scores no U term for r to scale, so its control is the reference that scores with SIMPLE mode's r-scaled importance term; it misses
    the gate by far (it shows that r is not applied there, not how tight the gate is).  The split K3 leaves the counter, the fused tail writes the same
    row and the split K4's U and action, bit for bit, and advances it by one."""
    N = 3
    case, cost, x, U = anneal_k3_case(T, nu, K, R, m, mode, seed=31 * T + nu + K + R)
    s, r, t0 = anneal_schedule_with_floor(N, T, ctr, seed=T + K)
    if case.simple:
        U[t0] = (U[t0].astype(np.float64) * 2.0 ** -40).astype(np.float32)     # r U stays of the size of the other steps
    S, sc, w, b, xr, ref = anneal_restate(case, cost, x, U, r[ctr])
    gate = anneal_gate(case, cost, x, U, r[ctr], S, sc, w, b, xr)
    outs = []
    for fused in (False, True):
        st = dev(ao.make_state(s, r, counter=float(ctr)))
        be = backend(nu, case.params, anneal=st, N=N)
        part, Ud = torch.zeros(2 + T * nu, device=DEV), dev(U)
        act, stats = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
        if fused:
            be.reduce_finalize(dev(cost), dev(x), Ud, part, act, stats)
        else:
            be.reduce(dev(cost), dev(x), Ud, part)
            torch.cuda.synchronize()
            assert float(st[0]) == ctr                                         # the split K3 does not move the counter
            be.finalize(part.view(1, -1), 1, Ud, act, stats)
        torch.cuda.synchronize()
        assert float(st[0]) == ctr + 1
        outs.append([t.cpu().numpy() for t in (part, Ud, act, stats)])
        be.destroy()
    for a_, b_ in zip(*outs):
        np.testing.assert_array_equal(a_.view(np.uint32), b_.view(np.uint32))
    row = outs[0][0]
    label = f"anneal-k3-T{T}nu{nu}-R{R}m{m}-K{K}-ctr{ctr}-{mode}"
    exc, line = _line(label, row, ref, gate)
    if case.simple:
        nb = ctr - 1 if ctr > 0 else ctr + 1
        alt = anneal_restate(case, cost, x, U, r[nb])[-1]
        what = f"r row {nb}"
    else:
        ps = copy.copy(case.params)
        ps.mode = MODE_SIMPLE
        alt = anneal_restate(case, cost, x, U, r[ctr], params=ps)[-1]
        what = "r applied"
    exc_alt, _ = row_excess(row, alt, gate)
    line += f", the reference with {what} misses it by {exc_alt:.2e}"
    print(line)
    assert exc <= 0, line
    assert exc_alt > 0, line + ": the gate cannot tell the schedule row apart"


# ------------------------------------------------------------------------------------------------------------------------------ anneal plan
def test_anneal_c2_shape_plans_agree_with_the_oracle_pipeline():
    """Panda reach at the C2 shape (T = 30, nu = 7: RPL 8, K = 2048) with anneal_iterations = 3, closed loop over three plans, graph on,
    against the same planner on the ``AnnealOracleBackend``."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from scenes import panda_cfg
    N = 3
    mk = lambda d: panda_cfg(K=2048, T=30, device=d, anneal_iterations=N, anneal_iter_decay=0.7, anneal_horizon_decay=0.9)
    gpu = MPPIisaacPlanner(mk(DEV), PandaReachObjective(), use_cuda_graph=True)
    cpu = MPPIisaacPlanner(mk("cpu"), PandaReachObjective(), backend=ao.AnnealOracleBackend(nthreads=8))
    q = np.array([0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0])
    qd = np.zeros_like(q)
    lim = float(gpu.mppi.backend.params.u_max[0])
    for it in range(3):
        ag, ac = gpu.compute_action(q, qd), cpu.compute_action(q, qd)
        err = float((ag.cpu() - ac).abs().max())
        print(f"MODES anneal-c2-plan{it} worst |da| {err:.2e} gate {2e-4 * max(1.0, lim):.2e}")
        assert err <= 2e-4 * max(1.0, lim), f"plan {it}"
        assert float(gpu.mppi.anneal_state[0]) == N
        q = q + 0.05 * ac.numpy(); qd = ac.numpy()
    assert gpu.mppi._graph is not None
    np.testing.assert_allclose(gpu.mppi.U.cpu().numpy(), cpu.mppi.U.numpy(), rtol=0, atol=2e-4 * max(1.0, lim))
