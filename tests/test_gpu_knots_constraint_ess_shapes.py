"""-m gpu: the kernels of spline MPPI (``control_knots``), constrained MPPI (``constraint_mode: feasible_first``) and the ESS-targeted
temperature (``lambda_mode: ess``) over every template instantiation and the accepted shape range, against the float64 references
``knots_oracle``, ``constraint_oracle`` and ``temperature_oracle``, on the generated cases of ``synth_mppi`` (the point robot's model with
nu set; no dynamics run).

* knots K1 (``mppib_sample_spline``) within the knot and interpolation bound of ``test_gpu_knots``, shards cut inside a tile bit for bit,
  the null row only in the shard that owns global K - 1, and actions inside the bounds;
* knots K3 (PLAIN rule over P*nu control rows and T cost rows, RPL 4 / 8 / 16, up to T = 256, P*nu = 512) within ``k3_gate(Tc = P)``;
  K4's theta and U_exec = B theta within the row's gate carried through the update and B; fused equals split; the shift;
* constrained K3 (FEASIBLE rule, RPL 4 / 8 / 16, up to the longest accepted horizons) with the feasible samples placed where the
  feasibility-first merge of tiles, warps, CTAs and shards can go wrong, within ``_row_gate`` of the regime that applies; the
  explicit-row K4 over G shard rows;
* the ESS pass at its own tile, half-tile and persistent-grid boundaries, the rule on the device's curve, and K3 / K4 at the chosen lambda
  (fixed, diagonal and full Sigma) within ``k3_gate``.

Each gate has a negative control, a deliberately wrong reference that must miss it.  Each case prints a ``SHAPES <id> worst |err| ...
worst err/gate ... gate ...`` line (shown with -s)."""
import dataclasses
import math

import numpy as np
import pytest
import torch

import adaptive_full_oracle as afo
import constraint_oracle as cn
import knots_oracle as ko
import temperature_oracle as tmo
from mppi_isaac_b200.model.blob import ESS_GRID, ESS_STATE_FLOATS, ess_grid, make_params, spline_basis, spline_table
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from synth_mppi import (EPS, NUM_SMS, WS_W, drop_tail_mask, k3_dS, k3_gate, k3_inputs, k3_restate, make_case, nu_model, row_excess, v_dS,
                        wrap_K, ws_layout)
from test_gpu_mode_shapes import _row_gate

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED, PLAN = 7, 3
U_RO = 2.0 ** -24                                                              # unit roundoff: the K1 bound of test_gpu_knots


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def backend(nu, p):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(nu_model(nu), p)
    return be


def excess(got, ref, gate):
    """row_excess over the flattened arrays."""
    return row_excess(*(np.asarray(v, np.float64).ravel() for v in (got, ref, gate)))


def line(label, got, ref, gate, extra=""):
    """(excess, the SHAPES line) of one gated comparison."""
    exc, err = excess(got, ref, gate)
    got, ref, gate = (np.asarray(v, np.float64).ravel() for v in (got, ref, gate))
    fin = np.isfinite(gate) & (gate > 0) & np.isfinite(ref)
    ratio = float((np.abs(got - ref)[fin] / gate[fin]).max(initial=0.0))
    return exc, f"SHAPES {label} worst |err| {err:.2e} worst err/gate {ratio:.3f} gate {float(gate[fin].max(initial=0.0)):.2e}{extra}"


def k_regimes(T, nu, **layout):
    """The K3 K regimes (multiples of 4): one CTA, a ragged last tile, one tile per SM minus / plus one, every CTA past three rings."""
    return {"gx1": 28, "ragged": WS_W * 37 + 4, "sms-": WS_W * NUM_SMS - 32, "sms+": WS_W * NUM_SMS + 32, "wrap": wrap_K(T, nu, "W", **layout)}


def mean_update(row, gate, U, simple, a):
    """K4's update from a row within `gate` of the float64 `row`: (U' in float64, its bound).  The kernel divides its own float32 W by
    its own eta, so W / eta moves by at most (|dW| + |W / eta| d_eta) / (eta - d_eta), plus the division's and the update's roundings."""
    e, W, de, dW = row[1], row[2:], gate[1], gate[2:]
    m = W / e
    dm = (dW + np.abs(m) * de) / (e - de) + 2 * EPS * np.abs(m)
    U = np.asarray(U, np.float64).ravel()
    if simple:
        new = U + m
        return new, dm + EPS * (np.abs(U) + np.abs(new))
    new = (1.0 - a) * U + a * m
    return new, a * dm + 2 * EPS * (np.abs(U) + np.abs(a * m) + np.abs(new))


# ======================================================================================================================== knots
def kparams(nu, T, K, P, d, mode="simple", gamma=0.95, **kw):
    return make_case(T, nu, K, mode=mode, gamma=gamma, control_knots=P, spline_degree=d, **kw)


# ---- K1
# (T, nu, P, d): d = 1, 2, 3 at P = d + 1 and at P = T; P*nu = 128 | 129, 256 | 258, 512 at T = 256; the T*nu = 4096 corner
K1_CELLS = [(2, 1, 2, 1), (9, 3, 3, 2), (9, 2, 4, 3), (9, 5, 9, 1), (9, 1, 9, 2), (9, 16, 9, 3), (256, 1, 2, 1), (256, 1, 128, 1),
            (256, 1, 129, 2), (256, 2, 128, 3), (256, 3, 86, 2), (256, 16, 32, 3)]
K1_KS = [1, 31, 32, 33, 1000, 65536]


def _k1_cases():
    out = []
    for i, (T, nu, P, d) in enumerate(K1_CELLS):
        big = T * nu * 1000 > 2_000_000                                        # the float64 action reference is T*nu*K doubles
        Ks = [1000] if T * nu >= 4096 else K1_KS if not big else [31, 33, 1000]
        for K in Ks:
            if T * nu * K > 10_000_000:
                continue
            out.append(pytest.param(T, nu, P, d, K, id=f"k1-T{T}nu{nu}-P{P}d{d}-K{K}"))
    return out


def spline_k1(nu, p, theta, k_offset=0, k_total=None):
    be = backend(nu, p)
    be.set_spline(dev(spline_table(p.T, p.control_knots, p.spline_degree, nu, theta)))
    K, T, P = p.K, p.T, p.control_knots
    a, x = torch.zeros((T, nu, K), device=DEV), torch.zeros((P, nu, K), device=DEV)
    be.sample_spline(SEED, PLAN, k_offset, k_total or K, dev(theta), a, x)
    torch.cuda.synchronize()
    be.destroy()
    return a.cpu().numpy(), x.cpu().numpy()


def k1_params(nu, T, K, P, d, k_offset=0):
    p = make_params(MPPIConfig(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.3 * np.eye(nu) + 0.05).tolist(),
                               u_min=[-0.6], u_max=[0.6], lambda_=0.05, sample_null_action=True, control_knots=P, spline_degree=d),
                    IsaacGymConfig(), nu, K, [])
    return p


@pytest.mark.parametrize("T,nu,P,d,K", _k1_cases())
def test_knots_k1_sweep(T, nu, P, d, K):
    """Knots |theta~ - ref| <= 2 eps ((nu + 1) |L||z| + 2 |theta| + 2 |ref|), actions the knots' bound carried through B plus
    eps (d + 2) |B| |theta~|.  Some knots sit at the bounds (theta = +-0.6): the actions stay inside [u_min, u_max].  Negative control:
    the reference interpolated with the basis of degree d + 1 (d - 1 where P = d + 1) misses the action bound."""
    p = k1_params(nu, T, K, P, d)
    rng = np.random.default_rng(T * 31 + nu * 7 + P + d)
    th = (0.3 * rng.standard_normal((P, nu))).astype(np.float32)
    th[0, 0], th[-1, -1] = 0.6, -0.6                                            # knots at the bounds
    a, x = spline_k1(nu, p, th)
    model = nu_model(nu)
    ar, xr, tr = ko.sample(model, p, SEED, PLAN, th, 0, K)
    z = np.abs(ko.co.white(model, ko.knot_params(p), SEED, PLAN, 0, K).astype(np.float64))
    L = np.abs(np.array(p.sigma_chol[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu))
    kb = U_RO * ((nu + 1) * np.einsum("ji,pik->pjk", L, z) + 2.0 * np.abs(th)[:, :, None] + 2.0 * np.abs(tr)) + 1e-30
    B = spline_basis(T, P, d)[0]
    ab = np.einsum("tp,pjk->tjk", B, kb + U_RO * (d + 2) * np.abs(tr)) + 1e-30
    label = f"k1-T{T}nu{nu}-P{P}d{d}-K{K}"
    exc_x, _ = line(label, x, xr, 2 * kb)
    exc, msg = line(label, a, ar, ab)
    d2 = d + 1 if P >= d + 2 and d < 3 else d - 1
    if d2 >= 1 and K > 1:                                                      # K = 1: the null row alone, zero at every degree
        B2 = spline_basis(T, P, d2)[0]
        lo, hi = np.float32(-0.6), np.float32(0.6)
        alt = np.minimum(np.maximum(np.einsum("tp,pjk->tjk", B2, tr), lo), hi)
        exc_alt, _ = excess(a, alt, ab)
        msg += f", the degree-{d2} interpolation misses it by {exc_alt:.2e}"
    else:
        exc_alt = None                                                         # P = 2, d = 1: no other degree has two knots
    print(msg)
    assert exc_x <= 0 and exc <= 0, msg
    if exc_alt is not None:
        assert exc_alt > 0, msg + ": the gate cannot tell the degree"
    assert np.all((a >= np.float32(-0.6)) & (a <= np.float32(0.6)))
    assert np.all(a[:, :, K - 1] == 0.0) and np.all(x[:, :, K - 1] == -th)   # the null row: every knot clamp(0) = 0


@pytest.mark.parametrize("T,nu,P,d", [(9, 3, 3, 2), (256, 1, 129, 2), (64, 16, 32, 3)])
def test_knots_k1_shards(T, nu, P, d):
    """Shards cut inside 32-sample tiles equal the whole launch bit for bit; the null row is global K - 1: only the last shard has one."""
    K = 1000
    th = (0.2 * np.random.default_rng(T + P).standard_normal((P, nu))).astype(np.float32)
    a, x = spline_k1(nu, k1_params(nu, T, K, P, d), th)
    cuts = [0, 45, 333, K]                                                      # 45, 333: inside tiles 1 and 10
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        sa, sx = spline_k1(nu, k1_params(nu, T, hi - lo, P, d), th, lo, K)
        np.testing.assert_array_equal(sa.view(np.uint32), a[:, :, lo:hi].view(np.uint32))
        np.testing.assert_array_equal(sx.view(np.uint32), x[:, :, lo:hi].view(np.uint32))
        owns = hi == K
        assert bool(np.all(sa[:, :, -1] == 0.0)) == owns                    # a shard without global K - 1 has no null row
    print(f"SHAPES k1-shards-T{T}nu{nu}-P{P}d{d} worst |err| 0 worst err/gate 0.000 gate 0 (bit for bit over cuts {cuts})")


# ---- K3 + K4 + shift
# (T, nu, P, d): P*nu = 1*nu, 128 | 129 (RPL 4 | 8), 256 | 258 (RPL 8 | 16), 512 at T = 2, 9, 256; P = d + 1 and P = T; the corner
# T = 256, nu = 16, P = 32, d = 3 (T*nu = 4096, the largest ring)
K3_CELLS = [(2, 1, 2, 1), (9, 3, 3, 2), (9, 2, 9, 3), (9, 16, 8, 1), (9, 16, 9, 2), (256, 1, 4, 3), (256, 1, 128, 1), (256, 1, 129, 2),
            (256, 2, 128, 3), (256, 2, 129, 1), (256, 4, 128, 2), (256, 2, 256, 1), (256, 16, 32, 3)]
GAMMAS = [0.5, 0.95, 1.05]


def _knots_k3_cases():
    out, i = [], 0
    for T, nu, P, d in K3_CELLS:
        rpl, ncons, nstage, _ = ws_layout(T, nu, "W", Tc=P)
        for name, K in k_regimes(T, nu, Tc=P).items():
            if P * nu * K > 12_000_000 and name == "wrap":                      # the largest cells stay at K <= ~4k
                continue
            mode = ["simple", "halton-spline"][i % 2]
            g = GAMMAS[(i // 2) % 3]
            i += 1
            tag = "simple" if mode == "simple" else f"g{g:g}"
            out.append(pytest.param(T, nu, P, d, K, mode, g,
                                    id=f"knots-RPL{rpl}-T{T}nu{nu}-P{P}d{d}-ncons{ncons}s{nstage}-{name}K{K}-{tag}"))
    return out


def run_knots(case, cost, x, th, fused):
    """(row, theta', action, U_exec) of K3 + K4 on a fresh handle and table."""
    p, nu, T = case.params, case.nu, case.T
    be = backend(nu, p)
    table = dev(spline_table(T, p.control_knots, p.spline_degree, nu, th))
    be.set_spline(table)
    part = torch.zeros(2 + case.Tc * nu, device=DEV)
    Ud, act, st = dev(th), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    if fused:
        be.reduce_finalize(dev(cost), dev(x), Ud, part, act, st)
    else:
        be.reduce(dev(cost), dev(x), Ud, part)
        be.finalize(part.view(1, -1), 1, Ud, act, st)
    torch.cuda.synchronize()
    out = [part.cpu().numpy(), Ud.cpu().numpy(), act.cpu().numpy(), table[-T * nu:].cpu().numpy().reshape(T, nu)]
    Us = Ud.clone()
    be.shift(Us, None)
    torch.cuda.synchronize()
    out.append(Us.cpu().numpy())
    be.destroy()
    return out


@pytest.mark.parametrize("T,nu,P,d,K,mode,gamma", _knots_k3_cases())
def test_knots_k3_k4_sweep(T, nu, P, d, K, mode, gamma):
    """The row within k3_gate(Tc = P); the reference without the last (ragged, favoured) tile misses it.  theta' within the row's gate
    carried through the update, U_exec = B theta' within that carried through B plus eps (d + 2) |B| |theta'|; U_exec from the
    un-updated theta misses it.  action = theta'_0 = U_exec[0] bit for bit; fused = split bit for bit; the shift against ko.shift,
    u_init where the shifted Greville abscissa leaves the horizon."""
    case = kparams(nu, T, K, P, d, mode, gamma, u_init=0.25)
    assert case.Tc == P
    cost, x, th = k3_inputs(case, seed=T * 13 + nu + P * 3 + d + K)
    S, w, ref = k3_restate(case, cost, x, th)
    gate = k3_gate(case, cost, x, th, S, w)
    split = run_knots(case, cost, x, th, fused=False)
    fused = run_knots(case, cost, x, th, fused=True)
    rpl, ncons, nstage, _ = ws_layout(T, nu, "W", Tc=P)
    label = f"knots-RPL{rpl}-T{T}nu{nu}-P{P}d{d}-ncons{ncons}s{nstage}-K{K}-{mode}"
    exc, msg = line(label, split[0], ref, gate)
    _, _, alt = k3_restate(case, cost, x, th, keep=drop_tail_mask(K))
    exc_alt, _ = excess(split[0], alt, gate)
    msg += f", without the last tile {exc_alt:.2e} over"
    # K4: theta' and U_exec
    a = float(np.float32(case.params.step_size_mean))
    th2, dth = mean_update(ref, gate, th, case.simple, a)
    B = spline_basis(T, P, d)[0]
    ue_ref = (B @ th2.reshape(P, nu)).ravel()
    ue_gate = np.abs(B) @ dth.reshape(P, nu) + EPS * (d + 2) * (np.abs(B) @ np.abs(th2.reshape(P, nu)))
    exc_th, _ = excess(split[1], th2, dth)
    exc_ue, msg_ue = line(label + "-Uexec", split[3], ue_ref, ue_gate.ravel())
    exc_ue_alt, _ = excess(split[3], (B @ th.astype(np.float64)).ravel(), ue_gate.ravel())
    msg += f"; theta' over by {exc_th:.2e}; {msg_ue.split(' ', 2)[2]}, U_exec of the old theta {exc_ue_alt:.2e} over"
    print(msg)
    assert exc <= 0, msg
    assert exc_alt > 0, msg + ": the gate cannot see the last tile"
    assert exc_th <= 0 and exc_ue <= 0, msg
    assert exc_ue_alt > 0, msg + ": the gate cannot see the update"
    for u, v in zip(split, fused):
        np.testing.assert_array_equal(u.view(np.uint32), v.view(np.uint32))
    np.testing.assert_array_equal(split[2], split[1].reshape(P, nu)[0])
    np.testing.assert_array_equal(split[3][0], split[1].reshape(P, nu)[0])
    # the shift of theta'
    thg = split[1].astype(np.float64).reshape(P, nu)
    sh_ref = ko.shift(case.params, nu, split[1])
    Sm = spline_basis(T, P, d)[1]
    edge = np.isnan(Sm).any(1)
    sh_gate = EPS * (d + 2) * (np.abs(np.nan_to_num(Sm)) @ np.abs(thg)) + EPS * np.abs(sh_ref)
    assert excess(split[4], sh_ref, sh_gate)[0] <= 0, "shift"
    assert np.all(split[4].reshape(P, nu)[edge] == np.float32(0.25)) and edge.any()


# ======================================================================================================================== constrained
TOL, LAM_C, LAM = 0.25, 0.125, 0.5
# T*nu = 1, 16 (T = 1), 128 | 129, 256 | 258, 512 (T = 32), and the longest accepted horizons: nu = 2 at T = 216, nu = 1 at T = 256
CN_CELLS = [(1, 1), (1, 16), (32, 4), (43, 3), (16, 16), (129, 2), (32, 16), (216, 2), (256, 1)]
PLACEMENTS = ["none", "all", "lastsample", "tile0", "wrapped", "lastwarp", "nancta"]


def cn_geometry(T, nu, K):
    _, ncons, nstage, _ = ws_layout(T, nu, "W", feasible=True)
    ntiles = -(-K // WS_W)
    return ncons, nstage, ntiles, min(ntiles, NUM_SMS)


def cn_K(T, nu, placement):
    if placement in ("wrapped", "lastwarp"):
        return wrap_K(T, nu, "W", feasible=True)
    if placement in ("tile0", "nancta"):
        return WS_W * NUM_SMS + 32
    return WS_W * 37 + 4


def _cn_cases():
    out, i = [], 0
    for T, nu in CN_CELLS:
        rpl, ncons, nstage, _ = ws_layout(T, nu, "W", feasible=True)
        for pl in PLACEMENTS:
            K = cn_K(T, nu, pl)
            mode = ["simple", "halton-spline"][i % 2]
            g = GAMMAS[(i // 2) % 3]
            lam_c = 1e-3 if pl == "none" and i % 3 == 0 else LAM_C            # every weight but the minimum underflows
            i += 1
            tag = "simple" if mode == "simple" else f"g{g:g}"
            out.append(pytest.param(T, nu, K, pl, mode, g, lam_c,
                                    id=f"cn-RPL{rpl}-T{T}nu{nu}-ncons{ncons}s{nstage}-{pl}-K{K}-{tag}-lc{lam_c:g}"))
    return out


def cn_case(T, nu, K, mode, gamma, lam_c=LAM_C):
    return make_case(T, nu, K, mode=mode, gamma=gamma, lam=LAM, constraint_mode="feasible_first", constraint_tol=TOL, constraint_lambda=lam_c)


def cn_feasible_set(T, nu, K, placement, rng):
    """The samples a placement makes feasible (bool [K]) and the samples whose costs are NaN."""
    ncons, nstage, ntiles, grid = cn_geometry(T, nu, K)
    feas, nan = np.zeros(K, bool), np.zeros(K, bool)
    tile = np.arange(K) // WS_W
    cta, local = tile % grid, tile // grid
    if placement == "all":
        feas[:] = True
    elif placement == "lastsample":
        feas[K - 1] = True                                                      # only the last sample of the ragged last tile
    elif placement == "tile0":
        feas[tile == 0] = True                                                  # tile 0 of CTA 0; CTA 0's next tile is infeasible
    elif placement == "wrapped":
        feas[(cta == grid - 1) & (local == nstage)] = True                     # the first tile of the last CTA's second ring pass
    elif placement == "lastwarp":
        feas[(local % ncons == ncons - 1) & (rng.random(K) < 0.5)] = True      # tiles of the last consumer warp only
    elif placement == "nancta":
        feas[(tile % 5 == 3) & (rng.random(K) < 0.5)] = True
        nan[cta == grid - 1] = True                                             # one CTA entirely non-finite
    return feas, nan


def cn_margins(T, K, feas, rng):
    """Margins g [T][K]: a feasible sample has g <= 0 everywhere (V = 0) or one step at g = tol exactly (V = tol, exact in float32); an
    infeasible one has two positive steps (one where T = 1) with V in [0.5, 2.5], far outside v_dS of tol."""
    g = -rng.uniform(0.0, 1.0, (T, K))
    inf = np.flatnonzero(~feas)
    if inf.size:
        V = 0.5 + 2.0 * rng.random(inf.size)
        t1 = rng.integers(0, T, inf.size)
        if T > 1:
            t2 = (t1 + 1 + rng.integers(0, T - 1, inf.size)) % T
            s = rng.uniform(0.2, 0.8, inf.size)
            g[t1, inf], g[t2, inf] = s * V, (1 - s) * V
        else:
            g[t1, inf] = V
    exact = np.flatnonzero(feas & (rng.random(K) < 0.3))
    g[0, exact] = TOL
    return np.ascontiguousarray(g, np.float32)


def cn_restate(case, cost, x, U, g, keep=None, lam_c=None, lam=None, gamma_v=False):
    """float64 FEASIBLE row (cn.row) and its gate: _row_gate of the feasible regime (S, k3_dS, lambda) over the feasible samples, or of
    the violation regime (S := V, v_dS, lambda_c) over the valid ones; n_feasible exact; min V within v_dS.  keep / lam_c / lam /
    gamma_v (V with gamma^t) change the reference for the negative controls."""
    p, T, nu, K = case.params, case.T, case.nu, case.K
    S = cn.scores(p, nu, cost, x, U)
    g64 = np.asarray(g, np.float64)
    V = cn.violations(g64)
    if gamma_v:
        with np.errstate(invalid="ignore"):
            V = ((float(np.float32(p.gamma)) ** np.arange(T))[:, None] * np.where(g64 <= 0, 0.0, g64)).sum(0)
    ok = np.isfinite(S) & np.isfinite(V)
    if keep is not None:
        ok &= keep
    feas = ok & (V <= float(np.float32(p.constraint_tol)))
    xr = np.asarray(x, np.float64).reshape(T * nu, K)
    ncons = ws_layout(T, nu, "W", feasible=True)[1]
    if feas.any():
        key, mask, lm, dS = S, feas, float(np.float32(p.lambda_)) if lam is None else lam, k3_dS(case, cost, x, U)
    else:
        key, mask, lm = V, ok, float(np.float32(p.constraint_lambda)) if lam_c is None else lam_c
        dS = v_dS(g)
    b = key[mask].min() if mask.any() else np.inf
    with np.errstate(over="ignore", invalid="ignore"):
        w = np.where(mask, np.exp(-(np.where(mask, key, b) - b) / lm), 0.0)
    gate, _, _ = _row_gate(key, np.where(mask, dS, 0.0), w, b, xr, lm, K, ncons)
    row = np.concatenate([[b, w.sum()], xr @ w, [feas.sum(), V[ok].min() if ok.any() else np.inf]])
    dv = v_dS(g)
    gate = np.concatenate([gate, [0.0, float(dv[ok].max()) if ok.any() else 0.0]])
    return row, gate, feas


def cn_k4(case, rows, U):
    """float64 K4 of the device's own rows (n_feasible from its bits): the feasibility-first merge, then the plain update; the bound
    is the merge's and the update's float32 rounding."""
    p, G = case.params, len(rows)
    r = cn.from_f32(np.asarray(rows, np.float32))
    b, e, W, n, vmin = cn.merge(p, r)
    lam = float(np.float32(p.lambda_ if n > 0 else p.constraint_lambda))
    match = ((r[:, -2] > 0) == (n > 0)) & (r[:, 1] > 0)
    sc = np.where(match, np.exp(-(np.where(match, r[:, 0], b) - b) / lam), 0.0)
    U64 = np.asarray(U, np.float64).ravel()
    a = float(np.float32(p.step_size_mean))
    if e > 0:
        m = W / e
        new = U64 + m if case.simple else (1 - a) * U64 + a * m
    else:
        m, new = np.zeros_like(U64), U64
    aw = (sc[:, None] * np.abs(r[:, 2:-2])).sum(0) / max(e, 1e-300)
    gate = (8 + 2 * G) * EPS * (np.abs(U64) + aw + np.abs(new)) + 1e-30
    return new, gate, n, vmin


def cn_run(case, cost, x, U, g, fused):
    p, nu, T = case.params, case.nu, case.T
    be = backend(nu, p)
    viol, cstate = dev(g), torch.zeros(2, device=DEV)
    be.set_constraint(viol, cstate)
    part = torch.zeros(4 + T * nu, device=DEV)
    Ud, act, st = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    if fused:
        be.reduce_finalize(dev(cost), dev(x), Ud, part, act, st)
    else:
        be.reduce(dev(cost), dev(x), Ud, part)
        be.finalize(part.view(1, -1), 1, Ud, act, st)
    torch.cuda.synchronize()
    out = [t.cpu().numpy() for t in (part, Ud, act, st, cstate)]
    be.destroy()
    return out


def i32(v):
    """The int32 whose bits a float32 holds (n_feasible in the row and in cstate)."""
    return int(np.array([v], np.float32).view(np.int32)[0])


@pytest.mark.parametrize("T,nu,K,placement,mode,gamma,lam_c", _cn_cases())
def test_constraint_k3_k4_sweep(T, nu, K, placement, mode, gamma, lam_c):
    """The FEASIBLE row within the gate of its regime, n_feasible exact, min V within v_dS; fused = split bit for bit; K4 within its
    rounding of the float64 K4 of the device's row, and cstate = (n_feasible, min V).  Negative controls: with feasible and infeasible
    samples, the plain row over every valid sample; with none, the violation row with lambda for lambda_c (and with gamma^t in MEAN mode);
    with a lone feasible sample, the reference without it; with all, the reference without the last tile."""
    case = cn_case(T, nu, K, mode, gamma, lam_c)
    rng = np.random.default_rng(T * 7 + nu * 3 + K + PLACEMENTS.index(placement))
    cost, x, U = k3_inputs(case, seed=T + nu + K)
    feas, nan = cn_feasible_set(T, nu, K, placement, rng)
    g = cn_margins(T, K, feas, rng)
    cost[0, nan] = np.nan
    ref, gate, feas_ref = cn_restate(case, cost, x, U, g)
    assert feas_ref.sum() == (feas & ~nan).sum()
    split = cn_run(case, cost, x, U, g, fused=False)
    fused = cn_run(case, cost, x, U, g, fused=True)
    row = split[0].astype(np.float64)
    row[-2] = i32(split[0][-2])
    ncons, nstage, ntiles, grid = cn_geometry(T, nu, K)
    label = f"cn-T{T}nu{nu}-ncons{ncons}s{nstage}-grid{grid}-{placement}-K{K}-{mode}-lc{lam_c:g}"
    exc, msg = line(label, row, ref, gate, f", n_feasible {int(row[-2])} of {K}")
    if placement == "none":
        alts = {"lambda for lambda_c": cn_restate(case, cost, x, U, g, lam_c=LAM)[0]}
        if not case.simple and gamma != 1.0 and T > 1:
            alts["V with gamma^t"] = cn_restate(case, cost, x, U, g, gamma_v=True)[0]
    elif placement == "all":
        alts = {"without the last tile": cn_restate(case, cost, x, U, g, keep=drop_tail_mask(K))[0]}
    elif placement == "lastsample":
        keep = np.ones(K, bool)
        keep[K - 1] = False
        alts = {"without the lone feasible sample": cn_restate(case, cost, x, U, g, keep=keep)[0]}
    else:
        S, w, plain = k3_restate(case, cost, x, U)
        alts = {"plain over every valid sample": np.concatenate([plain, ref[-2:]])}
    for name, alt in alts.items():
        e_alt, _ = excess(row, alt, gate)
        msg += f", {name} {e_alt:.2e} over"
        assert e_alt > 0, msg + f": the gate cannot tell {name}"
    print(msg)
    assert exc <= 0, msg
    for u, v in zip(split, fused):
        np.testing.assert_array_equal(u.view(np.uint32), v.view(np.uint32))
    Un, ugate, n, vmin = cn_k4(case, [split[0]], U)
    assert excess(split[1], Un, ugate)[0] <= 0, "K4 update"
    assert i32(split[4][0]) == n == int(ref[-2]) and split[4][1] == split[0][-1] and vmin == split[0][-1]


@pytest.mark.parametrize("G", [1, 2, 3, 8])
@pytest.mark.parametrize("T,nu", [(43, 3), (32, 16), (216, 2)])
def test_constraint_explicit_rows(T, nu, G):
    """G shard rows of separate K3 launches around one U, only rank G - 1's shard with feasible samples, merged by the explicit-row K4:
    each row within its gate, the merge within its rounding of the float64 K4 of the device rows.  Negative control: the merge without
    rank G - 1's row misses it (for G > 1); n_feasible is rank G - 1's."""
    Kl = WS_W * 37 + 4
    case = cn_case(T, nu, Kl, "simple", 1.0)
    U = k3_inputs(case, seed=99)[2]
    rows, nfs = [], []
    for r in range(G):
        rng = np.random.default_rng(1000 * G + r)
        cost, x, _ = k3_inputs(case, seed=100 + r)
        feas = np.zeros(Kl, bool)
        if r == G - 1:
            feas[rng.random(Kl) < 0.3] = True
        g = cn_margins(T, Kl, feas, rng)
        ref, gate, _ = cn_restate(case, cost, x, U, g)
        part = cn_run(case, cost, x, U, g, fused=False)[0]
        row = part.astype(np.float64)
        row[-2] = i32(part[-2])
        assert excess(row, ref, gate)[0] <= 0, f"rank {r}"
        rows.append(part)
        nfs.append(int(ref[-2]))
    be = backend(nu, case.params)
    cstate = torch.zeros(2, device=DEV)
    be.set_constraint(dev(np.zeros((T, Kl), np.float32)), cstate)
    Ud, act, st = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(dev(np.stack(rows)), G, Ud, act, st)
    torch.cuda.synchronize()
    got, cs = Ud.cpu().numpy(), cstate.cpu().numpy()
    be.destroy()
    Un, ugate, n, vmin = cn_k4(case, rows, U)
    exc, msg = line(f"cn-rows-T{T}nu{nu}-G{G}", got, Un, ugate, f", n_feasible {n}")
    if G > 1:
        alt, _, _, _ = cn_k4(case, rows[:-1], U)
        e_alt, _ = excess(got, alt, ugate)
        msg += f", without rank G - 1 {e_alt:.2e} over"
        assert e_alt > 0, msg
    print(msg)
    assert exc <= 0, msg
    assert i32(cs[0]) == n == nfs[-1] > 0 and sum(nfs[:-1]) == 0
    assert cs[1] == np.float32(vmin)


# ======================================================================================================================== ESS
# (T, nu): T = 1, 9, 256 and T*nu = 1, 16, 129, 512 (at T = 32 and at T = 256)
ESS_CELLS = [(1, 1), (1, 16), (9, 2), (43, 3), (129, 1), (32, 16), (256, 2)]
ESS_TNT = 64                                                                   # samples per tile of mppib_temperature_kernel
RHOS = [0.001, 0.05, 1.0]
KIND_OF = {"W": "fixed", "M2": "diag", "C": "full"}


def ess_Ks():
    g2 = ESS_TNT * 2 * NUM_SMS                                                 # one tile per persistent CTA
    return {"k1": 1, "k31": 31, "k32": 32, "k33": 33, "k64": 64, "k65": 65, "half": ESS_TNT * 50 + 20, "grid-": g2 - ESS_TNT, "grid": g2,
            "grid+": g2 + ESS_TNT, "three": 3 * g2 + 4, "k65536": 65536}


def _ess_cases():
    out, i = [], 0
    for T, nu in ESS_CELLS:
        for name, K in ess_Ks().items():
            if T * nu * K > 12_000_000:                                        # the float64 references of K3 are T*nu*K doubles
                continue
            kind = ["W", "M2", "C"][i % 3]
            mode = ["simple", "halton-spline"][(i // 3) % 2]
            g = GAMMAS[i % 3]
            rho = RHOS[(i // 2) % 3]
            i += 1
            tag = "simple" if mode == "simple" else f"g{g:g}"
            k3 = K % 4 == 0
            rpl = ws_layout(T, nu, kind)[0]
            out.append(pytest.param(T, nu, K, kind, mode, g, rho, id=f"ess-{KIND_OF[kind]}-T{T}nu{nu}-{name}K{K}-{tag}-rho{rho:g}"
                                    + (f"-k3RPL{rpl}" if k3 else "")))
    return out


def ess_rtol(case, cost, x, U, dist):
    """Per grid point: the relative error of ESS_j the float32 sums of C_k and q_k allow (test_gpu_temperature's Case.rtol), with the
    rounding of h = Sigma^-1 U over nu terms (diag: one division; full: nu products) added to dq."""
    p, T, nu = case.params, case.T, case.nu
    gm = float(p.gamma) ** np.arange(T)
    dC = (T + 2) * EPS * (np.abs(cost.astype(np.float64)) * gm[:, None]).sum(0)
    dq = np.zeros(case.K)
    if case.simple:
        Si = tmo.sigma_inv(p, nu, dist)
        h = U.astype(np.float64) @ Si.T
        habs = np.abs(U.astype(np.float64)) @ np.abs(Si).T
        xa = np.abs(x.reshape(T * nu, -1).astype(np.float64))
        dq = (T * nu + 2) * EPS * (np.abs(h.reshape(-1)) @ xa) + 4 * EPS * np.abs(h).sum() + (nu + 2) * EPS * (habs.reshape(-1) @ xa)
    inv = ess_grid(p.lambda_)[1].astype(np.float64)
    C, q = tmo.scores(p, nu, cost, x, U, dist)
    ok = np.isfinite(C) & np.isfinite(q)
    d = (inv[:, None] * dC[None, ok] + dq[None, ok]).max(1)
    return np.expm1(4 * d) + 1e-4


def ess_dist(case, lam):
    if case.kind == "C":
        return afo.make_dist(lam, case.sigma)
    return np.concatenate([[lam], np.diag(case.sigma)]).astype(np.float32)


def ess_k3(case, cost, x, U, dist, fused):
    """K3 (+ K4) after the temperature pass, on a fresh handle with dist[0] = the chosen lambda: (row, U', action, dist)."""
    be = backend(case.nu, case.params)
    dd = dev(dist)
    be.set_distribution(dd)
    st = np.zeros(ESS_STATE_FLOATS, np.float32)
    st[:ESS_GRID], st[ESS_GRID:2 * ESS_GRID] = ess_grid(case.params.lambda_)
    be.set_temperature(dev(st))
    part = torch.zeros(be.partial_row_floats(), device=DEV)
    Ud, act, stats = dev(U), torch.zeros(case.nu, device=DEV), torch.zeros(2, device=DEV)
    if fused:
        be.reduce_finalize(dev(cost), dev(x), Ud, part, act, stats)
    else:
        be.reduce(dev(cost), dev(x), Ud, part)
        be.finalize(part.view(1, -1), 1, Ud, act, stats)
    torch.cuda.synchronize()
    out = [t.cpu().numpy() for t in (part, Ud, act, dd)]
    be.destroy()
    return out


@pytest.mark.parametrize("T,nu,K,kind,mode,gamma,rho", _ess_cases())
def test_ess_pass_rule_and_k3_sweep(T, nu, K, kind, mode, gamma, rho):
    """The curve within ess_rtol of float64; lambda is the rule on the device's own curve (rel 2e-6), and the float64 oracle's lambda
    lies in the bracket the curve's bound allows.  Where K3 runs (K a multiple of 4), its row at the chosen lambda (read back from
    dist[0]) within k3_gate, fused = split bit for bit.  Negative controls: the curve against its neighbour grid point's; lambda without
    the log-linear interpolation outside the bracket (where the interpolation moves it by more than the bracket); K3 at the grid's
    bracketing lambda misses the gate."""
    lam0 = 0.3
    case = make_case(T, nu, K, mode=mode, gamma=gamma, lam=lam0, kind=kind, lambda_mode="ess", ess_target=rho)
    cost, x, U = k3_inputs(case, seed=T * 5 + nu + K)
    dist = ess_dist(case, lam0)
    be = backend(nu, case.params)
    dd = dev(dist)
    be.set_distribution(dd)
    st = np.zeros(ESS_STATE_FLOATS, np.float32)
    lam_grid32, inv32 = ess_grid(case.params.lambda_)
    st[:ESS_GRID], st[ESS_GRID:2 * ESS_GRID] = lam_grid32, inv32
    state = dev(st)
    be.set_temperature(state)
    row = torch.zeros(1 + 3 * ESS_GRID, device=DEV)
    be.temperature(dev(cost), dev(x), dev(U), row, solve=True)
    torch.cuda.synchronize()
    lam_dev, st_dev = float(dd[0]), state.cpu().numpy()
    be.destroy()
    N = int(st_dev[2 * ESS_GRID:2 * ESS_GRID + 1].view(np.int32)[0])
    ess_dev = st_dev[2 * ESS_GRID + 2:].astype(np.float64)
    ref_row = tmo.shard_row(case.params, nu, cost, x, U, inv32, dist)
    _, ess_ref = tmo.combine([ref_row])
    r = ess_rtol(case, cost, x, U, dist)
    label = f"ess-{KIND_OF[kind]}-T{T}nu{nu}-K{K}-{mode}-rho{rho:g}"
    exc, msg = line(label, ess_dev, ess_ref, r * ess_ref, f", lambda {lam_dev:.4g}")
    assert N == ref_row[0] == K
    nb = np.abs(ess_dev[:-1] / ess_ref[1:] - 1.0) - r[:-1]                     # the curve against its neighbour grid point
    msg += f", neighbour curve {nb.max():.2e} over"                           # (K = 1: ESS = 1 at every temperature)
    lam_grid = lam_grid32.astype(np.float64)
    rho32 = float(np.float32(rho))
    assert lam_dev == pytest.approx(tmo.rule(ess_dev, N, rho32, lam_grid, 0.0), rel=2e-6)
    lo = tmo.rule(ess_dev * (1 + r), N, rho32, lam_grid, 0.0)
    hi = tmo.rule(ess_dev * (1 - r), N, rho32, lam_grid, 0.0)
    lam_ref = tmo.rule(ess_ref, N, rho32, lam_grid, 0.0)
    assert lo * (1 - 1e-6) <= lam_ref <= hi * (1 + 1e-6), (lo, lam_ref, hi)
    hit = np.flatnonzero(ess_dev >= rho32 * N)
    j = int(hit[0]) if hit.size else None
    interp = j is not None and 0 < j and hi < lo * 2.0 ** 0.25                  # interpolated, and the bracket narrower than a grid step
    if interp:
        far = [v for v in (lam_grid[j - 1], lam_grid[j]) if not (lo * (1 - 1e-6) <= v <= hi * (1 + 1e-6))]
        msg += f", {len(far)} of the 2 bracketing grid points outside [{lo:.4g}, {hi:.4g}]"
    print(msg)
    assert exc <= 0, msg
    if K > 1:
        assert nb.max() > 0, msg + ": the curve bound cannot tell neighbour grid points"
    if interp:
        assert far, msg + ": the bracket cannot tell the interpolation"
    if K % 4:
        return
    # K3 + K4 at the chosen lambda
    kd = ess_dist(case, lam_dev)
    kcase = dataclasses.replace(case, dist=kd)
    S, w, ref = k3_restate(kcase, cost, x, U)
    gate = k3_gate(kcase, cost, x, U, S, w)
    split = ess_k3(kcase, cost, x, U, kd, fused=False)
    fused = ess_k3(kcase, cost, x, U, kd, fused=True)
    exc3, msg3 = line(label + f"-k3RPL{ws_layout(T, nu, kind)[0]}", split[0], ref, gate)
    other = min((v for v in lam_grid32 if v != np.float32(lam_dev)), key=lambda v: abs(math.log(v / lam_dev)))   # the nearest grid point
    _, _, alt = k3_restate(dataclasses.replace(case, dist=ess_dist(case, float(np.float32(other)))), cost, x, U)
    e_alt, _ = excess(split[0], alt, gate)
    C, q = tmo.scores(case.params, nu, cost, x, U, kd)
    spread = tmo.ess_at(C, q, lam_dev) > 1.5                                   # else the softmax keeps one sample at either lambda
    msg3 += f", at the grid's lambda {other:.4g} {e_alt:.2e} over" + ("" if spread else " (one sample carries the weight)")
    print(msg3)
    assert exc3 <= 0, msg3
    if spread:
        assert e_alt > 0, msg3 + ": the gate cannot tell the chosen lambda from the grid's"
    for u, v in zip(split, fused):
        np.testing.assert_array_equal(u.view(np.uint32), v.view(np.uint32))
    if kind == "W":
        U2, dU = mean_update(ref, gate, U, case.simple, float(np.float32(case.params.step_size_mean)))
        assert excess(split[1], U2, dU)[0] <= 0, "K4 update"
