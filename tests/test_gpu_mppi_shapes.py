"""-m gpu: K1 (Gaussian and Halton library), K3, K4 and the shift over every template instantiation and the accepted (T, nu, K) range,
against the float64 references, on the generated cases of ``synth_mppi`` (the point robot's model with nu set; no dynamics run).

K3 is gated per case by the float32 error bound of ``synth_mppi.k3_gate`` (not by a constant), and every sweep case must also
miss that gate against a reference that drops the samples of the last (ragged) tile: a gate that a wrong kernel passes is no test.
Each test prints its worst error next to its gate (``SHAPES`` lines, shown with -s)."""
import copy
import math
import os

import numpy as np
import pytest
import torch

import adaptive_full_oracle as afo
import adaptive_horizon_oracle as aho
import adaptive_oracle as ada
from synth_mppi import (EPS, KINDS, NUM_SMS, WS_W, drop_tail_mask, hz_C, hz_id, hz_k1_gate, k3_gate, k3_id, k3_inputs, k3_restate, last4_K,
                        make_case, mode_tag, nu_model, row_excess, shifted_from, syrk_split, wrap_K, ws_layout)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NTHREADS = min(16, os.cpu_count() or 1)


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def backend(case, dist=None, params=None):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(case.model, params or case.params)
    if dist is not None:
        be.set_distribution(dist)
    return be


# ------------------------------------------------------------------------------------------------------------------------------ K1
K1_NU = [1, 2, 4, 5, 8, 12, 13, 16]
K1_K = [1, 127, 129, 1000]


def _k1_cases():
    out, i = [], 0
    for nu in K1_NU:
        for T in sorted({1, 9, 512 // nu}):
            for kind in KINDS:
                K = K1_K[i % 4]
                i += 1
                out.append(pytest.param(T, nu, K, kind, id=f"k1-{kind}-T{T}nu{nu}-K{K}"))
    return out


def _bounds(nu, sig, rng):
    """Per-column bounds: every third column tight enough that the clamp binds on part of the samples, the others wide."""
    s = np.sqrt(np.diag(sig))
    lo = np.where(np.arange(nu) % 3 == 0, -0.5 * s, -1e3)
    hi = np.where(np.arange(nu) % 3 == 0, 0.3 * s, 1e3)
    return lo.tolist(), hi.tolist()


@pytest.mark.parametrize("T,nu,K,kind", _k1_cases())
def test_k1_gaussian(oracle, T, nu, K, kind):
    rng = np.random.default_rng(T * 17 + nu)
    case0 = make_case(T, nu, K, kind=kind)
    lo, hi = _bounds(nu, case0.sigma, rng)
    case = make_case(T, nu, K, kind=kind, u_min=lo, u_max=hi)
    p, nu = case.params, case.nu
    dist = dev(case.dist) if case.dist is not None else None
    be = backend(case, dist)
    U = rng.uniform(-0.05, 0.05, (T, nu)).astype(np.float32)
    prior = rng.uniform(-2, 2, (T, nu)).astype(np.float32)
    seed, plan0, ctr = 0x1_2345_6789, 2 ** 32 - 3, 5                       # seed and plan index >= 2^32, the plan through plan_ctr
    a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    be.sample(seed, plan0, 0, K, dev(U), dev(prior), a, n, torch.tensor([ctr], dtype=torch.int32, device=DEV))
    pref = p if kind == "W" else (ada.dist_params(p, nu, case.dist) if kind == "M2" else afo.dist_params(p, nu, case.dist))
    a_ref, n_ref = oracle.sample(case.model, pref, seed, plan0 + ctr, U, prior_row=prior)
    ag, ng = a.cpu().numpy(), n.cpu().numpy()
    L = case.chol().astype(np.float64)
    gate = 2e-6 * max(1.0, 6 * np.abs(L).sum(1).max())
    body = slice(0, max(K - 2, 0))
    err = max(float(np.abs(ag[:, :, body] - a_ref[:, :, body]).max(initial=0)), float(np.abs(ng[:, :, body] - n_ref[:, :, body]).max(initial=0)))
    print(f"SHAPES k1-{kind}-T{T}nu{nu}-K{K} worst {err:.2e} gate {gate:.2e}")
    assert err <= gate
    np.testing.assert_array_equal(ag[:, :, K - 1], a_ref[:, :, K - 1])      # null row
    np.testing.assert_array_equal(ag[:, :, K - 1], 0)
    if K >= 2:
        np.testing.assert_array_equal(ag[:, :, K - 2], prior)               # prior row, not clamped
        np.testing.assert_array_equal(ng[:, :, K - 2], n_ref[:, :, K - 2])
    tight = np.arange(nu) % 3 == 0
    if K > 100:
        at = (ag[:, tight, :-2] == np.asarray(hi, np.float32)[tight][None, :, None]).mean()
        assert 0.05 < at < 0.95                                              # the clamp binds on part of the samples of the tight columns
    # k_offset shards are bit-identical to one launch
    if K >= 2:
        k1 = K // 3 + 1
        parts = []
        for off, kk in ((0, k1), (k1, K - k1)):
            pp = copy.copy(p); pp.K = kk
            be2 = backend(case, dev(case.dist) if case.dist is not None else None, pp)
            aa = torch.zeros((T, nu, kk), device=DEV)
            be2.sample(seed, plan0 + ctr, off, K, dev(U), dev(prior), aa, None)
            parts.append(aa.cpu().numpy())
        np.testing.assert_array_equal(np.concatenate(parts, axis=2), ag)


# ------------------------------------------------------------------------------------------------------------------------------ Halton
def _halton_u(kg, base, mult):
    """float64 generalised Halton points of the global indices kg + 1 (vector) in one base."""
    idx = np.asarray(kg, np.int64) + 1
    r, f = np.zeros(idx.shape), 1.0 / base
    while np.any(idx > 0):
        r += ((idx % base) * mult % base) * f
        idx //= base
        f /= base
    return r


@pytest.mark.parametrize("nu", [7, 9, 12, 16])
@pytest.mark.parametrize("T", [12, 30, 128, 131])
@pytest.mark.parametrize("kind", KINDS)
def test_halton_library(oracle, nu, T, kind):
    from scipy.special import ndtri
    from mppi_isaac_b200.planner.mppi import halton_spline_operator, halton_table
    K, k_total = 1000, 65536
    k_off = k_total - K                                                       # global indices up to 65 536: points close to 0 and 1
    nk = T // 4
    case = make_case(T, nu, K, mode="halton-spline", kind=kind)
    p = case.params
    be = backend(case, dev(case.dist) if case.dist is not None else None)
    B, tab = halton_spline_operator(T, nk), halton_table(nk * nu, 11)
    Z = torch.zeros((T, nu, K), device=DEV)
    be.noise_library(k_off, k_total, dev(tab, torch.int32), dev(B), nk, Z)
    white = kind != "W"
    pref = p if kind == "W" else (ada.dist_params(p, nu, case.dist, white=True) if kind == "M2" else afo.dist_params(p, nu, case.dist, white=True))
    Z_ref = oracle.noise_library(case.model, pref, tab, B, nk, k_off, k_total)
    Zg = Z.cpu().numpy()
    # gate per element: slope of the quantile at the reference's u times the float32 error of u (radical inverse with up to
    # 17 digits, 2u - 1), plus erfinvf's own, through sum |B| sum |L|
    nd = nk * nu
    tab = np.asarray(tab).reshape(-1)                                        # [bases | multipliers]
    kg = np.arange(k_off, k_off + K)
    u = np.stack([_halton_u(kg, int(tab[d]), int(tab[nd + d])) for d in range(nd)])          # [nd][K]
    u32 = u.astype(np.float32).astype(np.float64)
    z = ndtri(u32)
    ndig = np.array([math.ceil(math.log(k_total + 1, int(tab[d]))) + 1 for d in range(nd)])[:, None]
    du = EPS * ((2 * ndig + 4) * u32 + 1.0)
    dz = (np.sqrt(2 * np.pi) * np.exp(0.5 * z * z) * du + 4 * EPS * np.abs(z)).reshape(nk, nu, K)
    Lc = np.eye(nu) if white else np.abs(np.array(p.sigma_chol[:nu * nu], np.float64).reshape(nu, nu))
    Bab = np.abs(np.asarray(B, np.float64))
    zc = np.einsum("ji,nik->njk", Lc, dz)                                    # [nk][nu][K]
    zmag = np.einsum("ji,nik->njk", Lc, np.abs(z.reshape(nk, nu, K)))
    gate = np.einsum("tn,njk->tjk", Bab, zc + EPS * (nk + nu + 2) * zmag)
    gate[:, :, -1] = 0                                                        # null row: exact
    err = np.abs(Zg - Z_ref)
    print(f"SHAPES halton-{kind}-T{T}nu{nu}-nk{nk} worst {err.max():.2e} gate(min/median) {gate[:, :, :-1].min():.2e}/{np.median(gate):.2e}"
          f" worst err/gate {(err / np.maximum(gate, 1e-30)).max():.2f} u in [{u.min():.2e}, {1 - u.max():.2e} from 1]")
    assert np.all(err <= gate)
    assert np.median(err) <= 1e-6
    assert u.min() < 1e-4 and u.max() > 1 - 1e-4
    # the library sampler: coloured (exact), WHITE x diag scale, WHITE x full L
    rng = np.random.default_rng(T + nu)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    prior = rng.uniform(-1, 1, (T, nu)).astype(np.float32)
    a, n = torch.zeros_like(Z), torch.zeros_like(Z)
    be.sample_library(k_off, k_total, dev(U), dev(prior), Z, a, n)
    if kind == "W":
        Zs = Zg
    elif kind == "M2":
        Zs = np.sqrt(case.dist[1:1 + nu].astype(np.float32))[None, :, None] * Zg
    else:
        Zs = afo.color_library(case.dist, nu, Zg)
    a_ref, n_ref = oracle.sample_library(case.model, p, U, Zs, k_off, k_total, prior_row=prior)
    if kind == "W":
        np.testing.assert_array_equal(a.cpu().numpy(), a_ref)
        np.testing.assert_array_equal(n.cpu().numpy(), n_ref)
    else:
        scale = max(1.0, np.abs(Zg).max() * np.abs(case.chol()).sum(1).max())
        assert np.abs(a.cpu().numpy() - a_ref).max() <= 2e-6 * scale
        assert np.abs(n.cpu().numpy() - n_ref).max() <= 2e-6 * scale
        np.testing.assert_array_equal(a.cpu().numpy()[:, :, -2:], a_ref[:, :, -2:])


# ------------------------------------------------------------------------------------------------------------------------------ K3 / K4
# (T, nu) cells: T*nu = 1, 128, 129, 256, 258 (257 is prime: T = 257 is refused), 512; consumer warps 6, 5, 4, 3, 2 (7 at every
# small shape); T = 256 at nu = 1 and 2; x boxes 7 x 37 and 2 x 251; nu = 13 .. 16
CELLS = [(1, 1), (32, 4), (43, 3), (16, 16), (129, 2), (32, 16), (125, 1), (146, 1), (174, 1), (216, 1), (187, 2), (256, 1), (256, 2), (37, 7),
         (251, 2), (20, 13), (9, 14), (30, 15), (3, 16)]
MODES = [("simple", 1.0), ("halton-spline", 0.0), ("halton-spline", 0.5), ("halton-spline", 0.95), ("halton-spline", 1.05)]


def _k3_cases():
    out = []
    for ci, (T, nu) in enumerate(CELLS):
        for kind in KINDS:
            if ws_layout(T, nu, kind) is None:
                continue
            for i, K in enumerate([4, 36, WS_W * NUM_SMS - 4, WS_W * NUM_SMS + 4, wrap_K(T, nu, kind)]):
                mode, g = MODES[(i + ci) % len(MODES)]
                tag = "simple" if mode == "simple" else f"g{g:g}"
                out.append(pytest.param(T, nu, K, kind, mode, g, id=k3_id(T, nu, K, kind, tag)))
    return out


def _ref_row(oracle, case, cost, x, U):
    if case.kind == "W":
        if case.K >= 32768:
            return oracle.reduce_mt(case.model, case.params, cost, x, U, NTHREADS)
        return oracle.reduce(case.model, case.params, cost, x, U)[0]
    if case.kind == "M2":
        return ada.reduce(case.model, case.params, cost, x, U, case.dist)
    return afo.reduce(case.model, case.params, cost, x, U, case.dist)


def _ref_finalize(case, row, U):
    if case.kind == "W":
        from oracle import oracle as orc
        Un, act, st = orc.finalize(case.model, case.params, row[None], U)
        return Un, act, st, None
    mod = ada if case.kind == "M2" else afo
    return mod.finalize(case.model, case.params, row[None], U, case.dist)


def _run_k3(case, cost, x, U):
    """reduce + finalize and the fused reduce_finalize from the same inputs: (row, U, action, stats, dist) of both."""
    out = []
    for fused in (False, True):
        dist = dev(case.dist) if case.dist is not None else None
        be = backend(case, dist)
        part, Ud = torch.zeros(case.row_floats(), device=DEV), dev(U)
        act, st = torch.zeros(case.nu, device=DEV), torch.zeros(2, device=DEV)
        c, xx = dev(cost), dev(x)
        if fused:
            be.reduce_finalize(c, xx, Ud, part, act, st)
        else:
            be.reduce(c, xx, Ud, part)
            be.finalize(part.view(1, -1), 1, Ud, act, st)
        out.append([t.cpu().numpy() for t in (part, Ud, act, st)] + [dist.cpu().numpy() if dist is not None else None])
    for a, b in zip(*out):
        if a is not None:
            np.testing.assert_array_equal(a, b)                                # the fused tail is the two launches, bit for bit
    return out[0]


def _check_k4(case, row, Ug, act, st, dg, U, label):
    """K4 on the kernel's own row against the reference's finalize: U, action, stats, dist."""
    T, nu, NR = case.T, case.nu, case.T * case.nu
    U_ref, act_ref, st_ref, d_ref = _ref_finalize(case, row, U)
    np.testing.assert_array_equal(st, row[:2])                                 # one row: (beta, eta) pass through unchanged
    np.testing.assert_array_equal(act, Ug[0])
    e = float(row[1])
    wm = np.abs(row[2:2 + NR].astype(np.float64) / e) if e > 0 else 0.0
    gate_u = 32 * EPS * (np.abs(U).max() + np.max(wm) + 1e-30) * (2.0 if case.params.filter_u else 1.0)
    err_u = float(np.abs(Ug - U_ref).max())
    msg = f"SHAPES {label} K4 U worst {err_u:.2e} gate {gate_u:.2e}"
    assert err_u <= gate_u, msg
    if dg is not None:
        assert dg[0] == d_ref[0]                                               # the lambda rule: the same float32 steps
        if case.kind == "M2" and e > 0:
            m2 = row[2 + NR:].astype(np.float64) / e
            d = (U_ref - U).reshape(-1).astype(np.float64)
            m1 = wm + (0.0 if case.simple else np.abs(U).reshape(-1))
            mag = (np.abs(m2) + 2 * np.abs(d) * m1 + d * d + (np.abs(U).reshape(-1) + wm) * m1).reshape(T, nu).mean(0)
            gate_c = float(case.params.step_size_cov) * EPS * (T + 16) * mag + 4 * EPS * np.abs(d_ref[1:])
            err_c = np.abs(dg[1:] - d_ref[1:])
            msg += f"; cov worst {err_c.max():.2e} gate {gate_c.min():.2e}"
            assert np.all(err_c <= gate_c), msg
        elif case.kind == "C" and e > 0:
            _, S, L, I = afo.unpack(dg, nu)
            _, Sr, _, _ = afo.unpack(d_ref, nu)
            W = row[2:2 + NR].astype(np.float64).reshape(T, nu) / e
            c = 0.0 if case.simple else U.astype(np.float64)
            a = np.abs(W) + np.abs(c) + np.abs(W - c)
            b = np.abs(U_ref - U) + np.abs(U) + np.abs(W)
            Cm = np.abs(afo.tril_unpack(row[2 + NR:].astype(np.float64), nu)) / e
            dV = EPS * (4 * Cm + (T + 12) * 4 * (a + b).T @ (a + b))
            gate_s = float(case.params.step_size_cov) / T * dV + 4 * EPS * np.abs(Sr)
            err_s = np.abs(S.astype(np.float64) - Sr)
            msg += f"; Sigma worst {err_s.max():.2e} gate {gate_s.min():.2e}"
            assert np.all(err_s <= gate_s), msg
            np.testing.assert_array_equal(S, S.T)
            np.testing.assert_array_equal(I, I.T)
            np.testing.assert_array_equal(L, np.tril(L))
            L64, S64 = L.astype(np.float64), S.astype(np.float64)
            assert np.all(np.abs(L64 @ L64.T - S64) <= (nu + 2) * EPS * (np.abs(L64) @ np.abs(L64).T)), msg
            assert np.abs(I.astype(np.float64) @ S64 - np.eye(nu)).max() <= 4 * nu * EPS * np.linalg.cond(S64), msg
    print(msg)


def _check_k3(oracle, case, cost, x, U, label, drop_check=False):
    S, w, _ = k3_restate(case, cost, x, U)
    gate = k3_gate(case, cost, x, U, S, w)
    ref = _ref_row(oracle, case, cost, x, U)
    row, Ug, act, st, dg = _run_k3(case, cost, x, U)
    exc, err = row_excess(row, ref, gate)
    finite = np.isfinite(gate) & (gate > 0)
    ratio = float((np.abs(row.astype(np.float64) - ref)[finite] / gate[finite]).max(initial=0.0))
    line = f"SHAPES {label} K3 worst |err| {err:.2e}, worst err/gate {ratio:.3f}, gate of eta {gate[1]:.2e}"
    if drop_check:
        _, _, alt = k3_restate(case, cost, x, U, keep=drop_tail_mask(case.K))
        exc_alt, _ = row_excess(row, alt, gate)
        line += f", the reference without the last tile misses it by {exc_alt:.2e}"
        assert exc_alt > 0, line + ": the gate cannot tell the ragged tail apart"
    print(line)
    assert exc <= 0, line
    _check_k4(case, row, Ug, act, st, dg, U, label)
    return row, Ug, st, dg


@pytest.mark.parametrize("T,nu,K,kind,mode,gamma", _k3_cases())
def test_k3_k4_sweep(oracle, T, nu, K, kind, mode, gamma):
    case = make_case(T, nu, K, mode=mode, gamma=gamma, kind=kind, filter_u=T >= 9, update_lambda=kind != "W")
    cost, x, U = k3_inputs(case, seed=31 * T + nu + K)
    _check_k3(oracle, case, cost, x, U, k3_id(T, nu, K, kind, mode_tag(case)), drop_check=True)


EDGE_SHAPES = [(30, 7, "W", "simple"), (16, 16, "C", "halton-spline"), (125, 1, "M2", "simple")]
EDGES = ["nonfinite", "tile", "cta", "none", "one", "min_ragged", "underflow", "tie", "lam_tiny", "lam_large"]


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("T,nu,kind,mode", EDGE_SHAPES, ids=[f"{k}-T{t}nu{n}-{m}" for t, n, k, m in EDGE_SHAPES])
def test_k3_edge_inputs(oracle, T, nu, kind, mode, edge):
    K = {"cta": WS_W * NUM_SMS * 2 + 64, "underflow": WS_W * NUM_SMS * 4, "tie": 4228}.get(edge, 4228)
    # lambda tiny: S spans 0.2 over 4 228 samples, so the weight sits on the best few (gaps ~ lambda / 2), while the float32 error
    # of S stays ~1e-6 -- a smaller lambda only widens the derived gate.  lambda large: near-uniform weights.
    lam = {"lam_tiny": 1e-4, "lam_large": 1e3}.get(edge, 0.5)
    base = make_case(T, nu, K, mode=mode, kind=kind, lam=0.05 if edge == "lam_tiny" else 0.5)
    cost, x, U = k3_inputs(base, seed=7, favour_tail=edge != "lam_tiny")
    case = make_case(T, nu, K, mode=mode, kind=kind, lam=lam)
    grid = min((K + WS_W - 1) // WS_W, NUM_SMS)
    if edge == "nonfinite":
        cost[:, 3] = np.nan
        cost[5, 7] = np.inf
        cost[2, 11] = -np.inf
        cost[T - 1, K - 1] = np.nan
    elif edge == "tile":
        cost[:, 32:64] = np.nan
    elif edge == "cta":
        for k0 in range(5 * WS_W, K, grid * WS_W):                             # every tile of CTA 5: its partial is (inf, 0, 0)
            cost[:, k0:k0 + WS_W] = np.nan
    elif edge == "none":
        cost[:] = np.nan
    elif edge == "one":
        keep = cost[:, 77].copy()
        cost[:] = np.nan
        cost[:, 77] = keep
    elif edge == "min_ragged":
        cost[0, K - 1] -= 3 * lam
    elif edge == "underflow":
        k = (9 + 3 * grid) * WS_W + 5                                          # in the last of the 4 tiles CTA 9 streams
        cost[0, k] -= 200 * lam                                                # exp(-200) underflows: s_old = 0
    elif edge == "tie":
        k1, k2 = 40, 40 + 7 * WS_W                                             # CTAs 1 and 8
        cost[0, k1] -= 50 * lam
        cost[:, k2], x[:, :, k2] = cost[:, k1], x[:, :, k1]
        if case.simple:
            pytest.skip("ties are built in MEAN mode")
    row, Ug, st, dg = _check_k3(oracle, case, cost, x, U, f"k3-edge-{edge}-{kind}-T{T}nu{nu}-K{K}-{mode_tag(case)}")
    NR = T * nu
    if edge == "none":
        assert row[0] == np.inf and row[1] == 0 and not row[2:].any()
        assert st[0] == np.inf and st[1] == 0
        if case.simple:
            np.testing.assert_array_equal(Ug, U)                               # U + 0
        else:
            assert np.abs(Ug - U).max() <= 4 * EPS * max(1.0, np.abs(U).max())
        if dg is not None:
            np.testing.assert_array_equal(dg, case.dist)
    elif edge == "one":
        assert row[1] == 1.0
        np.testing.assert_array_equal(row[2:2 + NR], x[:, :, 77].reshape(-1))
    elif edge == "tie":
        assert abs(row[1] - 2.0) <= 4 * EPS
        np.testing.assert_allclose(row[2:2 + NR], 2 * x[:, :, 40].reshape(-1), rtol=4 * EPS, atol=0)
    elif edge == "underflow":
        assert row[1] == 1.0
        np.testing.assert_array_equal(row[2:2 + NR], x[:, :, (9 + 3 * grid) * WS_W + 5].reshape(-1))


# ------------------------------------------------------------------------------------------------------------------------------ K4
@pytest.mark.parametrize("T", [9, 10, 11, 12, 13, 256])
def test_k4_savitzky_golay_and_clamp(oracle, T):
    """Hand-built row through K4 with filter_u: the edge and middle windows overlap at T = 9 .. 13; per-column bounds that the
    filtered U overshoots, so the clamp after the filter binds."""
    nu = 3
    rng = np.random.default_rng(T)
    y = np.cumsum(rng.normal(0, 0.3, (T, nu)), 0).astype(np.float32)
    lo, hi = np.quantile(y, 0.15, axis=0), np.quantile(y, 0.85, axis=0)
    case = make_case(T, nu, 4, mode="halton-spline", filter_u=True, u_min=lo.tolist(), u_max=hi.tolist())
    U = rng.normal(0, 0.1, (T, nu)).astype(np.float32)
    row = np.concatenate([[0.0, 1.0], y.ravel()]).astype(np.float32)
    be = backend(case)
    Ud, act, st = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(dev(row).view(1, -1), 1, Ud, act, st)
    U_ref, _, _ = oracle.finalize(case.model, case.params, row[None], U)
    Ug = Ud.cpu().numpy()
    gate = 64 * EPS * max(1.0, np.abs(y).max())
    err = float(np.abs(Ug - U_ref).max())
    lo32, hi32 = np.asarray(case.params.u_min[:nu], np.float32), np.asarray(case.params.u_max[:nu], np.float32)
    bound = (Ug == lo32) | (Ug == hi32)
    print(f"SHAPES k4-savgol-T{T} worst {err:.2e} gate {gate:.2e}, {bound.mean():.0%} of U on a bound")
    assert err <= gate
    assert 0.0 < bound.mean() < 0.9
    np.testing.assert_array_equal(act.cpu().numpy(), Ug[0])


@pytest.mark.parametrize("G", [2, 3, 5, 8])
@pytest.mark.parametrize("kind", KINDS)
def test_k4_combines_g_shard_rows(oracle, G, kind):
    """G shard rows (shards of different beta, one shard all invalid) through one K4 == one K3 launch over all samples."""
    T, nu, Ks = 16, 9, 1024
    K = G * Ks
    case = make_case(T, nu, K, mode="simple", kind=kind, filter_u=True)
    cost, x, U = k3_inputs(case, seed=G, favour_tail=False)
    for g in range(G):
        cost[0, g * Ks:(g + 1) * Ks] += 0.7 * g * case.lam                   # a different beta per shard
    cost[:, (G - 1) * Ks:] = np.nan                                            # the last shard has no valid sample
    one = _run_k3(case, cost, x, U)
    pg = copy.copy(case.params); pg.K = Ks
    dist = dev(case.dist) if case.dist is not None else None
    be = backend(case, dist, pg)
    P = case.row_floats()
    parts = torch.zeros((G, P), device=DEV)
    Ud = dev(U)
    for g in range(G):
        sl = slice(g * Ks, (g + 1) * Ks)
        be.reduce(dev(cost[:, sl]), dev(x[:, :, sl]), Ud, parts[g])
    act, st = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(parts, G, Ud, act, st)
    rows = parts.cpu().numpy()
    assert rows[-1, 0] == np.inf and rows[-1, 1] == 0
    assert len(set(rows[:-1, 0].tolist())) == G - 1
    Ug, stg = Ud.cpu().numpy(), st.cpu().numpy()
    err = float(np.abs(Ug - one[1]).max())
    gate = 4e-6 * max(1.0, np.abs(one[1]).max())
    print(f"SHAPES k4-G{G}-{kind} U against one launch {err:.2e} gate {gate:.2e}")
    assert err <= gate
    assert stg[0] == one[3][0] and abs(stg[1] - one[3][1]) <= 1e-5 * one[3][1]
    # and against the reference finalize of the same G rows
    if kind == "W":
        U_ref, _, st_ref = oracle.finalize(case.model, case.params, rows, U)
    else:
        U_ref, _, st_ref, d_ref = (ada if kind == "M2" else afo).finalize(case.model, case.params, rows, U, case.dist)
        np.testing.assert_allclose(dist.cpu().numpy()[1:], d_ref[1:], rtol=0, atol=2e-5 * np.abs(d_ref[1:]).max())
    assert np.abs(Ug - U_ref).max() <= gate
    assert stg[0] == st_ref[0]


# ------------------------------------------------------------------------------------------------------------------------------ shift
@pytest.mark.parametrize("T,nu", [(1, 5), (256, 2), (32, 16)])
def test_shift_and_plan_counter(oracle, T, nu):
    init = np.linspace(-0.3, 0.4, nu).tolist()
    case = make_case(T, nu, 4, u_init=init)
    be = backend(case)
    U = np.random.default_rng(T).normal(0, 1, (T, nu)).astype(np.float32)
    Ud, ctr = dev(U), torch.tensor([7], dtype=torch.int32, device=DEV)
    be.shift(Ud, ctr)
    be.shift(Ud, ctr)
    ref = oracle.shift(case.model, case.params, oracle.shift(case.model, case.params, U))
    np.testing.assert_array_equal(Ud.cpu().numpy(), ref)
    np.testing.assert_array_equal(ref[-1], np.asarray(init, np.float32))
    assert int(ctr) == 9


# ------------------------------------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("what", ["Tnu513", "T257", "K6", "knots33", "gamma_neg", "gamma_nan"])
def test_host_refuses_unsupported_shapes(what):
    """Refused on the host with an error, before any launch."""
    from mppi_isaac_b200.planner.mppi import halton_spline_operator, halton_table
    shapes = {"Tnu513": (57, 9, 64, "W"), "T257": (257, 1, 64, "W"), "K6": (8, 2, 6, "W"), "knots33": (132, 2, 64, "W"),
              "gamma_neg": (8, 2, 64, "W"), "gamma_nan": (8, 2, 64, "W")}
    T, nu, K, kind = shapes[what]
    case = make_case(T, nu, K, kind=kind)
    if what.startswith("gamma"):
        p = copy.copy(case.params)                                             # make_params refuses these too (test_oracle_mppi_shapes)
        p.gamma = -0.5 if what == "gamma_neg" else float("nan")
        with pytest.raises(RuntimeError, match="gamma"):
            backend(case, params=p)
        return
    be = backend(case, dev(case.dist) if case.dist is not None else None)
    x, cost, U = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, K), device=DEV), torch.zeros((T, nu), device=DEV)
    part = torch.zeros(case.row_floats(), device=DEV)
    if what == "knots33":
        nk = T // 4
        with pytest.raises(RuntimeError, match="n_knots = 33"):
            be.noise_library(0, K, dev(halton_table(nk * nu, 3), torch.int32), dev(halton_spline_operator(T, nk)), nk, torch.zeros((T, nu, K), device=DEV))
        return
    match = {"Tnu513": "T\\*nu = 513", "T257": "T = 257", "K6": "K=6"}[what]
    with pytest.raises(RuntimeError, match=match):
        be.reduce(cost, x, U, part)
    with pytest.raises(RuntimeError, match=match):
        be.reduce_finalize(cost, x, U, part, torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------------ cov_type horizon
# The "H" row kind (update_cov with cov_type: horizon, n = T*nu <= 256): the horizon K1, the two K3 instantiations that store S_k,
# the weighted SYRK (tiles, K-splits, the fold and the fused K4 of its last CTA) and horizon_update, each against float64.
def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _hz_backend(case, U, dist=None, params=None):
    """A horizon handle with U already shifted into place: mppib_shift computes the SIMPLE-mode g = lambda Sigma_H^-1 U of K3."""
    be = backend(case, dev(case.dist) if dist is None else dist, params)
    Ud = dev(shifted_from(U))
    be.shift(Ud)
    np.testing.assert_array_equal(Ud.cpu().numpy(), U)
    return be, Ud


def _white_z(case, seed, plan, k_offset, k_total, K):
    """K1's white Philox draws z [n][K] from the device: the fixed-Sigma K1 with identity colour, U = 0 and wide bounds returns
    1 * z + 0 * ... = z bit for bit (0 in the null row)."""
    wc = make_case(case.T, case.nu, K, kind="W", sigma=np.eye(case.nu))
    z = torch.zeros((case.T, case.nu, K), device=DEV)
    backend(wc).sample(seed, plan, k_offset, k_total, torch.zeros((case.T, case.nu), device=DEV), None, z, None)
    return z.cpu().numpy().reshape(case.n, K)


HZ_K1_CELLS = [(1, 1), (7, 1), (2, 4), (3, 3), (31, 1), (8, 4), (11, 3), (9, 7), (13, 5), (127, 1), (43, 3), (8, 16), (40, 5), (85, 3), (16, 16),
               (256, 1)]                                                      # n = 1 .. 256: the 32-row panels, 8-row warps and cend edges
HZ_K1_K = [1, 63, 64, 65, 1000]                                               # 64-sample tiles: one, ragged, exact, one over


def _hz_k1_check(case, L, z, U, ag, ng, K, label, prior=None):
    """The device's a and noise against the float64 colouring of z, per element; null row exact, prior row unclamped and exact, and
    every row must tell its own diagonal term apart."""
    n = case.n
    p = case.params
    a64 = np.asarray(U, np.float64).reshape(n, 1) + L.astype(np.float64) @ z.astype(np.float64)
    lo = np.tile(np.asarray(p.u_min[:case.nu], np.float64), case.T)[:, None]
    hi = np.tile(np.asarray(p.u_max[:case.nu], np.float64), case.T)[:, None]
    a_ref = np.clip(a64, lo, hi).astype(np.float32)
    gate = hz_k1_gate(L, z, U, a_ref)
    body = slice(0, max(K - 2, 0))
    ag, ng = ag.reshape(n, K), ng.reshape(n, K)
    err_a = np.abs(ag[:, body] - a_ref[:, body])
    n_ref = a_ref - np.asarray(U, np.float32).reshape(n, 1)
    err_n = np.abs(ng[:, body].astype(np.float64) - n_ref[:, body])
    gb = gate[:, body]
    ratio = float(max((err_a / gb).max(initial=0), (err_n / (gb + EPS * np.abs(n_ref[:, body]))).max(initial=0)))
    print(f"SHAPES {label} K1 worst |err| {err_a.max(initial=0):.2e}, worst err/gate {ratio:.3f}")
    assert np.all(err_a <= gb), label
    assert np.all(err_n <= gb + EPS * np.abs(n_ref[:, body])), label
    np.testing.assert_array_equal(ag[:, K - 1], 0)                            # null row
    if K >= 2 and prior is not None:
        np.testing.assert_array_equal(ag[:, K - 2], prior.reshape(-1))       # prior row, not clamped
        np.testing.assert_array_equal(ng[:, K - 2], (prior - U).reshape(-1).astype(np.float32))
    if K > 2:                                                                 # a reference without L_rr z_r in row r must miss
        d = np.diag(L).astype(np.float64)[:, None] * z[:, body]
        alt = np.clip(a64[:, body] - d, lo, hi)
        miss = (np.abs(ag[:, body] - alt) > gb).any(axis=1)
        assert miss.all(), f"{label}: rows {np.flatnonzero(~miss)[:8]} do not tell their diagonal term apart"
    return a_ref


@pytest.mark.parametrize("T,nu,K", [pytest.param(T, nu, K, id=f"hz-k1-T{T}nu{nu}-n{T * nu}-K{K}") for T, nu in HZ_K1_CELLS for K in HZ_K1_K])
def test_hz_k1_philox(T, nu, K):
    rng = np.random.default_rng(T * 31 + nu + K)
    case0 = make_case(T, nu, K, kind="H")
    lo, hi = _bounds(nu, case0.sigma, rng)
    case = make_case(T, nu, K, kind="H", u_min=lo, u_max=hi, sigma_h=["iid", "corr", 1e3][(T + nu) % 3])
    n, L = case.n, case.chol()
    U = rng.uniform(-0.05, 0.05, (T, nu)).astype(np.float32)
    prior = rng.uniform(-2, 2, (T, nu)).astype(np.float32)
    seed, plan0, ctr = 0x1_2345_6789, 2 ** 32 - 3, 5                       # seed and plan index >= 2^32, the plan through plan_ctr
    be = backend(case, dev(case.dist))
    a, nz = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    be.sample(seed, plan0, 0, K, dev(U), dev(prior), a, nz, torch.tensor([ctr], dtype=torch.int32, device=DEV))
    ag = a.cpu().numpy()
    z = _white_z(case, seed, plan0 + ctr, 0, K, K)
    _hz_k1_check(case, L, z, U, ag, nz.cpu().numpy(), K, f"hz-k1-T{T}nu{nu}-K{K}", prior)
    tight = np.tile(np.arange(nu) % 3 == 0, T)
    if K > 100:
        at = (ag.reshape(n, K)[tight, :-2] == np.tile(np.asarray(hi, np.float32), T)[tight][:, None]).mean()
        assert 0.05 < at < 0.95                                              # the clamp binds on part of the samples of the tight columns
    if K >= 2:                                                                # k_offset shards are bit-identical to one launch
        k1 = K // 3 + 1
        parts = []
        for off, kk in ((0, k1), (k1, K - k1)):
            pp = copy.copy(case.params); pp.K = kk
            aa = torch.zeros((T, nu, kk), device=DEV)
            backend(case, dev(case.dist), pp).sample(seed, plan0 + ctr, off, K, dev(U), dev(prior), aa, None)
            parts.append(aa.cpu().numpy())
        np.testing.assert_array_equal(np.concatenate(parts, axis=2), ag)


@pytest.mark.parametrize("T,nu", [(12, 7), (43, 3), (85, 3), (16, 16), (128, 2)])
def test_hz_k1_library(T, nu):
    """White Halton library at global indices up to 65 536, coloured by the live L_H."""
    from mppi_isaac_b200.planner.mppi import halton_spline_operator, halton_table
    K, k_total = 1000, 65536
    k_off = k_total - K
    nk = min(T // 4, 32)
    case = make_case(T, nu, K, mode="halton-spline", kind="H", sigma_h="corr")
    n, L = case.n, case.chol()
    be = backend(case, dev(case.dist))
    Z = torch.zeros((T, nu, K), device=DEV)
    be.noise_library(k_off, k_total, dev(halton_table(nk * nu, 11), torch.int32), dev(halton_spline_operator(T, nk)), nk, Z)
    rng = np.random.default_rng(T + nu)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    prior = rng.uniform(-1, 1, (T, nu)).astype(np.float32)
    a, nz = torch.zeros_like(Z), torch.zeros_like(Z)
    be.sample_library(k_off, k_total, dev(U), dev(prior), Z, a, nz)
    Zg = Z.cpu().numpy().reshape(n, K)
    _hz_k1_check(case, L, Zg, U, a.cpu().numpy(), nz.cpu().numpy(), K, f"hz-lib-T{T}nu{nu}", prior)


# (T, nu): n = 1, 64 | 65, 126, 128 | 129, 192 | 193, 195, 256 = 256 x 1 and 16 x 16; nu = 13 .. 16; SYRK tiles 1, 3, 6, 10
HZ_CELLS = [(1, 1), (64, 1), (5, 13), (9, 14), (32, 4), (43, 3), (12, 16), (193, 1), (13, 15), (256, 1), (16, 16)]
HZ_SIGMA = ["iid", "corr", 10.0, 1e3, 1e5]


def _hz_Ks(T, nu):
    n = T * nu
    Ks = [4, 36, last4_K(n), WS_W * NUM_SMS - 4, WS_W * NUM_SMS + 4, wrap_K(T, nu, "H")]
    return Ks + ([65536] if n in (64, 129, 256) else [])


def _hz_cases():
    out = []
    for ci, (T, nu) in enumerate(HZ_CELLS):
        for i, K in enumerate(_hz_Ks(T, nu)):
            mode, g = MODES[(i + ci) % len(MODES)]
            tag = "simple" if mode == "simple" else f"g{g:g}"
            sig = HZ_SIGMA[(i + 2 * ci) % len(HZ_SIGMA)]
            if mode == "simple" and not isinstance(sig, str) and sig > 10:
                # SIMPLE mode scores g.x with g = lambda Sigma_H^-1 U: at cond 1e3 .. 1e5 its float32 cancellation reaches lambda, and
                # the derived gate (rightly) no longer tells a dropped tile apart.  MEAN mode takes the ill-conditioned Sigma_H.
                sig = "corr"
            out.append(pytest.param(T, nu, K, mode, g, sig, id=hz_id(T, nu, K, tag)))
    return out


def _hz_run(case, cost, x, U):
    """reduce + finalize and the fused reduce_finalize from the same inputs: (row, U, action, stats, dist) of both, bit-equal."""
    out = []
    for fused in (False, True):
        dist = dev(case.dist)
        be, Ud = _hz_backend(case, U, dist)
        part, act, st = torch.zeros(case.row_floats(), device=DEV), torch.zeros(case.nu, device=DEV), torch.zeros(2, device=DEV)
        if fused:
            be.reduce_finalize(dev(cost), dev(x), Ud, part, act, st)
        else:
            be.reduce(dev(cost), dev(x), Ud, part)
            be.finalize(part.view(1, -1), 1, Ud, act, st)
        out.append([t.cpu().numpy() for t in (part, Ud, act, st, dist)])
    for a, b in zip(*out):
        np.testing.assert_array_equal(a, b)                                    # the SYRK-fused K4 is the two launches, bit for bit
    return out[0]


def _hz_check_dist(case, row, U, Ug, dg, label):
    """K4 of H on the device's own row against aho.finalize: U, lambda bit-equal, Sigma_H per entry, and L, Sigma_H^-1 on the device's
    own values (lower triangular, exactly symmetric, backward errors in n eps and cond)."""
    T, nu, n = case.T, case.nu, case.n
    U_ref, _, st_ref, d_ref = aho.finalize(case.model, case.params, row[None], U, case.dist)
    e = float(row[1])
    wm = np.abs(row[2:2 + n].astype(np.float64) / e) if e > 0 else 0.0
    gate_u = 32 * EPS * (np.abs(U).max() + np.max(wm) + 1e-30) * (2.0 if case.params.filter_u else 1.0)
    err_u = float(np.abs(Ug - U_ref).max())
    msg = f"SHAPES {label} K4 U worst {err_u:.2e} gate {gate_u:.2e}"
    assert err_u <= gate_u, msg
    assert dg[0] == d_ref[0], msg                                              # the lambda rule: the same float32 steps
    if not e > 0:
        np.testing.assert_array_equal(dg, case.dist)
        print(msg)
        return
    _, S, L, I = aho.unpack(dg, n)
    _, Sr, _, _ = aho.unpack(d_ref, n)
    W = row[2:2 + n].astype(np.float64) / e
    c = 0.0 if case.simple else U.astype(np.float64).reshape(n)
    a = np.abs(W) + np.abs(c) + np.abs(W - c)
    b = np.abs(U_ref - U).reshape(n) + np.abs(U).reshape(n) + np.abs(W)
    Cm = np.abs(aho.tril_unpack(row[2 + n:].astype(np.float64), n)) / e
    dV = EPS * (4 * Cm + 16 * np.outer(a + b, a + b))
    Sd = aho.unpack(case.dist, n)[1].astype(np.float64)
    dSn = float(case.params.step_size_cov) * dV + 4 * EPS * (np.abs(Sd) + float(case.params.kappa))
    gate_s = np.zeros((n, n))
    gate_s[:n - nu, :n - nu] = dSn[nu:, nu:]                                  # the shift: Sigma'[a][b] = Sigma_new[a + nu][b + nu]
    gate_s += 4 * EPS * np.abs(Sr)
    err_s = np.abs(S.astype(np.float64) - Sr)
    msg += f"; Sigma_H worst {err_s.max():.2e}, worst err/gate {(err_s / np.maximum(gate_s, 1e-300)).max():.3f}"
    assert np.all(err_s <= gate_s), msg
    np.testing.assert_array_equal(S, S.T)
    np.testing.assert_array_equal(I, I.T)
    np.testing.assert_array_equal(L, np.tril(L))
    L64, S64 = L.astype(np.float64), S.astype(np.float64)
    assert np.all(np.abs(L64 @ L64.T - S64) <= (n + 2) * EPS * (np.abs(L64) @ np.abs(L64).T)), msg
    assert np.abs(I.astype(np.float64) @ S64 - np.eye(n)).max() <= 4 * n * EPS * np.linalg.cond(S64), msg
    print(msg)


def _hz_check(case, cost, x, U, label, drop_check=False):
    S, w, ref = k3_restate(case, cost, x, U)
    gate = k3_gate(case, cost, x, U, S, w, sms=_sms())
    row, Ug, act, st, dg = _hz_run(case, cost, x, U)
    exc, err = row_excess(row, ref, gate)
    finite = np.isfinite(gate) & (gate > 0)
    rel = np.abs(row.astype(np.float64) - ref)
    n = case.n
    cpart = slice(2 + n, None)
    ratio = float((rel[:2 + n][finite[:2 + n]] / gate[:2 + n][finite[:2 + n]]).max(initial=0.0))
    cratio = float((rel[cpart][finite[cpart]] / gate[cpart][finite[cpart]]).max(initial=0.0))
    line = f"SHAPES {label} K3 worst err/gate {ratio:.3f}, C worst |err| {rel[cpart].max(initial=0):.2e} err/gate {cratio:.3f}"
    if drop_check:
        _, _, alt = k3_restate(case, cost, x, U, keep=drop_tail_mask(case.K))
        exc_alt, _ = row_excess(row[:2 + n], alt[:2 + n], gate[:2 + n])
        line += f", without the last tile by {exc_alt:.2e}"
        assert exc_alt > 0, line + ": the gate cannot tell the ragged tail apart"
        _, ksplit, kchunk = syrk_split(n, case.K, _sms())
        if ksplit > 1:
            worst = np.inf
            for s in range(ksplit):
                alt_c = ref[cpart] - hz_C(case, x, U, w, s * kchunk, min(case.K, (s + 1) * kchunk))
                worst = min(worst, row_excess(row[cpart], alt_c, gate[cpart])[0])
            line += f", without any one SYRK split by >= {worst:.2e}"
            assert worst > 0, line + ": the C gate cannot tell a SYRK split apart"
    print(line)
    assert exc <= 0, line
    np.testing.assert_array_equal(st, row[:2])
    np.testing.assert_array_equal(act, Ug[0])
    _hz_check_dist(case, row, U, Ug, dg, label)
    return row, Ug, st, dg


@pytest.mark.parametrize("T,nu,K,mode,gamma,sigma_h", _hz_cases())
def test_hz_k3_syrk_k4_sweep(T, nu, K, mode, gamma, sigma_h):
    case = make_case(T, nu, K, mode=mode, gamma=gamma, kind="H", filter_u=T >= 9, update_lambda=True, sigma_h=sigma_h)
    cost, x, U = k3_inputs(case, seed=31 * T + nu + K)
    _hz_check(case, cost, x, U, hz_id(T, nu, K, mode_tag(case)), drop_check=True)


HZ_EDGE_SHAPES = [(9, 7, "simple"), (16, 16, "halton-spline")]


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("T,nu,mode", HZ_EDGE_SHAPES, ids=[f"H-T{t}nu{n}-{m}" for t, n, m in HZ_EDGE_SHAPES])
def test_hz_edge_inputs(T, nu, mode, edge):
    K = {"cta": WS_W * NUM_SMS * 2 + 64, "underflow": WS_W * NUM_SMS * 4, "tie": 4228}.get(edge, 4228)
    lam = {"lam_tiny": 1e-4, "lam_large": 1e3}.get(edge, 0.5)
    base = make_case(T, nu, K, mode=mode, kind="H", lam=0.05 if edge == "lam_tiny" else 0.5)
    cost, x, U = k3_inputs(base, seed=7, favour_tail=edge != "lam_tiny")
    case = make_case(T, nu, K, mode=mode, kind="H", lam=lam, update_lambda=True)
    grid = min((K + WS_W - 1) // WS_W, NUM_SMS)
    if edge == "tie" and case.simple:
        pytest.skip("ties are built in MEAN mode")
    if edge == "nonfinite":
        cost[:, 3] = np.nan
        cost[5, 7] = np.inf
        cost[2, 11] = -np.inf
        cost[T - 1, K - 1] = np.nan
    elif edge == "tile":
        cost[:, 32:64] = np.nan
    elif edge == "cta":
        for k0 in range(5 * WS_W, K, grid * WS_W):
            cost[:, k0:k0 + WS_W] = np.nan
    elif edge == "none":
        cost[:] = np.nan
    elif edge == "one":
        keep = cost[:, 77].copy()
        cost[:] = np.nan
        cost[:, 77] = keep
    elif edge == "min_ragged":
        cost[0, K - 1] -= 3 * lam
    elif edge == "underflow":
        cost[0, (9 + 3 * grid) * WS_W + 5] -= 200 * lam
    elif edge == "tie":
        k1, k2 = 40, 40 + 7 * WS_W
        cost[0, k1] -= 50 * lam
        cost[:, k2], x[:, :, k2] = cost[:, k1], x[:, :, k1]
    row, Ug, st, dg = _hz_check(case, cost, x, U, f"hz-edge-{edge}-T{T}nu{nu}-K{K}-{mode_tag(case)}")
    n = case.n
    C = aho.tril_unpack(row[2 + n:], n)
    c = 0.0 if case.simple else U.reshape(n, 1)

    def dx(k):
        return (x.reshape(n, K)[:, k:k + 1] - c).astype(np.float32)            # fl(x - c)

    if edge == "none":
        assert row[0] == np.inf and row[1] == 0 and not row[2:].any()
        np.testing.assert_array_equal(dg, case.dist)
    elif edge in ("one", "underflow"):
        k = 77 if edge == "one" else (9 + 3 * grid) * WS_W + 5
        assert row[1] == 1.0
        np.testing.assert_array_equal(C, (dx(k) @ dx(k).T).astype(np.float32))   # exactly one sample's product
    elif edge == "tie":
        want = 2 * dx(40).astype(np.float64) @ dx(40).T.astype(np.float64)
        assert np.all(np.abs(C - want) <= 4 * EPS * np.abs(want))


@pytest.mark.parametrize("G", [2, 3, 5, 8])
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_hz_k4_combines_g_shard_rows(G, mode):
    """G shard rows (different beta, one shard all invalid) through one horizon K4 == one launch over all samples, and == aho.finalize."""
    T, nu, Ks = 16, 4, 1024
    K = G * Ks
    case = make_case(T, nu, K, mode=mode, kind="H", filter_u=True, update_lambda=True)
    cost, x, U = k3_inputs(case, seed=G, favour_tail=False)
    for g in range(G):
        cost[0, g * Ks:(g + 1) * Ks] += 0.7 * g * case.lam
    cost[:, (G - 1) * Ks:] = np.nan
    one = _hz_run(case, cost, x, U)
    pg = copy.copy(case.params); pg.K = Ks
    dist = dev(case.dist)
    be, Ud = _hz_backend(case, U, dist, pg)
    parts = torch.zeros((G, case.row_floats()), device=DEV)
    for g in range(G):
        sl = slice(g * Ks, (g + 1) * Ks)
        be.reduce(dev(cost[:, sl]), dev(x[:, :, sl]), Ud, parts[g])
    act, st = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(parts, G, Ud, act, st)
    rows = parts.cpu().numpy()
    assert rows[-1, 0] == np.inf and rows[-1, 1] == 0
    assert len(set(rows[:-1, 0].tolist())) == G - 1
    Ug, stg, dg = Ud.cpu().numpy(), st.cpu().numpy(), dist.cpu().numpy()
    gate = 4e-6 * max(1.0, np.abs(one[1]).max())
    err = float(np.abs(Ug - one[1]).max())
    err_d = float(np.abs(dg[1:] - one[4][1:]).max())
    print(f"SHAPES hz-k4-G{G}-{mode} U against one launch {err:.2e} gate {gate:.2e}, dist {err_d:.2e}")
    assert err <= gate
    assert stg[0] == one[3][0] and abs(stg[1] - one[3][1]) <= 1e-5 * one[3][1]
    assert err_d <= 2e-5 * np.abs(one[4][1:]).max()
    U_ref, _, st_ref, d_ref = aho.finalize(case.model, case.params, rows, U, case.dist)
    assert np.abs(Ug - U_ref).max() <= gate and stg[0] == st_ref[0] and dg[0] == d_ref[0]
    np.testing.assert_allclose(dg[1:], d_ref[1:], rtol=0, atol=2e-5 * np.abs(d_ref[1:]).max())


def _hz_finalize_row(case, row, U):
    be = backend(case, dev(case.dist))
    dd = be._dist_keepalive
    Ud, act, st = dev(U), torch.zeros(case.nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(dev(row).view(1, -1), 1, Ud, act, st)
    return dd.cpu().numpy(), Ud.cpu().numpy()


@pytest.mark.parametrize("what", ["fixed_point", "T1", "one_sample", "pivot_first", "pivot_mid", "pivot_last", "nan"])
def test_hz_k4_known_answers(what):
    """Hand-built rows through the horizon K4, set on the parameter block directly."""
    T, nu = (1, 5) if what == "T1" else (12, 3)
    n = T * nu
    P = 2 + n + n * (n + 1) // 2
    case = make_case(T, nu, 64, mode="simple", kind="H", sigma_h="iid" if what == "fixed_point" else "corr", update_lambda=True,
                     eta_u_bound=10.0, eta_l_bound=5.0)
    p = case.params
    rng = np.random.default_rng(n)
    S0 = np.asarray(p.sigma0[:nu * nu], np.float32).reshape(nu, nu)
    U = np.zeros((T, nu), np.float32)
    row = np.zeros(P, np.float32)
    row[1] = 1.0
    if what in ("fixed_point", "T1"):
        xv = rng.normal(0, 0.3, n)
        row[2:2 + n] = xv
        row[2 + n:] = aho.tril_pack(np.outer(xv, xv) + rng.normal(0, 0.01, (n, n)))
        if what == "fixed_point":
            p.step_size_cov, p.kappa = 0.0, 0.0
        d, _ = _hz_finalize_row(case, row, U)
        _, S, L, I = aho.unpack(d, n)
        if what == "fixed_point":
            np.testing.assert_array_equal(S, aho.unpack(case.dist, n)[1])     # I_T (x) Sigma0 is a fixed point, bit for bit
        else:
            np.testing.assert_array_equal(S, S0)                              # T = 1: Sigma' = Sigma0 for any row
        assert np.abs(L.astype(np.float64) @ L.T.astype(np.float64) - S).max() <= (n + 2) * EPS * np.abs(S).max()
        return
    if what == "one_sample":
        # SIMPLE, one valid sample x with exact products, U = 0, step_size_cov = 1: V = C - x x^T = 0, Sigma' = kappa I (+) Sigma0
        p.step_size_cov = 1.0
        xv = rng.choice([-1.0, -0.5, 0.25, 0.5, 1.0], n).astype(np.float32)
        row[2:2 + n] = xv
        row[2 + n:] = aho.tril_pack(np.outer(xv, xv))
        d, _ = _hz_finalize_row(case, row, U)
        _, S, L, _ = aho.unpack(d, n)
        m = n - nu
        kap = np.float32(p.kappa)
        want = np.zeros((n, n), np.float32)
        want[:m, :m] = kap * np.eye(m, dtype=np.float32)
        want[m:, m:] = S0
        np.testing.assert_array_equal(S, want)
        np.testing.assert_array_equal(L[:m, :m], np.sqrt(kap) * np.eye(m, dtype=np.float32))
        np.testing.assert_array_equal(L[m:, :m], 0)
        L0 = np.linalg.cholesky(S0.astype(np.float64))
        assert np.abs(L[m:, m:] - L0).max() <= (nu + 2) * EPS * np.abs(L0).max()
        return
    # a shifted update that is not positive definite (pivot k fails first) or holds a NaN: Sigma, L, Sigma^-1 bit-unchanged
    p.step_size_cov = 1.0
    Cd = np.eye(n)
    k = {"pivot_first": 0, "pivot_mid": (n - nu) // 2, "pivot_last": n - nu - 1, "nan": None}[what]
    if k is not None:
        Cd[k + nu, k + nu] = -1.0                                             # Sigma'[k][k] = C[k + nu][k + nu] + kappa < 0
    else:
        Cd[nu + 4, nu + 1] = np.nan
    row[2 + n:] = aho.tril_pack(Cd)
    d, _ = _hz_finalize_row(case, row, U)
    _, _, _, d_ref = aho.finalize(case.model, p, row[None], U, case.dist)
    np.testing.assert_array_equal(d[1:], case.dist[1:])
    np.testing.assert_array_equal(d_ref[1:], case.dist[1:])
    assert d[0] == d_ref[0] == np.float32(case.dist[0]) * (np.float32(1) + np.float32(p.lambda_mult))   # eta = 1 < eta_l_bound


def _hz_row(be, case, cost, x, Ud):
    part = torch.zeros(case.row_floats(), device=DEV)
    be.reduce(dev(cost), dev(x), Ud, part)
    return part.cpu().numpy()


def test_hz_reuse_and_resize():
    """Three plans on one handle give the same row (the SYRK tickets reset); handles of n = 36 and n = 256 interleaved on one device
    give a fresh handle's rows; set_params to a new K with the same n re-sizes hz_S and gives a fresh handle's row."""
    cases = {}
    for T, nu in ((12, 3), (16, 16)):
        c = make_case(T, nu, 4228, mode="simple", kind="H")
        cost, x, U = k3_inputs(c, seed=T)
        cases[T] = (c, cost, x, U)
    fresh = {}
    for T, (c, cost, x, U) in cases.items():
        be, Ud = _hz_backend(c, U)
        fresh[T] = _hz_row(be, c, cost, x, Ud)
        for _ in range(2):
            np.testing.assert_array_equal(_hz_row(be, c, cost, x, Ud), fresh[T])
    live = {T: _hz_backend(c, U) for T, (c, cost, x, U) in cases.items()}
    for _ in range(2):
        for T, (c, cost, x, U) in cases.items():
            be, Ud = live[T]
            np.testing.assert_array_equal(_hz_row(be, c, cost, x, Ud), fresh[T])
    c, cost, x, U = cases[12]
    be, Ud = live[12]
    for K2 in (65536, 36):
        c2 = make_case(c.T, c.nu, K2, mode="simple", kind="H")
        cost2, x2, _ = k3_inputs(c2, seed=K2)
        be.set_params(c2.params)
        Ud.copy_(dev(shifted_from(U)))                                       # hz_g is re-allocated with hz_S: shift into U again
        be.shift(Ud)
        got = _hz_row(be, c2, cost2, x2, Ud)
        bf, Uf = _hz_backend(c2, U)
        np.testing.assert_array_equal(got, _hz_row(bf, c2, cost2, x2, Uf))


@pytest.mark.parametrize("kind,T,K,plans", [("point", 85, 4096, 6)])
def test_hz_planner_tracks_the_reference(kind, T, K, plans):
    """Lock-step with AdaptiveHorizonOracleBackend at n = 255 (point robot, T = 85), filter_u and graph capture: the reference plans
    from the device's U and dist every plan."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    from scenes import point_cfg
    flags = dict(update_cov=True, update_lambda=True, cov_type="horizon", filter_u=True, eta_u_bound=40.0, eta_l_bound=4.0)
    gpu = MPPIisaacPlanner(point_cfg(K=K, T=T, device=DEV, **flags), PointReachObjective(), use_cuda_graph=True)
    cpu = MPPIisaacPlanner(point_cfg(K=K, T=T, device="cpu", **flags), PointReachObjective(), backend=aho.AdaptiveHorizonOracleBackend(nthreads=NTHREADS))
    q, qd = [0.1, 0.0, 0.0], [0.0] * 3
    n = gpu.mppi.T * gpu.mppi.nu
    assert n == 255
    d0 = gpu.mppi.dist.cpu().clone()
    worst = [0.0, 0.0]
    for it in range(plans):
        cpu.mppi.U.copy_(gpu.mppi.U.cpu())
        cpu.mppi.dist.copy_(gpu.mppi.dist.cpu())
        ag, ac = gpu.compute_action(q, qd), cpu.compute_action(q, qd)
        S_g, S_c = gpu.mppi.cov_action.cpu().numpy().astype(np.float64), cpu.mppi.cov_action.numpy().astype(np.float64)
        rel = np.abs(S_g - S_c).max() / max(1.0, np.abs(S_c).max())
        worst = [max(worst[0], float((ag.cpu() - ac).abs().max())), max(worst[1], rel)]
        assert float((ag.cpu() - ac).abs().max()) <= 5e-4, f"plan {it}"
        np.testing.assert_allclose(float(gpu.mppi.current_lambda), float(cpu.mppi.current_lambda), rtol=1e-5, err_msg=f"plan {it}")
        assert rel <= 1e-4, f"plan {it}"
    print(f"SHAPES hz-planner-{kind}-T{T}-K{K} worst action {worst[0]:.2e}, Sigma_H {worst[1]:.2e} relative")
    assert gpu.mppi._graph is not None
    assert not torch.equal(gpu.mppi.dist.cpu(), d0)


@pytest.mark.parametrize("what", ["n257", "K6", "set_params_T", "set_model_nu"])
def test_hz_host_refuses(what):
    """Refused on the host with an error, before any launch: n = 257 in a hand-built parameter block, K % 4 != 0 in the horizon reduce,
    and a registered horizon distribution that a new (T, nu) would outgrow."""
    case = make_case(12, 3, 64, kind="H")
    if what == "n257":
        from mppi_isaac_b200.backend import CudaBackend
        big = make_case(256, 1, 64, kind="H")
        p = copy.copy(big.params)
        p.T = 257
        with pytest.raises(RuntimeError, match="n = T\\*nu = 257 exceeds 256"):
            CudaBackend(DEV).create(nu_model(1), p)
        return
    if what == "K6":
        c6 = make_case(12, 3, 6, kind="H")
        be = backend(c6, dev(c6.dist))
        with pytest.raises(RuntimeError, match="K=6"):
            be.reduce(torch.zeros((12, 6), device=DEV), torch.zeros((12, 3, 6), device=DEV), torch.zeros((12, 3), device=DEV),
                      torch.zeros(c6.row_floats(), device=DEV))
        torch.cuda.synchronize()
        return
    be = backend(case, dev(case.dist))
    launches = be.launches
    if what == "set_params_T":
        p = copy.copy(case.params)
        p.T = 13
        with pytest.raises(RuntimeError, match="mppib_set_params: the registered distribution holds 3889 floats"):
            be.set_params(p)
    else:
        with pytest.raises(RuntimeError, match="mppib_set_model: the registered distribution holds 3889 floats"):
            be.set_model(nu_model(4))
        be.set_model(nu_model(3))                                             # a model that keeps nu goes on working
    assert be.params.T == 12 and be.model.nu == 3 and be.launches == launches
