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
import adaptive_oracle as ada
from synth_mppi import (EPS, KINDS, NUM_SMS, WS_W, drop_tail_mask, k3_gate, k3_id, k3_inputs, k3_restate, make_case, mode_tag, row_excess,
                        wrap_K, ws_layout)

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
@pytest.mark.parametrize("what", ["Tnu513", "T257", "K6", "m2_256x2", "knots33", "gamma_neg", "gamma_nan"])
def test_host_refuses_unsupported_shapes(what):
    """Refused on the host with an error, before any launch."""
    from mppi_isaac_b200.planner.mppi import halton_spline_operator, halton_table
    shapes = {"Tnu513": (57, 9, 64, "W"), "T257": (257, 1, 64, "W"), "K6": (8, 2, 6, "W"), "m2_256x2": (256, 2, 64, "M2"),
              "knots33": (132, 2, 64, "W"), "gamma_neg": (8, 2, 64, "W"), "gamma_nan": (8, 2, 64, "W")}
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
    match = {"Tnu513": "T\\*nu = 513", "T257": "T = 257", "K6": "K=6", "m2_256x2": "second-moment row"}[what]
    with pytest.raises(RuntimeError, match=match):
        be.reduce(cost, x, U, part)
    with pytest.raises(RuntimeError, match=match):
        be.reduce_finalize(cost, x, U, part, torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV))
    torch.cuda.synchronize()
