"""-m gpu: the kernels of the colored, CEM, smooth and risk-aware modes over every template instantiation and the accepted (T, nu, K)
range, against the float64 references (``risk_oracle``, ``smooth_oracle``, ``cem_oracle``, ``colored_oracle``, the adaptive ones), on
the generated cases of ``synth_mppi`` (the point robot's model with nu set; no dynamics run).

The K3 sweeps are gated per case by a float32 bound derived from the kernel's summation orders (``_row_gate``: the k3_gate reasoning,
with the m-term tail sum of the CVaR score under risk and the smoothness term of mode smooth), and every sweep case must also miss that
gate against a deliberately wrong reference.  Each case prints a ``MODES <id> worst ... gate ...`` line (shown with -s)."""
import copy

import numpy as np
import pytest
import torch

import adaptive_full_oracle as afo
import adaptive_oracle as ada
import cem_oracle as ce
import risk_oracle as ro
import smooth_oracle as so
from mppi_isaac_b200.model.blob import MODE_SIMPLE, make_params
from mppi_isaac_b200.planner.mppi import colored_noise_chol
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from synth_mppi import EPS, NUM_SMS, WS_W, drop_tail_mask, k3_dS, k3_inputs, make_case, nu_model, row_excess, wrap_K, ws_layout
from test_gpu_colored import _check_case, drop_one_term
from test_gpu_mppi_shapes import _check_k4, _run_k3
from test_gpu_smooth import k1_gate as smooth_k1_gate
from test_gpu_smooth import k4_check as smooth_k4_check

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED, PLAN = 0x1_2345_6789, 2 ** 32 + 7


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def backend(model, p, dist=None, smooth=None):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(model, p)
    if dist is not None:
        be.set_distribution(dist)
    if smooth is not None:
        be.set_smooth_state(smooth)
    return be


def white(model, p, nu, K, seed=SEED, plan=PLAN, k_offset=0, k_total=None):
    """The device's own white draws z[T][nu][K]: the fixed-Sigma K1 in mode simple with identity colour, no bounds, no null row."""
    w = copy.deepcopy(p)
    w.mode, w.sample_null_action, w.smooth_weight, w.n_worlds, w.risk_tail, w.update_cov, w.cov_full = MODE_SIMPLE, 0, 0.0, 0, 0, 0, 0
    for j in range(nu):
        w.u_min[j], w.u_max[j] = -3e38, 3e38
        for i in range(nu):
            w.sigma_chol[j * nu + i] = 1.0 if i == j else 0.0
    z = torch.zeros((p.T, nu, K), device=DEV)
    backend(model, w).sample(seed, plan, k_offset, k_total or K, torch.zeros((p.T, nu), device=DEV), None, z, None)
    return z.cpu().numpy()


def _row_gate(S, dS, w, b, rows, lam, K, ncons, sms=NUM_SMS):
    """The k3_gate bound on (beta, eta, W) of a row whose weights w_j = exp(-(S_j - b) / lambda) (w_j = 0 for an invalid j) come from
    float32 scores within dS_j of S: a weight moves at most to exp(-(S_j - b - dS_j - db) / lambda), the weighted sums then carry that
    spread plus the rounding of their own accumulation over K samples in 32-sample tiles on min(tiles, sms) CTAs of ncons consumer
    warps.  rows: [r][j] the vectors the row sums.  Returns (gate, dw, w_hi)."""
    ntiles = (K + WS_W - 1) // WS_W
    grid = min(ntiles, sms)
    per_warp = -(-(-(-ntiles // grid)) // ncons)
    rho = EPS * (64 + 3 * per_warp + grid / 4)
    ok = w > 0
    db = float(dS[ok].max()) if ok.any() else 0.0
    with np.errstate(over="ignore", invalid="ignore"):
        w_hi = np.where(ok, np.exp(np.minimum(-(np.where(ok, S, b) - b - dS - db) / lam, 700.0)), 0.0)
    dw = (w_hi - w) + w * rho
    gate = np.concatenate([[db + EPS * abs(b) if ok.any() else 0.0, dw.sum() + EPS * w.sum()], np.abs(rows) @ dw + EPS * np.abs(rows @ w)])
    return gate, dw, w_hi


def _line(label, row, ref, gate):
    exc, err = row_excess(row, ref, gate)
    fin = np.isfinite(gate) & (gate > 0)
    ratio = float((np.abs(row.astype(np.float64) - ref)[fin] / gate[fin]).max(initial=0.0))
    return exc, f"MODES {label} worst |err| {err:.2e} worst err/gate {ratio:.3f} gate of eta {gate[1]:.2e}"


# ------------------------------------------------------------------------------------------------------------------------------ risk
# (T, nu) cells: T*nu = 1, 16 (T = 1), 128 | 129 (RPL 4 | 8), 256 | 258 (RPL 8 | 16; 257 is prime, so T = 257 would be needed), 512 at
# T = 32 and at T = 256 (the second-moment row there runs two ring stages and two consumers)
RISK_CELLS = [(1, 1), (1, 16), (32, 4), (43, 3), (16, 16), (129, 2), (32, 16), (256, 2)]
RISK_KINDS = {"fixed": "W", "diag": "M2", "full": "C"}
RS = [2, 4, 8, 16, 32]
GAMMAS = [0.5, 0.95, 1.05]


def _risk_Ks(T, nu, kind, R):
    u = max(R, 4)                                                              # K3 needs K a multiple of 4, the worlds one of R
    return [("two", 2 * R), ("ragged", WS_W * 37 + (u if R < WS_W else 0)), ("sms-", WS_W * NUM_SMS - 32), ("sms+", WS_W * NUM_SMS + 32),
            ("wrap", wrap_K(T, nu, RISK_KINDS[kind]) // u * u)]


def _risk_cases():
    out, i = [], 0
    for T, nu in RISK_CELLS:
        for kind in RISK_KINDS:
            for ki in range(4):
                R = RS[i % 5]
                m = [1, max(R // 2, 1), R][(i // 5) % 3]
                mode = ["simple", "halton-spline"][i % 2]
                g = GAMMAS[(i // 2) % 3]
                name, K = _risk_Ks(T, nu, kind, R)[ki if ki < 2 else (2 + (i % 2) if ki == 2 else 4)]
                i += 1
                tag = "simple" if mode == "simple" else f"g{g:g}"
                rpl, ncons, _, _ = ws_layout(T, nu, RISK_KINDS[kind])
                out.append(pytest.param(T, nu, K, kind, R, m, mode, g, id=f"risk-RPL{rpl}-{kind}-T{T}nu{nu}-ncons{ncons}-R{R}m{m}-{name}K{K}-{tag}"))
    return out


def risk_case(T, nu, K, kind, R, m, mode="simple", gamma=0.95):
    return make_case(T, nu, K, mode=mode, gamma=gamma, kind=RISK_KINDS[kind], update_lambda=kind != "fixed", n_worlds=R, cvar_alpha=m / R)


def risk_inputs(case, R, seed):
    """k3_inputs (the last tile favoured) with +inf costs: one rollout of one group, and the m worst worlds of another."""
    cost, x, U = k3_inputs(case, seed=seed)
    Kc, m = case.K // R, int(case.params.risk_tail)
    if Kc >= 4:
        rng = np.random.default_rng(seed)
        g1, g2 = rng.choice(Kc - 2, 2, replace=False)
        cost[rng.integers(case.T), g1 * R + rng.integers(R)] = np.inf
        cost[0, g2 * R + R - m:g2 * R + R] = np.inf
    return cost, x, U


def risk_restate(case, cost, x, U, m=None, keep=None):
    """float64 risk K3 of the case: per-rollout S, control scores rho (risk_oracle), control weights, beta and the shard row; `m`
    overrides the tail, `keep` masks controls out."""
    p, nu, T, R = case.params, case.nu, case.T, int(case.params.n_worlds)
    m = int(p.risk_tail) if m is None else m
    S, lam = ro.scores(p, nu, cost, x, U, case.dist)
    rho = ro.rho(S, R, m)
    ok = np.isfinite(rho) if keep is None else np.isfinite(rho) & keep
    b = rho[ok].min() if ok.any() else np.inf
    w = np.where(ok, np.exp(-(np.where(ok, rho, b) - b) / lam), 0.0)
    xc = np.asarray(x, np.float64).reshape(T * nu, -1)[:, ::R]
    row = [np.array([b, w.sum()]), xc @ w]
    c = 0.0 if case.simple else np.asarray(U, np.float64).reshape(-1, 1)
    if case.kind == "M2":
        row.append(((xc - c) ** 2) @ w)
    elif case.kind == "C":
        d = (xc - c).reshape(T, nu, -1).transpose(1, 0, 2).reshape(nu, -1)
        row.append(((d * np.tile(w, T)[None]) @ d.T)[np.tril_indices(nu)])
    return S, rho, w, b, xc, np.concatenate(row)


def risk_gate(case, cost, x, U, S, rho, w, b, xc):
    """The row gate of the CVaR score: rho_c is the float32 tail of m sorted scores, each within dS (k3_dS) of its float64 value; the
    sum of the m largest moves by at most m max dS, and its m - 1 additions and the division round (m + 1) eps of sum |top|."""
    R, m, T, nu, lam = int(case.params.n_worlds), int(case.params.risk_tail), case.T, case.nu, case.lam
    dS = k3_dS(case, cost, x, U)
    Sg = np.where(np.isfinite(S), S, np.inf).reshape(-1, R)
    top = np.abs(-np.sort(-Sg, axis=1)[:, :m])
    with np.errstate(invalid="ignore"):
        drho = dS.reshape(-1, R).max(1) + (m + 2) * EPS * np.where(np.isfinite(top), top, 0).mean(1)
    _, ncons, _, _ = ws_layout(T, nu, case.kind)
    gate, dw, _ = _row_gate(rho, drho, w, b, xc, lam, case.K, ncons)
    c = 0.0 if case.simple else np.asarray(U, np.float64).reshape(-1, 1)
    if case.kind == "M2":
        d2 = (xc - c) ** 2
        gate = np.concatenate([gate, d2 @ (dw + 4 * EPS * w) + EPS * (d2 @ w)])
    elif case.kind == "C":
        d = np.abs(xc - c).reshape(T, nu, -1).transpose(1, 0, 2).reshape(nu, -1)
        M = (d * np.tile(dw + (T + 8) * EPS * w, T)[None]) @ d.T + EPS * ((d * np.tile(w, T)[None]) @ d.T)
        gate = np.concatenate([gate, M[np.tril_indices(nu)]])
    return gate


@pytest.mark.parametrize("T,nu,K,kind,R,m,mode,gamma", _risk_cases())
def test_risk_k3_k4_sweep(T, nu, K, kind, R, m, mode, gamma):
    case = risk_case(T, nu, K, kind, R, m, mode, gamma)
    assert int(case.params.risk_tail) == m
    cost, x, U = risk_inputs(case, R, seed=31 * T + nu + K + R)
    S, rho, w, b, xc, ref = risk_restate(case, cost, x, U)
    gate = risk_gate(case, cost, x, U, S, rho, w, b, xc)
    d = None if case.dist is None else case.dist
    np.testing.assert_allclose(ro.reduce(case.params, nu, cost, x, U, d), ref, rtol=EPS, atol=1e-9 * np.abs(ref[1:]).max())
    row, Ug, act, st, dg = _run_k3(case, cost, x, U)                           # fused == split, bit for bit
    label = f"risk-{kind}-T{T}nu{nu}-R{R}m{m}-K{K}-{mode}"
    exc, line = _line(label, row, ref, gate)
    if m > 1:                                                                  # a reference with one tail term dropped
        alt = risk_restate(case, cost, x, U, m=m - 1)[-1]
        what = "one tail term"
    else:                                                                      # a reference without the last control
        keep = np.ones(K // R, bool)
        keep[-1] = False
        alt = risk_restate(case, cost, x, U, keep=keep)[-1]
        what = "the last group"
    exc_alt, _ = row_excess(row, alt, gate)
    line += f", the reference without {what} misses it by {exc_alt:.2e}"
    print(line)
    assert exc <= 0, line
    assert exc_alt > 0, line + ": the gate cannot tell it apart"
    _check_k4(case, row, Ug, act, st, dg, U, label)                            # U, lambda and Sigma against the float64 finalize
    if K >= 4 * R:                                                             # a shard at k_offset = 3R: the same row
        p = copy.copy(case.params)
        p.k_offset = 3 * R
        be = backend(case.model, p, None if case.dist is None else dev(case.dist))
        part = torch.zeros(case.row_floats(), device=DEV)
        be.reduce(dev(cost), dev(x), dev(U), part)
        np.testing.assert_array_equal(part.cpu().numpy(), row)


@pytest.mark.parametrize("G", [1, 2, 3, 5])
@pytest.mark.parametrize("kind", list(RISK_KINDS))
def test_risk_k4_shard_rows_against_float64(kind, G):
    """G shard rows of risk_oracle.reduce (shards at k_offset = a multiple of R, each with its own beta) through the device K4 against
    the float64 finalize of the same rows: U, the lambda rule bit for bit, the diag / full Sigma update; for G = 1 the fused launch
    equals the split one."""
    T, nu, R, m, Ks = 16, 5, 8, 3, 512
    K = G * Ks
    case = risk_case(T, nu, K, kind, R, m, "halton-spline" if G % 2 else "simple")
    cost, x, U = risk_inputs(case, R, seed=G)
    rows = []
    for g in range(G):
        sl = slice(g * Ks, (g + 1) * Ks)
        pg = copy.copy(case.params)
        pg.K, pg.k_offset = Ks, g * Ks
        cg = np.ascontiguousarray(cost[:, sl]) - 0.5 * g * case.lam
        rows.append(ro.reduce(pg, nu, cg, np.ascontiguousarray(x[:, :, sl]), U, case.dist))
    rows = np.stack(rows)
    dist = None if case.dist is None else dev(case.dist)
    be = backend(case.model, case.params, dist)
    Ud, act, st = dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(dev(rows), G, Ud, act, st)
    Ug, stg = Ud.cpu().numpy(), st.cpu().numpy()
    b = rows[rows[:, 1] > 0, 0].min()                                           # the combined row, as K4 forms it
    s = np.where(rows[:, 1] > 0, np.exp(-(rows[:, 0].astype(np.float64) - b) / case.lam), 0.0)
    comb = (s[:, None] * rows.astype(np.float64)).sum(0)
    if kind == "fixed":
        from oracle import oracle as orc
        U_ref, _, st_ref = orc.finalize(case.model, case.params, rows, U)
    else:
        U_ref, _, st_ref, d_ref = (ada if kind == "diag" else afo).finalize(case.model, case.params, rows, U, case.dist)
        dg = dist.cpu().numpy()
        assert dg[0] == d_ref[0]                                               # the lambda rule: the same float32 steps
        gate_d = 2e-5 * np.abs(d_ref[1:]).max()
        print(f"MODES risk-k4-{kind}-G{G} dist worst {np.abs(dg[1:] - d_ref[1:]).max():.2e} gate {gate_d:.2e}")
        np.testing.assert_allclose(dg[1:], d_ref[1:], rtol=0, atol=gate_d)
    gate_u = 32 * EPS * (np.abs(U).max() + np.abs(comb[2:2 + T * nu] / comb[1]).max()) * G
    err = float(np.abs(Ug - U_ref).max())
    print(f"MODES risk-k4-{kind}-G{G} U worst {err:.2e} gate {gate_u:.2e}")
    assert err <= gate_u
    assert stg[0] == st_ref[0]
    if G == 1:
        out = []
        for fused in (False, True):
            dd = None if case.dist is None else dev(case.dist)
            bb = backend(case.model, case.params, dd)
            part, Uf, a1, s1 = torch.zeros(case.row_floats(), device=DEV), dev(U), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
            if fused:
                bb.reduce_finalize(dev(cost), dev(x), Uf, part, a1, s1)
            else:
                bb.reduce(dev(cost), dev(x), Uf, part)
                bb.finalize(part.view(1, -1), 1, Uf, a1, s1)
            out.append([t.cpu().numpy() for t in (part, Uf, a1, s1)] + ([dd.cpu().numpy()] if dd is not None else []))
        for a, c in zip(*out):
            np.testing.assert_array_equal(a, c)


# ------------------------------------------------------------------------------------------------------------------------------ smooth
# the risk cells plus shapes where the smoothness term's U region costs the ring a stage (fewer consumers than SIMPLE's)
SMOOTH_CELLS = [(1, 1), (1, 16), (32, 4), (43, 3), (16, 16), (129, 2), (32, 16), (256, 2), (145, 1), (186, 2), (20, 16)]
OMEGAS = [0.0, 0.5, 10.0]


def smooth_params(nu, T, K, k_offset=0, **kw):
    d = dict(num_samples=K, horizon=T, mppi_mode="smooth", sampling_method="random", noise_sigma=(0.3 * np.eye(nu) + 0.05).tolist(),
             u_min=[-0.2], u_max=[0.2], du_min=[-1.0], du_max=[1.0], lambda_=0.05, sample_null_action=True, smooth_weight=0.5)
    d.update(kw)
    p = make_params(MPPIConfig(**d), IsaacGymConfig(), nu, K, [])
    p.k_offset = k_offset
    return p


def _smooth_k3_cases():
    out, i = [], 0
    for T, nu in SMOOTH_CELLS:
        for name in ("36", "sms-", "sms+", "wrap"):
            om = OMEGAS[i % 3]
            i += 1
            K = {"36": 36, "sms-": WS_W * NUM_SMS - 4, "sms+": WS_W * NUM_SMS + 4}.get(name) or wrap_K(T, nu, "W", smooth=om != 0)
            rpl, ncons, _, _ = ws_layout(T, nu, "W", smooth=om != 0)
            out.append(pytest.param(T, nu, K, om, id=f"smooth-RPL{rpl}-T{T}nu{nu}-ncons{ncons}-K{K}-w{om:g}"))
    return out


def smooth_restate(p, nu, cost, x, U, keep=None):
    S = so.scores(p, nu, cost, x, U)
    lam = float(np.float32(p.lambda_))
    ok = np.isfinite(S) if keep is None else np.isfinite(S) & keep
    b = S[ok].min() if ok.any() else np.inf
    w = np.where(ok, np.exp(-(np.where(ok, S, b) - b) / lam), 0.0)
    xr = np.asarray(x, np.float64).reshape(p.T * nu, -1)
    return S, w, b, xr, np.concatenate([[b, w.sum()], xr @ w])


@pytest.mark.parametrize("T,nu,K,omega", _smooth_k3_cases())
def test_smooth_k3_sweep(T, nu, K, omega):
    """The smooth K3 (RPL 4 / 8 / 16) with the ring and consumers of its own layout; gate: SIMPLE's dS (k3_dS of the SIMPLE twin, gamma
    = 1) plus the smoothness term's: (NR/4 + 8) eps omega dt^2 sum_r (U_r + x_rk)^2 and 2 eps |S_k|.  The reference without the last
    tile must miss it; with omega = 0 the row is SIMPLE's bit for bit."""
    twin = make_case(T, nu, K, mode="simple", sigma=0.3 * np.eye(nu) + 0.05, lam=1.0)
    cost, x, U = k3_inputs(twin, seed=7 * T + nu + K)
    p = smooth_params(nu, T, K, smooth_weight=omega, lambda_=1.0)              # lambda 1: omega = 10 spreads S by about lambda / 4
    S, w, b, xr, ref = smooth_restate(p, nu, cost, x, U)
    wq = float(np.float32(p.smooth_weight)) * float(np.float32(p.dt)) ** 2
    q = ((U.astype(np.float64).reshape(-1, 1) + xr) ** 2).sum(0)
    dS = k3_dS(twin, cost, x, U) + EPS * ((T * nu / 4 + 8) * wq * q + 2 * np.abs(S))
    _, ncons, _, _ = ws_layout(T, nu, "W", smooth=omega != 0)
    gate, _, _ = _row_gate(S, dS, w, b, xr, float(np.float32(p.lambda_)), K, ncons)
    st = so.make_state(p, nu)
    be = backend(nu_model(nu), p, smooth=dev(st))
    part = torch.zeros(2 + T * nu, device=DEV)
    be.reduce(dev(cost), dev(x), dev(U), part)
    row = part.cpu().numpy()
    exc, line = _line(f"smooth-T{T}nu{nu}-K{K}-w{omega:g}", row, ref, gate)
    alt = smooth_restate(p, nu, cost, x, U, keep=drop_tail_mask(K))[-1]
    exc_alt, _ = row_excess(row, alt, gate)
    line += f", the reference without the last tile misses it by {exc_alt:.2e}"
    print(line)
    assert exc <= 0, line
    assert exc_alt > 0, line + ": the gate cannot tell the ragged tail apart"
    if omega == 0.0:                                                           # the smooth K3 without its term is SIMPLE's, bit for bit
        w_ = copy.deepcopy(p)
        w_.mode = MODE_SIMPLE
        ps = torch.zeros(2 + T * nu, device=DEV)
        backend(nu_model(nu), w_).reduce(dev(cost), dev(x), dev(U), ps)
        np.testing.assert_array_equal(row.view(np.uint32), ps.cpu().numpy().view(np.uint32))


SMOOTH_K1_NU = [1, 2, 5, 8, 13, 16]
BOUNDS = {"free": dict(u_min=[-1e30], u_max=[1e30], du_min=None, du_max=None), "action": dict(u_min=[-0.05], u_max=[0.08], du_min=None, du_max=None),
          "derivative": dict(u_min=[-1e30], u_max=[1e30], du_min=[-0.3], du_max=[0.2]), "both": dict(u_min=[-0.05], u_max=[0.05], du_min=[-0.6], du_max=[0.4])}
SMOOTH_K1_K = [1, 31, 33, 1000]


def _smooth_k1_cases():
    out, i = [], 0
    for nu in SMOOTH_K1_NU:
        for T in sorted({1, 9, min(512 // nu, 256)}):
            for bounds in BOUNDS:
                K = SMOOTH_K1_K[i % 4]
                i += 1
                out.append(pytest.param(T, nu, K, bounds, id=f"smooth-k1-{bounds}-T{T}nu{nu}-K{K}"))
    return out


@pytest.mark.parametrize("T,nu,K,bounds", _smooth_k1_cases())
def test_smooth_k1_sweep(T, nu, K, bounds):
    """The smooth K1 against so.sample on the device's own white draws, within the gate of test_gpu_smooth; a reference integrated from 0
    instead of a_prev must miss it; shards that split K are bit-identical to one launch."""
    p = smooth_params(nu, T, K, **BOUNDS[bounds])
    rng = np.random.default_rng(T * 17 + nu + K)
    U = rng.uniform(-0.4, 0.4, (T, nu)).astype(np.float32)
    st = so.make_state(p, nu, rng.uniform(0.02, 0.04, nu) * np.where(np.arange(nu) % 2, 1, -1))
    model = nu_model(nu)
    a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    backend(model, p, smooth=dev(st)).sample_smooth(SEED, PLAN, 0, K, dev(U), a, n)
    a, n = a.cpu().numpy(), n.cpu().numpy()
    z = white(model, p, nu, K)
    a_ref, n_ref = so.sample(p, nu, U, z, st, 0, K)
    gate = smooth_k1_gate(nu, p, U, z, st)
    err = np.abs(a.astype(np.float64) - a_ref)
    st0 = st.copy()
    st0[:nu] = 0.0
    a_bad, _ = so.sample(p, nu, U, z, st0, 0, K)
    miss = float((np.abs(a.astype(np.float64) - a_bad) - gate).max())
    print(f"MODES smooth-k1-{bounds}-T{T}nu{nu}-K{K} worst {err.max():.2e} gate {gate.min():.2e} worst err/gate {(err / gate).max():.3f},"
          f" the reference from a_prev = 0 misses it by {miss:.2e}")
    assert np.all(err <= gate)
    assert miss > 0
    lo, hi, dlo, dhi = so.bounds(p, nu)
    assert np.all(a >= lo[None, :, None]) and np.all(a <= hi[None, :, None])
    v = n.astype(np.float64) + U[:, :, None]
    assert np.all(v >= dlo[None, :, None] - 1e-6) and np.all(v <= dhi[None, :, None] + 1e-6)
    np.testing.assert_allclose(n, n_ref, rtol=0, atol=2 * gate.max() / float(np.float32(p.dt)) + 1e-5)
    np.testing.assert_array_equal(a[:, :, K - 1], np.broadcast_to(st[:nu], (T, nu)))      # the null row holds a_prev
    if K >= 2:
        cut = K // 3 + 1
        for lo_, hi_ in ((0, cut), (cut, K)):
            ps = smooth_params(nu, T, hi_ - lo_, k_offset=lo_, **BOUNDS[bounds])
            a_s = torch.zeros((T, nu, hi_ - lo_), device=DEV)
            backend(model, ps, smooth=dev(st)).sample_smooth(SEED, PLAN, lo_, K, dev(U), a_s, None)
            np.testing.assert_array_equal(a_s.cpu().numpy(), a[:, :, lo_:hi_])


@pytest.mark.parametrize("G", [1, 2, 5, 8])
@pytest.mark.parametrize("T,nu", [(1, 5), (9, 7), (256, 2), (32, 16)])
def test_smooth_k4_against_the_oracle(T, nu, G):
    """K3 on G shards, the smooth K4 on their rows against so.finalize (the gate of test_gpu_smooth); G = 1 fused equals split.  A
    reference integrated from a_prev = 0 misses the gate on A."""
    K = 1024 * G
    p = smooth_params(nu, T, K, du_min=[-0.3], du_max=[0.3], u_min=[-0.03], u_max=[0.03])
    rng = np.random.default_rng(G + T)
    cost = rng.uniform(0.0, 0.05, (T, K)).astype(np.float32)
    x = rng.normal(0.0, 0.4, (T, nu, K)).astype(np.float32)
    U = rng.uniform(-0.3, 0.3, (T, nu)).astype(np.float32)
    st = so.make_state(p, nu, rng.uniform(-0.02, 0.02, nu))
    model = nu_model(nu)
    rows = []
    for g in range(G):
        ps = smooth_params(nu, T, 1024, k_offset=g * 1024, du_min=[-0.3], du_max=[0.3], u_min=[-0.03], u_max=[0.03])
        part = torch.zeros(2 + T * nu, device=DEV)
        sl = slice(g * 1024, (g + 1) * 1024)
        backend(model, ps, smooth=dev(st)).reduce(dev(cost[:, sl]), dev(x[:, :, sl]), dev(U), part)
        rows.append(part.cpu().numpy())
    rows = np.stack(rows)
    stg, Ud = dev(st), dev(U)
    act, stats = torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    backend(model, p, smooth=stg).finalize(dev(rows), G, Ud, act, stats)
    Ug, stg, act = Ud.cpu().numpy(), stg.cpu().numpy(), act.cpu().numpy()
    smooth_k4_check(p, nu, rows, U, st, Ug, stg, act)
    st0 = st.copy()
    st0[:nu] = 0.0
    A_bad = so.unpack(so.finalize(p, nu, rows, U, st0)[3], T, nu)[1].astype(np.float64)
    A = so.unpack(stg, T, nu)[1].astype(np.float64)
    print(f"MODES smooth-k4-T{T}nu{nu}-G{G} |A - A(a_prev = 0)| {np.abs(A - A_bad).max():.2e}")
    assert np.abs(A - A_bad).max() > 1e-4
    if G == 1:
        out = []
        for fused in (False, True):
            sd, Uf = dev(st), dev(U)
            be = backend(model, p, smooth=sd)
            part, a1, s1 = torch.zeros(2 + T * nu, device=DEV), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
            if fused:
                be.reduce_finalize(dev(cost), dev(x), Uf, part, a1, s1)
            else:
                be.reduce(dev(cost), dev(x), Uf, part)
                be.finalize(part.view(1, -1), 1, Uf, a1, s1)
            out.append([t.cpu().numpy() for t in (part, Uf, a1, s1, sd)])
        for a, b in zip(*out):
            np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


# ------------------------------------------------------------------------------------------------------------------------------ CEM
EL_NEW = 896                                                                   # samples per elite-kernel chunk (EL_BUF - EL_KEEP)


def cem_params(nu, T, K, E, keep=0, alpha=0.3, k_offset=0, k_total=None, **kw):
    """A mode-cem parameter block on the generated model; E and keep set directly, so that shards smaller than E are accepted."""
    d = dict(num_samples=max(k_total or K, 2 * 128 + 2), horizon=T, mppi_mode="cem", sampling_method="colored", noise_sigma=(0.04 * np.eye(nu)).tolist(),
             u_min=[-0.5], u_max=[0.5], lambda_=0.5, sample_null_action=True, rollout_var_discount=0.99)
    d.update(kw)
    p = make_params(MPPIConfig(**d), IsaacGymConfig(), nu, K, [])
    p.n_elites, p.n_keep, p.elite_alpha, p.k_offset = E, keep, alpha, k_offset
    return p


def _elite_cases():
    out, i = [], 0
    for nu in (1, 4, 16):
        for T in sorted({1, 9, min(512 // nu, 256)}):
            for kname, K, off in (("under", EL_NEW - 1, 0), ("one", EL_NEW, 0), ("over", EL_NEW + 1, 0), ("ragged", 5003, 0),
                                  ("loop", NUM_SMS * EL_NEW + 1237, 0), ("offset", 3000, 77_777)):
                E = [1, 10, 128][i % 3]
                i += 1
                out.append(pytest.param(T, nu, K, E, off, id=f"elite-T{T}nu{nu}-E{E}-{kname}K{K}"))
    return out


@pytest.mark.parametrize("T,nu,K,E,k_offset", _elite_cases())
def test_cem_elite_kernel_sweep(T, nu, K, E, k_offset):
    """T = 1: the row equals ce.elite_row bit for bit.  T > 1: every elite's S within (T + 4) eps sum_t gamma^t |c| of the float64 S
    of its index, sorted and distinct, the selection exact wherever the float64 gap exceeds that bound, the gathered actions bit-exact;
    a reference without the last step's cost misses the bound."""
    rng = np.random.default_rng(T * 7 + nu + K + E)
    p = cem_params(nu, T, K, E, k_offset=k_offset)
    be = backend(nu_model(nu), p, dev(ce.make_state(np.full(nu, 0.04), T, nu, E)))
    cost = rng.uniform(0, 2, (T, K)).astype(np.float32)
    bad = rng.integers(0, K, max(1, K // 50))
    cost[rng.integers(0, T, bad.size), bad] = rng.choice(np.array([np.nan, np.inf, -np.inf], np.float32), bad.size)
    actions = rng.standard_normal((T, nu, K), dtype=np.float32)
    part = torch.full((ce.row_floats(T, nu, E),), 7.0, device=DEV)
    be.reduce(dev(cost), dev(actions), torch.zeros((T, nu), device=DEV), part)
    got = part.cpu().numpy()
    label = f"elite-T{T}nu{nu}-E{E}-K{K}"
    if T == 1:
        want = ce.elite_row(p, nu, cost, actions, k_offset)
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
        wrong = ce.elite_row(p, nu, cost, actions, k_offset + 1)               # the global indices of another shard
        assert not np.array_equal(got.view(np.uint32), wrong.view(np.uint32))
        print(f"MODES {label} worst 0 gate 0 (bit for bit)")
        return
    with np.errstate(invalid="ignore"):
        S = ce.scores(p, cost)
        bound = (T + 4) * EPS * ((np.float64(np.float32(p.gamma)) ** np.arange(T))[:, None] * np.abs(cost.astype(np.float64))).sum(0)
    fin = np.isfinite(S)
    idx = got[1:2 * E:2].view(np.uint32).astype(np.int64) - k_offset
    Sg = got[0:2 * E:2].astype(np.float64)
    assert np.all((idx >= 0) & (idx < K)) and len(set(idx.tolist())) == E and np.all(np.diff(Sg) >= 0)
    assert fin[idx].all()
    err = np.abs(Sg - S[idx])
    print(f"MODES {label} worst {err.max():.2e} gate {bound[idx].min():.2e} worst err/gate {(err / bound[idx]).max():.3f}")
    assert np.all(err <= bound[idx])
    order = np.flatnonzero(fin)[np.argsort(S[fin], kind="stable")]
    SE, bmax = S[order[E - 1]], bound[fin].max()
    sure_in = fin & (S < SE - 2 * bmax)                                        # its float32 S beats every float32 S from the E-th up
    sure_out = fin & (S > SE + 2 * bmax)                                       # E float32 S beat it
    assert set(np.flatnonzero(sure_in).tolist()) <= set(idx.tolist())
    assert not (set(np.flatnonzero(sure_out).tolist()) & set(idx.tolist()))
    for e, k in enumerate(idx):
        np.testing.assert_array_equal(got[2 * E + e * T * nu:2 * E + (e + 1) * T * nu], actions[:, :, k].ravel())
    with np.errstate(invalid="ignore"):
        S_bad = S - (np.float64(np.float32(p.gamma)) ** (T - 1)) * cost[T - 1].astype(np.float64)
    assert np.any(np.abs(Sg - S_bad[idx]) > bound[idx]), "a reference without the last step passes the bound"


@pytest.mark.parametrize("filt", [False, True])
@pytest.mark.parametrize("G,E", [(1, 10), (2, 128), (5, 1), (32, 128)])
@pytest.mark.parametrize("T,nu", [(9, 7), (256, 2)])
def test_cem_k4_against_float64(T, nu, G, E, filt):
    """K4 on G random shard rows (G E = 4096 candidates at G = 32, E = 128) against ce.finalize with the gates of test_gpu_cem: U
    within (E + 4) eps max|a| (x 4 with filter_u), sigma within 4 max|a| sqrt((E + 4) eps), elites, S and stats exact; a reference
    without the momentum (alpha = 0) misses the U gate."""
    K = 256
    rng = np.random.default_rng(G * E + T)
    p = cem_params(nu, T, K, E, alpha=0.3, k_total=G * K, filter_u=filt)
    st = ce.make_state(np.full(nu, 0.04), T, nu, E)
    rows = []
    for g in range(G):
        pg = copy.deepcopy(p)
        pg.k_offset = g * K
        cost = rng.uniform(0, 1, (T, K)).astype(np.float32)
        rows.append(ce.elite_row(pg, nu, cost, rng.uniform(-0.2, 0.2, (T, nu, K)).astype(np.float32), g * K))
    rows = np.stack(rows)
    U0 = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    Uw, aw, sw, stw = ce.finalize(p, nu, rows, U0, st)
    d_st = dev(st)
    be = backend(nu_model(nu), p, d_st)
    U, act, stats = dev(U0), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(dev(rows), G, U, act, stats)
    got, Ug = d_st.cpu().numpy(), U.cpu().numpy()
    amax = 0.2
    gate_u = (E + 4) * EPS * amax * (4 if filt else 1) + 2 * EPS * amax
    err = float(np.abs(Ug - Uw).max())
    p0 = copy.deepcopy(p)
    p0.elite_alpha = 0.0
    miss = float(np.abs(Ug - ce.finalize(p0, nu, rows, U0, st)[0]).max()) - gate_u
    print(f"MODES cem-k4-T{T}nu{nu}-G{G}E{E}-f{int(filt)} worst {err:.2e} gate {gate_u:.2e}, the reference without momentum misses by {miss:.2e}")
    assert err <= gate_u
    assert miss > 0
    sg, sw_ = ce.unpack(got, T, nu, E)[3], ce.unpack(stw, T, nu, E)[3]
    assert np.abs(sg - sw_).max() <= 4 * amax * np.sqrt((E + 4) * EPS)
    np.testing.assert_array_equal(ce.unpack(got, T, nu, E)[4], ce.unpack(stw, T, nu, E)[4])
    np.testing.assert_array_equal(got[:2 + E], stw[:2 + E])
    np.testing.assert_array_equal(stats.cpu().numpy(), sw)
    np.testing.assert_array_equal(act.cpu().numpy(), Ug[0])


def _cem_k1_cases():
    out = []
    for T, nu in ((30, 7), (9, 16)):
        for off in (0, 1):
            for keep in ("0", "1", "E"):
                out.append(pytest.param(T, nu, off, keep, id=f"cem-k1-T{T}nu{nu}-off{off}-keep{keep}"))
    return out


@pytest.mark.parametrize("T,nu,off,keep", _cem_k1_cases())
def test_cem_k1_carried_elites(T, nu, off, keep):
    """The CEM colored K1 with a live sigma and valid elites at carry offset 0 and 1, n_keep 0, 1 and E (E + E_keep + 2 = K_total):
    the carried rows are clamp(elites[e][t + off]) bit for bit, every row within the colored gate of test_gpu_cem of ce.sample, and
    shards split inside the carried block are bit-identical to one launch; a reference that ignores the carry offset misses."""
    E = 10
    n_keep = {"0": 0, "1": 1, "E": E}[keep]
    K = 2 * E + 2 if keep == "E" else 1000
    p = cem_params(nu, T, K, E, keep=n_keep, k_total=K)
    Lt = colored_noise_chol(T, 2.0)
    rng = np.random.default_rng(T + nu + off + n_keep)
    U0 = rng.uniform(-0.05, 0.05, (T, nu)).astype(np.float32)
    st = ce.make_state(np.full(nu, 0.04), T, nu, E)
    _, _, _, sig, el = ce.unpack(st, T, nu, E)
    sig[:] = rng.uniform(0.01, 0.3, sig.shape).astype(np.float32)
    el[:] = rng.uniform(-0.7, 0.7, el.shape).astype(np.float32)
    st[0], st[1] = float(off), 1.0
    model = nu_model(nu)
    a = torch.zeros((T, nu, K), device=DEV)
    backend(model, p, dev(st)).sample_colored(SEED, PLAN, 0, K, dev(U0), None, dev(Lt), a, None)
    a = a.cpu().numpy()
    z = white(model, p, nu, K)
    a_ref, _ = ce.sample(p, nu, U0, z, Lt, st, 0, K)
    w = np.einsum("ts,sik->tik", np.abs(Lt.astype(np.float64)), np.abs(z.astype(np.float64)))
    gate = EPS * ((np.arange(T) + 3)[:, None, None] * sig.astype(np.float64)[:, :, None] * w + np.abs(U0)[:, :, None] + 2 * np.abs(a_ref))
    err = np.abs(a - a_ref)
    st_bad = st.copy()
    st_bad[0] = 1.0 - off
    a_bad, _ = ce.sample(p, nu, U0, z, Lt, st_bad, 0, K)
    miss = float((np.abs(a - a_bad) - gate).max())
    print(f"MODES cem-k1-T{T}nu{nu}-off{off}-keep{n_keep}-K{K} worst {err.max():.2e} gate {gate.min():.2e}, "
          f"the reference with the other carry offset misses by {miss:.2e}")
    assert np.all(err <= gate)
    assert miss > 0 or n_keep == 0
    lo, hi = ce.bounds(p, nu)
    for e in range(n_keep):
        np.testing.assert_array_equal(a[:T - off, :, K - 3 - e], np.clip(el[e, off:], lo, hi))
    blk = K - 3 - max(n_keep, 1) // 2                                          # a split inside the carried block
    for cuts in ((0, blk, K), (0, K - 3 - n_keep + 1, K - 3, K)):
        for lo_, hi_ in zip(cuts[:-1], cuts[1:]):
            if hi_ <= lo_:
                continue
            ps = cem_params(nu, T, hi_ - lo_, E, keep=n_keep, k_offset=lo_, k_total=K)
            a_s = torch.zeros((T, nu, hi_ - lo_), device=DEV)
            backend(model, ps, dev(st)).sample_colored(SEED, PLAN, lo_, K, dev(U0), None, dev(Lt), a_s, None)
            np.testing.assert_array_equal(a_s.cpu().numpy(), a[:, :, lo_:hi_])


@pytest.mark.parametrize("T,nu", [(1, 7), (256, 2), (32, 16)])
def test_cem_shift(T, nu):
    E = 4
    p = cem_params(nu, T, 64, E, u_init=np.linspace(-0.2, 0.3, nu).tolist())
    st = ce.make_state(np.full(nu, 0.04), T, nu, E)
    st[2 + E:2 + E + T * nu] = 3.0
    d = dev(st)
    U0 = np.arange(T * nu, dtype=np.float32).reshape(T, nu)
    U, ctr = dev(U0), torch.tensor([7], dtype=torch.int32, device=DEV)
    backend(nu_model(nu), p, d).shift(U, ctr)
    Uw, stw = ce.shift(p, nu, U0, st)
    np.testing.assert_array_equal(U.cpu().numpy(), Uw)
    np.testing.assert_array_equal(d.cpu().numpy(), stw)
    assert int(ctr[0]) == 8


# ------------------------------------------------------------------------------------------------------------------------------ colored
def _colored_cases():
    out, i = [], 0
    for nu in (1, 5, 16):
        for T in sorted({1, 9, min(512 // nu, 256)}):
            for kind in ("M2", "C", "CEM"):
                K = [4, 63, 65, 1000][i % 4]
                beta = [1.0, 2.0, 2.5][i % 3]
                i += 1
                out.append(pytest.param(T, nu, K, kind, beta, id=f"colored-{kind}-T{T}nu{nu}-K{K}-b{beta:g}"))
    return out


@pytest.mark.parametrize("T,nu,K,kind,beta", _colored_cases())
def test_colored_instantiations(T, nu, K, kind, beta):
    """The <DIAG>, <FULL> and <CEM> colored K1 against colored_oracle.colour / cem_oracle.sample on the device's own white draws, within
    the per-element gates of test_gpu_colored and test_gpu_cem; a reference without one temporal term misses them."""
    if kind != "CEM":
        _check_case(make_case(T, nu, K, kind=kind), beta, tag=f"MODES {kind}")
        return
    E = 4
    p = cem_params(nu, T, K, E, keep=2, k_total=K)
    Lt = colored_noise_chol(T, beta)
    rng = np.random.default_rng(T + nu + K)
    U0 = rng.uniform(-0.05, 0.05, (T, nu)).astype(np.float32)
    st = ce.make_state(np.full(nu, 0.04), T, nu, E)
    st[2 + E:2 + E + T * nu] = rng.uniform(0.05, 0.3, T * nu).astype(np.float32)
    a = torch.zeros((T, nu, K), device=DEV)
    model = nu_model(nu)
    backend(model, p, dev(st)).sample_colored(SEED, PLAN, 0, K, dev(U0), None, dev(Lt), a, None)
    a = a.cpu().numpy()
    z = white(model, p, nu, K)
    sig = ce.unpack(st, T, nu, E)[3]
    a_ref, _ = ce.sample(p, nu, U0, z, Lt, st, 0, K)
    w = np.einsum("ts,sik->tik", np.abs(Lt.astype(np.float64)), np.abs(z.astype(np.float64)))
    gate = EPS * ((np.arange(T) + 3)[:, None, None] * sig.astype(np.float64)[:, :, None] * w + np.abs(U0)[:, :, None] + 2 * np.abs(a_ref))
    body = slice(0, K - 1)
    err = np.abs(a - a_ref)[:, :, body]
    a_bad, _ = ce.sample(p, nu, U0, z, drop_one_term(Lt, beta), st, 0, K)
    miss = float((np.abs(a - a_bad) - gate)[:, :, body].max())
    print(f"MODES colored-CEM-T{T}nu{nu}-K{K}-b{beta:g} worst {err.max():.2e} gate {gate.min():.2e}, without one temporal term by {miss:.2e}")
    assert np.all(err <= gate[:, :, body])
    assert miss > 0
    np.testing.assert_array_equal(a[:, :, K - 1], np.clip(0.0, -0.5, 0.5) * np.ones((T, nu), np.float32))


# ------------------------------------------------------------------------------------------------------------------------------ corners
CORNERS = [(256, 2), (32, 16), (1, 16)]
CORNER_MODES = ["simple", "halton-spline", "cem", "smooth", "risk-fixed", "risk-diag", "risk-full"]


def _corner_params(mode, T, nu, K):
    sig = (0.04 * np.eye(nu)).tolist()
    base = dict(num_samples=K, horizon=T, sampling_method="random", noise_sigma=sig, lambda_=0.5, sample_null_action=True, u_min=[-1.0], u_max=[1.0])
    if mode in ("simple", "halton-spline"):
        base.update(mppi_mode=mode)
    elif mode == "cem":
        base.update(mppi_mode="cem", sampling_method="colored", n_elites=10)
    elif mode == "smooth":
        base.update(mppi_mode="smooth", smooth_weight=0.5, du_min=[-1.0], du_max=[1.0])
    else:
        kind = mode.split("-")[1]
        base.update(mppi_mode="simple", n_worlds=8, cvar_alpha=0.25, update_cov=kind != "fixed", update_lambda=kind != "fixed",
                    cov_type="full" if kind == "full" else "diag")
    return make_params(MPPIConfig(**base), IsaacGymConfig(), nu, K, [])


def _corner_state(mode, p, T, nu):
    if mode == "cem":
        return dev(ce.make_state(np.full(nu, 0.04), T, nu, p.n_elites)), None
    if mode == "smooth":
        return None, dev(so.make_state(p, nu))
    if mode in ("risk-diag", "risk-full"):
        import adaptive_full_oracle as afo
        sig = 0.04 * np.eye(nu)
        return dev(np.concatenate([[0.5], np.diag(sig)]) if mode == "risk-diag" else afo.make_dist(0.5, sig)), None
    return None, None


def _corner_plan(mode, model, p, T, nu, K, dist, smooth):
    be = backend(model, p, dist, smooth)
    U = dev(np.zeros((T, nu)))
    a, n = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    if mode == "cem":
        be.sample_colored(SEED, PLAN, 0, K, U, None, dev(colored_noise_chol(T, 2.0)), a, n)
    elif mode == "smooth":
        be.sample_smooth(SEED, PLAN, 0, K, U, a, n)
    else:
        be.sample(SEED, PLAN, 0, K, U, None, a, n)
    cost = (a * a).sum(1).contiguous()
    x = a if mode == "cem" else n
    P = be.partial_row_floats()
    part, act, st = torch.zeros(P, device=DEV), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.reduce_finalize(cost, x, U, part, act, st)
    torch.cuda.synchronize()
    return U.cpu().numpy(), act.cpu().numpy(), st.cpu().numpy()


@pytest.mark.parametrize("mode", CORNER_MODES)
def test_accepted_corners_run(mode):
    """Every corner make_params accepts -- (T, nu) = (256, 2), (32, 16), (1, 16) -- runs K1 -> K3 -> K4 on the device without a refusal
    and with a finite plan; T*nu = 513 is refused by the device (the cem and smooth handles at creation, K3 otherwise), and by
    make_params wherever the host refuses it."""
    for T, nu in CORNERS:
        K = 1024
        p = _corner_params(mode, T, nu, K)
        dist, smooth = _corner_state(mode, p, T, nu)
        U, act, st = _corner_plan(mode, nu_model(nu), p, T, nu, K, dist, smooth)
        print(f"MODES corner-{mode}-T{T}nu{nu} action {act[:2]} stats {st}")
        assert np.isfinite(U).all() and np.isfinite(act).all() and np.isfinite(st).all()
        if mode != "smooth":                                                   # smooth plans a derivative U; its action is A_0
            np.testing.assert_array_equal(act, U[0])
    nu = 9
    if mode in ("cem", "smooth"):
        with pytest.raises(ValueError, match="horizon \\* nu <= 512"):
            _corner_params(mode, 57, nu, 1024)
    p = _corner_params(mode, 56, nu, 1024)
    p.T = 57                                                                   # T*nu = 513 past the host
    dist, smooth = _corner_state(mode, p, 57, nu)
    if mode in ("cem", "smooth"):                                              # these handles refuse the shape when they are created
        with pytest.raises(RuntimeError, match="513"):
            backend(nu_model(nu), p, dist, smooth)
        return
    be = backend(nu_model(nu), p, dist, smooth)
    cost, x, U = torch.zeros((57, 1024), device=DEV), torch.zeros((57, nu, 1024), device=DEV), torch.zeros((57, nu), device=DEV)
    with pytest.raises(RuntimeError, match="513"):
        be.reduce(cost, x, U, torch.zeros(be.partial_row_floats(), device=DEV))
    torch.cuda.synchronize()
