"""The ESS-targeted temperature (`lambda_mode: ess`) on the CPU: the rule's edge cases, the float64 restatement against K3's S, the
target quality on synthetic and recorded cost sets, scale invariance, composition with update_cov (diag and full), a stepwise plan with
a prior, and which features the mode admits -- make_params and the library refuse the same blocks with the same messages."""
import copy
import ctypes as C
import itertools
import os

import numpy as np
import pytest
import torch

import adaptive_full_oracle as adf
import adaptive_oracle as ada
import temperature_oracle as tmo
from mppi_isaac_b200 import MPPIisaacPlanner, backend
from mppi_isaac_b200.model.blob import ESS_GRID, MODE_MEAN, MODE_SIMPLE, ess_grid, make_params, mode_refusal
from mppi_isaac_b200.objectives import PandaReachObjective, PointReachObjective, PushObjective
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from oracle import oracle as orc
from scenes import boxer_cfg, panda_cfg, point_cfg, point_setup
from synth_mppi import nu_model

Q0, QD0 = [0.1, 0.0, 0.0], [0.0] * 3
ESS = dict(lambda_mode="ess")


def grid(lam0=1.0):
    lam, inv = ess_grid(lam0)
    return lam.astype(np.float64), inv


def choose(C, q, lam0, rho):
    """(lambda, N, ESS curve) of one shard by the restated pass and rule."""
    lam, inv = grid(lam0)
    row = _row(C, q, inv)
    N, ess = tmo.combine([row])
    return tmo.rule(ess, N, rho, lam, lam0), N, ess


def _row(C, q, inv):
    C, q = np.asarray(C, np.float64), np.asarray(q, np.float64)
    ok = np.isfinite(C) & np.isfinite(q)
    if not ok.any():
        return 0, np.full(ESS_GRID, np.inf), np.zeros(ESS_GRID), np.zeros(ESS_GRID)
    a = C[ok][None, :] * np.asarray(inv, np.float64)[:, None] + q[ok][None, :]
    m = a.min(1)
    e = np.exp(-(a - m[:, None]))
    return int(ok.sum()), m, e.sum(1), (e * e).sum(1)


# ---- the rule --------------------------------------------------------------------------------------------------------------------------

def test_no_bracket_takes_the_largest_grid_temperature():
    lam, _ = grid(1e-3)
    got, N, ess = choose([0.0, 1000.0], [0.0, 0.0], 1e-3, 1.0)
    assert N == 2 and ess.max() < 2.0 and got == lam[-1]


def test_all_equal_costs_take_the_smallest_grid_temperature():
    lam, _ = grid(0.5)
    got, N, ess = choose(np.full(100, 3.0), np.zeros(100), 0.5, 0.3)
    np.testing.assert_allclose(ess, 100.0, rtol=1e-12)
    assert got == lam[0]


def test_an_exact_hit_interpolates_to_the_grid_point():
    lam, _ = grid(1.0)
    ess = np.linspace(1.0, 100.0, ESS_GRID)
    N = 200
    rho = ess[10] / N
    assert tmo.rule(ess, N, rho, lam, 1.0) == pytest.approx(lam[10], rel=1e-7)     # the grid is rounded to float32
    # between two grid points the rule is linear in ln ESS over log2 lambda
    tau = np.sqrt(ess[10] * ess[11])
    assert tmo.rule(ess, N, tau / N, lam, 1.0) == pytest.approx(lam[10] * 2 ** (0.5 / 4), rel=1e-6)


def test_no_valid_sample_keeps_the_previous_temperature():
    got, N, ess = choose([np.nan, np.inf, -np.inf], [0.0, 0.0, 0.0], 1.0, 0.1)
    assert N == 0 and np.all(ess == 0.0)
    assert tmo.rule(ess, 0, 0.1, grid()[0], 0.123) == 0.123


def test_non_finite_samples_are_left_out():
    rng = np.random.default_rng(0)
    C, q = rng.exponential(size=64), rng.normal(size=64)
    _, inv = grid()
    clean = _row(C, q, inv)
    Cb, qb = np.concatenate([C, [np.nan, np.inf, -np.inf, 1.0]]), np.concatenate([q, [0.0, 0.0, 0.0, np.nan]])
    dirty = _row(Cb, qb, inv)
    assert dirty[0] == clean[0] == 64
    for a, b in zip(dirty[1:], clean[1:]):
        np.testing.assert_array_equal(a, b)


def test_ess_is_monotone_in_lambda():
    """Without the control cost (MEAN mode, q = 0) the weights flatten as lambda grows.  With it, S / lambda tends to q, so in SIMPLE mode
    the curve levels off at the ESS of exp(-q) and need not be monotone: the rule takes the first bracket."""
    rng = np.random.default_rng(1)
    for _ in range(5):
        C, q = rng.gamma(2.0, size=500) * 10, np.zeros(500)
        _, ess = tmo.combine([_row(C, q, grid(0.3)[1])])
        assert np.all(np.diff(ess) >= -1e-9 * ess[1:])


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_S_of_the_restatement_is_the_S_of_K3(mode):
    """min_k (C_k + lambda q_k) is K3's beta at that temperature, in SIMPLE (with the control cost) and MEAN mode."""
    sc, p, _ = point_setup(K=128, T=12, mode="simple" if mode == "simple" else "halton-spline", u_min=[-1e6], u_max=[1e6])
    nu = sc.model.nu
    rng = np.random.default_rng(2)
    cost = rng.exponential(size=(12, 128)).astype(np.float32)
    x = rng.normal(scale=0.3, size=(12, nu, 128)).astype(np.float32)
    U = rng.normal(scale=0.5, size=(12, nu)).astype(np.float32)
    C, q = tmo.scores(p, nu, cost, x, U)
    if p.mode == MODE_MEAN:
        assert np.all(q == 0)
    for lam in (0.05, 0.7):
        pl = copy.deepcopy(p)
        pl.lambda_ = lam
        row, _ = orc.reduce(sc.model, pl, cost, x, U)
        assert row[0] == pytest.approx((C + np.float32(lam) * q).min(), rel=1e-5, abs=1e-5)


# ---- target quality --------------------------------------------------------------------------------------------------------------------

def _quality(C, q, lam0, rho):
    lam, N, ess = choose(C, q, lam0, rho)
    grid_lam = grid(lam0)[0]
    bracketed = tmo.ess_at(C, q, grid_lam[0]) < rho * N <= tmo.ess_at(C, q, grid_lam[-1])
    return abs(tmo.ess_at(C, q, lam) / (rho * N) - 1.0), bracketed


def _recorded(kind):
    """(C, q) of one oracle plan's samples: panda reach (the C2 Objective) or boxer push (the C3 Objective), at a CPU-sized K."""
    if kind == "panda":
        p = MPPIisaacPlanner(panda_cfg(K=256, T=12, sampling_method="random"), PandaReachObjective(), backend=ada.AdaptiveOracleBackend())
        p.compute_action([0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0], [0.0] * 7)
    else:
        p = MPPIisaacPlanner(boxer_cfg(K=256, T=12, sampling_method="random"), PushObjective(robot="boxer", link="ee_link"),
                             backend=ada.AdaptiveOracleBackend())
        p.compute_action([0.0, 2.5, 0.0], [0.0] * 3)
    m = p.mppi
    return tmo.scores(m.backend.params, m.nu, m.cost.numpy(), m.noise.numpy(), m.U.numpy())


def test_target_quality():
    rng = np.random.default_rng(3)
    sets = {"gaussian": (rng.normal(10.0, 2.0, 4000), rng.normal(0, 0.1, 4000)),
            "exponential": (rng.exponential(5.0, 4000), np.zeros(4000)),
            "heavy-tailed": (np.abs(rng.standard_cauchy(4000)), np.zeros(4000)),
            "panda reach (recorded)": _recorded("panda"),
            "boxer push (recorded)": _recorded("boxer")}
    worst = 0.0
    for name, (C, q) in sets.items():
        for lam0 in (0.01, 0.1, 1.0):
            for rho in (0.01, 0.05, 0.2):
                err, bracketed = _quality(np.asarray(C, np.float64), np.asarray(q, np.float64), lam0, rho)
                if bracketed:
                    assert err < 0.05, (name, lam0, rho, err)
                    worst = max(worst, err)
    print(f"worst relative ESS error at the chosen lambda: {worst:.4f}")


# ---- the parameter block ---------------------------------------------------------------------------------------------------------------

def _cfg(**kw):
    d = dict(num_samples=256, horizon=12, mppi_mode="simple", sampling_method="random", noise_sigma=(0.1 * np.eye(3)).tolist(),
             u_min=[-1.0], u_max=[1.0], lambda_=0.1)
    d.update(kw)
    return MPPIConfig(**d)


def test_fixed_mode_keeps_the_block_byte_identical():
    base = make_params(_cfg(), IsaacGymConfig(), 3, 256, [])
    fixed = make_params(_cfg(lambda_mode="fixed", ess_target=0.5), IsaacGymConfig(), 3, 256, [])
    assert bytes(base) == bytes(fixed)
    ess = make_params(_cfg(lambda_mode="ess", ess_target=0.25), IsaacGymConfig(), 3, 256, [])
    assert ess.lambda_ess == 1 and ess.ess_target == 0.25


@pytest.mark.parametrize("rho", [0.0, -0.1, 1.5, float("nan"), float("inf")])
def test_ess_target_out_of_range_is_refused(rho):
    with pytest.raises(ValueError, match="ess_target"):
        make_params(_cfg(lambda_mode="ess", ess_target=rho), IsaacGymConfig(), 3, 256, [])


def test_unknown_lambda_mode_is_refused():
    with pytest.raises(ValueError, match="lambda_mode"):
        make_params(_cfg(lambda_mode="kl"), IsaacGymConfig(), 3, 256, [])


# ---- plans -----------------------------------------------------------------------------------------------------------------------------

class Scaled(PointReachObjective):
    def __init__(self, c):
        super().__init__()
        self.c = c

    def compute_cost(self, sim):
        return super().compute_cost(sim) * self.c


def test_scale_invariance():
    """Costs times c with lambda_ times c choose lambda times c and the same U (c a power of two: every rounding scales exactly)."""
    kw = dict(K=128, T=12, mppi_mode="simple", sampling_method="random", filter_u=False, **ESS, ess_target=0.05)
    a = MPPIisaacPlanner(point_cfg(lambda_=0.1, **kw), Scaled(1.0), backend=tmo.TemperatureOracleBackend())
    b = MPPIisaacPlanner(point_cfg(lambda_=0.8, **kw), Scaled(8.0), backend=tmo.TemperatureOracleBackend())
    for _ in range(4):
        np.testing.assert_allclose(b.compute_action(Q0, QD0).numpy(), a.compute_action(Q0, QD0).numpy(), rtol=0, atol=1e-5)
        np.testing.assert_allclose(b.mppi.U.numpy(), a.mppi.U.numpy(), rtol=0, atol=1e-5)
        assert float(b.mppi.current_lambda) == pytest.approx(8.0 * float(a.mppi.current_lambda), rel=1e-5)


class RecordingMixin:
    """Records what each plan's temperature pass saw and the temperature it chose."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.chosen, self.seen = [], []

    def temperature(self, cost, x, U, row, solve=True):
        self.seen.append((cost.clone(), None if x is None else x.clone(), U.clone()))
        super().temperature(cost, x, U, row, solve)
        self.chosen.append(float(self.dist[0]))


class Recording(RecordingMixin, tmo.TemperatureOracleBackend):
    pass


class RecordingFull(RecordingMixin, tmo.TemperatureFullOracleBackend):
    pass


class SubstitutedMixin:
    """An adaptive checker backend with dist[0] set to a given temperature before each plan's K3."""

    def __init__(self, lams, *a, **kw):
        super().__init__(*a, **kw)
        self.lams = list(lams)

    def reduce(self, cost, x, U, partial):
        self.dist[0] = self.lams.pop(0)
        return super().reduce(cost, x, U, partial)


class Substituted(SubstitutedMixin, ada.AdaptiveOracleBackend):
    pass


class SubstitutedFull(SubstitutedMixin, adf.AdaptiveFullOracleBackend):
    pass


@pytest.mark.parametrize("cov_type", ["diag", "full"])
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_composition_with_update_cov(cov_type, mode):
    """An ESS plan with update_cov is the adaptive plan with the chosen temperature substituted, plan after plan."""
    kw = dict(K=128, T=12, mppi_mode=mode, sampling_method="random", filter_u=False, update_cov=True, cov_type=cov_type)
    rec = Recording() if cov_type == "diag" else RecordingFull()
    e = MPPIisaacPlanner(point_cfg(**kw, **ESS, ess_target=0.1), PointReachObjective(), backend=rec)
    for _ in range(4):
        e.compute_action(Q0, QD0)
    sub = (Substituted if cov_type == "diag" else SubstitutedFull)(rec.chosen)
    a = MPPIisaacPlanner(point_cfg(**kw), PointReachObjective(), backend=sub)
    for _ in range(4):
        a.compute_action(Q0, QD0)
    np.testing.assert_allclose(e.mppi.U.numpy(), a.mppi.U.numpy(), rtol=0, atol=1e-6)
    np.testing.assert_allclose(e.mppi.dist[1:].numpy(), a.mppi.dist[1:].numpy(), rtol=1e-6, atol=1e-9)
    assert len(set(rec.chosen)) > 1                               # the temperature follows the plans


def test_chosen_lambda_is_the_rule_of_the_plan_and_the_views():
    rec = Recording()
    p = MPPIisaacPlanner(point_cfg(K=128, T=12, mppi_mode="simple", sampling_method="halton", **ESS, ess_target=0.1), PointReachObjective(),
                         backend=rec)
    for _ in range(3):
        p.compute_action(Q0, QD0)
        cost, x, U = rec.seen[-1]
        pp = p.mppi.backend.params
        C, q = tmo.scores(pp, p.mppi.nu, cost.numpy(), x.numpy(), U.numpy())
        lam, N, ess = choose(C, q, pp.lambda_, float(np.float32(0.1)))
        assert float(p.mppi.current_lambda) == pytest.approx(lam, rel=1e-6)
        assert p.mppi.valid_samples == N == 128
        np.testing.assert_allclose(p.mppi.ess_curve.numpy(), ess, rtol=1e-6)
        np.testing.assert_array_equal(p.mppi.ess_grid.numpy(), ess_grid(pp.lambda_)[0])


def test_stepwise_plan_with_a_prior():
    """The temperature sees the prior row's noise as K3 does: after the rewrite of the stepwise plan."""
    class Prior:
        def compute_command(self, sim):
            return torch.tensor([0.2, -0.1, 0.0])
    rec = Recording()
    p = MPPIisaacPlanner(point_cfg(K=64, T=10, mppi_mode="simple", sampling_method="random", use_priors=True, filter_u=False, **ESS),
                         PointReachObjective(), Prior(), backend=rec)
    assert p.mppi.rollout_mode == "stepwise"
    for _ in range(3):
        p.compute_action(Q0, QD0)
        cost, x, U = rec.seen[-1]
        row = 64 - 2
        np.testing.assert_allclose(x[:, :, row].numpy(), (p.mppi.actions[:, :, row] - U).numpy(), atol=1e-6)
        np.testing.assert_allclose(p.mppi.actions[0, :, row].numpy(), [0.2, -0.1, 0.0], atol=1e-6)
    assert p.mppi.valid_samples == 64


def test_planner_refuses_a_backend_without_the_temperature_entries():
    with pytest.raises(ValueError, match="set_temperature"):
        MPPIisaacPlanner(point_cfg(K=64, T=10, mppi_mode="simple", sampling_method="random", **ESS), PointReachObjective(),
                         backend=ada.AdaptiveOracleBackend())


def test_reduce_refuses_ess_without_a_state():
    be = tmo.TemperatureOracleBackend()
    p = MPPIisaacPlanner(point_cfg(K=64, T=10, mppi_mode="simple", sampling_method="random", **ESS), PointReachObjective(), backend=be)
    be.set_temperature(None)
    with pytest.raises(RuntimeError, match="temperature state"):
        p.compute_action(Q0, QD0)


# ---- admission: the harness of test_mode_admission.py restated for lambda_mode: ess -----------------------------------------------------

FEATURES = {
    "cem": dict(mppi_mode="cem"),
    "smooth": dict(mppi_mode="smooth"),
    "halton": dict(sampling_method="halton"),
    "colored": dict(sampling_method="colored"),
    "update_cov": dict(update_cov=True),
    "update_lambda": dict(update_lambda=True),
    "cov_full": dict(update_cov=True, cov_type="full"),
    "cov_horizon": dict(update_cov=True, cov_type="horizon"),
    "filter_u": dict(filter_u=True),
    "n_worlds": dict(n_worlds=2, cvar_alpha=0.5),
    "n_modes": dict(n_modes=2),
    "anneal": dict(anneal_iterations=2, anneal_iter_decay=0.8),
    "knots": dict(control_knots=4),
    "constraint": dict(constraint_mode="feasible_first"),
}
WHY = {
    "cem": "lambda_mode: ess excludes mode cem (it does not weight the samples with the temperature)",
    "smooth": "lambda_mode: ess excludes mode smooth (it does not weight the samples with the temperature)",
    "update_lambda": "lambda_mode: ess excludes update_lambda (two rules for one temperature)",
    "cov_horizon": "lambda_mode: ess excludes cov_horizon (the shift computes lambda Sigma_H^-1 U before the temperature is known)",
    "n_worlds": "lambda_mode: ess excludes n_worlds > 1",
    "n_modes": "lambda_mode: ess excludes n_modes > 1",
    "anneal": "lambda_mode: ess excludes annealed MPPI",
    "knots": "lambda_mode: ess excludes control_knots > 0",
    "constraint": "lambda_mode: ess excludes constraint_mode",
}


def _refusal(kw, T=12, nu=3, K=256):
    d = dict(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.1 * np.eye(nu)).tolist(),
             u_min=[-1.0], u_max=[1.0], lambda_=0.1, rollout_var_discount=0.95, **ESS)
    d.update(kw)
    try:
        make_params(MPPIConfig(**d), IsaacGymConfig(), nu, K, [])
        return None
    except ValueError as e:
        return str(e)


def _keys(names):
    kw = {}
    for n in names:
        kw.update(FEATURES[n])
    return kw


def _compatible_pairs():
    out = []
    for a, b in itertools.combinations(FEATURES, 2):
        if all(FEATURES[b].get(k, v) == v for k, v in FEATURES[a].items()):
            out.append((a, b))
    return out


@pytest.mark.parametrize("name", [None, *FEATURES])
def test_ess_against_each_feature(name):
    why = _refusal(_keys([] if name is None else [name]))
    assert why == WHY.get(name), why


ORDER = ["update_lambda", "cov_horizon", "cem", "smooth", "n_worlds", "n_modes", "knots", "constraint", "anneal"]   # the table's order


@pytest.mark.parametrize("pair", _compatible_pairs(), ids="+".join)
def test_ess_against_each_pair(pair):
    """A pair that refuses itself keeps its own message; otherwise the first feature of the pair that lambda_mode: ess excludes."""
    plain = _refusal({**_keys(pair), "lambda_mode": "fixed"})
    want = plain if plain is not None else next((WHY[n] for n in ORDER if n in pair), None)
    assert _refusal(_keys(pair)) == want


K_BLOCK = 256
BLOCK = {
    "cem": dict(mode=2, n_elites=4, n_keep=1, elite_alpha=0.1),
    "smooth": dict(mode=3),
    "update_cov": dict(update_cov=1),
    "update_lambda": dict(update_lambda=1),
    "cov_full": dict(update_cov=1, cov_full=1),
    "cov_horizon": dict(update_cov=1, cov_horizon=1),
    "filter_u": dict(filter_u=1),
    "n_worlds": dict(n_worlds=2, risk_tail=1),
    "n_modes": dict(n_modes=2, mode_samples=K_BLOCK // 2),
    "control_knots": dict(control_knots=4, spline_degree=1),
    "constraint_mode": dict(constraint_mode=1, constraint_tol=0.0, constraint_lambda=1.0),
}
SAME_KEY = ({"cem", "smooth"}, {"cov_full", "cov_horizon"})


def _block(names, **fields):
    p = make_params(MPPIConfig(num_samples=K_BLOCK, horizon=12, mppi_mode="simple", sampling_method="random",
                               noise_sigma=(0.1 * np.eye(3)).tolist(), u_min=[-1.0], u_max=[1.0], lambda_=0.1), IsaacGymConfig(), 3, K_BLOCK, [])
    fields = {"lambda_ess": 1, "ess_target": 0.01, **fields}
    for n in names:
        fields = {**BLOCK[n], **fields}
    for k, v in fields.items():
        setattr(p, k, v)
    for j in range(3):
        p.du_min[j], p.du_max[j] = -1e30, 1e30
    return p


def _library():
    if not os.path.exists(backend.lib_path()):
        import __graft_entry__
        __graft_entry__.build()
    return backend.load_library()


def _create(lib, p):
    h = C.c_void_p()
    rc = lib.mppib_create(C.byref(nu_model(3)), C.byref(p), C.c_int32(0), C.byref(h))
    if rc == 0:
        lib.mppib_destroy(h)
    return rc


def _block_cases():
    names = list(BLOCK)
    cases = [((), {})] + [((n,), {}) for n in names]
    cases += [((a, b), {}) for a, b in itertools.combinations(names, 2) if {a, b} not in SAME_KEY]
    cases += [((), dict(ess_target=v)) for v in (0.0, 1.0, 1.5, float("nan"))]
    return cases


@pytest.mark.parametrize("names, fields", _block_cases(), ids=lambda x: "+".join(x) if isinstance(x, tuple) else
                         "-".join(f"{k}{v}" for k, v in x.items()) or "base")
def test_the_table_and_the_library_refuse_the_same_blocks_with_the_same_messages(names, fields):
    lib = _library()
    p = _block(names, **fields)
    why = mode_refusal(p, 3)
    rc = _create(lib, p)
    err = lib.mppib_last_error().decode()
    assert rc in (-1, 0, -2), err
    if "ess_target" in fields and not 0.0 < fields["ess_target"] <= 1.0:
        assert rc == -1 and "ess_target" in err
        return
    assert (rc == -1) == (why is not None), (why, err)
    if why is not None and why.startswith("lambda_mode: ess"):
        assert err == why
