"""The shard-row length of every update rule: ``backend.shard_row_floats`` (the Python twin of shard_row_floats / partial_row_capacity in
csrc/common.cuh) pinned to literal values, and the ``partial`` buffer a planner on the oracle backends allocates for each rule."""
import pytest

from mppi_isaac_b200.backend import shard_row_floats
from mppi_isaac_b200.model.blob import MODE_CEM, MODE_SIMPLE, MODE_SMOOTH, MppibParams

# rule -> the parameter fields that select it
RULES = {
    "plain": {},
    "lambda": dict(update_lambda=1),
    "diag": dict(update_cov=1),
    "full": dict(update_cov=1, cov_full=1),
    "horizon": dict(update_cov=1, cov_horizon=1),
    "smooth": dict(mode=MODE_SMOOTH),
    "modes": dict(n_modes=4),
    "cem": dict(mode=MODE_CEM, n_elites=10),
    "risk": dict(n_worlds=4),
    "risk-diag": dict(n_worlds=4, update_cov=1),
    "risk-full": dict(n_worlds=4, update_cov=1, cov_full=1),
}
# floats of the row at (T, nu) = (30, 7), n = 210, and (12, 2), n = 24
EXPECTED = {
    (30, 7): dict(plain=212, **{"lambda": 212}, diag=422, full=240, horizon=22367, smooth=212, modes=848, cem=2120, risk=212,
                  **{"risk-diag": 422, "risk-full": 240}),
    (12, 2): dict(plain=26, **{"lambda": 26}, diag=50, full=29, horizon=326, smooth=26, modes=104, cem=260, risk=26,
                  **{"risk-diag": 50, "risk-full": 29}),
}


def _params(T, **fields):
    p = MppibParams()
    p.T, p.mode, p.n_modes, p.n_worlds = T, MODE_SIMPLE, 1, 1
    for k, v in fields.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("shape", sorted(EXPECTED))
@pytest.mark.parametrize("rule", sorted(RULES))
def test_shard_row_floats(rule, shape):
    T, nu = shape
    assert shard_row_floats(_params(T, **RULES[rule]), nu) == EXPECTED[shape][rule]


def _planner(rule):
    """A planner of `rule` on the oracle backend that implements it, and its (T, nu)."""
    import adaptive_full_oracle as afo
    import adaptive_horizon_oracle as aho
    import adaptive_oracle as ada
    import cem_oracle as ce
    import modes_oracle as mo
    import risk_oracle as ro
    import smooth_oracle as so
    from oracle.backend import OracleBackend
    from scenes import boxer_cfg, panda_cfg

    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective, PushObjective
    if rule.startswith("risk"):
        kw = dict(n_worlds=4, cvar_alpha=0.5, sampling_method="random", mppi_mode="simple")
        kw.update({"risk": {}, "risk-diag": dict(update_cov=True), "risk-full": dict(update_cov=True, cov_type="full")}[rule])
        return MPPIisaacPlanner(boxer_cfg(K=64, T=12, **kw), PushObjective(robot="boxer", link="ee_link"), backend=ro.RiskOracleBackend()), (12, 2)
    kw, backend = {
        "plain": ({}, OracleBackend),
        "lambda": (dict(update_lambda=True), ada.AdaptiveOracleBackend),
        "diag": (dict(update_cov=True), ada.AdaptiveOracleBackend),
        "full": (dict(update_cov=True, cov_type="full"), afo.AdaptiveFullOracleBackend),
        "horizon": (dict(update_cov=True, cov_type="horizon"), aho.AdaptiveHorizonOracleBackend),
        "smooth": (dict(mppi_mode="smooth", sampling_method="random", filter_u=False, smooth_weight=0.5, du_min=[-1.0], du_max=[1.0]),
                   so.SmoothOracleBackend),
        "modes": (dict(n_modes=4), mo.ModesOracleBackend),
        "cem": (dict(mppi_mode="cem", sampling_method="colored", n_elites=10), ce.CemOracleBackend),
    }[rule]
    return MPPIisaacPlanner(panda_cfg(K=128, T=30, device="cpu", **kw), PandaReachObjective(), backend=backend(), use_cuda_graph=False), (30, 7)


@pytest.mark.parametrize("rule", sorted(RULES))
def test_planner_allocates_the_shard_row(rule):
    pl, shape = _planner(rule)
    m = pl.mppi
    assert m.partial.numel() == shard_row_floats(m.backend.params, shape[1]) == EXPECTED[shape][rule]
    assert tuple(m.partials.shape) == (m.world, EXPECTED[shape][rule])
