"""The sweep of planning configurations that ``test_gpu_plan_paths.py`` runs through every way the planner runs a plan, and its scenes.

The configurations are derived from ``blob.FEATURES`` and ``blob.EXCLUSIONS``, not picked by hand: the plain planner, every feature on
its own and every maximal admitted combination, each in SIMPLE and MEAN mode where both are admitted and with cov_type diag and full
wherever update_cov is on.  A feature added to FEATURES without an entry in FEATURE_KEYS, or a pair newly admitted by EXCLUSIONS,
changes the sweep (``test_plan_paths_sweep.py`` checks both without a GPU)."""
from typing import NamedTuple, Optional, Tuple

import torch

from mppi_isaac_b200.model.blob import (ANNEALED, CEM, COLORED, CONSTRAINED, ESS, EXCLUSIONS, FEATURES, HALTON, KNOTS, MODES, SMOOTH,
                                        WORLDS)
from mppi_isaac_b200.objectives import PandaReachObjective, PointReachObjective, PushObjective
from scenes import boxer_cfg, panda_cfg, point_cfg

HORIZON = "cov_type: horizon"

# the config keys that switch each feature on, with parameters chosen so that the feature changes the plan within a few plans
FEATURE_KEYS = {
    CEM: dict(mppi_mode="cem", n_elites=8, cem_iterations=2),
    SMOOTH: dict(mppi_mode="smooth", smooth_weight=0.05, du_min=[-8.0], du_max=[8.0]),
    HALTON: dict(sampling_method="halton"),
    COLORED: dict(sampling_method="colored", noise_beta=2.0),
    "update_cov": dict(update_cov=True),
    # eta > 1 whenever two samples carry weight, so with the bounds at (0.5, 1) the temperature moves on almost every plan
    "update_lambda": dict(update_lambda=True, eta_u_bound=1.0, eta_l_bound=0.5),
    HORIZON: dict(update_cov=True, cov_type="horizon"),
    "filter_u": dict(filter_u=True),
    WORLDS: dict(n_worlds=4, cvar_alpha=0.5),
    MODES: dict(n_modes=2, mode_switch_margin=0.0),
    ANNEALED: dict(anneal_iterations=2, anneal_iter_decay=0.5, anneal_horizon_decay=0.9),
    KNOTS: dict(control_knots=5, spline_degree=2),
    CONSTRAINED: dict(constraint_mode="feasible_first"),
    ESS: dict(lambda_mode="ess", ess_target=0.1),
}

# what a configuration without any feature sets: the plain planner (SIMPLE mode, white Gaussian noise, no filter, fixed Sigma and lambda)
PLAIN = dict(mppi_mode="simple", sampling_method="random", filter_u=False, update_cov=False, update_lambda=False, cov_type="diag",
             use_priors=False)
MEAN = "halton-spline"


def merged_keys(features) -> Optional[dict]:
    """The config keys of a set of features, or None when two of them set one key to different values (halton and colored, cem and
    smooth)."""
    out = {}
    for f in sorted(features):
        for k, v in FEATURE_KEYS[f].items():
            if k in out and out[k] != v:
                return None
            out[k] = v
    return out


def implied(features):
    """The features the keys of `features` switch on: itself, plus every feature whose keys are all among them (horizon implies
    update_cov)."""
    keys = merged_keys(features)
    return frozenset(f for f, kv in FEATURE_KEYS.items() if all(k in keys and keys[k] == v for k, v in kv.items()))


def excluded(features) -> bool:
    """True when EXCLUSIONS refuses the set, as ``mode_refusal`` reads the table."""
    return any(name in features and set(features) & set(group) for subjects, group, _ in EXCLUSIONS for name in subjects)


def admitted(features) -> bool:
    return merged_keys(features) is not None and implied(features) == frozenset(features) and not excluded(features)


def maximal_combinations():
    """Every admitted set of features that no larger admitted set contains, computed from FEATURES, FEATURE_KEYS and EXCLUSIONS."""
    names = [f.name for f in FEATURES]
    sets = [frozenset(n for i, n in enumerate(names) if m >> i & 1) for m in range(1, 1 << len(names))]
    ok = [s for s in sets if admitted(s)]
    return {s for s in ok if not any(s < t for t in ok)}


class Case(NamedTuple):
    features: frozenset
    mode: Optional[str] = None          # "simple" or MEAN; None where cem / smooth fix the mode
    cov: Optional[str] = None           # "diag" or "full" with update_cov (not horizon); None otherwise
    scene: str = "point"                # point | boxer | panda
    u_per_command: int = 1

    @property
    def id(self):
        parts = sorted(self.features) or ["plain"]
        parts += [p for p in (self.mode, self.cov and f"cov {self.cov}", self.scene if self.scene != "point" else None,
                              f"u_per_command {self.u_per_command}" if self.u_per_command > 1 else None) if p]
        return "+".join(parts).replace(" ", "").replace(":", "=")

    def mppi_kw(self):
        kw = dict(PLAIN)
        kw.update(merged_keys(self.features))
        if self.mode:
            kw["mppi_mode"] = self.mode
        if self.cov:
            kw["cov_type"] = self.cov
        if self.u_per_command > 1:
            kw["u_per_command"] = self.u_per_command
        return kw

    def without(self, f):
        """The same case with feature `f` switched off (None when another feature implies it, so it cannot be switched off alone)."""
        rest = self.features - {f}
        if implied(rest) != rest:
            return None
        mode = self.mode or ("simple" if f in (CEM, SMOOTH) else None)
        cov = (self.cov or "diag") if "update_cov" in rest and HORIZON not in rest else None
        return self._replace(features=rest, mode=mode, cov=cov)


def expand(features, scene=None, u_per_command=1):
    """The cases of one feature set: SIMPLE and MEAN where the set leaves the mode open, diag and full where update_cov is on."""
    features = frozenset(features)
    modes = [None] if features & {CEM, SMOOTH} else ["simple", MEAN]
    covs = ["diag", "full"] if "update_cov" in features and HORIZON not in features else [None]
    scene = scene or ("boxer" if WORLDS in features else "point")
    return [Case(features, m, c, scene, u_per_command) for m in modes for c in covs]


def sweep():
    """The device sweep: plain, every feature alone, every maximal combination (each expanded), one panda case, and u_per_command = 2
    for the plain planner and every feature alone that admits it (smooth executes one action per plan)."""
    singles = [frozenset({f.name}) | implied({f.name}) for f in FEATURES]
    sets = list(dict.fromkeys([frozenset()] + singles + sorted(maximal_combinations(), key=sorted)))     # smooth and knots: single and maximal
    cases = [c for s in sets for c in expand(s)]
    cases.append(Case(frozenset({COLORED, "update_cov", "update_lambda", "filter_u"}), MEAN, "diag", "panda"))
    for s in [frozenset()] + [s for s in singles if SMOOTH not in s]:
        cases.append(expand(s, u_per_command=2)[0])
    return cases


class PointKeepOut(PointReachObjective):
    """Point reach that must stay left of the wall x = x_wall: the margin p_x - x_wall per row, built on the cost's device (the
    rollouts that cross the wall within the horizon violate it, the null sample and the slow ones do not)."""

    def __init__(self, x_wall=0.25, **kw):
        super().__init__(**kw)
        self.x_wall = x_wall

    def compute_constraint(self, sim):
        r = sim.get_actor_link_by_name(actor_name=self.actor, link_name=self.link)
        wall = torch.full((r.shape[0],), self.x_wall, dtype=torch.float32, device=r.device)
        return r[:, 0] - wall


Q0 = {"point": [0.1, 0.0, 0.0], "boxer": [0.0, 2.5, 0.0], "panda": [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]}


def cfg_of(case: Case, device, K=None, T=None):
    kw = case.mppi_kw()
    if case.scene == "point":
        return point_cfg(K=K or 128, T=T or 12, device=device, **kw)
    if case.scene == "boxer":
        return boxer_cfg(K=K or 128, T=T or 10, device=device, **kw)
    return panda_cfg(K=K or 256, T=T or 12, device=device, **kw)


def objective_of(case: Case):
    if case.scene == "boxer":
        return PushObjective(robot="boxer", link="ee_link")
    if case.scene == "panda":
        return PandaReachObjective()
    return PointKeepOut() if CONSTRAINED in case.features else PointReachObjective()


def case_ids(cases) -> Tuple[str, ...]:
    return tuple(c.id for c in cases)
