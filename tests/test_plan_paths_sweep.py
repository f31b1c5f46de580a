"""The sweep of ``test_gpu_plan_paths.py`` without a GPU: FEATURE_KEYS names every feature, every configuration is one the planner
admits and switches on exactly its features, and the maximal combinations are those EXCLUSIONS admits."""
import copy

import pytest

import plan_paths as pp
from mppi_isaac_b200.model.blob import CEM, COLORED, EXCLUSIONS, FEATURES, HALTON, WORLDS, make_params, mode_refusal

SWEEP = pp.sweep()


def test_feature_keys_cover_every_feature():
    assert set(pp.FEATURE_KEYS) == {f.name for f in FEATURES}


def test_exclusions_name_only_known_features():
    for subjects, group, _ in EXCLUSIONS:
        assert set(subjects) | set(group) <= set(pp.FEATURE_KEYS)


@pytest.mark.parametrize("case", SWEEP, ids=pp.case_ids(SWEEP))
def test_every_configuration_is_admitted_and_switches_on_its_features(case):
    cfg = pp.cfg_of(case, "cpu")
    nu = len(cfg.mppi.noise_sigma)
    p = make_params(cfg.mppi, cfg.isaacgym, nu, int(cfg.mppi.num_samples), [])
    assert mode_refusal(p, nu, cfg.mppi) is None
    assert {f.name for f in FEATURES if f.on(p, cfg.mppi)} == set(case.features)
    assert p.cov_full == int(case.cov == "full")


def test_maximal_combinations_are_those_the_exclusions_admit():
    """Computed here by trying every set through make_params: a pair newly admitted (or refused) joins (or leaves) the sweep."""
    names = [f.name for f in FEATURES]
    base = {scene: pp.cfg_of(pp.Case(frozenset(), "simple", scene=scene), "cpu") for scene in ("point", "boxer")}
    admitted = []
    for m in range(1 << len(names)):
        s = frozenset(n for i, n in enumerate(names) if m >> i & 1)
        if pp.merged_keys(s) is None:
            continue
        case = pp.Case(s, None if s & {CEM, pp.SMOOTH} else "simple", None, "boxer" if WORLDS in s else "point")
        cfg = base[case.scene]
        mc = copy.copy(cfg.mppi)
        for k, v in case.mppi_kw().items():
            setattr(mc, k, v)
        nu = len(mc.noise_sigma)
        try:
            p = make_params(mc, cfg.isaacgym, nu, int(mc.num_samples), [])
        except ValueError:
            continue
        if {f.name for f in FEATURES if f.on(p, mc)} == s:
            admitted.append(s)
    maximal = {s for s in admitted if not any(s < t for t in admitted)}
    assert maximal == pp.maximal_combinations()
    swept = {c.features for c in SWEEP}
    assert maximal <= swept


def test_sweep_covers_every_feature_alone_both_modes_both_cov_types_and_cem_noise():
    feats = {c.features for c in SWEEP}
    assert frozenset() in feats
    for f in FEATURES:
        assert frozenset({f.name}) | pp.implied({f.name}) in feats
    for c in (c for c in SWEEP if c.scene != "panda" and c.u_per_command == 1):
        if c.mode == "simple":
            assert c._replace(mode=pp.MEAN) in SWEEP
        if c.cov == "diag":
            assert c._replace(cov="full") in SWEEP
    cem = [c for c in SWEEP if CEM in c.features]
    assert any(COLORED in c.features for c in cem) and any(not c.features & {COLORED, HALTON} for c in cem)
    assert {c.scene for c in SWEEP} == {"point", "boxer", "panda"}


def test_feature_off_is_a_configuration_the_planner_admits():
    for case in SWEEP:
        for f in case.features:
            off = case.without(f)
            if off is None:
                continue
            cfg = pp.cfg_of(off, "cpu")
            nu = len(cfg.mppi.noise_sigma)
            p = make_params(cfg.mppi, cfg.isaacgym, nu, int(cfg.mppi.num_samples), [])
            assert mode_refusal(p, nu, cfg.mppi) is None
            assert {g.name for g in FEATURES if g.on(p, cfg.mppi)} == set(off.features), (case.id, f)
