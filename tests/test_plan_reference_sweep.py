"""The reference side of ``test_gpu_plan_reference.py`` without a GPU: every sweep case maps to a reference backend, the cost replay
reproduces a planner's own plans bit for bit, and with any one feature switched off the reference, on the same recorded costs, plans
differently on a quantity the device test compares -- so a backend that ignores a feature fails here rather than on the device."""
import numpy as np
import pytest

import plan_paths as pp
import plan_reference as pr
from mppi_isaac_b200.model.blob import CEM, FEATURES, MODES, WORLDS

SWEEP = pp.sweep()
P = 3


def _library_missing():
    try:
        from mppi_isaac_b200.backend import load_library
        load_library()
        return None
    except (OSError, RuntimeError) as e:
        return str(e)


def test_family_table_names_every_feature():
    assert set(pr.FAMILY) == {f.name for f in FEATURES}
    assert set(pr.IMPLEMENTS) == set(pr.FAMILY.values())


def test_lookup_refuses_what_no_backend_implements():
    with pytest.raises(ValueError, match="no reference backend is known"):
        pr.backend_class(frozenset({"a feature added later"}))
    with pytest.raises(ValueError, match="together"):
        pr.backend_class(frozenset({CEM, MODES}))
    with pytest.raises(ValueError, match="does not implement"):
        pr.backend_class(frozenset({MODES, "update_cov"}))


def test_every_case_and_every_case_with_a_feature_off_has_a_backend():
    for case in SWEEP:
        pr.backend_class(case.features)
        for f in case.features:
            off = case.without(f)
            if off is not None:
                pr.backend_class(off.features)


@pytest.mark.parametrize("case", SWEEP, ids=pp.case_ids(SWEEP))
def test_replayed_reference_plans_and_every_feature_binds(case):
    if WORLDS in case.features or case.scene == "boxer":
        why = _library_missing()
        if why:
            pytest.skip(f"the boxer scene sizes its contact capacity through libmppib.so, which does not load here: {why}")
    inputs, states, plans, own = pr.device_run(case, "cpu", P, backend=pr.reference_backend(case))
    assert len(own) == P and all(np.isfinite(s["action"]).all() for s in own)
    again = pr.reference_run(case, inputs, states, plans)
    for p, (a, b) in enumerate(zip(own, again)):
        assert a.keys() == b.keys()
        bad = [k for k in a if not np.array_equal(a[k], b[k], equal_nan=True)]
        assert not bad, f"plan {p}: the replayed plan differs from the planner's own in {bad}"
    for f in sorted(case.features):
        off = case.without(f)
        if off is None:
            continue
        got = pr.reference_run(off, inputs, states, plans, exact_calls=False)
        # lock-step, a feature may only show after the plan it acts in: update_lambda moves lambda in K4, after U's update
        changed = {k for r, g in zip(own, got) for k in r.keys() & g.keys() if r[k].shape == g[k].shape and not np.array_equal(r[k], g[k])}
        assert changed, f"{f} changes nothing the planner computes in {case.id}"
