"""-m gpu: every configuration of the plan sweep (plan_paths.py) against the float64 reference, plan by plan, on the device's own costs.

The device planner runs P eager batched plans; every cost (and constraint) its Objective returns is recorded and replayed, in call
order, to the CPU planner over the reference backend of the configuration (plan_reference.py), which starts every plan from the device's
carried state.  After every plan the samples, the returned action, U, mean_action (U_exec with knots), dist (Sigma, L, Sigma^-1 and
lambda, the ESS-chosen one included), smooth_state, mode_state, cstate, the temperature state and the anneal counter must agree within
the mode's plan gate (the samples within the K1 gate, the null columns of the actions bit for bit, the counts exactly).  Each case
prints one ``PLANREF <id> worst <quantity> <error/gate> gate <plan gate>`` line (-s).

Negative controls, each of which must miss a gate on at least one compared quantity over the P plans:
  * feature off: for every feature f of the case that can be switched off alone, the reference with f off on the same recorded costs;
  * stale plan: device plan p against reference plan p - 1."""
import pytest

import plan_paths as pp
import plan_reference as pr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
P = 4
SWEEP = pp.sweep()
IDS = pp.case_ids(SWEEP)
_RUNS = {}


def runs(case):
    """(inputs, device states before every plan, recorded costs, device snapshots, reference snapshots, gates) of `case`."""
    if case not in _RUNS:
        inputs, states, plans, dev = pr.device_run(case, DEV, P)
        ref = pr.reference_run(case, inputs, states, plans)
        cfg = pp.cfg_of(case, "cpu")
        gates = dict(k1=pr.k1_gate(case, cfg), plan=pr.plan_gate(case, max(abs(v) for v in cfg.mppi.u_max)))
        _RUNS[case] = (inputs, states, plans, dev, ref, gates)
    return _RUNS[case]


def worst_over(case, dev, ref, gates):
    return max((pr.worst(pr.errors(case, d, r, gates)) for d, r in zip(dev, ref)), key=lambda kv: kv[1])


@pytest.mark.parametrize("case", SWEEP, ids=IDS)
def test_plans_match_the_reference(case):
    _, _, _, dev, ref, gates = runs(case)
    worst = ("", 0.0)
    for p, (d, r) in enumerate(zip(dev, ref)):
        errs = pr.errors(case, d, r, gates)
        assert {"action", "U", "mean_action", "actions", "noise"} <= errs.keys(), f"plan {p}: compared only {sorted(errs)}"
        for name in ("lambda", "cov", "Sigma", "L", "Sigma_inv", "dist", "smooth_state", "mode_state", "cstate", "temp_state",
                     "anneal_counter", "knot_samples"):
            assert (name in d) == (name in errs), f"plan {p}: {name} is registered on one side only"
        bad = {k: v for k, v in errs.items() if not v <= 1.0}
        assert not bad, f"plan {p}: error / gate {bad}"
        worst = max(worst, pr.worst(errs), key=lambda kv: kv[1])
    print(f"PLANREF {case.id} worst {worst[0]} {worst[1]:.3f} gate {gates['plan']:.1e} k1 gate {gates['k1']:.1e}")


@pytest.mark.parametrize("case", [c for c in SWEEP if c.features], ids=[c.id for c in SWEEP if c.features])
def test_reference_with_a_feature_off_misses(case):
    inputs, states, plans, dev, _, gates = runs(case)
    checked = 0
    for f in sorted(case.features):
        off = case.without(f)
        if off is None:
            continue                                 # implied by another feature of the set (update_cov by cov_type: horizon)
        ref = pr.reference_run(off, inputs, states, plans, exact_calls=False)
        k, e = worst_over(case, dev, ref, gates)
        print(f"PLANREF-OFF {case.id} without {f}: worst {k} {e:.3g}")
        assert e > 1.0, f"the reference without {f} passes every gate of {case.id}"
        checked += 1
    assert checked > 0


@pytest.mark.parametrize("case", SWEEP, ids=IDS)
def test_stale_reference_plan_misses(case):
    _, _, _, dev, ref, gates = runs(case)
    k, e = worst_over(case, dev[1:], ref[:-1], gates)
    assert e > 1.0, f"device plans 1..{P - 1} pass against reference plans 0..{P - 2}"

