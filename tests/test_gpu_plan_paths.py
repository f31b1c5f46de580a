"""-m gpu: every configuration of the derived sweep (plan_paths.py) through every way ``MPPIisaacPlanner`` runs a plan on the device.

For each configuration P plans run with the same (q, qd) inputs -- those of the eager run, advanced by its actions -- and after every
plan the returned action, U, mean_action, the samples and every registered state (dist, smooth_state, mode_state, cstate, temp_state,
the anneal counter, the spline's U_exec) must be bit-identical to the eager planner's:

  A  eager batched plan (fused K3 + K4 tail), the baseline
  B  captured CUDA graph, replayed; captured exactly once
  C  the capture fails before it begins (torch.cuda.graph raises): eager fallback
  D  invalidate_graph() after plan 2 (update_weights, a base-pose change): re-captured
  E  stepwise rollout, split K3 / K4, one rollout launch per step
  F  keep_U rebuild after plan 2 (add_to_env, an obstacle added or resized), and once through a real obstacle change
  G  update_mppi_params after plan 2: equal to a freshly built planner on the same inputs

Every feature a configuration switches on must change U within the P plans, and with u_per_command = 2 every path returns
mean_action[:2].  Stepwise plans with a prior run against the float64 reference backends, lock-step, within each mode's plan gate."""
import numpy as np
import pytest
import torch

import plan_paths as pp
from mppi_isaac_b200.model.blob import FEATURES
from plan_reference import plan_gate, reference_backend

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
P = 4
SWEEP = pp.sweep()
IDS = pp.case_ids(SWEEP)
_EAGER = {}


def planner(case, device=DEV, **opts):
    from mppi_isaac_b200 import MPPIisaacPlanner
    return MPPIisaacPlanner(pp.cfg_of(case, device), pp.objective_of(case), **opts)


def snapshot(pl, returned):
    m = pl.mppi
    s = dict(action=returned.clone(), U=m.U.clone(), mean_action=m.mean_action.clone(), actions=m.actions.clone())
    for name, t in (("dist", m.dist), ("smooth_state", m.smooth_state), ("mode_state", m.mode_state), ("cstate", m.cstate),
                    ("temp_state", m.temp_state)):
        if t is not None:
            s[name] = t.clone()
    if m.anneal_state is not None:
        s["anneal_counter"] = m.anneal_state[:1].clone()
    if m.spline_table is not None:
        s["U_exec"] = m.spline_table[-m.T * m.nu:].clone()
    if m.u_per_command > 1:
        assert torch.equal(returned, m.mean_action[:m.u_per_command].cpu()), "u_per_command > 1 must return mean_action[:u_per_command]"
    return s


def run(pl, inputs, before=None):
    """The plans of `inputs` on `pl`; before(i, pl) runs ahead of plan i."""
    out = []
    for i, (q, qd) in enumerate(inputs):
        if before is not None:
            before(i, pl)
        out.append(snapshot(pl, pl.compute_action(q, qd)))
    return out


def eager(case):
    """Path A: the inputs (q advanced by the returned actions where the robot is velocity-driven in every joint) and the snapshots."""
    if case not in _EAGER:
        pl = planner(case, use_cuda_graph=False)
        q = np.asarray(pp.Q0[case.scene], np.float64)
        qd = np.zeros_like(q)
        inputs, out = [], []
        for _ in range(P):
            inputs.append((q.copy(), qd.copy()))
            a = pl.compute_action(q, qd)
            out.append(snapshot(pl, a))
            a0 = a.numpy().reshape(-1, pl.mppi.nu)[0].astype(np.float64)
            if a0.shape == q.shape:
                q, qd = q + 0.05 * a0, a0
        assert pl.mppi._graph is None
        _EAGER[case] = (inputs, out)
    return _EAGER[case]


def assert_equal_runs(ref, got, what, first=0):
    for i, (r, g) in enumerate(zip(ref, got)):
        assert r.keys() == g.keys(), f"{what}: plan {first + i + 1} registers {sorted(g)} instead of {sorted(r)}"
        bad = [k for k in r if not torch.equal(r[k], g[k])]
        assert not bad, f"{what}: plan {first + i + 1} differs from the eager plan in {bad}"


def _graphs(record):
    def before(i, pl):
        if i > 0:
            record.append(pl.mppi._graph)
    return before


@pytest.mark.parametrize("case", SWEEP, ids=IDS)
def test_b_graph_replay_equals_the_eager_plan(case):
    inputs, ref = eager(case)
    pl = planner(case, use_cuda_graph=True)
    graphs = []
    got = run(pl, inputs, _graphs(graphs))
    graphs.append(pl.mppi._graph)
    assert graphs[0] is not None and all(g is graphs[0] for g in graphs), "the plan must be captured once and replayed"
    assert_equal_runs(ref, got, "graph replay")


def _refuse(*a, **kw):
    raise RuntimeError("capture refused before it began")


@pytest.mark.parametrize("case", SWEEP, ids=IDS)
def test_c_failed_capture_falls_back_to_the_eager_plan(case, monkeypatch):
    """The warm-up plans of a capture that fails must leave no trace: the first action is the first plan's, not the third's."""
    inputs, ref = eager(case)
    monkeypatch.setattr(torch.cuda, "graph", _refuse)
    pl = planner(case, use_cuda_graph=True)
    got = run(pl, inputs)
    assert pl.mppi._graph_failed and pl.mppi._graph is None
    assert_equal_runs(ref, got, "capture fallback")


@pytest.mark.parametrize("case", SWEEP, ids=IDS)
def test_d_recapture_after_invalidate_equals_the_eager_plan(case):
    inputs, ref = eager(case)
    pl = planner(case, use_cuda_graph=True)
    graphs = []
    record = _graphs(graphs)

    def before(i, pl):
        record(i, pl)
        if i == 2:
            pl.mppi.invalidate_graph()
    got = run(pl, inputs, before)
    graphs.append(pl.mppi._graph)
    assert graphs[0] is not None and graphs[0] is graphs[1]
    assert graphs[2] is not None and graphs[2] is not graphs[1], "invalidate_graph() must lead to a new capture"
    assert_equal_runs(ref, got, "re-capture")


@pytest.mark.parametrize("case", SWEEP, ids=IDS)
def test_e_stepwise_equals_the_eager_plan(case):
    """Split K3 / K4 equals the fused tail and the stepwise rollout the batched one, bit for bit, for every rule."""
    inputs, ref = eager(case)
    pl = planner(case, rollout_mode="stepwise")
    assert pl.mppi.rollout_mode == "stepwise"
    assert_equal_runs(ref, run(pl, inputs), "stepwise")


@pytest.mark.parametrize("case", SWEEP, ids=IDS)
def test_f_keep_u_rebuild_continues_the_eager_plan(case):
    """A rebuild with keep_U (what add_to_env and the obstacle path do) carries everything a plan leaves for the next, the plan counter
    included: the rebuilt planner continues the random stream instead of repeating plans 0, 1, ..."""
    inputs, ref = eager(case)
    pl = planner(case, use_cuda_graph=False)

    def before(i, pl):
        if i == 2:
            pl._build_mppi(keep_U=True)
    assert_equal_runs(ref, run(pl, inputs, before), "keep_U rebuild")


@pytest.mark.parametrize("case", SWEEP, ids=IDS)
def test_g_update_mppi_params_resets_the_planner(case):
    inputs, ref = eager(case)
    pl = planner(case, use_cuda_graph=False)

    def before(i, pl):
        if i == 2:
            pl.update_mppi_params({"noise_sigma": pl.cfg.mppi.noise_sigma})
    got = run(pl, inputs, before)
    assert_equal_runs(ref[:2], got[:2], "update_mppi_params, before the update")
    fresh = run(planner(case, use_cuda_graph=False), inputs[2:])
    assert_equal_runs(fresh, got[2:], "update_mppi_params against a fresh planner", first=2)


@pytest.mark.parametrize("case", [c for c in SWEEP if c.features], ids=[c.id for c in SWEEP if c.features])
def test_every_feature_binds(case):
    """With one feature switched off the plans change: a configuration whose feature changes nothing would test nothing."""
    inputs, ref = eager(case)
    checked = 0
    for f in sorted(case.features):
        off = case.without(f)
        if off is None:
            continue                                 # implied by another feature of the set (update_cov by cov_type: horizon)
        got = run(planner(off, use_cuda_graph=False), inputs)
        key = "U" if got[0]["U"].shape == ref[0]["U"].shape else "mean_action"
        assert any(not torch.equal(r[key], g[key]) for r, g in zip(ref, got)), f"{f} changes no plan of {case.id}"
        checked += 1
    assert checked > 0


OBSTACLE = {"sphere": {"position": [2.0, -1.5, 0.0], "velocity": [0.0, 0.0, 0.0], "size": [0.1]}}
REBUILD = [c for c in SWEEP if c.scene == "point" and c.u_per_command == 1 and c.mode in (None, "simple") and c.cov in (None, "full")]


@pytest.mark.parametrize("case", REBUILD, ids=[c.id for c in REBUILD])
def test_f_obstacle_rebuild_carries_every_state(case):
    """An added sphere obstacle rebuilds the simulator and the planner (compute_action's path): right after the rebuild every carried
    state equals its value before, bit for bit."""
    inputs, _ = eager(case)
    pl = planner(case, use_cuda_graph=True)
    run(pl, inputs[:2])
    build, seen = pl._build_mppi, {}

    def spy(keep_U=False):
        seen["before"] = {k: t.clone() for k, t in pl.mppi.persistent_state().items()}
        build(keep_U=keep_U)
        seen["after"] = {k: t.clone() for k, t in pl.mppi.persistent_state().items()}
    pl._build_mppi = spy
    q, qd = inputs[2]
    a = pl.compute_action(q, qd, obst=OBSTACLE)
    assert seen, "adding an obstacle must rebuild the planner"
    assert seen["after"].keys() == seen["before"].keys()
    for k in seen["before"]:
        assert torch.equal(seen["after"][k], seen["before"][k]), f"{k} is not carried over the rebuild"
    assert torch.isfinite(a).all() and pl.mppi._graph is not None


# ------------------------------------------------------------------------------------------------------------------------------------
# stepwise plans with a prior against the float64 reference
# ------------------------------------------------------------------------------------------------------------------------------------
NO_PRIOR = {f.name for f in FEATURES if f.no_prior}
PRIOR_CASES = [c for c in SWEEP if c.scene == "point" and c.u_per_command == 1 and not c.features & NO_PRIOR]
PRIOR_COMMAND = (0.25, -0.125, 0.5)


class ConstPrior:
    def compute_command(self, sim):
        return torch.tensor(PRIOR_COMMAND)


@pytest.mark.parametrize("case", PRIOR_CASES, ids=[c.id for c in PRIOR_CASES])
def test_stepwise_plans_with_a_prior_match_the_reference(case):
    """Three stepwise plans with a prior on the device and through the float64 reference, lock-step (the reference starts every plan
    from the device's carried state): the prior row is the prior's command, bit for bit, and the actions agree within the gate."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    pls = []
    for device, backend in ((DEV, None), ("cpu", reference_backend(case))):
        cfg = pp.cfg_of(case, device)
        cfg.mppi.use_priors = True
        pls.append(MPPIisaacPlanner(cfg, pp.objective_of(case), ConstPrior(), **({} if backend is None else dict(backend=backend))))
    gpu, ref = pls
    assert gpu.mppi.rollout_mode == "stepwise" and ref.mppi.rollout_mode == "stepwise"
    K, lim = gpu.mppi.K, float(gpu.mppi.backend.params.u_max[0])
    gate = plan_gate(case, lim)
    prior = torch.tensor(PRIOR_COMMAND, dtype=torch.float32)
    q, qd = np.asarray(pp.Q0["point"], np.float64), np.zeros(3)
    for it in range(3):
        for k, t in gpu.mppi.persistent_state().items():
            ref.mppi.persistent_state()[k].copy_(t.cpu())
        ag, ar = gpu.compute_action(q, qd), ref.compute_action(q, qd)
        for pl in (gpu, ref):
            row = pl.mppi.actions[:, :, K - 2].cpu()
            assert torch.equal(row, prior.expand_as(row)), f"plan {it}: the prior row is not the prior's command"
        assert float((ag - ar).abs().max()) <= gate, f"plan {it}: |d action| = {float((ag - ar).abs().max()):.3g} > {gate:.3g}"
        q, qd = q + 0.05 * ar.numpy().astype(np.float64), ar.numpy().astype(np.float64)
