"""The float64 reference of every configuration of the plan sweep (plan_paths.py), and the cost replay that holds a device plan to it.

``reference_backend(case)`` is the checker backend that implements every feature of a sweep case.  ``FAMILY`` names, for every feature
of ``blob.FEATURES``, the backend family that implements it, and ``IMPLEMENTS`` what each family implements besides its own feature: a
case whose features no family implements together is refused, so a feature added to FEATURES must extend both tables.

Cost replay: ``Recording`` wraps the device planner's Objective and keeps a copy of every ``compute_cost`` (and, under constraint_mode,
``compute_constraint``) result in call order, one list per plan -- one call per iteration, so the anneal and CEM iterations come in order.
``Replay`` hands the same tensors, in the same order, to the CPU planner that runs the reference backend.  Before each plan the reference
takes the device's persistent_state() (U, plan_ctr, dist, smooth_state, mode_state), so it draws its own samples in float64 from the
same Philox counters and runs its own K3, K4 and shift on costs that are exact for the device's samples: what the float32 and float64
rollouts of a contact scene would make of those samples drops out of the comparison."""
import numpy as np
import torch

import plan_paths as pp
from mppi_isaac_b200.model.blob import (ANNEALED, CEM, COLORED, CONSTRAINED, ESS, FEATURES, HALTON, KNOTS, MODES, SMOOTH, WORLDS,
                                        spline_basis)
from mppi_isaac_b200.planner.mppi import colored_noise_chol

# the backend family of every feature: the family of a case is that of its one feature outside "constraint" ("constraint" if none)
FAMILY = {CEM: "cem", SMOOTH: "smooth", MODES: "modes", pp.HORIZON: "horizon", ESS: "ess", CONSTRAINED: "constraint",
          KNOTS: "constraint", ANNEALED: "constraint", WORLDS: "constraint", COLORED: "constraint", HALTON: "constraint",
          "update_cov": "constraint", "update_lambda": "constraint", "filter_u": "constraint"}
# the features each family's backend implements besides those FAMILY gives it (its parents in the oracle's class chain)
IMPLEMENTS = {"cem": {COLORED, "filter_u"}, "smooth": set(), "modes": {COLORED, HALTON, "filter_u"},
              "horizon": {"update_cov", "update_lambda", HALTON, "filter_u"},
              "ess": {COLORED, HALTON, "update_cov", "update_lambda", "filter_u"}, "constraint": set()}


def family(features):
    """The backend family that implements every feature of `features`; ValueError when FAMILY does not know a feature or no single
    family implements the set."""
    unknown = set(features) - set(FAMILY)
    if unknown:
        raise ValueError(f"no reference backend is known for {sorted(unknown)}: extend plan_reference.FAMILY")
    own = {FAMILY[f] for f in features} - {"constraint"}
    if len(own) > 1:
        raise ValueError(f"no reference backend implements {sorted(features)} together (families {sorted(own)})")
    fam = own.pop() if own else "constraint"
    rest = set(features) - {f for f in FAMILY if FAMILY[f] == fam} - IMPLEMENTS[fam]
    if rest:
        raise ValueError(f"the {fam} reference backend does not implement {sorted(rest)}")
    return fam


def backend_class(features):
    fam = family(features)
    if fam == "cem":
        import cem_oracle as ce
        return ce.CemOracleBackend
    if fam == "smooth":
        import smooth_oracle as sm
        return sm.SmoothOracleBackend
    if fam == "modes":
        import modes_oracle as mo
        return mo.ModesOracleBackend
    if fam == "horizon":
        import adaptive_horizon_oracle as aho
        return aho.AdaptiveHorizonOracleBackend
    if fam == "ess":
        return TemperatureColoredOracleBackend
    import constraint_oracle as cn
    return cn.ConstraintOracleBackend


def reference_backend(case, nthreads=8):
    return backend_class(case.features)(nthreads=nthreads)


def _temperature_colored():
    import colored_oracle as co
    import temperature_oracle as tmo

    class TemperatureColoredOracleBackend(tmo.TemperatureMixin, co.ColoredOracleBackend):
        """The temperature rule over the colored checker backend: ESS with colored or Halton noise, diag or full update_cov."""
    return TemperatureColoredOracleBackend


TemperatureColoredOracleBackend = _temperature_colored()


# ------------------------------------------------------------------------------------------------------------------------------------
# cost replay
# ------------------------------------------------------------------------------------------------------------------------------------
class Recording:
    """The Objective of the device planner: every cost and constraint it returns after new_plan() is copied to the host, per plan."""

    def __init__(self, objective):
        self.objective = objective
        self.plans = None

    def __getattr__(self, name):
        return getattr(self.objective, name)

    def new_plan(self):
        if self.plans is None:
            self.plans = []
        self.plans.append(dict(cost=[], constraint=[]))

    def _keep(self, kind, t):
        if self.plans is not None:
            self.plans[-1][kind].append(t.detach().to("cpu", torch.float32).clone())
        return t

    def compute_cost(self, sim):
        return self._keep("cost", self.objective.compute_cost(sim))

    def compute_constraint(self, sim):
        return self._keep("constraint", self.objective.compute_constraint(sim))


class Replay:
    """The Objective of the reference planner: before arm() (the trace at construction) the Objective itself, then the recorded
    tensors of one plan in call order."""

    def __init__(self, objective):
        self.objective = objective
        self.queue = None

    def __getattr__(self, name):
        return getattr(self.objective, name)

    def arm(self, plan):
        self.queue = {k: list(v) for k, v in plan.items()}

    def left(self):
        return sum(len(v) for v in self.queue.values())

    def _next(self, kind, sim):
        if self.queue is None:
            return getattr(self.objective, "compute_" + kind)(sim)
        if not self.queue[kind]:
            raise RuntimeError(f"the reference asked for more {kind} calls than the device plan made")
        return self.queue[kind].pop(0)

    def compute_cost(self, sim):
        return self._next("cost", sim)

    def compute_constraint(self, sim):
        return self._next("constraint", sim)


def snapshot(pl, returned):
    """Everything a plan computes that the reference computes too, as float64 numpy arrays (integer counts as int64)."""
    m = pl.mppi
    f = lambda t: t.detach().cpu().double().numpy().copy()
    s = dict(action=f(returned), U=f(m.U), mean_action=f(m.mean_action), actions=f(m.actions), noise=f(m.noise))
    if m.xk is not None:
        s["knot_samples"] = f(m.xk)
    if m.current_lambda is not None:
        # lambda apart from the covariance and each of Sigma, L, Sigma^-1 apart, so each is measured against its own magnitude
        s["lambda"] = f(m.dist[:1])
        n = m.T * m.nu if m.cov_horizon else m.nu
        blocks = ("Sigma", "L", "Sigma_inv") if m.cov_full or m.cov_horizon else ("cov",)
        for i, name in enumerate(blocks):
            s[name] = f(m.dist[1 + i * n * n:1 + (i + 1) * n * n] if len(blocks) > 1 else m.dist[1:])
    elif m.dist is not None:
        s["dist"] = f(m.dist)
    for name, t in (("smooth_state", m.smooth_state), ("mode_state", m.mode_state)):
        if t is not None:
            s[name] = f(t)
    if m.cstate is not None:
        s["cstate"] = f(m.cstate[1:])
        s["n_feasible"] = m.cstate[0:1].cpu().view(torch.int32).numpy().astype(np.int64)
    if m.temp_state is not None:
        s["temp_state"] = np.delete(f(m.temp_state), 2 * len(m.ess_grid))
        s["n_valid"] = np.array([m.valid_samples], np.int64)
    if m.anneal_state is not None:
        s["anneal_counter"] = f(m.anneal_state[:1])
    return s


SAMPLES = ("actions", "noise", "knot_samples")
EXACT = ("n_feasible", "n_valid", "anneal_counter")
RELATIVE = ("lambda",)


def planner(case, device, objective, **opts):
    from mppi_isaac_b200 import MPPIisaacPlanner
    return MPPIisaacPlanner(pp.cfg_of(case, device), objective, **opts)


def advance(q, a, nu):
    """The next plan's (q, qd): q moved by the first returned action where the robot is velocity-driven in every joint."""
    a0 = a.numpy().reshape(-1, nu)[0].astype(np.float64)
    if a0.shape == q.shape:
        return q + 0.05 * a0, a0
    return q, np.zeros_like(q)


def device_run(case, device, P, **opts):
    """P eager plans on `device`: (inputs, device state before every plan, recorded costs of every plan, snapshots)."""
    rec = Recording(pp.objective_of(case))
    pl = planner(case, device, rec, use_cuda_graph=False, **opts)
    q = np.asarray(pp.Q0[case.scene], np.float64)
    qd = np.zeros_like(q)
    inputs, states, snaps = [], [], []
    for _ in range(P):
        inputs.append((q.copy(), qd.copy()))
        states.append({k: t.detach().cpu().clone() for k, t in pl.mppi.persistent_state().items()})
        rec.new_plan()
        a = pl.compute_action(q, qd)
        snaps.append(snapshot(pl, a))
        q, qd = advance(q, a, pl.mppi.nu)
    assert pl.mppi.rollout_mode == "batched" and pl.mppi._graph is None
    return inputs, states, rec.plans, snaps


def reference_run(case, inputs, states, plans, backend=None, exact_calls=True):
    """The reference planner of `case` through the same plans, lock-step: before plan p it takes states[p] (where it has a buffer of
    that name and shape) and replays plans[p]."""
    rep = Replay(pp.objective_of(case))
    pl = planner(case, "cpu", rep, backend=backend or reference_backend(case))
    snaps = []
    for (q, qd), state, plan in zip(inputs, states, plans):
        own = pl.mppi.persistent_state()
        for k, t in state.items():
            if k in own and own[k].shape == t.shape:
                own[k].copy_(t)
        rep.arm(plan)
        snaps.append(snapshot(pl, pl.compute_action(q, qd)))
        if exact_calls:
            assert rep.left() == 0, f"the reference used fewer cost calls than the device plan made ({rep.left()} left)"
    return snaps


# ------------------------------------------------------------------------------------------------------------------------------------
# gates
# ------------------------------------------------------------------------------------------------------------------------------------
def plan_gate(case, u_lim):
    """The whole-plan gate of the mode's own test: test_gpu_adaptive_horizon's and, off the panda, test_gpu_adaptive_full's 5e-4; the
    plan-parity gate 2e-4 max(1, u_lim) of every other mode (DESIGN.md section 2)."""
    if pp.HORIZON in case.features or case.cov == "full":
        return 5e-4
    return 2e-4 * max(1.0, u_lim)


def k1_gate(case, cfg):
    """The K1 gate of test_gpu_mppi_shapes, 2e-6 max(1, 6 |L|_inf), with L the control factor of the configured Sigma times, with
    colored noise, the temporal factor; the coloured Halton library's 1e-4 max(1, |L|_inf) (test_gpu_adaptive_full)."""
    L = np.linalg.cholesky(np.asarray(cfg.mppi.noise_sigma, np.float64))
    n = np.abs(L).sum(1).max()
    if HALTON in case.features:
        return 1e-4 * max(1.0, n)
    if COLORED in case.features:
        n *= np.abs(colored_noise_chol(int(cfg.mppi.horizon), float(cfg.mppi.noise_beta))).sum(1).max()
    if KNOTS in case.features:
        B, _, _ = spline_basis(int(cfg.mppi.horizon), int(cfg.mppi.control_knots), int(cfg.mppi.spline_degree))
        n *= max(1.0, np.abs(B).sum(1).max())
    return 2e-6 * max(1.0, 6 * n)


def null_columns(case):
    """The sample columns drawn as the null action: the last control sample (its n_worlds rollouts with risk)."""
    R = pp.FEATURE_KEYS[WORLDS]["n_worlds"] if WORLDS in case.features else 1
    return slice(-R, None)


def errors(case, dev, ref, gates):
    """{quantity: error / gate} of one plan over the quantities both snapshots hold in the same shape.  Samples: the largest error over the
    K1 gate (of the non-null columns for the actions, and inf unless their null columns are equal bit for bit).  Counts and the anneal counter: inf unless
    equal.  Everything else: the largest error relative to max(1, |reference|) (to |reference| for lambda) over the plan gate, inf
    where +-inf or NaN differ."""
    out = {}
    for k in dev.keys() & ref.keys():
        g, r = dev[k], ref[k]
        if g.shape != r.shape:
            continue
        if k in EXACT:
            out[k] = 0.0 if np.array_equal(g, r) else np.inf
        elif k == "actions":
            null = null_columns(case)
            body = slice(0, g.shape[-1] + null.start)
            e = float(np.abs(g[..., body] - r[..., body]).max(initial=0.0)) / gates["k1"]
            out[k] = e if np.array_equal(g[..., null], r[..., null]) else np.inf
        elif k in SAMPLES:
            # the null columns of noise and knot samples are -U, and U differs by K4's rounding after the first iteration of a plan
            out[k] = float(np.abs(g - r).max(initial=0.0)) / gates["k1"]
        else:
            fin = np.isfinite(r)
            if not np.array_equal(fin, np.isfinite(g)) or not np.array_equal(g[~fin], r[~fin]):
                out[k] = np.inf
                continue
            mag = float(np.abs(r[fin]).max(initial=0.0))
            scale = mag if k in RELATIVE and mag > 0 else max(1.0, mag)
            out[k] = float(np.abs(g[fin] - r[fin]).max(initial=0.0)) / scale / gates["plan"]
    return out


def worst(errs):
    """(quantity, error / gate) of the largest ratio in a {quantity: ratio} dict."""
    k = max(errs, key=errs.get)
    return k, errs[k]
