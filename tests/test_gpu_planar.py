"""-m gpu: the planar differential-drive base (synth_planar.py) on every team instantiation it reaches and on the thread-per-rollout
kernel, against the float64 oracle.  The test id names the instantiation: team <G, NB> contact-free (<8,4>, <8,8>, <16,12>, <16,16>),
team <G, NB, true, NCS, 8> with contacts (NCS 1-4 on NB 4 and 8, 2-5 on NB 12, 2-4 on NB 16), and "thread" (MPPIB_K2_TEAM=0).

The planar rule recomputes the targets of joints 0-2 every substep from the current yaw and fwd_axis, with friction-cone effort
limits that nearly always bind (virtual-joint gains n kd / r^2 ~ 1e5): the lock-step exclusion of test_gpu_synth.py is extended to
those targets and limits.  Each test prints its worst errors ("SYNTH-PLANAR ..." lines, visible with -s)."""
import copy
import math

import numpy as np
import pytest
import torch

from synth_planar import (CONTACT_CASES, FREE_CASES, G, WALL_FACE, contact_case_id, free_case_id, make_contact_case, make_planar_robot,
                          planar_states, planar_targets, rot_z, symmetric_base)
from test_gpu_contact_synth import gates
from test_gpu_synth import FREE_GATES, GUARD, GUARD_VALUE, _compare_free_running, _guarded, _unlimited, backend, dev

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MAPPINGS = ("team", "thread")
PROBE = 2e-6


def _id(cid, mapping):
    return cid if mapping == "team" else cid.rsplit("-", 1)[0] + "-thread"


FREE_PARAMS = [pytest.param(c, mp, id=_id(free_case_id(c), mp)) for c in FREE_CASES for mp in MAPPINGS]
CONTACT_PARAMS = [pytest.param(c, mp, id=_id(contact_case_id(c), mp)) for c in CONTACT_CASES for mp in MAPPINGS]


@pytest.fixture(scope="module")
def synth_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("synth_planar_gpu")


def report(test, **vals):
    print(f"SYNTH-PLANAR {test} " + " ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}" for k, v in vals.items()))


def _robot(synth_dir, case, **kw):
    nw, narm, topo = case
    return make_planar_robot(synth_dir, 0, narm, topo, nwheels=nw, **kw)


def _near_saturation(oracle, sc, p, actions, t, state):
    """Rollouts whose unsaturated drive force lies within 1e-3 (relative) of an effort limit -- the planar targets and friction-cone
    limits of joints 0-2 included: float32 may take the other saturation decision there."""
    m, nb = sc.model, sc.ndof
    unsat, _ = oracle.rollout(_unlimited(m), p, None, actions, t, 1, state=state.copy(), want_obs=False, use_double=True)
    tgt = planar_targets(sc, p, state, actions[t])
    eff = np.array(m.effort[:nb], np.float64)[:, None]
    kd = np.array(m.kd[:nb], np.float64)[:, None]
    td = kd * (tgt - unsat[nb:2 * nb].astype(np.float64))
    return (np.abs(np.abs(td) / eff - 1.0) <= 1e-3).any(axis=0)


def lockstep(oracle, monkeypatch, sc, p, mapping, actions, state, steps, obs_rows=False):
    """The oracle's state re-injected before every step (substeps = 1: the yaw of the targets is the step's starting yaw).  Returns
    worst |dq| (yaw apart), |dyaw|, |dqd|, the worst chassis-row position / quaternion (up to sign) errors and the excluded
    rollout-steps."""
    be = backend(monkeypatch, sc, p, mapping)
    nb, K = sc.ndof, p.K
    assert p.substeps == 1
    a_d = dev(actions)
    w = dict(dq=0.0, dyaw=0.0, dqd=0.0, pos=0.0, quat=0.0)
    excluded = 0
    obs = torch.zeros((be.obs_size(), p.T, K), device=DEV)
    for t in range(steps):
        st = dev(state)
        be.rollout(None, st, a_d, t, 1, obs)
        ref, o_ref = oracle.rollout(sc.model, p, None, actions, t, 1, state=state.copy(), use_double=True)
        near = _near_saturation(oracle, sc, p, actions, t, state)
        g, o = st.cpu().numpy(), obs[:, t].cpu().numpy()
        assert np.isfinite(g).all() and np.isfinite(o).all()
        excluded += int(near.sum())
        keep = ~near
        d = np.abs(g[:, keep] - ref[:, keep])
        w["dq"] = max(w["dq"], float(np.delete(d[:nb], 2, axis=0).max()))
        w["dyaw"] = max(w["dyaw"], float(d[2].max()))
        w["dqd"] = max(w["dqd"], float(d[nb:2 * nb].max()))
        w["pos"] = max(w["pos"], float(np.abs(o[0:3, keep] - o_ref[0:3, t, keep]).max()))
        qa, qb = o[3:7, keep], o_ref[3:7, t, keep]
        w["quat"] = max(w["quat"], float(np.minimum(np.abs(qa - qb).max(axis=0), np.abs(qa + qb).max(axis=0)).max()))
        state = ref
    return w, excluded


@pytest.mark.parametrize("case,mapping", FREE_PARAMS)
def test_one_step_lockstep(oracle, monkeypatch, synth_dir, case, mapping):
    K, T = 128, 6
    sc, p, s0 = _robot(synth_dir, case, K=K, T=T)
    rng = np.random.default_rng(sc.ndof)
    actions = rng.uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    actions[:, :, : K // 4] *= 0.05                                          # a quarter of the rollouts drives gently
    w, excl = lockstep(oracle, monkeypatch, sc, p, mapping, actions, planar_states(sc, s0, K, rng), T)
    report("lockstep", id=_id(free_case_id(case), mapping), excluded=excl, **w)
    assert w["dq"] <= 1e-5 and w["dyaw"] <= 1e-5                              # stated gate
    assert w["dq"] <= 2e-6 and w["dyaw"] <= 2e-6 and w["dqd"] <= 1e-4, w     # what float32 delivers (test_gpu_synth.py)
    assert w["pos"] <= 2e-6 and w["quat"] <= 2e-6, w
    assert excl <= K * T // 50                                                # the exclusion stays a rare edge case


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("case", [FREE_CASES[0], FREE_CASES[2], FREE_CASES[6], FREE_CASES[8]],
                         ids=[free_case_id(c) for c in (FREE_CASES[0], FREE_CASES[2], FREE_CASES[6], FREE_CASES[8])])
def test_large_yaw_lockstep(oracle, monkeypatch, synth_dir, case, mapping):
    """Every rollout at |yaw| in [20, 50] rad, in lock-step with the oracle from the same float32 state: the range reduction of the
    yaw target's sincos and the chassis quaternion's half angle.  One float32 ulp of yaw is up to 3.8e-6 there."""
    K, T = 128, 6
    sc, p, s0 = _robot(synth_dir, case, K=K, T=T)
    rng = np.random.default_rng(7 + sc.ndof)
    actions = rng.uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    state = planar_states(sc, s0, K, rng, big_yaw_every=1)
    assert (np.abs(state[2]) >= 20).all()
    w, excl = lockstep(oracle, monkeypatch, sc, p, mapping, actions, state, T)
    report("large-yaw", id=_id(free_case_id(case), mapping), excluded=excl, **w)
    assert w["dq"] <= 2e-6 and w["dqd"] <= 1e-4, w
    assert w["dyaw"] <= 1e-5 and w["quat"] <= 1e-5 and w["pos"] <= 2e-6, w   # a few ulps of yaw
    assert excl <= K * T // 50


# The saturation decision of a velocity drive is taken on the first solve of a substep and the saturated joints are re-solved once
# (oracle.cpp rollout_one).  When a joint sits at its limit while other joints saturate, taking the other decision changes its torque in
# the re-solve by a finite amount: the result jumps.  The planar base's virtual drives (gains ~1e5, friction-cone limits) reach that
# point often, and float32 may decide either way within ~1e-4 of the limit.  The effort probe finds those rollouts: the float64 oracle
# is run again with every effort limit scaled by 1 +- SAT_PROBE; a continuous result moves by ~SAT_PROBE * mu g h, a decision at its
# threshold jumps.
SAT_PROBE = 1e-3
# The kernels take spatial quantities about the world origin, so the float32 first solve loses precision with the base's distance from
# it: 28 m away (the far rollouts of the contact scenes) a decision is ambiguous within ~1 % of the limit (measured: the float64 oracle
# takes the kernels' branch between scales 1.001 and 1.01).  The contact tests look for decisions within SAT_BAND of the limits.
SAT_BAND = 1e-2


def _efforts_scaled(model, f):
    out = copy.deepcopy(model)
    for i in range(model.nb):
        out.effort[i] = model.effort[i] * f
    return out


def effort_probe(oracle, model, run):
    """max over the two probes of |run(probed model) - run(model)| per rollout: run(model) -> (NS, K) or (R, K) float64 result."""
    base = run(model)
    return np.max([np.abs(run(_efforts_scaled(model, f)) - base) for f in (1 + SAT_PROBE, 1 - SAT_PROBE)], axis=0)


@pytest.mark.parametrize("substeps", [1, 3])
@pytest.mark.parametrize("case,mapping", FREE_PARAMS)
def test_free_running(oracle, monkeypatch, synth_dir, case, mapping, substeps):
    """T = 12 steps from per-rollout states: the quantile gates of test_gpu_synth.FREE_GATES on q, qd, the chassis / arm / wheel rows
    and the DOF rows over every rollout; the loose bound on the worst rollout over the rollouts whose float64 result does not jump
    under the effort probe (a saturation decision at its threshold somewhere in the 12 steps, then amplified by the coupled base and
    arm)."""
    K, T = 256, 12
    sc, p, s0 = _robot(synth_dir, case, K=K, T=T, dt=0.03, substeps=substeps)
    be = backend(monkeypatch, sc, p, mapping)
    rng = np.random.default_rng(100 + sc.ndof)
    actions = rng.uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    actions[:, :, : K // 4] *= 0.05
    st0 = planar_states(sc, s0, K, rng)
    obs, state = torch.zeros((be.obs_size(), T, K), device=DEV), dev(st0)
    be.rollout(None, state, dev(actions), 0, T, obs)
    st_ref, obs_ref = oracle.rollout(sc.model, p, None, actions, state=st0.copy(), use_double=True, nthreads=8)
    o, s = obs.cpu().numpy(), state.cpu().numpy()
    assert np.isfinite(o).all() and np.isfinite(s).all()
    nb = sc.ndof
    sens = effort_probe(oracle, sc.model, lambda mm: oracle.rollout(mm, p, None, actions, state=st0.copy(), want_obs=False,
                                                                    use_double=True, nthreads=8)[0].astype(np.float64))
    jump = (sens[:nb].max(axis=0) > 100 * FREE_GATES["q"][1]) | (sens[nb:2 * nb].max(axis=0) > 100 * FREE_GATES["qd"][1])
    err = _compare_free_running(sc, o, s, obs_ref, st_ref)
    report("free", id=f"{_id(free_case_id(case), mapping)}-sub{substeps}", jumps=int(jump.sum()),
           **{f"{k}_med": float(np.median(v)) for k, v in err.items()},
           **{f"{k}_q97": float(np.quantile(v, 0.97)) for k, v in err.items()}, **{f"{k}_max": float(v[~jump].max()) for k, v in err.items()},
           **{f"{k}_max_at_jumps": float(v[jump].max()) if jump.any() else 0.0 for k, v in err.items() if k in ("q", "qd")})
    for k, (g_med, g_q97) in FREE_GATES.items():
        assert np.median(err[k]) <= g_med and np.quantile(err[k], 0.97) <= g_q97, (k, np.median(err[k]), np.quantile(err[k], 0.97))
        assert err[k][~jump].max() <= 100 * g_q97, (k, err[k][~jump].max())
    assert jump.sum() <= K // 4, int(jump.sum())         # a minority: up to 31 of 256 rollouts (the 16-body chain at 3 substeps)
    assert np.abs(s[0:2] - st0[0:2]).max() > 1e-2 and np.abs(s[2] - st0[2]).max() > 1e-2    # the base really drove and turned


# ---------------------------------------------------------------------------------------------------------------------------
# contacts
# ---------------------------------------------------------------------------------------------------------------------------
def _rows(sc):
    nb, nf = sc.ndof, sc.model.nfree
    pos = list(range(nb)) + [2 * nb + 13 * f + r for f in range(nf) for r in range(7)]
    vel = list(range(nb, 2 * nb)) + [2 * nb + 13 * f + r for f in range(nf) for r in range(7, 13)]
    return np.array(pos), np.array(vel)


def _errors(sc, s, o, s_ref, o_ref):
    """Per-rollout errors of one step: positions, velocities, observed chassis and free-body rows, contact forces (relative to
    max(1, |F|)).  Observation rows: chassis (13), DOF state (2 nb), free bodies (13 each), contact slots (3 each)."""
    nb, nf = sc.ndof, sc.model.nfree
    pos, vel = _rows(sc)
    b0 = 13 + 2 * nb
    f0 = b0 + 13 * nf
    F_ref = o_ref[f0:]
    scale = np.maximum(1.0, np.abs(F_ref).max(axis=0)) if len(F_ref) else 1.0
    qa, qb = o[3:7], o_ref[3:7]
    return {"pos": np.maximum(np.abs(s[pos] - s_ref[pos]).max(axis=0), np.abs(o[0:3] - o_ref[0:3]).max(axis=0),
                              np.minimum(np.abs(qa - qb), np.abs(qa + qb)).max(axis=0)),
            "vel": np.maximum(np.abs(s[vel] - s_ref[vel]).max(axis=0), np.abs(o[7:13] - o_ref[7:13]).max(axis=0)),
            "obs_free": np.abs(o[b0:f0] - o_ref[b0:f0]).max(axis=0) if nf else np.zeros(s.shape[1]),
            "force": (np.abs(o[f0:] - F_ref).max(axis=0) / scale) if len(F_ref) else np.zeros(s.shape[1])}


def thresholds(oracle, sc, p, m, actions, t, state, root0, gate, rng):
    """(at a contact threshold, at a saturation threshold) per rollout of step t: the float64 result moves by more than a gate when
    every position row moves by +-PROBE, or under the effort probe."""
    pos, _ = _rows(sc)
    K = state.shape[1]

    def ref(s, mm=m):
        return oracle.rollout(mm, p, None, actions, t, 1, state=s.copy(), root0=root0, use_double=True, nthreads=8)
    s_ref, o_ref = ref(state)
    at_contact, at_sat = np.zeros(K, bool), np.zeros(K, bool)
    for sign in (1.0, -1.0):
        d = np.zeros_like(state)
        d[pos] = sign * PROBE * rng.choice([-1.0, 1.0], (len(pos), K))
        s_p, o_p = ref(state + d)
        e = _errors(sc, s_p, o_p[:, t], s_ref, o_ref[:, t])
        for k in gate:
            at_contact |= e[k] > gate[k]
    # a decision at its threshold within SAT_BAND of the limits: the response to scaling them by 1 +- SAT_BAND is not SAT_BAND / SAT_PROBE
    # times the response to 1 +- SAT_PROBE (a continuous result is linear in the scale there, a flipped decision jumps)
    for sign in (1.0, -1.0):
        (s_b, o_b), (s_s, o_s) = (ref(state, _efforts_scaled(m, 1 + sign * eps)) for eps in (SAT_BAND, SAT_PROBE))
        r = SAT_BAND / SAT_PROBE
        e = _errors(sc, s_ref + (s_b - s_ref) - r * (s_s - s_ref), o_ref[:, t] + (o_b[:, t] - o_ref[:, t]) - r * (o_s[:, t] - o_ref[:, t]),
                    s_ref, o_ref[:, t])
        for k in gate:
            at_sat |= e[k] > gate[k]
    return s_ref, o_ref, at_contact, at_sat


# Open: with the base 20 - 28 m from the world origin (the far rollouts) and no free box or one, these five miss the 2e-3 velocity
# gate by up to 1.5x (2.0e-3 - 3.1e-3, thread kernel), and the 16-body chain by 14x (2.8e-2, both kernels), outside any threshold the
# probes find.  The kernels' spatial quantities about the world origin lose float32 precision with that distance; strict, so the
# marks have to go when that is fixed.
FAR_PRECISION = {"w2chain0-nfree0-thread", "w2chain0-nfree1-thread", "w2chain4-nfree0-thread", "w2chain8-nfree0-team_G16_NB16_NCS2",
                 "w2chain8-nfree0-thread"}
CONTACT_LOCKSTEP_PARAMS = [pytest.param(*prm.values, id=prm.id, marks=[pytest.mark.xfail(reason="float32 precision far from the world "
                           "origin (see FAR_PRECISION)", strict=True)] if prm.id in FAR_PRECISION else []) for prm in CONTACT_PARAMS]


@pytest.mark.parametrize("case,mapping", CONTACT_LOCKSTEP_PARAMS)
def test_contact_lockstep_against_float64_oracle(oracle, monkeypatch, synth_dir, case, mapping):
    """The gates of test_gpu_contact_synth.test_lockstep_against_float64_oracle on the planar contact scenes, with its +-2e-6 position
    probe that leaves out the rollout-steps at a contact threshold and the effort probe that leaves out those at a saturation
    threshold of a drive; both are counted, reported and bounded apart."""
    K, T = 128, 8
    sc, p, state, root0 = make_contact_case(synth_dir, case, K=K, T=T)
    m = sc.model
    be = backend(monkeypatch, sc, p, mapping, model=m)
    rng = np.random.default_rng(7)
    actions = rng.uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    a_d, root_d = dev(actions), dev(root0)
    gate = gates(sc)
    worst = {k: 0.0 for k in gate}
    n_contact = n_sat = excluded = contact_steps = 0
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    f0 = 13 + 2 * sc.ndof + 13 * m.nfree
    for t in range(T):
        st = dev(state)
        be.rollout(None, st, a_d, t, 1, obs, root0=root_d)
        s_ref, o_ref, at_contact, at_sat = thresholds(oracle, sc, p, m, actions, t, state, root0, gate, rng)
        near = at_contact | at_sat
        g, o = st.cpu().numpy(), obs[:, t].cpu().numpy()
        assert np.isfinite(g).all() and np.isfinite(o).all()
        err = _errors(sc, g, o, s_ref, o_ref[:, t])
        keep = ~near
        n_contact, n_sat, excluded = n_contact + int(at_contact.sum()), n_sat + int(at_sat.sum()), excluded + int(near.sum())
        contact_steps += int((np.abs(o_ref[f0:, t]).max(axis=0) > 0).sum())
        for k in gate:
            if keep.any():
                worst[k] = max(worst[k], float(err[k][keep].max()))
        state = s_ref
    report("contact-lockstep", id=_id(contact_case_id(case), mapping), at_contact_threshold=n_contact, at_saturation_threshold=n_sat,
           excluded=excluded, contact_frac=contact_steps / (K * T), **worst)
    # contact thresholds stay a rare edge case (up to 2.7 %: three free boxes pressed into the chassis); decisions within 1 % of a
    # drive limit are common on a planar base (2 - 9 % of the rollout-steps of these scenes, counted on the float64 oracle)
    assert n_contact <= 0.03 * K * T and n_sat <= 0.1 * K * T, (n_contact, n_sat)
    assert contact_steps >= (0.1 if m.nfree == 0 else 0.5) * K * T, contact_steps      # the case really is a contact case
    for k in gate:
        assert worst[k] <= gate[k], (k, worst[k])


# ---------------------------------------------------------------------------------------------------------------------------
# known answers on the device
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mapping", MAPPINGS)
def test_known_answers_on_device(monkeypatch, synth_dir, mapping):
    """test_oracle_planar.py's known answers on the device: from rest with a large v along world x the saturated x drive accelerates
    the base at exactly mu g while y stays 0; driven square-on into a wall the wall's net contact force converges to mu m_tot g along
    the normal with no vertical component."""
    dt = 0.01
    axis_angle = 0.9
    fwd = np.cross([math.cos(axis_angle), math.sin(axis_angle), 0.0], [0, 0, 1.0])
    psi0 = -math.atan2(fwd[1], fwd[0])
    sc, p, s0, kn = symmetric_base(synth_dir, axis_angle=axis_angle, yaw0=psi0, T=10, dt=dt, substeps=2)
    nb = sc.ndof
    be = backend(monkeypatch, sc, p, mapping)
    acts = np.zeros((p.T, sc.nu, p.K), np.float32)
    acts[:, 0] = 5.0
    obs, st = torch.zeros((be.obs_size(), p.T, p.K), device=DEV), torch.zeros((be.state_size(), p.K), device=DEV)
    be.rollout(dev(s0), st, dev(acts), 0, p.T, obs)
    o = obs.cpu().numpy()
    qd_x = o[39 + 1, :, 0].astype(np.float64)                                 # DOF rows after the three link rows: q0, qd0, q1, qd1
    y = o[39 + 2, :, 0].astype(np.float64)
    acc = np.diff(np.concatenate([[0.0], qd_x])) / dt
    err_acc = float(np.abs(acc / (kn["mu"] * G) - 1).max())
    assert err_acc <= 1e-4, acc                                               # float32 velocity differences (measured on an H100 below)
    assert np.abs(y).max() <= 1e-5
    # the wall
    sc, p, s0, kn = symmetric_base(synth_dir, axis_angle=np.pi / 2, yaw0=0.0, wall=True, T=100, dt=0.01, substeps=2)
    m, nb = sc.model, sc.ndof
    be = backend(monkeypatch, sc, p, mapping, model=m)
    acts = np.zeros((p.T, sc.nu, p.K), np.float32)
    acts[:, 0] = 1.0
    obs, st = torch.zeros((be.obs_size(), p.T, p.K), device=DEV), torch.zeros((be.state_size(), p.K), device=DEV)
    be.rollout(dev(s0), st, dev(acts), 0, p.T, obs, root0=dev(sc.root_state0))
    o = obs.cpu().numpy()
    x = o[13, :, 0].astype(np.float64)
    slot = sc.contact_slot[sc.body_offset[sc.actor_names.index("wall")]]
    F = o[13 + 2 * nb + 3 * slot: 13 + 2 * nb + 3 * slot + 3, :, 0].astype(np.float64)
    drive = kn["mu"] * kn["m_tot"] * G
    err_F = float(np.abs(F[0, -10:] / drive - 1).max())
    report("known", id=mapping, acc_rel=err_acc, wall_F_rel=err_F, Fz=float(np.abs(F[2]).max()),
           face=float(np.abs(x[-20:] + sc.layout["box"][2][0] - WALL_FACE).max()))
    assert np.abs(x[-20:] + sc.layout["box"][2][0] - WALL_FACE).max() <= m.contact_margin
    assert err_F <= 2e-3 and (F[2] == 0).all(), (F[:, -10:], drive)


# ---------------------------------------------------------------------------------------------------------------------------
# bookkeeping: ragged K, shards, team against thread
# ---------------------------------------------------------------------------------------------------------------------------
RAGGED = [("free", FREE_CASES[0]), ("free", FREE_CASES[4]), ("free", FREE_CASES[8]), ("contact", CONTACT_CASES[3]),
          ("contact", CONTACT_CASES[11]), ("contact", CONTACT_CASES[14])]


def _ragged_id(kind, case):
    return free_case_id(case) if kind == "free" else contact_case_id(case)


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("kind,case", RAGGED, ids=[_ragged_id(*r) for r in RAGGED])
def test_ragged_k(monkeypatch, synth_dir, kind, case, mapping):
    """K that leaves the last warp partly empty: every rollout below K is bit-identical to the same rollout of a launch with K rounded
    up to the rollouts per warp, every output below K is written and nothing past K is.  Broadcast state0, per-rollout state, and
    observe only."""
    T = 4
    if kind == "free":
        nb = 3 + case[0] + case[1]
        rpw = (32 // (8 if nb <= 8 else 16)) if mapping == "team" else 32
    else:
        rpw = 4 if mapping == "team" else 32
    n = 3
    Ks = sorted({1, max(1, rpw - 1), rpw * n + 1, rpw * n + rpw - 1}) if mapping == "team" else [31, 33]
    K_max = -(-Ks[-1] // rpw) * rpw
    if kind == "free":
        sc, p0, s0 = _robot(synth_dir, case, K=K_max, T=T, substeps=2, dt=0.03)
        states = planar_states(sc, s0, K_max, np.random.default_rng(3))
        root_d = None
    else:
        sc, p0, states, root0 = make_contact_case(synth_dir, case, K=K_max, T=T)
        s0 = states[:2 * sc.ndof, 0].copy()
        root_d = dev(root0)
    m = sc.model
    acts = np.random.default_rng(3).uniform(-0.5, 0.5, (T, sc.nu, K_max)).astype(np.float32)
    checked = 0
    for K in Ks:
        Kup = -(-K // rpw) * rpw
        assert Kup > K
        outs = {}
        for KK in (K, Kup):
            p = copy.copy(p0)
            p.K = KK
            be = backend(monkeypatch, sc, p, mapping, model=m)
            R, NS = be.obs_size(), be.state_size()
            a_d = dev(acts[:, :, :KK])
            res = {}
            for mode in ("state0", "state", "observe"):
                obuf, obs = _guarded(R * T * KK, float("nan"))
                if mode == "state0":
                    sbuf, st = _guarded(NS * KK, float("nan"))
                    be.rollout(dev(s0), st.view(NS, KK), a_d, 0, T, obs.view(R, T, KK), root0=root_d)
                else:
                    sbuf, st = _guarded(NS * KK, 0.0)
                    st.copy_(dev(states[:, :KK]).reshape(-1))
                    nsteps = T if mode == "state" else 0
                    be.rollout(None, st.view(NS, KK), a_d, 0 if nsteps else 2, nsteps, obs.view(R, T, KK), root0=root_d)
                torch.cuda.synchronize()
                assert bool((obuf[-GUARD:] == GUARD_VALUE).all()) and bool((sbuf[-GUARD:] == GUARD_VALUE).all()), (mode, K, KK)
                res[mode] = (obs.view(R, T, KK)[:, :, :K].cpu().numpy(), st.view(NS, KK)[:, :K].cpu().numpy())
            outs[KK] = res
        for mode in ("state0", "state", "observe"):
            (o, s), (o_up, s_up) = outs[K][mode], outs[Kup][mode]
            written = o if mode != "observe" else o[:, 2]
            assert not np.isnan(written).any() and not np.isnan(s).any(), (mode, K)
            if mode == "observe":
                assert np.isnan(np.delete(o, 2, axis=1)).all()
            np.testing.assert_array_equal(o, o_up, err_msg=f"{mode} K={K}")
            np.testing.assert_array_equal(s, s_up, err_msg=f"{mode} K={K}")
            checked += 1
    report("ragged", id=_id(_ragged_id(kind, case), mapping), Ks=",".join(map(str, Ks)), checked=checked)


SHARD = [c for c in CONTACT_CASES if c[3] >= 2 and c[5]]


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("case", SHARD, ids=[contact_case_id(c) for c in SHARD])
def test_shard_offset_with_randomised_free_boxes(monkeypatch, synth_dir, case, mapping):
    """A k_offset shard reproduces its slice of the whole launch bit for bit: the randomisation of every free box is keyed by the
    global sample index."""
    K, T, KS, off = 64, 4, 16, 24
    sc, p, st, root0 = make_contact_case(synth_dir, case, K=K, T=T)
    m = sc.model
    acts = np.random.default_rng(4).uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    be = backend(monkeypatch, sc, p, mapping, model=m)
    obs, s = torch.zeros((be.obs_size(), T, K), device=DEV), dev(st)
    be.rollout(None, s, dev(acts), 0, T, obs, root0=dev(root0))
    ps = copy.copy(p)
    ps.K, ps.k_offset = KS, off
    bs = backend(monkeypatch, sc, ps, mapping, model=m)
    obs_s, s_s = torch.zeros((bs.obs_size(), T, KS), device=DEV), dev(st[:, off:off + KS])
    bs.rollout(None, s_s, dev(acts[:, :, off:off + KS]), 0, T, obs_s, root0=dev(root0))
    assert torch.isfinite(obs).all()
    assert torch.equal(obs_s, obs[:, :, off:off + KS]) and torch.equal(s_s, s[:, off:off + KS])


CROSS_FAR_PRECISION = {"w2chain8-nfree0-team_G16_NB16_NCS2", "w2tree8-nfree1-team_G16_NB16_NCS3"}     # 16-body chains: see FAR_PRECISION
CROSS_PARAMS = [pytest.param(c, id=contact_case_id(c), marks=[pytest.mark.xfail(reason="float32 precision far from the world origin "
                "(see FAR_PRECISION)", strict=True)] if contact_case_id(c) in CROSS_FAR_PRECISION else []) for c in CONTACT_CASES]


@pytest.mark.parametrize("case", CROSS_PARAMS)
def test_mappings_agree_on_one_step(oracle, monkeypatch, synth_dir, case):
    """Team and thread-per-rollout kernels from the same per-rollout state, one model step, no oracle in between: the 0.98-quantile
    gates of test_gpu_contact_synth.test_mappings_agree_on_one_step over the rollouts that are at no contact or saturation threshold
    (the probes of the lock-step test; at a threshold the two float32 kernels may branch apart like either may from the oracle)."""
    K, T = 256, 2
    sc, p, st, root0 = make_contact_case(synth_dir, case, K=K, T=T)
    m = sc.model
    acts = dev(np.random.default_rng(5).uniform(-0.5, 0.5, (T, sc.nu, K)))
    out = {}
    for mapping in MAPPINGS:
        be = backend(monkeypatch, sc, p, mapping, model=m)
        s = dev(st)
        obs = torch.zeros((be.obs_size(), T, K), device=DEV)
        be.rollout(None, s, acts, 0, 1, obs, root0=dev(root0))
        out[mapping] = (s.cpu().numpy(), obs[:, 0].cpu().numpy())
    gate = gates(sc)
    _, _, at_contact, at_sat = thresholds(oracle, sc, p, m, acts.cpu().numpy(), 0, st, root0, gate, np.random.default_rng(6))
    keep = ~(at_contact | at_sat)
    err = {k: v[keep] for k, v in _errors(sc, out["team"][0], out["team"][1], out["thread"][0], out["thread"][1]).items()}
    q98 = {k: float(np.quantile(v, 0.98)) for k, v in err.items()}
    report("cross", id=contact_case_id(case), at_contact_threshold=int(at_contact.sum()), at_saturation_threshold=int(at_sat.sum()),
           **{f"{k}_med": float(np.median(v)) for k, v in err.items()}, **{f"{k}_q98": v for k, v in q98.items()})
    assert keep.sum() >= 0.85 * K, int(keep.sum())
    for k in gate:
        assert q98[k] <= gate[k], (k, q98[k])
    # measured on an H100 over the other cases (0.98 quantiles): positions 4.8e-5, velocities 3.2e-3, free rows 8e-5, forces 4.3e-4
    # relative -- far above the fixed-base suite's 6.7e-7 / 5.1e-5 because of the world-origin precision at 20 - 28 m (FAR_PRECISION)
    assert q98["pos"] <= 6e-5 and q98["vel"] <= 4e-3 and q98["obs_free"] <= 2e-4 and q98["force"] <= 1e-3, q98
