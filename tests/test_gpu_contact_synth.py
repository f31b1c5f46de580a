"""-m gpu: every contact instantiation of the rollout kernels on generated scenes with several free bodies (synth_scenes.py) against the
float64 oracle, on both contact mappings: team of lanes (the default; <G, NB, true, NCS, 8, COMPACT>, the test id names it) and thread
per rollout (MPPIB_K2_TEAM=0).

Contacts switch on margins, face choices and the contact cap, and float32 may take the other branch at a threshold: the lock-step
test runs the float64 oracle also from two copies of the state with every position row moved by +-2e-6 (more than float32 rounding
does) and leaves out the rollout-steps whose result moves by more than a gate under that probe (a threshold was crossed: no
float32 implementation can be held to the float64 branch there); it counts them and bounds them at 2 %.  Each test
prints its worst errors ("SYNTH-CONTACT ..." lines, visible with -s)."""
import copy

import numpy as np
import pytest
import torch

from mppi_isaac_b200.model.blob import OBS_CONTACT, OBS_DOF_STATE, OBS_FREE_STATE, OBS_WIDTH
from synth_scenes import CASES, G, case_id, cube_collision_scene, make_case, resting_boxes_scene, slider_scene, stack_scene
from test_gpu_synth import GUARD, GUARD_VALUE, _guarded, backend, dev
from test_oracle_contact_synth import _initial_momenta, cube_kw, free_rows, momenta, stack_model, step_kw, step_params

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MAPPINGS = ("team", "thread")


def _pid(c, mp):
    return f"{case_id(c)}-{mp}" if mp == "team" else f"{case_id(c).rsplit('-', 1)[0]}-thread"


PARAMS = [pytest.param(c, mp, id=_pid(c, mp)) for c in CASES for mp in MAPPINGS]
PROBE = 2e-6
# the shipped steps (conf/isaacgym/): push.yaml 0.1 / 1, normal.yaml 0.05 / 2, pick.yaml 0.04 / 2; None = the case's own 0.02 / 2
H01, H0025, H002 = (0.1, 1), (0.05, 2), (0.04, 2)
STEP_ID = {None: "", H01: "-h0.1", H0025: "-h0.025", H002: "-h0.02", (0.02, 2): "-h0.01"}
# one case per NB template (4, 8, 12, 16), each with free bodies
PER_NB = [c for c in CASES if c[:3] in ((4, "tree", 2), (8, "tree", 4), (12, "tree", 3), (13, "tree", 3))]
# Open, not run: at h = 0.1 the contact cases without free bodies (tree6, tree10, tree13) put 101 - 503 of 1 024 rollout-steps at a
# contact threshold (the +-2e-6 probe moves the float64 result by more than a gate), and tree8 with four free boxes 21 of 1 024 at
# h = 0.025, above the 2 % bound; the rollout-steps kept are within every gate (measured on an H100, both mappings).
OPEN_THRESHOLDS = {((6, "tree", 0), H01), ((10, "tree", 0), H01), ((13, "tree", 0), H01), ((8, "tree", 4), H0025)}
LOCK_PARAMS = ([pytest.param(c, mp, None, "velocity", id=_pid(c, mp)) for c in CASES for mp in MAPPINGS]
               + [pytest.param(c, mp, H01, "velocity", id=_pid(c, mp) + STEP_ID[H01]) for c in CASES for mp in MAPPINGS
                  if (c[:3], H01) not in OPEN_THRESHOLDS]
               + [pytest.param(c, mp, st, "velocity", id=_pid(c, mp) + STEP_ID[st]) for st in (H0025, H002) for c in PER_NB for mp in MAPPINGS
                  if (c[:3], st) not in OPEN_THRESHOLDS]
               + [pytest.param(c, mp, st, "effort", id=_pid(c, mp) + STEP_ID[st] + "-effort") for st in ((0.02, 2), H01) for c in PER_NB
                  for mp in MAPPINGS])


@pytest.fixture(scope="module")
def synth_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("synth_contact_gpu")


def report(test, **vals):
    print(f"SYNTH-CONTACT {test} " + " ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}" for k, v in vals.items()))


def _rows(sc):
    """State rows: positions (joint q, free x and quaternion) and velocities (joint qd, free v and w)."""
    nb, nf = sc.ndof, sc.model.nfree
    pos = list(range(nb)) + [2 * nb + 13 * f + r for f in range(nf) for r in range(7)]
    vel = list(range(nb, 2 * nb)) + [2 * nb + 13 * f + r for f in range(nf) for r in range(7, 13)]
    return np.array(pos), np.array(vel)


def _errors(sc, s, o, s_ref, o_ref):
    """Per-rollout errors of one step: positions, velocities, observed free-body rows, contact forces (relative to max(1, |F|))."""
    nb, nf = sc.ndof, sc.model.nfree
    pos, vel = _rows(sc)
    f0 = 2 * nb + 13 * nf
    F_ref = o_ref[f0:]
    scale = np.maximum(1.0, np.abs(F_ref).max(axis=0)) if len(F_ref) else 1.0
    return {"pos": np.abs(s[pos] - s_ref[pos]).max(axis=0), "vel": np.abs(s[vel] - s_ref[vel]).max(axis=0),
            "obs_free": np.abs(o[2 * nb:f0] - o_ref[2 * nb:f0]).max(axis=0) if nf else np.zeros(s.shape[1]),
            "force": (np.abs(o[f0:] - F_ref).max(axis=0) / scale) if len(F_ref) else np.zeros(s.shape[1])}


def gates(sc, h=None):
    """Stated gates of the contact path (test_gpu_parity.py): positions / quaternions 1e-4, velocities 2e-3 (5e-3 with several free
    bodies), net forces 5e-2 max(1, |F|); the observed free-body rows hold both positions and velocities.  One step moves a position
    by h times its velocity, so a velocity error within its gate moves the position by up to h times that gate; where that exceeds
    1e-4 it is the position gate (h = 0.1: 2e-4 / 5e-4; h = 0.025 with several free bodies: 1.25e-4; h <= 0.02: 1e-4)."""
    v = 5e-3 if sc.model.nfree >= 2 else 2e-3
    return {"pos": max(1e-4, (h or 0.0) * v), "vel": v, "obs_free": v, "force": 5e-2}


@pytest.mark.parametrize("case,mapping,step,dof_mode", LOCK_PARAMS)
def test_lockstep_against_float64_oracle(oracle, monkeypatch, synth_dir, case, mapping, step, dof_mode):
    """Lock-step at the case's own step (h = 0.01), at every shipped step (h = 0.1 on every case; 0.025 and 0.02 on one case per NB
    template) and with torque drives (dof_mode effort, drive damping 10: commands of up to 3 N / N m press the links into the statics)."""
    K, T = 128, 8
    sc, p, state, root0 = make_case(synth_dir, case, K=K, T=T, dof_mode=dof_mode, **step_kw(step))
    m = sc.model
    be = backend(monkeypatch, sc, p, mapping, model=m)
    rng = np.random.default_rng(7)
    amp = 3.0 if dof_mode == "effort" else 0.5
    actions = rng.uniform(-amp, amp, (T, sc.nu, K)).astype(np.float32)
    a_d, root_d = dev(actions), dev(root0)
    pos, _ = _rows(sc)
    gate = gates(sc, p.dt / p.substeps)
    worst = {k: 0.0 for k in gate}
    excluded = contact_steps = 0
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    f0 = 2 * sc.ndof + 13 * m.nfree
    for t in range(T):
        st = dev(state)
        be.rollout(None, st, a_d, t, 1, obs, root0=root_d)

        def ref(s):
            return oracle.rollout(m, p, None, actions, t, 1, state=s.copy(), root0=root0, use_double=True, nthreads=8)
        s_ref, o_ref = ref(state)
        sens = {k: np.zeros(K) for k in gate}
        for sign in (1.0, -1.0):
            d = np.zeros_like(state)
            d[pos] = sign * PROBE * rng.choice([-1.0, 1.0], (len(pos), K))
            s_p, o_p = ref(state + d)
            e = _errors(sc, s_p, o_p[:, t], s_ref, o_ref[:, t])
            sens = {k: np.maximum(sens[k], e[k]) for k in gate}
        near = np.zeros(K, bool)
        for k in gate:
            near |= sens[k] > gate[k]
        g, o = st.cpu().numpy(), obs[:, t].cpu().numpy()
        assert np.isfinite(g).all() and np.isfinite(o).all()
        err = _errors(sc, g, o, s_ref, o_ref[:, t])
        keep = ~near
        excluded += int(near.sum())
        contact_steps += int((np.abs(o_ref[f0:, t]).max(axis=0) > 0).sum()) if m.ncontact_slots else 0
        for k in gate:
            if keep.any():
                worst[k] = max(worst[k], float(err[k][keep].max()))
        state = s_ref
    report("lockstep", id=f"{_pid(case, mapping)}{STEP_ID[step]}{'-effort' if dof_mode == 'effort' else ''}", excluded=excluded,
           contact_frac=contact_steps / (K * T), **worst)
    assert excluded <= 0.02 * K * T, excluded                                  # discontinuities stay a rare edge case
    assert contact_steps >= 0.5 * K * T, contact_steps                        # the case really is a contact case
    for k in gate:
        assert worst[k] <= gate[k], (k, worst[k])
    # what float32 delivers on an H100 over every case and both mappings at h = 0.01: positions 1.5e-5, velocities 2.7e-3 (forest9,
    # two free bodies), forces 5.0e-3 relative; at most 13 of 1 024 rollout-steps excluded.  At h = 0.1: positions 3.6e-5, velocities
    # 6.0e-4, forces 1.2e-3, at most 5 excluded; h = 0.025 / 0.02: 3.3e-5, 1.0e-3, 4.7e-3, at most 18 excluded; effort drives (h = 0.01
    # and 0.1): 2.4e-4 (h = 0.1, gate 5e-4), 2.4e-3, 3.2e-3, at most 5 excluded
    if step is None:
        assert worst["pos"] <= 3e-5 and worst["force"] <= 1e-2, worst


@pytest.mark.parametrize("ncubes,mapping,step", step_params([(n, mp) for mp in MAPPINGS for n in (2, 3, 4)]))
def test_colliding_cubes_conserve_momentum_on_device(oracle, monkeypatch, synth_dir, ncubes, mapping, step):
    """The known answer of test_oracle_contact_synth.py on the device: free cubes without gravity or ground keep their total linear
    momentum and their angular momentum about the origin on every step."""
    sc, p, st, mass, h = cube_collision_scene(synth_dir, 0, ncubes, **cube_kw(step))
    T, K = p.T, p.K
    be = backend(monkeypatch, sc, p, mapping, model=sc.model)
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    be.rollout(None, dev(st), dev(np.zeros((T, sc.nu, K), np.float32)), 0, T, obs, root0=dev(sc.root_state0))
    rows = free_rows(obs.cpu().numpy(), ncubes)
    P0, L0 = _initial_momenta(st, sc.ndof, mass, h)
    P, L = momenta(rows, mass, h)
    dP = float(np.abs(P - P0[None]).max()) / max(1.0, float(np.abs(P0).max()))
    dL = float(np.abs(L - L0[None]).max()) / max(1.0, float(np.abs(L0).max()))
    report("momentum", id=f"cubes{ncubes}-{mapping}{STEP_ID[step]}", dP_rel=dP, dL_rel=dL)
    assert dP <= 5e-6 and dL <= 5e-6, (dP, dL)                             # float32: measured 1.0e-6 / 1.8e-6 on an H100
    v0 = st[2 * sc.ndof:].reshape(ncubes, 13, K)[:, 7:10]
    assert np.abs(rows[:, 7:10, -1] - v0).max(axis=(0, 1)).min() > 0.1


@pytest.mark.parametrize("nboxes,mapping,step", step_params([(n, mp) for mp in MAPPINGS for n in (2, 3)]))
def test_stack_settles_on_device(monkeypatch, synth_dir, nboxes, mapping, step):
    """The stack of test_oracle_contact_synth.py on the device: each box's net contact force converges to its weight, the stack rests
    (at the shipped steps with 32 Gauss-Seidel sweeps: test_oracle_contact_synth.stack_model)."""
    sc, p, st, mass = stack_scene(synth_dir, 0, nboxes, **step_kw(step))
    T, K = p.T, p.K
    m = sc.model = stack_model(sc.model, step)
    be = backend(monkeypatch, sc, p, mapping, model=m)
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    be.rollout(None, dev(st), dev(np.zeros((T, sc.nu, K), np.float32)), 0, T, obs, root0=dev(sc.root_state0))
    o = obs.cpu().numpy()
    rows = free_rows(o, nboxes)
    worst_f = worst_v = 0.0
    for f in range(nboxes):
        s = m.free_slot[f]
        force = o[13 * nboxes + 3 * s: 13 * nboxes + 3 * s + 3, -5:]
        worst_f = max(worst_f, float(np.abs(force[2] - mass[f] * G).max() / max(1.0, mass[f] * G)), float(np.abs(force[0:2]).max()))
        worst_v = max(worst_v, float(np.abs(rows[f, 7:13, -1]).max()))
    report("stack", id=f"stack{nboxes}-{mapping}{STEP_ID[step]}", dF=worst_f, v=worst_v)
    assert worst_f <= 2e-2 and worst_v <= 2e-3, (worst_f, worst_v)


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("nboxes,cap", [(2, None), (3, None), (4, None), (3, 12)])
def test_resting_boxes_carry_their_weight_at_the_push_step_on_device(monkeypatch, synth_dir, nboxes, cap, mapping):
    """test_oracle_contact_synth.test_resting_boxes_each_carry_their_weight_at_the_push_step on the device: at h = 0.1 only the 4 lowest
    corners of a box are ground points, so the cap of 24 (12) carries 6 (3) resting boxes; each carries m g and none moves."""
    sc, p, st, mass = resting_boxes_scene(synth_dir, 0, nboxes, max_contacts=cap)
    T, K = p.T, p.K
    m = sc.model
    be = backend(monkeypatch, sc, p, mapping, model=m)
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    be.rollout(None, dev(st), dev(np.zeros((T, sc.nu, K), np.float32)), 0, T, obs, root0=dev(sc.root_state0))
    o = obs.cpu().numpy()
    rows = free_rows(o, nboxes)
    x0 = st[2 * sc.ndof:].reshape(nboxes, 13, K)[:, :3]
    worst_f = worst_v = worst_x = 0.0
    for f in range(nboxes):
        s = m.free_slot[f]
        force = o[13 * nboxes + 3 * s: 13 * nboxes + 3 * s + 3, -5:]
        worst_f = max(worst_f, float(np.abs(force[2] - mass[f] * G).max() / (mass[f] * G)), float(np.abs(force[0:2]).max()))
        worst_v = max(worst_v, float(np.abs(rows[f, 7:13, -1]).max()))
        worst_x = max(worst_x, float(np.abs(rows[f, 0:3] - x0[f][:, None, :]).max()))
    report("resting", id=f"boxes{nboxes}-cap{cap or 24}-{mapping}", dF=worst_f, v=worst_v, dx=worst_x)
    assert worst_f <= 2e-2 and worst_v <= 2e-3 and worst_x <= 5e-3, (worst_f, worst_v, worst_x)


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("drive,u,step", [("velocity", 0.4, None), ("velocity", 0.4, H01), ("effort", 3.0, (0.02, 2)), ("effort", 8.0, (0.02, 2)),
                                          ("effort", 3.0, H01), ("effort", 8.0, H01)])
def test_link_sphere_pressed_into_a_wall_on_device(monkeypatch, synth_dir, drive, u, step, mapping):
    """The slider of test_oracle_contact_synth.py on the device: at rest the wall carries the drive's force -- kd u for the velocity
    drive, clamp(u, +-5 N) for the torque drive (its damping term is zero at rest) -- and the sphere sits F / contact_kp deep."""
    r, face = 0.1, 0.6
    if drive == "effort":
        sc, p, s0 = slider_scene(synth_dir, r=r, face=face, effort=5.0, T=60, dof_mode="effort", **step_kw(step))
        s0[0] = face - r - 0.01
        F = min(u, 5.0)
    else:
        sc, p, s0 = slider_scene(synth_dir, r=r, face=face, **step_kw(step))
        F = float(sc.model.kd[0]) * u
    T, K = p.T, p.K
    m = sc.model
    be = backend(monkeypatch, sc, p, mapping, model=m)
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    be.rollout(dev(s0), None, dev(np.full((T, 1, K), u, np.float32)), 0, T, obs, root0=dev(sc.root_state0))
    o = obs.cpu().numpy()
    wall = sc.contact_slot[sc.body_offset[1]]
    fx, q, qd = o[2 + 3 * wall, -5:], o[0, -5:], o[1, -5:]
    dF = float(np.abs(fx - F).max() / F)
    dd = float(np.abs((q - (face - r)) - F / m.contact_kp).max() / (F / m.contact_kp))
    report("slider", id=f"{drive}-u{u}-{mapping}{STEP_ID[step]}", dF=dF, depth=dd, qd=float(np.abs(qd).max()))
    assert dF <= 2e-2 and dd <= 2e-2 and np.abs(qd).max() < 1e-2, (dF, dd)


def _exact_rows(p, nb):
    """Observation rows that a stepwise launch must reproduce bit for bit (free bodies, contact forces) -- the link and DOF rows come
    from the kinematics pass, which a batched launch shares with the next step's sweep and a single step runs on its own (float32
    contraction order: test_gpu_parity.test_k2_stepwise_equals_batched_and_observe_only) -- and the contact rows."""
    exact, contact, r = [], [], 0
    for i in range(p.nobs):
        kind = p.obs[i].kind
        w = 2 * nb if kind == OBS_DOF_STATE else OBS_WIDTH[kind]
        if kind in (OBS_FREE_STATE, OBS_CONTACT):
            exact += range(r, r + w)
        if kind == OBS_CONTACT:
            contact += range(r, r + w)
        r += w
    return np.array(exact, int), np.array(contact, int)


def _stepwise_scene(synth_dir, kind):
    from synth_planar import CONTACT_CASES, make_contact_case
    from synth_robots import make_robot
    K, T = 64, 6
    if kind.startswith("tree"):                                                # contact-free: team <8, 8> and <16, 12>
        nb = int(kind[4:])
        sc, p, s0 = make_robot(synth_dir, 0, nb, "tree", K=K, T=T)
        st = np.repeat(s0[:, None], K, 1) + np.random.default_rng(nb).uniform(-0.05, 0.05, (2 * nb, K)).astype(np.float32)
        return sc, p, st, None
    if kind == "planar":
        return make_contact_case(synth_dir, CONTACT_CASES[11], K=K, T=T)      # 4 wheels, a 5-joint tree, 4 randomised free boxes
    if kind == "effort":
        return make_case(synth_dir, PER_NB[1], K=K, T=T, dof_mode="effort")
    return make_case(synth_dir, {"random2": CASES[1], "random4": CASES[11]}[kind], K=K, T=T)


# Open: on the thread-per-rollout kernel the T one-step launches of a contact scene do not reproduce the T-step launch's state bit
# for bit (the four contact kinds below; measured on an H100); the contact-free trees do, and the team kernel does on every kind.
STEPWISE = [pytest.param(k, mp, id=f"{k}-{mp}") for k in ("tree6", "tree12", "random2", "random4", "planar", "effort") for mp in MAPPINGS
            if mp == "team" or k.startswith("tree")]


@pytest.mark.parametrize("kind,mapping", STEPWISE)
def test_stepwise_equals_batched_and_observe_only(monkeypatch, synth_dir, kind, mapping):
    """The launch protocol of the planner's stepwise path (planner/mppi.py: taken whenever a prior is configured) on the team and
    thread kernels: T one-step launches (actions[t:t+1], act_t0 = t) give the state of one T-step launch bit for bit, and the free-body
    and contact-force rows too; link and DOF rows agree to 2e-6.  An observe-only launch (nsteps = 0) writes its own slot only, with
    zero contact forces.  Contact-free trees on both team G, two randomised contact cases with free bodies, a planar contact case and
    an effort-drive contact case."""
    sc, p, st0, root0 = _stepwise_scene(synth_dir, kind)
    T, K = p.T, p.K
    m = sc.model
    be = backend(monkeypatch, sc, p, mapping, model=m)
    amp = 3.0 if kind == "effort" else 0.5
    acts = dev(np.random.default_rng(6).uniform(-amp, amp, (T, sc.nu, K)).astype(np.float32))
    root_d = dev(root0) if root0 is not None else None
    R = be.obs_size()
    obs_a, obs_b = torch.zeros((R, T, K), device=DEV), torch.zeros((R, T, K), device=DEV)
    st_a, st_b = dev(st0), dev(st0)
    be.rollout(None, st_a, acts, 0, T, obs_a, root0=root_d)
    for t in range(T):
        be.rollout(None, st_b, acts[t:t + 1], t, 1, obs_b, act_t0=t, root0=root_d)
    exact, contact = _exact_rows(p, sc.ndof)
    other = np.setdiff1d(np.arange(R), exact)
    assert torch.isfinite(obs_a).all() and torch.equal(st_a, st_b)
    a, b = obs_a.cpu().numpy(), obs_b.cpu().numpy()
    np.testing.assert_array_equal(a[exact], b[exact])
    d_other = float(np.abs(a[other] - b[other]).max()) if len(other) else 0.0
    if len(contact):
        assert np.abs(a[contact]).max() > 0                                    # forces were there to compare
    obs_c = torch.full((R, T, K), float("nan"), device=DEV)
    be.rollout(None, st_b, acts, T - 1, 0, obs_c, root0=root_d)                # observe-only into slot T - 1: the state after step T - 1
    c = obs_c.cpu().numpy()
    assert np.isnan(c[:, :T - 1]).all()
    noncontact = np.setdiff1d(np.arange(R), contact)
    np.testing.assert_array_equal(c[contact, T - 1], 0.0)
    d_obs = float(np.abs(c[noncontact, T - 1] - b[noncontact, T - 1]).max())
    report("stepwise", id=f"{kind}-{mapping}", rows_other=d_other, observe_only=d_obs)
    assert d_other <= 2e-6 and d_obs <= 2e-6, (d_other, d_obs)


RAGGED = [c for c in CASES if c[:3] in ((3, "chain", 3), (8, "tree", 4), (9, "forest", 2), (13, "tree", 4))]


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("case", RAGGED, ids=[case_id(c) for c in RAGGED])
def test_ragged_k(monkeypatch, synth_dir, case, mapping):
    """K that leaves the last warp partly empty (4 rollouts per warp in the team kernel's contact phase, 32 in the thread kernel):
    every rollout below K is bit-identical to the same rollout of a launch with K rounded up, every output below K is written and
    nothing past K is.  Broadcast state0, per-rollout state, and observe only."""
    rpw = 4 if mapping == "team" else 32
    Ks = [1, 3, 4 * 3 + 1, 4 * 3 + 3] if mapping == "team" else [31, 33]
    K_max = -(-Ks[-1] // rpw) * rpw
    T = 4
    sc, p0, states, root0 = make_case(synth_dir, case, K=K_max, T=T)
    m = sc.model
    nb = sc.ndof
    s0 = states[:2 * nb, 0].copy()
    acts = np.random.default_rng(3).uniform(-0.5, 0.5, (T, sc.nu, K_max)).astype(np.float32)
    root_d = dev(root0)
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
                    n = T if mode == "state" else 0
                    be.rollout(None, st.view(NS, KK), a_d, 0 if n else 2, n, obs.view(R, T, KK), root0=root_d)
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
    report("ragged", id=f"{case_id(case)}-{mapping}", Ks=",".join(map(str, Ks)), checked=checked)


SHARD = [c for c in CASES if c[2] >= 2 and c[7]]


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("case", SHARD, ids=[case_id(c) for c in SHARD])
def test_shard_offset_with_several_randomised_free_actors(monkeypatch, synth_dir, case, mapping):
    """A k_offset shard reproduces its slice of the whole launch bit for bit: the size / mass / friction draws of every free actor are
    keyed by the global sample index."""
    K, T, KS, off = 64, 4, 16, 24
    sc, p, st, root0 = make_case(synth_dir, case, K=K, T=T)
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


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_mappings_agree_on_one_step(monkeypatch, synth_dir, case):
    """Team and thread-per-rollout kernels from the same per-rollout state, one model step, no oracle in between: float32 rounding
    apart, except at the rare contact thresholds (at most 2 % of the rollouts)."""
    K, T = 256, 2
    sc, p, st, root0 = make_case(synth_dir, case, K=K, T=T)
    m = sc.model
    acts = dev(np.random.default_rng(5).uniform(-0.5, 0.5, (T, sc.nu, K)))
    out = {}
    for mapping in MAPPINGS:
        be = backend(monkeypatch, sc, p, mapping, model=m)
        s = dev(st)
        obs = torch.zeros((be.obs_size(), T, K), device=DEV)
        be.rollout(None, s, acts, 0, 1, obs, root0=dev(root0))
        out[mapping] = (s.cpu().numpy(), obs[:, 0].cpu().numpy())
    err = _errors(sc, out["team"][0], out["team"][1], out["thread"][0], out["thread"][1])
    gate = gates(sc)
    q98 = {k: float(np.quantile(v, 0.98)) for k, v in err.items()}
    report("cross", id=case_id(case), **{f"{k}_med": float(np.median(v)) for k, v in err.items()}, **{f"{k}_q98": v for k, v in q98.items()})
    for k in gate:
        assert q98[k] <= gate[k], (k, q98[k])
    # measured on an H100 (0.98 quantiles over every case): positions 6.7e-7, velocities 5.1e-5, forces 9.7e-5 relative
    assert q98["pos"] <= 2e-6 and q98["vel"] <= 2e-4 and q98["obs_free"] <= 2e-4 and q98["force"] <= 5e-4, q98
