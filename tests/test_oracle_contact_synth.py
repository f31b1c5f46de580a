"""The oracle's contact path on generated scenes with several free bodies (synth_scenes.py), pinned by answers that do not come from
its code: conservation of momentum between colliding cubes, a stack settling on the ground, a box on a ramp, a link sphere driven into
a wall.  Plus the bookkeeping of several free actors (stepwise == batched, seeded / shard-invariant randomisation, float32 == float64
in lock-step), the binding contact cap, and the kernel each generated case is routed to."""
import copy
import math
import os

import numpy as np
import pytest

from synth_scenes import (CASES, G, case_id, contact_bodies, cube_collision_scene, make_case, make_contact_scene, ramp_scene,
                          resting_boxes_scene, slider_scene, stack_scene, team_template)

IDS = [case_id(c) for c in CASES]
# the substeps h = dt / substeps of the shipped configurations (conf/isaacgym/): normal.yaml 0.05 / 2, push.yaml 0.1 / 1; None = the
# scene's own step (h = 0.005 - 0.01).  The ground margin max(0.01, 1.5 g h^2) is 0.147 m at h = 0.1, and the soft constraint is
# nearly hard there (beta = 0.91, gamma = 9.1e-4).
SHIPPED = (((0.05, 2), "h0.025"), ((0.1, 1), "h0.1"))


def step_params(values):
    """pytest params (*value, step) for every value at the scene's own step (step None, the value's plain id) and at each shipped step
    (the id gets "-h0.025" / "-h0.1" appended)."""
    out = []
    for v in values:
        v = v if isinstance(v, tuple) else (v,)
        vid = "-".join(str(x) for x in v)
        out.append(pytest.param(*v, None, id=vid))
        out += [pytest.param(*v, step, id=f"{vid}-{sid}") for step, sid in SHIPPED]
    return out


def step_kw(step):
    return {} if step is None else dict(dt=step[0], substeps=step[1])


def stack_model(m, step):
    """At the shipped steps a stack runs with 32 Gauss-Seidel sweeps (a copy of the model).  The contact rows of a stack are coupled
    and, at gamma = 1 / (h (h kp + kd)) = 9.1e-4 (h = 0.1), nearly hard: 8 sweeps leave a residual every step.  With 8 sweeps the 2-box
    stack still carries its weights exactly but creeps 6 mm (h = 0.025) and 4.8 cm (h = 0.1) in 6 s, and the 3-box stack at h = 0.1
    jitters (net forces up to 3.7 % off the weights, 0.39 m/s on the middle box); with 32 sweeps every case is exact and at rest."""
    if step is None:
        return m
    m = copy.deepcopy(m)
    m.contact_iters = 32
    return m


def cube_kw(step):
    """Box pairs are found within the 1 cm contact margin, with no sweep between substeps: cubes sent at 1 - 3 m/s pass through one
    another at h = 0.1.  The speeds scale with 0.01 / h, so that every step moves them the 1 - 3 cm per substep they move at h = 0.01."""
    kw = step_kw(step)
    if kw:
        kw["speed"] = 0.01 / (kw["dt"] / kw["substeps"])
    return kw


@pytest.fixture(scope="module")
def synth_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("synth_contact")


def free_rows(obs, nfree):
    """(nfree, 13, T, K) free-body rows of an observation laid out as synth_scenes' known-answer scenes observe them."""
    return obs[:13 * nfree].reshape(nfree, 13, *obs.shape[1:])


def momenta(rows, mass, h):
    """Total linear momentum and angular momentum about the world origin of free cubes: rows (nfree, 13, ...) -> (3, ...), (3, ...)."""
    P = np.zeros(rows.shape[2:] + (3,))
    L = np.zeros_like(P)
    for f in range(rows.shape[0]):
        x, v, w = (np.moveaxis(rows[f, a:a + 3].astype(np.float64), 0, -1) for a in (0, 7, 10))
        P += mass[f] * v
        L += mass[f] * np.cross(x, v) + (2.0 / 3.0) * mass[f] * h[f] ** 2 * w          # cube: I = m (2 h)^2 / 6
    return P, L


def _initial_momenta(state, nb, mass, h):
    nf = len(mass)
    rows = state[2 * nb:].reshape(nf, 13, -1)
    return momenta(rows, mass, h)


@pytest.mark.parametrize("ncubes,step", step_params([2, 3, 4]))
def test_colliding_cubes_conserve_momentum(oracle, synth_dir, ncubes, step):
    """No gravity, no ground, no randomisation: the contact impulses are the only forces, applied equal and opposite at the same point,
    so the total linear momentum and the angular momentum about the origin stay what they were on every step; x += h v adds none."""
    sc, p, st, mass, h = cube_collision_scene(synth_dir, 0, ncubes, **cube_kw(step))
    T, K = p.T, p.K
    nb = sc.ndof
    _, obs = oracle.rollout(sc.model, p, None, np.zeros((T, sc.nu, K), np.float32), state=st.copy(), use_double=True)
    P0, L0 = _initial_momenta(st, nb, mass, h)
    rows = free_rows(obs, ncubes)
    P, L = momenta(rows, mass, h)                                               # (T, K, 3)
    dP = np.abs(P - P0[None]).max() / max(1.0, float(np.abs(P0).max()))
    dL = np.abs(L - L0[None]).max() / max(1.0, float(np.abs(L0).max()))
    assert dP <= 1e-6 and dL <= 1e-6, (dP, dL)             # the rows are reported in float32: measured 4e-8 / 7e-8 (relative)
    # the cubes really collided: their velocities changed by far more than round-off
    v0 = st[2 * nb:].reshape(ncubes, 13, K)[:, 7:10]
    assert np.abs(rows[:, 7:10, -1] - v0).max(axis=(0, 1)).min() > 0.1


@pytest.mark.parametrize("nboxes,step", step_params([2, 3]))
def test_stack_settles_with_each_box_carrying_its_weight(oracle, synth_dir, nboxes, step):
    """A stack on the ground: the net contact force on box i converges to its weight m_i g (the box below pushes up with the weight
    of everything above it, the box above pushes down with the weight of the rest) and the stack comes to rest.  A stack of n boxes
    takes 4 + 10 (n - 1) contact points (4 bottom corners on the ground; per pair, the 9 bottom-face sample points of the upper box
    and the top-face centre of the wider lower one), so 3 boxes fill the cap of 24 and a fourth would lose its support."""
    sc, p, st, mass = stack_scene(synth_dir, 0, nboxes, **step_kw(step))
    T, K = p.T, p.K
    m = sc.model = stack_model(sc.model, step)
    _, obs = oracle.rollout(m, p, None, np.zeros((T, sc.nu, K), np.float32), state=st.copy(), root0=sc.root_state0, use_double=True)
    rows = free_rows(obs, nboxes)
    base = 13 * nboxes
    for f in range(nboxes):
        s = m.free_slot[f]
        force = obs[base + 3 * s: base + 3 * s + 3, -5:]
        np.testing.assert_allclose(force[2], mass[f] * G, atol=2e-2 * max(1.0, mass[f] * G))
        np.testing.assert_allclose(force[0:2], 0, atol=2e-2)
        np.testing.assert_allclose(rows[f, 7:13, -1], 0, atol=2e-3)
        assert np.abs(rows[f, 0, -1] - 5.0).max() < 5e-3 and np.abs(rows[f, 1, -1]).max() < 5e-3     # no drift


@pytest.mark.parametrize("mu,step", step_params([0.8, 0.1]))
def test_box_on_a_rotated_ramp(oracle, synth_dir, mu, step):
    """A box on a static box tilted by 0.35 rad: with the average friction above tan(0.35) = 0.365 it stays; below, it slides down the
    slope with a = g (sin - mu cos).  About 0.5 s at every step (at least 8 steps), so the box stays on the ramp."""
    angle = 0.35
    kw = step_kw(step)
    if kw:
        kw["T"] = max(8, round(0.5 / kw["dt"]))
    sc, p, st = ramp_scene(synth_dir, angle, mu, mu, **kw)
    T, K = p.T, p.K
    _, obs = oracle.rollout(sc.model, p, None, np.zeros((T, sc.nu, K), np.float32), state=st.copy(), root0=sc.root_state0, use_double=True)
    v = obs[7:10, :, 0].astype(np.float64)                                      # (3, T)
    down = np.array([math.cos(angle), 0.0, -math.sin(angle)])                   # down the slope of a ramp tilted about +y
    speed = down @ v
    if mu > math.tan(angle):
        assert np.abs(v[:, 3:]).max() < 5e-3
    else:
        a = G * (math.sin(angle) - mu * math.cos(angle))
        dt = p.dt
        np.testing.assert_allclose(np.diff(speed[3:]) / dt, a, rtol=0.03)
        assert speed[-1] > 0.5 * a * T * dt


def test_link_sphere_stops_at_a_wall_and_holds_the_stall_force(oracle, synth_dir):
    """A one-joint prismatic robot drives its link sphere (r = 0.1) into a static box whose face is at x = 0.6: the sphere stops at the
    face plus its radius (within the contact margin) and the wall carries the velocity drive's stall force kd * target.  At rest the
    contact's soft constraint sits at its fixed point ln = bias / gamma, i.e. F = contact_kp * d: the sphere is F / kp deep."""
    _velocity_slider(oracle, synth_dir, None)


@pytest.mark.parametrize("step", [pytest.param(step, id=sid) for step, sid in SHIPPED])
def test_link_sphere_stops_at_a_wall_at_the_shipped_steps(oracle, synth_dir, step):
    """The velocity-drive slider of test_link_sphere_stops_at_a_wall_and_holds_the_stall_force at h = 0.025 and h = 0.1."""
    _velocity_slider(oracle, synth_dir, step)


def _velocity_slider(oracle, synth_dir, step):
    r, face, u = 0.1, 0.6, 0.4
    sc, p, s0 = slider_scene(synth_dir, r=r, face=face, **step_kw(step))
    T, K = p.T, p.K
    m = sc.model
    actions = np.full((T, 1, K), u, np.float32)
    _, obs = oracle.rollout(m, p, s0, actions, root0=sc.root_state0, use_double=True)
    q, qd = obs[0], obs[1]
    # the sphere-wall pair is found within the contact margin only, and a substep moves the sphere u h: it may enter that deep first
    h = p.dt / p.substeps
    assert q.max() <= face - r + max(m.contact_margin, u * h) and q[-1, 0] >= face - r - 5e-3
    assert np.abs(qd[-5:]).max() < 1e-2
    wall = sc.contact_slot[sc.body_offset[1]]
    fx = obs[2 + 3 * wall, -5:]
    np.testing.assert_allclose(fx, m.kd[0] * u, rtol=0.02)                      # 600 N/(m/s) * 0.4 m/s = 240 N into the wall
    np.testing.assert_allclose(q[-5:] - (face - r), m.kd[0] * u / m.contact_kp, rtol=0.02)     # 2.4 mm


@pytest.mark.parametrize("step", [pytest.param((0.02, 2), id="h0.01"), pytest.param((0.1, 1), id="h0.1")])
@pytest.mark.parametrize("u", [3.0, 8.0, -3.0])
def test_effort_drive_presses_a_link_sphere_into_a_wall(oracle, synth_dir, u, step):
    """The slider with a torque drive (dof_mode effort, drive damping kd = 10) and a URDF effort limit of 5 N, started 1 cm from the
    wall: at rest the damping term kd * qd is zero, so the wall carries clamp(u, +-5 N) -- 3 N below the limit, 5 N above it -- and the
    sphere sits F / contact_kp deep (the soft constraint's fixed point ln = bias / gamma).  Pulled away (u < 0) it leaves the wall."""
    r, face, effort = 0.1, 0.6, 5.0
    sc, p, s0 = slider_scene(synth_dir, r=r, face=face, effort=effort, T=60, dof_mode="effort", **step_kw(step))
    T, K = p.T, p.K
    m = sc.model
    assert m.drive_mode == 1 and float(m.kd[0]) == 10.0 and float(m.effort[0]) == effort
    s0[0] = face - r - 0.01
    actions = np.full((T, 1, K), u, np.float32)
    _, obs = oracle.rollout(m, p, s0, actions, root0=sc.root_state0, use_double=True)
    q, qd = obs[0], obs[1]
    wall = sc.contact_slot[sc.body_offset[1]]
    fx = obs[2 + 3 * wall, -5:]
    if u < 0:
        assert q[-1, 0] < face - r - 0.1 and np.abs(fx).max() == 0
        return
    F = min(u, effort)
    assert np.abs(qd[-5:]).max() < 1e-3
    np.testing.assert_allclose(fx, F, rtol=0.02)
    np.testing.assert_allclose(q[-5:] - (face - r), F / m.contact_kp, rtol=0.02)           # 30 / 50 um


@pytest.mark.parametrize("nboxes,cap", [(2, None), (3, None), (4, None), (3, 12)])
def test_resting_boxes_each_carry_their_weight_at_the_push_step(oracle, synth_dir, nboxes, cap):
    """n boxes 10 cm tall resting apart on the ground at h = 0.1 s (push.yaml), where the ground margin 1.5 g h^2 = 0.147 m puts all 8
    corners of each box within reach of the ground.  Only the 4 lowest corners are ground points, so the cap of 24 (or 12) carries
    floor(cap / 4) resting boxes; each box carries m g on its slot and none moves in 50 steps.  (With all 8 corners the cap carried
    floor(cap / 8): the 4th box -- the 2nd with cap 12 -- got no point and fell through the ground.)"""
    sc, p, st, mass = resting_boxes_scene(synth_dir, 0, nboxes, max_contacts=cap)
    T, K = p.T, p.K
    m = sc.model
    assert float(m.ground_margin) > 0.14 and m.max_contacts == (cap or 24)
    _, obs = oracle.rollout(m, p, None, np.zeros((T, sc.nu, K), np.float32), state=st.copy(), root0=sc.root_state0, use_double=True)
    rows = free_rows(obs, nboxes)
    base = 13 * nboxes
    x0 = st[2 * sc.ndof:].reshape(nboxes, 13, K)[:, :3]
    for f in range(nboxes):
        s = m.free_slot[f]
        force = obs[base + 3 * s: base + 3 * s + 3, -5:]
        np.testing.assert_allclose(force[2], mass[f] * G, rtol=2e-2, err_msg=f"box {f}")
        np.testing.assert_allclose(force[0:2], 0, atol=2e-2)
        np.testing.assert_allclose(rows[f, 7:13, -1], 0, atol=2e-3, err_msg=f"box {f}")
        np.testing.assert_allclose(rows[f, 0:3], x0[f][:, None, :].repeat(T, 1), atol=5e-3, err_msg=f"box {f}")     # no fall, no drift


def test_scenarios_keep_their_meaning_at_the_push_step(synth_dir):
    """At h = 0.1 s the generated starting states still mean what they say: a falling box has the clearance above the (14.7 cm) ground
    margin it has at h = 0.01 above the 1 cm one, and a far box is out of every margin: ground and every other shape."""
    case = (8, "tree", 4, 3, 1, 3, 1, True, None)
    out = {}
    for dt, sub in ((0.02, 2), (0.1, 1)):
        sc, p, st, root0 = make_case(synth_dir, case, K=40, T=1, dt=dt, substeps=sub)
        out[dt] = (sc, st)
    nb = 8
    (sc1, st1), (sc2, st2) = out[0.02], out[0.1]
    m1, m2 = sc1.model, sc2.model
    assert abs(float(m2.ground_margin) - 1.5 * 9.8 * 0.01) < 1e-6
    np.testing.assert_array_equal(st1[:2 * nb], st2[:2 * nb])
    for k in range(40):
        for f in range(4):
            r1, r2 = st1[2 * nb + 13 * f: 2 * nb + 13 * (f + 1), k], st2[2 * nb + 13 * f: 2 * nb + 13 * (f + 1), k]
            scen = k % 10
            if scen == 6:                                                       # falling
                assert r2[2] - r1[2] == pytest.approx(float(m2.ground_margin) - float(m1.ground_margin), abs=1e-6)
                np.testing.assert_array_equal(np.delete(r1, 2), np.delete(r2, 2))
            else:
                np.testing.assert_array_equal(r1, r2)
            if scen == 7:                                                       # far
                half = np.array(m2.free_half[f][:], float)
                lowest = r2[2] - np.linalg.norm(half)
                assert lowest > float(m2.ground_margin) + 1.0
                for g in range(4):
                    if g != f:
                        d = np.linalg.norm(r2[:3] - st2[2 * nb + 13 * g: 2 * nb + 13 * g + 3, k])
                        assert d > 2 * np.linalg.norm(half) + 0.01 + 0.5


def test_sixteen_body_contact_scene_is_refused(synth_dir):
    """With collision shapes a 16-body model leaves the thread kernel less than the 12 contact points build_scene requires, so the
    NB = 16 contact template is reached with 13 bodies (the case table) and a 16-body scene is refused, not silently truncated."""
    with pytest.raises(NotImplementedError, match="shared memory"):
        make_contact_scene(synth_dir, 0, 16, "deep", 1)


def test_case_table_covers_every_contact_team_template(synth_dir):
    """All 16 (NB, NCS) instantiations of the contact team kernel, computed from the built models, and the features the table claims:
    four free bodies, link spheres, rotated statics, more than 8 contact bodies, lowered caps."""
    seen = set()
    features = dict(nfree4=0, link_sphere=0, rotated=0, many_bodies=0, cap=0, noise=0, gravity_off=0)
    for c in CASES:
        sc, p, st, root0 = make_case(synth_dir, c, K=4, T=1)
        m = sc.model
        _, NB, ncs = team_template(m.nb, m.nfree)
        assert ncs == -(-(m.nb + 6 * m.nfree) // 8)
        seen.add((NB, ncs))
        features["nfree4"] += m.nfree == 4
        features["link_sphere"] += any(m.shape_type[s] == 1 and m.shape_owner_kind[s] == 1 for s in range(m.nshapes))
        features["rotated"] += any(m.shape_owner_kind[s] == 0 and abs(root0[m.shape_actor[s], 3:6]).max() > 0.1 for s in range(m.nshapes))
        features["many_bodies"] += contact_bodies(sc) > 8 and any(m.shape_slot[s] < 0 for s in range(m.nshapes))
        features["cap"] += m.max_contacts <= 8
        features["noise"] += any(m.free_mass_pct[f] > 0 for f in range(m.nfree))
        features["gravity_off"] += any(m.free_gravity[f] == 0 for f in range(m.nfree))
        assert m.nshapes <= 24 and m.max_contacts <= 24
    expect = {(4, 1), (4, 2), (4, 3), (4, 4), (8, 1), (8, 2), (8, 3), (8, 4), (12, 2), (12, 3), (12, 4), (12, 5), (16, 2), (16, 3), (16, 4), (16, 5)}
    assert seen == expect, expect - seen
    assert len(CASES) == len(set(IDS))
    assert features["many_bodies"] >= 3 and features["cap"] >= 3 and all(v >= 2 for v in features.values()), features


def _mapping(model, **env):
    import ctypes as C
    from mppi_isaac_b200 import backend
    lib = backend.load_library()
    old = {k: os.environ.get(k) for k in ("MPPIB_K2_LANES", "MPPIB_K2_TEAM")}
    try:
        for k in old:
            os.environ.pop(k, None)
        os.environ.update(env)
        return backend.CudaBackend.MAPPING_NAMES[lib.mppib_rollout_mapping_for_model(C.byref(model))].split("-")[0]
    finally:
        for k, v in old.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_case_routing(synth_dir, case):
    """Every contact case runs on the team kernel by default (chains too: contact scenes never take the lanes kernel) and on the
    thread-per-rollout kernel with MPPIB_K2_TEAM=0."""
    sc, _, _, _ = make_case(synth_dir, case, K=4, T=1)
    assert _mapping(sc.model) == "team"
    assert _mapping(sc.model, MPPIB_K2_TEAM="0") == "thread"


def _one_step(oracle, m, p, st, root0, **kw):
    s, o = oracle.rollout(m, p, None, np.zeros((p.T, m.nu, p.K), np.float32), 0, 1, state=st.copy(), root0=root0, use_double=True, **kw)
    return s, o[:, 0]


@pytest.mark.parametrize("case", [c for c in CASES if c[8] is not None], ids=[case_id(c) for c in CASES if c[8] is not None])
def test_lowered_cap_binds(oracle, synth_dir, case):
    """The cases that lower max_contacts to c really saturate it: one step at c differs from one step at c - 1 (the c-th point is kept
    and used), and raising the cap changes the result too (points past c were dropped)."""
    sc, p, st, root0 = make_case(synth_dir, case, K=40, T=1)
    m = sc.model
    c = m.max_contacts
    lower, higher = copy.deepcopy(m), copy.deepcopy(m)
    lower.max_contacts, higher.max_contacts = c - 1, 24
    s_c, _ = _one_step(oracle, m, p, st, root0)
    s_lo, _ = _one_step(oracle, lower, p, st, root0)
    s_hi, _ = _one_step(oracle, higher, p, st, root0)
    assert (np.abs(s_c - s_lo).max(axis=0) > 0).sum() >= 4
    assert (np.abs(s_c - s_hi).max(axis=0) > 0).sum() >= 4


BOOK = [c for c in CASES if c[2] >= 2]


@pytest.mark.parametrize("case", BOOK, ids=[case_id(c) for c in BOOK])
def test_bookkeeping_with_several_free_actors(oracle, synth_dir, case):
    """Stepwise == batched, the per-rollout randomisation is reproducible and keyed by the global sample index (a k_offset shard is
    its slice of the whole launch), and the float32 oracle follows the float64 one in lock-step."""
    K, T = 40, 4
    sc, p, st, root0 = make_case(synth_dir, case, K=K, T=T)
    m = sc.model
    acts = np.random.default_rng(1).uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    s_all, o_all = oracle.rollout(m, p, None, acts, state=st.copy(), root0=root0)
    s, o = st.copy(), np.zeros_like(o_all)
    for t in range(T):
        s, ot = oracle.rollout(m, p, None, acts, t, 1, state=s, root0=root0)
        o[:, t] = ot[:, t]
    np.testing.assert_array_equal(s, s_all)
    np.testing.assert_array_equal(o, o_all)
    s2, o2 = oracle.rollout(m, p, None, acts, state=st.copy(), root0=root0)
    np.testing.assert_array_equal(o2, o_all)
    ps = copy.copy(p)
    ps.K, ps.k_offset = 16, 24
    s3, o3 = oracle.rollout(m, ps, None, np.ascontiguousarray(acts[:, :, 24:40]), state=st[:, 24:40].copy(), root0=root0)
    np.testing.assert_array_equal(o3, o_all[:, :, 24:40])
    np.testing.assert_array_equal(s3, s_all[:, 24:40])
    # float32 against float64, one step at a time from the float64 state
    s64 = st.copy()
    nb = sc.ndof
    worst = 0.0
    for t in range(T):
        a, _ = oracle.rollout(m, p, None, acts, t, 1, state=s64.copy(), root0=root0, want_obs=False)
        s64, _ = oracle.rollout(m, p, None, acts, t, 1, state=s64, root0=root0, want_obs=False, use_double=True)
        pos = np.r_[0:nb, [2 * nb + 13 * f + r for f in range(m.nfree) for r in range(7)]]
        worst = max(worst, float(np.median(np.abs(a[pos] - s64[pos]).max(axis=0))))
    assert worst <= 1e-5, worst
