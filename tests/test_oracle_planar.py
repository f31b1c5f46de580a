"""The oracle's planar differential-drive base (DESIGN.md section 2, "Differential-drive bases") on generated robots (synth_planar.py),
pinned by code it shares nothing with: the Lagrangian dynamics of lagrange_ref.py with the planar targets of joints 0-2 recomputed
from the current yaw and their friction-cone effort limits, host forward kinematics with the virtual joints, and known answers on a
symmetric wheel-only base.  Plus the kernel each generated planar model is routed to and the contact templates it reaches."""
import math

import numpy as np
import pytest
import torch

from lagrange_ref import forward_dynamics, mass_matrix_and_potential
from mppi_isaac_b200.model.urdf import forward_kinematics
from synth_planar import (CONTACT_CASES, FREE_CASES, G, WALL_FACE, contact_case_id, free_case_id, make_contact_case, make_planar_contact_scene,
                          make_planar_robot, planar_targets, rot_z, symmetric_base, template, wheel_dofs, yaw_quat)
from synth_robots import is_chain
from test_oracle_synth import _mapping


@pytest.fixture(scope="module")
def synth_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("synth_planar")


def _qdd_reference(sc, p, q, qd, u, h):
    """Lagrangian qdd of one substep: velocity drives towards the planar targets (joints 0-2, from the current yaw) and the
    command-map targets (wheels, arm), the friction-cone limits of joints 0-2, the saturation re-solve.  Returns (qdd, saturated
    mask)."""
    m, nb = sc.model, sc.ndof
    kd, b = np.array(m.kd[:nb], np.float64), np.array(m.damping[:nb], np.float64)
    eff = np.array(m.effort[:nb], np.float64)
    tgt = planar_targets(sc, p, q[:, None], u[:, None])[:, 0]
    grav = tuple(np.array(m.gravity[:], np.float64)) if m.gravity_on else (0.0, 0.0, 0.0)
    tau, dimp = kd * (tgt - qd) - b * qd, h * (kd + b)
    qdd, _ = forward_dynamics(sc.robot, q, qd, tau, dimp, grav)
    td = kd * (tgt - (qd + h * qdd.numpy()))
    sat = np.abs(td) > eff
    if sat.any():
        tau = np.where(sat, np.sign(td) * eff - b * qd, tau)
        dimp = np.where(sat, h * b, dimp)
        qdd, _ = forward_dynamics(sc.robot, q, qd, tau, dimp, grav)
    return qdd.numpy(), sat


LAGRANGE = [(2, 0, "chain"), (2, 4, "chain"), (4, 5, "tree"), (2, 11, "tree")]     # 5, 9, 12 and 16 bodies


@pytest.mark.parametrize("case", LAGRANGE, ids=[free_case_id(c) for c in LAGRANGE])
def test_oracle_qdd_matches_lagrangian(oracle, synth_dir, case):
    """One substep of the float64 oracle (qdd = (qd_new - qd) / h) against the Lagrangian, both saturated and unsaturated virtual
    drives: a base moving near its targets needs less than the friction cone, a base far from them saturates it."""
    nw, narm, topo = case
    h = 1e-3
    sc, p, _ = make_planar_robot(synth_dir, 0, narm, topo, nwheels=nw, K=2, T=1, dt=h, substeps=1)
    m, nb = sc.model, sc.ndof
    rng = np.random.default_rng(nb)
    counts = {"sat": 0, "unsat": 0}
    for trial in range(6):
        q = np.zeros(nb)
        q[0:2] = rng.uniform(-2.0, 2.0, 2)
        q[2] = rng.uniform(-np.pi, np.pi) + (40.0 if trial == 5 else 0.0)
        for i in range(3, nb):
            q[i] = rng.uniform(max(m.q_lo[i], -2.0) + 0.05, min(m.q_hi[i], 2.0) - 0.05) if m.q_hi[i] < 1e29 else rng.uniform(-np.pi, np.pi)
        q = q.astype(np.float32).astype(np.float64)
        u = rng.uniform(-0.5, 0.5, sc.nu)
        if trial % 2 == 0:
            u[2:] *= 0.02                                     # a quiet arm: the base's own drives decide
        u = u.astype(np.float32).astype(np.float64)
        qd = rng.uniform(-0.8, 0.8, nb)
        if trial % 2 == 0:                                    # the base within 2e-4 of its targets: unsaturated virtual drives
            qd[0:3] = planar_targets(sc, p, q[:, None], u[:, None])[0:3, 0] + rng.uniform(-2e-4, 2e-4, 3)
            qd[3:] *= 0.05
        qd = qd.astype(np.float32).astype(np.float64)
        qdd_ref, sat = _qdd_reference(sc, p, q, qd, u, h)
        counts["sat"] += int(sat[:3].sum())
        counts["unsat"] += int((~sat[:3]).sum())
        actions = np.repeat(u.astype(np.float32)[None, :, None], 2, axis=2)
        st, _ = oracle.rollout(m, p, np.concatenate([q, qd]).astype(np.float32), actions, 0, 1, want_obs=False, use_double=True)
        qdd = (st[nb:2 * nb, 0].astype(np.float64) - qd) / h
        np.testing.assert_allclose(qdd, qdd_ref, rtol=2e-4, atol=2e-3, err_msg=f"trial {trial}")
    print(f"SYNTH-PLANAR lagrange id={free_case_id(case)} saturated_virtual={counts['sat']} unsaturated_virtual={counts['unsat']}")
    assert counts["sat"] > 0 and counts["unsat"] > 0, counts


FK = [(1, 0, "chain"), (4, 1, "chain"), (2, 7, "tree"), (2, 11, "tree")]


@pytest.mark.parametrize("case", FK, ids=[free_case_id(c) for c in FK])
def test_oracle_rows_match_forward_kinematics(oracle, synth_dir, case):
    """Every observed row (chassis, arm link or mount, wheel) at every step == host FK of the observed q, virtual joints included; the
    chassis row is (x, y, z0, quat(yaw)) with linear velocity (xd, yd, 0) and angular velocity (0, 0, yawd)."""
    nw, narm, topo = case
    K, T = 8, 6
    sc, p, s0 = make_planar_robot(synth_dir, 1, narm, topo, nwheels=nw, K=K, T=T)
    m, nb = sc.model, sc.ndof
    actions = np.random.default_rng(nb).uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    _, obs = oracle.rollout(m, p, s0, actions, use_double=True)
    base_pos, base_quat = np.array(m.base_pos[:], np.float64), np.array(m.base_quat[:], np.float64)
    links = [p.obs[j].index for j in range(3)]
    assert sc.robot.link_names[links[0]] == "base" and m.link_body[links[0]] == 2
    for t in range(T):
        for k in range(K):
            q = obs[39::2, t, k][:nb].astype(np.float64)
            qd = obs[40::2, t, k][:nb].astype(np.float64)
            pos, quat = forward_kinematics(sc.robot, q, base_pos, base_quat)
            for j, l in enumerate(links):
                row = obs[13 * j:13 * j + 13, t, k].astype(np.float64)
                np.testing.assert_allclose(row[0:3], pos[l], atol=4e-6, rtol=0)
                qa, qb = row[3:7], quat[l]
                assert min(np.abs(qa - qb).max(), np.abs(qa + qb).max()) <= 2e-6
            c = obs[0:13, t, k].astype(np.float64)
            np.testing.assert_allclose(c[0:3], [q[0], q[1], base_pos[2]], atol=1e-6, rtol=0)
            qy = yaw_quat(q[2])
            assert min(np.abs(c[3:7] - qy).max(), np.abs(c[3:7] + qy).max()) <= 2e-6
            np.testing.assert_allclose(c[7:13], [qd[0], qd[1], 0.0, 0.0, 0.0, qd[2]], atol=2e-6, rtol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------------
# known answers on the symmetric wheel-only base
# ---------------------------------------------------------------------------------------------------------------------------
def _run(oracle, sc, p, s0, v, w, T=None):
    """Constant command (v, w) for T steps from s0 in float64: (q (T, nb), qd (T, nb)) after every step."""
    T = p.T if T is None else T
    nb = sc.ndof
    acts = np.zeros((p.T, sc.nu, p.K), np.float32)
    acts[:, 0], acts[:, 1] = v, w
    _, obs = oracle.rollout(sc.model, p, s0, acts, use_double=True)
    off = 13 * sum(1 for o in range(p.nobs) if p.obs[o].kind == 0)
    q, qd = obs[off:off + 2 * nb:2, :T, 0].T.astype(np.float64), obs[off + 1:off + 2 * nb:2, :T, 0].T.astype(np.float64)
    return q, qd


def _heading(sc, psi):
    return rot_z(psi) @ sc.layout["fwd"]


def test_known_answer_straight_and_turn_in_place(oracle, synth_dir):
    """(v, 0) from yaw psi0: the base settles at v R(psi0) fwd with no lateral velocity, yaw unmoved.  (0, w): x, y fixed, yaw rate w.  The
    wheels reach v / r -+ w L / (2 r) (left -, right +): the command map through the oracle, not arithmetic alone."""
    sc, p, s0, kn = symmetric_base(synth_dir, axis_angle=0.7, yaw0=2.1, T=60)
    psi0 = 2.1
    left, right = wheel_dofs(sc)
    d = _heading(sc, psi0)
    v = 0.4
    q, qd = _run(oracle, sc, p, s0, v, 0.0)
    lateral = -qd[-10:, 0] * d[1] + qd[-10:, 1] * d[0]                      # steady state (x and y saturate separately on the way)
    assert np.abs(qd[-10:, 0:2] - v * d[:2]).max() <= 1e-6 * v
    assert np.abs(lateral).max() <= 4 * np.spacing(np.float32(v)), np.abs(lateral).max()     # float32 rounding of the stored state
    assert np.abs(q[:, 2] - psi0).max() <= 1e-7 and np.abs(qd[:, 2]).max() <= 1e-9
    np.testing.assert_allclose(qd[-1, left + right], v / kn["r"], rtol=1e-5)
    w = 0.9
    q, qd = _run(oracle, sc, p, s0, 0.0, w)
    assert np.abs(q[:, 0:2] - s0[0:2]).max() <= 1e-9 and np.abs(qd[:, 0:2]).max() <= 1e-9
    assert abs(qd[-1, 2] - w) <= 1e-6 * w
    np.testing.assert_allclose(qd[-1, left], -w * kn["L"] / (2 * kn["r"]), rtol=1e-5)
    np.testing.assert_allclose(qd[-1, right], w * kn["L"] / (2 * kn["r"]), rtol=1e-5)
    v, w = 0.3, -0.7
    q, qd = _run(oracle, sc, p, s0, v, w)
    np.testing.assert_allclose(qd[-1, left], v / kn["r"] - w * kn["L"] / (2 * kn["r"]), rtol=1e-5)
    np.testing.assert_allclose(qd[-1, right], v / kn["r"] + w * kn["L"] / (2 * kn["r"]), rtol=1e-5)


def test_known_answer_circle(oracle, synth_dir):
    """Constant (v, w) from the steady motion: the path is a circle of radius |v / w| about p0 + (v / w) z x heading, to O(h)."""
    dt = 0.005
    v, w = 0.4, 1.3
    T = int(round(2 * np.pi / w / dt)) + 1
    sc, p, s0, kn = symmetric_base(synth_dir, axis_angle=-1.1, yaw0=0.4, T=T, dt=dt, substeps=1)
    left, right = wheel_dofs(sc)
    d = _heading(sc, 0.4)
    s0 = s0.copy()
    nb = sc.ndof
    s0[nb:nb + 2], s0[nb + 2] = v * d[:2], w
    s0[nb + np.array(left)] = v / kn["r"] - w * kn["L"] / (2 * kn["r"])
    s0[nb + np.array(right)] = v / kn["r"] + w * kn["L"] / (2 * kn["r"])
    q, qd = _run(oracle, sc, p, s0, v, w)
    R = v / w
    c = s0[0:2] + R * np.array([-d[1], d[0]])
    rad = np.linalg.norm(q[:, 0:2] - c, axis=1)
    err = float(np.abs(rad - abs(R)).max())
    print(f"SYNTH-PLANAR circle R={R:.4g} h={dt} radius_err={err:.3g} yaw_rate_err={np.abs(qd[:, 2] - w).max():.3g}")
    assert err <= 2 * v * dt, err                                           # O(h): the drive lags its turning target by ~ one substep
    assert np.abs(qd[:, 2] - w).max() <= 1e-6
    assert abs(q[-1, 2] - q[0, 2] - 2 * np.pi) <= 2 * w * dt                # one turn
    assert np.linalg.norm(q[-1, 0:2] - s0[0:2]) <= 4 * v * dt               # the path closes


@pytest.mark.parametrize("heading", ["x", "diagonal"])
def test_known_answer_friction_cone_acceleration(oracle, synth_dir, heading):
    """From rest with a large v: while a virtual joint's drive is saturated its acceleration is exactly mu g (the saturated joint's
    implicit damping is h b = 0).  The limit is per virtual joint -- a box, not a cone: heading along world x only x accelerates (y
    stays 0); on the diagonal x and y both accelerate at mu g, so the speed grows at sqrt(2) mu g.  Under a large w the yaw
    accelerates at mu m g (L / 2) / I_zz."""
    dt = 0.01
    axis_angle = 0.9
    fwd = np.cross([math.cos(axis_angle), math.sin(axis_angle), 0.0], [0, 0, 1.0])
    target = 0.0 if heading == "x" else np.pi / 4
    psi0 = target - math.atan2(fwd[1], fwd[0])
    sc, p, s0, kn = symmetric_base(synth_dir, axis_angle=axis_angle, yaw0=psi0, T=20, dt=dt, substeps=2)
    a_ref = kn["mu"] * G
    d = _heading(sc, psi0)
    np.testing.assert_allclose(d[:2], [math.cos(target), math.sin(target)], atol=1e-12)
    q, qd = _run(oracle, sc, p, s0, 5.0, 0.0)
    n = 10                                                                   # 0.1 s: far from 5 m/s, saturated throughout
    acc = np.diff(np.concatenate([s0[None, sc.ndof:sc.ndof + 2], qd[:n, 0:2]]), axis=0) / dt
    if heading == "x":
        np.testing.assert_allclose(acc[:, 0], a_ref, rtol=2e-6)
        tiny = 4 * 5.0 * np.finfo(np.float32).eps                            # v times the float32 rounding of fwd_axis
        assert np.abs(q[:n, 1]).max() <= tiny and np.abs(qd[:n, 1]).max() <= tiny
    else:
        np.testing.assert_allclose(acc, a_ref, rtol=2e-6)
        np.testing.assert_allclose(np.linalg.norm(acc, axis=1), math.sqrt(2) * a_ref, rtol=2e-6)
    # the Lagrangian I_zz agrees with the hand-computed total inertia about the yaw axis, and x, y, yaw decouple
    M, _ = mass_matrix_and_potential(sc.robot, torch.tensor(s0[:sc.ndof], dtype=torch.float64), (0.0, 0.0, -G))
    M = M.numpy()
    np.testing.assert_allclose(M[2, 2], kn["I_zz"], rtol=1e-9)
    np.testing.assert_allclose(M[0, 0], kn["m_tot"], rtol=1e-9)
    assert np.abs(M[0:3][:, [i for i in range(sc.ndof) if i not in (0, 1, 2)]]).max() <= 1e-12 and abs(M[0, 2]) + abs(M[1, 2]) <= 1e-12
    q, qd = _run(oracle, sc, p, s0, 0.0, 40.0)
    alpha = np.diff(np.concatenate([[s0[sc.ndof + 2]], qd[:n, 2]])) / dt
    np.testing.assert_allclose(alpha, kn["mu"] * kn["m_tot"] * G * kn["L"] / 2 / kn["I_zz"], rtol=2e-6)
    assert np.abs(q[:n, 0:2] - s0[0:2]).max() <= 1e-9


def test_known_answer_wall_force(oracle, synth_dir):
    """Driven square-on into a static wall (chassis box unrotated in its link frame, forward axis along the wall normal): the box
    stops at the face (its +x face within the contact margin of it), the wall's net contact force converges to the saturated drive
    force mu m_tot g along the normal, and the vertical force is 0 -- the vertical friction row has no effective inverse mass through
    x, y and yaw and is dropped."""
    sc, p, s0, kn = symmetric_base(synth_dir, axis_angle=np.pi / 2, yaw0=0.0, wall=True, T=100, dt=0.01, substeps=2)
    m, nb = sc.model, sc.ndof
    np.testing.assert_allclose(np.array(m.fwd_axis[:]), [1.0, 0.0], atol=1e-12)
    hx = sc.layout["box"][2][0]
    acts = np.zeros((p.T, sc.nu, p.K), np.float32)
    acts[:, 0] = 1.0
    _, obs = oracle.rollout(m, p, s0, acts, use_double=True, root0=sc.root_state0)
    x = obs[13, :, 0].astype(np.float64)
    wall_slot = sc.contact_slot[sc.body_offset[sc.actor_names.index("wall")]]
    f0 = 13 + 2 * nb
    F = obs[f0 + 3 * wall_slot: f0 + 3 * wall_slot + 3, :, 0].astype(np.float64)
    front = x[-20:] + hx
    print(f"SYNTH-PLANAR wall face_gap={WALL_FACE - front.max():.3g}..{WALL_FACE - front.min():.3g} F={F[:, -1]} drive={kn['mu'] * kn['m_tot'] * G:.6g}")
    assert np.abs(front - WALL_FACE).max() <= m.contact_margin
    assert (np.abs(F[:, :20]).max(axis=0) == 0).all() and np.abs(F).max() > 0  # no contact before it gets there
    np.testing.assert_allclose(F[0, -10:], kn["mu"] * kn["m_tot"] * G, rtol=1e-3)
    assert (F[2] == 0).all()
    y, yaw = obs[13 + 2, :, 0].astype(np.float64), obs[13 + 4, :, 0].astype(np.float64)       # DOF rows: q0, qd0, q1, qd1, ...
    assert np.abs(y).max() <= 1e-4 and np.abs(yaw).max() <= 1e-4                            # square-on: no sideways or turning motion


# ---------------------------------------------------------------------------------------------------------------------------
# routing and template coverage
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", FREE_CASES, ids=[free_case_id(c) for c in FREE_CASES])
def test_planar_models_route_to_team(synth_dir, case):
    """Every generated planar model runs on the team kernel by default, also the 4-body serial chain x -> y -> yaw -> wheel that the
    lanes kernel would otherwise take (the lanes kernel has no planar rule); MPPIB_K2_TEAM=0 -> thread per rollout."""
    nw, narm, topo = case
    sc, _, _ = make_planar_robot(synth_dir, 0, narm, topo, nwheels=nw, K=8, T=2)
    m = sc.model
    if (nw, narm) == (1, 0):
        assert is_chain(m) and m.nb == 4
    assert _mapping(m) == "team"
    assert _mapping(m, MPPIB_K2_LANES="0") == "team"
    assert _mapping(m, MPPIB_K2_TEAM="0") == "thread"


def test_template_coverage_and_refusals(synth_dir):
    """The cases reach every team template a planar base can reach: contact-free <8,4>, <8,8>, <16,12>, <16,16>; with contacts
    <8,4,NCS 1-4>, <8,8,NCS 1-4>, <16,12,NCS 2-5>, <16,16,NCS 2-4>.  build_scene refuses 13 bodies with four free boxes and twelve
    shapes, and 15 or more bodies with a single link shape (the thread kernel's 12-contact shared-memory floor)."""
    free = {template(3 + nw + narm, 0, False)[:2] for nw, narm, _ in FREE_CASES}
    assert free == {(8, 4), (8, 8), (16, 12), (16, 16)}
    got = {template(3 + c[0] + c[1], c[3]) for c in CONTACT_CASES}
    want = ({(8, 4, n) for n in range(1, 5)} | {(8, 8, n) for n in range(1, 5)} | {(16, 12, n) for n in range(2, 6)}
            | {(16, 16, n) for n in range(2, 5)})
    assert got == want, sorted(want - got)
    assert len({contact_case_id(c) for c in CONTACT_CASES}) == len(CONTACT_CASES)
    with pytest.raises(NotImplementedError, match="12 needed"):
        make_planar_contact_scene(synth_dir, 0, 8, "tree", 2, 4, arm_shapes=3, K=4, T=1)
    for narm in (10, 11):
        with pytest.raises(NotImplementedError, match="12 needed"):
            make_planar_contact_scene(synth_dir, 0, narm, "tree", 2, 0, arm_shapes=1, K=4, T=1)


@pytest.mark.parametrize("case", CONTACT_CASES, ids=[contact_case_id(c) for c in CONTACT_CASES])
def test_contact_case_routing_and_contacts(oracle, synth_dir, case):
    """Every planar contact case runs on the team kernel by default and on thread per rollout with MPPIB_K2_TEAM=0, and it has
    contacts: at least 30 % of the rollouts carry a contact force after one step."""
    sc, p, st, root0 = make_contact_case(synth_dir, case, K=40, T=1)
    m = sc.model
    assert _mapping(m) == "team" and _mapping(m, MPPIB_K2_TEAM="0") == "thread"
    acts = np.zeros((1, sc.nu, 40), np.float32)
    _, o = oracle.rollout(m, p, None, acts, 0, 1, state=st.copy(), root0=root0, use_double=True)
    f0 = 13 + 2 * sc.ndof + 13 * m.nfree
    frac = float((np.abs(o[f0:, 0]).max(axis=0) > 0).mean())
    assert frac >= 0.3, frac
