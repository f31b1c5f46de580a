"""Deterministic generated CONTACT scenes for the rollout tests: the generated robots of synth_robots.py with collision geometry on
some of their links (boxes, spheres, cylinders -- a cylinder becomes its bounding box -- one of them on the root link), 0-4 free boxes,
rotated static boxes (one of them a ramp) and static spheres, all compiled through the real path (parse_urdf -> compile_urdf ->
build_scene).

    make_contact_scene(tmp_path, seed, nb, topology, nfree, ...) -> (scene, params, state, root0)

`state` is the (2 nb + 13 nfree, K) per-rollout starting state.  The free-body rows put each rollout in one of the SCENARIOS below --
resting on the ground, stacked, on an edge or a corner, pressed into the rotated static box, touching a link shape, falling with spin,
far from everything, squeezed against each other, on the ramp -- with a period (10) that is not a multiple of the 4 rollouts a warp
of the team kernel's contact phase holds, so one warp mixes rollouts with no contacts and rollouts at the contact cap.

CASES covers every (NB, NCS) instantiation of the contact team kernel <G, NB, true, NCS, 8, COMPACT> (launch_team_g): NB from the
body count (4, 8, 12, 16), NCS = ceil((nb + 6 nfree) / 8) coordinate slots per lane.  Several cases have more than 8 contact bodies
(MPPIB_MAX_SLOTS: some shapes get no force slot) and several lower the contact cap to 4 or 8 so that it binds.

Also the scenes of the known-answer tests (test_oracle_contact_synth.py): free cubes colliding without gravity or ground, a stack of
boxes, a box on a ramp, a one-joint prismatic robot driving a link sphere into a static box."""
import copy
import math
import os

import numpy as np

from mppi_isaac_b200.model.blob import OBS_CONTACT, OBS_DOF_STATE, OBS_FREE_STATE, build_scene, make_params
from mppi_isaac_b200.model.urdf import R_to_quat_xyzw, forward_kinematics, quat_xyzw_to_R
from mppi_isaac_b200.utils.config_store import ActorWrapper, IsaacGymConfig, MPPIConfig
from synth_robots import TOPOLOGIES, make_robot

G = 9.8
SCENARIOS = ("ground", "stack", "edge", "corner", "pressed", "link", "falling", "far", "squeeze", "ramp")
RAMP_POS, RAMP_HALF, RAMP_ANGLE = np.array([0.0, 6.0, 0.6]), np.array([0.8, 0.6, 0.1]), 0.35
ROT_POS = np.array([0.0, -6.0, 0.8])
STACK_POS, SQUEEZE_POS, FAR_POS = np.array([-6.0, 0.0, 0.0]), np.array([-6.0, 6.0, 2.5]), np.array([40.0, 40.0, 10.0])


def team_template(nb, nfree):
    """(G, NB, NCS) of the contact team kernel launch_rollout_team / launch_team_g pick for nb bodies and nfree free bodies."""
    G, NB = (8, 4) if nb <= 4 else (8, 8) if nb <= 8 else (16, 12) if nb <= 12 else (16, 16)
    return G, NB, -(-(nb + 6 * nfree) // 8)


def template_id(nb, nfree):
    G, NB, ncs = team_template(nb, nfree)
    return f"team_G{G}_NB{NB}_NCS{ncs}"


# (nb, topology, nfree, static boxes, static spheres, link shapes, link spheres, randomisation, max_contacts or None)
CASES = [
    (3, "chain", 0, 3, 2, 3, 1, False, None),
    (4, "tree", 2, 2, 1, 3, 1, True, 8),
    (3, "chain", 3, 3, 1, 3, 2, False, None),
    (4, "star", 4, 2, 1, 3, 1, True, 4),
    (6, "tree", 0, 3, 2, 4, 2, False, None),
    (5, "tree", 1, 3, 1, 3, 1, True, None),
    (7, "chain", 2, 2, 1, 4, 2, False, 4),
    (8, "tree", 4, 3, 1, 3, 1, True, None),
    (10, "tree", 0, 3, 2, 5, 2, True, 8),
    (9, "forest", 2, 2, 1, 3, 1, True, None),
    (12, "tree", 3, 3, 1, 4, 2, False, 8),
    (11, "tree", 4, 2, 1, 3, 1, True, None),
    (13, "tree", 0, 3, 2, 5, 2, False, None),
    (13, "tree", 1, 2, 1, 3, 1, False, 4),
    (13, "tree", 3, 2, 1, 2, 1, True, None),
    (13, "tree", 4, 2, 0, 1, 0, True, 8),
]
# With collision shapes, 14 or more bodies leave the thread-per-rollout kernel's shared memory too little room for the 12 contact
# points build_scene requires once free bodies join (a 16-body model not even without them), so the NB = 16 template is reached with
# 13 bodies; the 16-body deep chain runs contact-free only (test_gpu_synth.py).


def case_id(case):
    nb, topology, nfree = case[:3]
    return f"{topology}{nb}-nfree{nfree}-{template_id(nb, nfree)}"


def _yaw(a):
    return np.array([0.0, 0.0, math.sin(a / 2), math.cos(a / 2)])


def _axis_angle(axis, a):
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    return np.concatenate([axis * math.sin(a / 2), [math.cos(a / 2)]])


def _qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def _random_quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q) * np.sign(q[3])


def on_ground(half, quat, xy, sink=5e-4):
    """Centre of a box of half extents `half` at orientation `quat` whose lowest point is `sink` below the ground."""
    R = quat_xyzw_to_R(quat)
    return np.array([xy[0], xy[1], float(np.abs(R[2]) @ half) - sink])


def _link_shapes_world(sc, q):
    """World centre and bounding radius of every collision primitive on the robot's links at joint positions q."""
    m = sc.model
    pos, quat = forward_kinematics(sc.robot, q, np.array(m.base_pos[:], float), np.array(m.base_quat[:], float))
    out = []
    for l, cols in enumerate(sc.robot.link_collisions):
        for col in cols:
            c = pos[l] + quat_xyzw_to_R(quat[l]) @ np.asarray(col["p"], float)
            if col["kind"] == "sphere":
                r = float(col["size"][0])
            elif col["kind"] == "box":
                r = 0.5 * float(np.linalg.norm(col["size"]))
            else:
                r = float(np.hypot(col["size"][0] * math.sqrt(2), 0.5 * col["size"][1]))
            out.append((c, r, col["kind"]))
    return out


def _free_rows(scenario, f, fb, rng, link_world, rot_quat, rot_half, lift=0.0):
    """(13,) root-state row of free box f (half extents fb[f]) in `scenario`.  `lift`: how far the ground margin exceeds its 1 cm floor
    (1.5 g h^2 - 0.01 above h = 0.026 s); a falling box starts that much higher, so that it keeps its clearance above the margin."""
    half = fb[f]
    spot = np.array([6.0, -6.0 + 1.5 * f])                           # a spot of its own on the ground for every box
    v, w = rng.uniform(-0.05, 0.05, 3), rng.uniform(-0.1, 0.1, 3)
    quat = _yaw(rng.uniform(-np.pi, np.pi))
    if scenario == "ground" or (scenario in ("pressed", "link", "ramp") and f > 0) or (scenario == "squeeze" and len(fb) < 2):
        x = on_ground(half, quat, spot)
    elif scenario == "stack":
        quat = _yaw(rng.uniform(-0.2, 0.2))
        z = sum(2 * fb[g][2] for g in range(f)) + half[2] - 5e-4 * (f + 1)
        x = np.array([STACK_POS[0] + rng.uniform(-0.01, 0.01), STACK_POS[1] + rng.uniform(-0.01, 0.01), z])
        v, w = 0.1 * v, 0.1 * w
    elif scenario == "edge":
        quat = _qmul(_yaw(rng.uniform(-np.pi, np.pi)), _axis_angle([1, 0, 0], np.pi / 4 + rng.uniform(-0.05, 0.05)))
        x = on_ground(half, quat, spot)
    elif scenario == "corner":
        quat = _qmul(_axis_angle([1, 0, 0], np.pi / 4), _axis_angle([0, 1, 0], 0.6155 + rng.uniform(-0.05, 0.05)))
        x = on_ground(half, quat, spot)
    elif scenario == "pressed":                                        # into a face of the rotated static box, 5 mm deep
        quat = rot_quat
        ax = int(rng.integers(0, 3))
        d = np.zeros(3)
        d[ax] = rng.choice([-1.0, 1.0]) * (rot_half[ax] + half[ax] - 5e-3)
        x = ROT_POS + quat_xyzw_to_R(rot_quat) @ d
        v = quat_xyzw_to_R(rot_quat) @ (-0.3 * np.sign(d))              # and moving into it
    elif scenario == "link":                                           # overlapping a link shape
        c, r, _ = link_world[int(rng.integers(0, len(link_world)))]
        d = rng.normal(size=3)
        x = c + d / np.linalg.norm(d) * (r + half.min() - 0.01)
        v = -0.2 * d / np.linalg.norm(d)
    elif scenario == "falling":
        x = np.array([spot[0], spot[1], 0.2 + lift + rng.uniform(0.0, 0.4)])
        v, w = np.array([0.0, 0.0, -1.0]) + rng.uniform(-0.5, 0.5, 3), rng.uniform(-4, 4, 3)
        quat = _random_quat(rng)
    elif scenario == "far":
        x, v, w = FAR_POS + np.array([3.0 * f, 0, 0]), np.zeros(3), np.zeros(3)
    elif scenario == "squeeze":                                        # in a row in the air, each 5 mm into the next, closing in
        quat = _yaw(rng.uniform(-0.1, 0.1))
        x0 = sum(2 * fb[g][0] for g in range(f)) + half[0] - 5e-3 * f
        x = SQUEEZE_POS + np.array([x0, 0.0, 0.0])
        v = np.array([0.5 if f % 2 == 0 else -0.5, 0.0, 0.0]) + rng.uniform(-0.1, 0.1, 3)
        w = rng.uniform(-1, 1, 3)
    else:                                                              # ramp: flush on the ramp's top face
        Rr = quat_xyzw_to_R(_axis_angle([0, 1, 0], RAMP_ANGLE))
        quat = R_to_quat_xyzw(Rr)
        x = RAMP_POS + Rr @ np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), RAMP_HALF[2] + half[2] - 5e-4])
    return np.concatenate([x, quat, v, w])


def make_contact_scene(tmp_path, seed, nb, topology, nfree, *, statics=2, static_spheres=1, link_shapes=3, link_spheres=1, noise=False,
                       max_contacts=None, K=64, T=8, dt=0.02, substeps=2, gravity_off=True, dof_mode="velocity"):
    """One generated contact scene: (scene, params, state (NS, K), root0 (A, 13)).  The robot gets `link_shapes` collision primitives
    (the root link's box, `link_spheres` spheres, the rest boxes and cylinders); free box f > 0 has gravity off if `gravity_off` and f is
    odd.  Static boxes: the ramp, a randomly rotated box, and the rest (like the static spheres) overlapping link shapes at the starting
    joint positions.  `max_contacts` lowers the model's contact cap (on a copy of the model) so that it binds often.  `dof_mode` is the
    robot's drive (velocity, or effort: torque commands).  Observed: the DOF state, every free body, every contact slot."""
    assert 0 <= nfree <= 4 and statics >= 2 and 1 <= link_shapes <= nb + 1
    rng = np.random.default_rng([seed, nb, TOPOLOGIES.index(topology), nfree, 3])
    links = ["l0"] + [f"l{i}" for i in sorted(rng.choice(np.arange(1, nb + 1), link_shapes - 1, replace=False))]
    kinds = ["box"] + ["sphere"] * link_spheres + [("box", "cylinder")[i % 2] for i in range(link_shapes - 1 - link_spheres)]
    collisions = dict(zip(links, kinds))
    nsig = dict(noise_sigma_size=[0.01, 0.01, 0.01], noise_percentage_mass=0.2, noise_percentage_friction=0.3) if noise else {}
    fb = [rng.uniform(0.04, 0.12, 3) for _ in range(nfree)]
    actors = []
    for f in range(nfree):
        actors.append(ActorWrapper(type="box", name=f"box{f}", size=(2 * fb[f]).tolist(), mass=float(rng.uniform(0.3, 2.0)),
                                   friction=float(rng.uniform(0.3, 1.0)), fixed=False, gravity=not (gravity_off and f % 2 == 1), **nsig))
    rot_quat, rot_half = _random_quat(rng), rng.uniform(0.15, 0.3, 3)
    actors.append(ActorWrapper(type="box", name="ramp", size=(2 * RAMP_HALF).tolist(), fixed=True, friction=float(rng.uniform(0.4, 1.0)),
                               init_pos=RAMP_POS.tolist(), init_ori=_axis_angle([0, 1, 0], RAMP_ANGLE).tolist()))
    actors.append(ActorWrapper(type="box", name="rotated", size=(2 * rot_half).tolist(), fixed=True, friction=float(rng.uniform(0.4, 1.0)),
                               init_pos=ROT_POS.tolist(), init_ori=rot_quat.tolist(), **nsig))
    base_pos = [0.0, 0.0, 1.5]
    # the joint positions of make_robot's state0: the statics at the link shapes are placed against them
    sc0, _, s0 = make_robot(tmp_path, seed, nb, topology, K=2, T=1, base_pos=base_pos, collisions=collisions)
    link_world = _link_shapes_world(sc0, s0[:nb].astype(np.float64))
    targets = rng.permutation(len(link_world))
    for j in range(statics - 2 + static_spheres):
        c, r, _ = link_world[targets[j % len(link_world)]]
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        if j < statics - 2:
            half = rng.uniform(0.05, 0.15, 3)
            actors.append(ActorWrapper(type="box", name=f"static{j}", size=(2 * half).tolist(), fixed=True, init_pos=(c + d * (0.5 * r + half.min())).tolist(),
                                       init_ori=_random_quat(rng).tolist(), friction=float(rng.uniform(0.4, 1.0))))
        else:
            rad = float(rng.uniform(0.05, 0.12))
            actors.append(ActorWrapper(type="sphere", name=f"ball{j}", size=[rad], fixed=True, init_pos=(c + d * (0.8 * r + rad)).tolist(),
                                       friction=float(rng.uniform(0.4, 1.0))))

    def obs(sc):
        return ([(OBS_DOF_STATE, 0)] + [(OBS_FREE_STATE, f) for f in range(sc.model.nfree)]
                + [(OBS_CONTACT, s) for s in range(sc.model.ncontact_slots)])
    sc, p, s0 = make_robot(tmp_path, seed, nb, topology, K=K, T=T, dt=dt, substeps=substeps, base_pos=base_pos, collisions=collisions,
                           actors=actors, obs=obs, dof_mode=dof_mode)
    m = sc.model
    assert m.nfree == nfree and m.nshapes == nfree + statics + static_spheres + link_shapes and m.nshapes <= 24 and m.max_contacts >= 12
    if max_contacts is not None:
        sc.model = m = copy.deepcopy(m)
        m.max_contacts = int(max_contacts)
    # per-rollout starting states
    st = np.zeros((2 * nb + 13 * nfree, K), np.float64)
    lo, hi = np.array(m.q_lo[:nb], np.float64), np.array(m.q_hi[:nb], np.float64)
    st[:nb] = np.clip(s0[:nb, None] + rng.uniform(-0.03, 0.03, (nb, K)), lo[:, None], hi[:, None])
    st[nb:2 * nb] = rng.uniform(-0.3, 0.3, (nb, K))
    root0 = sc.root_state0.copy()
    lift = max(0.0, float(m.ground_margin) - 0.01)
    for k in range(K):
        scen = SCENARIOS[k % len(SCENARIOS)]
        for f in range(nfree):
            st[2 * nb + 13 * f: 2 * nb + 13 * (f + 1), k] = _free_rows(scen, f, fb, rng, link_world, rot_quat, rot_half, lift)
    for f in range(nfree):                                  # the broadcast starting rows of the free bodies: resting on the ground
        root0[m.free_actor[f]] = _free_rows("ground", f, fb, rng, link_world, rot_quat, rot_half).astype(np.float32)
    return sc, p, st.astype(np.float32), root0


def make_case(tmp_path, case, **kw):
    nb, topology, nfree, statics, spheres, link_shapes, link_spheres, noise, cap = case
    return make_contact_scene(tmp_path, 0, nb, topology, nfree, statics=statics, static_spheres=spheres, link_shapes=link_shapes,
                              link_spheres=link_spheres, noise=noise, max_contacts=cap, **kw)


def contact_bodies(sc):
    """Distinct bodies carrying a collision shape (free boxes, statics, links); more than MPPIB_MAX_SLOTS leaves some without a slot."""
    actors = sum(1 for i, a in enumerate(sc.actor_cfgs) if i != sc.robot_actor and a.collision)
    return actors + sum(1 for cols in sc.robot.link_collisions if cols)


# ---------------------------------------------------------------------------------------------------------------------------
# known-answer scenes: a contact-free two-body robot far away, the boxes where the answer is known
# ---------------------------------------------------------------------------------------------------------------------------
def _aside_robot(tmp_path, actors, K, T, dt, substeps):
    """A 2-body generated robot without collision geometry (it takes part in no contact) plus `actors`; observes every free body
    and every contact slot."""
    def obs(sc):
        return [(OBS_FREE_STATE, f) for f in range(sc.model.nfree)] + [(OBS_CONTACT, s) for s in range(sc.model.ncontact_slots)]
    sc, p, s0 = make_robot(tmp_path, 7, 2, "chain", K=K, T=T, dt=dt, substeps=substeps, base_pos=[0.0, 0.0, 1.0], actors=actors, obs=obs)
    return sc, p, s0


def cube_collision_scene(tmp_path, seed, ncubes, K=8, T=30, dt=0.02, substeps=2, speed=1.0):
    """2-4 free cubes, gravity off, no ground, no randomisation, sent into one another with random velocities and spins (scaled by
    `speed`): the contacts are the only forces.  Returns (scene, params, state (NS, K), masses, half sizes)."""
    rng = np.random.default_rng([seed, ncubes, 11])
    h = rng.uniform(0.05, 0.12, ncubes)
    mass = rng.uniform(0.3, 2.0, ncubes)
    actors = [ActorWrapper(type="box", name=f"cube{f}", size=[2 * h[f]] * 3, mass=float(mass[f]), friction=float(rng.uniform(0.3, 1.0)),
                           fixed=False, gravity=False, init_pos=[5.0 + f, 0.0, 1.0]) for f in range(ncubes)]
    sc, p, s0 = _aside_robot(tmp_path, actors, K, T, dt, substeps)
    sc.model = copy.deepcopy(sc.model)
    sc.model.ground_plane = 0
    nb = sc.ndof
    st = np.zeros((2 * nb + 13 * ncubes, K), np.float64)
    st[:nb] = s0[:nb, None]
    centre = np.array([5.0, 0.0, 1.0])
    for k in range(K):
        for f in range(ncubes):
            d = rng.normal(size=3)
            d /= np.linalg.norm(d)
            x = centre + d * rng.uniform(0.15, 0.35)
            v = (centre - x) / np.linalg.norm(centre - x) * rng.uniform(1.0, 3.0) + rng.uniform(-0.3, 0.3, 3)
            st[2 * nb + 13 * f: 2 * nb + 13 * (f + 1), k] = np.concatenate([x, _random_quat(rng), speed * v, speed * rng.uniform(-5, 5, 3)])
    return sc, p, st.astype(np.float32), mass, h


def stack_scene(tmp_path, seed, nboxes, K=4, T=60, dt=0.02, substeps=4):
    """`nboxes` boxes stacked flush on the ground at rest, no randomisation.  Returns (scene, params, state, masses)."""
    rng = np.random.default_rng([seed, nboxes, 12])
    half = [np.array([rng.uniform(0.12, 0.2), rng.uniform(0.12, 0.2), rng.uniform(0.05, 0.1)]) for _ in range(nboxes)]
    half = sorted(half, key=lambda a: -a[0] * a[1])                    # the wider ones below
    mass = np.sort(rng.uniform(0.5, 2.0, nboxes))[::-1]                # and the heavier ones
    actors = [ActorWrapper(type="box", name=f"box{f}", size=(2 * half[f]).tolist(), mass=float(mass[f]), friction=float(rng.uniform(0.5, 1.0)),
                           fixed=False, init_pos=[5.0, 0.0, 0.0]) for f in range(nboxes)]
    sc, p, s0 = _aside_robot(tmp_path, actors, K, T, dt, substeps)
    nb = sc.ndof
    st = np.zeros((2 * nb + 13 * nboxes, K), np.float32)
    st[:nb] = s0[:nb, None]
    z = 0.0
    for f in range(nboxes):
        row = np.concatenate([[5.0, 0.0, z + half[f][2]], [0, 0, 0, 1.0], np.zeros(6)])
        st[2 * nb + 13 * f: 2 * nb + 13 * (f + 1)] = row[:, None]
        z += 2 * half[f][2]
    return sc, p, st, mass


def resting_boxes_scene(tmp_path, seed, nboxes, K=4, T=50, dt=0.1, substeps=1, max_contacts=None):
    """`nboxes` boxes of 16 x 14 x 10 cm and 1.0 - 1.6 kg flat on the ground, 0.6 m apart, at rest, no randomisation; `max_contacts`
    lowers the contact cap on a copy of the model.  Returns (scene, params, state, masses)."""
    rng = np.random.default_rng([seed, nboxes, 13])
    half = np.array([0.08, 0.07, 0.05])
    mass = rng.uniform(1.0, 1.6, nboxes)
    actors = [ActorWrapper(type="box", name=f"box{f}", size=(2 * half).tolist(), mass=float(mass[f]), friction=float(rng.uniform(0.5, 1.0)),
                           fixed=False, init_pos=[5.0, 0.6 * f, half[2]]) for f in range(nboxes)]
    sc, p, s0 = _aside_robot(tmp_path, actors, K, T, dt, substeps)
    if max_contacts is not None:
        sc.model = copy.deepcopy(sc.model)
        sc.model.max_contacts = int(max_contacts)
    nb = sc.ndof
    st = np.zeros((2 * nb + 13 * nboxes, K), np.float32)
    st[:nb] = s0[:nb, None]
    for f in range(nboxes):
        st[2 * nb + 13 * f: 2 * nb + 13 * (f + 1)] = np.concatenate([[5.0, 0.6 * f, half[2]], [0, 0, 0, 1.0], np.zeros(6)])[:, None]
    return sc, p, st, mass


def ramp_scene(tmp_path, angle, mu_box, mu_ramp, K=4, T=25, dt=0.02, substeps=2):
    """A box flush on the top face of a static box tilted by `angle` about y.  Returns (scene, params, state); the box slides
    along -x' (down the slope) if the average friction is below tan(angle)."""
    half = np.array([0.1, 0.1, 0.05])
    rq = _axis_angle([0, 1, 0], angle)
    actors = [ActorWrapper(type="box", name="box", size=(2 * half).tolist(), mass=1.0, friction=mu_box, fixed=False, init_pos=[0.0, 0.0, 3.0]),
              ActorWrapper(type="box", name="ramp", size=(2 * RAMP_HALF * [2, 1, 1]).tolist(), fixed=True, friction=mu_ramp,
                           init_pos=[5.0, 0.0, 1.0], init_ori=rq.tolist())]
    sc, p, s0 = _aside_robot(tmp_path, actors, K, T, dt, substeps)
    nb = sc.ndof
    Rr = quat_xyzw_to_R(rq)
    x = np.array([5.0, 0.0, 1.0]) + Rr @ np.array([0.0, 0.0, RAMP_HALF[2] + half[2]])
    st = np.zeros((2 * nb + 13, K), np.float32)
    st[:nb] = s0[:nb, None]
    st[2 * nb:] = np.concatenate([x, rq, np.zeros(6)])[:, None]
    return sc, p, st


SLIDER_URDF = """<robot name="slider">
<link name="base"><inertial><mass value="2.0"/><inertia ixx="0.01" iyy="0.01" izz="0.01" ixy="0" ixz="0" iyz="0"/></inertial></link>
<link name="tip"><inertial><mass value="0.5"/><inertia ixx="0.002" iyy="0.002" izz="0.002" ixy="0" ixz="0" iyz="0"/></inertial>
<collision><origin xyz="0 0 0"/><geometry><sphere radius="{r}"/></geometry></collision></link>
<joint name="slide" type="prismatic"><parent link="base"/><child link="tip"/><origin xyz="0 0 0"/><axis xyz="1 0 0"/>
<limit lower="-1" upper="2" effort="{effort}" velocity="2"/><dynamics damping="0.0"/></joint>
</robot>
"""


def slider_scene(tmp_path, r=0.1, face=0.6, effort=1000.0, K=4, T=100, dt=0.02, substeps=2, dof_mode="velocity"):
    """A one-joint prismatic robot (a velocity or effort drive along world x) whose link is a sphere of radius r, and a static box
    whose -x face is at x = face.  Returns (scene, params, state0)."""
    fn = "slider.urdf"
    with open(os.path.join(str(tmp_path), fn), "w") as f:
        f.write(SLIDER_URDF.format(r=r, effort=effort))
    robot = ActorWrapper(type="robot", name="slider", urdf_file=fn, fixed=True, init_pos=[0.0, 0.0, 0.3], dof_mode=dof_mode, collision=True)
    wall = ActorWrapper(type="box", name="wall", size=[0.4, 0.6, 0.6], fixed=True, init_pos=[face + 0.2, 0.0, 0.3])
    sc = build_scene([robot, wall], assets_dirs=[str(tmp_path)], substep=dt / substeps)
    obs = [(OBS_DOF_STATE, 0)] + [(OBS_CONTACT, s) for s in range(sc.model.ncontact_slots)]
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=[[0.1]], u_min=[-1.0], u_max=[1.0],
                    lambda_=0.05, sample_null_action=True)
    p = make_params(mc, IsaacGymConfig(dt=dt, substeps=substeps), sc.nu, K, obs)
    return sc, p, np.zeros(2, np.float32)
