"""Deterministic generated DIFFERENTIAL-DRIVE robots for the rollout tests: a planar base (virtual joints x, y, yaw -- DESIGN.md section
2, "Differential-drive bases") carrying 1, 2 or 4 wheels and an arm, compiled through the real path (parse_urdf -> compile_urdf ->
build_scene) with `fixed: False, differential_drive: True`.

    make_planar_robot(tmp_path, seed, narm, topology, nwheels=..., ...) -> (scene, params, state0)
    make_planar_contact_scene(tmp_path, seed, narm, topology, nwheels, nfree, ...) -> (scene, params, state (NS, K), root0)

The generated base has what the shipped ones (boxer, jackal, albert) do not: a chassis with an off-centre, rotated inertia frame; a
wheel axis that is no coordinate axis of the chassis (so fwd_axis is not +-x / +-y); wheels on the chassis or on a rotated fixed-joint
child of it ("mount": the host reads the first wheel's tree_R, both placements give the same fwd_axis); one, two or four wheels; and an
arm of `narm` joints (a chain or a tree, the joint mixes of synth_robots.robot_urdf) on the chassis, so nu = 2 + narm and
nb = 3 + nwheels + narm.  Observed: the chassis link (the root row the RolloutSim getters return for a planar robot), one arm link (the
mount when there is no arm), the first wheel link, and the DOF state.

CASES reach every team template a planar base can reach, contact-free and with contacts (NCS = ceil((nb + 6 nfree) / 8)); see
CONTACT_CASES for the contact combinations that do not fit in shared memory.  Also the symmetric wheel-only base of the known-answer
tests (test_oracle_planar.py, test_gpu_planar.py)."""
import math
import os

import numpy as np

from mppi_isaac_b200.model.blob import OBS_CONTACT, OBS_DOF_STATE, OBS_FREE_STATE, OBS_LINK_STATE, build_scene, make_params
from mppi_isaac_b200.model.urdf import rpy_to_R
from mppi_isaac_b200.utils.config_store import ActorWrapper, IsaacGymConfig, MPPIConfig
from synth_robots import _collision, _f, _parents, _unit

G = 9.8
ARM_TOPOLOGIES = ("chain", "tree")
WALL_FACE, WALL_HALF = 3.0, np.array([0.1, 3.0, 0.5])          # static wall: its -x face at x = WALL_FACE
SPHERE_POS, SPHERE_R = np.array([-3.0, 0.0, 0.0]), 0.15         # static sphere (its height is set to the chassis box's)
FAR_POS = np.array([20.0, 20.0])
SCENARIOS = ("wall", "sphere", "front", "pressed", "far")       # period 5: not a multiple of the 4 rollouts of a contact-phase warp


def yaw_quat(a):
    return np.array([0.0, 0.0, math.sin(a / 2), math.cos(a / 2)])


def rot_z(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def _rpy_of(R):
    """URDF rpy of a rotation matrix (R = Rz(y) Ry(p) Rx(r))."""
    return np.array([math.atan2(R[2, 1], R[2, 2]), math.asin(-max(-1.0, min(1.0, R[2, 0]))), math.atan2(R[1, 0], R[0, 0])])


def _z_to(a):
    """A rotation whose z column is the unit vector a."""
    a = np.asarray(a, float) / np.linalg.norm(a)
    x = np.cross([0.0, 0.0, 1.0], a) if abs(a[2]) < 0.9 else np.array([1.0, 0.0, 0.0])
    x = x - a * (x @ a)
    x /= np.linalg.norm(x)
    return np.column_stack([x, np.cross(a, x), a])


def _inertia_xml(I):
    return (f'<inertia ixx="{I[0, 0]:.9g}" iyy="{I[1, 1]:.9g}" izz="{I[2, 2]:.9g}" ixy="{I[0, 1]:.9g}" ixz="{I[0, 2]:.9g}" '
            f'iyz="{I[1, 2]:.9g}"/>')


def planar_urdf(seed, narm, topology, nwheels, *, on_mount=False, collisions=None, symmetric=False, axis_angle=None,
                chassis_box=None):
    """URDF text and a layout dict: `axis` (the wheel axis in the chassis frame, in its plane), `radius`, `base` (wheel base L),
    `left` / `right` (wheel joint names), `wheel_links`, `tip` (observed arm link), `box` ((centre, yaw in the link frame, half
    extents) of the chassis box or None).

    symmetric=True is the known-answer base: no arm, no mount, chassis inertial at the link origin and unrotated, two undamped wheels
    at +-L/2 along the axis with their centres of mass on it and an inertia symmetric about it -- the total centre of mass is on the yaw
    axis and x, y, yaw and the wheels do not couple in M(q).  `collisions` ({arm link name: box | sphere | cylinder}) adds arm link
    shapes; `chassis_box` (True or (centre, yaw)) a chassis box, and with it every wheel gets a cylinder along its axis."""
    assert nwheels in (1, 2, 4) and narm >= 0 and topology in ARM_TOPOLOGIES and not (symmetric and (narm or on_mount))
    rng = np.random.default_rng([seed, narm, ARM_TOPOLOGIES.index(topology), nwheels, 21])
    col_rng = np.random.default_rng([seed, narm, ARM_TOPOLOGIES.index(topology), nwheels, 22])
    alpha = float(rng.uniform(-np.pi, np.pi)) if axis_angle is None else float(axis_angle)
    a = np.array([math.cos(alpha), math.sin(alpha), 0.0])              # wheel axis, left wheels on its + side
    fwd = np.cross(a, [0.0, 0.0, 1.0])
    r, L = float(rng.uniform(0.05, 0.12)), float(rng.uniform(0.3, 0.6))
    left, right, wheel_links = [], [], []
    out = ['<robot name="planar">']
    if symmetric:
        mc, d = float(rng.uniform(4.0, 10.0)), rng.uniform(0.05, 0.3, 3)
        Ic = np.diag([d[1] + d[2], d[0] + d[2], d[0] + d[1]])
        origin = '<origin xyz="0 0 0"/>'
    else:
        mc, d = float(rng.uniform(4.0, 12.0)), rng.uniform(0.05, 0.3, 3)
        Ic = np.diag([d[1] + d[2], d[0] + d[2], d[0] + d[1]])
        origin = f'<origin xyz="{_f(rng.uniform(-0.08, 0.08, 3))}" rpy="{_f(rng.uniform(-np.pi, np.pi, 3))}"/>'
    box = None
    chassis_col = ""
    if chassis_box is not None and chassis_box is not False:
        half = np.array([rng.uniform(0.18, 0.28), rng.uniform(0.14, 0.22), rng.uniform(0.06, 0.1)])
        if chassis_box is True:
            cen = np.array([*col_rng.uniform(-0.03, 0.03, 2), 0.0])
            byaw = float(col_rng.uniform(-np.pi, np.pi)) if col_rng.uniform() < 0.5 else 0.0      # sometimes rotated in the link frame
        else:
            cen, byaw = np.asarray(chassis_box[0], float), float(chassis_box[1])
        box = (cen, byaw, half)
        chassis_col = (f'<collision><origin xyz="{_f(cen)}" rpy="0 0 {byaw:.9g}"/><geometry><box size="{_f(2 * half)}"/></geometry>'
                       '</collision>')
    out.append(f'<link name="base"><inertial>{origin}<mass value="{mc:.9g}"/>{_inertia_xml(Ic)}</inertial>{chassis_col}</link>')
    # the mount: a fixed-joint child of the chassis with a random rotation (its mass merges into the chassis body)
    Rm = np.eye(3)
    pm = np.zeros(3)
    if not symmetric:
        rpy_m = rng.uniform(-np.pi, np.pi, 3)
        Rm, pm = rpy_to_R(rpy_m), np.array([*rng.uniform(-0.05, 0.05, 2), -0.02])
        out.append(f'<link name="mount"><inertial><origin xyz="{_f(rng.uniform(-0.05, 0.05, 3))}"/><mass value="{rng.uniform(0.2, 0.6):.9g}"/>'
                   '<inertia ixx="0.002" iyy="0.003" izz="0.004" ixy="0" ixz="0" iyz="0"/></inertial></link>')
        out.append(f'<joint name="jmount" type="fixed"><parent link="base"/><child link="mount"/><origin xyz="{_f(pm)}" rpy="{_f(rpy_m)}"/>'
                   '</joint>')
    # wheels: left on the + side of the axis, right on the - side; four wheels add a front / rear offset along the forward axis
    sides = {1: [(1, 0.0)], 2: [(1, 0.0), (-1, 0.0)], 4: [(1, 0.15), (-1, 0.15), (1, -0.15), (-1, -0.15)]}[nwheels]
    mw = float(rng.uniform(0.3, 1.2))
    Ia, Ip = mw * r * r / 2, mw * (3 * r * r + 0.04 ** 2) / 12
    parent, Rp, pp = ("mount", Rm, pm) if on_mount else ("base", np.eye(3), np.zeros(3))
    for w, (s, df) in enumerate(sides):
        name = f"wheel_{'left' if s > 0 else 'right'}_{w}"
        (left if s > 0 else right).append(name)
        wheel_links.append(f"w{w}")
        pos = s * L / 2 * a + df * fwd + np.array([0.0, 0.0, -0.04])      # chassis frame
        ap = Rp.T @ a                                                       # the axis in the parent's frame = in the wheel link's frame
        Iw = Ip * (np.eye(3) - np.outer(ap, ap)) + Ia * np.outer(ap, ap)
        wcol = ""
        if box is not None:
            wcol = (f'<collision><origin xyz="0 0 0" rpy="{_f(_rpy_of(_z_to(ap)))}"/><geometry><cylinder radius="{r:.9g}" length="0.04"/>'
                    '</geometry></collision>')
        out.append(f'<link name="w{w}"><inertial><origin xyz="0 0 0"/><mass value="{mw:.9g}"/>{_inertia_xml(Iw)}</inertial>{wcol}</link>')
        out.append(f'<joint name="{name}" type="continuous"><parent link="{parent}"/><child link="w{w}"/>'
                   f'<origin xyz="{_f(Rp.T @ (pos - pp))}" rpy="0 0 0"/><axis xyz="{_f(ap)}"/>'
                   f'<limit effort="{rng.uniform(20, 80):.9g}" velocity="{rng.uniform(25, 40):.9g}"/><dynamics damping="{0.0 if symmetric else rng.uniform(0.0, 0.1):.9g}"/></joint>')
    # the arm: the joint mixes of synth_robots.robot_urdf, link 0 is the chassis
    cols = {name: _collision(col_rng, kind) for name, kind in sorted((collisions or {}).items())}
    parents = _parents(rng, narm, topology) if narm else []
    for i in range(1, narm + 1):
        m = float(rng.uniform(0.3, 2.0))
        dd = rng.uniform(0.004, 0.04, 3) * m
        out.append(f'<link name="a{i}"><inertial><origin xyz="{_f(rng.uniform(-0.1, 0.1, 3))}" rpy="{_f(rng.uniform(-np.pi, np.pi, 3))}"/>'
                   f'<mass value="{m:.9g}"/><inertia ixx="{dd[1] + dd[2]:.9g}" iyy="{dd[0] + dd[2]:.9g}" izz="{dd[0] + dd[1]:.9g}" ixy="0" '
                   f'ixz="0" iyz="0"/></inertial>{cols.get(f"a{i}", "")}</link>')
        jt = str(rng.choice(["revolute", "continuous", "prismatic"], p=[0.5, 0.2, 0.3]))
        lo, hi = ((-rng.uniform(0.2, 0.4), rng.uniform(0.2, 0.4)) if jt == "prismatic" else (-rng.uniform(1.2, 2.6), rng.uniform(1.2, 2.6)))
        par = "base" if parents[i - 1] == 0 else f"a{parents[i - 1]}"
        xyz = np.array([*rng.uniform(-0.1, 0.1, 2), 0.12]) if par == "base" else rng.uniform(-0.15, 0.15, 3)
        out.append(f'<joint name="j{i}" type="{jt}"><parent link="{par}"/><child link="a{i}"/>'
                   f'<origin xyz="{_f(xyz)}" rpy="{_f(rng.uniform(-np.pi, np.pi, 3))}"/><axis xyz="{_f(_unit(rng))}"/>'
                   f'<limit lower="{lo:.9g}" upper="{hi:.9g}" effort="{rng.uniform(15, 150):.9g}" velocity="{rng.uniform(2.0, 4.0):.9g}"/>'
                   f'<dynamics damping="{rng.uniform(0.05, 0.5):.9g}"/></joint>')
    out.append("</robot>")
    tip = f"a{narm}" if narm else ("mount" if not symmetric else wheel_links[-1])
    layout = dict(axis=a, fwd=fwd, radius=r, base=L, left=left, right=right, wheel_links=wheel_links, tip=tip, box=box,
                  wheel_mass=mw, wheel_Ip=Ip, chassis_mass=mc, chassis_I=Ic)
    return "\n".join(out) + "\n", layout


def make_planar_robot(tmp_path, seed, narm, topology="chain", *, nwheels=2, on_mount=None, collisions=None, actors=(), obs=None,
                      symmetric=False, axis_angle=None, chassis_box=None, friction=None, yaw0=None, pos0=None, z0=None, gravity=True,
                      K=64, T=12, dt=0.02, substeps=1, u_lim=0.5):
    """Write the URDF to `tmp_path`, compile it into a one-robot scene and return (scene, params, state0).  state0 = (q, qd): the
    base at init_pos / init_ori's yaw (random unless given) moving roughly along its forward axis, wheel angles and arm joints random
    (the arm inside its limits, as make_robot).  `on_mount` (default: odd seeds) puts the wheels on the mount.  planar_urdf's layout
    dict is kept as `scene.layout`."""
    on_mount = bool(seed % 2) if on_mount is None else on_mount
    text, lay = planar_urdf(seed, narm, topology, nwheels, on_mount=on_mount and not symmetric, collisions=collisions, symmetric=symmetric,
                            axis_angle=axis_angle, chassis_box=chassis_box)
    fn = f"planar_{topology}{narm}_w{nwheels}_s{seed}{'_m' if on_mount else ''}{'_sym' if symmetric else ''}{'_col' if lay['box'] else ''}.urdf"
    with open(os.path.join(str(tmp_path), fn), "w") as f:
        f.write(text)
    rng = np.random.default_rng([seed, narm, ARM_TOPOLOGIES.index(topology), nwheels, 23])
    mu = float(rng.uniform(0.3, 1.0)) if friction is None else float(friction)
    psi = float(rng.uniform(-np.pi, np.pi)) if yaw0 is None else float(yaw0)
    xy = rng.uniform(-1.0, 1.0, 2) if pos0 is None else np.asarray(pos0, float)
    if z0 is None:
        z0 = 0.15 if lay["box"] is None else 0.04 + lay["box"][2][2]      # a chassis box reaches down to 4 cm above the ground
    actor = ActorWrapper(type="robot", name="planar", urdf_file=fn, fixed=False, differential_drive=True, init_pos=[float(xy[0]), float(xy[1]), z0],
                         init_ori=yaw_quat(psi).tolist(), friction=mu, wheel_radius=lay["radius"], wheel_base=lay["base"], wheel_count=nwheels,
                         left_wheel_joints=list(lay["left"]), right_wheel_joints=list(lay["right"]), dof_mode="velocity", gravity=gravity,
                         collision=lay["box"] is not None or bool(collisions))
    sc = build_scene([actor] + list(actors), assets_dirs=[str(tmp_path)], substep=dt / substeps)
    m = sc.model
    nb = sc.ndof
    assert nb == 3 + nwheels + narm and sc.nu == 2 + narm and m.planar_base == 1 and sc.virtual_dofs == 3
    assert np.allclose(np.array(m.fwd_axis[:]), lay["fwd"][:2], atol=1e-6)                # on the chassis or the mount: the same axis
    sc.layout = lay
    names = sc.robot.link_names
    if obs is not None:
        obs = obs(sc)
    else:
        obs = [(OBS_LINK_STATE, names.index("base")), (OBS_LINK_STATE, names.index(lay["tip"])),
               (OBS_LINK_STATE, names.index(lay["wheel_links"][0])), (OBS_DOF_STATE, 0)]
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.1 * np.eye(sc.nu)).tolist(),
                    u_min=[-u_lim], u_max=[u_lim], lambda_=0.05, sample_null_action=True)
    p = make_params(mc, IsaacGymConfig(dt=dt, substeps=substeps), sc.nu, K, obs)
    q0, qd0 = np.zeros(nb), np.zeros(nb)
    q0[0:3] = sc.dof_state0[[0, 2, 4]]
    f = rot_z(q0[2]) @ lay["fwd"]
    qd0[0:2] = rng.uniform(-0.3, 0.3) * f[:2] + rng.uniform(-0.02, 0.02, 2)
    qd0[2] = rng.uniform(-0.5, 0.5)
    for i in range(3, nb):
        if m.q_hi[i] < 1e29:
            lo, hi = max(m.q_lo[i], -2.0), min(m.q_hi[i], 2.0)
            gap = min(0.3, 0.25 * (hi - lo))
            q0[i] = rng.uniform(lo + gap, hi - gap)
            qd0[i] = rng.uniform(-0.3, 0.3)
        else:
            q0[i] = rng.uniform(-np.pi, np.pi)
            qd0[i] = rng.uniform(-2.0, 2.0)
    return sc, p, np.concatenate([q0, qd0]).astype(np.float32)


def wheel_dofs(sc):
    """(left, right) DOF indices of the wheel joints."""
    a = sc.actor_cfgs[sc.robot_actor]
    names = sc.robot.dof_names
    return [names.index(n) for n in a.left_wheel_joints], [names.index(n) for n in a.right_wheel_joints]


def planar_states(sc, s0, K, rng, *, spread=0.2, big_yaw_every=0):
    """(2 nb, K) per-rollout states: yaw over [-pi, pi] (every `big_yaw_every`-th rollout at |yaw| in [20, 50] rad), x, y around
    s0's, base velocities around the forward axis, wheels and arm as planar_robot's state0, the arm inside its limits."""
    m, nb = sc.model, sc.ndof
    st = np.repeat(s0[:, None], K, 1).astype(np.float64)
    st[0:2] += rng.uniform(-0.5, 0.5, (2, K))
    st[2] = rng.uniform(-np.pi, np.pi, K)
    if big_yaw_every:
        big = np.arange(K) % big_yaw_every == big_yaw_every - 1
        st[2, big] = rng.choice([-1.0, 1.0], big.sum()) * rng.uniform(20.0, 50.0, big.sum())
    fwd = np.array(m.fwd_axis[:], np.float64)
    c, s = np.cos(st[2]), np.sin(st[2])
    v = rng.uniform(-0.4, 0.4, K)
    st[nb + 0] = v * (fwd[0] * c - fwd[1] * s) + rng.uniform(-0.02, 0.02, K)
    st[nb + 1] = v * (fwd[0] * s + fwd[1] * c) + rng.uniform(-0.02, 0.02, K)
    st[nb + 2] = rng.uniform(-0.8, 0.8, K)
    for i in range(3, nb):
        st[i] += rng.uniform(-spread, spread, K)
        if m.q_hi[i] < 1e29:
            st[i] = np.clip(st[i], m.q_lo[i] + 0.02, m.q_hi[i] - 0.02)
        st[nb + i] += rng.uniform(-0.3, 0.3, K)
    return st.astype(np.float32)


def planar_targets(sc, p, state, u):
    """Float64 velocity targets (nb, K) of one substep at `state`: joints 0-2 from the current yaw (the planar-base rule), the
    others from the command map.  u: (nu, K)."""
    m, nb = sc.model, sc.ndof
    u = np.asarray(u, np.float64) * p.u_scale
    tgt = np.array([m.cmd_c0[i] * u[m.cmd_i0[i]] + m.cmd_c1[i] * u[m.cmd_i1[i]] for i in range(nb)], np.float64)
    yaw = np.asarray(state[2], np.float64)
    fx, fy = float(m.fwd_axis[0]), float(m.fwd_axis[1])
    tgt[0] = u[0] * (fx * np.cos(yaw) - fy * np.sin(yaw))
    tgt[1] = u[0] * (fx * np.sin(yaw) + fy * np.cos(yaw))
    tgt[2] = u[1]
    return tgt


# ---------------------------------------------------------------------------------------------------------------------------
# contact scenes
# ---------------------------------------------------------------------------------------------------------------------------
def template(nb, nfree, contact=True):
    """(G, NB, NCS) of the team kernel for nb bodies and nfree free bodies (launch_rollout_team / launch_team_g)."""
    G, NB = (8, 4) if nb <= 4 else (8, 8) if nb <= 8 else (16, 12) if nb <= 12 else (16, 16)
    return G, NB, (-(-(nb + 6 * nfree) // 8) if contact else None)


def template_id(nb, nfree=0, contact=False):
    G, NB, ncs = template(nb, nfree, contact)
    return f"team_G{G}_NB{NB}" + (f"_NCS{ncs}" if contact else "")


# contact-free: (nwheels, narm, topology) -- <8,4>, <8,8>, <16,12>, <16,16>
FREE_CASES = [(1, 0, "chain"), (2, 0, "chain"), (2, 3, "tree"), (4, 1, "chain"), (2, 4, "chain"), (2, 7, "tree"), (4, 5, "tree"),
              (2, 8, "chain"), (2, 11, "tree")]
# with contacts: (nwheels, narm, topology, nfree, arm shapes, randomisation).  NCS 1-4 on <8,4> and <8,8>, 2-5 on <16,12>, 2-4 on
# <16,16>.  With collision shapes a planar base of 13 bodies leaves the thread-per-rollout kernel room for the 12 contact points
# build_scene requires with at most three free boxes (four free boxes and about ten shapes are refused), and 15 or more bodies with
# any link shape are refused: NCS 5 on NB 16 is not reachable by a planar base (test_oracle_planar.py asserts both refusals).
CONTACT_CASES = [
    (1, 0, "chain", 0, 0, False), (1, 0, "chain", 2, 0, True), (1, 0, "chain", 3, 0, False), (1, 0, "chain", 4, 0, True),
    (2, 0, "chain", 0, 0, False), (2, 0, "chain", 1, 0, True), (2, 0, "chain", 2, 0, False), (2, 0, "chain", 4, 0, True),
    (2, 4, "chain", 0, 2, False), (2, 7, "tree", 2, 3, True), (4, 3, "tree", 3, 2, False), (4, 5, "tree", 4, 1, True),
    (2, 8, "chain", 0, 3, False), (2, 8, "tree", 1, 2, True), (2, 8, "tree", 3, 1, True), (2, 9, "tree", 0, 1, False),
]


def free_case_id(case):
    nw, narm, topo = case
    return f"w{nw}{topo}{narm}-{template_id(3 + nw + narm)}"


def contact_case_id(case):
    nw, narm, topo, nfree = case[:4]
    return f"w{nw}{topo}{narm}-nfree{nfree}-{template_id(3 + nw + narm, nfree, True)}"


def _chassis_box_world(lay, x, y, yaw, z0):
    """World centre, rotation and half extents of the chassis box with the base at (x, y, yaw)."""
    cen, byaw, half = lay["box"]
    R = rot_z(yaw)
    return np.array([x, y, z0]) + R @ cen, rot_z(yaw + byaw), half


def _free_row(scenario, f, fb, rng, lay, base, z0):
    """(13,) root-state row of free box f (half extents fb[f]) with the base at `base` = (x, y, yaw)."""
    half = fb[f]
    spot = np.array([0.7 * f - 1.0, -3.0])
    v, w = rng.uniform(-0.05, 0.05, 3), rng.uniform(-0.1, 0.1, 3)
    byaw = float(rng.uniform(-np.pi, np.pi))
    c, Rb, bh = _chassis_box_world(lay, *base, z0)
    if scenario in ("front", "pressed"):
        face = f % 4 if scenario == "pressed" else 0
        d = Rb[:, 0] if face % 2 == 0 else Rb[:, 1]
        d = d * (1 if face < 2 else -1)
        ext_c, ext_b = bh[0 if face % 2 == 0 else 1], half[0]
        gap = -4e-3 if scenario == "pressed" else float(rng.uniform(0.02, 0.15)) + 0.05 * f
        byaw = math.atan2(d[1], d[0])
        x = c + d * (ext_c + ext_b + gap)
        if scenario == "front" and f:                         # side by side in front of the chassis
            x = x + Rb[:, 1] * (0.3 * ((f + 1) // 2) * (-1) ** f)
        x[2] = half[2] - 5e-4
        if scenario == "pressed":
            v = -0.2 * d
    else:
        x = np.array([spot[0], spot[1], half[2] - 5e-4])
    return np.concatenate([x, yaw_quat(byaw), v, w])


def make_planar_contact_scene(tmp_path, seed, narm, topology, nwheels, nfree, *, arm_shapes=1, noise=False, K=64, T=8, dt=0.02,
                              substeps=2):
    """One generated planar contact scene: (scene, params, state (NS, K), root0 (A, 13)).  Collision geometry: a box on the chassis
    (sometimes rotated in the link frame), a cylinder on every wheel (its bounding box spins with the wheel), `arm_shapes` shapes on
    arm links; 0-4 free boxes (every other one randomised if `noise`), the static wall and the static sphere.  Per rollout the
    SCENARIOS put the chassis against the wall or the sphere, the free boxes in front of it, pressed against its faces (beside it
    too), or everything far apart; yaw over [-pi, pi], every 16th rollout at |yaw| in [20, 50] rad.  Observed: the chassis, the
    DOF state, every free body, every contact slot."""
    assert 0 <= nfree <= 4 and (narm == 0 or 1 <= arm_shapes <= narm) and (narm > 0 or arm_shapes == 0)
    rng = np.random.default_rng([seed, narm, ARM_TOPOLOGIES.index(topology), nwheels, nfree, 24])
    links = [f"a{i}" for i in sorted(rng.choice(np.arange(1, narm + 1), arm_shapes, replace=False))] if narm else []
    collisions = {l: ("box", "sphere", "cylinder")[j % 3] for j, l in enumerate(links)}
    nsig = dict(noise_sigma_size=[0.01, 0.01, 0.01], noise_percentage_mass=0.2, noise_percentage_friction=0.3)
    fb = [rng.uniform(0.05, 0.12, 3) for _ in range(nfree)]
    actors = [ActorWrapper(type="box", name=f"box{f}", size=(2 * fb[f]).tolist(), mass=float(rng.uniform(0.3, 2.0)),
                           friction=float(rng.uniform(0.3, 1.0)), fixed=False, **(nsig if noise and f % 2 == 0 else {}))
              for f in range(nfree)]
    _, lay0 = planar_urdf(seed, narm, topology, nwheels, on_mount=bool(seed % 2), collisions=collisions, chassis_box=True)
    z0 = 0.04 + lay0["box"][2][2]
    zc = z0 + lay0["box"][0][2]
    actors.append(ActorWrapper(type="box", name="wall", size=(2 * WALL_HALF).tolist(), fixed=True, friction=float(rng.uniform(0.4, 1.0)),
                               init_pos=[WALL_FACE + WALL_HALF[0], 0.0, WALL_HALF[2]]))
    actors.append(ActorWrapper(type="sphere", name="ball", size=[SPHERE_R], fixed=True, friction=float(rng.uniform(0.4, 1.0)),
                               init_pos=[SPHERE_POS[0], SPHERE_POS[1], zc]))

    def obs(sc):
        return ([(OBS_LINK_STATE, sc.robot.link_names.index("base")), (OBS_DOF_STATE, 0)] + [(OBS_FREE_STATE, f) for f in range(sc.model.nfree)]
                + [(OBS_CONTACT, s) for s in range(sc.model.ncontact_slots)])
    sc, p, s0 = make_planar_robot(tmp_path, seed, narm, topology, nwheels=nwheels, collisions=collisions, chassis_box=True, actors=actors,
                                  obs=obs, K=K, T=T, dt=dt, substeps=substeps, pos0=[0.0, 0.0])
    m, lay, nb = sc.model, sc.layout, sc.ndof
    assert m.nfree == nfree and m.nshapes == nfree + 2 + 1 + nwheels + arm_shapes and m.max_contacts >= 12
    st = np.zeros((2 * nb + 13 * nfree, K), np.float64)
    st[:2 * nb] = planar_states(sc, s0, K, rng, big_yaw_every=16)
    cen, byaw, half = lay["box"]
    for k in range(K):
        scen = SCENARIOS[k % len(SCENARIOS)]
        yaw = float(st[2, k])
        Rb = rot_z(yaw + byaw)
        if scen == "wall":                                    # a chassis corner or face 4 mm into the wall
            ext = float(np.abs(Rb[0]) @ half)
            cx = WALL_FACE + 4e-3 - ext
            st[0, k] = cx - (rot_z(yaw) @ cen)[0]
            st[1, k] = rng.uniform(-1.0, 1.0)
            st[nb:nb + 2, k] = [rng.uniform(0.1, 0.3), rng.uniform(-0.05, 0.05)]      # and moving into it
        elif scen == "sphere":                                # a chassis face 4 mm into the sphere
            d = Rb[:, int(rng.integers(0, 2))] * rng.choice([-1.0, 1.0])
            ext = float(np.abs(Rb.T @ d) @ half)
            c = SPHERE_POS - d * (ext + SPHERE_R - 4e-3)
            st[0:2, k] = c[:2] - (rot_z(yaw) @ cen)[:2]
            st[nb:nb + 2, k] = rng.uniform(0.1, 0.3) * d[:2]
        elif scen == "far":
            st[0:2, k] = FAR_POS + rng.uniform(-1.0, 1.0, 2)
        for f in range(nfree):
            base = (float(st[0, k]), float(st[1, k]), yaw)
            st[2 * nb + 13 * f: 2 * nb + 13 * (f + 1), k] = _free_row(scen, f, fb, rng, lay, base, z0)
    root0 = sc.root_state0.copy()
    for f in range(nfree):                                  # the broadcast starting rows of the free bodies: on the ground at their spots
        root0[m.free_actor[f]] = _free_row("far", f, fb, rng, lay, (0.0, 0.0, 0.0), z0).astype(np.float32)
    return sc, p, st.astype(np.float32), root0


def make_contact_case(tmp_path, case, **kw):
    nw, narm, topo, nfree, arm_shapes, noise = case
    return make_planar_contact_scene(tmp_path, 0, narm, topo, nw, nfree, arm_shapes=arm_shapes, noise=noise, **kw)


# ---------------------------------------------------------------------------------------------------------------------------
# known answers: the symmetric wheel-only base
# ---------------------------------------------------------------------------------------------------------------------------
def symmetric_base(tmp_path, *, axis_angle=0.7, friction=0.6, yaw0=0.0, wall=False, K=4, T=50, dt=0.01, substeps=2):
    """The symmetric two-wheel base (planar_urdf symmetric=True), gravity on.  Returns (scene, params, state0, known) with
    known = dict(m_tot, I_zz (total inertia about the yaw axis), mu, r, L).  wall=True gives the chassis an unrotated box centred on
    the yaw axis and adds a static wall whose -x face is at WALL_FACE; the base then starts 0.5 m in front of it."""
    actors, obs = [], None
    if wall:
        actors = [ActorWrapper(type="box", name="wall", size=(2 * WALL_HALF).tolist(), fixed=True, friction=0.8,
                               init_pos=[WALL_FACE + WALL_HALF[0], 0.0, WALL_HALF[2]])]

        def obs(sc):
            return ([(OBS_LINK_STATE, sc.robot.link_names.index("base")), (OBS_DOF_STATE, 0)]
                    + [(OBS_CONTACT, s) for s in range(sc.model.ncontact_slots)])
    sc, p, s0 = make_planar_robot(tmp_path, 5, 0, "chain", nwheels=2, symmetric=True, axis_angle=axis_angle, friction=friction, yaw0=yaw0,
                                  pos0=[0.0, 0.0] if not wall else None, chassis_box=((np.zeros(3), 0.0) if wall else None), actors=actors,
                                  obs=obs, K=K, T=T, dt=dt, substeps=substeps)
    lay, m = sc.layout, sc.model
    mtot = lay["chassis_mass"] + 2 * lay["wheel_mass"]
    Izz = lay["chassis_I"][2, 2] + 2 * (lay["wheel_Ip"] + lay["wheel_mass"] * (lay["base"] / 2) ** 2)
    s0[:] = 0.0
    s0[2] = yaw0
    if wall:
        s0[0] = WALL_FACE - lay["box"][2][0] - 0.5
    return sc, p, s0, dict(m_tot=mtot, I_zz=Izz, mu=friction, r=lay["radius"], L=lay["base"])
