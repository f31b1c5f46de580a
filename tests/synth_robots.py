"""Deterministic generated robots for the rollout tests: random URDFs compiled through the real path (parse_urdf -> compile_urdf ->
build_scene), so the rollout kernels are exercised on geometry the shipped robots never have -- arbitrary joint axes and origins, a
rotated and shifted base, rotated inertial frames with off-centre centres of mass, prismatic / revolute / continuous mixes, a
fixed-joint link merged into its body, a very light link -- and on every body count and topology the kernels are specialised for.

    make_robot(tmp_path, seed, nb, topology) -> (scene, params, state0)     (shaped like the builders of scenes.py)

Topologies: "chain" (body i hangs below body i - 1), "tree" (random, depth first, at least one branch), "forest" (several joints on
the root link), "star" (every body on the root link), "deep" (a serial chain of exactly 16 bodies: the depth the team kernel's four
pointer-jumping rounds reach).  Observed: the root link (it belongs to no body), the fixed-joint link, the tip link, and the DOF state.
"""
import os

import numpy as np

from mppi_isaac_b200.model.blob import OBS_DOF_STATE, OBS_LINK_STATE, build_scene, make_params
from mppi_isaac_b200.utils.config_store import ActorWrapper, IsaacGymConfig, MPPIConfig

TOPOLOGIES = ("chain", "tree", "forest", "star", "deep")


def _parents(rng, nb, topology):
    """URDF parent link of links 1..nb (link 0 is the root link)."""
    if topology in ("chain", "deep"):
        return [i - 1 for i in range(1, nb + 1)]
    if topology == "star":
        return [0] * nb
    if topology == "forest":
        nroot = min(nb, 3)
        par = [0] * nroot + [int(rng.integers(1, i)) for i in range(nroot + 1, nb + 1)]
        return par
    # tree: a single root body, random ancestors among the last few links (so the tree has some depth), at least one branch point
    while True:
        par = [0] + [int(rng.integers(max(1, i - 3), i)) for i in range(2, nb + 1)]
        if nb < 3 or len(set(par)) < len(par):
            return par


def _unit(rng):
    v = rng.normal(size=3)
    return v / np.linalg.norm(v)


def _f(v):
    return " ".join(f"{x:.9g}" for x in np.atleast_1d(v))


def _collision(rng, kind):
    """One <collision> element of the given kind (box / sphere / cylinder) at a random offset and rotation in its link frame."""
    if kind == "box":
        geom = f'<box size="{_f(rng.uniform(0.06, 0.2, 3))}"/>'
    elif kind == "sphere":
        geom = f'<sphere radius="{rng.uniform(0.04, 0.1):.9g}"/>'
    else:
        geom = f'<cylinder radius="{rng.uniform(0.03, 0.08):.9g}" length="{rng.uniform(0.08, 0.2):.9g}"/>'
    return (f'<collision><origin xyz="{_f(rng.uniform(-0.05, 0.05, 3))}" rpy="{_f(rng.uniform(-np.pi, np.pi, 3))}"/>'
            f'<geometry>{geom}</geometry></collision>')


def robot_urdf(seed, nb, topology, collisions=None):
    """URDF text and the names of the fixed-joint link and the tip link.  Joint 1 is prismatic for even nb (the prismatic axis of a
    body on the base is rotated by the base pose), revolute for odd nb; the other joints are a random revolute / continuous /
    prismatic mix.  `collisions` ({link name: box | sphere | cylinder}) adds one collision primitive to each named link; its sizes
    and poses come from an RNG stream of their own, so the rest of the URDF is the same with and without them."""
    assert topology in TOPOLOGIES and 1 <= nb <= 16 and (topology != "deep" or nb == 16)
    rng = np.random.default_rng([seed, nb, TOPOLOGIES.index(topology)])
    col_rng = np.random.default_rng([seed, nb, TOPOLOGIES.index(topology), 2])
    cols = {name: _collision(col_rng, kind) for name, kind in sorted((collisions or {}).items())}
    parents = _parents(rng, nb, topology)
    fixed_on = max(1, nb // 2)                   # link carrying the fixed-joint child "fx"; its child joints hang below "fx"
    light = max(1, nb - 1)                       # the light link (mass 1e-3)
    out = ['<robot name="synth">',
           f'<link name="l0"><inertial><origin xyz="{_f(rng.uniform(-0.05, 0.05, 3))}"/><mass value="3.0"/>'
           f'<inertia ixx="0.02" iyy="0.03" izz="0.04" ixy="0" ixz="0" iyz="0"/></inertial>{cols.get("l0", "")}</link>']

    def inertial(m):
        d = rng.uniform(0.004, 0.04, 3) * m
        return (f'<inertial><origin xyz="{_f(rng.uniform(-0.1, 0.1, 3))}" rpy="{_f(rng.uniform(-np.pi, np.pi, 3))}"/><mass value="{m:.9g}"/>'
                f'<inertia ixx="{d[1] + d[2]:.9g}" iyy="{d[0] + d[2]:.9g}" izz="{d[0] + d[1]:.9g}" ixy="0" ixz="0" iyz="0"/></inertial>')

    for i in range(1, nb + 1):
        m = 1e-3 if i == light else float(rng.uniform(0.3, 2.0))
        out.append(f'<link name="l{i}">{inertial(m)}{cols.get(f"l{i}", "")}</link>')
        if i == 1:
            jt = "prismatic" if nb % 2 == 0 else "revolute"
        else:
            jt = str(rng.choice(["revolute", "continuous", "prismatic"], p=[0.5, 0.2, 0.3]))
        par = "fx" if parents[i - 1] == fixed_on else f"l{parents[i - 1]}"
        if jt == "prismatic":
            lo, hi = -rng.uniform(0.2, 0.4), rng.uniform(0.2, 0.4)
        else:
            lo, hi = -rng.uniform(1.2, 2.6), rng.uniform(1.2, 2.6)
        lim = f'<limit lower="{lo:.9g}" upper="{hi:.9g}" effort="{rng.uniform(15, 150):.9g}" velocity="{rng.uniform(2.0, 4.0):.9g}"/>'
        out.append(f'<joint name="j{i}" type="{jt}"><parent link="{par}"/><child link="l{i}"/>'
                   f'<origin xyz="{_f(rng.uniform(-0.15, 0.15, 3))}" rpy="{_f(rng.uniform(-np.pi, np.pi, 3))}"/><axis xyz="{_f(_unit(rng))}"/>'
                   f'{lim}<dynamics damping="{rng.uniform(0.05, 0.5):.9g}"/></joint>')
    out.append(f'<link name="fx">{inertial(float(rng.uniform(0.2, 0.6)))}{cols.get("fx", "")}</link>')
    out.append(f'<joint name="jfx" type="fixed"><parent link="l{fixed_on}"/><child link="fx"/>'
               f'<origin xyz="{_f(rng.uniform(-0.1, 0.1, 3))}" rpy="{_f(rng.uniform(-np.pi, np.pi, 3))}"/></joint>')
    out.append("</robot>")
    return "\n".join(out) + "\n", "fx", f"l{nb}"


def make_robot(tmp_path, seed, nb, topology="chain", *, dof_mode="velocity", gravity=True, K=64, T=12, dt=0.02, substeps=1, u_lim=0.5,
               base_pos=None, base_ori=None, collisions=None, actors=(), obs=None):
    """Write the URDF to `tmp_path`, compile it into a one-robot scene and return (scene, params, state0).  The base pose is a random
    non-identity one unless given; state0 = (q, qd) with q inside the joint limits (a quarter of the range, at most 0.3, from a stop) and
    small random qd.  `collisions` (see robot_urdf) gives links collision geometry and builds the robot actor with collision on;
    `actors` are further actors of the scene and `obs(scene)`, if given, returns the observation items instead of the default ones."""
    text, fixed_link, tip = robot_urdf(seed, nb, topology, collisions)
    fn = f"synth_{topology}{nb}_s{seed}{'_col' if collisions else ''}.urdf"
    with open(os.path.join(str(tmp_path), fn), "w") as f:
        f.write(text)
    rng = np.random.default_rng([seed, nb, TOPOLOGIES.index(topology), 1])
    if base_pos is None:
        base_pos = rng.uniform(-0.5, 0.5, 3).tolist()
    if base_ori is None:
        qb = rng.normal(size=4)
        base_ori = (np.sign(qb[3]) * qb / np.linalg.norm(qb)).tolist()
    actor = ActorWrapper(type="robot", name="synth", urdf_file=fn, fixed=True, init_pos=list(base_pos), init_ori=list(base_ori),
                         dof_mode=dof_mode, gravity=gravity, collision=bool(collisions))
    sc = build_scene([actor] + list(actors), assets_dirs=[str(tmp_path)], substep=dt / substeps)
    assert sc.ndof == nb and (actors or (sc.model.nfree == 0 and sc.model.nshapes == 0))
    names = sc.robot.link_names
    if obs is not None:
        obs = obs(sc)
    else:
        obs = [(OBS_LINK_STATE, names.index("l0")), (OBS_LINK_STATE, names.index(fixed_link)), (OBS_LINK_STATE, names.index(tip)), (OBS_DOF_STATE, 0)]
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.1 * np.eye(sc.nu)).tolist(),
                    u_min=[-u_lim], u_max=[u_lim], lambda_=0.05, sample_null_action=True)
    p = make_params(mc, IsaacGymConfig(dt=dt, substeps=substeps), sc.nu, K, obs)
    m = sc.model
    lo = np.maximum([m.q_lo[i] for i in range(nb)], -2.0)
    hi = np.minimum([m.q_hi[i] for i in range(nb)], 2.0)
    gap = np.minimum(0.3, 0.25 * (hi - lo))
    q0 = rng.uniform(lo + gap, hi - gap)
    qd0 = rng.uniform(-0.3, 0.3, nb)
    state0 = np.concatenate([q0, qd0]).astype(np.float32)
    return sc, p, state0


def depth(model):
    """Bodies on the longest root-to-leaf path."""
    best = 0
    for i in range(model.nb):
        d, j = 0, i
        while j >= 0:
            d, j = d + 1, model.parent[j]
        best = max(best, d)
    return best


def is_chain(model):
    return all(model.parent[i] == i - 1 for i in range(model.nb))
