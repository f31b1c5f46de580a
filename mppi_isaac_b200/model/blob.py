"""ctypes mirror of ``include/mppib.h`` (MppibModel / MppibParams) and the scene builder.

``build_scene`` does the host-side job of ``IsaacGymWrapper.start_sim`` /
``_create_actor`` (``mppiisaac/planner/isaacgym_wrapper.py:124-236,429-508``) and
``load_asset`` (``mppiisaac/utils/isaacgym_utils.py:14-58``) for the rollout path: it turns
the actor list into one constant block -- the articulated robot, the free rigid bodies,
the static shapes, drive gains and the command map of ``apply_robot_cmd`` (``:524-572``).
"""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass, field
from typing import Callable, Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from .urdf import RobotModel, compile_urdf, load_compiled, quat_xyzw_to_R, R_to_quat_xyzw

ABI_VERSION = 24
MAX_BODIES, MAX_LINKS, MAX_NU, MAX_OBS, MAX_FREE, MAX_SHAPES = 16, 32, 16, 64, 4, 24
MAX_CONTACTS, MAX_SLOTS = 24, 8
HZ_MAX_N = 256                                  # cov_type horizon: largest T*nu

JOINT_REVOLUTE, JOINT_PRISMATIC = 0, 1
DRIVE_VELOCITY, DRIVE_EFFORT = 0, 1
OBS_LINK_STATE, OBS_DOF_STATE, OBS_FREE_STATE, OBS_CONTACT = 0, 1, 2, 3
SHAPE_BOX, SHAPE_SPHERE = 0, 1
OWNER_STATIC, OWNER_LINK, OWNER_FREE = 0, 1, 2
MODE_SIMPLE, MODE_MEAN, MODE_CEM, MODE_SMOOTH = 0, 1, 2, 3
CEM_MAX_ELITES = 128
MAX_WORLDS = 32                                 # risk-aware MPPI: largest n_worlds
MAX_MODES = 16                                  # multi-modal MPPI: largest n_modes
MAX_ANNEAL = 16                                 # annealed MPPI: largest anneal_iterations
ANNEAL_MIN_SCALE = 2.0 ** -20                   # annealed MPPI: smallest noise scale, so that r = 1 / s^2 stays finite in float32
MAX_SPLINE_DEGREE = 3                           # spline MPPI: largest spline_degree
ESS_GRID, ESS_ROW_FLOATS, ESS_STATE_FLOATS = 65, 196, 197   # ESS-targeted temperature: grid points, shard row, state (include/mppib.h)

f32, i32 = C.c_float, C.c_int32


class MppibModel(C.Structure):
    _fields_ = [
        ("abi_version", i32), ("nb", i32), ("nlinks", i32), ("nu", i32), ("drive_mode", i32),
        ("gravity_on", i32), ("nfree", i32), ("nshapes", i32),
        ("gravity", f32 * 3), ("base_pos", f32 * 3), ("base_quat", f32 * 4),
        ("parent", i32 * MAX_BODIES), ("jtype", i32 * MAX_BODIES),
        ("tree_R", (f32 * 9) * MAX_BODIES), ("tree_p", (f32 * 3) * MAX_BODIES), ("tree_quat", (f32 * 4) * MAX_BODIES),
        ("mass", f32 * MAX_BODIES), ("mcom", (f32 * 3) * MAX_BODIES), ("inertia", (f32 * 6) * MAX_BODIES),
        ("q_lo", f32 * MAX_BODIES), ("q_hi", f32 * MAX_BODIES), ("qd_max", f32 * MAX_BODIES),
        ("effort", f32 * MAX_BODIES), ("damping", f32 * MAX_BODIES), ("kd", f32 * MAX_BODIES),
        ("armature", f32 * MAX_BODIES),
        ("cmd_i0", i32 * MAX_BODIES), ("cmd_i1", i32 * MAX_BODIES),
        ("cmd_c0", f32 * MAX_BODIES), ("cmd_c1", f32 * MAX_BODIES), ("planar_base", i32), ("fwd_axis", f32 * 2),
        ("link_body", i32 * MAX_LINKS), ("link_R", (f32 * 9) * MAX_LINKS), ("link_p", (f32 * 3) * MAX_LINKS), ("link_quat", (f32 * 4) * MAX_LINKS),
        ("free_actor", i32 * MAX_FREE), ("free_mass", f32 * MAX_FREE), ("free_mass_pct", f32 * MAX_FREE),
        ("free_half", (f32 * 3) * MAX_FREE), ("free_gravity", i32 * MAX_FREE), ("free_slot", i32 * MAX_FREE),
        ("shape_type", i32 * MAX_SHAPES), ("shape_owner_kind", i32 * MAX_SHAPES), ("shape_owner", i32 * MAX_SHAPES),
        ("shape_actor", i32 * MAX_SHAPES), ("shape_slot", i32 * MAX_SHAPES),
        ("shape_half", (f32 * 3) * MAX_SHAPES), ("shape_pos", (f32 * 3) * MAX_SHAPES),
        ("shape_quat", (f32 * 4) * MAX_SHAPES), ("shape_friction", f32 * MAX_SHAPES), ("shape_fric_pct", f32 * MAX_SHAPES),
        ("shape_size_sigma", (f32 * 3) * MAX_SHAPES),
        ("ncontact_slots", i32), ("ground_plane", i32), ("ground_friction", f32), ("contact_kp", f32), ("contact_kd", f32),
        ("max_depen", f32), ("ground_margin", f32), ("contact_margin", f32), ("contact_iters", i32), ("nactors", i32), ("max_contacts", i32),
    ]


class MppibObsItem(C.Structure):
    _fields_ = [("kind", i32), ("index", i32)]


class MppibParams(C.Structure):
    _fields_ = [
        ("K", i32), ("T", i32), ("substeps", i32), ("dt", f32), ("mode", i32), ("lambda_", f32),
        ("gamma", f32), ("step_size_mean", f32), ("u_scale", f32), ("sample_null_action", i32),
        ("filter_u", i32),
        ("u_min", f32 * MAX_NU), ("u_max", f32 * MAX_NU), ("u_init", f32 * MAX_NU),
        ("sigma_chol", f32 * (MAX_NU * MAX_NU)), ("sigma_inv", f32 * (MAX_NU * MAX_NU)),
        ("k_offset", C.c_uint32), ("rand_seed", C.c_uint32),
        ("nobs", i32), ("obs", MppibObsItem * MAX_OBS),
        ("update_cov", i32), ("update_lambda", i32), ("eta_u_bound", f32), ("eta_l_bound", f32),
        ("step_size_cov", f32), ("kappa", f32), ("lambda_mult", f32), ("cov_full", i32),
        ("cov_horizon", i32), ("sigma0", f32 * (MAX_NU * MAX_NU)),
        ("n_elites", i32), ("n_keep", i32), ("elite_alpha", f32),
        ("du_min", f32 * MAX_NU), ("du_max", f32 * MAX_NU), ("smooth_weight", f32),
        ("n_worlds", i32), ("risk_tail", i32),
        ("n_modes", i32), ("mode_margin", f32), ("mode_samples", i32),
        ("constraint_mode", i32), ("constraint_tol", f32), ("constraint_lambda", f32), ("constraint_pad", i32),
        ("lambda_ess", i32), ("ess_target", f32),
        ("control_knots", i32), ("spline_degree", i32),
    ]


OBS_WIDTH = {OBS_LINK_STATE: 13, OBS_FREE_STATE: 13, OBS_CONTACT: 3}


def obs_width(kind: int, ndof: int) -> int:
    return 2 * ndof if kind == OBS_DOF_STATE else OBS_WIDTH[kind]


# ----------------------------------------------------------------------------------------
@dataclass
class Scene:
    """Everything the host needs to know about one environment (identical for all K)."""
    model: MppibModel
    robot: RobotModel
    actor_cfgs: list
    actor_names: List[str]
    robot_actor: int                      # index of the (single) robot actor
    body_names: List[List[str]]           # per actor: rigid-body (link) names
    body_offset: List[int]                # per actor: first env-domain rigid-body index
    free_actor: Dict[int, int]            # actor index -> free-body slot
    root_state0: np.ndarray               # (A,13) float32 initial root states
    dof_state0: np.ndarray                # (2*ndof,) interleaved
    contact_slot: Dict[int, int] = field(default_factory=dict)  # env rigid-body index -> slot
    shape_bodies: frozenset = frozenset()  # env rigid-body indices that own a collision shape (slotted or not)
    ndof: int = 0
    nu: int = 0
    virtual_dofs: int = 0                 # leading virtual joints of a planar (differential-drive) base: x, y, yaw

    @property
    def num_bodies(self) -> int:
        return self.body_offset[-1] + len(self.body_names[-1])


def find_urdf(urdf_file: str, assets_dirs: Optional[Sequence[str]] = None) -> Optional[str]:
    dirs = list(assets_dirs or [])
    env = os.environ.get("MPPI_ISAAC_ASSETS")
    if env:
        dirs += env.split(os.pathsep)
    for d in dirs:
        for cand in (os.path.join(d, "urdf", urdf_file), os.path.join(d, urdf_file)):
            if os.path.exists(cand):
                return cand
    return None


def compiled_path(urdf_file: str) -> str:
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    stem = os.path.splitext(urdf_file)[0].replace("/", "__")
    return os.path.join(here, "models_compiled", stem + ".json")


def load_robot(urdf_file: str, fixed: bool, assets_dirs=None) -> RobotModel:
    """Compile from the URDF when an assets tree is available, else use the pre-compiled
    constant block shipped in ``models_compiled/`` (made by ``tools/compile_models.py``)."""
    path = find_urdf(urdf_file, assets_dirs)
    if path is not None:
        return compile_urdf(path, fixed_base=fixed)
    cp = compiled_path(urdf_file)
    if os.path.exists(cp):
        return load_compiled(cp)
    raise FileNotFoundError(
        f"URDF '{urdf_file}' not found (set MPPI_ISAAC_ASSETS or cfg.assets_dirs) and no pre-compiled model at {cp}")


def _set(arr, values):
    for i, v in enumerate(np.asarray(values).reshape(-1)):
        arr[i] = v


def _box_of_collision(col: dict):
    """Collision geometry -> (half extents, centre offset in the geometry frame).  Everything is a box on this path."""
    kind = col["kind"]
    if kind == "box":
        return 0.5 * np.asarray(col["size"], float), np.zeros(3)
    if kind == "sphere":
        return np.full(3, float(col["size"][0])), np.zeros(3)
    if kind == "cylinder":
        r, l = float(col["size"][0]), float(col["size"][1])
        return np.array([r, r, 0.5 * l]), np.zeros(3)
    if kind == "mesh" and "aabb_half" in col:
        return np.asarray(col["aabb_half"], float), np.asarray(col["aabb_center"], float)
    return None, None


def build_scene(actor_cfgs: list, gravity=(0.0, 0.0, -9.8), assets_dirs=None, substep: float = 0.025,
                contact_kp: float = 1.0e5, contact_kd: float = 1.0e3, contact_iters: int = 8) -> Scene:
    robots = [i for i, a in enumerate(actor_cfgs) if a.type == "robot"]
    if len(robots) != 1:
        raise NotImplementedError("exactly one robot actor per environment is supported on this path "
                                  "(the reference's own initial-pose code is single-robot too: isaacgym_wrapper.py:220-229)")
    ra = robots[0]
    rcfg = actor_cfgs[ra]
    planar = not rcfg.fixed
    if planar and not rcfg.differential_drive:
        raise NotImplementedError("floating-base robots are supported as differential-drive bases only (planar reduction)")
    robot = load_robot(rcfg.urdf_file, fixed=not planar, assets_dirs=assets_dirs)
    if rcfg.differential_drive and not (rcfg.left_wheel_joints or rcfg.right_wheel_joints):
        # the reference's jackal.yaml names no wheel joints although apply_robot_cmd needs them (isaacgym_wrapper.py:553-556): take the
        # URDF's own naming (front_left_wheel, rear_right_wheel, ...)
        rcfg.left_wheel_joints = [n for n in robot.dof_names if "wheel" in n and "left" in n]
        rcfg.right_wheel_joints = [n for n in robot.dof_names if "wheel" in n and "right" in n]
    if planar != bool(robot.planar_base):
        raise ValueError(f"compiled model of {rcfg.urdf_file} does not match `fixed: {rcfg.fixed}`")
    if robot.nb > MAX_BODIES or robot.nlinks > MAX_LINKS:
        raise ValueError("robot exceeds MPPIB_MAX_BODIES / MPPIB_MAX_LINKS")

    m = MppibModel()
    m.abi_version = ABI_VERSION
    m.nb, m.nlinks = robot.nb, robot.nlinks
    m.gravity_on = 1 if rcfg.gravity else 0
    _set(m.gravity, gravity)
    if planar:      # the pose lives in the virtual joints (x, y, yaw); only the height of the plane is a constant
        _set(m.base_pos, [0.0, 0.0, float(rcfg.init_pos[2])])
        _set(m.base_quat, [0.0, 0.0, 0.0, 1.0])
    else:
        _set(m.base_pos, rcfg.init_pos)
        _set(m.base_quat, rcfg.init_ori)
    if rcfg.dof_mode == "velocity":
        m.drive_mode, kd, arm = DRIVE_VELOCITY, 600.0, 0.0       # isaacgym_wrapper.py:497-500
    elif rcfg.dof_mode == "effort":
        m.drive_mode, kd, arm = DRIVE_EFFORT, 10.0, 0.0          # :492-496
    elif rcfg.dof_mode == "position":
        raise NotImplementedError("dof_mode 'position' is broken in the reference (isaacgym_wrapper.py:571-572) and not provided")
    else:
        raise ValueError("Invalid dof_mode")                         # :506
    for i in range(robot.nb):
        m.parent[i], m.jtype[i] = robot.parent[i], robot.jtype[i]
        _set(m.tree_R[i], robot.tree_R[i]); _set(m.tree_p[i], robot.tree_p[i])
        _set(m.tree_quat[i], R_to_quat_xyzw(robot.tree_R[i]))
        m.mass[i] = robot.mass[i]
        _set(m.mcom[i], robot.mcom[i])
        I = robot.inertia_o[i]
        _set(m.inertia[i], [I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]])
        m.q_lo[i], m.q_hi[i] = max(robot.q_lo[i], -1e30), min(robot.q_hi[i], 1e30)
        m.qd_max[i], m.effort[i] = min(robot.qd_max[i], 1e30), min(robot.effort[i], 1e30)
        m.damping[i], m.kd[i], m.armature[i] = robot.damping[i], kd, arm
    if planar:
        # wheel traction reduced to drives on the virtual joints: n wheels of radius r with velocity gain kd give a linear
        # gain n kd / r^2 and a yaw gain kd sum(x_i^2) / r^2 (x_i = +-L/2); the reachable force is the friction cone mu m g
        r, L, nw = float(rcfg.wheel_radius), float(rcfg.wheel_base), int(rcfg.wheel_count or 2)
        mtot, mu, g = float(np.sum(robot.mass)), float(rcfg.friction), float(np.linalg.norm(gravity))
        for j, (gain, lim) in enumerate(((nw * kd / r**2, mu * mtot * g), (nw * kd / r**2, mu * mtot * g),
                                         (nw * kd * (L / 2) ** 2 / r**2, mu * mtot * g * L / 2))):
            m.kd[j], m.effort[j], m.damping[j] = gain, lim, 0.0
        wheels = [i for i, n in enumerate(robot.dof_names) if n in (rcfg.left_wheel_joints or []) + (rcfg.right_wheel_joints or [])]
        if not wheels:
            raise NotImplementedError(f"differential-drive robot '{rcfg.name}' names no left_wheel_joints / right_wheel_joints: the command map of "
                                      "isaacgym_wrapper.py:510-522 cannot be built (the reference's jackal.yaml has this gap too)")
        axis = np.asarray(robot.tree_R[wheels[0]])[:, 2]                     # wheel axis in the root-link frame
        fwd = np.cross(axis, [0.0, 0.0, 1.0])                                # a wheel turning +omega about `axis` rolls the base along axis x z
        m.planar_base = 1
        _set(m.fwd_axis, fwd[:2] / np.linalg.norm(fwd[:2]))
    # command map (apply_robot_cmd, isaacgym_wrapper.py:524-559)
    u_idx = 0
    if rcfg.differential_drive:
        r, L = float(rcfg.wheel_radius), float(rcfg.wheel_base)
        u_idx = 2
    for i, name in enumerate(robot.dof_names):
        if planar and i < 3:
            m.cmd_i0[i], m.cmd_c0[i], m.cmd_i1[i], m.cmd_c1[i] = 0, 0.0, 0, 0.0     # targets come from the planar-base rule
            continue
        if rcfg.differential_drive and name in (rcfg.left_wheel_joints or []):
            m.cmd_i0[i], m.cmd_c0[i], m.cmd_i1[i], m.cmd_c1[i] = 0, 1.0 / r, 1, -L / (2 * r)   # _ik :510-522
        elif rcfg.differential_drive and name in (rcfg.right_wheel_joints or []):
            m.cmd_i0[i], m.cmd_c0[i], m.cmd_i1[i], m.cmd_c1[i] = 0, 1.0 / r, 1, L / (2 * r)
        else:
            m.cmd_i0[i], m.cmd_c0[i], m.cmd_i1[i], m.cmd_c1[i] = u_idx, 1.0, 0, 0.0
            u_idx += 1
    m.nu = u_idx
    for l in range(robot.nlinks):
        m.link_body[l] = robot.link_body[l]
        _set(m.link_R[l], robot.link_R[l]); _set(m.link_p[l], robot.link_p[l])
        _set(m.link_quat[l], R_to_quat_xyzw(robot.link_R[l]))

    # rigid-body bookkeeping in the env domain (actor order, links in URDF depth-first order)
    body_names, body_offset, off = [], [], 0
    root0 = np.zeros((len(actor_cfgs), 13), np.float32)
    for ai, a in enumerate(actor_cfgs):
        root0[ai, 0:3] = a.init_pos
        root0[ai, 3:7] = a.init_ori
        names = list(robot.link_names) if ai == ra else [a.type]   # box link is "box" (examples/boxer_push/planner.py:51)
        body_names.append(names)
        body_offset.append(off)
        off += len(names)

    # ---- free bodies, collision boxes, contact slots (replaces _create_actor's shape setup, isaacgym_wrapper.py:429-482)
    free_actor: Dict[int, int] = {}
    contact_slot: Dict[int, int] = {}
    shapes = []          # dicts: kind, owner, actor, half, pos, quat, friction, fric_pct, sigma, body (env rigid body index)
    nfree = 0
    for ai, a in enumerate(actor_cfgs):
        if ai == ra or not a.collision:
            continue
        if a.type not in ("box", "sphere"):
            raise NotImplementedError(f"actor asset of type {a.type} is not yet implemented!")      # isaacgym_utils.py:54-56
        stype = SHAPE_BOX
        if a.type == "sphere":
            # a true sphere primitive (gym.create_sphere(radius = size[0]), isaacgym_utils.py:42-52): one analytic contact against
            # boxes / other spheres.  Only FIXED spheres: the obstacles of compute_action(obst=...), whose pose is re-read from the
            # root state at the start of every plan; like every `fixed: True` actor of the reference (fix_base_link) they are static
            # bodies -- the velocity columns of their root-state row are data for the Objective, not motion.
            if not a.fixed:
                raise NotImplementedError(f"free sphere actor '{a.name}': only fixed sphere obstacles are supported")
            half = np.full(3, float(a.size[0]))
            stype = SHAPE_SPHERE
        else:
            half = 0.5 * np.asarray(a.size, float)[:3]
        sigma = np.asarray(a.noise_sigma_size if a.noise_sigma_size is not None else [0, 0, 0], float).reshape(-1)
        if stype == SHAPE_SPHERE:
            sigma = np.full(3, 2.0 * float(sigma[0]) if sigma.size else 0.0)      # the noise acts on the RADIUS (half extents take sigma / 2)
        else:
            sigma = np.resize(sigma, 3) if sigma.size >= 3 else np.zeros(3)
        sh = dict(stype=stype, kind=OWNER_STATIC, owner=-1, actor=ai, half=half, pos=np.zeros(3), quat=np.array([0, 0, 0, 1.0]),
                  friction=float(a.friction), fric_pct=float(a.noise_percentage_friction), sigma=sigma, body=body_offset[ai])
        if not a.fixed:
            if nfree >= MAX_FREE:
                raise ValueError("too many free rigid bodies (MPPIB_MAX_FREE)")
            f = nfree
            nfree += 1
            free_actor[ai] = f
            m.free_actor[f], m.free_mass[f], m.free_mass_pct[f] = ai, float(a.mass), float(a.noise_percentage_mass)
            _set(m.free_half[f], half)
            m.free_gravity[f] = 1 if a.gravity else 0
            sh.update(kind=OWNER_FREE, owner=f)
        shapes.append(sh)
    have_world = len(shapes) > 0
    if have_world and rcfg.collision:
        for l, cols in enumerate(robot.link_collisions):
            for col in cols:
                half, cen = _box_of_collision(col)
                if half is None:
                    continue
                Rg, pg = np.asarray(col["R"], float), np.asarray(col["p"], float)
                R_bl, p_bl = robot.link_R[l], robot.link_p[l]            # link frame in its owning body's frame
                pos = p_bl + R_bl @ (pg + Rg @ cen)
                shapes.append(dict(stype=SHAPE_SPHERE if col["kind"] == "sphere" else SHAPE_BOX, kind=OWNER_LINK, owner=int(robot.link_body[l]), actor=-1, half=half, pos=pos,
                                   quat=R_to_quat_xyzw(R_bl @ Rg), friction=float(rcfg.friction), fric_pct=0.0, sigma=np.zeros(3),
                                   body=body_offset[ra] + l))
    if len(shapes) > MAX_SHAPES:
        raise ValueError(f"{len(shapes)} collision boxes exceed MPPIB_MAX_SHAPES")
    # contact-force slots: non-robot bodies first, then robot links while slots remain
    for sh in sorted(shapes, key=lambda d: (d["kind"] == OWNER_LINK, d["body"])):
        if sh["body"] not in contact_slot and len(contact_slot) < MAX_SLOTS:
            contact_slot[sh["body"]] = len(contact_slot)
    for si, sh in enumerate(shapes):
        m.shape_type[si], m.shape_owner_kind[si], m.shape_owner[si], m.shape_actor[si] = sh["stype"], sh["kind"], sh["owner"], sh["actor"]
        m.shape_slot[si] = contact_slot.get(sh["body"], -1)
        _set(m.shape_half[si], sh["half"]); _set(m.shape_pos[si], sh["pos"]); _set(m.shape_quat[si], sh["quat"])
        m.shape_friction[si], m.shape_fric_pct[si] = sh["friction"], sh["fric_pct"]
        _set(m.shape_size_sigma[si], sh["sigma"])
        if sh["kind"] == OWNER_FREE:
            m.free_slot[sh["owner"]] = m.shape_slot[si]
    m.nfree, m.nshapes, m.ncontact_slots = nfree, len(shapes), len(contact_slot)
    m.nactors = len(actor_cfgs)
    # contact capacity: as many points as the rollout kernel's shared-memory working set allows -- the library reports the bytes
    # one 32-rollout CTA needs for a model (mppib_rollout_smem_bytes, include/mppib.h); 226 KB of an SM are usable
    if nfree or shapes:
        import ctypes as C
        from ..backend import load_library
        lib = load_library()
        cap = MAX_CONTACTS
        while cap >= 1:
            m.max_contacts = cap
            if lib.mppib_rollout_smem_bytes(C.byref(m)) <= 226 * 1024:
                break
            cap -= 1
        if cap < 12:
            raise NotImplementedError(f"scene too large for one SM's shared memory: {m.nb} bodies, {len(shapes)} collision boxes leave room for "
                                      f"{cap} contact points per rollout (12 needed)")
    else:
        m.max_contacts = MAX_CONTACTS
    m.ground_plane, m.ground_friction = 1, 1.0                        # isaacgym_utils.py:61-68
    m.contact_kp, m.contact_kd, m.contact_iters = contact_kp, contact_kd, contact_iters
    # speculative contacts: a body may not close a gap faster than gap / h (keeps resting contacts alive at large h)
    m.ground_margin = max(0.01, 1.5 * abs(gravity[2]) * substep * substep)
    m.max_depen = 0.25
    m.contact_margin = 0.01                                           # isaacgym_wrapper.py:33 contact_offset

    ndof = robot.nb
    nvirt = 3 if planar else 0
    dof0 = np.zeros(2 * ndof, np.float32)
    if rcfg.init_joint_pose:
        real = np.asarray(rcfg.init_joint_pose, np.float32)[: 2 * (ndof - nvirt)]
        dof0[2 * nvirt: 2 * nvirt + len(real)] = real
    if planar:
        qx, qy, qz, qw = (float(v) for v in rcfg.init_ori)
        dof0[0], dof0[2] = float(rcfg.init_pos[0]), float(rcfg.init_pos[1])
        dof0[4] = math.atan2(2 * (qw * qz + qx * qy), 1 - 2 * (qy * qy + qz * qz))
    return Scene(model=m, robot=robot, actor_cfgs=actor_cfgs, actor_names=[a.name for a in actor_cfgs],
                 robot_actor=ra, body_names=body_names, body_offset=body_offset, free_actor=free_actor,
                 root_state0=root0, dof_state0=dof0, contact_slot=contact_slot, shape_bodies=frozenset(sh["body"] for sh in shapes), ndof=ndof, nu=int(m.nu), virtual_dofs=nvirt)


def _cem_params(p: MppibParams, mppi_cfg, nu: int) -> None:
    """The `mppi_mode: cem` keys (DESIGN.md section 2, "Cross-entropy planning"): E elites, momentum alpha, E_keep = floor(xi E)
    carried elites, I iterations per plan."""
    E = int(getattr(mppi_cfg, "n_elites", 10))
    alpha = float(getattr(mppi_cfg, "elite_momentum", 0.1))
    xi = float(getattr(mppi_cfg, "keep_elites", 0.3))
    iters = int(getattr(mppi_cfg, "cem_iterations", 3))
    k_total = int(mppi_cfg.num_samples)
    if not 1 <= E <= CEM_MAX_ELITES:
        raise ValueError(f"n_elites = {E} must lie in 1 .. {CEM_MAX_ELITES}")
    if not 0.0 <= alpha <= 1.0:
        raise ValueError(f"elite_momentum = {alpha} must lie in [0, 1]")
    if not 0.0 <= xi <= 1.0:
        raise ValueError(f"keep_elites = {xi} must lie in [0, 1]")
    if iters < 1:
        raise ValueError(f"cem_iterations = {iters} must be at least 1")
    keep = int(math.floor(xi * E))
    if E + keep + 2 > k_total:
        raise ValueError(f"mppi_mode: cem needs n_elites + floor(keep_elites * n_elites) + 2 <= num_samples; {E} + {keep} + 2 > {k_total}")
    sigma = np.asarray(mppi_cfg.noise_sigma, np.float64).reshape(nu, nu)
    if np.any(sigma != np.diag(np.diag(sigma))):
        raise ValueError("mppi_mode: cem adapts a diagonal per-step sigma: noise_sigma must be diagonal")
    p.n_elites, p.n_keep, p.elite_alpha = E, keep, alpha


def _smooth_params(p: MppibParams, mppi_cfg, nu: int, bc) -> None:
    """The `mppi_mode: smooth` keys (DESIGN.md section 2, "Smooth MPPI"): the smoothness weight omega and the derivative bounds
    du_min / du_max (length 1 broadcasts, None is unbounded)."""
    w = float(getattr(mppi_cfg, "smooth_weight", 0.0))
    if not (math.isfinite(w) and w >= 0.0):
        raise ValueError(f"smooth_weight = {w} must be finite and >= 0")
    dlo, dhi = bc(getattr(mppi_cfg, "du_min", None), -1e30), bc(getattr(mppi_cfg, "du_max", None), 1e30)
    if len(dlo) != nu or len(dhi) != nu:
        raise ValueError(f"du_min / du_max need 1 or nu = {nu} values, got {len(dlo)} / {len(dhi)}")
    for j in range(nu):
        if not float(np.float32(dlo[j])) <= float(np.float32(dhi[j])):
            raise ValueError(f"du_min[{j}] = {dlo[j]} must not exceed du_max[{j}] = {dhi[j]}")
    if not p.dt > 0.0:
        raise ValueError(f"mppi_mode: smooth integrates the derivative over isaacgym.dt, which must be positive; dt = {p.dt}")
    p.smooth_weight = w
    for j in range(nu):
        p.du_min[j], p.du_max[j] = dlo[j], dhi[j]


def risk_tail(n_worlds: int, alpha: float) -> int:
    """m = ceil(alpha R) in float64: the number of worst worlds whose mean scores a control (1 .. R)."""
    return min(max(int(math.ceil(float(alpha) * int(n_worlds))), 1), int(n_worlds))


def _risk_params(p: MppibParams, mppi_cfg, K_local: int) -> None:
    """The risk-aware MPPI keys (DESIGN.md section 2, "Risk-aware MPPI"): R = n_worlds rollouts per control sample, scored by the mean
    of their m = ceil(cvar_alpha R) largest costs.  n_worlds = 1 leaves the block as it was."""
    R = int(getattr(mppi_cfg, "n_worlds", 1))
    if R == 1:
        return
    alpha = float(getattr(mppi_cfg, "cvar_alpha", 1.0))
    k_total = int(mppi_cfg.num_samples)
    if not (1 <= R <= MAX_WORLDS and R & (R - 1) == 0):
        raise ValueError(f"n_worlds = {R} must be a power of two in 1 .. {MAX_WORLDS}")
    if not (math.isfinite(alpha) and 0.0 < alpha <= 1.0):
        raise ValueError(f"cvar_alpha = {alpha} must lie in (0, 1]")
    if k_total % R != 0 or k_total // R < 2:
        raise ValueError(f"n_worlds = {R} needs num_samples = {k_total} to be a multiple of it with at least two control samples")
    if K_local % R != 0:
        raise ValueError(f"n_worlds = {R}: the shard of {K_local} samples must hold whole groups of worlds")
    p.n_worlds, p.risk_tail = R, risk_tail(R, alpha)


def _modes_params(p: MppibParams, mppi_cfg) -> None:
    """The multi-modal MPPI keys (DESIGN.md section 2, "Multi-modal MPPI"): M = n_modes nominal sequences, each drawn around by its
    block of Kc = K_total / M samples, and the switching margin.  n_modes = 1 leaves the block as it was."""
    M = int(getattr(mppi_cfg, "n_modes", 1))
    margin = float(getattr(mppi_cfg, "mode_switch_margin", 0.0))
    if not 1 <= M <= MAX_MODES:
        raise ValueError(f"n_modes = {M} must lie in 1 .. {MAX_MODES}")
    if not (math.isfinite(margin) and margin >= 0.0):
        raise ValueError(f"mode_switch_margin = {margin} must be finite and >= 0")
    if M == 1:
        return
    k_total = int(mppi_cfg.num_samples)
    if k_total % M != 0 or k_total // M < 32:
        raise ValueError(f"n_modes = {M} needs num_samples = {k_total} to be a multiple of it with at least 32 samples per mode")
    p.n_modes, p.mode_margin, p.mode_samples = M, margin, k_total // M


def anneal_schedule(n_iterations: int, iter_decay: float, horizon_decay: float, T: int):
    """(s, r) float64 (N, T) arrays of annealed MPPI (DESIGN.md section 2, "Annealed MPPI"): s[i][t] = c_i^i c_h^(T-1-t), r = 1 / s^2.
    The caller rounds each once to float32."""
    i = np.arange(int(n_iterations), dtype=np.float64)[:, None]
    t = np.arange(int(T), dtype=np.float64)[None, :]
    s = float(iter_decay) ** i * float(horizon_decay) ** (int(T) - 1 - t)
    return s, 1.0 / (s * s)


def anneal_config(mppi_cfg):
    """(N, c_i, c_h) of the annealed-MPPI keys, defaults (1, 1.0, 1.0): one MPPI iteration at unit noise, today's planner."""
    return (int(getattr(mppi_cfg, "anneal_iterations", 1)), float(getattr(mppi_cfg, "anneal_iter_decay", 1.0)),
            float(getattr(mppi_cfg, "anneal_horizon_decay", 1.0)))


def anneal_on(mppi_cfg) -> bool:
    """True when the annealed-MPPI keys ask for more than today's planner: N > 1 or a decay below 1."""
    n, ci, ch = anneal_config(mppi_cfg)
    return n > 1 or ci < 1.0 or ch < 1.0


def _anneal_params(p: MppibParams, mppi_cfg) -> None:
    """The annealed-MPPI keys (DESIGN.md section 2, "Annealed MPPI").  The schedule itself is a device buffer the planner registers
    (mppib_set_anneal), so the parameter block does not change."""
    n, ci, ch = anneal_config(mppi_cfg)
    if not 1 <= n <= MAX_ANNEAL:
        raise ValueError(f"anneal_iterations = {n} must lie in 1 .. {MAX_ANNEAL}")
    for name, c in (("anneal_iter_decay", ci), ("anneal_horizon_decay", ch)):
        if not (math.isfinite(c) and 0.0 < c <= 1.0):
            raise ValueError(f"{name} = {c} must lie in (0, 1]")
    if not anneal_on(mppi_cfg):
        return
    s, _ = anneal_schedule(n, ci, ch, p.T)
    if s.min() < ANNEAL_MIN_SCALE:
        raise ValueError(f"annealed MPPI: the smallest noise scale c_i^(N-1) c_h^(T-1) = {s.min():.3g} is below 2^-20 (anneal_iterations = {n}, "
                         f"anneal_iter_decay = {ci}, anneal_horizon_decay = {ch}, horizon = {p.T})")


def spline_knot_vector(T: int, P: int, d: int):
    """The clamped uniform knot vector of spline MPPI on [0, T-1] (float64): d+1 zeros, i (T-1) / (P-d) for i = 1 .. P-d-1, d+1 copies
    of T-1.  The interior knots are integers divided once, so they are exact wherever the quotient is."""
    inner = [i * (T - 1) / (P - d) for i in range(1, P - d)]
    return np.array([0.0] * (d + 1) + inner + [float(T - 1)] * (d + 1), np.float64)


def _bspline_row(u, P: int, d: int, x: float):
    """(P,) float64 values N_{p,d}(x) of the B-splines of knot vector u by Cox-de Boor (0/0 = 0); at the right end x = u[-1] the last
    basis function is 1."""
    if x >= u[-1]:
        row = np.zeros(P)
        row[P - 1] = 1.0
        return row
    N = np.array([1.0 if u[i] <= x < u[i + 1] else 0.0 for i in range(len(u) - 1)])
    for k in range(1, d + 1):
        M = np.zeros(len(u) - 1 - k)
        for i in range(len(M)):
            a = (x - u[i]) / (u[i + k] - u[i]) * N[i] if u[i + k] > u[i] else 0.0
            b = (u[i + k + 1] - x) / (u[i + k + 1] - u[i + 1]) * N[i + 1] if u[i + k + 1] > u[i + 1] else 0.0
            M[i] = a + b
        N = M
    return N[:P]


def spline_basis(T: int, P: int, d: int):
    """(B, S, xi) in float64 of spline MPPI (DESIGN.md section 2, "Spline MPPI"): B[T][P] = N_{p,d}(t) at the steps, xi[P] the Greville
    abscissae (u_{p+1} + ... + u_{p+d}) / d, and the shift map S[P][P] with row p = N(xi_p + 1) where xi_p + 1 <= T-1 and NaN otherwise
    (that knot takes u_init)."""
    u = spline_knot_vector(T, P, d)
    B = np.stack([_bspline_row(u, P, d, float(t)) for t in range(T)])
    xi = np.array([u[p + 1:p + d + 1].sum() / d for p in range(P)])
    S = np.full((P, P), np.nan)
    for p in range(P):
        if xi[p] + 1.0 <= T - 1:
            S[p] = _bspline_row(u, P, d, xi[p] + 1.0)
    return B, S, xi


def spline_table(T: int, P: int, d: int, nu: int, theta=None):
    """The float32 spline table of include/mppib.h (mppib_set_spline): rows[T + P][d + 3] of (first, count, weights) over the non-zero
    weights of B's rows, then of the shift rows (count 0: u_init), then U_exec[T][nu] = B theta (zeros without theta), from float64
    rounded once."""
    B, S, _ = spline_basis(T, P, d)
    rows = np.zeros((T + P, d + 3), np.float64)
    for r, w in enumerate(list(B) + list(S)):
        if np.isnan(w).any():
            continue
        nz = np.nonzero(w)[0]
        lo, hi = int(nz[0]), int(nz[-1])
        rows[r, 0], rows[r, 1] = lo, hi - lo + 1
        rows[r, 2:2 + hi - lo + 1] = w[lo:hi + 1]
    ue = np.zeros((T, nu)) if theta is None else B @ np.asarray(theta, np.float64).reshape(P, nu)
    return np.concatenate([rows.reshape(-1), ue.reshape(-1)]).astype(np.float32)


def spline_initial_knots(T: int, P: int, d: int, U_init):
    """(P, nu) float32 knots of a (T, nu) initial sequence: theta_p = U_init at xi_p by linear interpolation of its rows, in float64."""
    _, _, xi = spline_basis(T, P, d)
    U = np.asarray(U_init, np.float64).reshape(T, -1)
    return np.stack([np.interp(xi, np.arange(T, dtype=np.float64), U[:, j]) for j in range(U.shape[1])], axis=1).astype(np.float32)


def _spline_params(p: MppibParams, mppi_cfg) -> None:
    """The `control_knots` / `spline_degree` keys of spline MPPI (DESIGN.md section 2, "Spline MPPI").  P = 0 leaves both fields 0, so the
    block is today's byte for byte."""
    P, d = int(getattr(mppi_cfg, "control_knots", 0)), int(getattr(mppi_cfg, "spline_degree", 1))
    if P < 0:
        raise ValueError(f"control_knots = {P} must be >= 0 (0: off)")
    if P == 0:
        return
    if not 1 <= d <= MAX_SPLINE_DEGREE:
        raise ValueError(f"spline_degree = {d} must be 1, 2 or 3")
    if not d + 1 <= P <= p.T:
        raise ValueError(f"control_knots = {P} must lie in spline_degree + 1 = {d + 1} .. horizon = {p.T}")
    p.control_knots, p.spline_degree = P, d


def constraint_on(mppi_cfg) -> bool:
    """True when the config asks for constrained MPPI (`constraint_mode: feasible_first`)."""
    return str(getattr(mppi_cfg, "constraint_mode", "none")) == "feasible_first"


def _constraint_params(p: MppibParams, mppi_cfg) -> None:
    """The `constraint_mode` / `constraint_tol` / `constraint_lambda` keys of constrained MPPI (DESIGN.md section 2, "Constrained MPPI").
    With the mode "none" the three fields stay 0, so the block is today's byte for byte."""
    mode = str(getattr(mppi_cfg, "constraint_mode", "none"))
    if mode not in ("none", "feasible_first"):
        raise ValueError(f"unknown constraint_mode {mode!r} (none | feasible_first)")
    if mode == "none":
        return
    tol = float(getattr(mppi_cfg, "constraint_tol", 0.0))
    if not (math.isfinite(tol) and tol >= 0.0):
        raise ValueError(f"constraint_tol = {tol} must be finite and >= 0")
    lam_c = getattr(mppi_cfg, "constraint_lambda", None)
    lam_c = float(p.lambda_ if lam_c is None else lam_c)
    if not (math.isfinite(lam_c) and lam_c > 0.0):
        raise ValueError(f"constraint_lambda = {lam_c} must be finite and > 0")
    p.constraint_mode, p.constraint_tol, p.constraint_lambda = 1, tol, lam_c


def ess_on(mppi_cfg) -> bool:
    """True when the config asks for the ESS-targeted temperature (`lambda_mode: ess`)."""
    return str(getattr(mppi_cfg, "lambda_mode", "fixed")) == "ess"


def _ess_params(p: MppibParams, mppi_cfg) -> None:
    """The `lambda_mode` / `ess_target` keys of the ESS-targeted temperature (DESIGN.md section 2, "ESS-targeted temperature").  With
    lambda_mode fixed both fields stay 0, so the block is today's byte for byte."""
    mode = str(getattr(mppi_cfg, "lambda_mode", "fixed"))
    if mode not in ("fixed", "ess"):
        raise ValueError(f"unknown lambda_mode {mode!r} (fixed | ess)")
    if mode == "fixed":
        return
    rho = float(getattr(mppi_cfg, "ess_target", 0.01))
    if not (math.isfinite(rho) and 0.0 < rho <= 1.0):
        raise ValueError(f"ess_target = {rho} must be finite and in (0, 1]")
    p.lambda_ess, p.ess_target = 1, rho


def ess_grid(lambda0: float):
    """(65,) float32 grid temperatures lambda_j = lambda0 2^((j - 32)/4) and (65,) float32 1/lambda_j, each computed in float64 from the
    float32 lambda0 of the parameter block and rounded once: the first 130 floats of the temperature state."""
    lam0 = float(np.float32(lambda0))
    lam = lam0 * 2.0 ** ((np.arange(ESS_GRID, dtype=np.float64) - 32.0) / 4.0)
    return lam.astype(np.float32), (1.0 / lam).astype(np.float32)


class Feature(NamedTuple):
    name: str                                     # how the messages name it
    on: Callable                                  # (params, mppi_cfg or None) -> bool; without a config the block alone decides
    limit: Optional[Tuple[Optional[int], int, str]] = None   # (largest horizon or None, largest rows * nu, the rows: "T" or "control_knots")
    no_prior: Optional[str] = None                # why the planner refuses a prior with it; None: it takes one
    setter: Optional[str] = None                  # the backend method that registers its device state


CEM, SMOOTH, HALTON, COLORED = "mppi_mode: cem", "mppi_mode: smooth", "sampling_method: halton", "sampling_method: colored"
WORLDS, MODES, ANNEALED, KNOTS, CONSTRAINED = "n_worlds > 1", "n_modes > 1", "annealed MPPI", "control_knots > 0", "constraint_mode: feasible_first"
ESS = "lambda_mode: ess"
FEATURES = (
    Feature(CEM, lambda p, c: p.mode == MODE_CEM, (256, 512, "T"), setter="set_distribution"),
    Feature(SMOOTH, lambda p, c: p.mode == MODE_SMOOTH, (256, 512, "T"),
            "the prior row would be an action, the samples are derivatives", "set_smooth_state"),
    Feature(HALTON, lambda p, c: c is not None and str(getattr(c, "sampling_method", "halton")) == "halton"),
    Feature(COLORED, lambda p, c: c is not None and str(getattr(c, "sampling_method", "halton")) == "colored", (256, 512, "T")),
    Feature("update_cov", lambda p, c: bool(p.update_cov), setter="set_distribution"),
    Feature("update_lambda", lambda p, c: bool(p.update_lambda), setter="set_distribution"),
    Feature("cov_type: horizon", lambda p, c: bool(p.cov_horizon)),
    Feature("filter_u", lambda p, c: bool(p.filter_u)),
    Feature(WORLDS, lambda p, c: p.n_worlds > 1, no_prior="the prior row would have to fill a whole group of worlds"),
    Feature(MODES, lambda p, c: p.n_modes > 1, (None, 512, "T"), "the prior row would belong to no mode", "set_distribution"),
    Feature(ANNEALED, lambda p, c: c is not None and anneal_on(c), setter="set_anneal"),
    Feature(KNOTS, lambda p, c: p.control_knots > 0, (256, 512, "control_knots"),
            "the prior row is an action sequence and cannot be written as knots", "set_spline"),
    Feature(CONSTRAINED, lambda p, c: bool(p.constraint_mode), setter="set_constraint"),
    Feature(ESS, lambda p, c: bool(p.lambda_ess), setter="set_temperature"),
)
_CEM_SMOOTH, _ADAPTIVE = (CEM, SMOOTH), ("update_cov", "update_lambda")
K3_SMEM = 224 * 1024                              # the shared memory K3 sizes its ring in (reduce_ws_stages, csrc/reduce.cu)


def feasible_k3_bytes(T: int, nu: int) -> int:
    """Shared memory of constraint_mode's K3 at its smallest ring, two stages next to two warp partials (``WsLayout`` of RULE_FEASIBLE in
    csrc/reduce.cu): a stage holds T*nu control, T cost and T violation rows of 32 samples; the shard row is 4 + T*nu floats.  The
    library refuses the mode where this exceeds K3_SMEM (validate, csrc/api.cu), so a horizon too long for the ring is refused here too."""
    NR = T * nu
    P4 = (4 + NR + 3) & ~3
    floats = max(2 * (NR + 2 * T) * 32, 512 + 4 * P4) + ((NR + 3) & ~3) + ((T + 3) & ~3) + 8 * 32 + 2 * P4 + 8
    return ((floats * 4 + 15) & ~15) + 2 * 8 * 2 + 128
# (features, what each of them excludes, the wording after its name); mode_refusal reports the first that applies.  csrc/api.cu: the same pairs
EXCLUSIONS = (
    ((COLORED,), ("cov_type: horizon",), "excludes cov_type: horizon, whose Sigma_H already models the time correlation"),
    ((CEM,), _ADAPTIVE, "has its own update rule and excludes update_cov and update_lambda"),
    ((CEM,), (HALTON,), "samples with sampling_method random or colored, not halton"),
    ((SMOOTH, KNOTS, CONSTRAINED), _ADAPTIVE, "excludes update_cov and update_lambda"),
    ((SMOOTH,), ("filter_u",), "excludes filter_u: the actions are already smooth, switch filter_u off"),
    ((SMOOTH,), (HALTON,), "samples its derivative with sampling_method random, not halton"),
    ((SMOOTH,), (COLORED,), "samples its derivative with sampling_method random, not colored"),
    ((WORLDS, MODES, KNOTS, CONSTRAINED), _CEM_SMOOTH, "excludes mppi_mode cem and smooth"),
    ((WORLDS,), ("cov_type: horizon",), "excludes cov_type: horizon"),
    ((MODES,), _ADAPTIVE, "excludes update_cov and update_lambda: the adapted distribution belongs to one mean"),
    ((MODES, CONSTRAINED), (WORLDS,), "excludes n_worlds > 1"),
    ((ANNEALED,), (CEM,), "excludes mppi_mode cem, which has its own sigma"),
    ((ANNEALED,), (SMOOTH,), "excludes mppi_mode smooth"),
    ((ANNEALED,), (HALTON,), "excludes sampling_method halton: the library is drawn once, so every iteration would reuse the same directions; use random or colored"),
    ((ANNEALED,), _ADAPTIVE, "excludes update_cov and update_lambda (and so every cov_type)"),
    ((ANNEALED,), (MODES,), "excludes n_modes > 1: the Stein coupling's Sigma^-1 metric would need the schedule"),
    ((KNOTS,), (HALTON,), "samples its knots with sampling_method random, not halton"),
    ((KNOTS,), (COLORED,), "samples its knots with sampling_method random, not colored"),
    ((KNOTS,), (MODES, WORLDS), "excludes n_modes > 1 and n_worlds > 1"),
    ((KNOTS, CONSTRAINED), (ANNEALED,), "excludes annealed MPPI"),
    ((KNOTS,), ("filter_u",), "excludes filter_u: the spline is smooth already, switch filter_u off"),
    ((CONSTRAINED,), (MODES,), "excludes n_modes > 1"),
    ((CONSTRAINED,), (KNOTS,), "excludes control_knots > 0"),
    # the library names the excluded features in its own words (csrc/api.cu kFeatureNames); these texts repeat them, so both sides refuse a
    # block with lambda_mode: ess with the same message
    ((ESS,), ("update_lambda",), "excludes update_lambda (two rules for one temperature)"),
    ((ESS,), ("cov_type: horizon",), "excludes cov_horizon (the shift computes lambda Sigma_H^-1 U before the temperature is known)"),
    ((ESS,), (CEM,), "excludes mode cem (it does not weight the samples with the temperature)"),
    ((ESS,), (SMOOTH,), "excludes mode smooth (it does not weight the samples with the temperature)"),
    ((ESS,), (WORLDS,), "excludes n_worlds > 1"),
    ((ESS,), (MODES,), "excludes n_modes > 1"),
    ((ESS,), (KNOTS,), "excludes control_knots > 0"),
    ((ESS,), (CONSTRAINED,), "excludes constraint_mode"),
    ((ESS,), (ANNEALED,), "excludes annealed MPPI"),
)


def mode_refusal(p: MppibParams, nu: int, mppi_cfg=None, anneal: bool = False) -> Optional[str]:
    """Why the FEATURES a block switches on cannot run together, or None: the first size limit, then the first exclusion.  mppi_cfg adds
    the sampling and annealing keys; anneal=True counts a registered annealing schedule as on."""
    on = [f for f in FEATURES if f.on(p, mppi_cfg) or (anneal and f.name == ANNEALED)]
    for f in on:
        if f.limit:
            t_max, n_max, rows = f.limit
            n = getattr(p, rows) * nu
            if p.T > (t_max or p.T) or n > n_max:
                need = (f"horizon <= {t_max} and " if t_max else "") + ("horizon" if rows == "T" else rows) + f" * nu <= {n_max}"
                return f"{f.name} needs {need}; T = {p.T}, {rows}*nu = {n}"
    if any(f.name == CONSTRAINED for f in on) and feasible_k3_bytes(p.T, nu) > K3_SMEM:
        return (f"{CONSTRAINED} needs two K3 ring stages of (horizon * nu + 2 * horizon) * 32 floats, with their working set, in shared memory "
                f"<= {K3_SMEM} bytes; T = {p.T}, T*nu = {p.T * nu} needs {feasible_k3_bytes(p.T, nu)}")
    names = {f.name for f in on}
    for subjects, group, text in EXCLUSIONS:
        for name in subjects:
            if name in names and names.intersection(group):
                return f"{name} {text}"
    return None


def make_params(mppi_cfg, sim_cfg, nu: int, K_local: int, obs_items: Sequence[tuple]) -> MppibParams:
    """MPPIConfig + IsaacGymConfig -> MppibParams (float32 block for the kernels)."""
    p = MppibParams()
    p.K, p.T = int(K_local), int(mppi_cfg.horizon)
    p.substeps, p.dt = int(sim_cfg.substeps), float(sim_cfg.dt)
    mode = str(mppi_cfg.mppi_mode)
    if mode == "simple":
        p.mode, p.gamma = MODE_SIMPLE, 1.0
    elif mode == "halton-spline":
        p.mode, p.gamma = MODE_MEAN, float(mppi_cfg.rollout_var_discount)
    elif mode == "cem":
        p.mode, p.gamma = MODE_CEM, float(mppi_cfg.rollout_var_discount)
    elif mode == "smooth":
        p.mode, p.gamma = MODE_SMOOTH, 1.0
    else:
        raise ValueError(f"unknown mppi_mode {mode}")
    if not (math.isfinite(p.gamma) and p.gamma >= 0.0):     # gamma = 0 is legal: score only the first step
        raise ValueError(f"rollout_var_discount = {p.gamma} must be finite and >= 0")
    p.lambda_ = float(mppi_cfg.lambda_)
    p.step_size_mean = 0.98
    # adaptive MPPI (DESIGN.md section 2): the two flags and the eta bounds are config keys, the step sizes are constants
    p.update_cov = int(bool(getattr(mppi_cfg, "update_cov", False)))
    p.update_lambda = int(bool(getattr(mppi_cfg, "update_lambda", False)))
    p.eta_u_bound = float(getattr(mppi_cfg, "eta_u_bound", 10.0))
    p.eta_l_bound = float(getattr(mppi_cfg, "eta_l_bound", 5.0))
    p.step_size_cov, p.kappa, p.lambda_mult = 0.7, 0.005, 0.1
    cov_type = str(getattr(mppi_cfg, "cov_type", "diag"))
    if cov_type not in ("diag", "full", "horizon"):
        raise ValueError(f"unknown cov_type {cov_type!r} (diag | full | horizon)")
    if cov_type in ("full", "horizon") and not p.update_cov:
        raise ValueError(f"cov_type: {cov_type} selects the update rule of update_cov and needs update_cov: true")
    p.cov_full = int(cov_type == "full")
    p.cov_horizon = int(cov_type == "horizon")
    if p.cov_horizon and p.T * nu > HZ_MAX_N:
        raise ValueError(f"cov_type: horizon adapts a (T*nu) x (T*nu) covariance with T*nu <= {HZ_MAX_N}; T*nu = {p.T * nu}")
    beta = float(getattr(mppi_cfg, "noise_beta", 2.0))
    if not (math.isfinite(beta) and beta >= 0.0):
        raise ValueError(f"noise_beta = {beta} must be finite and >= 0")
    if p.mode == MODE_CEM:
        _cem_params(p, mppi_cfg, nu)
    p.u_scale = float(mppi_cfg.u_scale)
    p.sample_null_action = int(bool(mppi_cfg.sample_null_action))
    p.filter_u = int(bool(mppi_cfg.filter_u))
    if p.filter_u and p.T < 9:
        raise ValueError("filter_u needs horizon >= 9 (Savitzky-Golay window 9)")
    if nu > MAX_NU:
        raise ValueError("nu exceeds MPPIB_MAX_NU")

    def bc(v, default):
        if v is None:
            return [default] * nu
        v = [float(x) for x in (v if hasattr(v, "__len__") else [v])]
        return v * nu if len(v) == 1 else v          # length-1 bounds broadcast (conf/mppi/panda.yaml:9-10)
    umin, umax = bc(mppi_cfg.u_min, -1e30), bc(mppi_cfg.u_max, 1e30)
    uinit = bc(mppi_cfg.u_init, 0.0)
    sigma = np.asarray(mppi_cfg.noise_sigma, np.float64).reshape(nu, nu)
    if (p.cov_full or p.cov_horizon) and (np.any(sigma != sigma.T) or np.any(np.linalg.eigvalsh(sigma) <= 0)):
        raise ValueError(f"cov_type: {cov_type} needs a symmetric positive-definite noise_sigma")
    chol = np.linalg.cholesky(sigma)
    sinv = np.linalg.inv(sigma)
    for j in range(nu):
        p.u_min[j], p.u_max[j], p.u_init[j] = umin[j], umax[j], uinit[j]
        for i in range(nu):
            p.sigma_chol[j * nu + i] = chol[j, i]
            p.sigma_inv[j * nu + i] = sinv[j, i]
            p.sigma0[j * nu + i] = sigma[j, i]
    if p.mode == MODE_SMOOTH:
        _smooth_params(p, mppi_cfg, nu, bc)
    if len(obs_items) > MAX_OBS:
        raise ValueError("too many observation items")
    p.k_offset = int(getattr(mppi_cfg, "_k_offset", 0))
    _risk_params(p, mppi_cfg, int(K_local))
    _modes_params(p, mppi_cfg)
    _anneal_params(p, mppi_cfg)
    _spline_params(p, mppi_cfg)
    _constraint_params(p, mppi_cfg)
    _ess_params(p, mppi_cfg)
    why = mode_refusal(p, nu, mppi_cfg)
    if why:
        raise ValueError(why)
    p.rand_seed = int(getattr(mppi_cfg, "seed_val", 0)) & 0xFFFFFFFF
    p.nobs = len(obs_items)
    for i, (kind, index) in enumerate(obs_items):
        p.obs[i].kind, p.obs[i].index = int(kind), int(index)
    return p
