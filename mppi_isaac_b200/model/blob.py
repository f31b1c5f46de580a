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
from typing import Dict, List, Optional, Sequence

import numpy as np

from .urdf import RobotModel, compile_urdf, load_compiled, quat_xyzw_to_R, R_to_quat_xyzw

ABI_VERSION = 15
MAX_BODIES, MAX_LINKS, MAX_NU, MAX_OBS, MAX_FREE, MAX_SHAPES = 16, 32, 16, 64, 4, 24
MAX_CONTACTS, MAX_SLOTS = 24, 8

JOINT_REVOLUTE, JOINT_PRISMATIC = 0, 1
DRIVE_VELOCITY, DRIVE_EFFORT = 0, 1
OBS_LINK_STATE, OBS_DOF_STATE, OBS_FREE_STATE, OBS_CONTACT = 0, 1, 2, 3
SHAPE_BOX, SHAPE_SPHERE = 0, 1
OWNER_STATIC, OWNER_LINK, OWNER_FREE = 0, 1, 2
MODE_SIMPLE, MODE_MEAN = 0, 1

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
                 root_state0=root0, dof_state0=dof0, contact_slot=contact_slot, ndof=ndof, nu=int(m.nu), virtual_dofs=nvirt)


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
    if cov_type not in ("diag", "full"):
        raise ValueError(f"unknown cov_type {cov_type!r} (diag | full)")
    if cov_type == "full" and not p.update_cov:
        raise ValueError("cov_type: full selects the update rule of update_cov and needs update_cov: true")
    p.cov_full = int(cov_type == "full")
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
    if p.cov_full and (np.any(sigma != sigma.T) or np.any(np.linalg.eigvalsh(sigma) <= 0)):
        raise ValueError("cov_type: full needs a symmetric positive-definite noise_sigma")
    chol = np.linalg.cholesky(sigma)
    sinv = np.linalg.inv(sigma)
    for j in range(nu):
        p.u_min[j], p.u_max[j], p.u_init[j] = umin[j], umax[j], uinit[j]
        for i in range(nu):
            p.sigma_chol[j * nu + i] = chol[j, i]
            p.sigma_inv[j * nu + i] = sinv[j, i]
    if len(obs_items) > MAX_OBS:
        raise ValueError("too many observation items")
    p.k_offset = int(getattr(mppi_cfg, "_k_offset", 0))
    p.rand_seed = int(getattr(mppi_cfg, "seed_val", 0)) & 0xFFFFFFFF
    p.nobs = len(obs_items)
    for i, (kind, index) in enumerate(obs_items):
        p.obs[i].kind, p.obs[i].index = int(kind), int(index)
    return p
