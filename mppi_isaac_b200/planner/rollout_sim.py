"""``RolloutSim`` -- the ``sim`` handle Objectives and priors see.

Drop-in for the Objective-visible surface of ``IsaacGymWrapper``
(``mppiisaac/planner/isaacgym_wrapper.py:83-774``): same constructor arguments, the same named
getters (``:292-356``), ``apply_robot_cmd`` (``:524-572``), ``step`` (``:639-655``), the state
reset / save methods (``:574-619``, ``:662-758``) and the attributes ``env_cfg``, ``num_envs``,
``device``, ``_dof_state``, ``_root_state``, ``_rigid_body_state``, ``_net_contact_force``,
``visualize_link_buffer``, ``_visualize_link_present``.  ``gym.simulate()`` is replaced by the
batched CUDA rollout kernel (``mppib_rollout``); nothing here computes dynamics on the host.

Storage
-------
All K rollouts start from ONE world state, so static data is stored once and handed out as
stride-0 ``expand`` views; what differs per rollout lives in ``obs[R][T][K]`` (k innermost,
written coalesced by the kernel).  A getter returns a strided *view* of those rows:

* step mode (the reference protocol, one ``step()`` per call): shape ``(K, w)``, strides ``(1, T*K)``
* batched mode (whole horizon rolled out by one launch):        shape ``(T*K, w)``, row ``t*K + k``

Every reference Objective is row-wise over dim 0, so the same ``compute_cost`` code serves both
(SURVEY.md section 7, hard part 3).  Which rows the kernel has to write is found by tracing the
Objective once against a recording facade (``trace()``); reading a row that was not traced raises.
"""
from __future__ import annotations

import copy
import math
from typing import List, Optional, Sequence

import numpy as np
import torch

from ..model.blob import (MAX_SLOTS, OBS_CONTACT, OBS_DOF_STATE, OBS_FREE_STATE, OBS_LINK_STATE, MppibParams, Scene, build_scene,
                          make_params, obs_width)
from ..utils.config_store import ActorWrapper, IsaacGymConfig, MPPIConfig, load_actor_cfgs


class ObservationError(KeyError):
    pass


class RolloutSim:
    def __init__(self, cfg: IsaacGymConfig, actors: List[str], init_positions: Optional[List[List[float]]] = None,
                 num_envs: int = 1, viewer: bool = False, device: str = "cuda:0", interactive_goal: bool = True, *,
                 horizon: int = 1, mppi_cfg: Optional[MPPIConfig] = None, conf_dirs: Optional[Sequence[str]] = None,
                 assets_dirs: Optional[Sequence[str]] = None, backend=None, observe="auto", k_offset: int = 0):
        if viewer or getattr(cfg, "viewer", False):
            raise NotImplementedError("the viewer is outside the rollout path (SURVEY.md section 2, row 12)")
        self.cfg = cfg
        self.k_offset = int(k_offset)          # global index of this shard's first rollout (sharded plans)
        self.device = device
        self.num_envs = int(num_envs)
        self.interactive_goal = interactive_goal
        self.viewer = None
        self._conf_dirs, self._assets_dirs = conf_dirs, assets_dirs
        self.env_cfg = load_actor_cfgs(actors, conf_dirs)
        robots = [a for a in self.env_cfg if a.type == "robot"]
        if init_positions is not None:
            assert len(robots) == len(init_positions)          # isaacgym_wrapper.py:103
            for init_pos, actor_cfg in zip(init_positions, robots):
                actor_cfg.init_pos = list(init_pos)
        for i, a in enumerate(self.env_cfg):
            a.handle = i
        self._T = int(horizon)
        self._mppi_cfg = mppi_cfg
        self._observe = observe
        self._obs_items: List[tuple] = []
        self._backend = backend
        self._recording = False
        self.saved_root_state = None
        # what a captured CUDA graph bakes in: `model_epoch` counts changes of the kernel constant block (MppibModel is a
        # by-value kernel parameter) and of the K-indexed buffers; `build_epoch` counts re-creations of the kernel handle
        self.model_epoch = 0
        self.build_epoch = 0
        self.start_sim()

    # ------------------------------------------------------------------------------------------
    # construction (start_sim, isaacgym_wrapper.py:124-236)
    # ------------------------------------------------------------------------------------------
    def start_sim(self):
        self.scene: Scene = build_scene(self.env_cfg, assets_dirs=self._assets_dirs, substep=float(self.cfg.dt) / int(self.cfg.substeps))
        sc = self.scene
        self._visualize_link_present = any(a.visualize_link for a in self.env_cfg)
        self.visualize_link_buffer = []
        dev = self.device
        self.robot_indices = torch.tensor([i for i, a in enumerate(self.env_cfg) if a.type == "robot"], device=dev)
        self.obstacle_indices = torch.tensor(
            [i for i, a in enumerate(self.env_cfg) if a.type in ("sphere", "box") and a.name != "dummy"], device=dev)
        # ONE world state for all K rollouts, kept in a single device buffer [state0 (NS) | root0 (A*13)] so that a
        # world update is one host->device copy from a pinned staging buffer
        dof0 = sc.dof_state0
        ns, na = 2 * sc.ndof, len(self.env_cfg)
        host = np.concatenate([dof0[0::2], dof0[1::2], sc.root_state0.reshape(-1)]).astype(np.float32)
        self._world = torch.from_numpy(host.copy()).to(dev)
        self._state0 = self._world[:ns]                                           # (NS,) [q | qd]
        self._root0 = self._world[ns:].view(na, 13)                               # (A,13)
        self._stage = torch.from_numpy(host.copy())
        if torch.device(dev).type == "cuda":
            self._stage = self._stage.pin_memory()
        self._stage_np = self._stage.numpy()
        self._act_host = None
        if self._visualize_link_present:
            rcfg = self.env_cfg[sc.robot_actor]
            if rcfg.visualize_link not in sc.robot.link_names:
                raise ValueError(f"visualize_link '{rcfg.visualize_link}' is not a link of {rcfg.urdf_file}: {sc.robot.link_names}")
            self._viz_link = sc.robot.link_names.index(rcfg.visualize_link)
            self.robot_rigid_body_viz_idx = sc.body_offset[sc.robot_actor] + self._viz_link
        self._mode = "step"        # "step" | "batched"
        self._t = 0                # slot the next step() writes
        self._slot = 0             # slot holding the current observation (step mode)
        self._have_obs = False
        self._allocate()

    def _default_mppi_cfg(self) -> MPPIConfig:
        nu = self.scene.nu
        return MPPIConfig(num_samples=self.num_envs, horizon=self._T, mppi_mode="simple", sampling_method="random",
                          noise_sigma=np.eye(nu).tolist(), lambda_=1.0)

    def _make_params(self) -> MppibParams:
        mc = self._mppi_cfg if self._mppi_cfg is not None else self._default_mppi_cfg()
        mc = copy.copy(mc)
        mc.horizon = self._T
        mc._k_offset = self.k_offset           # the kernels key per-rollout randomisation and CEM elite indices by the global index
        return make_params(mc, self.cfg, self.scene.nu, self.num_envs, self._obs_items)

    def _allocate(self):
        """(Re)create the kernel handle and the K-indexed buffers for the current obs plan."""
        sc, K, T, dev = self.scene, self.num_envs, self._T, self.device
        if self._observe == "all":
            self._obs_items = ([(OBS_LINK_STATE, l) for l in range(sc.robot.nlinks)] + [(OBS_DOF_STATE, 0)]
                               + [(OBS_FREE_STATE, f) for f in range(sc.model.nfree)] + [(OBS_CONTACT, s) for s in range(sc.model.ncontact_slots)])
        elif self._visualize_link_present and (OBS_LINK_STATE, self._viz_link) not in self._obs_items:
            self._obs_items.append((OBS_LINK_STATE, self._viz_link))
        self._obs_row = {}
        r = 0
        for kind, idx in self._obs_items:
            self._obs_row[(kind, idx)] = r
            r += obs_width(kind, sc.ndof)
        self._R = r
        self.params = self._make_params()
        if self._backend is None:
            from ..backend import CudaBackend
            self._backend = CudaBackend(dev)
        self._backend.create(sc.model, self.params)
        self.model_epoch += 1
        self.build_epoch += 1
        assert self._backend.obs_size() == self._R
        NS = self._backend.state_size()
        self._state = torch.zeros((NS, K), dtype=torch.float32, device=dev)            # (NS,K) step-protocol state
        self._state_stale = True
        self._obs = torch.zeros((max(self._R, 1), T, K), dtype=torch.float32, device=dev)
        self._cmd = torch.zeros((sc.nu, K), dtype=torch.float32, device=dev)
        self._state_is_broadcast = True

    def _sync_step_state(self):
        """(NS,K) step-protocol state <- the broadcast world state (DOF row + initial states of the free bodies)."""
        if self._state_stale:
            nd2 = 2 * self.scene.ndof
            self._state[:nd2].copy_(self._state0[:, None].expand(-1, self.num_envs))
            for actor_idx, f in self.scene.free_actor.items():
                self._state[nd2 + 13 * f: nd2 + 13 * (f + 1)].copy_(self._root0[actor_idx][:, None].expand(-1, self.num_envs))
            self._state_stale = False

    @property
    def backend(self):
        return self._backend

    @property
    def horizon(self) -> int:
        return self._T

    def configure(self, mppi_cfg: MPPIConfig = None, horizon: int = None, num_envs: int = None):
        """Change the plan shape / MPPI parameters (used by MPPIPlanner and update_mppi_params)."""
        if mppi_cfg is not None:
            self._mppi_cfg = mppi_cfg
        if horizon is not None:
            self._T = int(horizon)
        if num_envs is not None:
            self.num_envs = int(num_envs)
        self._allocate()

    # ------------------------------------------------------------------------------------------
    # observation plan
    # ------------------------------------------------------------------------------------------
    def trace(self, fn):
        """Run ``fn(self)`` against dummy rows and record which observations it reads."""
        if self._observe == "all":
            return
        before = list(self._obs_items)
        self._recording = True
        try:
            fn(self)
        finally:
            self._recording = False
        if self._obs_items != before:
            self._allocate()

    def _rows(self, kind: int, idx: int, width: int) -> torch.Tensor:
        """View of `width` observed rows as (N, width): N = K in step mode, T*K in batched mode."""
        key = (kind, idx)
        if self._recording:
            if key not in self._obs_items:
                self._obs_items.append(key)
            n = 2
            out = torch.ones((n, width), dtype=torch.float32, device=self.device)
            if kind in (OBS_LINK_STATE, OBS_FREE_STATE):
                out[:, 3:6] = 0.0   # identity quaternion xyzw
            return out
        if key not in self._obs_row:
            raise ObservationError(
                f"observation {key} was not part of the traced observation plan {self._obs_items}; construct the planner "
                "with observe='all' or call sim.trace(objective.compute_cost) after changing the Objective")
        r0 = self._obs_row[key]
        T, K = self._T, self.num_envs
        if self._mode == "batched":
            return self._obs[r0:r0 + width].view(width, T * K).t()
        if not self._have_obs:
            self._refresh_initial()
        return self._obs[r0:r0 + width, self._slot, :].t()

    def _n(self) -> int:
        if self._recording:
            return 2
        return self._T * self.num_envs if self._mode == "batched" else self.num_envs

    def _refresh_initial(self):
        """Observe the current state into slot 0 (reference: refresh_* right after a reset)."""
        self._sync_step_state()
        self._backend.rollout(None, self._state, self._cmd, 0, 0, self._obs, act_t0=0, root0=self._root0)
        self._have_obs = True
        self._slot = 0

    # ------------------------------------------------------------------------------------------
    # index helpers / getters (isaacgym_wrapper.py:292-356)
    # ------------------------------------------------------------------------------------------
    def _get_actor_index_by_name(self, name: str):
        return [a.name for a in self.env_cfg].index(name)

    def _get_actor_index_by_robot_index(self, robot_idx: int):
        return int(self.robot_indices[robot_idx])

    def _actor_root_rows(self, actor_idx: int) -> torch.Tensor:
        actor_idx = int(actor_idx)
        if actor_idx in self.scene.free_actor:
            return self._rows(OBS_FREE_STATE, self.scene.free_actor[actor_idx], 13)
        if actor_idx == self.scene.robot_actor and self.scene.virtual_dofs:
            return self._rows(OBS_LINK_STATE, 0, 13)          # planar (differential-drive) base: the root link moves
        return self._root0[actor_idx].unsqueeze(0).expand(self._n(), 13)

    def get_actor_position_by_actor_index(self, actor_idx: int):
        return self._actor_root_rows(actor_idx)[:, 0:3]

    def get_actor_position_by_name(self, name: str):
        return self.get_actor_position_by_actor_index(self._get_actor_index_by_name(name))

    def get_actor_position_by_robot_index(self, robot_idx: int):
        return self.get_actor_position_by_actor_index(self._get_actor_index_by_robot_index(robot_idx))

    def get_actor_velocity_by_actor_index(self, idx: int):
        return self._actor_root_rows(idx)[:, 7:10]

    def get_actor_velocity_by_name(self, name: str):
        return self.get_actor_velocity_by_actor_index(self._get_actor_index_by_name(name))

    def get_actor_velocity_by_robot_index(self, robot_idx: int):
        return self.get_actor_velocity_by_actor_index(self._get_actor_index_by_robot_index(robot_idx))

    def get_actor_orientation_by_actor_index(self, idx: int):
        return self._actor_root_rows(idx)[:, 3:7]

    def get_actor_orientation_by_name(self, name: str):
        return self.get_actor_orientation_by_actor_index(self._get_actor_index_by_name(name))

    def get_actor_orientation_by_robot_index(self, robot_idx: int):
        return self.get_actor_orientation_by_actor_index(self._get_actor_index_by_robot_index(robot_idx))

    def find_actor_rigid_body_index(self, actor_idx: int, link_name: str) -> int:
        sc = self.scene
        return sc.body_offset[actor_idx] + sc.body_names[actor_idx].index(link_name)

    def get_rigid_body_by_rigid_body_index(self, rigid_body_idx: int):
        sc = self.scene
        rigid_body_idx = int(rigid_body_idx)
        for a in range(len(self.env_cfg)):
            off, n = sc.body_offset[a], len(sc.body_names[a])
            if off <= rigid_body_idx < off + n:
                if a == sc.robot_actor:
                    return self._rows(OBS_LINK_STATE, rigid_body_idx - off, 13)
                return self._actor_root_rows(a)
        raise IndexError(rigid_body_idx)

    def get_actor_link_by_name(self, actor_name: str, link_name: str):
        actor_idx = self._get_actor_index_by_name(actor_name)
        return self.get_rigid_body_by_rigid_body_index(self.find_actor_rigid_body_index(actor_idx, link_name))

    def get_actor_contact_forces_by_name(self, actor_name: str, link_name: str):
        actor_idx = self._get_actor_index_by_name(actor_name)
        rb = self.find_actor_rigid_body_index(actor_idx, link_name)
        if rb in self.scene.contact_slot:
            return self._rows(OBS_CONTACT, self.scene.contact_slot[rb], 3)
        if rb in self.scene.shape_bodies:
            # the body collides, but the rollout kernel reports no force for it: zeros would silently drop a collision term
            raise ObservationError(
                f"net contact force of '{actor_name}' / '{link_name}': the body has a collision shape but no contact-force slot; "
                f"forces are reported for at most {MAX_SLOTS} bodies (non-robot bodies first, then robot links while slots remain)")
        return torch.zeros((1, 3), dtype=torch.float32, device=self.device).expand(self._n(), 3)     # no collision shape: no force

    def get_dof_state(self):
        return self._dof_state

    @property
    def _dof_state(self):
        """(N, 2*ndof) interleaved q0,qd0,q1,qd1,... (isaacgym_wrapper.py:190-192); the virtual joints of a planar base
        are not DOFs of the reference's robot and are left out."""
        return self._rows(OBS_DOF_STATE, 0, 2 * self.scene.ndof)[:, 2 * self.scene.virtual_dofs:]

    @property
    def _root_state(self):
        """(N, A, 13).  Static actors are stride-0 views of the single world state."""
        rows = [self._actor_root_rows(a) for a in range(len(self.env_cfg))]
        if all(r.stride(0) == 0 for r in rows):
            return self._root0.unsqueeze(0).expand(self._n(), *self._root0.shape)
        return torch.stack(rows, dim=1)

    @property
    def _rigid_body_state(self):
        """(N, B, 13) -- materialised on demand; prefer the named getters."""
        sc = self.scene
        rows = [self.get_rigid_body_by_rigid_body_index(b) for b in range(sc.num_bodies)]
        return torch.stack(rows, dim=1)

    @property
    def _net_contact_force(self):
        sc = self.scene
        out = torch.zeros((self._n(), sc.num_bodies, 3), dtype=torch.float32, device=self.device)
        for rb, slot in sc.contact_slot.items():
            out[:, rb] = self._rows(OBS_CONTACT, slot, 3)
        return out

    @property
    def num_robots(self):
        return len(self.robot_indices)

    @property
    def robot_positions(self):
        return torch.index_select(self._root_state, 1, self.robot_indices)[:, :, 0:3]

    @property
    def robot_velocities(self):
        return torch.index_select(self._root_state, 1, self.robot_indices)[:, :, 7:10]

    @property
    def obstacle_positions(self):
        return torch.index_select(self._root_state, 1, self.obstacle_indices)[:, :, 0:3]

    @property
    def ostacle_velocities(self):      # (sic) reference spelling, isaacgym_wrapper.py:286
        return torch.index_select(self._root_state, 1, self.obstacle_indices)[:, :, 7:10]

    @property
    def visualize_link_pos(self):
        return self._rows(OBS_LINK_STATE, self._viz_link, 13)[:, 0:3]

    # ------------------------------------------------------------------------------------------
    # setters (isaacgym_wrapper.py:366-406)
    # ------------------------------------------------------------------------------------------
    def _as_row(self, v, n):
        return torch.as_tensor(v, dtype=torch.float32, device=self.device).reshape(-1)[:n]

    def set_actor_position_by_actor_index(self, position, actor_idx: int) -> None:
        self._root0[int(actor_idx), 0:3] = self._as_row(position, 3)
        self._root_changed(int(actor_idx))

    def set_actor_position_by_name(self, position, name: str) -> None:
        self.set_actor_position_by_actor_index(position, self._get_actor_index_by_name(name))

    def set_actor_position_by_robot_index(self, position, robot_idx) -> None:
        self.set_actor_position_by_actor_index(position, self._get_actor_index_by_robot_index(robot_idx))

    def set_actor_velocity_by_actor_index(self, velocity, actor_idx: int) -> None:
        self._root0[int(actor_idx), 7:10] = self._as_row(velocity, 3)

    def set_actor_velocity_by_name(self, velocity, name: str) -> None:
        self.set_actor_velocity_by_actor_index(velocity, self._get_actor_index_by_name(name))

    def set_actor_velocity_by_robot_index(self, velocity, robot_idx) -> None:
        self.set_actor_velocity_by_actor_index(velocity, self._get_actor_index_by_robot_index(robot_idx))

    def _root_changed(self, actor_idx: int):
        """A robot base pose lives in the kernel's constant block; push it when it moves."""
        if actor_idx == self.scene.robot_actor:
            self.sync_base_pose()

    def sync_base_pose(self):
        return self._sync_base_pose_from(self._root0[self.scene.robot_actor].detach().cpu())

    def _sync_base_pose_from(self, row, staged=False):
        row = row.numpy() if hasattr(row, "numpy") else row
        m = self.scene.model
        if self.scene.virtual_dofs:
            # planar base: the pose is STATE (virtual joints), only the height of the plane is a kernel constant
            x, y, yaw, vx, vy, wz = self._base_from_root(row)
            nd = self.scene.ndof
            if not staged:                     # the host fast path has already put these into the staged copy
                vals = torch.tensor([x, y, yaw, vx, vy, wz], dtype=torch.float32)
                self._stage[0:3] = vals[0:3]; self._stage[nd:nd + 3] = vals[3:6]
                self._state0[0:3].copy_(vals[0:3].to(self.device)); self._state0[nd:nd + 3].copy_(vals[3:6].to(self.device))
            self._state_stale = True
            if m.base_pos[2] != float(row[2]):
                m.base_pos[2] = float(row[2])
                self._set_model(m)
                return True
            return False
        changed = False
        for i in range(3):
            if m.base_pos[i] != float(row[i]):
                m.base_pos[i] = float(row[i]); changed = True
        for i in range(4):
            if m.base_quat[i] != float(row[3 + i]):
                m.base_quat[i] = float(row[3 + i]); changed = True
        if changed:
            self._set_model(m)
        return changed

    def _set_model(self, m):
        """Push the model block to the handle; planners compare `model_epoch` before replaying a captured graph."""
        self._backend.set_model(m)
        self.model_epoch += 1

    def _base_from_root(self, root_row):
        """(x, y, yaw, vx, vy, wz) of a planar base from a 13-float root state (host tensor / array)."""
        r = [float(v) for v in root_row]
        yaw = math.atan2(2 * (r[6] * r[5] + r[3] * r[4]), 1 - 2 * (r[4] * r[4] + r[5] * r[5]))
        return r[0], r[1], yaw, r[7], r[8], r[12]

    def set_actor_dof_state(self, state):
        """(K, 2*ndof) or (2*ndof,) interleaved DOF state -> per-rollout simulator state (real DOFs; a planar base keeps its pose)."""
        state = torch.as_tensor(state, dtype=torch.float32, device=self.device)
        nd, nv = self.scene.ndof, self.scene.virtual_dofs
        if nv:
            nr = nd - nv
            if not (state.dim() == 1 or state.shape[0] == 1):
                raise NotImplementedError("per-rollout DOF states are not supported for planar-base robots")
            row = state.reshape(-1)
            self._state0[nv:nd].copy_(row[0:2 * nr:2])
            self._state0[nd + nv:2 * nd].copy_(row[1:2 * nr:2])
            self._state_is_broadcast = True
            self._state_stale = True
            self._have_obs = False
            self._t = 0
            return
        if state.dim() == 1 or state.shape[0] == 1:
            row = state.reshape(-1)
            self._state0.copy_(torch.cat([row[0:2 * nd:2], row[1:2 * nd:2]]))   # in place: the pointer is baked into CUDA graphs
            self._state_is_broadcast = True
            self._state_stale = True          # the (NS,K) step-protocol buffer is refreshed lazily
        else:
            self._state[:nd] = state[:, 0:2 * nd:2].t()
            self._state[nd:2 * nd] = state[:, 1:2 * nd:2].t()
            self._state_is_broadcast = False
        self._have_obs = False
        self._t = 0

    def set_dof_velocity_target_tensor(self, u):
        self._cmd.copy_(torch.as_tensor(u, dtype=torch.float32, device=self.device).t())

    def set_dof_actuation_force_tensor(self, u):
        self._cmd.copy_(torch.as_tensor(u, dtype=torch.float32, device=self.device).t())

    # ------------------------------------------------------------------------------------------
    # command + step (isaacgym_wrapper.py:524-572, 639-655)
    # ------------------------------------------------------------------------------------------
    def apply_robot_cmd(self, u_desired):
        """Store the (K, nu) command; the kernel applies the DOF map / diff-drive IK itself."""
        if u_desired.dim() == 1:
            u_desired = u_desired.unsqueeze(0)
        if u_desired.shape[0] == 1 and self.num_envs > 1:
            u_desired = u_desired.expand(self.num_envs, -1)
        us = float(self.params.u_scale)
        self._cmd.copy_(u_desired.t() if us == 1.0 else u_desired.t() / us)   # the kernel multiplies by u_scale

    def step(self):
        """One model step of length dt for all K rollouts (mppib_rollout with nsteps = 1)."""
        self._mode = "step"
        self._sync_step_state()
        t = self._t % self._T
        self._backend.rollout(None, self._state, self._cmd, t, 1, self._obs, act_t0=t, root0=self._root0)
        self._state_is_broadcast = False
        self._have_obs = True
        self._slot = t
        self._t = t + 1
        if self._visualize_link_present:
            self.visualize_link_buffer.append(self.visualize_link_pos.clone())

    def rollout_all(self, actions: torch.Tensor):
        """Whole horizon in ONE launch from the broadcast world state; switches getters to batched views."""
        self._backend.rollout(self._state0, None, actions, 0, self._T, self._obs, act_t0=0, root0=self._root0)
        self.mark_batched()

    def mark_batched(self):
        """Host-side bookkeeping after a whole-horizon rollout (also called after a CUDA-graph replay)."""
        self._mode = "batched"
        self._have_obs = True
        self._t = 0
        if self._visualize_link_present:
            r0 = self._obs_row[(OBS_LINK_STATE, self._viz_link)]
            self.visualize_link_buffer = [self._obs[r0:r0 + 3, t, :].t() for t in range(self._T)]

    def begin_step_mode(self):
        """Re-arm the step protocol from the broadcast world state."""
        self._mode = "step"
        self._state_stale = True
        self._sync_step_state()
        self._state_is_broadcast = True
        self._have_obs = False
        self._t = 0

    # ------------------------------------------------------------------------------------------
    # reset / save (isaacgym_wrapper.py:238-266, 574-619, 662-758)
    # ------------------------------------------------------------------------------------------
    def reset_to_initial_poses(self):
        sc = self.scene
        self._root0.copy_(torch.from_numpy(sc.root_state0).to(self.device))
        dof0 = sc.dof_state0
        self.set_actor_dof_state(torch.from_numpy(dof0))
        self.sync_base_pose()

    def reset_robot_state(self, q, qdot):
        """pybullet-style (q, qdot) -> every rollout (isaacgym_wrapper.py:574-619)."""
        dof_state = []
        q_idx = 0
        for actor in self.env_cfg:
            if actor.type != "robot":
                continue
            n = self.scene.ndof - self.scene.virtual_dofs
            if actor.differential_drive:
                # (x, y, yaw) + remaining joints; the wheel DOFs sit at the back and start at rest (isaacgym_wrapper.py:588-604)
                nw = int(actor.wheel_count)
                n_q = n - (nw - 3)
                actor_q, actor_qdot = list(q[q_idx:q_idx + n_q]), list(qdot[q_idx:q_idx + n_q])
                self.set_state_tensor_by_pos_vel(actor.handle, actor_q[:3], actor_qdot[:3])
                actor_q, actor_qdot = actor_q[3:] + [0.0] * nw, actor_qdot[3:] + [0.0] * nw
                for _q, _qdot in zip(actor_q, actor_qdot):
                    dof_state += [float(_q), float(_qdot)]
                q_idx += n_q
                continue
            actor_q, actor_qdot = q[q_idx:q_idx + n], qdot[q_idx:q_idx + n]
            for _q, _qdot in zip(actor_q, actor_qdot):
                dof_state += [float(_q), float(_qdot)]
            q_idx += n
        if self.scene.virtual_dofs == 0:
            # staged upload: one async H2D copy of [q | qd] instead of a pageable tensor + gather kernels
            nd = self.scene.ndof
            row = np.asarray(dof_state, dtype=np.float32)
            self._stage_np[0:nd] = row[0::2]
            self._stage_np[nd:2 * nd] = row[1::2]
            self._state0.copy_(self._stage[:2 * nd], non_blocking=True)
            self._state_is_broadcast = True
            self._state_stale = True
            self._have_obs = False
            self._t = 0
            return
        self.set_actor_dof_state(torch.tensor(dof_state, dtype=torch.float32))

    def set_world_state(self, dof_state_row: torch.Tensor, root_state: torch.Tensor):
        """(1,2*ndof) + (1,A,13) world snapshot -> all rollouts (mppi_isaac.py:87-99).
        Host tensors go through the pinned staging buffer: one H2D copy, no device->host traffic.
        Returns True when the robot base pose (a kernel constant) changed."""
        dof = torch.as_tensor(dof_state_row).reshape(-1)
        nd = self.scene.ndof
        self.visualize_link_buffer = []
        if root_state is None:                 # unchanged root states: only the DOF row travels
            root = self._stage[2 * nd:].view(-1, 13)
        else:
            root = torch.as_tensor(root_state).reshape(-1, 13)
        if root.device.type != "cpu" or dof.device.type != "cpu":
            self._root0.copy_(root.to(self.device, dtype=torch.float32))
            self.set_actor_dof_state(dof.to(self.device, dtype=torch.float32))
            return self.sync_base_pose()
        return self.set_world_state_host(dof.to(torch.float32).numpy(), None if root_state is None else root.to(torch.float32).reshape(-1).numpy())

    def set_world_state_host(self, dof, root=None):
        """Host fast path of ``set_world_state``: flat float32 numpy arrays (interleaved DOF row, optional A*13 root rows)
        -> pinned staging buffer -> ONE async H2D copy.  ``root=None`` keeps the root states already on the device."""
        nd, nv = self.scene.ndof, self.scene.virtual_dofs
        nr = nd - nv
        st = self._stage_np
        st[nv:nd] = dof[0:2 * nr:2]
        st[nd + nv:2 * nd] = dof[1:2 * nr:2]
        if root is not None:
            st[2 * nd:] = root
        robot_row = st[2 * nd + 13 * self.scene.robot_actor: 2 * nd + 13 * self.scene.robot_actor + 13]
        if nv:
            x, y, yaw, vx, vy, wz = self._base_from_root(robot_row)
            st[0], st[1], st[2], st[nd], st[nd + 1], st[nd + 2] = x, y, yaw, vx, vy, wz
        self.visualize_link_buffer = []
        if root is None:
            self._state0.copy_(self._stage[:2 * nd], non_blocking=True)   # device root states (possibly edited by setters) stay as they are
        else:
            self._world.copy_(self._stage, non_blocking=True)
        self._state_is_broadcast = True
        self._state_stale = True
        self._have_obs = False
        self._t = 0
        return self._sync_base_pose_from(robot_row, staged=True)

    def read_action(self, action: torch.Tensor):
        """Device action -> pinned host buffer (one D2H copy + a stream synchronize); returns a float32 numpy view."""
        if self._act_host is None or self._act_host.shape != action.shape:
            self._act_host = torch.empty(action.shape, dtype=torch.float32, pin_memory=self._stage.is_pinned())
        self._act_host.copy_(action, non_blocking=True)
        if action.is_cuda:
            torch.cuda.current_stream(action.device).synchronize()
        return self._act_host.numpy()

    def save_root_state(self):
        self.saved_root_state = self._root0.clone()

    def get_saved_root_state(self):
        return self.saved_root_state

    def reset_root_state(self):
        if self._visualize_link_present:
            self.visualize_link_buffer = []
        if self.saved_root_state is not None:
            self._root0.copy_(self.saved_root_state)

    def set_root_state_tensor_by_actor_idx(self, state_tensor, idx):
        self._root0[int(idx)] = self._as_row(state_tensor, 13)
        self._root_changed(int(idx))

    def set_state_tensor_by_pos_vel(self, handle, pos, vel):
        """(x, y, yaw) + velocities -> root pose, yaw -> quaternion (isaacgym_wrapper.py:677-693, intent)."""
        yaw = float(pos[2])
        self._root0[handle, 0:2] = self._as_row(pos[:2], 2)
        self._root0[handle, 3:7] = torch.tensor([0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2)], device=self.device)
        self._root0[handle, 7:9] = self._as_row(vel[:2], 2)
        self._root0[handle, 12] = float(vel[2])               # yaw rate (the reference writes vel into the linear slots, :693)
        self._root_changed(int(handle))

    def update_root_state_tensor_by_obstacles(self, obstacles):
        """dict of {position, velocity, size} -> actors named sphere<i> (isaacgym_wrapper.py:695-746)."""
        env_cfg_changed = False
        for i, obst in enumerate(list(obstacles.values())):
            name = f"sphere{i}"
            idxs = [j for j, a in enumerate(self.env_cfg) if a.name == name]
            if not idxs:
                self.env_cfg.append(ActorWrapper(type="sphere", name=name, handle=None, size=list(obst["size"]), fixed=True))
                env_cfg_changed = True
                continue
            j = idxs[0]
            if list(obst["size"]) != list(self.env_cfg[j].size):
                self.env_cfg[j].size = list(obst["size"])
                env_cfg_changed = True
            self._root0[j] = torch.tensor([*obst["position"], 0, 0, 0, 1, *obst["velocity"], 0, 0, 0], dtype=torch.float32, device=self.device)
        if env_cfg_changed:
            keep = self._root0.clone()
            for i, a in enumerate(self.env_cfg):
                a.handle = i
            self.stop_sim()
            self.start_sim()           # new kernel handle, new buffers (build_epoch / model_epoch tell the planner)
            n = min(keep.shape[0], self._root0.shape[0])
            self._root0[:n] = keep[:n]
            for i, obst in enumerate(list(obstacles.values())):     # rows of the obstacles that were just created
                j = [a.name for a in self.env_cfg].index(f"sphere{i}")
                self._root0[j] = torch.tensor([*obst["position"], 0, 0, 0, 1, *obst["velocity"], 0, 0, 0], dtype=torch.float32, device=self.device)
            self._stage[2 * self.scene.ndof:].copy_(self._root0.reshape(-1).cpu())
        return env_cfg_changed

    def update_root_state_tensor_by_obstacles_tensor(self, obst_tensor):
        for o_tensor in obst_tensor:
            obst_idx = [i for i, a in enumerate(self.env_cfg) if a.type != "robot" and not a.fixed][0]
            self._root0[obst_idx] = self._as_row(o_tensor, 13)

    def stop_sim(self):
        self._backend.destroy()

    def add_to_envs(self, additions):
        for a in additions:
            self.env_cfg.append(ActorWrapper(**a))
        for i, a in enumerate(self.env_cfg):
            a.handle = i
        self.stop_sim()
        self.start_sim()

    # viewer-only entry points keep their names as no-ops (SURVEY.md 8(a) W9)
    def draw_lines(self, lines, env_idx=0):
        return None

    def interactive_goal_update(self):
        return None

    def initialize_keyboard_listeners(self):
        return None
