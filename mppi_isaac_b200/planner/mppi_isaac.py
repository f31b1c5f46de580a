"""``MPPIisaacPlanner`` -- the drop-in boundary (``mppiisaac/planner/mppi_isaac.py:18-138``).

Same constructor, public methods, attributes and plugin protocols as the reference class:
``MPPIisaacPlanner(cfg, objective, prior=None)``, ``dynamics``, ``running_cost``, ``compute_action``,
``reset_rollout_sim``, ``compute_action_tensor``, ``command``, ``add_to_env``, ``get_rollouts``,
``update_objective``, ``update_weights``, ``update_mppi_params``; ``objective.compute_cost(sim)`` /
``objective.reset()`` / ``prior.compute_command(sim)`` are called exactly as there.  What changed is what
runs underneath: the IsaacGym simulator is replaced by the CUDA rollout kernel behind ``RolloutSim`` and
mppi_torch by the fused sample / reduce / finalize kernels behind ``MPPIPlanner``.

Extra keyword arguments (all optional): ``rollout_mode`` ("auto" | "batched" | "stepwise"),
``use_cuda_graph``, ``observe`` ("auto" traces the Objective, "all" writes every link),
``backend`` (tests inject a checker backend; the product default is the CUDA library), ``process_group``.
Under ``torch.distributed`` with world_size G the K samples are sharded over the ranks (one process per GPU).
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from ..model.blob import constraint_on
from ..utils.transport import FastDecoder, FastEncoder, bytes_to_torch, torch_to_bytes
from .mppi import MPPIPlanner, shard_samples
from .rollout_sim import RolloutSim

torch.set_printoptions(precision=2, sci_mode=False)   # mppi_isaac.py:15


class MPPIisaacPlanner(object):
    def __init__(self, cfg, objective: Callable, prior: Optional[Callable] = None, *, rollout_mode: str = "auto",
                 use_cuda_graph: bool = True, observe: str = "auto", backend=None, process_group=None):
        self.cfg = cfg
        self.objective = objective
        self.done = False
        self._last_root_bytes = None
        self._dec_dof, self._dec_root, self._enc = FastDecoder(), FastDecoder(), FastEncoder()
        self._opts = dict(rollout_mode=rollout_mode, use_cuda_graph=use_cuda_graph, process_group=process_group)

        rank, world = 0, 1
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            rank = torch.distributed.get_rank(process_group)
            world = torch.distributed.get_world_size(process_group)
        self.k_total = int(cfg.mppi.num_samples)
        self.k_local, self.k_offset = shard_samples(self.k_total, rank, world, unit=max(4, int(getattr(cfg.mppi, "n_worlds", 1))))

        self.sim = RolloutSim(
            cfg.isaacgym,
            actors=cfg.actors,
            init_positions=cfg.initial_actor_positions,
            num_envs=self.k_local,
            device=cfg.mppi.device,
            horizon=int(cfg.mppi.horizon),
            mppi_cfg=cfg.mppi,
            conf_dirs=getattr(cfg, "conf_dirs", None) or None,
            assets_dirs=getattr(cfg, "assets_dirs", None) or None,
            backend=backend,
            observe=observe,
            k_offset=self.k_offset,
        )
        self.constrained = constraint_on(cfg.mppi)
        self._check_constraint(objective)
        # which rows does the Objective read?  (one dry run against dummy rows)
        self._trace()

        if prior:
            self.prior = lambda state, t: prior.compute_command(self.sim)
        else:
            self.prior = None
        self._build_mppi()

        # place holder handed to mppi, the real state is the rollout simulator itself (mppi_isaac.py:51-52)
        self.state_place_holder = torch.zeros((self.k_local, self.cfg.nx))

    def _build_mppi(self, keep_U: bool = False):
        old = getattr(self, "mppi", None) if keep_U else None
        self._last_root_bytes = None           # whatever was uploaded belonged to the previous handle / buffers
        self._sim_build = self.sim.build_epoch
        self.mppi = self._make_mppi()
        self._sim_build = self.sim.build_epoch         # MPPIPlanner.__init__ re-configures the sim (one more handle)
        if old is not None and old.U.shape == self.mppi.U.shape:
            # the warm start survives a rebuilt simulator, as in the reference (mppi is not rebuilt there): U, the plan counter (so the
            # random stream continues instead of repeating the draws of plans 0, 1, ...), the adapted distribution, the last executed
            # action of mppi_mode smooth and the mode state of n_modes > 1 -- each where the new planner has it in the same shape
            new = self.mppi.persistent_state()
            for name, t in old.persistent_state().items():
                if name in new and new[name].shape == t.shape:
                    new[name].copy_(t)
            # the annealing schedule is rebuilt from the config, not carried over: a keep_U rebuild starts from the configured decays
            self.mppi.refresh_mean_action()              # spline MPPI: U_exec of the carried knots

    def _check_constraint(self, objective):
        if self.constrained and not callable(getattr(objective, "compute_constraint", None)):
            raise ValueError(f"constraint_mode: feasible_first needs an Objective with compute_constraint(sim) ({type(objective).__name__} has none)")

    def _trace(self):
        """Record which rows the Objective reads: the cost and, with constrained MPPI, the constraint, so the plan observes their union."""
        def observed(sim):
            self.objective.compute_cost(sim)
            if self.constrained:
                self.objective.compute_constraint(sim)
        self.sim.trace(observed)

    def _make_mppi(self):
        return MPPIPlanner(
            self.cfg.mppi,
            self.cfg.nx,
            dynamics=self.dynamics,
            running_cost=self.running_cost,
            prior=self.prior,
            sim=self.sim,
            k_total=self.k_total,
            k_offset=self.k_offset,
            running_constraint=self.running_constraint if self.constrained else None,
            **self._opts,
        )

    def update_objective(self, objective):
        self._check_constraint(objective)
        self.objective = objective
        self._trace()
        self._build_mppi()

    def dynamics(self, _, u, t=None):
        # the state lives in the rollout simulator; `_` and `t` are ignored exactly as in the reference (:57-65)
        self.sim.apply_robot_cmd(u)
        self.sim.step()
        return (self.state_place_holder, u)

    def running_cost(self, _):
        return self.objective.compute_cost(self.sim)

    def running_constraint(self, _):
        return self.objective.compute_constraint(self.sim)

    def compute_action(self, q, qdot, obst=None, obst_tensor=None):
        self.sim.reset_root_state()
        self.sim.reset_robot_state(q, qdot)
        if obst:
            self.sim.update_root_state_tensor_by_obstacles(obst)
            if self.sim.build_epoch != self._sim_build:
                # an obstacle was added / resized: the simulator was rebuilt (stop_sim / start_sim as isaacgym_wrapper.py:743-746),
                # i.e. a new kernel handle, new buffers and scene-default joint states.  Re-trace, re-bind the planner to the new
                # handle (action mirror, captured graph) and re-apply the robot state the caller has just handed over.
                self._trace()
                self._build_mppi(keep_U=True)
                self.sim.reset_robot_state(q, qdot)
        if obst_tensor is not None and len(obst_tensor) > 0:
            self.sim.update_root_state_tensor_by_obstacles_tensor(obst_tensor)
        self.sim.save_root_state()
        actions = self.mppi.command(self.state_place_holder)
        if self.mppi.u_per_command == 1 and actions.is_cuda:
            return torch.from_numpy(self.mppi.action_on_host().copy())       # K4 already stored it into pinned host memory
        return actions.cpu()

    def reset_rollout_sim(self, dof_state_tensor, root_state_tensor, rigid_body_state_tensor=None):
        self.sim.visualize_link_buffer = []
        if any(isinstance(t, torch.Tensor) and t.is_cuda for t in (dof_state_tensor, root_state_tensor)):
            changed = self.sim.set_world_state(bytes_to_torch(dof_state_tensor), bytes_to_torch(root_state_tensor))   # in-process device tensors
        else:
            # torch.load costs ~0.1 ms per tensor: the payload is read in place (transport.FastDecoder), and a root-state
            # message identical to the previous one (static scene, fixed base) is neither parsed nor uploaded again
            root = None
            if not (isinstance(root_state_tensor, (bytes, bytearray)) and root_state_tensor == self._last_root_bytes):
                root, _ = self._dec_root(root_state_tensor)
                self._last_root_bytes = bytes(root_state_tensor) if isinstance(root_state_tensor, (bytes, bytearray)) else None
            dof, _ = self._dec_dof(dof_state_tensor)
            changed = self.sim.set_world_state_host(dof, root)
        if changed:
            self.mppi.invalidate_graph()       # the robot base pose is a kernel constant

    def compute_action_tensor(self, dof_state_tensor, root_state_tensor):
        self.objective.reset()
        self.reset_rollout_sim(dof_state_tensor, root_state_tensor)
        return self.command()

    def command(self):
        action = self.mppi.command(self.state_place_holder)
        # same bytes as torch_to_bytes(action) (a pickled tensor on the planner's device): one D2H copy into pinned
        # memory, then payload + CRC patched into the cached archive (transport.FastEncoder)
        host = self.mppi.action_on_host() if self.mppi.u_per_command == 1 else self.sim.read_action(action)
        return self._enc(action, host)

    def add_to_env(self, env_cfg_additions):
        self.sim.add_to_envs(env_cfg_additions)
        self._trace()
        self._build_mppi(keep_U=True)

    def get_rollouts(self):
        if not self.sim._visualize_link_present:
            return torch_to_bytes(torch.zeros((1, 1, 1)))
        return torch_to_bytes(torch.stack(self.sim.visualize_link_buffer))

    def update_weights(self, weights):
        self.objective.weights = weights
        self.mppi.invalidate_graph()           # weights are python floats baked into a captured graph

    def update_mppi_params(self, params):
        self.cfg.mppi.noise_sigma = params["noise_sigma"]
        self._build_mppi()                     # reference rebuilds MPPIPlanner (and so resets U and, mppi_mode smooth, a_prev), :129-138
