"""Plugin fixtures: the example Objectives of the BASELINE configs, restated.

The reference ships its cost functions inside ``examples/*/planner.py``; they are *user* plugins of the
planner (protocol: ``compute_cost(sim) -> (N,) tensor``, ``reset()``, optional ``weights``), not part of
the library.  They are restated here so the parity tests and ``bench.py`` can drive the drop-in surface
with the same arithmetic:

* ``PandaReachObjective``   <- ``examples/panda/planner.py:22-40``      (O1, config C2)
* ``PointReachObjective``   <- ``examples/heijn_reach/planner.py:15-24`` (O4 template, config C1)
* ``PushObjective``         <- ``examples/{boxer,heijn}_push/planner.py:26-67`` (O2, configs C3 / C4)
* ``PandaPickObjective``    <- ``examples/panda_pick/planner.py:24-53``  (O3, config C5)

Every term is row-wise over dim 0, so the functions work unchanged on the (K, .) step views and the
(T*K, .) batched views of ``RolloutSim``.
"""
import torch

from .ops import _zyx_first_two, pose_cost
from .utils.conversions import matrix_to_euler_angles, quaternion_to_matrix, quaternion_to_yaw


class PandaReachObjective:
    """w_goal * |p_ee - p_goal| + w_ori * |euler_ZYX(R(q_ee))[:2]| for the stick tip."""

    def __init__(self, cfg=None, actor: str = "panda", link: str = "panda_ee_tip", goal: str = "goal", literal: bool = False, fused: bool = True):
        self.weights = {"robot_to_goal": 1.0, "robot_ori": 0.5}
        self.actor, self.link, self.goal = actor, link, goal
        self.literal = literal          # True: the reference's op-by-op formulation (full 3x3 matrix, stack, norm)
        self.fused = fused              # True: both terms in one kernel (ops.pose_cost); False: torch ops, same arithmetic

    def reset(self):
        pass

    def compute_cost(self, sim):
        ee = sim.get_actor_link_by_name(self.actor, self.link)
        goal = sim.get_actor_position_by_name(self.goal)
        if self.fused and not self.literal:
            return pose_cost(ee, goal, self.weights["robot_to_goal"], self.weights["robot_ori"])
        dist = torch.linalg.norm(ee[:, 0:3] - goal[:, 0:3], axis=1)
        if self.literal:
            # the reference hands the xyzw quaternion to a real-first API; reproduced literally (Appendix A #11)
            zyx = matrix_to_euler_angles(quaternion_to_matrix(ee[:, 3:7]), "ZYX")[:, 0:2]
            ori = torch.linalg.norm(zyx, axis=1)
        else:
            ori = _zyx_first_two(ee[:, 3:7])
        return self.weights["robot_to_goal"] * dist + self.weights["robot_ori"] * ori


class PandaReachKeepOutObjective(PandaReachObjective):
    """The panda reach cost with a spherical keep-out region for the tip: ``compute_constraint`` returns the margin
    radius - |p_ee - centre| per row (> 0 inside the sphere), for ``constraint_mode: feasible_first``."""

    def __init__(self, cfg=None, centre=(0.5, 0.0, 0.5), radius: float = 0.1, **kw):
        super().__init__(cfg, **kw)
        self.centre = tuple(float(c) for c in centre)
        self.radius = float(radius)
        self._centre_t = None

    def compute_constraint(self, sim):
        ee = sim.get_actor_link_by_name(self.actor, self.link)
        if self._centre_t is None or self._centre_t.device != ee.device:
            self._centre_t = torch.tensor(self.centre, dtype=torch.float32, device=ee.device)
        return self.radius - torch.linalg.norm(ee[:, 0:3] - self._centre_t, axis=1)


class PointReachObjective:
    """Planar distance of a robot link to the goal actor (+ optional wall contact force)."""

    def __init__(self, cfg=None, actor: str = "point_robot", link: str = "base_link", goal: str = "goal", wall: str = None):
        self.actor, self.link, self.goal, self.wall = actor, link, goal, wall
        self.weights = {}

    def reset(self):
        pass

    def compute_cost(self, sim):
        r = sim.get_actor_link_by_name(actor_name=self.actor, link_name=self.link)
        g = sim.get_actor_position_by_name(self.goal)
        cost = torch.linalg.norm(g[:, 0:2] - r[:, 0:2], axis=1)
        if self.wall is not None:
            f = sim.get_actor_contact_forces_by_name(self.wall, "box")
            cost = cost + torch.sum(torch.abs(f[:, 0:3]), axis=1)
        return cost


class PushObjective:
    """Non-prehensile push cost (2-D): robot-block distance, block-goal distance and yaw, push alignment, block speed and
    the contact force on the two static obstacles.  The alignment term divides by dist*dist without an epsilon, exactly
    as the reference does (SURVEY.md Appendix A #12) -- a 0/0 NaN gives that sample weight 0 in the fused reduction."""

    def __init__(self, cfg=None, robot: str = "heijn", link: str = "front_link", block: str = "block", goal: str = "goal",
                 obstacles=("paper_obst1", "paper_obst2")):
        self.weights = {"robot_to_block": 0.1, "block_to_goal": 2.0, "block_to_goal_ort": 3.0, "push_align": 0.6,
                        "collision": 100, "velocity": 0.0}
        self.goal_yaw = 0.0
        self.robot, self.link, self.block, self.goal, self.obstacles = robot, link, block, goal, tuple(obstacles)

    def reset(self):
        pass

    def compute_cost(self, sim):
        r = sim.get_actor_link_by_name(actor_name=self.robot, link_name=self.link)
        b_pos = sim.get_actor_position_by_name(self.block)
        b_vel = sim.get_actor_velocity_by_name(self.block)
        b_ort = sim.get_actor_orientation_by_name(self.block)
        g_pos = sim.get_actor_position_by_name(self.goal)
        r2b = r[:, 0:2] - b_pos[:, 0:2]
        b2g = g_pos[:, 0:2] - b_pos[:, 0:2]
        r2b_dist = torch.linalg.norm(r2b, axis=1)
        b2g_dist = torch.linalg.norm(b2g, axis=1)
        yaw_err = torch.abs(quaternion_to_yaw(b_ort) - self.goal_yaw)
        align = torch.sum(r2b * b2g, 1) / (r2b_dist * b2g_dist) + 1
        coll = 0.0
        for name in self.obstacles:
            f = sim.get_actor_contact_forces_by_name(actor_name=name, link_name="box")
            coll = coll + torch.sum(torch.abs(f[:, 0:2]), axis=1)
        vel = torch.linalg.norm(b_vel[:, 0:2], axis=1)
        w = self.weights
        return (w["robot_to_block"] * r2b_dist + w["block_to_goal"] * b2g_dist + w["block_to_goal_ort"] * yaw_err
                + w["push_align"] * align + w["velocity"] * vel + w["collision"] * coll)


class PandaPickObjective:
    """40 |ee - block| + 10 |block - goal| + 26 sum|F(table)| + 2 |euler_ZYX(ee)[:2]| for the gripper frame ``panda_ee``."""

    def __init__(self, cfg=None, actor: str = "panda", link: str = "panda_ee", block: str = "panda_pick_block", goal: str = "goal",
                 table: str = "table"):
        self.weights = {"robot_to_block": 40.0, "block_to_goal": 10.0, "collision": 26.0, "robot_ori": 2.0}
        self.actor, self.link, self.block, self.goal, self.table = actor, link, block, goal, table
        self.reset()

    def reset(self):
        self.prev_block_to_goal_dist = 1
        self.prev_robot_to_block_dist = 1

    def compute_cost(self, sim):
        ee = sim.get_actor_link_by_name(self.actor, self.link)
        blk = sim.get_actor_position_by_name(self.block)
        goal = sim.get_actor_position_by_name(self.goal)
        f_table = sim.get_actor_contact_forces_by_name(self.table, "box")
        r2b = torch.linalg.norm(ee[:, 0:3] - blk[:, 0:3], axis=1)
        b2g = torch.linalg.norm(blk[:, 0:3] - goal[:, 0:3], axis=1)
        forces = torch.sum(torch.abs(f_table[:, 0:3]), axis=1)
        w = self.weights
        self.prev_block_to_goal_dist = b2g
        return w["robot_to_block"] * r2b + w["block_to_goal"] * b2g + w["collision"] * forces + w["robot_ori"] * _zyx_first_two(ee[:, 3:7])
