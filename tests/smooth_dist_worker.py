"""One rank of the two-rank gloo test of Smooth MPPI (test_oracle_smooth_dist.py): a sharded panda plan in mppi_mode smooth on the
checker backend; saves the actions, U and the smooth state of every plan."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
SMOOTH = dict(mppi_mode="smooth", sampling_method="random", filter_u=False, smooth_weight=0.5, du_min=[-1.0], du_max=[1.0])


def plan(K=64, T=12, plans=3):
    """(actions of `plans` plans, U, smooth state) of a panda reach planner in mppi_mode smooth on the checker backend."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    import smooth_oracle as so
    from scenes import panda_cfg
    p = MPPIisaacPlanner(panda_cfg(K=K, T=T, **SMOOTH), PandaReachObjective(), backend=so.SmoothOracleBackend())
    acts = np.stack([p.compute_action(Q0, [0] * 7).numpy() for _ in range(plans)])
    return p, acts


def run(rank, world, port, out_dir):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    p, acts = plan()
    assert p.sim.num_envs == 64 // world and p.k_offset == rank * (64 // world)
    np.save(os.path.join(out_dir, f"act_{rank}.npy"), acts)
    np.save(os.path.join(out_dir, f"U_{rank}.npy"), p.mppi.U.numpy())
    np.save(os.path.join(out_dir, f"state_{rank}.npy"), p.mppi.smooth_state.numpy())
    dist.destroy_process_group()
