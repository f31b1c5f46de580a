"""One rank of the gloo test of multi-modal MPPI (test_oracle_modes_dist.py): a sharded point-robot plan with n_modes = 4 on the checker
backend, with K_total chosen so that every shard boundary falls inside a mode; saves the actions, U and the mode state of every plan."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
Q0 = [0.1, 0.0, 0.0]
MODES = dict(n_modes=4, mode_switch_margin=0.01)


def plan(K=192, T=10, plans=3):
    """(planner, actions, mode states of `plans` plans) of a point-robot planner with n_modes = 4 on the checker backend."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    import modes_oracle as mo
    from scenes import point_cfg
    p = MPPIisaacPlanner(point_cfg(K=K, T=T, **MODES), PointReachObjective(), backend=mo.ModesOracleBackend())
    acts, states = [], []
    for _ in range(plans):
        acts.append(p.compute_action(Q0, [0] * 3).numpy().copy())
        states.append(p.mppi.mode_state.numpy().copy())
    return p, np.stack(acts), np.stack(states)


def run(rank, world, port, out_dir, K):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    p, acts, states = plan(K)
    from mppi_isaac_b200.planner.mppi import shard_samples
    assert (p.sim.num_envs, p.k_offset) == shard_samples(K, rank, world)
    np.save(os.path.join(out_dir, f"act_{rank}.npy"), acts)
    np.save(os.path.join(out_dir, f"state_{rank}.npy"), states)
    np.save(os.path.join(out_dir, f"U_{rank}.npy"), p.mppi.U.numpy())
    dist.destroy_process_group()
