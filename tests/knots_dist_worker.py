"""One rank of the gloo test of spline MPPI (test_oracle_knots_dist.py): a sharded point-robot plan with P = 4 knots of degree 3 on the
checker backend; saves the actions, U and U_exec of every plan."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
Q0 = [0.1, 0.0, 0.0]
KNOTS = dict(control_knots=4, spline_degree=3, sampling_method="random", filter_u=False)


def plan(K=128, T=10, plans=3):
    """(planner, actions, U_exec of `plans` plans) of a point-robot spline planner on the checker backend."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    import knots_oracle as ko
    from scenes import point_cfg
    p = MPPIisaacPlanner(point_cfg(K=K, T=T, **KNOTS), PointReachObjective(), backend=ko.KnotsOracleBackend())
    acts, exe = [], []
    for _ in range(plans):
        acts.append(p.compute_action(Q0, [0] * 3).numpy().copy())
        exe.append(p.mppi.mean_action.numpy().copy())
    return p, np.stack(acts), np.stack(exe)


def run(rank, world, port, out_dir, K):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    p, acts, exe = plan(K)
    from mppi_isaac_b200.planner.mppi import shard_samples
    assert (p.sim.num_envs, p.k_offset) == shard_samples(K, rank, world)
    assert p.mppi.partial.numel() == 2 + 4 * p.mppi.nu                 # the shard row carries the knots, not the steps
    np.save(os.path.join(out_dir, f"act_{rank}.npy"), acts)
    np.save(os.path.join(out_dir, f"exe_{rank}.npy"), exe)
    np.save(os.path.join(out_dir, f"U_{rank}.npy"), p.mppi.U.numpy())
    dist.destroy_process_group()
