"""One rank of the gloo test of annealed MPPI (test_oracle_anneal_dist.py): a sharded point-robot plan with three iterations per plan on
the checker backend; saves the actions, U and the schedule counter of every plan."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
Q0 = [0.1, 0.0, 0.0]
ANNEAL = dict(anneal_iterations=3, anneal_iter_decay=0.6, anneal_horizon_decay=0.9)


def plan(K=128, T=10, plans=3):
    """(planner, actions, counters of `plans` plans) of a point-robot planner with three annealed iterations on the checker backend."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    import anneal_oracle as ao
    from scenes import point_cfg
    p = MPPIisaacPlanner(point_cfg(K=K, T=T, **ANNEAL), PointReachObjective(), backend=ao.AnnealOracleBackend())
    acts, ctrs = [], []
    for _ in range(plans):
        acts.append(p.compute_action(Q0, [0] * 3).numpy().copy())
        ctrs.append(float(p.mppi.anneal_state[0]))
    return p, np.stack(acts), np.array(ctrs)


def run(rank, world, port, out_dir, K):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    p, acts, ctrs = plan(K)
    from mppi_isaac_b200.planner.mppi import shard_samples
    assert (p.sim.num_envs, p.k_offset) == shard_samples(K, rank, world)
    np.save(os.path.join(out_dir, f"act_{rank}.npy"), acts)
    np.save(os.path.join(out_dir, f"ctr_{rank}.npy"), ctrs)
    np.save(os.path.join(out_dir, f"U_{rank}.npy"), p.mppi.U.numpy())
    dist.destroy_process_group()
