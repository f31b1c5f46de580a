"""One rank of the two-rank gloo test of risk-aware MPPI (test_oracle_risk_dist.py): a sharded boxer push plan with n_worlds = 4 on the
checker backend; saves the actions and U of every plan."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
Q0 = [0.0, 2.5, 0.0]
RISK = dict(mppi_mode="simple", sampling_method="random", n_worlds=4, cvar_alpha=0.5)


def plan(K=64, T=10, plans=2):
    """(planner, actions of `plans` plans) of a boxer push planner with n_worlds = 4 on the checker backend."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PushObjective
    import risk_oracle as ro
    from scenes import boxer_cfg
    p = MPPIisaacPlanner(boxer_cfg(K=K, T=T, **RISK), PushObjective(robot="boxer", link="ee_link"), backend=ro.RiskOracleBackend())
    acts = np.stack([p.compute_action(Q0, [0] * 3).numpy() for _ in range(plans)])
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
    dist.destroy_process_group()
