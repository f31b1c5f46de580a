"""One rank of the gloo test of the ESS-targeted temperature (test_oracle_temperature_dist.py): a sharded point-robot plan on the checker
backend, with every sample valid or only the first 40 (all on the first rank); saves the actions, U and the chosen temperatures."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
Q0 = [0.1, 0.0, 0.0]


def objective(case):
    from mppi_isaac_b200.objectives import PointReachObjective

    class Obj(PointReachObjective):
        def compute_cost(self, sim):
            c = super().compute_cost(sim)
            if case == "one_rank":                                  # NaN makes a sample invalid for the temperature and for K3
                kg = sim.k_offset + torch.arange(c.shape[0]) % sim.num_envs
                c = torch.where(kg < 40, c, torch.full_like(c, float("nan")))
            return c
    return Obj()


def plan(case, K=140, T=10, plans=3):
    """(planner, actions, (lambda, valid samples) of `plans` plans) of an ESS point-robot planner on the checker backend."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    import temperature_oracle as tmo
    from scenes import point_cfg
    p = MPPIisaacPlanner(point_cfg(K=K, T=T, sampling_method="random", filter_u=False, lambda_mode="ess", ess_target=0.1),
                         objective(case), backend=tmo.TemperatureOracleBackend())
    acts, lams = [], []
    for _ in range(plans):
        acts.append(p.compute_action(Q0, [0] * 3).numpy().copy())
        lams.append((float(p.mppi.current_lambda), p.mppi.valid_samples))
    return p, np.stack(acts), np.array(lams)


def run(rank, world, port, out_dir, case):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    p, acts, lams = plan(case)
    np.save(os.path.join(out_dir, f"act_{rank}.npy"), acts)
    np.save(os.path.join(out_dir, f"U_{rank}.npy"), p.mppi.U.numpy())
    np.save(os.path.join(out_dir, f"lam_{rank}.npy"), lams)
    np.save(os.path.join(out_dir, f"K_{rank}.npy"), np.array([p.mppi.K]))
    dist.destroy_process_group()
