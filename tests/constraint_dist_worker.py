"""One rank of the gloo test of constrained MPPI (test_oracle_constraint_dist.py): a sharded point-robot plan on the checker backend whose
feasible samples lie on the first rank, the second or neither; saves the actions, U and the constraint state of every plan."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
Q0 = [0.1, 0.0, 0.0]
HALF = 68                          # the first rank's samples of K = 136 over two ranks


def margin(case):
    """g of a row from the robot position p and the global sample index kg: feasible on the first half, the second half or nowhere."""
    def fn(p, kg):
        viol = 0.5 + p[:, 0].abs()
        if case == "neither":
            return viol
        feas = kg < HALF if case == "first" else kg >= HALF
        return torch.where(feas, -torch.ones_like(viol), viol)
    return fn


def plan(case, K=136, T=10, plans=3):
    """(planner, actions, (n_feasible, min V) of `plans` plans) of a constrained point-robot planner on the checker backend."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    import constraint_oracle as cn
    from scenes import point_cfg
    from test_oracle_constraint import PointKeepOut
    p = MPPIisaacPlanner(point_cfg(K=K, T=T, sampling_method="random", filter_u=False, constraint_mode="feasible_first"),
                         PointKeepOut(margin(case)), backend=cn.ConstraintOracleBackend())
    acts, cst = [], []
    for _ in range(plans):
        acts.append(p.compute_action(Q0, [0] * 3).numpy().copy())
        cst.append((p.mppi.feasible_samples, float(p.mppi.min_violation)))
    return p, np.stack(acts), np.array(cst)


def run(rank, world, port, out_dir, case):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    p, acts, cst = plan(case)
    assert p.mppi.partial.numel() == 4 + p.mppi.T * p.mppi.nu
    np.save(os.path.join(out_dir, f"act_{rank}.npy"), acts)
    np.save(os.path.join(out_dir, f"U_{rank}.npy"), p.mppi.U.numpy())
    np.save(os.path.join(out_dir, f"cst_{rank}.npy"), cst)
    dist.destroy_process_group()
