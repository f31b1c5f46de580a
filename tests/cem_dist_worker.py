"""One rank of the two-rank gloo test of cross-entropy planning (test_oracle_cem_dist.py): a sharded panda plan in mppi_mode cem with
three iterations per plan and carried elites on the checker backend; saves the actions, U, the CEM state and the global indices of
the elites every update chose."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
CEM = dict(mppi_mode="cem", sampling_method="colored", n_elites=6, keep_elites=0.5, cem_iterations=3)


def _backend():
    import cem_oracle as ce

    class Recording(ce.CemOracleBackend):
        """The CEM checker backend that keeps the global sample indices of the elites of every K4 (best first)."""

        def __init__(self):
            super().__init__()
            self.elite_index = []

        def finalize(self, partials, G, U, action_out, stats):
            rows = partials.detach().cpu().numpy().reshape(G, -1)
            E = int(self.params.n_elites)
            self.elite_index.append([int(rows[g, 2 * e + 1:2 * e + 2].view(np.uint32)[0]) for g, e in ce.merge(rows, E)])
            return super().finalize(partials, G, U, action_out, stats)

    return Recording()


def plan(K=64, T=12, plans=2):
    """(planner, actions of `plans` plans) of a panda reach planner in mppi_mode cem on the checker backend."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from scenes import panda_cfg
    p = MPPIisaacPlanner(panda_cfg(K=K, T=T, **CEM), PandaReachObjective(), backend=_backend())
    acts = np.stack([p.compute_action(Q0, [0] * 7).numpy() for _ in range(plans)])
    return p, acts


def run(rank, world, port, out_dir):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    p, acts = plan()
    Ks = 64 // world
    assert p.sim.num_envs == Ks and p.k_offset == rank * Ks
    n_keep = int(p.mppi.backend.params.n_keep)
    assert n_keep >= 1 and 64 - 3 - (n_keep - 1) >= (world - 1) * Ks       # the carried rows K_total - 3 - e lie in the last shard
    np.save(os.path.join(out_dir, f"act_{rank}.npy"), acts)
    np.save(os.path.join(out_dir, f"U_{rank}.npy"), p.mppi.U.numpy())
    np.save(os.path.join(out_dir, f"state_{rank}.npy"), p.mppi.dist.numpy())
    np.save(os.path.join(out_dir, f"elites_{rank}.npy"), np.array(p.mppi.backend.elite_index, np.int64))
    dist.destroy_process_group()
