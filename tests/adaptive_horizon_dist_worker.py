"""One rank of the 2-GPU horizon-covariance exchange test (run under torch.distributed.run by test_gpu_adaptive_horizon.py): a sharded
panda plan with update_cov, cov_type horizon and update_lambda, CUDA graph on, over the exchange MPPIB_EXCHANGE selects; prints the
action bit patterns and a digest of the dist bits."""
import hashlib
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

rank, local = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))

from mppi_isaac_b200 import MPPIisaacPlanner  # noqa: E402
from mppi_isaac_b200.objectives import PandaReachObjective  # noqa: E402
from scenes import panda_cfg  # noqa: E402

A = np.random.default_rng(3).normal(0, 1.0, (7, 7))
sigma = A @ A.T / 7 + 0.3 * np.eye(7)
sigma = 0.1 * sigma / np.mean(np.diag(sigma))
cfg = panda_cfg(K=4000, T=30, device=f"cuda:{local}", update_cov=True, update_lambda=True, cov_type="horizon",
                noise_sigma=(0.5 * (sigma + sigma.T)).tolist(), eta_u_bound=40.0, eta_l_bound=4.0)
planner = MPPIisaacPlanner(cfg, PandaReachObjective(), use_cuda_graph=True)
q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
for _ in range(6):
    a = planner.compute_action(q0, [0.0] * 7)
torch.cuda.synchronize()
exch = "peer" if planner.mppi._peer_exchange else "nccl"
digest = hashlib.sha256(planner.mppi.dist.cpu().numpy().tobytes()).hexdigest()
bits = [float(v).hex() for v in a.tolist()] + ["|", digest]
print(f"RESULT {exch} {rank} " + " ".join(bits), flush=True)
planner.mppi.close_peers()
dist.destroy_process_group()
