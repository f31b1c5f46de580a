import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, numpy as np
import bench
from mppi_isaac_b200 import MPPIisaacPlanner
K = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
pl = MPPIisaacPlanner(bench.load_cfg("c5", K, "cuda:0"), bench.make_objective("c5"), use_cuda_graph=False)
bench.init_world(pl, "c5")
m, be, sim = pl.mppi, pl.mppi.backend, pl.sim
def step(name, fn):
    fn(); torch.cuda.synchronize(); print("ok", name, flush=True)
step("shift", lambda: be.shift(m.U, m.plan_ctr))
step("sample", lambda: m._sample())
step("rollout", lambda: sim.rollout_all(m.actions))
cost = None
def c():
    global cost
    cost = m._cost_batched()
step("cost", c)
print("cost", cost.shape, cost.dtype, cost.is_contiguous(), cost.data_ptr() % 16, float(cost.max()), flush=True)
from mppi_isaac_b200.model.blob import MODE_SIMPLE
x = m.noise if be.params.mode == MODE_SIMPLE else m.actions
step("reduce", lambda: be.reduce(cost, x, m.U, m.partial))
step("reduce_finalize", lambda: be.reduce_finalize(cost, x, m.U, m.partial, m._action, m.stats))
print(m._action)
