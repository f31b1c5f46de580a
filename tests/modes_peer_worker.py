"""One rank of the peer-window test of multi-modal MPPI (test_gpu_modes_peer.py).

Every rank owns a handle for its shard (uneven shards whose boundaries fall inside modes) and a peer window sized for the row
[M][2 + T*nu]; K3 stores its row into every rank's window and release-stores one flag per rank, K4 with partials = NULL acquires its
flags and reads the M blocks of every rank back at the window's stride pcap.  Several processes share one device through CUDA IPC, and
the host orders every step: all ranks finish K3 and meet at a barrier before any rank launches K4, so no K4 waits for a flag of a
context that has not run yet.  Each rank pickles one record per exchange (its shard row, U and the mode state before K4, every K4
output) to ``<out>/<case>_<rank>.pkl``.
"""
import os
import pickle
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (HERE, os.path.dirname(HERE)):
    if _p not in sys.path:
        sys.path.insert(0, _p)

# name -> (T, nu, M, Kc, shard offsets [0, ..., M*Kc], exchanges, mppi_mode, filter_u); P = M*(2 + T*nu) and pcap = P rounded up to 4
CASES = {
    "M4-simple-T10nu3-w2": (10, 3, 4, 64, [0, 100, 256], 3, "simple", False),             # P 128
    "M4-mean-filter-T13nu3-w2": (13, 3, 4, 40, [0, 76, 160], 3, "halton-spline", True),   # P 164
    "M16-simple-T7nu3-w4": (7, 3, 16, 32, [0, 100, 236, 376, 512], 3, "simple", False),   # P 368
    "M4-simple-T9nu1-w4": (9, 1, 4, 48, [0, 20, 92, 140, 192], 3, "simple", False),       # P 44
    "M3-simple-T7nu3-w2": (7, 3, 3, 48, [0, 68, 144], 3, "simple", False),               # P 69, pcap 72
    "M5-mean-filter-T9nu1-w4": (9, 1, 5, 32, [0, 36, 76, 120, 160], 3, "halton-spline", True),   # P 55, pcap 56
    "M16-mean-T5nu2-w2": (5, 2, 16, 32, [0, 244, 512], 3, "halton-spline", False),        # P 192
}


def world_of(name):
    return len(CASES[name][4]) - 1


def params(name, rank):
    """The parameter block of rank `rank`'s shard."""
    from mppi_isaac_b200.model.blob import make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    T, nu, M, Kc, offs, _, mode, filt = CASES[name]
    K = offs[rank + 1] - offs[rank]
    mc = MPPIConfig(num_samples=M * Kc, horizon=T, mppi_mode=mode, sampling_method="random", noise_sigma=(0.2 * np.eye(nu) + 0.02).tolist(),
                    u_min=[-0.4], u_max=[0.4], lambda_=0.1, sample_null_action=True, rollout_var_discount=0.9, filter_u=filt, n_modes=M,
                    mode_switch_margin=0.02)
    p = make_params(mc, IsaacGymConfig(), nu, K, [])
    p.k_offset = offs[rank]
    return p


def start(name):
    """(U [M][T][nu], mode state) every rank starts from."""
    T, nu, M = CASES[name][:3]
    U = np.random.default_rng(T * M + nu).uniform(-0.2, 0.2, (M, T, nu)).astype(np.float32)
    return U, np.concatenate([[0.0], np.full(M, np.inf), U[0].ravel()]).astype(np.float32)


def inputs(name, rank, j):
    """(cost [T][K], x [T][nu][K]) of exchange j on this rank: a few costs are +inf, and at j = 1 the last rank has no valid sample."""
    T, nu, M, Kc, offs = CASES[name][:5]
    K = offs[rank + 1] - offs[rank]
    rng = np.random.default_rng(1000 * j + rank + 1)
    cost = rng.uniform(0.0, 1.0, (T, K)).astype(np.float32)
    cost[0] += np.float32(0.05 * rank)
    cost[rng.integers(0, T, 3), rng.integers(0, K, 3)] = np.inf
    if j == 1 and rank == len(offs) - 2:
        cost[:] = np.nan
    x = rng.normal(0.0, 0.2, (T, nu, K)).astype(np.float32)
    return cost, x


def run(rank, world, store, out_dir, names):
    os.environ["MPPIB_PEER_TIMEOUT_S"] = "10"
    import torch
    import torch.distributed as dist
    from mppi_isaac_b200.backend import CudaBackend
    from synth_mppi import nu_model
    dist.init_process_group("gloo", init_method="file://" + store, rank=rank, world_size=world)
    device = f"cuda:{rank % torch.cuda.device_count()}"
    torch.cuda.set_device(device)
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(device)
    host = lambda a: a.detach().cpu().numpy().copy()
    for name in names:
        T, nu, M, _, _, n = CASES[name][:6]
        be = CudaBackend(device)
        be.create(nu_model(nu), params(name, rank))
        U0, st0 = start(name)
        U, st = t(U0), t(st0)
        be.set_distribution(st)
        part = torch.zeros(be.partial_row_floats(), device=device)
        act, stats = torch.zeros(nu, device=device), torch.zeros(2, device=device)
        h = be.peer_alloc(world, rank)
        hs = [None] * world
        dist.all_gather_object(hs, h)
        for g in range(world):
            if g != rank:
                be.peer_open(g, hs[g])
        dist.barrier()
        recs = []
        for j in range(n):
            cost, x = inputs(name, rank, j)
            pre = dict(U0=host(U), st0=host(st))
            be.reduce(t(cost), t(x), U, part)
            torch.cuda.synchronize(device)
            dist.barrier()
            be.finalize(None, world, U, act, stats)
            torch.cuda.synchronize(device)
            recs.append(dict(pre, row=host(part), U=host(U), act=host(act), stats=host(stats), st=host(st)))
            dist.barrier()
        torch.cuda.synchronize(device)
        dist.barrier()
        be.peer_close()
        dist.barrier()
        be.destroy()
        with open(os.path.join(out_dir, f"{name}_{rank}.pkl"), "wb") as f:
            pickle.dump(recs, f)
        dist.barrier()
    dist.destroy_process_group()
