"""One rank of the peer-window test of constrained MPPI (test_gpu_constraint_peer.py).

Every rank owns a handle for its shard of K_TOTAL samples, a registered violation buffer and a peer window sized for the constrained row
4 + T*nu.  A plan is the shift, the Gaussian K1, a synthetic cost and margin of the actions, K3 into every rank's window and K4 from the
window; the host puts a barrier between K3 and the K4 that reads its rows, so several processes can share one device.  The margin is
feasible only for global samples in [lo, hi), so a case decides which ranks hold feasible samples.  Each rank saves U, the action, the
constraint state and the gathered rows after every plan to ``<out>/<rank>.npz``; ``plan`` runs the same plans on one handle."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (HERE, os.path.dirname(HERE)):
    if _p not in sys.path:
        sys.path.insert(0, _p)

T, NU, K_TOTAL, PLANS = 12, 3, 1024, 3
CASES = {"first": (0, 300), "last": (800, 1024), "none": (0, 0), "all": (0, 1024)}


def params(K, k_offset):
    from mppi_isaac_b200.model.blob import make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    mc = MPPIConfig(num_samples=K_TOTAL, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.2 * np.eye(NU)).tolist(),
                    u_min=[-0.5], u_max=[0.5], lambda_=0.1, sample_null_action=True, filter_u=True, constraint_mode="feasible_first",
                    constraint_tol=0.0, constraint_lambda=0.3)
    p = make_params(mc, IsaacGymConfig(), NU, K, [])
    p.k_offset = k_offset
    return p


def cost_and_margin(actions, k_offset, case):
    """A synthetic running cost [T][K] of the actions [T][nu][K] and a margin [T][K]: <= 0 for global samples in the case's range,
    0.05 + |a_0| (so the violation depends on the sample) elsewhere."""
    import torch
    tgt = torch.linspace(-0.3, 0.3, T * NU, device=actions.device).view(T, NU, 1)
    cost = ((actions - tgt) ** 2).sum(1).contiguous()
    lo, hi = CASES[case]
    kg = k_offset + torch.arange(actions.shape[-1], device=actions.device)
    feas = ((kg >= lo) & (kg < hi)).view(1, -1)
    g = torch.where(feas, -actions[:, 0, :].abs(), 0.05 + actions[:, 0, :].abs()).contiguous()
    return cost, g


def plan(device, K, k_offset, case, exchange=None, world=1):
    """(U, action, cstate) after each of PLANS constrained plans of the shard [k_offset, k_offset + K); `exchange` runs between K3 and K4."""
    import torch
    from mppi_isaac_b200.backend import CudaBackend
    from synth_mppi import nu_model
    be = CudaBackend(device)
    be.create(nu_model(NU), params(K, k_offset))
    viol, cstate = torch.zeros((T, K), device=device), torch.zeros(2, device=device)
    be.set_constraint(viol, cstate)
    if exchange is not None:
        exchange("open", be)
    U = torch.zeros((T, NU), device=device)
    a, x = torch.zeros((T, NU, K), device=device), torch.zeros((T, NU, K), device=device)
    part, act, st = torch.zeros(4 + T * NU, device=device), torch.zeros(NU, device=device), torch.zeros(2, device=device)
    ctr = torch.zeros(1, dtype=torch.int32, device=device)
    out, extra = [], []
    for _ in range(PLANS):
        be.shift(U, ctr)
        be.sample(11, 0, k_offset, K_TOTAL, U, None, a, x, ctr)
        cost, g = cost_and_margin(a, k_offset, case)
        viol.copy_(g)
        Ubefore = U.clone()
        be.reduce(cost, x, U, part)
        if exchange is None:
            be.finalize(part.view(1, -1), 1, U, act, st)
        else:
            exchange("barrier", be)
            rows = exchange("gather", part)                                   # every rank's row, for the explicit-row K4
            U2 = U.clone()
            be.finalize(rows, world, U2, torch.zeros(NU, device=device), torch.zeros(2, device=device))
            torch.cuda.synchronize(device)
            extra.append((rows.cpu().numpy(), U2.cpu().numpy(), Ubefore.cpu().numpy()))
            be.finalize(None, world, U, act, st)
        torch.cuda.synchronize(device)
        out.append((U.cpu().numpy().copy(), act.cpu().numpy().copy(), cstate.cpu().numpy().copy()))
    if exchange is not None:
        exchange("close", be)
    be.destroy()
    return (out, extra) if exchange is not None else out


def run(rank, world, store, out_dir, case):
    os.environ["MPPIB_PEER_TIMEOUT_S"] = "10"
    import torch
    import torch.distributed as dist
    from mppi_isaac_b200.planner.mppi import shard_samples
    dist.init_process_group("gloo", init_method="file://" + store, rank=rank, world_size=world)
    device = f"cuda:{rank % torch.cuda.device_count()}"
    torch.cuda.set_device(device)

    def exchange(what, be):
        if what == "gather":
            got = [torch.zeros(be.numel()) for _ in range(world)]
            dist.all_gather(got, be.cpu())
            return torch.stack(got).to(device)
        if what == "open":
            hs = [None] * world
            dist.all_gather_object(hs, be.peer_alloc(world, rank))
            for g in range(world):
                if g != rank:
                    be.peer_open(g, hs[g])
        elif what == "close":
            torch.cuda.synchronize(device)
            dist.barrier()
            be.peer_close()
        torch.cuda.synchronize(device)
        dist.barrier()

    K, off = shard_samples(K_TOTAL, rank, world)
    out, extra = plan(device, K, off, case, exchange, world)
    np.savez(os.path.join(out_dir, f"{rank}.npz"), U=np.stack([o[0] for o in out]), act=np.stack([o[1] for o in out]),
             cst=np.stack([o[2] for o in out]), rows=np.stack([e[0] for e in extra]), U_rows=np.stack([e[1] for e in extra]),
             U_before=np.stack([e[2] for e in extra]))
    dist.barrier()
    dist.destroy_process_group()
