"""One rank of the peer-window test of the ESS-targeted temperature (test_gpu_temperature_peer.py).

Every rank owns a handle for its shard of K_TOTAL samples (uneven shards), a registered distribution and temperature state, and a peer
window sized for the temperature row.  A plan is the shift, the Gaussian K1, a synthetic cost, the temperature pass with the fused solve
(its row into every rank's window, every rank's row from its own), K3 into every window and K4 from the window -- two exchanges per plan on
one window, over several plans, so both slots are reused by both.  After each plan the rank also gathers the temperature rows over gloo and
runs the explicit-row solve of the same rows.  Each rank saves lambda, the state, U and the rows of every plan to ``<out>/<rank>.npz``."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (HERE, os.path.dirname(HERE)):
    if _p not in sys.path:
        sys.path.insert(0, _p)

T, NU, K_TOTAL, PLANS = 12, 3, 2036, 5


def params(K, k_offset):
    from mppi_isaac_b200.model.blob import make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
    mc = MPPIConfig(num_samples=K_TOTAL, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.2 * np.eye(NU)).tolist(),
                    u_min=[-0.5], u_max=[0.5], lambda_=0.1, sample_null_action=True, filter_u=True, lambda_mode="ess", ess_target=0.05)
    p = make_params(mc, IsaacGymConfig(), NU, K, [])
    p.k_offset = k_offset
    return p


def run(rank, world, store, out_dir):
    os.environ["MPPIB_PEER_TIMEOUT_S"] = "30"
    import torch
    import torch.distributed as dist
    from mppi_isaac_b200.backend import CudaBackend
    from mppi_isaac_b200.model.blob import ESS_GRID, ESS_ROW_FLOATS, ESS_STATE_FLOATS, ess_grid
    from mppi_isaac_b200.planner.mppi import shard_samples
    from synth_mppi import nu_model
    dist.init_process_group("gloo", init_method="file://" + store, rank=rank, world_size=world)
    device = f"cuda:{rank % torch.cuda.device_count()}"
    torch.cuda.set_device(device)
    K, off = shard_samples(K_TOTAL, rank, world)
    p = params(K, off)
    be = CudaBackend(device)
    be.create(nu_model(NU), p)
    dist_buf = torch.tensor([p.lambda_] + [0.04] * NU, dtype=torch.float32, device=device)
    be.set_distribution(dist_buf)
    lam, inv = ess_grid(p.lambda_)
    st = torch.zeros(ESS_STATE_FLOATS)
    st[:ESS_GRID], st[ESS_GRID:2 * ESS_GRID] = torch.from_numpy(lam), torch.from_numpy(inv)
    state = st.to(device)
    be.set_temperature(state)
    hs = [None] * world
    dist.all_gather_object(hs, be.peer_alloc(world, rank))
    for g in range(world):
        if g != rank:
            be.peer_open(g, hs[g])
    torch.cuda.synchronize(device)
    dist.barrier()
    U = torch.zeros((T, NU), device=device)
    a, x = torch.zeros((T, NU, K), device=device), torch.zeros((T, NU, K), device=device)
    part, act, stats = torch.zeros(2 + T * NU, device=device), torch.zeros(NU, device=device), torch.zeros(2, device=device)
    row = torch.zeros(ESS_ROW_FLOATS, device=device)
    ctr = torch.zeros(1, dtype=torch.int32, device=device)
    tgt = torch.linspace(-0.3, 0.3, T * NU, device=device).view(T, NU, 1)
    out = {k: [] for k in ("lam", "state", "U", "rows", "lam_rows", "state_rows")}
    for _ in range(PLANS):
        be.shift(U, ctr)
        be.sample(11, 0, off, K_TOTAL, U, None, a, x, ctr)
        cost = (4.0 * ((a - tgt) ** 2).sum(1)).contiguous()
        be.temperature(cost, x, U, row, solve=True)                  # exchange s: temperature rows through the window
        be.reduce(cost, x, U, part)                                   # exchange s + 1: K3 rows
        torch.cuda.synchronize(device)
        dist.barrier()
        be.finalize(None, world, U, act, stats)
        torch.cuda.synchronize(device)
        out["lam"].append(dist_buf[0].item())
        out["state"].append(state.cpu().numpy().copy())
        out["U"].append(U.cpu().numpy().copy())
        got = [torch.zeros(ESS_ROW_FLOATS) for _ in range(world)]
        dist.all_gather(got, row.cpu())
        rows = torch.stack(got).to(device).contiguous()
        out["rows"].append(rows.cpu().numpy())
        keep_lam, keep_state = dist_buf[0].clone(), state.clone()
        be.temperature_solve(rows, world)                            # the explicit-row solve of the same rows
        torch.cuda.synchronize(device)
        out["lam_rows"].append(dist_buf[0].item())
        out["state_rows"].append(state.cpu().numpy().copy())
        dist_buf[0] = keep_lam
        state.copy_(keep_state)
        torch.cuda.synchronize(device)
        dist.barrier()
    torch.cuda.synchronize(device)
    dist.barrier()
    be.peer_close()
    be.destroy()
    np.savez(os.path.join(out_dir, f"{rank}.npz"), **{k: np.stack(v) for k, v in out.items()}, K=np.array([K]))
    dist.barrier()
    dist.destroy_process_group()
