"""-m gpu: the peer-window exchange of multi-modal MPPI (the [M][2 + T*nu] shard row), with two and four ranks on one GPU (CUDA IPC
between processes) and uneven shards whose boundaries fall inside modes.  ``modes_peer_worker`` runs the ranks; for every exchange:

(a) every rank holds the same K4 outputs (U, action, stats, mode state), bit for bit;
(b) ``mppib_finalize`` on one handle here, with the saved shard rows stacked at stride P and the saved U and mode state before K4,
    gives the peer K4's outputs bit for bit -- a difference is the window path's own (block offset, stride pcap, parity or counter);
(c) every rank's shard row matches the float64 per-mode row of its shard (``modes_oracle.reduce``), block by block."""
import os
import pickle
import subprocess
import sys
import time

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import modes_oracle as mo  # noqa: E402
import modes_peer_worker as w  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 2.0 ** -24


def _exclusive_process():
    """The compute mode of the visible devices, read without changing it: several contexts per device need Default."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=compute_mode", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout
    except (OSError, subprocess.SubprocessError):
        return False
    return "Exclusive_Process" in out


def _spawn(tmp_path, world, names, timeout=600):
    """Run `world` ranks of the worker over `names`; the ranks are joined with a timeout and none outlives this call."""
    out = tmp_path / f"world{world}"
    out.mkdir()
    ctx = mp.spawn(w.run, args=(world, str(tmp_path / f"store{world}"), str(out), names), nprocs=world, join=False)
    deadline = time.monotonic() + timeout
    try:
        while not ctx.join(timeout=max(1.0, deadline - time.monotonic())):
            if time.monotonic() >= deadline:
                raise TimeoutError(f"world {world}: the ranks did not finish within {timeout} s")
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.terminate()
        for p in ctx.processes:
            p.join(10)
            if p.is_alive():
                p.kill()
                p.join()
    res = {}
    for name in names:
        res[name] = []
        for r in range(world):
            with open(out / f"{name}_{r}.pkl", "rb") as f:
                res[name].append(pickle.load(f))
    return res


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def explicit_k4(name, world, rec, rows):
    from mppi_isaac_b200.backend import CudaBackend
    from synth_mppi import nu_model
    nu = w.CASES[name][1]
    be = CudaBackend(DEV)
    be.create(nu_model(nu), w.params(name, 0))
    st = torch.as_tensor(rec["st0"]).to(DEV)
    be.set_distribution(st)
    U, act, stats = torch.as_tensor(rec["U0"]).to(DEV), torch.zeros(nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(torch.as_tensor(np.ascontiguousarray(rows)).to(DEV), world, U, act, stats)
    got = dict(U=U.cpu().numpy(), act=act.cpu().numpy(), stats=stats.cpu().numpy(), st=st.cpu().numpy())
    be.destroy()
    return got


@pytest.mark.parametrize("world", [2, 4])
def test_modes_peer_window_exchange(tmp_path, world):
    if _exclusive_process():
        pytest.skip("the device is in Exclusive_Process compute mode: several ranks cannot share it")
    names = [n for n in w.CASES if w.world_of(n) == world]
    res = _spawn(tmp_path, world, names)
    for name in names:
        T, nu, M, Kc, offs = w.CASES[name][:5]
        ranks = res[name]
        for j, rec0 in enumerate(ranks[0]):
            for r in range(1, world):                                        # (a)
                for k in ("U", "act", "stats", "st"):
                    assert _same(ranks[r][j][k], rec0[k]), f"{name} exchange {j}: rank {r} {k} differs from rank 0"
            rows = np.stack([ranks[r][j]["row"] for r in range(world)])
            got = explicit_k4(name, world, rec0, rows)                       # (b)
            for k in ("U", "act", "stats", "st"):
                assert _same(got[k], rec0[k]), f"{name} exchange {j}: the peer K4's {k} differs from the explicit-row K4"
            for r in range(world):                                           # (c)
                p = w.params(name, r)
                cost, x = w.inputs(name, r, j)
                ref = mo.reduce(p, nu, cost, x, rec0["U0"]).reshape(M, -1)
                row = ranks[r][j]["row"].reshape(M, -1)
                mag = float(np.where(np.isfinite(cost), np.abs(cost), 0).sum(0).max()) + 1.0
                gb = (T + T * nu + 8) * EPS * (mag + np.abs(x).sum((0, 1)).max() * 10)
                gw = 64 * EPS * Kc + gb / float(np.float32(p.lambda_)) * 2
                for m in range(M):
                    if ref[m, 1] == 0:
                        assert row[m, 0] == np.inf and row[m, 1] == 0 and (row[m, 2:] == 0).all(), (name, j, r, m)
                        continue
                    assert abs(float(row[m, 0]) - float(ref[m, 0])) <= gb, (name, j, r, m)
                    np.testing.assert_allclose(row[m, 1], ref[m, 1], rtol=gw, atol=0)
                    np.testing.assert_allclose(row[m, 2:], ref[m, 2:], rtol=0, atol=gw * max(1.0, float(np.abs(ref[m, 2:]).max())))
        assert any(np.isinf(ranks[r][1]["row"].reshape(M, -1)[:, 0]).all() for r in range(world))   # a shard without a valid sample
