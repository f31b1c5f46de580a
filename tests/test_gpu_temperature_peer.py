"""-m gpu: the ESS-targeted temperature over the peer-window exchange, two and four ranks on one GPU (CUDA IPC between processes), over
five consecutive plans so that both window slots are reused by the temperature and K3 exchanges: every rank writes the same lambda, state
and U bits, and lambda equals the explicit-row solve of the same rows and the float64 rule on them."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import temperature_oracle as tmo  # noqa: E402
import temperature_peer_worker as w  # noqa: E402

pytestmark = pytest.mark.gpu


def _exclusive_process():
    """The compute mode of the visible devices, read without changing it: several contexts per device need Default."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=compute_mode", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout
    except (OSError, subprocess.SubprocessError):
        return False
    return "Exclusive_Process" in out


def _spawn(tmp_path, world, timeout=600):
    """Run `world` ranks of the worker; the ranks are joined with a timeout and none outlives this call."""
    out = tmp_path / f"world{world}"
    out.mkdir()
    ctx = mp.spawn(w.run, args=(world, str(tmp_path / f"store{world}"), str(out)), nprocs=world, join=False)
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
    return [np.load(out / f"{r}.npz") for r in range(world)]


@pytest.mark.parametrize("world", [2, 4])
def test_temperature_over_the_peer_window(tmp_path, world):
    if _exclusive_process():
        pytest.skip("the device is in Exclusive_Process compute mode: several ranks cannot share it")
    from mppi_isaac_b200.model.blob import ESS_GRID, ess_grid
    res = _spawn(tmp_path, world)
    assert sum(int(r["K"][0]) for r in res) == w.K_TOTAL and len({int(r["K"][0]) for r in res}) > 1   # uneven shards
    for r in range(1, world):
        for k in ("lam", "state", "U", "rows"):
            np.testing.assert_array_equal(res[r][k], res[0][k])
    np.testing.assert_array_equal(res[0]["lam"], res[0]["lam_rows"])            # window solve == explicit-row solve, bit for bit
    np.testing.assert_array_equal(res[0]["state"], res[0]["state_rows"])
    lam_grid = ess_grid(w.params(w.K_TOTAL, 0).lambda_)[0].astype(np.float64)
    assert len(set(res[0]["lam"].tolist())) > 1
    for j in range(w.PLANS):
        N, ess = tmo.combine([tmo.from_f32(r) for r in res[0]["rows"][j]])
        st = res[0]["state"][j]
        assert N == w.K_TOTAL == int(st[2 * ESS_GRID:2 * ESS_GRID + 1].view(np.int32)[0])
        np.testing.assert_allclose(st[2 * ESS_GRID + 2:], ess, rtol=1e-5)
        assert res[0]["lam"][j] == pytest.approx(tmo.rule(st[2 * ESS_GRID + 2:].astype(np.float64), N, float(np.float32(0.05)), lam_grid, 0.0),
                                                 rel=2e-6)
