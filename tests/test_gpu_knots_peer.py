"""-m gpu: spline MPPI over the peer-window exchange, two and four ranks on one GPU (CUDA IPC between processes), P = 4 knots of degree 3:
every rank ends every plan with the same knots, action and U_exec, bit for bit, and its K4 from the window equals the explicit-row K4 of the
same G rows bit for bit; the sharded plans reproduce the plans of one handle holding all samples.  The overlapped exchange across two GPUs
(no barrier between K3 and K4) is not covered here."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import knots_peer_worker as w  # noqa: E402

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
def test_spline_plans_over_the_peer_window(tmp_path, world):
    if _exclusive_process():
        pytest.skip("the device is in Exclusive_Process compute mode: several ranks cannot share it")
    res = _spawn(tmp_path, world)
    for r in range(1, world):
        for k in ("U", "act", "exe", "rows"):
            np.testing.assert_array_equal(res[r][k], res[0][k])
    np.testing.assert_array_equal(res[0]["U"], res[0]["U_rows"])               # window K4 == explicit-row K4 of the same rows
    np.testing.assert_array_equal(res[0]["exe"], res[0]["exe_rows"])
    ref = w.plan("cuda:0", w.K_TOTAL, 0)
    for j, (U, act, exe) in enumerate(ref):
        np.testing.assert_allclose(res[0]["U"][j], U, rtol=0, atol=2e-5)      # the shards' rows combine in another order: fp32 only
        np.testing.assert_allclose(res[0]["act"][j], act, rtol=0, atol=2e-5)
        np.testing.assert_allclose(res[0]["exe"][j], exe, rtol=0, atol=2e-5)
