"""-m gpu: constrained MPPI over the peer-window exchange, two and four ranks on one GPU (CUDA IPC between processes), with the feasible
samples on the first ranks only, the last rank only, no rank or every rank: every rank ends every plan with the same U, action and
constraint state, bit for bit; its K4 from the window equals the explicit-row K4 of the same G rows bit for bit and the float64 merge of
those rows; the sharded plans reproduce the plans of one handle holding all samples.  The overlapped exchange across two GPUs (no barrier
between K3 and K4) is not covered here."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import constraint_oracle as cn  # noqa: E402
import constraint_peer_worker as w  # noqa: E402

pytestmark = pytest.mark.gpu


def _exclusive_process():
    """The compute mode of the visible devices, read without changing it: several contexts per device need Default."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=compute_mode", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout
    except (OSError, subprocess.SubprocessError):
        return False
    return "Exclusive_Process" in out


def _spawn(tmp_path, world, case, timeout=600):
    """Run `world` ranks of the worker; the ranks are joined with a timeout and none outlives this call."""
    out = tmp_path / f"world{world}"
    out.mkdir()
    ctx = mp.spawn(w.run, args=(world, str(tmp_path / f"store{world}"), str(out), case), nprocs=world, join=False)
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
@pytest.mark.parametrize("case", ["first", "last", "none", "all"])
def test_constrained_plans_over_the_peer_window(tmp_path, world, case):
    if _exclusive_process():
        pytest.skip("the device is in Exclusive_Process compute mode: several ranks cannot share it")
    from synth_mppi import nu_model
    res = _spawn(tmp_path, world, case)
    for r in range(1, world):
        for k in ("U", "act", "cst", "rows"):
            np.testing.assert_array_equal(res[r][k], res[0][k])
    np.testing.assert_array_equal(res[0]["U"], res[0]["U_rows"])               # window K4 == explicit-row K4 of the same rows
    p = w.params(w.K_TOTAL, 0)
    for j in range(w.PLANS):
        rows = cn.from_f32(res[0]["rows"][j])
        feas_ranks = rows[:, -2] > 0
        lo, hi = w.CASES[case]
        assert feas_ranks.any() == (hi > lo)
        Un, _, _, (n, vmin) = cn.finalize(nu_model(w.NU), p, rows, res[0]["U_before"][j])
        np.testing.assert_allclose(res[0]["U"][j], Un, rtol=0, atol=1e-4)    # the float64 merge of the same rows
        cst = res[0]["cst"][j]
        assert int(np.ascontiguousarray(cst[:1]).view(np.int32)[0]) == n
        np.testing.assert_allclose(cst[1], vmin, rtol=1e-6)
    ref = w.plan("cuda:0", w.K_TOTAL, 0, case)
    for j, (U, act, cst) in enumerate(ref):
        np.testing.assert_allclose(res[0]["U"][j], U, rtol=0, atol=2e-5)      # the shards' rows combine in another order: fp32 only
        np.testing.assert_allclose(res[0]["act"][j], act, rtol=0, atol=2e-5)
        np.testing.assert_array_equal(res[0]["cst"][j][:1], cst[:1])           # the feasible count is exact
