"""Spline MPPI sharded over two gloo ranks on the checker backend (P = 4 knots of degree 3): every rank ends every plan with the same
actions, knots and U_exec, and the sharded plan reproduces the single-process one."""
import os
import socket
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.timeout(300)
def test_sharded_spline_plan_matches_single_process(tmp_path):
    sys.path.insert(0, HERE)
    import knots_dist_worker as w
    world, K = 2, 136
    mp.spawn(w.run, args=(world, _free_port(), str(tmp_path), K), nprocs=world, join=True)
    single, ref, ref_exe = w.plan(K)
    for name in ("act", "exe", "U"):
        a0 = np.load(tmp_path / f"{name}_0.npy")
        np.testing.assert_array_equal(np.load(tmp_path / f"{name}_1.npy"), a0)   # both ranks hold the same bits
    np.testing.assert_allclose(np.load(tmp_path / "act_0.npy"), ref, rtol=0, atol=2e-5)   # == the unsharded plan (fp32 reassociation only)
    np.testing.assert_allclose(np.load(tmp_path / "exe_0.npy"), ref_exe, rtol=0, atol=2e-5)
    np.testing.assert_allclose(np.load(tmp_path / "U_0.npy"), single.mppi.U.numpy(), rtol=0, atol=2e-5)
