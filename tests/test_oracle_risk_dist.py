"""Risk-aware MPPI sharded over two gloo ranks on the checker backend: every rank ends with the same actions and U, and the sharded
plan reproduces the single-process one."""
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
def test_two_rank_risk_plan_matches_single_process(tmp_path):
    sys.path.insert(0, HERE)
    import risk_dist_worker as w
    mp.spawn(w.run, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    single, ref = w.plan()
    a0, a1 = np.load(tmp_path / "act_0.npy"), np.load(tmp_path / "act_1.npy")
    np.testing.assert_array_equal(a0, a1)                                 # every rank executes the same command
    np.testing.assert_allclose(a0, ref, rtol=0, atol=2e-5)                # == the unsharded plan (fp32 reassociation only)
    np.testing.assert_array_equal(np.load(tmp_path / "U_0.npy"), np.load(tmp_path / "U_1.npy"))
    np.testing.assert_allclose(np.load(tmp_path / "U_0.npy"), single.mppi.U.numpy(), rtol=0, atol=2e-5)
