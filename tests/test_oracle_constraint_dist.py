"""Constrained MPPI sharded over two gloo ranks on the checker backend: the feasible samples lie on the first rank only, on the second only,
or on neither; every rank ends every plan with the same actions, U and constraint state, and the sharded plan reproduces the
single-process one."""
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
@pytest.mark.parametrize("case", ["first", "second", "neither"])
def test_sharded_constrained_plan_matches_single_process(tmp_path, case):
    sys.path.insert(0, HERE)
    import constraint_dist_worker as w
    world = 2
    mp.spawn(w.run, args=(world, _free_port(), str(tmp_path), case), nprocs=world, join=True)
    single, ref, ref_cst = w.plan(case)
    for name in ("act", "U", "cst"):
        np.testing.assert_array_equal(np.load(tmp_path / f"{name}_1.npy"), np.load(tmp_path / f"{name}_0.npy"))   # the same bits on both ranks
    np.testing.assert_allclose(np.load(tmp_path / "act_0.npy"), ref, rtol=0, atol=2e-5)
    np.testing.assert_allclose(np.load(tmp_path / "U_0.npy"), single.mppi.U.numpy(), rtol=0, atol=2e-5)
    cst = np.load(tmp_path / "cst_0.npy")
    np.testing.assert_array_equal(cst[:, 0], ref_cst[:, 0])
    np.testing.assert_allclose(cst[:, 1], ref_cst[:, 1], rtol=1e-6)
    assert np.all(cst[:, 0] == 0) if case == "neither" else np.all(cst[:, 0] > 0)
