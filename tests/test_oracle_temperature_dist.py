"""The ESS-targeted temperature sharded over two and three gloo ranks on the checker backend, with uneven shards and with the valid samples
on the first rank only: every rank ends every plan with the same temperature, actions and U, and the sharded plan reproduces the
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
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("case", ["all", "one_rank"])
def test_sharded_ess_plan_matches_single_process(tmp_path, world, case):
    sys.path.insert(0, HERE)
    import temperature_dist_worker as w
    mp.spawn(w.run, args=(world, _free_port(), str(tmp_path), case), nprocs=world, join=True)
    single, ref, ref_lam = w.plan(case)
    shards = [int(np.load(tmp_path / f"K_{r}.npy")[0]) for r in range(world)]
    assert sum(shards) == 140 and len(set(shards)) > 1                      # uneven shards
    for r in range(1, world):
        for name in ("act", "U", "lam"):
            np.testing.assert_array_equal(np.load(tmp_path / f"{name}_{r}.npy"), np.load(tmp_path / f"{name}_0.npy"))   # the same bits
    lam = np.load(tmp_path / "lam_0.npy")
    np.testing.assert_array_equal(lam[:, 1], ref_lam[:, 1])
    assert np.all(lam[:, 1] == (140 if case == "all" else 40))
    np.testing.assert_allclose(lam[:, 0], ref_lam[:, 0], rtol=1e-5)
    np.testing.assert_allclose(np.load(tmp_path / "act_0.npy"), ref, rtol=0, atol=2e-5)
    np.testing.assert_allclose(np.load(tmp_path / "U_0.npy"), single.mppi.U.numpy(), rtol=0, atol=2e-5)
