"""Multi-modal MPPI sharded over two and three gloo ranks on the checker backend, every shard boundary inside a mode: every rank ends with
the same actions, modes and mode state, and the sharded plan reproduces the single-process one."""
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


# (world, K_total): two shards of 68 / 64 samples with Kc = 33 (the boundary 68 cuts mode 2), three of 64 with Kc = 48 (64 and 128
# cut modes 1 and 2)
@pytest.mark.timeout(300)
@pytest.mark.parametrize("world, K", [(2, 132), (3, 192)])
def test_sharded_modes_plan_matches_single_process(tmp_path, world, K):
    sys.path.insert(0, HERE)
    import modes_dist_worker as w
    from mppi_isaac_b200.planner.mppi import shard_samples
    mp.spawn(w.run, args=(world, _free_port(), str(tmp_path), K), nprocs=world, join=True)
    single, ref, ref_states = w.plan(K)
    Kc = int(single.mppi.backend.params.mode_samples)
    assert Kc == K // 4 and all(shard_samples(K, r, world)[1] % Kc != 0 for r in range(1, world))   # every boundary cuts a mode
    for name in ("act", "state", "U"):
        a0 = np.load(tmp_path / f"{name}_0.npy")
        for r in range(1, world):
            np.testing.assert_array_equal(np.load(tmp_path / f"{name}_{r}.npy"), a0)   # every rank holds the same bits
    a0, st0 = np.load(tmp_path / "act_0.npy"), np.load(tmp_path / "state_0.npy")
    np.testing.assert_allclose(a0, ref, rtol=0, atol=2e-5)                    # == the unsharded plan (fp32 reassociation only)
    np.testing.assert_array_equal(st0[:, 0], ref_states[:, 0])                # the same executed mode after every plan
    np.testing.assert_allclose(st0[:, 1:], ref_states[:, 1:], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(np.load(tmp_path / "U_0.npy"), single.mppi.U.numpy(), rtol=0, atol=2e-5)
