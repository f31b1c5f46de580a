"""Cross-entropy planning sharded over two gloo ranks on the checker backend: three iterations per plan with carried elites, which K1
writes into rows K_total - 3 - e of the last shard.  Every rank ends with the same actions, U and CEM state, the sharded plans choose
the same elites as the single-process plan, and reproduce its U, sigma and actions."""
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
def test_two_rank_cem_plan_matches_single_process(tmp_path):
    sys.path.insert(0, HERE)
    import cem_dist_worker as w
    import cem_oracle as ce
    mp.spawn(w.run, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    single, ref = w.plan()
    load = lambda name, r: np.load(tmp_path / f"{name}_{r}.npy")               # noqa: E731
    for name in ("act", "U", "state", "elites"):
        np.testing.assert_array_equal(load(name, 0), load(name, 1))          # every rank holds the same plan
    idx = load("elites", 0)
    assert idx.shape == (2 * 3, int(single.mppi.backend.params.n_elites))     # two plans of three iterations
    np.testing.assert_array_equal(idx, np.array(single.mppi.backend.elite_index, np.int64))
    K_total, n_keep = 64, int(single.mppi.backend.params.n_keep)
    carried = set(range(K_total - 3 - n_keep + 1, K_total - 2))
    assert carried & set(idx[3:].ravel().tolist()), "no carried elite was chosen again: the carry is not exercised"
    p = single.mppi.backend.params
    T, nu, E = int(p.T), single.mppi.nu, int(p.n_elites)
    np.testing.assert_allclose(load("act", 0), ref, rtol=0, atol=2e-6)       # == the unsharded plan (fp32 reassociation only)
    np.testing.assert_allclose(load("U", 0), single.mppi.U.numpy(), rtol=0, atol=2e-6)
    st, st1 = load("state", 0), single.mppi.dist.numpy()
    np.testing.assert_allclose(ce.unpack(st, T, nu, E)[3], ce.unpack(st1, T, nu, E)[3], rtol=0, atol=2e-6)    # sigma
    np.testing.assert_allclose(st, st1, rtol=0, atol=2e-6)
