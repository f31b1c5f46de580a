"""The restatements of the spline and constrained K3 launches in ``synth_mppi`` pinned to literal values.  Knots keep T cost rows but
have P*nu control rows (``ctrl_rows``), so the RPL, the consumer count and the ring depth follow P*nu + T; the FEASIBLE rule of
constraint_mode carries T violation rows more per tile ((T*nu + 2T) * 32 floats) and a shard row of 4 + T*nu floats (``WsLayout`` in
csrc/reduce.cu).  The GPU sweep names its cases by these, so a drift here would mislabel what it covers; and the FEASIBLE restatement is
what admission (``blob.feasible_k3_bytes``, ``validate`` in csrc/api.cu) refuses."""
import pytest

from mppi_isaac_b200.model.blob import feasible_k3_bytes
from synth_mppi import _ws_bytes, row_floats, wrap_K, ws_layout, ws_stages


def test_row_floats():
    assert row_floats(256, 2, "W", Tc=32) == 2 + 64                    # knots: the row holds P*nu control rows
    assert row_floats(32, 16, "W", feasible=True) == 4 + 512            # (beta, eta, W, n_feasible, min V)
    assert row_floats(12, 3, "W") == row_floats(12, 3, "W", Tc=12) == 38


@pytest.mark.parametrize("T,P,nu,layout,nbytes", [
    (256, 128, 1, (4, 4, 4, 128), 201504),                              # P*nu = 128: RPL 4
    (256, 129, 1, (8, 4, 4, 129), 202032),                              # 129: RPL 8, a prime row count in one box
    (256, 128, 2, (8, 3, 3, 256), 203008),                              # 256: RPL 8
    (256, 129, 2, (16, 3, 3, 129), 203792),                             # 258: RPL 16, two boxes of 129 rows
    (256, 32, 16, (16, 2, 2, 256), 205024),                             # 512 at T = 256: the largest tile of any mode, two stages
    (256, 256, 2, (16, 2, 2, 256), 205024),
    (2, 2, 1, (4, 7, 7, 2), 5024),                                      # the smallest spline: T = P = d + 1 = 2
])
def test_knots_layout(T, P, nu, layout, nbytes):
    assert ws_layout(T, nu, "W", Tc=P) == layout
    assert _ws_bytes(T, nu, layout[2], "W", Tc=P) == nbytes
    if P < T:                                                           # the plain T*nu layout would name another launch
        assert ws_layout(T, nu, "W") != layout


@pytest.mark.parametrize("T,nu,layout,nbytes", [
    (1, 1, (4, 7, 7, 1), 4240),                                         # T*nu = 1
    (32, 16, (16, 2, 2, 256), 154976),                                  # T*nu = 512: plain runs three stages, FEASIBLE two
    (216, 2, (16, 2, 2, 216), 228480),                                  # the longest nu = 2 horizon: 896 bytes under 224 KiB
    (217, 2, None, None),                                               # two stages need 229568 bytes: refused
    (256, 1, (8, 2, 2, 256), 201952),                                   # the longest horizon
])
def test_feasible_layout(T, nu, layout, nbytes):
    assert ws_layout(T, nu, "W", feasible=True) == layout
    if layout is None:
        assert ws_stages(T, nu, "W", feasible=True) < 2 and ws_layout(T, nu, "W") is not None
        assert feasible_k3_bytes(T, nu) == 229568 > 224 * 1024
    else:
        assert _ws_bytes(T, nu, layout[2], "W", feasible=True) == nbytes
        assert feasible_k3_bytes(T, nu) <= 224 * 1024


def test_wrap_K_follows_the_ring():
    """wrap_K streams more than three rings on every CTA: with fewer stages it is a smaller K."""
    assert wrap_K(32, 16, "W") == 32 * 132 * 10 - 12                   # three stages
    assert wrap_K(32, 16, "W", feasible=True) == 32 * 132 * 7 - 12     # two
    assert wrap_K(256, 1, "W", Tc=128) == 32 * 132 * 13 - 12           # four


def test_feasible_refuses_exactly_nu2_long_horizons():
    """Among the shapes the plain K3 accepts (T <= 256, T*nu <= 512), the FEASIBLE ring refuses exactly nu = 2 with 217 <= T <= 256, and
    feasible_k3_bytes (make_params' limit) is the restatement's two-stage size at every one of them."""
    plain = [(T, nu) for nu in range(1, 17) for T in range(1, 257) if T * nu <= 512]
    assert all(ws_layout(T, nu, "W") is not None for T, nu in plain)
    refused = {(T, nu) for T, nu in plain if ws_layout(T, nu, "W", feasible=True) is None}
    assert refused == {(T, 2) for T in range(217, 257)}
    for T, nu in plain:
        assert feasible_k3_bytes(T, nu) == _ws_bytes(T, nu, 2, "W", feasible=True)
        assert (feasible_k3_bytes(T, nu) > 224 * 1024) == ((T, nu) in refused)
