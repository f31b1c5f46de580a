"""The restatements of the MODES K3 launch in ``synth_mppi`` pinned to literal values: ``modes_fin_floats`` (the shared floats of
``modes_rows``, csrc/reduce.cu), the floor it puts under the ring region of ``WsLayout`` for n_modes > 1, and the (gx, M) grid of
``launch_reduce_ws_t``.  The GPU sweep of multi-modal MPPI names its cases by these, so a drift here would mislabel what it covers."""
import pytest

from synth_mppi import NUM_SMS, _ws_bytes, mode_range, mode_tiles, modes_fin_floats, modes_grid, ws_layout


def test_modes_fin_floats():
    # 3 M NR + 16 * 16 + M G + 4 M + 2 M^2 + 4
    assert modes_fin_floats(512, 16, 1) == 25428                    # M = 16 at T*nu = 512: the largest of the fused K4
    assert modes_fin_floats(512, 16, 16) == 25668                   # ... and of the split K4 with MPPIB_MAX_PEERS rows
    assert modes_fin_floats(36, 2, 1) == 494


@pytest.mark.parametrize("T,nu,layout,plain,modes16", [
    (32, 16, (16, 3, 3, 256), 218496, 218496),                       # T*nu = 512: the ring exceeds the floor
    (256, 2, (16, 2, 2, 256), 205024, 205024),
    (12, 3, (4, 7, 7, 36), 45616, 45616),
    (1, 1, (4, 7, 7, 1), 3552, 5040),                                # T*nu + T = 2: the floor sizes the ring region
    (1, 3, (4, 7, 7, 3), 5136, 5536),
])
def test_modes_layout(T, nu, layout, plain, modes16):
    """The ring depth and consumer count of the MODES launch are those of the plain row; only the bytes may grow by the floor."""
    assert ws_layout(T, nu, "W") == layout
    assert ws_layout(T, nu, "W", modes=16) == layout
    nstage = layout[2]
    assert _ws_bytes(T, nu, nstage, "W") == plain
    assert _ws_bytes(T, nu, nstage, "W", modes=16) == modes16
    assert _ws_bytes(T, nu, nstage, "W", modes=2) >= plain


def test_modes_grid():
    assert NUM_SMS == 132
    assert modes_grid(64, 0, 32, 2) == 1                             # Kc = 32 aligned: one tile per mode
    assert modes_grid(16 * 256, 0, 256, 16) == 8 == NUM_SMS // 16    # 8 tiles per mode fill 132 // 16 CTAs
    assert modes_grid(2 * 2112, 0, 2112, 2) == 66 == NUM_SMS // 2
    assert modes_grid(2 * 2048, 0, 2048, 2) == 64                    # fewer tiles than 132 // 2
    assert modes_grid(5 * 33, 0, 33, 5) == 2                         # every boundary inside a tile: two tiles per mode
    # a shard [48, 144) of M = 5, Kc = 96: modes 0 and 1 are local, 2 .. 4 have no local sample
    assert [mode_range(96, 48, 96, m) for m in range(3)] == [(0, 48), (48, 96), (144, 96)]
    assert [mode_tiles(96, 48, 96, m) for m in range(5)] == [2, 2, 0, 0, 0]
    assert modes_grid(96, 48, 96, 5) == 2
    # a shard whose first mode has 5 local samples, all in one partial tile
    assert mode_range(100, 27, 32, 0) == (0, 5) and mode_tiles(100, 27, 32, 0) == 1
    assert mode_tiles(100, 27, 32, 1) == 2                           # [5, 37): tiles 0 and 1
