"""-m gpu: the fused pose-cost kernel (``mppib_cost_pose_kernel`` through ``ops.pose_cost``) against the float64 reference of
``tests/pose_cost_ref.py``, gated per entry by its derived float32 bound.

Covered: every strided view the ``RolloutSim`` getters hand out, sizes around the launcher's grid cap (8 CTAs of 256 threads per
SM, so the grid-stride loop runs up to 8 passes at C5 size), the quaternion edges (gimbal lock, yaw at +-pi, non-unit and zero
quaternions, q vs -q), the weight and accumulate paths, a guard band around ``out``, side streams, graph capture and a second
device."""
import numpy as np
import pytest
import torch

import pose_cost_ref as pr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = -1.0e30                     # no cost is negative: an entry still holding it was not written
GUARD = 4099


def _ops():
    from mppi_isaac_b200 import ops
    return ops


def grid_cap(device=DEV):
    """Threads of the launcher's largest grid: 8 CTAs of 256 per SM."""
    return 8 * torch.cuda.get_device_properties(device).multi_processor_count * 256


_WORST = {}


def _report(group, ratio, nan=0):
    w, c = _WORST.get(group, (0.0, 0))
    _WORST[group] = (max(w, ratio), c + nan)
    print(f"[pose-cost] {group}: worst err/gate {_WORST[group][0]:.3g}, NaN {_WORST[group][1]}")


def _guarded_out(n, device=DEV, fill=None):
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.float32, device=device)
    out = buf[GUARD:GUARD + n]
    if fill is not None:
        out.copy_(fill)
    return buf, out


def check(group, a, b, w_pos, w_ori, out=None, buf=None, accumulate=False, out0=None, got=None):
    """Run the kernel (unless ``got`` is given) and compare with the reference: NaN only where allowed, every other entry
    finite and inside its gate, every entry written and the guard band untouched."""
    n = a.shape[0]
    if got is None:
        if out is None:
            buf, out = _guarded_out(n, a.device)
        _ops().pose_cost(a, b, w_pos, w_ori, out=out, accumulate=accumulate)
        torch.cuda.synchronize(a.device)
        got = out
    ah = a.detach().cpu().numpy()
    bh = None if b is None else b.detach().cpu().numpy()
    ref = pr.pose_cost_ref(ah, bh, w_pos, w_ori)
    gate = pr.pose_cost_gate(ah, bh, w_pos, w_ori, out0=out0)
    if out0 is not None:
        ref = ref + np.asarray(out0, np.float64)
    g = got.cpu().numpy().astype(np.float64)
    assert (g != SENTINEL).all(), f"{int((g == SENTINEL).sum())} of {n} entries not written"
    if buf is not None:
        band = torch.cat([buf[:GUARD], buf[GUARD + n:]])
        assert bool((band == SENTINEL).all()), "the kernel wrote outside [0, n)"
    nan = np.isnan(g)
    allowed = pr.nan_allowed(ah[:, 3:7]) if (w_ori and ah.shape[1] >= 7) else np.zeros(n, bool)
    if out0 is not None:
        allowed |= np.isnan(out0)
    assert not nan[~allowed].any(), f"NaN at rows {np.flatnonzero(nan & ~allowed)[:8]}"
    fin = ~nan & np.isfinite(ref)
    with np.errstate(invalid="ignore"):                           # inf - inf on the accumulated +-inf rows
        err = np.abs(g - ref)
    ratio = err[fin] / gate[fin]
    bad = np.flatnonzero(fin)[ratio > 1]
    assert bad.size == 0, f"{bad.size} entries outside the gate, first {bad[:4]}: got {g[bad[:4]]}, ref {ref[bad[:4]]}, gate {gate[bad[:4]]}"
    assert nan[np.isnan(ref)].all(), "the reference is NaN (zero quaternion or NaN in out) where the kernel is not"
    inf = ~nan & np.isinf(ref)
    assert (g[inf] == ref[inf]).all()
    _report(group, float(ratio.max()) if ratio.size else 0.0, int(nan.sum()))
    return g


def _mixed_rows(n, seed):
    """(n, 13) float32 rows on the device: random positions, random unit quaternions with every edge quaternion of
    ``edge_quaternions`` planted at random rows (the zero quaternion included)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = (torch.rand((n, 13), device=DEV, generator=g) - 0.5) * 4
    q = torch.randn((n, 4), device=DEV, generator=g)
    a[:, 3:7] = q / q.norm(dim=1, keepdim=True)
    edges = torch.from_numpy(np.concatenate(list(pr.edge_quaternions(seed).values()))).to(DEV)
    m = min(n, edges.shape[0])
    idx = torch.randperm(n, device=DEV, generator=g)[:m]
    a[idx, 3:7] = edges[:m]
    return a


def _view(layout, rows, T=1):
    """The getters' views of (n, 13) rows ``rows``: 'batched' obs view (strides (1, n)), 'step' view of one slot (non-zero
    storage offset), 'link_mid' rows of a link in the middle of a wider obs, 'dense' (n, 13)."""
    n = rows.shape[0]
    if layout == "dense":
        return rows.contiguous()
    if layout == "batched":
        obs = torch.empty((13 + 14, n), device=DEV)
        obs[:13] = rows.t()
        return obs[:13].view(13, n).t()
    if layout == "link_mid":
        obs = torch.full((13 * 3 + 14, n), float("nan"), device=DEV)
        obs[27:40] = rows.t()
        return obs[27:40].t()
    if layout == "step":
        Ts, slot = 3, 2
        obs = torch.full((13 * 2 + 14, Ts, n), float("nan"), device=DEV)
        obs[13:26, slot, :] = rows.t()
        v = obs[13:26, slot, :].t()
        assert v.storage_offset() != 0 and v.stride() == (1, Ts * n)
        return v
    raise ValueError(layout)


def _goal(kind, n, seed=7):
    if kind == "stride0":
        return torch.tensor([0.4, -0.1, 0.6], device=DEV).unsqueeze(0).expand(n, 3)
    g = torch.Generator(device=DEV).manual_seed(seed)
    wide = torch.full((5, n + 3), float("nan"), device=DEV)
    wide[1:4, 3:] = (torch.rand((3, n), device=DEV, generator=g) - 0.5) * 4
    v = wide[1:4, 3:].t()                                         # strides (1, n + 3), offset n + 6
    assert v.stride() == (1, n + 3)
    return v


@pytest.mark.parametrize("layout", ["batched", "step", "link_mid", "dense"])
@pytest.mark.parametrize("goal", ["stride0", "per_row"])
@pytest.mark.parametrize("which", ["257", "cap+1"])
def test_pose_cost_layouts(layout, goal, which):
    n = 257 if which == "257" else grid_cap() + 1
    rows = _mixed_rows(n, seed=n)
    a = _view(layout, rows)
    assert torch.equal(a.nan_to_num(7.0), rows.nan_to_num(7.0))
    check("layouts", a, _goal(goal, n), 1.0, 0.5)


def _sizes():
    cap = grid_cap() if torch.cuda.is_available() else 8 * 132 * 256
    return [1, 2, 255, 256, 257, cap - 1, cap, cap + 1, 3 * cap + 7, 300_000, 65_536 * 30]


@pytest.mark.parametrize("n", _sizes())
def test_pose_cost_sizes(n):
    """The batched obs view of the plan at every size around the grid cap: the grid-stride loop runs 1 to 8 passes."""
    rows = _mixed_rows(n, seed=n % 1000 + 1)
    check("sizes", _view("batched", rows), _goal("stride0", n), 1.0, 0.5)
    check("sizes", _view("batched", rows), _goal("per_row", n), 40.0, 2.0)


def test_pose_cost_quaternion_edges():
    """Gimbal lock (pitch = +-(pi/2 - delta), delta = 1e-1 ... 0), yaw at and next to +-pi, quaternions scaled by 10^-3 ... 10^3,
    q next to -q (bit-identical costs) and the zero quaternion (NaN, as in the reference)."""
    groups = pr.edge_quaternions(seed=11, per_group=512)
    for name, q in groups.items():
        qq = q
        if name == "q_negq":
            qq = q[: q.shape[0] // 2]
        a = pr.rows_with_quaternions(qq, seed=2)
        if name == "q_negq":
            neg = a.copy()
            neg[:, 3:7] = -neg[:, 3:7]
            a = np.concatenate([a, neg])
        b = np.random.default_rng(3).uniform(-2, 2, (a.shape[0], 3)).astype(np.float32)
        if name == "q_negq":
            b[b.shape[0] // 2:] = b[: b.shape[0] // 2]
        ad, bd = torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)
        for w in ((1.0, 0.5), (0.0, 1.0)):
            g = check(f"edge:{name}", ad, bd if w[0] else None, *w)
            if name == "zero":
                assert np.isnan(g).all()
            if name == "q_negq":
                h = g.shape[0] // 2
                assert np.array_equal(g[:h].astype(np.float32).view(np.int32), g[h:].astype(np.float32).view(np.int32))
            if name == "gimbal" and w == (0.0, 1.0):
                print(f"[pose-cost] gimbal-lock edge: {int(np.isnan(g).sum())} NaN of {g.shape[0]} rows "
                      f"({int(pr.nan_allowed(a[:, 3:7]).sum())} allowed)")


def test_pose_cost_weights_guard_columns():
    """w_pos = 0 with b = None never reads the position columns, w_ori = 0 never reads the quaternion columns: NaN there
    must not reach the result."""
    n = 5000
    rows = _mixed_rows(n, seed=21)
    ok = ~torch.from_numpy(pr.nan_allowed(rows[:, 3:7].cpu().numpy())).to(DEV)
    rows = rows[ok].contiguous()
    n = rows.shape[0]
    poisoned = rows.clone()
    poisoned[:, 0:3] = float("nan")
    obs = poisoned.t().contiguous()
    a = obs.t()
    got = check("weights", a, None, 0.0, 0.75)
    assert np.isfinite(got).all()
    poisoned = rows.clone()
    poisoned[:, 3:13] = float("nan")
    a3 = poisoned.t().contiguous()[:3].t()                         # a 3-column view over NaN quaternion storage
    goal = _goal("per_row", n)
    got = check("weights", a3, goal, 2.5, 0.0)
    assert np.isfinite(got).all()


def test_pose_cost_accumulate():
    """accumulate=True adds to what ``out`` holds: finite values, +-inf and NaN stay out + c, bit for bit."""
    n = grid_cap() + 5
    rows = _mixed_rows(n, seed=31)
    a, goal = _view("batched", rows), _goal("stride0", n)
    fresh = _ops().pose_cost(a, goal, 1.0, 0.5)
    g = torch.Generator(device=DEV).manual_seed(5)
    base = torch.rand(n, device=DEV, generator=g) * 10 - 5
    base[::11] = float("inf")
    base[1::11] = float("-inf")
    base[2::11] = float("nan")
    base[3::11] = 1e30
    buf, out = _guarded_out(n, fill=base)
    out0 = base.cpu().numpy().astype(np.float64)
    check("accumulate", a, goal, 1.0, 0.5, out=out, buf=buf, accumulate=True, out0=out0)
    want = base + fresh
    assert torch.equal(out.view(torch.int32)[~want.isnan()], want.view(torch.int32)[~want.isnan()])
    assert bool(out[want.isnan()].isnan().all())


def test_pose_cost_on_a_side_stream_after_a_writer():
    """ops.pose_cost runs on the caller's current stream: it sees what the kernel before it on that stream wrote into a."""
    n = 3 * grid_cap() + 7
    src = _mixed_rows(n, seed=42)
    obs = torch.zeros((13, n), device=DEV)
    a, goal = obs.t(), _goal("stride0", n)
    s = torch.cuda.Stream(device=DEV)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(2_000_000)                              # keep the writer late: a launch on another stream would race it
        obs.copy_(src.t())
        buf, out = _guarded_out(n)
        _ops().pose_cost(a, goal, 1.0, 0.5, out=out)
    s.synchronize()
    check("streams", src, goal, 1.0, 0.5, buf=buf, got=out)


def test_pose_cost_in_a_captured_graph():
    """A captured launch replays bit-identical to the eager call and reads the current contents of a."""
    n = grid_cap() + 1
    obs = _mixed_rows(n, seed=51).t().contiguous()
    a, goal = obs.t(), _goal("per_row", n)
    out = torch.empty(n, device=DEV)
    s = torch.cuda.Stream(device=DEV)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _ops().pose_cost(a, goal, 1.0, 0.5, out=out)             # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _ops().pose_cost(a, goal, 1.0, 0.5, out=out)
    for seed in (51, 52):
        obs.copy_(_mixed_rows(n, seed=seed).t())
        out.fill_(SENTINEL)
        graph.replay()
        eager = _ops().pose_cost(a, goal, 1.0, 0.5)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), eager.view(torch.int32))
        check("graph", a, goal, 1.0, 0.5, got=out)


def test_pose_cost_on_another_device():
    """cost on cuda:1 while the current device is cuda:0: the launcher switches to the device that owns `out` and back."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    torch.cuda.set_device(0)
    n = grid_cap("cuda:1") + 3
    rows = _mixed_rows(n, seed=61).to("cuda:1")
    a = rows.t().contiguous().t()
    goal = torch.tensor([0.4, -0.1, 0.6], device="cuda:1").unsqueeze(0).expand(n, 3)
    buf, out = _guarded_out(n, "cuda:1")
    _ops().pose_cost(a, goal, 1.0, 0.5, out=out)
    assert torch.cuda.current_device() == 0
    torch.cuda.synchronize("cuda:1")
    check("devices", a, goal, 1.0, 0.5, buf=buf, got=out)
