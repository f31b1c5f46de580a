"""The float64 reference and the float32 gate of the fused pose cost (``tests/pose_cost_ref.py``), on the CPU.

The GPU test (``tests/test_gpu_pose_cost.py``) compares ``mppib_cost_pose_kernel`` with this reference under this gate, so
both are pinned here: the reference against scipy's rotations, the gate against a float32 restatement of the kernel's
operation order (inside everywhere) and against wrong variants of it (outside somewhere), and the oracle's ``cost_pose``
against both."""
import warnings

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import pose_cost_ref as pr


def _all_quats():
    g = pr.edge_quaternions(seed=3)
    return np.concatenate([v for k, v in g.items() if k != "zero"]), g


def _worst(err, gate):
    ok = np.isfinite(err)
    return float((err[ok] / gate[ok]).max())


def test_reference_equals_scipy_rotation():
    """quaternion_to_matrix of (r, i, j, k) == scipy's matrix of the scalar-last (i, j, k, r), i.e. the xyzw row read as wxyz;
    the ZYX angles equal scipy's away from gimbal lock, and |yaw| at +-pi."""
    q, _ = _all_quats()
    q = q.astype(np.float64)
    rot = Rotation.from_quat(np.roll(q, -1, axis=1))
    m = pr.quaternion_to_matrix(q)
    np.testing.assert_allclose(m, rot.as_matrix(), rtol=0, atol=1e-12)
    e = pr.matrix_to_euler_zyx(m)
    ok = np.abs(m[:, 2, 0]) < 1 - 1e-6
    assert ok.sum() > 100
    with warnings.catch_warnings():
        warnings.simplefilter("error")                                 # scipy warns at gimbal lock; these rows are away from it
        s = rot[np.flatnonzero(ok)].as_euler("ZYX")
    np.testing.assert_allclose(np.abs(e[ok, 0]), np.abs(s[:, 0]), rtol=0, atol=1e-9)
    np.testing.assert_allclose(np.cos(e[ok, 0]), np.cos(s[:, 0]), rtol=0, atol=1e-9)
    np.testing.assert_allclose(e[ok, 1], s[:, 1], rtol=0, atol=1e-9)
    # the identity xyzw quaternion (0, 0, 0, 1) read real first is a half turn about z: cost term pi
    np.testing.assert_allclose(pr.orientation_ref(np.array([[0.0, 0.0, 0.0, 1.0]])), [np.pi], rtol=1e-15)
    np.testing.assert_allclose(pr.orientation_ref(np.array([[1.0, 0.0, 0.0, 0.0]])), [0.0], atol=0)
    # euler angles round trip through the generator the edge inputs are made with
    ang = np.array([[0.3, -0.7, 1.1], [-2.9, 0.2, -0.4], [np.pi - 1e-3, 1.5, 0.0]])
    np.testing.assert_allclose(pr.matrix_to_euler_zyx(pr.quaternion_to_matrix(pr.quat_from_zyx(*ang.T))), ang, atol=1e-12)
    assert np.isnan(pr.orientation_ref(np.zeros((1, 4))))[0]


def _inputs(seed=0):
    q, g = _all_quats()
    q = np.concatenate([q, g["zero"]])
    a = pr.rows_with_quaternions(q, seed=seed)
    b = np.random.default_rng(seed + 1).uniform(-2, 2, (q.shape[0], 3)).astype(np.float32)
    b[::7] = a[::7, 0:3]                                               # zero distance rows
    b[1::7] = a[1::7, 0:3] + np.float32(1e-6)                          # tiny distance rows
    return a, b


@pytest.mark.parametrize("w_pos,w_ori", [(1.0, 0.5), (40.0, 2.0), (0.0, 1.0), (1.0, 0.0), (-3.0, 0.25)])
def test_float32_restatement_stays_inside_the_gate(w_pos, w_ori):
    a, b = _inputs()
    ref = pr.pose_cost_ref(a, b, w_pos, w_ori)
    gate = pr.pose_cost_gate(a, b, w_pos, w_ori)
    got = pr.pose_cost_f32(a, b, w_pos, w_ori).astype(np.float64)
    allowed = pr.nan_allowed(a[:, 3:7]) if w_ori else np.zeros(a.shape[0], bool)
    assert not np.isnan(got[~allowed]).any()
    if w_ori:
        zero = (a[:, 3:7] == 0).all(1)
        assert np.isnan(got[zero]).all() and np.isnan(ref[zero]).all()
    fin = ~np.isnan(got)
    err = np.abs(got - ref)
    assert (err[fin] <= gate[fin]).all(), np.flatnonzero(fin)[np.argmax((err[fin] / gate[fin]))]
    w = _worst(err[fin], gate[fin])
    print(f"float32 restatement w=({w_pos}, {w_ori}): worst err/gate {w:.3g}, NaN {int((~fin).sum())} of {a.shape[0]}")
    if w_ori:
        # the gate is not vacuous: within 100x of what the float32 order actually loses on these inputs
        assert w > 1e-2


@pytest.mark.parametrize("mutation", ["real_last", "yaw_m01", "no_two_s"])
def test_wrong_variants_miss_the_gate(mutation):
    a, b = _inputs(seed=5)
    ref = pr.pose_cost_ref(a, b, 1.0, 0.5)
    gate = pr.pose_cost_gate(a, b, 1.0, 0.5)
    bad = pr.pose_cost_f32(a, b, 1.0, 0.5, mutation=mutation).astype(np.float64)
    fin = np.isfinite(bad) & np.isfinite(ref)
    assert (np.abs(bad - ref)[fin] > gate[fin]).sum() >= 10


def test_nan_rule_bounds_the_float32_m20():
    """The float32 m20 can only leave [-1, 1] where the float64 |m20| >= 1 - 4 eps: e20 <= 8u for every quaternion."""
    q, _ = _all_quats()
    qq = q.astype(np.float64)
    m20 = pr.m20_ref(qq)
    r, i, j, k = qq.T
    t = 2.0 / (qq * qq).sum(1)
    e20 = 2 * pr.U * t * (np.abs(i * k) + np.abs(j * r)) + 6 * pr.U * np.abs(m20)
    assert e20.max() <= 8 * pr.U * (1 + 1e-6)
    f = q.astype(np.float32)
    m20_f = (np.float32(2.0) / (f * f).sum(1, dtype=np.float32)) * (f[:, 1] * f[:, 3] - f[:, 2] * f[:, 0])
    out = np.abs(m20_f.astype(np.float64)) > 1
    assert (np.abs(m20[out]) >= 1 - 4 * pr.EPS).all()


def test_oracle_cost_pose_within_the_gate(oracle):
    """The oracle's threaded cost_pose (the CPU arm's Objective) == the float64 reference within the gate, on the obs layout."""
    a, b = _inputs(seed=9)
    n = a.shape[0]
    obs = np.ascontiguousarray(a.T)                                   # (13, N): the obs rows
    av = obs.T                                                        # (N, 13) strides (4, 4N)
    goal = np.broadcast_to(np.array([0.4, -0.1, 0.6], np.float32), (n, 3))
    for bb, w_pos, w_ori in ((goal, 1.0, 0.5), (b, 40.0, 2.0), (None, 0.0, 0.5)):
        out = np.full(n, -1.0e30, np.float32)
        oracle.cost_pose(av, bb, w_pos, w_ori, out, 4)
        bref = None if bb is None else np.ascontiguousarray(bb)
        ref, gate = pr.pose_cost_ref(a, bref, w_pos, w_ori), pr.pose_cost_gate(a, bref, w_pos, w_ori)
        allowed = pr.nan_allowed(a[:, 3:7])
        got = out.astype(np.float64)
        assert not np.isnan(got[~allowed]).any() and (got != -1.0e30).all()
        fin = ~np.isnan(got)
        assert (np.abs(got - ref)[fin] <= gate[fin]).all()
