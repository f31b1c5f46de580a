"""Float64 reference of the fused pose cost (``mppib_cost_pose_kernel``, ``ops.pose_cost``) and its per-entry float32 gate.

The reference restates the route of the panda Objective of the reference project (examples/panda/planner.py:22-40) with
pytorch3d's public formulas, in float64 NumPy:

    cost = w_pos * |a[0:3] - b[0:3]|  +  w_ori * |matrix_to_euler_angles(quaternion_to_matrix(a[3:7]), "ZYX")[0:2]|

where the simulator's xyzw quaternion is handed to the REAL-FIRST ``quaternion_to_matrix`` as it is (column 3 is read as the
real part).  It imports neither ``ops``, ``objectives`` nor ``utils/conversions``, so a mistake shared by the kernel and the
torch formulation of the library does not cancel here.

The gate bounds, per entry, what float32 evaluation in the kernel's operation order may add to the float64 value.  The
library is compiled without ``--use_fast_math``, ``-ftz``, ``-prec-div=false`` or ``-prec-sqrt=false`` (``NVCC_FLAGS`` of
``__graft_entry__.py``), so every +, -, *, / and ``sqrtf`` is correctly rounded (relative error <= u = 2^-24, an FMA
contraction only removes roundings) and denormals are kept.  The two library functions are allowed their documented error
(CUDA math documentation, single precision): ``atan2f`` 3 ulp, ``asinf`` 2 ulp -- taken as 4 here.  One ulp of a float32
x is at most 2u|x|.  First-order terms, per row, with the float64 values of the (float32) inputs:

* position: the inputs are float32 numbers, so ``a - b`` is correctly rounded and brings no cancellation error of its own;
  squares, two additions, ``sqrtf`` and the weight give ``|d(w_pos dist)| <= 5u |w_pos| dist`` (4.5u to first order).
* matrix entries (real-first r, i, j, k; s = r^2+i^2+j^2+k^2, t = 2/s): ``two_s`` carries 5u, so
  ``e00 = 8u t(j^2+k^2) + u|m00|``, ``e10 = 2u t(|ij| + |kr|) + 6u|m10|``, ``e20 = 2u t(|ik| + |jr|) + 6u|m20|``.
* yaw = atan2(m10, m00): the vector (m00, m10) of length rho = hypot(m00, m10) moves by at most e = hypot(e00, e10), which
  turns it by at most asin(e / rho) (pi once e >= rho); |yaw| is continuous across the branch cut at +-pi and the cost only
  sees yaw^2.  Plus 3 ulp of atan2f.
* pitch = asin(-m20): e20 / sqrt(1 - (|m20| + e20)^2) by the mean value theorem while |m20| + e20 < 1, never more than
  acos(1 - e20) (the steepest interval of that length ends at 1).  Plus 4 ulp of asinf.  Since t(|ik| + |jr|) <= 1,
  e20 <= 8u = 4 eps: the float32 m20 can leave [-1, 1] -- and asinf return NaN -- only where the float64 |m20| >= 1 - 4 eps.
  The NaN rule of the tests allows it from 1 - 8 eps on.
* norm of (yaw, pitch): moves by at most hypot(E_yaw, E_pitch); squares, sum, ``sqrtf`` and the weight add 4u.
* the sum of both terms adds u|c|, accumulation into ``out`` u|out + c|.

The sum is scaled by (1 + 64u) for the second-order terms.  An absolute floor of 1e-30 (|w_pos| + |w_ori|) covers squares
that leave the normal range (differences below ~1e-19 m).
"""
import numpy as np

U = 2.0 ** -24                 # unit roundoff of float32
EPS = 2.0 ** -23               # float32 machine epsilon
ULP_ATAN2F, ULP_ASINF = 3, 4


def quaternion_to_matrix(q):
    """pytorch3d.transforms.quaternion_to_matrix in float64: q = (r, i, j, k) real first, any norm (two_s = 2 / |q|^2)."""
    q = np.asarray(q, np.float64)
    r, i, j, k = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        two_s = 2.0 / (q * q).sum(-1)
        o = np.stack([1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                      two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                      two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)], -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def matrix_to_euler_zyx(m):
    """pytorch3d.transforms.matrix_to_euler_angles(m, "ZYX") in float64: (angle about Z, about Y, about X).  m20 is clipped
    to [-1, 1]: the exact m20 of a quaternion lies there, only float64 rounding can put it one ulp past (NaN stays NaN)."""
    with np.errstate(invalid="ignore"):
        z = np.arctan2(m[..., 1, 0], m[..., 0, 0])
        y = np.arcsin(np.clip(-m[..., 2, 0], -1.0, 1.0))
        x = np.arctan2(m[..., 2, 1], m[..., 2, 2])
    return np.stack([z, y, x], -1)


def _cols(a, lo, hi):
    return np.asarray(a, np.float64)[:, lo:hi]


def orientation_ref(quat):
    """|euler_ZYX(R(q))[0:2]| for (N, 4) quaternions read real first; NaN for the zero quaternion and where |m20| > 1."""
    e = matrix_to_euler_zyx(quaternion_to_matrix(quat))
    return np.hypot(e[:, 0], e[:, 1])


def pose_cost_ref(a, b, w_pos, w_ori):
    """Float64 cost of (N, >=7) rows ``a`` (xyz, quaternion) against (N, >=3) ``b`` (None when w_pos == 0)."""
    n = np.asarray(a).shape[0]
    c = np.zeros(n)
    if w_pos != 0:
        c = c + float(w_pos) * np.linalg.norm(_cols(a, 0, 3) - _cols(b, 0, 3), axis=1)
    if w_ori != 0:
        c = c + float(w_ori) * orientation_ref(_cols(a, 3, 7))
    return c


def m20_ref(quat):
    return quaternion_to_matrix(quat)[:, 2, 0]


def nan_allowed(quat):
    """Rows where the float32 kernel may return NaN: the zero quaternion, and |m20| >= 1 - 8 eps (asinf of a float32 m20
    rounded past 1)."""
    q = np.asarray(quat, np.float64)
    zero = (q == 0).all(axis=1)
    with np.errstate(invalid="ignore"):
        edge = np.abs(m20_ref(q)) >= 1 - 8 * EPS
    return zero | edge


def pose_cost_gate(a, b, w_pos, w_ori, out0=None):
    """Per-entry bound on |float32 kernel - pose_cost_ref| (module docstring); ``out0``: the values accumulated into."""
    n = np.asarray(a).shape[0]
    wp, wo = abs(float(w_pos)), abs(float(w_ori))
    g = np.zeros(n)
    c = np.zeros(n)
    if w_pos != 0:
        dist = np.linalg.norm(_cols(a, 0, 3) - _cols(b, 0, 3), axis=1)
        g += 5 * U * wp * dist
        c += wp * dist
    if w_ori != 0:
        q = _cols(a, 3, 7)
        r, i, j, k = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        with np.errstate(divide="ignore", invalid="ignore"):
            t = 2.0 / (q * q).sum(1)
            m = quaternion_to_matrix(q)
            m00, m10, m20 = m[:, 0, 0], m[:, 1, 0], m[:, 2, 0]
            e00 = 8 * U * t * (j * j + k * k) + U * np.abs(m00)
            e10 = 2 * U * t * (np.abs(i * j) + np.abs(k * r)) + 6 * U * np.abs(m10)
            e20 = 2 * U * t * (np.abs(i * k) + np.abs(j * r)) + 6 * U * np.abs(m20)
            rho, ev = np.hypot(m00, m10), np.hypot(e00, e10)
            yaw, pitch = np.arctan2(m10, m00), np.arcsin(np.clip(-m20, -1, 1))
            e_yaw = np.where(ev < rho, np.arcsin(np.minimum(ev / rho, 1.0)), np.pi)
            e_yaw = e_yaw + ULP_ATAN2F * 2 * U * (np.abs(yaw) + e_yaw)
            top = np.abs(m20) + e20
            e_mvt = np.where(top < 1, e20 / np.sqrt(np.maximum(1 - top * top, 1e-300)), np.inf)
            e_pitch = np.minimum(e_mvt, np.arccos(np.clip(1 - e20, -1, 1)))
            e_pitch = e_pitch + ULP_ASINF * 2 * U * (np.abs(pitch) + e_pitch)
            ori = np.hypot(yaw, pitch)
            e_ori = np.hypot(e_yaw, e_pitch)
        g += wo * (e_ori + 4 * U * (ori + e_ori))
        c += wo * ori
    g += U * c
    if out0 is not None:
        g += U * (np.abs(np.asarray(out0, np.float64)) + c)
    return g * (1 + 64 * U) + 1e-30 * (wp + wo)


def pose_cost_f32(a, b, w_pos, w_ori, mutation=None):
    """Float32 NumPy restatement of the kernel's operation order.  atan2 / asin are evaluated in float64 from the float32
    matrix entries and rounded once (what a correctly rounded library would return).  ``mutation`` gives the wrong
    variants the gate must reject: "real_last" (xyzw read as such), "yaw_m01" (yaw from m01 instead of m10), "no_two_s"
    (2 instead of 2 / |q|^2)."""
    f = np.float32
    a = np.asarray(a, np.float32)
    c = np.zeros(a.shape[0], np.float32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if w_pos != 0:
            b = np.asarray(b, np.float32)
            dx, dy, dz = a[:, 0] - b[:, 0], a[:, 1] - b[:, 1], a[:, 2] - b[:, 2]
            c = f(w_pos) * np.sqrt(dx * dx + dy * dy + dz * dz)
        if w_ori != 0:
            r, qi, qj, qk = a[:, 3], a[:, 4], a[:, 5], a[:, 6]
            if mutation == "real_last":
                qi, qj, qk, r = a[:, 3], a[:, 4], a[:, 5], a[:, 6]
            two_s = f(2.0) / (r * r + qi * qi + qj * qj + qk * qk)
            if mutation == "no_two_s":
                two_s = np.full_like(r, 2.0)
            m00 = f(1.0) - two_s * (qj * qj + qk * qk)
            m10 = two_s * (qi * qj + qk * r)
            if mutation == "yaw_m01":
                m10 = two_s * (qi * qj - qk * r)
            m20 = two_s * (qi * qk - qj * r)
            yaw = np.arctan2(m10.astype(np.float64), m00.astype(np.float64)).astype(np.float32)
            pitch = np.arcsin(-m20.astype(np.float64)).astype(np.float32)
            c = c + f(w_ori) * np.sqrt(yaw * yaw + pitch * pitch)
    return c


# ---------------------------------------------------------------------------------------------------------------------
# inputs: quaternions in the order the kernel reads them, (r, i, j, k) = columns 3..6 of a row
# ---------------------------------------------------------------------------------------------------------------------
def quat_from_zyx(yaw, pitch, roll):
    """Real-first quaternion of R = Rz(yaw) Ry(pitch) Rx(roll), i.e. matrix_to_euler_zyx(quaternion_to_matrix(q)) = angles."""
    cy, sy, cp, sp, cr, sr = np.cos(yaw / 2), np.sin(yaw / 2), np.cos(pitch / 2), np.sin(pitch / 2), np.cos(roll / 2), np.sin(roll / 2)
    return np.stack([cy * cp * cr + sy * sp * sr, cy * cp * sr - sy * sp * cr, cy * sp * cr + sy * cp * sr, sy * cp * cr - cy * sp * sr], -1)


GIMBAL_DELTAS = (1e-1, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6, 1e-7, 0.0)


def edge_quaternions(seed=0, per_group=64):
    """Dict of named float32 (n, 4) quaternion groups: random unit ones, pitch +-(pi/2 - delta) for every GIMBAL_DELTAS, yaw
    at and next to +-pi (the identity xyzw quaternion read real first is yaw = pi), unit quaternions scaled by 10^-3 ... 10^3,
    q next to -q, and the zero quaternion."""
    rng = np.random.default_rng(seed)
    f = np.float32
    def unit(n):
        q = rng.normal(size=(n, 4))
        return q / np.linalg.norm(q, axis=1, keepdims=True)
    g = {"random": unit(per_group)}
    rows = []
    for d in GIMBAL_DELTAS:
        for sgn in (1.0, -1.0):
            yaw, roll = rng.uniform(-np.pi, np.pi, 4), rng.uniform(-np.pi, np.pi, 4)
            rows.append(quat_from_zyx(yaw, np.full(4, sgn * (np.pi / 2 - d)), roll))
            rows.append(quat_from_zyx(np.zeros(2), np.full(2, sgn * (np.pi / 2 - d)), np.zeros(2)))
    g["gimbal"] = np.concatenate(rows)
    yaws = np.array([np.pi, -np.pi, np.pi - 1e-7, -np.pi + 1e-7, np.pi - 1e-3, -np.pi + 1e-3])
    rows = [quat_from_zyx(yaws, rng.uniform(-1, 1, yaws.size), rng.uniform(-1, 1, yaws.size)),
            quat_from_zyx(yaws, np.zeros(yaws.size), np.zeros(yaws.size)),
            np.array([[0.0, 0.0, 0.0, 1.0], [0.0, 0.0, 0.0, -1.0], [1e-8, 0.0, 0.0, 1.0], [-1e-8, 0.0, 0.0, 1.0]])]
    g["yaw_pi"] = np.concatenate(rows)
    g["scaled"] = np.concatenate([unit(8) * 10.0 ** e for e in (-3, -2, -1, 1, 2, 3)])
    q = unit(per_group // 2).astype(f)
    g["q_negq"] = np.concatenate([q, -q])
    g["zero"] = np.zeros((2, 4))
    return {k: np.asarray(v, f) for k, v in g.items()}


def rows_with_quaternions(quat, seed=1, pos_scale=2.0):
    """(n, 13) float32 rows: random positions and velocities, the given quaternions in columns 3:7."""
    rng = np.random.default_rng(seed)
    n = quat.shape[0]
    a = rng.uniform(-pos_scale, pos_scale, (n, 13)).astype(np.float32)
    a[:, 3:7] = quat
    return a
