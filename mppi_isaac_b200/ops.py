"""Fused cost terms for Objectives (optional).

An Objective is user code: anything written with torch ops on the views ``RolloutSim`` hands out works.  The terms below
are the ones the reference's example Objectives are made of, as single CUDA kernels of ``libmppib.so`` -- the pose-reach
cost of ``examples/panda/planner.py:22-40`` costs ~28 element-wise torch launches (~61 us at K = 10 000, T = 30 on an H100) and
one launch (~4 us) here.  CPU tensors (the checker backend of the tests) take the torch formulation.
"""
import ctypes as C

import torch


def _zyx_first_two(quat: torch.Tensor) -> torch.Tensor:
    """|euler_ZYX(R(q))[:, 0:2]| for a (N,4) quaternion handed REAL-FIRST to the matrix formula (so the xyzw tensor of
    the simulator is read as w=x, x=y, y=z, z=w: the reference's literal arithmetic, Appendix A #11).  Only the three
    matrix entries the two angles need are formed -- same numbers as
    ``matrix_to_euler_angles(quaternion_to_matrix(q), "ZYX")[:, 0:2]`` with a fraction of the element-wise kernels."""
    r, i, j, k = quat[:, 0], quat[:, 1], quat[:, 2], quat[:, 3]
    two_s = 2.0 / (quat * quat).sum(-1)
    m00 = 1 - two_s * (j * j + k * k)
    m10 = two_s * (i * j + k * r)
    m20 = two_s * (i * k - j * r)
    yaw = torch.atan2(m10, m00)
    pitch = torch.asin(-m20)
    return torch.sqrt(yaw * yaw + pitch * pitch)


def pose_cost_torch(a: torch.Tensor, b, w_pos: float, w_ori: float) -> torch.Tensor:
    c = 0.0
    if w_pos:
        c = w_pos * torch.linalg.norm(a[:, 0:3] - b[:, 0:3], axis=1)
    if w_ori:
        c = c + w_ori * _zyx_first_two(a[:, 3:7])
    return c


def pose_cost(a: torch.Tensor, b, w_pos: float, w_ori: float, out: torch.Tensor = None, accumulate: bool = False) -> torch.Tensor:
    """``w_pos * |a[:, 0:3] - b[:, 0:3]| + w_ori * |euler_ZYX(R(a[:, 3:7]))[:2]|`` row-wise, one kernel.

    ``a``: (N, >=7) link / root state view (xyz, quaternion xyzw); ``b``: (N, >=3) view (may be a stride-0 expand of
    one row) or None when ``w_pos == 0``.  Any strides are accepted; the obs layout (stride 1 along N) is coalesced."""
    if not a.is_cuda:
        res = pose_cost_torch(a, b, w_pos, w_ori)
        if out is None:
            return res
        return out.add_(res) if accumulate else out.copy_(res)
    from .backend import load_library
    lib = load_library()
    n = a.shape[0]
    if a.dtype != torch.float32 or (b is not None and (b.dtype != torch.float32 or b.device != a.device)):
        raise TypeError("pose_cost: float32 tensors on one device expected")
    if w_ori and a.shape[1] < 7:
        raise ValueError("pose_cost: the orientation term needs the quaternion columns 3:7")
    if out is None:
        out = torch.empty((n,), dtype=torch.float32, device=a.device)
        accumulate = False
    elif out.dtype != torch.float32 or not out.is_contiguous() or out.numel() != n:
        raise ValueError("pose_cost: `out` must be a contiguous float32 tensor of N elements")
    bp, bsi, bsr = (C.c_void_p(b.data_ptr()), b.stride(0), b.stride(1)) if b is not None else (C.c_void_p(0), 0, 0)
    rc = lib.mppib_cost_pose(C.c_int64(n), C.c_void_p(a.data_ptr()), C.c_int64(a.stride(0)), C.c_int64(a.stride(1)), bp, C.c_int64(bsi),
                             C.c_int64(bsr), C.c_float(w_pos), C.c_float(w_ori), C.c_void_p(out.data_ptr()), C.c_int32(1 if accumulate else 0),
                             C.c_void_p(torch.cuda.current_stream(a.device).cuda_stream))
    if rc != 0:
        raise RuntimeError(f"mppib_cost_pose failed ({rc}): {lib.mppib_last_error().decode()}")
    return out
