"""Orientation helpers used by Objectives.

``quaternion_to_yaw`` restates ``mppiisaac/utils/conversions.py:4-11`` (xyzw quaternions).
``quaternion_to_matrix`` / ``matrix_to_euler_angles`` restate the two pytorch3d 0.3.0 functions the panda
Objectives call (``examples/panda/planner.py:30-32``); pytorch3d is not installed here.  NOTE the reference
feeds an *xyzw* quaternion into pytorch3d's *wxyz* API (SURVEY.md Appendix A #11) -- ``quaternion_to_matrix``
keeps pytorch3d's real-first convention so that the literal arithmetic of those Objectives is reproduced.

Provenance: ``quaternion_to_matrix``, ``_angle_from_tan`` and ``matrix_to_euler_angles`` follow the public formulas of
pytorch3d's ``transforms/rotation_conversions.py`` (Meta Platforms, BSD licence) -- third-party code the reference depends on,
not code of the reference repository; they have to reproduce that library's numbers exactly, so their structure is the library's.
"""
import torch


def quaternion_to_yaw(quat: torch.Tensor) -> torch.Tensor:
    x, y, z, w = quat[:, 0], quat[:, 1], quat[:, 2], quat[:, -1]
    return torch.atan2(2.0 * (w * z + x * y), w * w + x * x - y * y - z * z)


def quaternion_to_matrix(quaternions: torch.Tensor) -> torch.Tensor:
    """Real-part-first quaternions (..., 4) -> rotation matrices (..., 3, 3)."""
    r, i, j, k = torch.unbind(quaternions, -1)
    two_s = 2.0 / (quaternions * quaternions).sum(-1)
    o = torch.stack(
        (
            1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
            two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
            two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j),
        ),
        -1,
    )
    return o.reshape(quaternions.shape[:-1] + (3, 3))


def _angle_from_tan(axis: str, other_axis: str, data, horizontal: bool, tait_bryan: bool):
    i1, i2 = {"X": (2, 1), "Y": (0, 2), "Z": (1, 0)}[axis]
    if horizontal:
        i2, i1 = i1, i2
    even = (axis + other_axis) in ["XY", "YZ", "ZX"]
    if horizontal == even:
        return torch.atan2(data[..., i1], data[..., i2])
    if tait_bryan:
        return torch.atan2(-data[..., i2], data[..., i1])
    return torch.atan2(data[..., i2], -data[..., i1])


def matrix_to_euler_angles(matrix: torch.Tensor, convention: str) -> torch.Tensor:
    """Rotation matrices (..., 3, 3) -> Euler angles (..., 3) for a 3-letter convention such as "ZYX"."""
    idx = {"X": 0, "Y": 1, "Z": 2}
    i0, i2 = idx[convention[0]], idx[convention[2]]
    tait_bryan = i0 != i2
    if tait_bryan:
        central = torch.asin(matrix[..., i0, i2] * (-1.0 if i0 - i2 in [-1, 2] else 1.0))
    else:
        central = torch.acos(matrix[..., i0, i0])
    o = (
        _angle_from_tan(convention[0], convention[1], matrix[..., i2], False, tait_bryan),
        central,
        _angle_from_tan(convention[2], convention[1], matrix[..., i0, :], True, tait_bryan),
    )
    return torch.stack(o, -1)
