#!/usr/bin/env python
"""Generates the golden fixtures in this directory:  python tests/golden/make_golden.py <path to an mppi-isaac checkout>

* savgol_w9_o2.json : scipy.signal.savgol_filter(window_length=9, polyorder=2, mode='interp', axis=0) on seeded
  random (T, 7) sequences -- the filter mppi_torch applies when filter_u is set (SURVEY.md Appendix C).
* fk_reference_urdf.json : forward-kinematics known answers computed straight from the reference URDFs
  (<checkout>/assets/urdf/**) by an independent 4x4 homogeneous-transform walk (no model compiler).
"""
import json
import math
import os
import sys
import xml.etree.ElementTree as ET

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def savgol():
    from scipy.signal import savgol_filter
    rng = np.random.default_rng(20260924)
    cases = []
    for T in (9, 12, 20, 30):
        y = rng.normal(size=(T, 7)).astype(np.float32)
        f = savgol_filter(y.astype(np.float64), 9, 2, mode="interp", axis=0)
        cases.append(dict(y=y.tolist(), filtered=f.tolist()))
    with open(os.path.join(HERE, "savgol_w9_o2.json"), "w") as fh:
        json.dump(dict(source="scipy.signal.savgol_filter(9, 2, mode='interp', axis=0)", cases=cases), fh)


def _T(xyz, rpy):
    r, p, y = rpy
    Rx = np.array([[1, 0, 0], [0, math.cos(r), -math.sin(r)], [0, math.sin(r), math.cos(r)]])
    Ry = np.array([[math.cos(p), 0, math.sin(p)], [0, 1, 0], [-math.sin(p), 0, math.cos(p)]])
    Rz = np.array([[math.cos(y), -math.sin(y), 0], [math.sin(y), math.cos(y), 0], [0, 0, 1]])
    T = np.eye(4); T[:3, :3] = Rz @ Ry @ Rx; T[:3, 3] = xyz
    return T


def _axis_T(axis, q, prismatic):
    a = np.asarray(axis, float); a /= np.linalg.norm(a)
    T = np.eye(4)
    if prismatic:
        T[:3, 3] = a * q
        return T
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    T[:3, :3] = np.eye(3) + math.sin(q) * K + (1 - math.cos(q)) * K @ K
    return T


def urdf_fk(path, qmap, base=np.eye(4)):
    root = ET.parse(path).getroot()
    joints = [j for j in root.findall("joint") if j.find("parent") is not None]
    children = {j.find("child").get("link") for j in joints}
    links = [l.get("name") for l in root.findall("link")]
    out = {}

    def walk(link, T):
        out[link] = T
        for j in joints:
            if j.find("parent").get("link") != link:
                continue
            o = j.find("origin")
            xyz = [float(v) for v in (o.get("xyz", "0 0 0") if o is not None else "0 0 0").split()]
            rpy = [float(v) for v in (o.get("rpy", "0 0 0") if o is not None else "0 0 0").split()]
            Tj = T @ _T(xyz, rpy)
            if j.get("type") in ("revolute", "continuous", "prismatic"):
                ax = [float(v) for v in j.find("axis").get("xyz").split()]
                Tj = Tj @ _axis_T(ax, qmap.get(j.get("name"), 0.0), j.get("type") == "prismatic")
            walk(j.find("child").get("link"), Tj)

    roots = [l for l in links if l not in children]
    sizes = {}
    for r in roots:
        out.clear(); walk(r, base); sizes[r] = len(out)
    out.clear(); walk(max(roots, key=lambda r: sizes[r]), base)
    return {k: v.copy() for k, v in out.items()}


def fk():
    A = os.path.join(sys.argv[1], "assets", "urdf") + os.sep
    rng = np.random.default_rng(7)
    cases = []
    specs = [
        ("panda_isaac/robots/franka_panda_stick.urdf", [f"panda_joint{i}" for i in range(1, 8)], (0, 0, 0)),
        ("panda_isaac/robots/franka_panda_gripper.urdf", [f"panda_joint{i}" for i in range(1, 8)] + ["panda_finger_joint1", "panda_finger_joint2"], (0, 0, 0)),
        ("heijn/heijn.urdf", ["mobile_joint_x", "mobile_joint_y", "mobile_joint_theta"], (0.0, 1.5, 0.05)),
        ("point_robot.urdf", ["mobile_joint_x", "mobile_joint_y", "mobile_joint_theta"], (0, 0, 0)),
    ]
    for rel, names, base_p in specs:
        for trial in range(3):
            q = rng.uniform(-1.2, 1.2, len(names))
            if "panda" in rel:
                q[3] = rng.uniform(-2.8, -0.3); q[5] = rng.uniform(0.2, 3.0)
                if len(q) == 9:
                    q[7:] = rng.uniform(0, 0.04, 2)
            base = np.eye(4); base[:3, 3] = base_p
            Ts = urdf_fk(A + rel, dict(zip(names, q)), base)
            cases.append(dict(urdf=rel, base_pos=list(base_p), q=q.tolist(),
                              links={k: dict(p=v[:3, 3].tolist(), R=v[:3, :3].tolist()) for k, v in Ts.items()}))
    with open(os.path.join(HERE, "fk_reference_urdf.json"), "w") as fh:
        json.dump(dict(source="independent homogeneous-transform FK over the reference's assets/urdf", cases=cases), fh)


if __name__ == "__main__":
    savgol()
    fk()
    print("golden fixtures written to", HERE)
