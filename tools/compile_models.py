#!/usr/bin/env python
"""Pre-compile the hot-path robots into mppi_isaac_b200/models_compiled/*.json.

The reference's URDF + collision meshes (assets/urdf/**, 96 MB) are not part of this repository, so the constant blocks
derived from them are generated once and committed.  Usage:  python tools/compile_models.py <mppi-isaac checkout>/assets
"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from mppi_isaac_b200.model.blob import compiled_path  # noqa: E402
from mppi_isaac_b200.model.urdf import compile_urdf, save_compiled  # noqa: E402

ROBOTS = [
    "point_robot.urdf",
    "heijn/heijn.urdf",
    "panda_isaac/robots/franka_panda.urdf",
    "panda_isaac/robots/franka_panda_stick.urdf",
    "panda_isaac/robots/franka_panda_gripper.urdf",
    "omni_panda/omniPandaWithGripper.urdf",
]
FLOATING = ["boxer/boxer.urdf", "albert/albert.urdf", "jackal/jackal.urdf"]   # differential-drive bases: compiled with the planar virtual-joint root
ROOT_MASS = {"jackal/jackal.urdf": 40.0}                              # ActorWrapper.mass of the actor file (conf/actors/jackal.yaml:8); default 1.0


def main():
    assets = sys.argv[1]
    for rel in ROBOTS:
        model = compile_urdf(os.path.join(assets, "urdf", rel), fixed_base=True)
        out = compiled_path(rel)
        save_compiled(model, out)
        print(f"{rel}: nb={model.nb} links={model.nlinks} -> {os.path.relpath(out)}")
    for rel in FLOATING:
        model = compile_urdf(os.path.join(assets, "urdf", rel), fixed_base=False, root_mass_override=ROOT_MASS.get(rel, 1.0))   # ActorWrapper.mass
        out = compiled_path(rel)
        save_compiled(model, out)
        print(f"{rel}: nb={model.nb} links={model.nlinks} planar base -> {os.path.relpath(out)}")


if __name__ == "__main__":
    main()
