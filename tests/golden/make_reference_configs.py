"""Regenerates reference_configs.json: what this package's loaders and URDF compiler make of the upstream mppi-isaac checkout
(its example task YAMLs, its conf/ actor YAMLs and three of its URDFs).  The test suite compares the shipped pre-compiled models
and the package's own conf/ against these values, so it needs no upstream checkout at test time.

    python tests/golden/make_reference_configs.py <path to an mppi-isaac checkout>
"""
import glob
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from mppi_isaac_b200.model.blob import build_scene  # noqa: E402
from mppi_isaac_b200.model.urdf import compile_urdf  # noqa: E402
from mppi_isaac_b200.utils.config_store import load_actor_cfgs, load_config  # noqa: E402

URDFS = ("point_robot.urdf", "heijn/heijn.urdf", "panda_isaac/robots/franka_panda_stick.urdf")
ACTOR_FIELDS = ("urdf_file", "init_joint_pose", "init_pos")


def main(ref):
    conf = [os.path.join(ref, "conf")]
    assets = [os.path.join(ref, "assets")]
    tasks = {}
    for t in sorted(glob.glob(os.path.join(ref, "examples", "*", "*.yaml"))):
        cfg = load_config(t, conf)
        name = os.path.relpath(t, os.path.join(ref, "examples"))
        entry = {"num_samples": cfg.mppi.num_samples, "horizon": cfg.mppi.horizon, "actors": list(cfg.actors),
                 "dt": cfg.isaacgym.dt, "substeps": cfg.isaacgym.substeps}
        try:
            sc = build_scene(load_actor_cfgs(cfg.actors, conf), assets_dirs=assets, substep=cfg.isaacgym.dt / cfg.isaacgym.substeps)
            entry["scene"] = [sc.model.nb, sc.nu]
        except NotImplementedError as e:
            entry["scene"] = str(e)
        tasks[name] = entry
    urdfs = {}
    for rel in URDFS:
        m = compile_urdf(os.path.join(ref, "assets", "urdf", rel))
        urdfs[rel] = {"mass": [float(v) for v in m.mass], "inertia_o": [[float(v) for v in row] for row in
                      [list(x.ravel()) for x in m.inertia_o]], "link_names": list(m.link_names), "dof_names": list(m.dof_names)}
    names = ["panda_stick", "goal"]
    actors = {n: {f: getattr(a, f) for f in ACTOR_FIELDS} for n, a in zip(names, load_actor_cfgs(names, conf))}
    out = dict(source="mppi-isaac examples/*/*.yaml, conf/actors and assets/urdf, read by this package's loaders",
               tasks=tasks, urdfs=urdfs, actors=actors)
    with open(os.path.join(HERE, "reference_configs.json"), "w") as fh:
        json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main(sys.argv[1])
