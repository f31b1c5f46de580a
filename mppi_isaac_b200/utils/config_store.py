"""Config schema and loader for the rollout path.

Mirrors the reference's Hydra structured configs
(``mppiisaac/utils/config_store.py:9-18`` ``ExampleConfig``; ``MPPIConfig`` field names from
``benchmarks/panda_arm/setup/mppi.yaml:5-77`` + ``conf/mppi/omnipanda_effort.yaml:29-31``;
``IsaacGymConfig`` ``mppiisaac/planner/isaacgym_wrapper.py:10-18``; ``ActorWrapper``
``isaacgym_wrapper.py:49-77``) without depending on hydra/omegaconf, which are not installed
in the build image.  The loader composes the same YAML trees: a task file with a ``defaults``
list (``- mppi: panda``, ``- isaacgym: normal``) resolved against ``<conf>/<group>/<name>.yaml``,
``base_*`` defaults coming from the dataclasses below, and ``key=value`` dotted overrides.
Objects that already look like a config (an OmegaConf ``DictConfig`` or any attribute bag)
are accepted unchanged by the planner.
"""
from __future__ import annotations

import copy
import os
from dataclasses import dataclass, field, fields, is_dataclass
from typing import Any, List, Optional

import yaml

PKG_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILTIN_CONF = os.path.join(PKG_DIR, "conf")


@dataclass
class MPPIConfig:
    num_samples: int = 100
    horizon: int = 30
    mppi_mode: str = "halton-spline"     # halton-spline | simple | cem | smooth
    sampling_method: str = "halton"      # halton | random | colored
    noise_sigma: Optional[List[List[float]]] = None
    noise_mu: Optional[List[float]] = None
    device: str = "cuda:0"
    lambda_: float = 1.0
    update_lambda: bool = False
    update_cov: bool = False
    cov_type: str = "diag"               # update rule of update_cov: diag | full | horizon (T*nu <= 256) (DESIGN.md section 2)
    noise_beta: float = 2.0              # sampling_method colored: power-law exponent of the temporal spectrum, 0 = white (DESIGN.md section 2)
    n_elites: int = 10                   # mppi_mode cem (iCEM, DESIGN.md section 2): elites E in 1 .. 128
    elite_momentum: float = 0.1          # mppi_mode cem: momentum alpha of the mean and sigma updates, in [0, 1]
    keep_elites: float = 0.3             # mppi_mode cem: fraction xi of the elites carried into the next samples, floor(xi E) rows
    cem_iterations: int = 3              # mppi_mode cem: sample / roll out / update iterations per plan, at least 1
    smooth_weight: float = 0.0           # mppi_mode smooth (DESIGN.md section 2): omega >= 0 of the cost omega sum_t |a_t - a_{t-1}|^2
    du_min: Optional[List[float]] = None  # mppi_mode smooth: bounds of the action derivative (length 1 broadcasts; None: unbounded)
    du_max: Optional[List[float]] = None
    n_worlds: int = 1                    # risk-aware MPPI (DESIGN.md section 2): R rollouts per control sample in R fixed worlds, 1 .. 32
    cvar_alpha: float = 1.0              # risk-aware MPPI: a control scores the mean of its ceil(alpha R) worst world costs, alpha in (0, 1]
    n_modes: int = 1                     # multi-modal MPPI (DESIGN.md section 2): M nominal sequences planned side by side, 1 .. 16, K / M >= 32 samples each
    mode_switch_margin: float = 0.0      # multi-modal MPPI: keep the executed mode while its free energy is within this margin (cost units) of the lowest
    anneal_iterations: int = 1           # annealed MPPI (DESIGN.md section 2): N MPPI iterations per plan, 1 .. 16
    anneal_iter_decay: float = 1.0       # annealed MPPI: c_i in (0, 1], the noise std factor per iteration
    anneal_horizon_decay: float = 1.0    # annealed MPPI: c_h in (0, 1], the noise std factor per step towards the start of the horizon
    control_knots: int = 0               # spline MPPI (DESIGN.md section 2): P control knots per horizon, interpolated to every step; 0 = off
    spline_degree: int = 1               # spline MPPI: B-spline degree d in 1 .. 3, P in d + 1 .. horizon
    constraint_mode: str = "none"        # constrained MPPI (DESIGN.md section 2): "none" or "feasible_first" (needs Objective.compute_constraint)
    constraint_tol: float = 0.0          # constrained MPPI: a sample is feasible when its summed violation is <= tol (finite, >= 0)
    constraint_lambda: Optional[float] = None   # constrained MPPI: temperature of the fallback over violations when no sample is feasible; None: lambda_
    lambda_mode: str = "fixed"           # ESS-targeted temperature (DESIGN.md section 2): "fixed" (lambda_) or "ess" (chosen on the device every plan)
    ess_target: float = 0.01             # lambda_mode ess: rho in (0, 1], the share of the valid samples the weights keep (Kish ESS = rho N)
    u_min: Optional[List[float]] = None
    u_max: Optional[List[float]] = None
    u_init: float = 0.0
    U_init: Optional[List[List[float]]] = None
    u_scale: float = 1.0
    u_per_command: int = 1
    rollout_var_discount: float = 0.95
    sample_null_action: bool = False
    noise_abs_cost: bool = False
    filter_u: bool = False
    use_priors: bool = False
    eta_u_bound: float = 10.0
    eta_l_bound: float = 5.0
    seed_val: int = 0


@dataclass
class IsaacGymConfig:
    dt: float = 0.05
    substeps: int = 2
    use_gpu_pipeline: bool = True
    num_client_threads: int = 0
    viewer: bool = False
    num_obstacles: int = 10
    spacing: float = 6.0


@dataclass
class ActorWrapper:
    type: str
    name: str
    dof_mode: str = "velocity"
    init_pos: List[float] = field(default_factory=lambda: [0, 0, 0])
    init_ori: List[float] = field(default_factory=lambda: [0, 0, 0, 1])
    size: List[float] = field(default_factory=lambda: [0.1, 0.1, 0.1])
    mass: float = 1.0
    color: List[float] = field(default_factory=lambda: [1.0, 1.0, 1.0])
    fixed: bool = False
    collision: bool = True
    friction: float = 1.0
    handle: Optional[int] = None
    flip_visual: bool = False
    urdf_file: Optional[str] = None
    visualize_link: Optional[str] = None
    gravity: bool = True
    differential_drive: bool = False
    init_joint_pose: Optional[List[float]] = None
    wheel_radius: Optional[float] = None
    wheel_base: Optional[float] = None
    wheel_count: Optional[float] = None
    left_wheel_joints: Optional[List[str]] = None
    right_wheel_joints: Optional[List[str]] = None
    caster_links: Optional[List[str]] = None
    noise_sigma_size: Optional[List[float]] = None
    noise_percentage_mass: float = 0.0
    noise_percentage_friction: float = 0.0


@dataclass
class ExampleConfig:
    render: bool = False
    n_steps: int = 1000
    mppi: MPPIConfig = field(default_factory=MPPIConfig)
    isaacgym: IsaacGymConfig = field(default_factory=IsaacGymConfig)
    goal: List[float] = field(default_factory=list)
    nx: int = 0
    actors: List[str] = field(default_factory=list)
    initial_actor_positions: List[List[float]] = field(default_factory=list)
    # extension: extra places to look for conf/actors and assets/urdf (user trees, e.g. the reference checkout)
    conf_dirs: List[str] = field(default_factory=list)
    assets_dirs: List[str] = field(default_factory=list)


def _fill(dc_type, data: dict):
    names = {f.name for f in fields(dc_type)}
    unknown = set(data) - names
    if unknown:
        raise KeyError(f"unknown keys for {dc_type.__name__}: {sorted(unknown)}")
    return dc_type(**data)


def conf_search_path(extra: Optional[List[str]] = None) -> List[str]:
    dirs = list(extra or [])
    env = os.environ.get("MPPI_ISAAC_CONF")
    if env:
        dirs += env.split(os.pathsep)
    dirs.append(BUILTIN_CONF)
    return [d for d in dirs if d and os.path.isdir(d)]


def _find(group: str, name: str, dirs: List[str]) -> str:
    for d in dirs:
        p = os.path.join(d, group, name + ".yaml")
        if os.path.exists(p):
            return p
    raise FileNotFoundError(f"config '{group}/{name}.yaml' not found in {dirs}")


def _load_group(group: str, name: str, dirs: List[str]) -> dict:
    with open(_find(group, name, dirs)) as f:
        d = yaml.safe_load(f) or {}
    d.pop("defaults", None)  # only ever "- base_<group>": the dataclass defaults
    return d


def _set_dotted(d: dict, key: str, value):
    parts = key.split(".")
    for p in parts[:-1]:
        d = d.setdefault(p, {})
    d[parts[-1]] = value


def load_config(task_file: str, conf_dirs: Optional[List[str]] = None, overrides: Optional[List[str]] = None) -> ExampleConfig:
    """Compose a task YAML (e.g. the reference's ``examples/panda/config_panda.yaml``)."""
    dirs = conf_search_path(conf_dirs)
    with open(task_file) as f:
        top = yaml.safe_load(f) or {}
    top.pop("hydra", None)
    merged: dict = {}
    for item in top.pop("defaults", []) or []:
        if isinstance(item, dict):
            for group, name in item.items():
                merged[group] = _load_group(group, name, dirs)
    for k, v in top.items():
        if isinstance(v, dict) and isinstance(merged.get(k), dict):
            merged[k].update(v)
        else:
            merged[k] = v
    for ov in overrides or []:
        k, v = ov.split("=", 1)
        _set_dotted(merged, k, yaml.safe_load(v))
    merged["mppi"] = _fill(MPPIConfig, merged.get("mppi", {}))
    merged["isaacgym"] = _fill(IsaacGymConfig, merged.get("isaacgym", {}))
    cfg = _fill(ExampleConfig, merged)
    cfg.conf_dirs = list(conf_dirs or [])
    return cfg


def load_isaacgym_config(name: str, conf_dirs: Optional[List[str]] = None) -> ExampleConfig:
    """Reference entry point name (config_store.py:42-46): compose ``<conf>/<name>.yaml``."""
    for d in conf_search_path(conf_dirs):
        p = os.path.join(d, name + ".yaml")
        if os.path.exists(p):
            return load_config(p, conf_dirs)
    raise FileNotFoundError(name)


def load_actor_cfgs(actors: List[str], conf_dirs: Optional[List[str]] = None) -> List[ActorWrapper]:
    """``isaacgym_utils.py:70-78``: plain YAML -> ActorWrapper(**d) per actor name."""
    dirs = conf_search_path(conf_dirs)
    out = []
    for a in actors:
        if isinstance(a, ActorWrapper):
            out.append(copy.deepcopy(a))
            continue
        with open(_find("actors", a, dirs)) as f:
            d = yaml.safe_load(f)
        if d.get("handle") == "None":  # the shipped files write `handle: None` (a YAML string)
            d["handle"] = None
        out.append(_fill(ActorWrapper, d))
    return out


def to_plain(cfg: Any):
    """dataclass / DictConfig / dict -> plain nested python containers."""
    if is_dataclass(cfg):
        return {f.name: to_plain(getattr(cfg, f.name)) for f in fields(cfg)}
    if isinstance(cfg, dict):
        return {k: to_plain(v) for k, v in cfg.items()}
    if isinstance(cfg, (list, tuple)):
        return [to_plain(v) for v in cfg]
    if hasattr(cfg, "items") and hasattr(cfg, "keys"):
        return {k: to_plain(cfg[k]) for k in cfg.keys()}
    if hasattr(cfg, "__iter__") and not isinstance(cfg, (str, bytes)):
        return [to_plain(v) for v in cfg]
    return cfg
