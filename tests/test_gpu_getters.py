"""-m gpu: the ``RolloutSim`` getters on the device against the same getters over the CPU oracle, on the shipped scenes.

The Objective reads the rollout through these getters, so a wrong row, column, slot or stride in them is a wrong cost even
where the rollout kernel itself is right.  Each scene rolls the same actions through a GPU ``RolloutSim`` and one backed by
``oracle.backend.OracleBackend`` (float64 dynamics), in batched mode (one whole-horizon launch) and in stepwise mode (one
``step()`` per time step), and every getter the shipped Objectives call, ``get_dof_state``, ``_root_state``, every rigid body
and the contact force of every slotted body are compared under the gates of ``tests/test_gpu_parity.py``: positions 1e-4 m,
quaternions 2e-5 up to sign (1e-4 for free bodies, the lock-step gate of their root state), link velocities and DOF rows
2e-3 (5e-3 for planar-base robots), net contact forces 5e-2 * max(1, |F|).  Contact scenes use a horizon of 3 steps, as
contact onsets make longer free-running comparisons statistical."""
import copy

import numpy as np
import pytest
import torch

from scenes import boxer_cfg, panda_cfg, pick_cfg, point_cfg, push_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _shipped(name):
    from mppi_isaac_b200 import load_isaacgym_config
    return copy.deepcopy(load_isaacgym_config(name))


def _jackal_cfg():
    from mppi_isaac_b200.utils.config_store import MPPIConfig
    cfg = _shipped("config_point_robot_b200")
    cfg.actors = ["jackal", "goal"]
    cfg.initial_actor_positions = [[0.0, 0.0, 0.05]]
    cfg.mppi = MPPIConfig(num_samples=64, horizon=5, mppi_mode="simple", sampling_method="random", noise_sigma=[[1.0, 0], [0, 1.0]],
                          u_min=[-1.0, -2.0], u_max=[1.0, 2.0], lambda_=0.1)
    return cfg


def _scene(name):
    """(config, Objective, horizon, planar base?) of each shipped scene."""
    from mppi_isaac_b200.objectives import PandaPickObjective, PandaReachObjective, PointReachObjective, PushObjective
    if name == "point":
        return point_cfg(K=64, T=5), PointReachObjective(), 5, False
    if name == "panda":
        return panda_cfg(K=64, T=9, filter_u=False), PandaReachObjective(), 9, False
    if name == "push":
        return push_cfg(K=64, T=3), PushObjective(), 3, False
    if name == "pick":
        return pick_cfg(K=64, T=3, filter_u=False), PandaPickObjective(), 3, False
    if name == "boxer":
        return boxer_cfg(K=64, T=3, filter_u=False), PushObjective(robot="boxer", link="ee_link"), 3, True
    if name == "omnipanda":
        return _shipped("config_omnipanda_pick_b200"), PandaPickObjective(actor="omnipanda", link="panda_hand"), 3, False
    if name == "albert":
        return _shipped("config_albert_b200"), PandaReachObjective(actor="albert", link="mmrobot_link7"), 5, True
    if name == "jackal":
        return _jackal_cfg(), PointReachObjective(actor="jackal", link="ee_link"), 5, True
    raise ValueError(name)


SCENES = ["point", "panda", "push", "pick", "boxer", "omnipanda", "albert", "jackal"]
K = 64


def _sim(cfg, T, device, backend=None, observe="all"):
    from mppi_isaac_b200.planner.rollout_sim import RolloutSim
    mc = copy.copy(cfg.mppi)
    mc.num_samples, mc.horizon, mc.device, mc.filter_u = K, T, device, False
    return RolloutSim(cfg.isaacgym, actors=cfg.actors, init_positions=cfg.initial_actor_positions, num_envs=K, device=device, horizon=T,
                      mppi_cfg=mc, conf_dirs=getattr(cfg, "conf_dirs", None) or None, backend=backend, observe=observe)


def _actions(sim, T, seed):
    nu = sim.scene.nu
    lo = np.resize(np.asarray(sim.params.u_min, np.float32)[:nu], nu)
    hi = np.resize(np.asarray(sim.params.u_max, np.float32)[:nu], nu)
    u = np.random.default_rng(seed).uniform(0.0, 1.0, (T, nu, K)).astype(np.float32)
    return lo[None, :, None] + (hi - lo)[None, :, None] * u


def _getters(sim, objective_names):
    """name -> (tensor, kind) for every getter compared; kind picks the gate."""
    sc = sim.scene
    out = {"dof_state": (sim.get_dof_state(), "dof"), "root_state": (sim._root_state, "root")}
    for b in range(sc.num_bodies):
        out[f"body{b}"] = (sim.get_rigid_body_by_rigid_body_index(b), "root" if b in _free_bodies(sc) else "link")
    for rb, slot in sc.contact_slot.items():
        a = next(i for i in range(len(sc.body_names)) if sc.body_offset[i] <= rb < sc.body_offset[i] + len(sc.body_names[i]))
        out[f"force:{sc.actor_names[a]}/{sc.body_names[a][rb - sc.body_offset[a]]}"] = (
            sim.get_actor_contact_forces_by_name(sc.actor_names[a], sc.body_names[a][rb - sc.body_offset[a]]), "force")
    for kind, (actor, link) in objective_names:
        if kind == "link":
            out[f"link:{actor}/{link}"] = (sim.get_actor_link_by_name(actor, link), "link")
        else:
            for g in ("position", "velocity", "orientation"):
                out[f"{g}:{actor}"] = (getattr(sim, f"get_actor_{g}_by_name")(actor), g)
    return out


def _free_bodies(sc):
    return {sc.body_offset[a] for a in sc.free_actor}


def _objective_names(sim, objective):
    """The (actor, link) pairs and actors an Objective reads, recorded by calling it against a recording facade."""
    names = []

    class Rec:
        def __getattr__(self, k):
            return getattr(sim, k)

        def get_actor_link_by_name(self, actor_name, link_name):
            names.append(("link", (actor_name, link_name)))
            return sim.get_actor_link_by_name(actor_name, link_name)

        def _actor(self, g, name):
            names.append(("actor", (name, None)))
            return getattr(sim, f"get_actor_{g}_by_name")(name)

        def get_actor_position_by_name(self, name):
            return self._actor("position", name)

        def get_actor_velocity_by_name(self, name):
            return self._actor("velocity", name)

        def get_actor_orientation_by_name(self, name):
            return self._actor("orientation", name)

    objective.compute_cost(Rec())
    return list(dict.fromkeys(names))


def _gates(planar):
    return {"pos": 1e-4, "quat": 2e-5, "quat_free": 1e-4, "vel": 5e-3 if planar else 2e-3}


def _cmp13(a, b, g, free, what):
    worst = {}
    worst["pos"] = float(np.abs(a[..., 0:3] - b[..., 0:3]).max())
    q = np.minimum(np.abs(a[..., 3:7] - b[..., 3:7]), np.abs(a[..., 3:7] + b[..., 3:7])).max()
    worst["quat"] = float(q)
    worst["vel"] = float(np.abs(a[..., 7:13] - b[..., 7:13]).max()) if a.shape[-1] >= 13 else 0.0
    assert worst["pos"] <= g["pos"], (what, worst)
    assert worst["quat"] <= (g["quat_free"] if free else g["quat"]), (what, worst)
    assert worst["vel"] <= g["vel"], (what, worst)
    return max(worst["pos"] / g["pos"], worst["quat"] / (g["quat_free"] if free else g["quat"]), worst["vel"] / g["vel"])


def compare(gpu, cpu, names, planar, label):
    g = _gates(planar)
    G, C = _getters(gpu, names), _getters(cpu, names)
    assert G.keys() == C.keys()
    worst = 0.0
    for key, (tg, kind) in G.items():
        tc = C[key][0]
        assert tg.shape == tc.shape, key
        a, b = tg.detach().cpu().numpy().astype(np.float64), tc.detach().numpy().astype(np.float64)
        assert np.isfinite(a).all(), key
        if kind == "dof":
            err = float(np.abs(a - b).max())
            assert err <= g["vel"], (label, key, err)
            worst = max(worst, err / g["vel"])
        elif kind == "force":
            err, lim = float(np.abs(a - b).max()), 5e-2 * max(1.0, float(np.abs(b).max()))
            assert err <= lim, (label, key, err, lim)
            worst = max(worst, err / lim)
        elif kind == "root":
            free = gpu.scene.free_actor
            for ai in range(a.shape[1]) if a.ndim == 3 else [None]:
                aa, bb = (a, b) if ai is None else (a[:, ai], b[:, ai])
                worst = max(worst, _cmp13(aa, bb, g, ai is None or ai in free, (label, key, ai)))
        elif kind in ("link", "position", "velocity", "orientation"):
            if kind == "link":
                worst = max(worst, _cmp13(a, b, g, False, (label, key)))
            else:
                lim = {"position": g["pos"], "velocity": g["vel"], "orientation": g["quat_free"]}[kind]
                err = float((np.minimum(np.abs(a - b), np.abs(a + b)) if kind == "orientation" else np.abs(a - b)).max())
                assert err <= lim, (label, key, err)
                worst = max(worst, err / lim)
    return worst


@pytest.mark.parametrize("scene", SCENES)
def test_getters_on_device_match_the_oracle(scene):
    from oracle.backend import OracleBackend
    cfg, objective, T, planar = _scene(scene)
    gpu = _sim(cfg, T, DEV)
    cpu = _sim(cfg, T, "cpu", backend=OracleBackend(use_double=True, nthreads=8))
    names = _objective_names(cpu, objective)
    actions = _actions(gpu, T, seed=len(scene))
    worst = {}
    # batched: one whole-horizon launch, (T*K, w) views
    gpu.rollout_all(torch.from_numpy(actions).to(DEV))
    cpu.rollout_all(torch.from_numpy(actions))
    worst["batched"] = compare(gpu, cpu, names, planar, "batched")
    # stepwise: the reference protocol, (K, w) views; the first read comes before any step
    for s in (gpu, cpu):
        s.begin_step_mode()
    worst["initial"] = compare(gpu, cpu, names, planar, "before step 0")
    for t in range(T):
        for s, dev in ((gpu, DEV), (cpu, "cpu")):
            s.apply_robot_cmd(torch.from_numpy(actions[t].T.copy()).to(dev))
            s.step()
        worst["stepwise"] = max(worst.get("stepwise", 0.0), compare(gpu, cpu, names, planar, f"step {t}"))
    print(f"[getters] {scene}: worst err/gate " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


@pytest.mark.parametrize("scene", SCENES)
def test_traced_rows_equal_observe_all_and_initial_observation(scene):
    """observe='auto' (only the traced rows are written) gives bit for bit the rows observe='all' gives; in stepwise mode a
    read before the first step() is the observe-only launch (nsteps = 0) of the starting state."""
    cfg, objective, T, _ = _scene(scene)
    full = _sim(cfg, T, DEV, observe="all")
    auto = _sim(cfg, T, DEV, observe="auto")
    auto.trace(objective.compute_cost)
    assert auto._obs_items and len(auto._obs_items) <= len(full._obs_items)
    actions = torch.from_numpy(_actions(full, T, seed=7)).to(DEV)
    for s in (full, auto):
        s.rollout_all(actions)
    torch.cuda.synchronize()

    def same_rows(label):
        for item in auto._obs_items:
            ra, rf = auto._obs_row[item], full._obs_row[item]
            w = _width(auto, item)
            assert torch.equal(auto._obs[ra:ra + w], full._obs[rf:rf + w]), (label, item)
    same_rows("batched")
    assert torch.equal(objective.compute_cost(auto).view(torch.int32), objective.compute_cost(full).view(torch.int32))
    for s in (full, auto):
        s.begin_step_mode()
    first = objective.compute_cost(auto)                              # triggers the observe-only launch of the start state
    full.get_dof_state()                                              # and in the observe='all' sim
    torch.cuda.synchronize()
    same_rows("before step 0")
    # the same rows from an explicit observe-only launch of the broadcast start state
    st = torch.zeros_like(auto._state)
    nd2 = 2 * auto.scene.ndof
    st[:nd2] = auto._state0[:, None]
    for actor_idx, f in auto.scene.free_actor.items():
        st[nd2 + 13 * f: nd2 + 13 * (f + 1)] = auto._root0[actor_idx][:, None]
    obs = torch.full_like(auto._obs, float("nan"))
    auto.backend.rollout(None, st, torch.zeros_like(auto._cmd), 0, 0, obs, act_t0=0, root0=auto._root0)
    torch.cuda.synchronize()
    for item in auto._obs_items:
        r0, w = auto._obs_row[item], _width(auto, item)
        assert torch.equal(obs[r0:r0 + w, 0], auto._obs[r0:r0 + w, 0]), item
    assert torch.equal(first.view(torch.int32), objective.compute_cost(auto).view(torch.int32))
    for s in (full, auto):
        s.apply_robot_cmd(actions[0].t())
        s.step()
    same_rows("step 0")


def _width(sim, item):
    from mppi_isaac_b200.model.blob import obs_width
    return obs_width(item[0], sim.scene.ndof)
