"""-m gpu: the CUDA path against the oracle AT THE BASELINE SIZES (C2* K = 10 000 / T = 30, C3 K = 4 000 / T = 20, the C4 shard
K = 4 000 / T = 25, the C5 shard K = 8 192 / T = 30 -- the two-wave, 222 KB shared-memory case -- and C5's full K = 65 536).

Contact-free rollouts are compared free-running over the whole horizon; contact rollouts in lock-step (the oracle's state is
re-injected before every model step: contact dynamics are chaotic, SURVEY.md 8(c)), with the tolerances of test_gpu_parity.py.
The oracle runs on all host cores; every test finishes in seconds on the GPU box."""
import copy
import os

import numpy as np
import pytest
import torch

from scenes import boxer_setup, panda_setup, pick_cfg, push_setup

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NTH = max(1, os.cpu_count() or 1)


def gpu_backend(sc, p):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(sc.model, p)
    return be


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def test_c2_headline_size_free_running_parity(oracle):
    """BASELINE C2*: panda 7-DoF, K = 10 000, T = 30 -- every rollout, every step, against the float64 oracle."""
    K, T = 10000, 30
    sc, p, state0 = panda_setup(K=K, T=T)
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(11)
    actions = rng.uniform(-0.2, 0.2, (T, sc.nu, K)).astype(np.float32)
    obs, state = torch.zeros((be.obs_size(), T, K), device=DEV), torch.zeros((be.state_size(), K), device=DEV)
    be.rollout(dev(state0), state, dev(actions), 0, T, obs)
    st_ref, obs_ref = oracle.rollout(sc.model, p, state0, actions, use_double=True, nthreads=NTH)
    o, s = obs.cpu().numpy(), state.cpu().numpy()
    nb = sc.ndof
    assert np.abs(s[:nb] - st_ref[:nb]).max() <= 1e-3                      # stated gate (free-running, T = 30)
    assert np.abs(s[:nb] - st_ref[:nb]).max() <= 5e-5                      # what float32 delivers
    assert np.abs(o[0:3] - obs_ref[0:3]).max() <= 1e-4                     # link position, every step [m]
    qa, qb = o[3:7], obs_ref[3:7]
    assert np.minimum(np.abs(qa - qb), np.abs(qa + qb)).max() <= 2e-5
    assert np.abs(o[13:13 + 2 * nb] - obs_ref[13:13 + 2 * nb]).max() <= 2e-3


def _lockstep(oracle, sc, p, s0_rows, free_rows, actions, T, K, steps, tol_x=1e-4, tol_v=2e-3):
    """Oracle state re-injected before every step; returns the worst one-step errors (positions / quaternions, velocities)."""
    be = gpu_backend(sc, p)
    a_d, root_d = dev(actions), dev(sc.root_state0)
    NS = be.state_size()
    nd2 = 2 * sc.ndof
    state_ref = np.zeros((NS, K), np.float32)
    state_ref[:nd2] = s0_rows[:, None]
    for f, actor in enumerate(free_rows):
        state_ref[nd2 + 13 * f: nd2 + 13 * (f + 1)] = sc.root_state0[actor][:, None]
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    worst_x = worst_v = 0.0
    nb = sc.ndof
    for t in steps:
        st = dev(state_ref)
        be.rollout(None, st, a_d, t, 1, obs, root0=root_d)
        state_ref, _ = oracle.rollout(sc.model, p, None, actions, t, 1, state=state_ref.copy(), root0=sc.root_state0, want_obs=False, nthreads=NTH)
        g = st.cpu().numpy()
        assert np.isfinite(g).all()
        pos_rows = list(range(nb)) + [nd2 + 13 * f + r for f in range(len(free_rows)) for r in range(7)]
        vel_rows = list(range(nb, nd2)) + [nd2 + 13 * f + r for f in range(len(free_rows)) for r in range(7, 13)]
        worst_x = max(worst_x, float(np.abs(g[pos_rows] - state_ref[pos_rows]).max()))
        worst_v = max(worst_v, float(np.abs(g[vel_rows] - state_ref[vel_rows]).max()))
    assert worst_x <= tol_x and worst_v <= tol_v, (worst_x, worst_v)
    return worst_x, worst_v


def test_c3_boxer_push_size_lockstep(oracle):
    """BASELINE C3: boxer_push, K = 4 000, T = 20, per-rollout size / mass / friction randomisation on."""
    K, T = 4000, 20
    sc, p, s0 = boxer_setup(K=K, T=T)
    rng = np.random.default_rng(0)
    actions = np.stack([rng.uniform(0.3, 1.2, (T, K)), rng.uniform(-1.0, 1.0, (T, K))], axis=1).astype(np.float32)
    _lockstep(oracle, sc, p, s0, [1], actions, T, K, range(T), tol_x=1e-4, tol_v=5e-3)


def test_c4_heijn_push_shard_size_lockstep(oracle):
    """BASELINE C4 on one of its 4 GPUs: heijn_push, K = 4 000, T = 25, dt 0.1 / 1 substep; the robot really pushes the block."""
    K, T = 4000, 25
    sc, p, s0 = push_setup(K=K, T=T, noise=True, block_pos=(0.62, 1.5, 0.1))
    a = np.random.default_rng(3).uniform(-0.6, 0.6, (T, 3, K)).astype(np.float32)
    a[:, 0] = 0.5 + 0.1 * a[:, 0]
    _lockstep(oracle, sc, p, s0, [1], a, T, K, range(T))


def _pick_scene(K, T):
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaPickObjective
    from oracle.backend import OracleBackend
    pl = MPPIisaacPlanner(pick_cfg(K=K, T=T, device="cpu", sampling_method="random", mppi_mode="simple"), PandaPickObjective(), backend=OracleBackend())
    sc, p = pl.sim.scene, pl.sim.params
    dof0 = sc.dof_state0
    s0 = np.concatenate([dof0[0::2], dof0[1::2]]).astype(np.float32)
    return sc, p, s0


def test_c5_panda_pick_shard_size_lockstep(oracle):
    """BASELINE C5 on one of its 8 GPUs: panda_pick, K = 8 192, T = 30 (two waves of 222 KB CTAs on 132 SMs): the gripper closes on
    the block while the arm moves; every fifth step of the horizon in lock-step."""
    K, T = 8192, 30
    sc, p, s0 = _pick_scene(K, T)
    assert sc.model.nfree >= 1 and sc.model.nshapes > 4
    rng = np.random.default_rng(5)
    a = rng.uniform(-0.2, 0.2, (T, sc.nu, K)).astype(np.float32)
    a[:, 7:9] = -0.15 + 0.05 * a[:, 7:9]                                   # fingers closing
    free_actors = [sc.model.free_actor[f] for f in range(sc.model.nfree)]
    _lockstep(oracle, sc, p, s0, free_actors, a, T, K, range(0, T, 5), tol_x=1e-4, tol_v=5e-3)


def test_c5_full_size_determinism_and_shard_invariance():
    """BASELINE C5 at its full K = 65 536 on one GPU: two launches are bit-identical, and the 8 192-sample shard a rank of the
    8-GPU job owns (k_offset keys the per-rollout randomisation) reproduces its slice of the full launch bit for bit."""
    K, T = 65536, 30
    sc, p, s0 = _pick_scene(K, T)
    be = gpu_backend(sc, p)
    a = (np.random.default_rng(6).uniform(-0.2, 0.2, (T, sc.nu, K))).astype(np.float32)
    a_d, root_d, s0_d = dev(a), dev(sc.root_state0), dev(s0)
    R = be.obs_size()
    o1, o2 = torch.zeros((R, T, K), device=DEV), torch.zeros((R, T, K), device=DEV)
    be.rollout(s0_d, None, a_d, 0, T, o1, root0=root_d)
    be.rollout(s0_d, None, a_d, 0, T, o2, root0=root_d)
    assert torch.isfinite(o1).all() and torch.equal(o1, o2)
    p8 = copy.copy(p); p8.K, p8.k_offset = 8192, 3 * 8192
    be8 = gpu_backend(sc, p8)
    o8 = torch.zeros((R, T, 8192), device=DEV)
    be8.rollout(s0_d, None, dev(a[:, :, 3 * 8192:4 * 8192]), 0, T, o8, root0=root_d)
    assert torch.equal(o8, o1[:, :, 3 * 8192:4 * 8192])


def test_c3_shard_invariance_across_team_layouts():
    """BASELINE C3 at K = 4 000: the whole launch and a 512-sample shard of it (k_offset keys the per-rollout randomisation) are
    bit-identical, also where the two launches take different shared-memory layouts of the team kernel (on 132 SMs the 4 000-sample
    launch takes the compact one, which fits its 1 000 CTAs in one wave, and the shard the roomy one)."""
    K, T, KS, off = 4000, 20, 512, 1024
    sc, p, s0 = boxer_setup(K=K, T=T)
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(12)
    a = np.stack([rng.uniform(0.3, 1.2, (T, K)), rng.uniform(-1.0, 1.0, (T, K))], axis=1).astype(np.float32)
    a_d, root_d, s0_d = dev(a), dev(sc.root_state0), dev(s0)
    R = be.obs_size()
    o = torch.zeros((R, T, K), device=DEV)
    be.rollout(s0_d, None, a_d, 0, T, o, root0=root_d)
    ps = copy.copy(p); ps.K, ps.k_offset = KS, off
    bs = gpu_backend(sc, ps)
    o_s = torch.zeros((R, T, KS), device=DEV)
    bs.rollout(s0_d, None, dev(a[:, :, off:off + KS]), 0, T, o_s, root0=root_d)
    assert torch.isfinite(o).all() and torch.equal(o_s, o[:, :, off:off + KS])


@pytest.mark.parametrize("which,K", [("gripper", 65536), ("point", 65536), ("panda", 131072), ("gripper", 8192)])
def test_k3_ring_parity_at_streaming_sizes(oracle, which, K):
    """K3 against the oracle at sizes where every CTA streams more tiles than the ring holds (the producer waits on `empty`
    barriers, stages are refilled several times): C5's shapes (nu = 9: 300-row tiles, 5 stages / 5 consumers, two TMA boxes per
    tile), a narrow one (nu = 3: 7 stages of 48 rows) and the headline's (nu = 7, 7 stages)."""
    from mppi_isaac_b200.model.blob import MODE_SIMPLE
    from scenes import gripper_setup, point_setup
    setup, T = {"gripper": (gripper_setup, 30), "point": (point_setup, 12), "panda": (panda_setup, 30)}[which]
    sc, p, _ = setup(K=K, T=T)
    nu = sc.nu
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(7)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    x = (rng.standard_normal((T, nu, K)) * 0.3).astype(np.float32)
    cost = rng.uniform(0, 10, (T, K)).astype(np.float32)
    cost[:, K // 3] = np.nan
    partial = torch.zeros(2 + T * nu, device=DEV)
    for _ in range(2):                                                     # twice: the barriers start from a clean phase every launch
        be.reduce(dev(cost), dev(x), dev(U), partial)
    torch.cuda.synchronize()
    p_ref = oracle.reduce_mt(sc.model, p, cost, x, U, NTH)
    pg = partial.cpu().numpy()
    assert abs(pg[0] - p_ref[0]) <= 1e-5 * max(1, abs(p_ref[0]))
    np.testing.assert_allclose(pg[1], p_ref[1], rtol=5e-5)
    np.testing.assert_allclose(pg[2:], p_ref[2:], rtol=0, atol=5e-5 * max(1.0, np.abs(p_ref[2:]).max()))


# ------------------------------------------------------------------------------------------------------------------
# regressions of the round-1 review (ADVICE.md)
# ------------------------------------------------------------------------------------------------------------------
def test_compute_action_with_obstacles_rebuilds_the_gpu_planner():
    """compute_action(obst=...) adds an actor -> the simulator (kernel handle, buffers) is rebuilt; the planner must re-bind to it:
    fresh action in the pinned mirror, graph re-captured, robot state re-applied."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PointReachObjective
    from oracle.backend import OracleBackend
    from scenes import point_cfg
    obst = {"o0": {"position": [0.75, 0.0, 0.1], "velocity": [0.0, 0.0, 0.0], "size": [0.2]}}
    gpu = MPPIisaacPlanner(point_cfg(K=256, T=12, device=DEV), PointReachObjective(), use_cuda_graph=True)
    cpu = MPPIisaacPlanner(point_cfg(K=256, T=12, device="cpu"), PointReachObjective(), backend=OracleBackend())
    q, qd = [0.1, 0.0, 0.0], [0.0, 0.0, 0.0]
    a0 = gpu.compute_action(q, qd)                                       # no obstacle yet: graph captured on the first handle
    cpu.compute_action(q, qd)
    for it in range(3):
        ag, ac = gpu.compute_action(q, qd, obst=obst), cpu.compute_action(q, qd, obst=obst)
        assert torch.isfinite(ag).all() and float(ag.abs().max()) > 0.0
        torch.testing.assert_close(ag, gpu.mppi._action.cpu(), atol=0, rtol=0)     # the host mirror IS the device action of this plan
        assert float((ag - ac).abs().max()) <= 2e-2 * 1.5, (it, ag, ac)
    assert [a.name for a in gpu.sim.env_cfg][-1] == "sphere0" and gpu.mppi._graph is not None
    np.testing.assert_allclose(gpu.sim._state0.cpu().numpy()[:3], q, atol=1e-6)    # the caller's joint state survived the rebuild
    assert a0.shape == ag.shape


def test_captured_graph_follows_a_base_moved_through_a_setter():
    """The robot base pose is a by-value kernel parameter baked into the captured graph: moving the base with a sim setter (not
    through reset_rollout_sim) must invalidate the graph, otherwise the rollouts keep starting from the old base."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from scenes import panda_cfg
    pl = MPPIisaacPlanner(panda_cfg(K=256, T=10, device=DEV), PandaReachObjective(), use_cuda_graph=True)
    q = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
    pl.compute_action(q, [0.0] * 7)
    pl.compute_action(q, [0.0] * 7)
    assert pl.mppi._graph is not None
    ee0 = pl.sim.get_actor_link_by_name("panda", "panda_ee_tip")[:, 0:3].clone()
    base = pl.sim.get_actor_position_by_robot_index(0)[0].clone()
    pl.sim.set_actor_position_by_robot_index(base + torch.tensor([0.25, 0.0, 0.0], device=DEV), 0)
    pl.sim.save_root_state()
    pl.mppi.U.zero_(); pl.mppi.plan_ctr.zero_()
    pl.compute_action(q, [0.0] * 7)
    ee1 = pl.sim.get_actor_link_by_name("panda", "panda_ee_tip")[:, 0:3]
    # null-action row K-1: identical joint trajectory in both plans, so its tip moves by exactly the base shift
    K = pl.sim.num_envs
    d = (ee1.view(-1, K, 3)[0, K - 1] - ee0.view(-1, K, 3)[0, K - 1]).cpu().numpy()
    np.testing.assert_allclose(d, [0.25, 0.0, 0.0], atol=2e-3)


def test_c_abi_runs_on_the_handles_device_from_any_thread():
    """A planner on cuda:N served from a thread whose current device is cuda:0 (the RPC server case): launches must select the
    handle's device and restore the caller's."""
    import threading
    n = torch.cuda.device_count()
    dev_idx = n - 1
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from scenes import panda_cfg
    pl = MPPIisaacPlanner(panda_cfg(K=128, T=10, device=f"cuda:{dev_idx}"), PandaReachObjective(), use_cuda_graph=False)
    q = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
    ref = pl.compute_action(q, [0.0] * 7)
    out = {}

    def worker():
        try:
            torch.cuda.set_device(0)
            pl.mppi.U.zero_(); pl.mppi.plan_ctr.zero_()
            out["a"] = pl.compute_action(q, [0.0] * 7)
            out["dev"] = torch.cuda.current_device()
        except Exception as e:  # noqa: BLE001
            out["err"] = repr(e)
    pl.mppi.U.zero_(); pl.mppi.plan_ctr.zero_()
    ref = pl.compute_action(q, [0.0] * 7)
    th = threading.Thread(target=worker)
    th.start(); th.join(timeout=120)
    assert "err" not in out, out.get("err")
    assert out["dev"] == 0
    torch.testing.assert_close(out["a"], ref, atol=1e-6, rtol=0)


def test_sphere_obstacle_rollout_lockstep(oracle):
    """True sphere primitives (the obstacles of compute_action(obst=...)): the robot's collision box against a fixed sphere, GPU
    kernel against the oracle in lock-step while the point robot is driven into the sphere from several directions."""
    from mppi_isaac_b200.model.blob import SHAPE_SPHERE, build_scene, make_params
    from mppi_isaac_b200.utils.config_store import ActorWrapper, IsaacGymConfig, load_actor_cfgs
    from scenes import point_mppi
    from mppi_isaac_b200.model.blob import OBS_CONTACT, OBS_DOF_STATE, OBS_LINK_STATE
    K, T = 256, 20
    actors = load_actor_cfgs(["point_robot", "goal"]) + [ActorWrapper(type="sphere", name="sphere0", handle=None, size=[0.2], fixed=True, init_pos=[0.8, 0.8, 0.1])]
    sc = build_scene(actors)
    m = sc.model
    assert SHAPE_SPHERE in [m.shape_type[s] for s in range(m.nshapes)]
    obs = [(OBS_LINK_STATE, sc.robot.link_names.index("base_link")), (OBS_DOF_STATE, 0)] + [(OBS_CONTACT, s) for s in range(m.ncontact_slots)]
    p = make_params(point_mppi(K, T), IsaacGymConfig(), sc.nu, K, obs)
    rng = np.random.default_rng(8)
    ang = rng.uniform(0.2, 1.37, K)                                        # headings that hit the sphere head-on, by a corner, or graze it
    a = np.zeros((T, 3, K), np.float32)
    a[:, 0] = 1.4 * np.cos(ang); a[:, 1] = 1.4 * np.sin(ang)
    s0 = np.array([0.1, 0.1, 0.0, 0.0, 0.0, 0.0], np.float32)
    wx, wv = _lockstep(oracle, sc, p, s0, [], a, T, K, range(T), tol_x=1e-4, tol_v=5e-3)
    # the rollouts really reach the sphere: some of them are stopped short of where free motion would take them (0.1 + 1.4 cos * 1 s)
    st, _ = oracle.rollout(sc.model, p, s0, a, root0=sc.root_state0, nthreads=NTH)
    assert (np.hypot(st[0] - 0.1, st[1] - 0.1) < 1.0).mean() > 0.3
