"""-m gpu: parity of the CUDA path against the oracle, through the C ABI (CudaBackend = ctypes on libmppib.so).

Tolerances (float32 path; SURVEY.md 8(c)):
  K1  Philox integers exact -> Gaussians |d| <= 2e-6 * max(1,|z|) (double Box-Muller vs logf/sincospif)
  K2  one model step |dq| <= 1e-5 ; free-running T=30 |dq| <= 1e-3 rad, link position <= 1e-4 m... (measured ~1e-6)
  K3/K4  |U_gpu - U_oracle|_inf <= 1e-5 * max(1, |U|_inf)
Full-size properties at BASELINE sizes (K = 10 000 / 65 536): shard-combine invariance, replica determinism,
uniform-cost and dominant-sample limits."""
import copy
import os

import numpy as np
import pytest
import torch

from mppi_isaac_b200.model.blob import MODE_SIMPLE, OBS_DOF_STATE, OBS_LINK_STATE
from scenes import boxer_cfg, boxer_setup, gripper_setup, panda_cfg, panda_setup, pick_cfg, point_cfg, point_setup, push_cfg, push_setup

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def gpu_backend(sc, p):
    from mppi_isaac_b200.backend import CudaBackend
    be = CudaBackend(DEV)
    be.create(sc.model, p)
    return be


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


def test_native_library_is_loaded():
    from mppi_isaac_b200 import backend
    backend.load_library()
    with open("/proc/self/maps") as f:
        assert "libmppib.so" in f.read()


@pytest.mark.parametrize("setup,K,T", [(panda_setup, 1000, 30), (point_setup, 128, 12)])
def test_k1_sample_parity(oracle, setup, K, T):
    sc, p, _ = setup(K=K, T=T)
    nu = sc.nu
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(0)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    prior = rng.uniform(-0.3, 0.3, (T, nu)).astype(np.float32)
    actions, noise = torch.zeros((T, nu, K), device=DEV), torch.zeros((T, nu, K), device=DEV)
    ctr = torch.tensor([5], dtype=torch.int32, device=DEV)
    be.sample(1234, 2, 0, K, dev(U), dev(prior), actions, noise, ctr)       # effective plan index 7
    a_ref, n_ref = oracle.sample(sc.model, p, 1234, 7, U, prior_row=prior)
    a, n = actions.cpu().numpy(), noise.cpu().numpy()
    scale = float(np.sqrt(max(p.sigma_chol[0] ** 2, 1e-12)))
    assert np.abs(a - a_ref).max() <= 2e-6 * max(1.0, 6 * scale)
    assert np.abs(n - n_ref).max() <= 2e-6 * max(1.0, 6 * scale)
    np.testing.assert_array_equal(a[:, :, -1], 0)
    np.testing.assert_array_equal(a[:, :, -2], prior)
    # shard invariance on the device: two shards with k_offset reproduce the single launch
    p2 = copy.copy(p); p2.K = K // 2
    be2 = gpu_backend(sc, p2)
    parts = []
    for g in range(2):
        aa = torch.zeros((T, nu, K // 2), device=DEV)
        be2.sample(1234, 7, g * (K // 2), K, dev(U), dev(prior), aa, None)
        parts.append(aa.cpu().numpy())
    np.testing.assert_array_equal(np.concatenate(parts, axis=2), a)


@pytest.mark.parametrize("setup,K,T", [(panda_setup, 1000, 30), (point_setup, 128, 12), (gripper_setup, 512, 30)])
def test_k2_rollout_parity_free_running(oracle, setup, K, T):
    sc, p, state0 = setup(K=K, T=T)
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(1)
    lim = float(p.u_max[0])
    actions = rng.uniform(-lim, lim, (T, sc.nu, K)).astype(np.float32)
    R = be.obs_size()
    obs, state = torch.zeros((R, T, K), device=DEV), torch.zeros((be.state_size(), K), device=DEV)
    be.rollout(dev(state0), state, dev(actions), 0, T, obs)
    st_ref, obs_ref = oracle.rollout(sc.model, p, state0, actions, use_double=True, nthreads=8)
    o, s = obs.cpu().numpy(), state.cpu().numpy()
    nb = sc.ndof
    assert np.abs(s[:nb] - st_ref[:nb]).max() <= 1e-3                      # stated gate
    assert np.abs(s[:nb] - st_ref[:nb]).max() <= 2e-5                      # what float32 actually delivers
    assert np.abs(o[0:3] - obs_ref[0:3]).max() <= 1e-4                     # link position [m]
    qa, qb = o[3:7], obs_ref[3:7]
    assert np.minimum(np.abs(qa - qb), np.abs(qa + qb)).max() <= 2e-5      # quaternion up to sign
    assert np.abs(o[7:13] - obs_ref[7:13]).max() <= 2e-3                   # link velocities (x kd amplification)
    dof_rows = slice(13, 13 + 2 * nb)
    assert np.abs(o[dof_rows] - obs_ref[dof_rows]).max() <= 2e-3
    for r0 in range(13 + 2 * nb, o.shape[0], 13):                          # further observed links (gripper fingers)
        assert np.abs(o[r0:r0 + 3] - obs_ref[r0:r0 + 3]).max() <= 1e-4
        assert np.minimum(np.abs(o[r0 + 3:r0 + 7] - obs_ref[r0 + 3:r0 + 7]), np.abs(o[r0 + 3:r0 + 7] + obs_ref[r0 + 3:r0 + 7])).max() <= 2e-5


def test_k2_one_step_lockstep(oracle):
    """Oracle state re-injected before every step: one-step error of the kernel alone."""
    sc, p, state0 = panda_setup(K=256, T=30)
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(2)
    actions = rng.uniform(-0.2, 0.2, (30, 7, 256)).astype(np.float32)
    a_d = dev(actions)
    state_ref = np.repeat(state0[:, None], 256, 1).astype(np.float32)
    R = be.obs_size()
    obs = torch.zeros((R, 30, 256), device=DEV)
    worst = 0.0
    for t in range(30):
        st = dev(state_ref)
        be.rollout(None, st, a_d, t, 1, obs)
        state_ref, _ = oracle.rollout(sc.model, p, None, actions, t, 1, state=state_ref.copy(), want_obs=False)
        worst = max(worst, float(np.abs(st.cpu().numpy()[:7] - state_ref[:7]).max()))
    assert worst <= 1e-5


def test_k2_stepwise_equals_batched_and_observe_only(oracle):
    sc, p, state0 = panda_setup(K=64, T=6)
    be = gpu_backend(sc, p)
    actions = dev(np.random.default_rng(3).uniform(-0.2, 0.2, (6, 7, 64)).astype(np.float32))
    R = be.obs_size()
    obs_a, obs_b = torch.zeros((R, 6, 64), device=DEV), torch.zeros((R, 6, 64), device=DEV)
    st_a, st_b = torch.zeros((14, 64), device=DEV), dev(np.repeat(state0[:, None], 64, 1))
    be.rollout(dev(state0), st_a, actions, 0, 6, obs_a)
    for t in range(6):
        be.rollout(None, st_b, actions[t:t + 1], t, 1, obs_b, act_t0=t)
    assert torch.equal(st_a, st_b)                                         # the dynamics are bit-identical ...
    # ... the observed rows come from two differently scheduled copies of the same kinematics (the batched launch reuses the
    # next step's sweep 1, a single step runs the standalone pass): identical up to float32 contraction order
    torch.testing.assert_close(obs_a, obs_b, atol=2e-6, rtol=0)
    obs_c = torch.zeros_like(obs_a)
    be.rollout(None, st_b, actions, 5, 0, obs_c)                           # observe-only into slot 5
    assert torch.equal(obs_c[:, 5], obs_b[:, 5])


def test_k2_replica_determinism_full_size():
    """K = 10 000 identical inputs -> bit-identical trajectories (reference test invariant, full BASELINE size)."""
    sc, p, state0 = panda_setup(K=10000, T=30)
    be = gpu_backend(sc, p)
    a = np.random.default_rng(4).uniform(-0.2, 0.2, (30, 7, 1)).astype(np.float32)
    actions = dev(np.repeat(a, 10000, axis=2))
    obs = torch.zeros((be.obs_size(), 30, 10000), device=DEV)
    be.rollout(dev(state0), None, actions, 0, 30, obs)
    assert bool((obs == obs[:, :, :1]).all())


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("K", [64, 1000, 4100])
def test_k3_k4_parity(oracle, mode, K):
    sc, p, _ = panda_setup(K=K, T=30, mode=mode, filter_u=True)
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(5)
    U = rng.uniform(-0.1, 0.1, (30, 7)).astype(np.float32)
    a, n = oracle.sample(sc.model, p, 3, 0, U)
    cost = rng.uniform(0, 10, (30, K)).astype(np.float32)
    cost[:, K // 3] = np.nan                                                # a diverged rollout gets weight 0
    x = n if p.mode == MODE_SIMPLE else a
    partial = torch.zeros(2 + 210, device=DEV)
    be.reduce(dev(cost), dev(x), dev(U), partial)
    p_ref, _ = oracle.reduce(sc.model, p, cost, x, U)
    pg = partial.cpu().numpy()
    assert abs(pg[0] - p_ref[0]) <= 1e-5 * max(1, abs(p_ref[0]))
    np.testing.assert_allclose(pg[1], p_ref[1], rtol=2e-5)
    np.testing.assert_allclose(pg[2:], p_ref[2:], rtol=0, atol=2e-5 * max(1.0, np.abs(p_ref[2:]).max()))
    Ud, act, stats = dev(U), torch.zeros(7, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(partial.view(1, -1), 1, Ud, act, stats)
    U_ref, act_ref, st_ref = oracle.finalize(sc.model, p, p_ref[None], U)
    assert np.abs(Ud.cpu().numpy() - U_ref).max() <= 1e-5 * max(1.0, np.abs(U_ref).max())
    np.testing.assert_array_equal(act.cpu().numpy(), Ud.cpu().numpy()[0])
    Us = dev(U); be.shift(Us)
    np.testing.assert_array_equal(Us.cpu().numpy(), oracle.shift(sc.model, p, U))


def test_k3_properties_at_baseline_sizes():
    """Size-independent properties at K = 65 536 (C5 size on one GPU) and K = 10 000 (headline)."""
    for K in (10000, 65536):
        sc, p, _ = panda_setup(K=K, T=30, filter_u=False)
        be = gpu_backend(sc, p)
        g = torch.Generator(device=DEV).manual_seed(0)
        x = torch.randn((30, 7, K), device=DEV, generator=g) * 0.3
        U = torch.zeros((30, 7), device=DEV)
        partial = torch.zeros(212, device=DEV)
        # uniform cost -> W/eta is the plain mean
        be.reduce(torch.ones((30, K), device=DEV), x, U, partial)
        assert abs(float(partial[1]) - K) <= 1e-3 * K
        torch.testing.assert_close(partial[2:] / partial[1], x.mean(dim=2).reshape(-1), atol=2e-5, rtol=0)
        # one dominant sample -> W/eta is that sample
        cost = torch.rand((30, K), device=DEV, generator=g)
        cost[:, 777] = -1e3
        be.reduce(cost, x, U, partial)
        torch.testing.assert_close(partial[2:] / partial[1], x[:, :, 777].reshape(-1), atol=1e-6, rtol=0)
        # shard-combine invariance: G shards through K4 == 1 shard through K4
        cost = torch.rand((30, K), device=DEV, generator=g) * 5
        be.reduce(cost, x, U, partial)
        U1, act = torch.zeros((30, 7), device=DEV), torch.zeros(7, device=DEV)
        be.finalize(partial.view(1, -1), 1, U1, act, None)
        G = 8 if K % 32 == 0 else 4                                        # shards must stay multiples of 4
        p8 = copy.copy(p); p8.K = K // G
        be8 = gpu_backend(sc, p8)
        parts = torch.zeros((G, 212), device=DEV)
        for s in range(G):
            sl = slice(s * p8.K, (s + 1) * p8.K)
            be8.reduce(cost[:, sl].contiguous(), x[:, :, sl].contiguous(), U, parts[s])
        U8 = torch.zeros((30, 7), device=DEV)
        be8.finalize(parts, G, U8, act, None)
        torch.testing.assert_close(U8, U1, atol=2e-6, rtol=0)


@pytest.mark.parametrize("robot", ["panda", "point"])
def test_full_plan_parity_through_planner_api(robot):
    """MPPIisaacPlanner on the GPU (CUDA graph on) vs the same planner on the checker backend, closed loop."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective, PointReachObjective
    from oracle.backend import OracleBackend
    if robot == "panda":
        mk, obj, q = (lambda d: panda_cfg(K=1000, T=30, device=d)), PandaReachObjective, np.array([0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0])
    else:
        mk, obj, q = (lambda d: point_cfg(K=128, T=12, device=d)), PointReachObjective, np.array([0.1, 0.0, 0.0])
    gpu = MPPIisaacPlanner(mk(DEV), obj(), use_cuda_graph=True)
    cpu = MPPIisaacPlanner(mk("cpu"), obj(), backend=OracleBackend(nthreads=8))
    qd = np.zeros_like(q)
    for it in range(5):
        ag, ac = gpu.compute_action(q, qd), cpu.compute_action(q, qd)
        lim = float(gpu.mppi.backend.params.u_max[0])
        assert float((ag - ac).abs().max()) <= 2e-4 * max(1.0, lim), f"plan {it}"
        q = q + 0.05 * ac.numpy(); qd = ac.numpy()
    assert gpu.mppi._graph is not None, "CUDA-graph capture of the plan failed"
    np.testing.assert_allclose(gpu.mppi.U.cpu().numpy(), cpu.mppi.U.numpy(), atol=2e-4)
    rg, rc = torch.load(__import__("io").BytesIO(gpu.get_rollouts())), torch.load(__import__("io").BytesIO(cpu.get_rollouts()))
    assert rg.shape == rc.shape
    assert float((rg.cpu() - rc).abs().max()) <= 1e-3


def _stepwise_matches_batched(mk, obj, q):
    from mppi_isaac_b200 import MPPIisaacPlanner
    a = MPPIisaacPlanner(mk(), obj(), rollout_mode="batched", use_cuda_graph=False)
    b = MPPIisaacPlanner(mk(), obj(), rollout_mode="stepwise")
    for it in range(3):
        ua, ub = a.compute_action(q, [0] * len(q)), b.compute_action(q, [0] * len(q))
        assert float((ua - ub).abs().max()) <= 1e-6
    assert torch.equal(a.mppi.actions, b.mppi.actions)


def test_stepwise_protocol_on_gpu_matches_batched():
    from mppi_isaac_b200.objectives import PandaReachObjective
    _stepwise_matches_batched(lambda: panda_cfg(K=256, T=12, device=DEV), PandaReachObjective, [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0])


@pytest.mark.parametrize("config", ["push", "boxer"])
def test_stepwise_protocol_on_gpu_matches_batched_with_contacts(config):
    """The planner's stepwise path against its batched one on the contact scenes of configs C4 (push, h = 0.1 s) and C3 (the boxer's
    planar base, h = 0.1 s)."""
    from mppi_isaac_b200.objectives import PushObjective
    if config == "push":
        _stepwise_matches_batched(lambda: push_cfg(K=256, T=10, device=DEV), PushObjective, [0.0, 0.0, 0.0])
    else:
        _stepwise_matches_batched(lambda: boxer_cfg(K=256, T=12, device=DEV), lambda: PushObjective(robot="boxer", link="ee_link"), [0.0, 2.5, 0.0])


# ---------------------------------------------------------------------------------------------------------------
# free bodies + contacts (configs C4 / C5).  Contact dynamics are discontinuous (a sample point flips between "inside"
# and "outside"), so the tight gate is LOCK-STEP: the oracle's state is re-injected before every step.  Free-running
# agreement is checked statistically (SURVEY.md 8(c): "drift reported, not gated").
# ---------------------------------------------------------------------------------------------------------------
def _push_actions(T, K, seed=0, vx=0.5):
    a = np.random.default_rng(seed).uniform(-0.6, 0.6, (T, 3, K)).astype(np.float32)
    a[:, 0] = vx + 0.1 * a[:, 0]
    return a


def test_contact_rollout_lockstep_parity(oracle):
    K, T = 128, 12
    sc, p, s0 = push_setup(K=K, T=T, noise=True, block_pos=(0.62, 1.5, 0.1))
    be = gpu_backend(sc, p)
    actions = _push_actions(T, K)
    a_d, root_d = dev(actions), dev(sc.root_state0)
    NS = be.state_size()
    assert NS == 6 + 13
    state_ref = np.zeros((NS, K), np.float32)
    state_ref[6:] = sc.root_state0[1][:, None]
    R = be.obs_size()
    obs = torch.zeros((R, T, K), device=DEV)
    worst_q, worst_x, worst_v, touched = 0.0, 0.0, 0.0, 0
    for t in range(T):
        st = dev(state_ref)
        be.rollout(None, st, a_d, t, 1, obs, root0=root_d)
        state_ref, o_ref = oracle.rollout(sc.model, p, None, actions, t, 1, state=state_ref.copy(), root0=sc.root_state0)
        g = st.cpu().numpy()
        worst_q = max(worst_q, float(np.abs(g[:6] - state_ref[:6]).max()))
        worst_x = max(worst_x, float(np.abs(g[6:13] - state_ref[6:13]).max()))
        worst_v = max(worst_v, float(np.abs(g[13:19] - state_ref[13:19]).max()))
        f_g, f_r = obs[32:35, t].cpu().numpy(), o_ref[32:35, t]
        touched += int((np.abs(f_r[0]) > 1.0).sum())
        assert np.abs(f_g - f_r).max() <= 5e-2 * max(1.0, np.abs(f_r).max())          # net contact force on the block [N]
    assert touched > K                                                                 # the robot really pushes the block in this test
    assert worst_q <= 1e-4 and worst_x <= 1e-4 and worst_v <= 2e-3                     # one-step root state: 1e-4 (m, -), 2e-3 m/s


def test_contact_rollout_free_running_statistics(oracle):
    K, T = 512, 15
    sc, p, s0 = push_setup(K=K, T=T, noise=True, block_pos=(0.62, 1.5, 0.1))
    be = gpu_backend(sc, p)
    actions = _push_actions(T, K, seed=1)
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    be.rollout(dev(s0), None, dev(actions), 0, T, obs, root0=dev(sc.root_state0))
    _, o_ref = oracle.rollout(sc.model, p, s0, actions, root0=sc.root_state0, nthreads=8)
    o = obs.cpu().numpy()
    assert np.isfinite(o).all()
    dx = np.abs(o[19:22, -1] - o_ref[19:22, -1]).max(axis=0)                           # final block position per rollout
    assert np.median(dx) <= 1e-4 and np.mean(dx < 5e-3) >= 0.95, (np.median(dx), np.mean(dx < 5e-3))
    assert abs(o[19, -1].mean() - o_ref[19, -1].mean()) <= 2e-3                        # ensemble mean of the pushed distance
    np.testing.assert_allclose(o[13:19], o_ref[13:19], atol=5e-3)                      # robot DOF state (velocity drive dominates)


def test_contact_randomisation_and_shard_offset_on_device(oracle):
    sc, p, s0 = push_setup(K=64, T=2, noise=True, block_pos=(3.0, 3.0, 0.1), obstacles=False, dt=0.05)
    root0 = sc.root_state0.copy(); root0[1, 7] = 1.0
    a = np.zeros((2, 3, 64), np.float32)
    be = gpu_backend(sc, p)
    obs = torch.zeros((be.obs_size(), 2, 64), device=DEV)
    be.rollout(dev(s0), None, dev(a), 0, 2, obs, root0=dev(root0))
    _, o_ref = oracle.rollout(sc.model, p, s0, a, root0=root0)
    np.testing.assert_allclose(obs.cpu().numpy(), o_ref, atol=2e-4)                   # same per-rollout size / mass / friction draws
    p2 = copy.copy(p); p2.K, p2.k_offset = 32, 32
    be2 = gpu_backend(sc, p2)
    obs2 = torch.zeros((be2.obs_size(), 2, 32), device=DEV)
    be2.rollout(dev(s0), None, dev(a[:, :, :32]), 0, 2, obs2, root0=dev(root0))
    assert torch.equal(obs2, obs[:, :, 32:])                                           # global sample index keys the draws


@pytest.mark.parametrize("task", ["push", "pick", "omnipick"])
def test_contact_plan_through_planner_api(task):
    """First plan from the same world state, GPU (CUDA graph) vs checker backend, configs C4 / C5 at test size, and the omnipanda
    pick scene (12 bodies + 14 boxes: contact capacity 17, sized to the SM's shared memory)."""
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaPickObjective, PushObjective
    from oracle.backend import OracleBackend
    if task == "push":
        mk, obj, q = (lambda d: push_cfg(K=512, T=10, device=d)), PushObjective, [0.0, 0.0, 0.0]
    elif task == "pick":
        mk, obj, q = (lambda d: pick_cfg(K=256, T=12, device=d)), PandaPickObjective, [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0, 0.02, 0.02]
    else:
        from mppi_isaac_b200 import load_isaacgym_config
        def mk(d):
            cfg = copy.deepcopy(load_isaacgym_config("config_omnipanda_pick_b200"))
            cfg.mppi.num_samples, cfg.mppi.device, cfg.mppi.sampling_method, cfg.mppi.mppi_mode = 256, d, "random", "simple"
            return cfg
        obj, q = (lambda: PandaPickObjective(actor="omnipanda", link="panda_hand")), [0.0, 0.0, 0.0, 0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0, 0.02, 0.02]
    gpu = MPPIisaacPlanner(mk(DEV), obj(), use_cuda_graph=True)
    cpu = MPPIisaacPlanner(mk("cpu"), obj(), backend=OracleBackend(nthreads=8))
    ag, ac = gpu.compute_action(q, [0.0] * len(q)), cpu.compute_action(q, [0.0] * len(q))
    assert torch.isfinite(ag).all()
    lim = float(gpu.mppi.backend.params.u_max[0])
    assert float((ag - ac).abs().max()) <= 2e-2 * lim
    for _ in range(3):
        ag = gpu.compute_action(q, [0.0] * len(q))
    assert gpu.mppi._graph is not None and torch.isfinite(ag).all()
    if task == "omnipick":
        assert gpu.sim.scene.model.max_contacts == 17
    blk = "block" if task == "push" else "panda_pick_block"
    zg, zc = gpu.sim.get_actor_position_by_name(blk)[:, 2], cpu.sim.get_actor_position_by_name(blk)[:, 2]
    assert abs(float(zg.mean()) - float(zc.mean())) <= 5e-3


def test_boxer_planar_base_rollout_parity(oracle):
    """Config C3 geometry: differential-drive planar base + block + obstacles, lock-step against the oracle."""
    K, T = 64, 10
    sc, p, s0 = boxer_setup(K=K, T=T)
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(0)
    actions = np.stack([rng.uniform(0.3, 1.2, (T, K)), rng.uniform(-1.0, 1.0, (T, K))], axis=1).astype(np.float32)
    a_d, root_d = dev(actions), dev(sc.root_state0)
    NS = be.state_size()
    state_ref = np.zeros((NS, K), np.float32)
    state_ref[:10] = s0[:, None]
    state_ref[10:] = sc.root_state0[1][:, None]
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    worst, moved = 0.0, 0.0
    for t in range(T):
        st = dev(state_ref)
        be.rollout(None, st, a_d, t, 1, obs, root0=root_d)
        state_ref, _ = oracle.rollout(sc.model, p, None, actions, t, 1, state=state_ref.copy(), root0=sc.root_state0)
        g = st.cpu().numpy()
        worst = max(worst, float(np.abs(g[[0, 1, 2, 10, 11, 12]] - state_ref[[0, 1, 2, 10, 11, 12]]).max()))
        assert np.abs(g[5:10] - state_ref[5:10]).max() <= 5e-3                # joint velocities incl. the wheels
        moved = max(moved, float(np.abs(state_ref[11] - 1.75).max()))
    assert worst <= 1e-4 and moved > 0.05                                     # base / block positions to 1e-4; the block really gets pushed


def test_boxer_plan_through_planner_api():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PushObjective
    from oracle.backend import OracleBackend
    gpu = MPPIisaacPlanner(boxer_cfg(K=512, T=12, device=DEV), PushObjective(robot="boxer", link="ee_link"))
    cpu = MPPIisaacPlanner(boxer_cfg(K=512, T=12, device="cpu"), PushObjective(robot="boxer", link="ee_link"), backend=OracleBackend(nthreads=8))
    q = [0.0, 2.5, 0.0]
    ag, ac = gpu.compute_action(q, [0.0] * 3), cpu.compute_action(q, [0.0] * 3)
    assert torch.isfinite(ag).all() and float((ag - ac).abs().max()) <= 2e-2 * 3.5
    for _ in range(2):
        gpu.compute_action(q, [0.0] * 3)
    assert gpu.mppi._graph is not None


def test_halton_library_parity(oracle):
    from mppi_isaac_b200.planner.mppi import halton_spline_operator, halton_table
    K, T, nk = 1000, 30, 7
    sc, p, _ = panda_setup(K=K, T=T, mode="halton-spline")
    be = gpu_backend(sc, p)
    B, tab = halton_spline_operator(T, nk), halton_table(nk * 7, 11)
    Z = torch.zeros((T, 7, K), device=DEV)
    be.noise_library(0, K, dev(tab, torch.int32), dev(B), nk, Z)
    Z_ref = oracle.noise_library(sc.model, p, tab, B, nk)
    # float32 radical inverse + erfinvf vs double + AS241: the quantile's slope sqrt(2 pi) exp(z^2/2) amplifies 1 ulp of u in the tails
    assert np.abs(Z.cpu().numpy() - Z_ref).max() <= 1e-4
    assert np.median(np.abs(Z.cpu().numpy() - Z_ref)) <= 1e-6
    U = np.random.default_rng(0).uniform(-0.1, 0.1, (T, 7)).astype(np.float32)
    a, n = torch.zeros_like(Z), torch.zeros_like(Z)
    be.sample_library(0, K, dev(U), None, Z, a, n)
    a_ref, n_ref = oracle.sample_library(sc.model, p, U, Z.cpu().numpy())
    np.testing.assert_array_equal(a.cpu().numpy(), a_ref)
    np.testing.assert_array_equal(n.cpu().numpy(), n_ref)


def test_halton_spline_plan_through_planner_api():
    from mppi_isaac_b200 import MPPIisaacPlanner
    from mppi_isaac_b200.objectives import PandaReachObjective
    from oracle.backend import OracleBackend
    kw = dict(mppi_mode="halton-spline", sampling_method="halton")
    gpu = MPPIisaacPlanner(panda_cfg(K=1000, T=30, device=DEV, **kw), PandaReachObjective())
    cpu = MPPIisaacPlanner(panda_cfg(K=1000, T=30, device="cpu", **kw), PandaReachObjective(), backend=OracleBackend(nthreads=8))
    q = np.array([0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0])
    for it in range(4):
        ag, ac = gpu.compute_action(q, np.zeros(7)), cpu.compute_action(q, np.zeros(7))
        assert float((ag - ac).abs().max()) <= 2e-4, f"plan {it}"
        q = q + 0.05 * ac.numpy()
    assert gpu.mppi._graph is not None


def point_nu1_setup(K, T):
    """The point robot driven through one input: both command maps point at input 0 (nu = 1)."""
    sc, p, state0 = point_setup(K=K, T=T)
    sc.model.nu = 1
    for i in range(sc.model.nb):
        sc.model.cmd_i0[i] = sc.model.cmd_i1[i] = 0
    return sc, p, state0


@pytest.mark.parametrize("setup,T", [(point_setup, 12), (point_setup, 25), (point_setup, 9), (gripper_setup, 30), (gripper_setup, 11), (gripper_setup, 29),
                                     (point_nu1_setup, 1)])
def test_k3_shapes_and_alignment(oracle, setup, T):
    """K3 across (T, nu) shapes: T*nu = 27..270 rows, odd row counts, two TMA boxes for T*nu > 256 (270 = 2 x 135) and three for 261 = 3 x 87;
    T = nu = 1, where the last CTA's fold needs more shared memory than the ring stages hold."""
    K = 1000
    sc, p, _ = setup(K=K, T=T) if setup is not gripper_setup else setup(K=K, T=T, filter_u=False)
    p.filter_u = 0
    nu = sc.model.nu
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(T)
    U = rng.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
    x = rng.normal(0, 0.3, (T, nu, K)).astype(np.float32)
    cost = rng.uniform(0, 5, (T, K)).astype(np.float32)
    partial = torch.zeros(2 + T * nu, device=DEV)
    be.reduce(dev(cost), dev(x), dev(U), partial)
    torch.cuda.synchronize()
    p_ref, _ = oracle.reduce(sc.model, p, cost, x, U)
    pg = partial.cpu().numpy()
    np.testing.assert_allclose(pg[:2], p_ref[:2], rtol=2e-5)
    np.testing.assert_allclose(pg[2:], p_ref[2:], rtol=0, atol=2e-5 * max(1.0, np.abs(p_ref[2:]).max()))


@pytest.mark.gpu
def test_peer_memory_exchange_matches_nccl_two_gpus():
    """2 ranks (one per GPU): the exchange fused into K3/K4 over peer memory (mppib_peer_*) gives the same plan as the
    NCCL all-gather path, eagerly and under CUDA-graph replay, and all ranks agree on the action."""
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    acts = {}
    for mode in ("graph", "eager"):
        for exch in ("peer", "nccl"):
            env = dict(os.environ, MPPIB_EXCHANGE=exch, MPPIB_PEER_TIMEOUT_S="10")
            out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                                  "--master-port", "29533", os.path.join(root, "tools", "dist_smoke.py"), mode],
                                 capture_output=True, text=True, timeout=240, env=env, cwd=root)
            assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
            line = [ln for ln in out.stdout.splitlines() if ln.startswith("ACTION ")][-1].split()
            assert line[1] == exch, f"asked for the {exch} exchange, ran {line[1]}"
            acts[(mode, exch)] = np.array([float(v) for v in line[2:]])
        np.testing.assert_array_equal(acts[(mode, "peer")], acts[(mode, "nccl")])
    np.testing.assert_array_equal(acts[("graph", "peer")], acts[("eager", "peer")])


@pytest.mark.gpu
def test_fused_pose_cost_matches_torch_ops():
    """ops.pose_cost (one CUDA kernel) == the torch-op formulation of the reference's panda cost (examples/panda/planner.py:22-40)
    on the obs layout (stride 1 along N), a stride-0 broadcast goal, a dense (N,13) tensor, and with accumulation; and the
    fused Objective gives the same plan cost as the op-by-op one (literal=True: full matrix -> euler route)."""
    from mppi_isaac_b200 import ops
    from mppi_isaac_b200.objectives import PandaReachObjective
    g = torch.Generator(device="cuda").manual_seed(11)
    T, K = 5, 4000
    rows = torch.randn((13, T, K), device="cuda", generator=g)
    rows[3:7] /= rows[3:7].norm(dim=0, keepdim=True)
    a = rows.view(13, T * K).t()                                   # (N,13) strides (1, N): the RolloutSim view
    goal = torch.tensor([0.4, -0.1, 0.6], device="cuda").unsqueeze(0).expand(T * K, 3)
    ref = ops.pose_cost_torch(a, goal, 1.0, 0.5)
    out = ops.pose_cost(a, goal, 1.0, 0.5)
    torch.testing.assert_close(out, ref, rtol=2e-6, atol=2e-6)
    dense = a.contiguous()
    per_row = torch.randn((T * K, 3), device="cuda", generator=g)
    torch.testing.assert_close(ops.pose_cost(dense, per_row, 2.0, 0.0), ops.pose_cost_torch(dense, per_row, 2.0, 0.0), rtol=2e-6, atol=2e-6)
    acc = ref.clone()
    ops.pose_cost(a, None, 0.0, 2.0, out=acc, accumulate=True)
    torch.testing.assert_close(acc, ref + ops.pose_cost_torch(a, None, 0.0, 2.0), rtol=2e-6, atol=2e-6)

    class Sim:                                                      # the two getters the Objective uses
        def get_actor_link_by_name(self, *_):
            return a
        def get_actor_position_by_name(self, *_):
            return goal
    fused, literal = PandaReachObjective(fused=True).compute_cost(Sim()), PandaReachObjective(literal=True).compute_cost(Sim())
    torch.testing.assert_close(fused, literal, rtol=1e-4, atol=2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("setup,K", [(panda_setup, 512), (gripper_setup, 256)])
def test_k2_drive_saturation_resolve_path(oracle, setup, K):
    """Velocity targets that jump by several rad/s saturate the drives (URDF <limit effort>): the fused sweep-3/sweep-1 loop
    of the contact-free kernel must hand those rollouts to its re-solve path and still match the oracle; with the effort
    limits lifted the trajectories differ, i.e. the path was really taken."""
    T = 12
    sc, p, state0 = setup(K=K, T=T)
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(5)
    actions = rng.uniform(-2.5, 2.5, (T, sc.nu, K)).astype(np.float32)
    actions[:, :, : K // 4] *= 0.02                                          # a quarter of the rollouts never saturates (divergent warps)
    R = be.obs_size()
    obs, state = torch.zeros((R, T, K), device=DEV), torch.zeros((be.state_size(), K), device=DEV)
    be.rollout(dev(state0), state, dev(actions), 0, T, obs)
    st_ref, obs_ref = oracle.rollout(sc.model, p, state0, actions, use_double=True, nthreads=8)
    s, o = state.cpu().numpy(), obs.cpu().numpy()
    nb = sc.ndof
    # a saturation decision taken at the threshold can flip between float32 (kernel) and float64 (oracle) and changes that
    # joint's torque for one substep, so the gate is on quantiles over the rollouts, not on the worst one
    err_q = np.abs(s[:nb] - st_ref[:nb]).max(axis=0)
    assert np.median(err_q) <= 2e-5 and np.quantile(err_q, 0.97) <= 1e-3 and err_q.max() <= 5e-2
    err_p = np.abs(o[0:3] - obs_ref[0:3]).max(axis=(0, 1))
    assert np.median(err_p) <= 2e-5 and np.quantile(err_p, 0.97) <= 1e-3
    free = copy.deepcopy(sc.model)
    for i in range(nb):
        free.effort[i] = 1e9
    be_free = gpu_backend(sc, p)
    be_free.set_model(free)
    state2 = torch.zeros_like(state)
    be_free.rollout(dev(state0), state2, dev(actions), 0, T, None)
    diff = np.abs(state2.cpu().numpy()[:nb] - s[:nb]).max(axis=0)
    assert diff[K // 4:].max() > 1e-2 and diff[: K // 4].max() < 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("actor,link,u_lim", [("albert", "mmrobot_link7", 0.4), ("omnipanda", "panda_hand", 0.3), ("panda_effort", "panda_link7", 8.0),
                                               ("panda", "panda_link7", 0.2), ("jackal", "ee_link", 1.0)])
def test_k2_rollout_parity_further_robots(oracle, actor, link, u_lim):
    """SURVEY 8(f) N4: the remaining robots of the reference's example set run through the same kernel and match the oracle --
    albert (differential-drive base reduced to the plane + 7-DoF arm, 12 bodies, tree), omnipanda (x / y / yaw base joints + arm +
    gripper, 12 DOF), the panda in EFFORT mode (commands are torques, isaacgym_wrapper.py:492-496), the plain panda, jackal (four-wheel
    differential drive, planar base)."""
    from scenes import robot_setup
    K, T = 256, 12
    sc, p, state0 = robot_setup(actor, link, K=K, T=T, u_lim=u_lim)
    be = gpu_backend(sc, p)
    rng = np.random.default_rng(8)
    actions = rng.uniform(-u_lim, u_lim, (T, sc.nu, K)).astype(np.float32)
    obs, state = torch.zeros((be.obs_size(), T, K), device=DEV), torch.zeros((be.state_size(), K), device=DEV)
    root0 = dev(sc.root_state0.astype(np.float32))
    be.rollout(dev(state0), state, dev(actions), 0, T, obs, root0=root0)
    st_ref, obs_ref = oracle.rollout(sc.model, p, state0, actions, use_double=True, nthreads=8, root0=sc.root_state0.astype(np.float32))
    s, o = state.cpu().numpy(), obs.cpu().numpy()
    nd = sc.ndof
    assert np.abs(s[:nd] - st_ref[:nd]).max() <= 1e-4
    assert np.abs(s[nd:2 * nd] - st_ref[nd:2 * nd]).max() <= 5e-3
    assert np.abs(o[0:3] - obs_ref[0:3]).max() <= 1e-4
    assert np.abs(s[:nd] - state0[:nd, None]).max() > 1e-2            # something actually moved


@pytest.mark.gpu
@pytest.mark.parametrize("mode,filt", [("simple", True), ("halton-spline", False), ("simple", False)])
def test_fused_reduce_finalize_equals_two_launches(mode, filt):
    """mppib_reduce_finalize (K4 done by the last CTA of K3) == mppib_reduce + mppib_finalize, bit for bit."""
    K, T = 4100, 30
    sc, p, _ = panda_setup(K=K, T=T, mode=mode, filter_u=filt)
    be = gpu_backend(sc, p)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn((T, sc.nu, K), device=DEV, generator=g) * 0.2
    cost = torch.rand((T, K), device=DEV, generator=g) * 5
    cost[3, 17] = float("nan")                                           # a rejected sample goes through both paths
    U0 = torch.randn((T, sc.nu), device=DEV, generator=g) * 0.05
    Ua, Ub = U0.clone(), U0.clone()
    pa, pb = torch.zeros(2 + T * sc.nu, device=DEV), torch.zeros(2 + T * sc.nu, device=DEV)
    aa, ab = torch.zeros(sc.nu, device=DEV), torch.zeros(sc.nu, device=DEV)
    sa, sb = torch.zeros(2, device=DEV), torch.zeros(2, device=DEV)
    be.reduce(cost, x, Ua, pa)
    be.finalize(pa.view(1, -1), 1, Ua, aa, sa)
    be.reduce_finalize(cost, x, Ub, pb, ab, sb)
    torch.cuda.synchronize()
    assert torch.equal(pa, pb) and torch.equal(Ua, Ub) and torch.equal(aa, ab) and torch.equal(sa, sb)
    assert not torch.equal(Ua, U0)


@pytest.mark.gpu
def test_examples_panda_closed_loop_on_gpu():
    """examples/panda planner (K = 10 000, CUDA graph) + world (one-env RolloutSim on the GPU) over the RPC layer: the tip approaches
    the goal and the loop runs far faster than real time (dt = 0.05 s)."""
    import sys
    import threading
    import time
    ex = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "panda")
    sys.path.insert(0, ex)
    try:
        import planner as ex_planner
        import world as ex_world
    finally:
        sys.path.remove(ex)
    from mppi_isaac_b200.utils.rpc import RpcClient, RpcServer
    pl = ex_planner.build_planner(device=DEV)
    cfg, sim = ex_world.build_world(device=DEV)
    server = RpcServer(pl).bind("tcp://127.0.0.1:*")
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    try:
        client = RpcClient(server.last_endpoint, timeout_s=60)
        d0 = ex_world.goal_distance(sim)
        for _ in range(5):
            ex_world.control_step(sim, client)
        t0 = time.perf_counter()
        for _ in range(60):
            ex_world.control_step(sim, client)
        hz = 60 / (time.perf_counter() - t0)
        d1 = ex_world.goal_distance(sim)
        print(f"closed loop: |ee - goal| {d0:.3f} -> {d1:.3f} m in 65 steps, {hz:.0f} control steps/s incl. RPC and the world's own step")
        assert d1 < d0 - 0.1 and hz > 1.0 / cfg.isaacgym.dt
        client.close()
    finally:
        server.stop()
        th.join(timeout=5)
