"""Host logic of the drop-in boundary (planner sequencing, facade views, transport, sharding), driven on CPU
through the checker backend.  No CUDA here; the same code paths run on the GPU with CudaBackend."""
import numpy as np
import pytest
import torch

from mppi_isaac_b200 import MPPIisaacPlanner
from mppi_isaac_b200.objectives import PandaPickObjective, PandaReachObjective, PointReachObjective, PushObjective
from mppi_isaac_b200.planner.mppi import shard_samples
from mppi_isaac_b200.planner.rollout_sim import ObservationError, RolloutSim
from mppi_isaac_b200.utils.config_store import IsaacGymConfig
from mppi_isaac_b200.utils.conversions import matrix_to_euler_angles, quaternion_to_matrix, quaternion_to_yaw
from mppi_isaac_b200.utils.transport import bytes_to_torch, torch_to_bytes
from oracle.backend import OracleBackend
from scenes import boxer_cfg, panda_cfg, pick_cfg, point_cfg, push_cfg

Q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]


def make(cfg, obj, **kw):
    return MPPIisaacPlanner(cfg, obj, backend=OracleBackend(), **kw)


def test_public_surface_matches_reference_names():
    p = make(panda_cfg(K=16, T=10), PandaReachObjective())
    for name in ("update_objective", "dynamics", "running_cost", "compute_action", "reset_rollout_sim", "compute_action_tensor",
                 "command", "add_to_env", "get_rollouts", "update_weights", "update_mppi_params"):
        assert callable(getattr(p, name))
    for attr in ("cfg", "objective", "sim", "mppi", "prior", "state_place_holder"):
        assert hasattr(p, attr)
    assert p.state_place_holder.shape == (16, 14)
    s = p.sim
    for name in ("get_actor_position_by_name", "get_actor_velocity_by_name", "get_actor_orientation_by_name", "get_actor_link_by_name",
                 "get_rigid_body_by_rigid_body_index", "get_actor_contact_forces_by_name", "get_dof_state", "apply_robot_cmd", "step",
                 "reset_robot_state", "save_root_state", "reset_root_state", "reset_to_initial_poses",
                 "update_root_state_tensor_by_obstacles", "set_actor_position_by_name"):
        assert callable(getattr(s, name))
    assert s.num_envs == 16 and s._visualize_link_present and isinstance(s.env_cfg, list)


def test_point_robot_plan_c1_converges():
    """BASELINE config C1 (point_robot reach, K=128, T=12): closed loop drives the base towards the goal."""
    cfg = point_cfg()
    p = make(cfg, PointReachObjective())
    q, qd = np.array([0.1, 0.0, 0.0]), np.zeros(3)
    d0 = np.hypot(1 - q[0], 1 - q[1])
    for it in range(25):
        a = p.compute_action(q, qd).numpy()
        assert a.shape == (3,) and np.all(np.abs(a) <= 1.5 + 1e-6)
        q = q + cfg.isaacgym.dt * a          # kinematic world: the velocity drive tracks the command
        qd = a
    assert np.hypot(1 - q[0], 1 - q[1]) < 0.35 * d0


def test_batched_equals_stepwise_protocol():
    """One T-step launch + one batched cost call == the reference's T x (dynamics, running_cost) protocol."""
    a = make(panda_cfg(K=32, T=12), PandaReachObjective(), rollout_mode="batched")
    b = make(panda_cfg(K=32, T=12), PandaReachObjective(), rollout_mode="stepwise")
    for it in range(3):
        ua = a.compute_action(Q0, [0] * 7)
        ub = b.compute_action(Q0, [0] * 7)
        np.testing.assert_allclose(ua.numpy(), ub.numpy(), atol=1e-6)
    np.testing.assert_allclose(a.mppi.U.numpy(), b.mppi.U.numpy(), atol=1e-6)
    np.testing.assert_array_equal(a.mppi.actions.numpy(), b.mppi.actions.numpy())
    ra, rb = bytes_to_torch(a.get_rollouts()), bytes_to_torch(b.get_rollouts())
    assert ra.shape == (12, 32, 3)
    np.testing.assert_allclose(ra.numpy(), rb.numpy(), atol=1e-6)


def test_getter_views_shapes_and_values():
    p = make(panda_cfg(K=8, T=5, filter_u=False), PandaReachObjective())
    p.compute_action(Q0, [0] * 7)
    s = p.sim                                             # batched mode after a plan
    ee = s.get_actor_link_by_name("panda", "panda_ee_tip")
    assert ee.shape == (40, 13) and s.get_actor_position_by_name("goal").shape == (40, 3)
    assert s.get_actor_position_by_name("goal").stride(0) == 0       # static actor: one row, expanded
    np.testing.assert_allclose(s.get_actor_position_by_name("goal")[7].numpy(), [1.0, 1.0, 0.5])
    assert s._root_state.shape == (40, 2, 13)
    assert s.get_actor_contact_forces_by_name("goal", "sphere").shape == (40, 3)
    # row t*K + k of the batched view is sample k at step t
    np.testing.assert_array_equal(ee[2 * 8 + 3].numpy(), s._obs[0:13, 2, 3].numpy())
    with pytest.raises(ObservationError):
        s.get_actor_link_by_name("panda", "panda_link3")              # not in the traced plan
    # step mode: (K, .) views
    s.begin_step_mode()
    assert s.get_actor_link_by_name("panda", "panda_ee_tip").shape == (8, 13)
    u = torch.zeros(8, 7)
    p.dynamics(None, u)
    assert s.get_actor_link_by_name("panda", "panda_ee_tip").shape == (8, 13)
    assert p.running_cost(None).shape == (8,)


def test_observe_all_exposes_dense_tensors():
    p = make(panda_cfg(K=8, T=4, filter_u=False), PandaReachObjective(), observe="all")
    p.compute_action(Q0, [0] * 7)
    s = p.sim
    assert s._rigid_body_state.shape == (32, 11, 13) and s._dof_state.shape == (32, 14) and s._net_contact_force.shape == (32, 11, 3)
    dof = s.get_dof_state()
    np.testing.assert_allclose(dof[:, 0::2][0].numpy(), np.array(Q0) + 0.05 * p.mppi.actions[0, :, 0].numpy(), atol=2e-3)
    np.testing.assert_array_equal(s.get_actor_link_by_name("panda", "panda_link3").numpy(), s._rigid_body_state[:, 3].numpy())


def test_compute_action_tensor_roundtrip_and_warm_start():
    p = make(panda_cfg(K=32, T=12), PandaReachObjective())
    dof = torch.tensor([[v for q in Q0 for v in (q, 0.0)]], dtype=torch.float32)
    root = p.sim._root_state[:1].clone()
    root[0, 1, :3] = torch.tensor([0.5, 0.2, 0.4])                     # move the goal
    out = p.compute_action_tensor(torch_to_bytes(dof), torch_to_bytes(root))
    act = bytes_to_torch(out)
    assert act.shape == (7,) and act.dtype == torch.float32
    np.testing.assert_allclose(p.sim.get_actor_position_by_name("goal")[0].numpy(), [0.5, 0.2, 0.4])
    U1 = p.mppi.U.clone()
    bytes_to_torch(p.command())
    # warm start: the new plan started from U shifted by one step (last row u_init = 0)
    assert not torch.equal(U1, p.mppi.U)
    assert int(p.mppi.plan_ctr[0]) == 2


def test_update_weights_and_mppi_params():
    p = make(panda_cfg(K=32, T=12), PandaReachObjective())
    p.compute_action(Q0, [0] * 7)
    p.update_weights({"robot_to_goal": 2.0, "robot_ori": 0.0})
    assert p.objective.weights["robot_to_goal"] == 2.0
    p.update_mppi_params({"noise_sigma": (0.05 * np.eye(7)).tolist()})
    assert abs(p.mppi.backend.params.sigma_chol[0] - np.sqrt(0.05)) < 1e-6
    assert float(p.mppi.U.abs().max()) == 0.0                          # reference rebuilds MPPIPlanner -> U reset


def test_prior_goes_to_row_k_minus_2_stepwise():
    class Prior:
        def compute_command(self, sim):
            assert sim.get_actor_link_by_name("panda", "panda_ee_tip").shape[0] == sim.num_envs
            return torch.full((7,), 0.123)
    cfg = panda_cfg(K=16, T=9, use_priors=True)
    p = make(cfg, PandaReachObjective(), prior=Prior())
    assert p.mppi.rollout_mode == "stepwise"
    p.compute_action(Q0, [0] * 7)
    np.testing.assert_allclose(p.mppi.actions[:, :, 14].numpy(), 0.123)
    assert np.all(p.mppi.actions[:, :, 15].numpy() == 0)               # null action row


def test_shard_samples_and_errors():
    assert shard_samples(10000, 0, 1) == (10000, 0)
    parts = [shard_samples(10000, r, 8) for r in range(8)]
    assert sum(k for k, _ in parts) == 10000 and all(k % 4 == 0 for k, _ in parts)
    assert [o for _, o in parts] == list(np.cumsum([0] + [k for k, _ in parts[:-1]]))
    with pytest.raises(ValueError):
        shard_samples(10, 0, 2)
    with pytest.raises(ValueError, match="horizon"):
        make(panda_cfg(K=16, T=6, filter_u=True), PandaReachObjective())
    with pytest.raises(NotImplementedError):
        RolloutSim(IsaacGymConfig(), ["panda_stick", "goal"], viewer=True, device="cpu", backend=OracleBackend())


def test_transport_and_conversions():
    t = torch.arange(12, dtype=torch.float32).reshape(3, 4)
    assert torch.equal(bytes_to_torch(torch_to_bytes(t)), t)
    psi = torch.tensor([0.3, -1.2, 2.9])
    quat = torch.stack([torch.zeros(3), torch.zeros(3), torch.sin(psi / 2), torch.cos(psi / 2)], 1)
    np.testing.assert_allclose(quaternion_to_yaw(quat).numpy(), psi.numpy(), atol=1e-6)       # conversions.py:4-11
    # real-first quaternion API: identity and a 90 deg yaw
    R = quaternion_to_matrix(torch.tensor([[1.0, 0, 0, 0], [np.cos(np.pi / 4), 0, 0, np.sin(np.pi / 4)]]))
    np.testing.assert_allclose(R[0].numpy(), np.eye(3), atol=1e-7)
    np.testing.assert_allclose(R[1].numpy(), [[0, -1, 0], [1, 0, 0], [0, 0, 1]], atol=1e-6)
    e = matrix_to_euler_angles(R, "ZYX")
    np.testing.assert_allclose(e[1].numpy(), [np.pi / 2, 0, 0], atol=1e-6)
    # scipy cross-check of the ZYX convention on random rotations
    from scipy.spatial.transform import Rotation
    rot = Rotation.random(20, random_state=0)
    ours = matrix_to_euler_angles(torch.tensor(rot.as_matrix(), dtype=torch.float64), "ZYX").numpy()
    np.testing.assert_allclose(ours, rot.as_euler("ZYX"), atol=1e-9)
    wxyz = np.roll(rot.as_quat(), 1, axis=1)
    np.testing.assert_allclose(quaternion_to_matrix(torch.tensor(wxyz)).numpy(), rot.as_matrix(), atol=1e-12)


def test_heijn_push_c4_through_the_planner():
    """BASELINE config C4 geometry: free block + static obstacles + contact-force cost through the drop-in surface."""
    p = make(push_cfg(K=64, T=10), PushObjective())
    s = p.sim
    assert s.scene.model.nfree == 1 and s.scene.num_bodies == 12                       # SURVEY section 8 table, C4: 8 / 12 bodies
    a = p.compute_action([0.0, 0.0, 0.0], [0.0, 0.0, 0.0])
    assert a.shape == (3,) and torch.isfinite(a).all()
    blk = s.get_actor_position_by_name("block")
    assert blk.shape == (640, 3) and blk.stride(0) != 0                                # per-rollout rows, not the static expand
    assert s.get_actor_velocity_by_name("block").shape == (640, 3) and s.get_actor_orientation_by_name("block").shape == (640, 4)
    assert s.get_actor_link_by_name("block", "box").shape == (640, 13)
    f = s.get_actor_contact_forces_by_name(actor_name="paper_obst1", link_name="box")
    assert f.shape == (640, 3)
    np.testing.assert_allclose(blk[:, 2].numpy(), 0.1, atol=0.02)                      # the block rests on the ground in every rollout
    assert s._root_state.shape == (640, 5, 13)
    with pytest.raises(ObservationError):
        s._net_contact_force                                                               # dense tensors need observe='all'
    dense = make(push_cfg(K=8, T=4), PushObjective(), observe="all")
    dense.compute_action([0.0] * 3, [0.0] * 3)
    assert dense.sim._net_contact_force.shape == (32, 12, 3) and dense.sim._rigid_body_state.shape == (32, 12, 13)
    # closed loop: the planner drives the base towards the block (robot_to_block / push_align terms)
    q = np.zeros(3)
    d0 = np.hypot(2.5 - 0.31, 1.8 - 1.5)
    for it in range(6):
        a = p.compute_action(q, np.zeros(3)).numpy()
        q = q + 0.1 * a
    front = np.array([q[0] + 0.31 * np.cos(q[2]), 1.5 + q[1] + 0.31 * np.sin(q[2])])
    assert np.hypot(2.5 - front[0], 1.8 - front[1]) < d0


def test_panda_pick_c5_scene_and_cost():
    p = make(pick_cfg(K=16, T=9), PandaPickObjective())
    s = p.sim
    assert s.scene.num_bodies == 17 and s.scene.model.nfree == 1 and s.scene.nu == 9   # SURVEY section 8 table, C5
    q0 = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0, 0.02, 0.02]
    a = p.compute_action(q0, [0.0] * 9)
    assert a.shape == (9,) and torch.isfinite(a).all()
    blk = s.get_actor_position_by_name("panda_pick_block")
    assert blk.shape == (144, 3)
    assert float(blk[-16:, 2].min()) > 0.14 - 0.02 + 0.02 - 0.01                       # the cube fell onto the table (top at 0.14), not through it
    assert s.get_actor_contact_forces_by_name("table", "box").shape == (144, 3)


def test_streamlined_orientation_cost_equals_the_literal_formulation():
    """PandaReachObjective's default arithmetic (3 matrix entries) == the reference's op-by-op version (full matrix)."""
    a = make(panda_cfg(K=64, T=12), PandaReachObjective())
    a.compute_action(Q0, [0] * 7)
    fast = a.objective.compute_cost(a.sim)
    a.objective.literal = True
    lit = a.objective.compute_cost(a.sim)
    np.testing.assert_allclose(fast.numpy(), lit.numpy(), rtol=0, atol=2e-6)
    q = torch.nn.functional.normalize(torch.randn(500, 4, dtype=torch.float64), dim=1)
    from mppi_isaac_b200.objectives import _zyx_first_two
    ref = torch.linalg.norm(matrix_to_euler_angles(quaternion_to_matrix(q), "ZYX")[:, 0:2], axis=1)
    np.testing.assert_allclose(_zyx_first_two(q).numpy(), ref.numpy(), atol=1e-12)


def test_boxer_push_c3_planar_differential_drive():
    """BASELINE config C3: floating differential-drive base (reduced to the plane), 2 wheel DOFs, (v, omega) command."""
    p = make(boxer_cfg(K=32, T=12), PushObjective(robot="boxer", link="ee_link"), observe="all")
    s = p.sim
    assert s.scene.num_bodies == 12 and s.scene.nu == 2 and s.scene.virtual_dofs == 3              # SURVEY section 8 table, C3
    a = p.compute_action([0.0, 2.5, 0.0], [0.0, 0.0, 0.0])
    assert a.shape == (2,) and torch.isfinite(a).all()
    assert s._dof_state.shape == (32 * 12, 4)                                                       # only the wheel DOFs are DOFs
    # diff-drive kinematics: u = (v, 0) for 0.5 s moves the base along its forward axis (-y of the root link) by ~v t
    s.begin_step_mode()
    u = torch.zeros(32, 2); u[:, 0] = 0.8
    for _ in range(10):
        p.dynamics(None, u)
    pos = s.get_actor_position_by_name("boxer")[0].numpy()
    assert abs(pos[0]) < 1e-3 and abs((2.5 - pos[1]) - 0.8 * 0.5) < 0.06
    wheels = s._dof_state[0].numpy()
    np.testing.assert_allclose(wheels[[1, 3]], 0.8 / 0.08, rtol=0.02)                               # both wheels v / r (isaacgym_wrapper.py:510-522)
    u[:, 0], u[:, 1] = 0.0, 1.0
    for _ in range(10):
        p.dynamics(None, u)
    quat = s.get_actor_orientation_by_name("boxer")[0:1]
    assert abs(abs(float(quaternion_to_yaw(quat)[0])) - 0.5) < 0.03                                 # yaw = omega t
    w = s._dof_state[0].numpy()[[1, 3]]
    np.testing.assert_allclose(w, [0.494 / (2 * 0.08), -0.494 / (2 * 0.08)], rtol=0.03)             # right +, left - for a left turn
    # world-state round trip: the base pose arrives in the root state, the wheels in the DOF state
    dof = torch.zeros(1, 4)
    root = torch.from_numpy(s.scene.root_state0.copy()).unsqueeze(0)
    root[0, 0, 0:3] = torch.tensor([0.3, 2.0, 0.05]); root[0, 0, 3:7] = torch.tensor([0.0, 0.0, np.sin(0.35), np.cos(0.35)])
    p.reset_rollout_sim(torch_to_bytes(dof), torch_to_bytes(root))
    np.testing.assert_allclose(s._state0[:3].numpy(), [0.3, 2.0, 0.7], atol=1e-6)
    out = bytes_to_torch(p.command())
    assert out.shape == (2,)
    np.testing.assert_allclose(s.get_actor_position_by_name("boxer")[:32, 0:2].numpy(), [[0.3, 2.0]] * 32, atol=0.08)


def test_halton_spline_mode_runs_the_shipped_style_config():
    """mppi_mode halton-spline + sampling_method halton (what 17 of the 18 shipped conf/mppi files select)."""
    p = make(panda_cfg(K=128, T=12, mppi_mode="halton-spline", sampling_method="halton"), PandaReachObjective())
    assert p.mppi.use_library and p.mppi.n_knots == 3 and p.mppi.backend.params.mode == 1
    z0 = p.mppi.Z.clone()
    a1 = p.compute_action(Q0, [0] * 7)
    a2 = p.compute_action(Q0, [0] * 7)
    assert torch.equal(p.mppi.Z, z0)                                       # the library is drawn once and reused
    assert a1.shape == (7,) and torch.isfinite(a2).all() and float(a1.abs().max()) <= 0.2 + 1e-6
    # mean update: U <- 0.02 U + 0.98 sum_k w_k a_k stays inside the bounds
    assert float(p.mppi.U.abs().max()) <= 0.2 + 1e-6


def test_fast_wire_codec_matches_torch_save_load():
    """transport.FastDecoder / FastEncoder give exactly what torch.load / torch.save give (reference wire format,
    mppiisaac/utils/transport.py:5-14), including after a shape change and for tensors the fast path must refuse."""
    import numpy as np
    from mppi_isaac_b200.utils.transport import FastDecoder, FastEncoder, bytes_to_torch, torch_to_bytes

    g = torch.Generator().manual_seed(5)
    dec, enc = FastDecoder(), FastEncoder()
    for shape in [(1, 14), (1, 14), (1, 9, 13), (2, 7), (1, 14), (3,)]:
        t = torch.randn(shape, generator=g)
        flat, shp = dec(torch_to_bytes(t))
        assert shp == tuple(shape) and np.array_equal(flat, t.reshape(-1).numpy())
    assert dec._tpl[len(torch_to_bytes(torch.zeros(1, 14)))] is not None        # the template path is really in use
    view = torch.randn(14, 2, generator=g)[:, 0]                                 # non-contiguous: payload != tensor
    flat, shp = FastDecoder()(torch_to_bytes(view))
    assert shp == (14,) and np.array_equal(flat, view.numpy())
    f64 = torch.randn(4, generator=g, dtype=torch.float64)
    flat, _ = FastDecoder()(torch_to_bytes(f64))
    assert flat.dtype == np.float32 and np.allclose(flat, f64.numpy())
    like = torch.zeros(7)
    for _ in range(3):
        v = torch.randn(7, generator=g).numpy()
        back = bytes_to_torch(enc(like, v))
        assert back.dtype == torch.float32 and back.shape == (7,) and np.array_equal(back.numpy(), v)
    assert enc._tpl[((7,), "cpu")] is not None


def test_rpc_server_client_speak_the_zerorpc_wire_format():
    """utils/rpc.py: ROUTER/DEALER framing, msgpack [header, name, args] events, OK / ERR answers on the request's channel,
    heart-beats answered in kind -- the request/reply subset of zerorpc v3 the reference uses
    (examples/panda/planner.py:46-48, world.py:21-22,35-50).  The planner methods carry torch.save bytes unchanged."""
    import threading
    import msgpack
    import zmq
    from mppi_isaac_b200.utils.rpc import RemoteError, RpcClient, RpcServer
    from mppi_isaac_b200.utils.transport import bytes_to_torch, torch_to_bytes

    class FakePlanner:
        def compute_action_tensor(self, dof_bytes, root_bytes):
            return torch_to_bytes(bytes_to_torch(dof_bytes)[0, 0:3] + bytes_to_torch(root_bytes).sum())
        def update_weights(self, weights):
            self.weights = weights
            return None
        def boom(self):
            raise ValueError("bad thing")

    planner = FakePlanner()
    server = RpcServer(planner).bind("tcp://127.0.0.1:*")
    endpoint = server.last_endpoint
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    try:
        cli = RpcClient(endpoint, timeout_s=10)
        dof, root = torch.arange(14.0).reshape(1, 14), torch.ones(1, 2, 13)
        out = bytes_to_torch(cli.compute_action_tensor(torch_to_bytes(dof), torch_to_bytes(root)))
        assert torch.equal(out, dof[0, 0:3] + 26.0)
        assert cli.update_weights({"robot_to_goal": 2.0, "robot_ori": 0.25}) is None and planner.weights["robot_ori"] == 0.25
        with pytest.raises(RemoteError, match="ValueError: bad thing"):
            cli.boom()
        with pytest.raises(RemoteError, match="no such method"):
            cli.not_there()
        assert bytes_to_torch(cli.compute_action_tensor(torch_to_bytes(dof), torch_to_bytes(root))).shape == (3,)   # still serving
        # raw frames, as a zerorpc client would put them on the wire
        raw = zmq.Context.instance().socket(zmq.DEALER)
        raw.setsockopt(zmq.LINGER, 0)
        raw.connect(endpoint)
        raw.send_multipart([b"", msgpack.packb([{"message_id": "abc", "v": 3}, "_zpc_hb", []], use_bin_type=True)])
        assert raw.poll(5000)
        frames = raw.recv_multipart()
        header, name, args = msgpack.unpackb(frames[-1], raw=False)
        assert frames[0] == b"" and name == "_zpc_hb" and header["response_to"] == "abc" and header["v"] == 3
        raw.send_multipart([b"", msgpack.packb([{"message_id": "m2", "v": 3}, "update_weights", [{"a": 1.0}]], use_bin_type=True)])
        assert raw.poll(5000)
        header, name, args = msgpack.unpackb(raw.recv_multipart()[-1], raw=False)
        assert name == "OK" and args == [None] and header["response_to"] == "m2" and "message_id" in header
        # malformed events (a non-string method name, a header that is no map, args that are no list) are dropped, the server lives on
        for bad in ([{"message_id": "m3", "v": 3}, 17, []], [["not", "a", "map"], "update_weights", []], [{"message_id": "m4", "v": 3}, "update_weights", 5],
                    [{"message_id": "m5"}, None, None]):
            raw.send_multipart([b"", msgpack.packb(bad, use_bin_type=True)])
        raw.send_multipart([b"", b"\xc1 not msgpack"])
        raw.send_multipart([b"", msgpack.packb([{"message_id": "m6", "v": 3}, "update_weights", [{"b": 2.0}]], use_bin_type=True)])
        assert raw.poll(5000)
        header, name, args = msgpack.unpackb(raw.recv_multipart()[-1], raw=False)
        assert name == "OK" and header["response_to"] == "m6" and planner.weights == {"b": 2.0}
        raw.close()
        cli.close()
    finally:
        server.stop()
        th.join(timeout=5)


@pytest.mark.parametrize("task,objective,q", [
    ("config_albert_b200", lambda: PandaReachObjective(actor="albert", link="mmrobot_link7"), [0, 0, 0, 0, -0.94, 0, -2.8, 0, 1.8675, 0]),
    ("config_panda_effort_b200", lambda: PandaReachObjective(actor="panda", link="panda_link7"), [0, -0.94, 0, -2.8, 0, 1.8675, 0]),
    ("config_omnipanda_pick_b200", lambda: PandaPickObjective(actor="omnipanda", link="panda_hand"), [0, 0, 0, 0, -0.94, 0, -2.8, 0, 1.8675, 0, 0.02, 0.02]),
])
def test_further_example_robots_plan_through_the_api(task, objective, q):
    """SURVEY 8(f) N4: albert (differential-drive base + arm), the panda in effort mode and omnipanda picking from a table build
    from the shipped conf/ + compiled models and plan through the drop-in API (checker backend on the CPU)."""
    import copy
    from mppi_isaac_b200 import load_isaacgym_config
    cfg = copy.deepcopy(load_isaacgym_config(task))
    cfg.mppi.num_samples, cfg.mppi.device = 48, "cpu"
    p = MPPIisaacPlanner(cfg, objective(), backend=OracleBackend(nthreads=8))
    sc = p.sim.scene
    assert cfg.nx == 2 * (sc.ndof - sc.virtual_dofs)                                          # nx of the reference's task files (real DOFs)
    a0 = p.compute_action(q, [0.0] * len(q))
    a1 = p.compute_action(q, [0.0] * len(q))
    assert a0.shape == (sc.nu,) and torch.isfinite(a0).all() and torch.isfinite(a1).all()
    lo, hi = torch.tensor(p.mppi.backend.params.u_min[:sc.nu]), torch.tensor(p.mppi.backend.params.u_max[:sc.nu])
    assert bool(((a1 >= lo - 1e-6) & (a1 <= hi + 1e-6)).all())
    if sc.model.nshapes:
        assert 12 <= sc.model.max_contacts <= 24                                               # sized to the SM's shared memory


def test_examples_panda_planner_and_world_close_the_loop_over_rpc():
    """examples/panda: the planner process' object behind RpcServer, the world process' one-env RolloutSim driving it through
    RpcClient with torch.save bytes (the reference's planner.py / world.py split, examples/panda/planner.py:43-48, world.py:35-50)."""
    import os
    import sys
    import threading
    ex = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "panda")
    sys.path.insert(0, ex)
    try:
        import planner as ex_planner
        import world as ex_world
    finally:
        sys.path.remove(ex)
    from mppi_isaac_b200.utils.rpc import RpcClient, RpcServer
    pl = ex_planner.build_planner(samples=96, device="cpu", backend=OracleBackend(nthreads=8))
    cfg, sim = ex_world.build_world(device="cpu", backend=OracleBackend(nthreads=1))
    server = RpcServer(pl).bind("tcp://127.0.0.1:*")
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    try:
        client = RpcClient(server.last_endpoint, timeout_s=60)
        d0 = ex_world.goal_distance(sim)
        for _ in range(8):
            a = ex_world.control_step(sim, client)
        assert a.shape == (7,) and torch.isfinite(a).all()
        assert ex_world.goal_distance(sim) < d0 - 0.01 and server.calls == 8
        client.close()
    finally:
        server.stop()
        th.join(timeout=5)


def test_compute_action_with_sphere_obstacles():
    """compute_action(q, qdot, obst={...}) (mppi_isaac.py:71-85, isaacgym_wrapper.py:695-746): obstacles become fixed actors named
    sphere<i>; on this path they collide through their bounding boxes and are held at their pose over the horizon."""
    p = make(point_cfg(K=64, T=12), PointReachObjective(), observe="all")
    obst = {"o0": {"position": [0.75, 0.0, 0.1], "velocity": [0.0, 0.0, 0.0], "size": [0.2]}}
    a0 = p.compute_action([0.1, 0.0, 0.0], [0.0, 0.0, 0.0], obst=obst)         # first call: actor added, rollout model rebuilt
    a1 = p.compute_action([0.1, 0.0, 0.0], [0.0, 0.0, 0.0], obst=obst)
    assert [a.name for a in p.sim.env_cfg][-1] == "sphere0" and p.sim.scene.model.nshapes >= 2
    assert torch.isfinite(a0).all() and torch.isfinite(a1).all()
    np.testing.assert_allclose(p.sim.get_actor_position_by_name("sphere0")[0].numpy(), [0.75, 0.0, 0.1], atol=1e-6)
    # the obstacle is solid: driving the point robot along +x for 2 s stops at the box face instead of reaching x = 0.1 + 1.5 * 2
    s = p.sim
    s.reset_robot_state([0.1, 0.0, 0.0], [0.0, 0.0, 0.0])
    s.begin_step_mode()
    u = torch.zeros(64, 3); u[:, 0] = 1.5
    for _ in range(40):
        p.dynamics(None, u)
    x = float(s._dof_state[0, 0])
    assert 0.2 < x < 0.75 - 0.2 + 0.05, x
    moved = obst | {"o0": {"position": [0.75, 2.0, 0.1], "velocity": [0.0, 0.0, 0.0], "size": [0.2]}}
    p.compute_action([0.1, 0.0, 0.0], [0.0, 0.0, 0.0], obst=moved)             # same actor, new pose: no rebuild, free path now
    s.reset_robot_state([0.1, 0.0, 0.0], [0.0, 0.0, 0.0])
    s.begin_step_mode()
    for _ in range(40):
        p.dynamics(None, u)
    assert float(s._dof_state[0, 0]) > 1.5


def test_sphere_obstacle_is_a_sphere_not_its_bounding_box():
    """compute_action(obst=...) obstacles are gym.create_sphere actors (isaacgym_utils.py:42-52): a robot approaching along the
    diagonal is stopped when the CORNER of its collision box reaches the sphere (centre distance r), 5.9 cm later than the corner
    of the sphere's bounding box would stop it.  Point robot (collision box half extent 0.2) driven along (1, 1) from (0.1, 0.1)
    towards a sphere of radius 0.2 at (0.8, 0.8): it comes to rest at x = y = 0.8 - 0.2 / sqrt(2) - 0.2 = 0.4586."""
    p = make(point_cfg(K=16, T=12), PointReachObjective(), observe="all")
    obst = {"o0": {"position": [0.8, 0.8, 0.1], "velocity": [0.0, 0.0, 0.0], "size": [0.2]}}
    p.compute_action([0.1, 0.1, 0.0], [0.0, 0.0, 0.0], obst=obst)
    p.compute_action([0.1, 0.1, 0.0], [0.0, 0.0, 0.0], obst=obst)
    from mppi_isaac_b200.model.blob import SHAPE_SPHERE
    m = p.sim.scene.model
    assert SHAPE_SPHERE in [m.shape_type[s] for s in range(m.nshapes)]
    s = p.sim
    s.reset_robot_state([0.1, 0.1, 0.0], [0.0, 0.0, 0.0])
    s.begin_step_mode()
    u = torch.zeros(16, 3); u[:, 0] = 1.0; u[:, 1] = 1.0
    for _ in range(60):
        p.dynamics(None, u)
    x, y = float(s._dof_state[0, 0]), float(s._dof_state[0, 2])
    assert abs(x - y) < 1e-2, (x, y)         # (the x joint carries the y body: slightly different contact compliance)
    assert 0.445 < x < 0.475 and 0.445 < y < 0.475, (x, y)      # bounding-box contact would hold it at 0.40


def test_jackal_four_wheel_differential_drive():
    """SURVEY 8(f) N4: jackal (conf/actors/jackal.yaml: 4 wheels, r = 0.14, L = 0.4, no wheel-joint lists in the reference's file
    -> inferred from the URDF joint names).  Command map of isaacgym_wrapper.py:510-522 on all four wheels, planar base follows
    the commanded body twist: 1 s of v = 0.5 m/s advances the base by 0.5 m along its heading; omega turns it."""
    from mppi_isaac_b200.model.blob import OBS_DOF_STATE, OBS_LINK_STATE, build_scene, make_params
    from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig, load_actor_cfgs
    from oracle import oracle as orc
    sc = build_scene(load_actor_cfgs(["jackal", "goal"]))
    m = sc.model
    assert m.nb == 7 and m.nu == 2 and m.planar_base == 1 and sc.virtual_dofs == 3
    r, L = 0.14, 0.4
    wheels = {n: i for i, n in enumerate(sc.robot.dof_names)}
    for n, sign in (("front_left_wheel", -1), ("rear_left_wheel", -1), ("front_right_wheel", 1), ("rear_right_wheel", 1)):
        i = wheels[n]
        assert abs(m.cmd_c0[i] - 1 / r) < 1e-5 and abs(m.cmd_c1[i] - sign * L / (2 * r)) < 1e-5
    K, T = 4, 20
    mc = MPPIConfig(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=[[1.0, 0], [0, 1.0]],
                    u_min=[-1.0, -2.0], u_max=[1.0, 2.0], lambda_=0.1)
    p = make_params(mc, IsaacGymConfig(), sc.nu, K, [(OBS_LINK_STATE, 0), (OBS_DOF_STATE, 0)])
    a = np.zeros((T, 2, K), np.float32)
    a[:, 0, :] = 0.5
    a[:, 1, 1] = 1.0                                                         # rollout 1 also turns
    dof0 = sc.dof_state0
    s0 = np.concatenate([dof0[0::2], dof0[1::2]]).astype(np.float32)
    st, obs = orc.rollout(m, p, s0, a, root0=sc.root_state0)
    fwd = np.array([m.fwd_axis[0], m.fwd_axis[1]])
    adv = (st[0:2, 0] - s0[0:2]) @ fwd
    assert abs(adv - 0.5) < 0.03 and abs(st[2, 0] - s0[2]) < 1e-3            # straight: 0.5 m in 1 s, no yaw
    assert abs((st[2, 1] - s0[2]) - 1.0) < 0.06                              # omega = 1 rad/s for 1 s
    assert abs(st[7 + wheels["front_left_wheel"], 0] - 0.5 / r) < 0.05      # wheel speed v / r


# ---------------------------------------------------------------------------------------------------------------------
# net contact forces: at most MAX_SLOTS bodies get a force slot; a read of any other colliding body is refused
# ---------------------------------------------------------------------------------------------------------------------
def _boxes(n):
    from mppi_isaac_b200.utils.config_store import ActorWrapper
    return [ActorWrapper(type="box", name=f"box{i}", size=[0.1, 0.1, 0.1], init_pos=[3.0 + 0.5 * i, -3.0, 0.05], fixed=True) for i in range(n)]


class _ContactReadObjective:
    """Distance to the goal plus the net contact force of each named (actor, link) -- the shape of the push and pick costs."""

    def __init__(self, reads):
        self.reads = reads

    def reset(self):
        pass

    def compute_cost(self, sim):
        r = sim.get_actor_link_by_name("point_robot", "base_link")
        cost = torch.linalg.norm(r[:, 0:2] - sim.get_actor_position_by_name("goal")[:, 0:2], axis=1)
        for actor, link in self.reads(sim):
            cost = cost + torch.sum(torch.abs(sim.get_actor_contact_forces_by_name(actor, link)), axis=1)
        return cost


def test_contact_force_read_without_a_slot_is_refused():
    """Nine static boxes: the first eight get the eight force slots, the ninth collides without one.  An Objective that reads
    its force is refused while the planner traces it, instead of seeing zeros."""
    cfg = point_cfg(K=16, T=9)
    cfg.actors = list(cfg.actors) + _boxes(9)
    with pytest.raises(ObservationError, match=r"'box8'.*no contact-force slot.*at most 8 bodies"):
        make(cfg, _ContactReadObjective(lambda s: [("box8", "box")]))
    # robot links that collide lost their slots to the boxes: refused as well
    with pytest.raises(ObservationError, match="no contact-force slot"):
        make(cfg, _ContactReadObjective(lambda s: [("point_robot", "base_link")]))


def test_contact_force_read_of_a_slotted_or_shapeless_body_builds():
    cfg = point_cfg(K=16, T=9)
    cfg.actors = list(cfg.actors) + _boxes(9)
    reads = [("box0", "box"), ("box7", "box"), ("point_robot", "base_link_x"), ("goal", "sphere")]
    p = make(cfg, _ContactReadObjective(lambda s: reads))
    sc = p.sim.scene
    assert len(sc.contact_slot) == 8 and sc.body_offset[2 + 8] in sc.shape_bodies and sc.body_offset[2 + 8] not in sc.contact_slot
    a = p.compute_action([0.1, 0.0, 0.0], [0.0, 0.0, 0.0])
    assert torch.isfinite(a).all()
    s = p.sim
    assert s.get_actor_contact_forces_by_name("box0", "box").shape == (144, 3)
    for actor, link in reads[2:]:                                   # no collision shape: the force really is zero
        f = s.get_actor_contact_forces_by_name(actor, link)
        assert f.shape == (144, 3) and f.stride(0) == 0 and float(f.abs().max()) == 0.0


def test_obstacle_rebuild_retraces_and_refuses_the_ninth_obstacle():
    """compute_action(obst=...) adds sphere actors and rebuilds the simulator; the re-trace refuses an Objective that reads
    the force on an obstacle that got no slot (the ninth)."""
    def spheres(n):
        return {f"o{i}": {"position": [2.0 + 0.6 * i, -2.0, 0.1], "velocity": [0.0, 0.0, 0.0], "size": [0.1]} for i in range(n)}
    p = make(point_cfg(K=16, T=9), _ContactReadObjective(lambda s: [(a.name, "sphere") for a in s.env_cfg if a.name.startswith("sphere")]))
    a = p.compute_action([0.1, 0.0, 0.0], [0.0, 0.0, 0.0], obst=spheres(8))
    assert torch.isfinite(a).all() and len(p.sim.scene.contact_slot) == 8
    with pytest.raises(ObservationError, match=r"'sphere8'.*no contact-force slot"):
        p.compute_action([0.1, 0.0, 0.0], [0.0, 0.0, 0.0], obst=spheres(9))
