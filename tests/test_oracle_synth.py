"""The oracle (the float64 spec every rollout kernel is held to) on generated robots (synth_robots.py): arbitrary joint axes, a rotated
base, rotated inertial frames, prismatic / revolute / continuous mixes, saturating drives, chains of 1..8 bodies and trees / forests of
up to 16.  Checked against code it shares nothing with -- the Lagrangian dynamics of lagrange_ref.py and the host forward kinematics --
and against the float64 restatements of the lanes / team kernels; plus the kernel each generated model is routed to."""
import ctypes as C
import os

import numpy as np
import pytest

from mppi_isaac_b200.model.urdf import forward_kinematics, quat_xyzw_to_R
from lagrange_ref import forward_dynamics
from synth_robots import depth, is_chain, make_robot

CHAINS = [(nb, "chain") for nb in range(1, 9)]
TREES = [(5, "tree"), (9, "forest"), (12, "tree"), (13, "tree"), (16, "forest")]
# every generated model of the GPU suite (test_gpu_synth.py), for the mapping check
ALL = CHAINS + [(4, "star"), (5, "tree"), (9, "forest"), (12, "tree"), (13, "tree"), (16, "forest"), (16, "tree"), (16, "deep")]


def _ids(cases):
    return [f"{topology}{nb}" for nb, topology in cases]


@pytest.fixture(scope="module")
def synth_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("synth")


def _qdd_reference(sc, q, qd, u, h):
    """Lagrangian qdd of one substep with the velocity drive, the saturation re-solve included; the base rotation enters as gravity
    expressed in the base frame."""
    m, nb = sc.model, sc.ndof
    kd, b = np.array(m.kd[:nb], np.float64), np.array(m.damping[:nb], np.float64)
    eff = np.array(m.effort[:nb], np.float64)
    tgt = np.array([m.cmd_c0[i] * u[m.cmd_i0[i]] + m.cmd_c1[i] * u[m.cmd_i1[i]] for i in range(nb)])
    Rb = quat_xyzw_to_R(np.array(m.base_quat[:], np.float64))
    grav = tuple(Rb.T @ np.array(m.gravity[:], np.float64)) if m.gravity_on else (0.0, 0.0, 0.0)
    tau, dimp = kd * (tgt - qd) - b * qd, h * (kd + b)
    qdd, _ = forward_dynamics(sc.robot, q, qd, tau, dimp, grav)
    td = kd * (tgt - (qd + h * qdd.numpy()))
    sat = np.abs(td) > eff
    if sat.any():
        tau = np.where(sat, np.sign(td) * eff - b * qd, tau)
        dimp = np.where(sat, h * b, dimp)
        qdd, _ = forward_dynamics(sc.robot, q, qd, tau, dimp, grav)
    return qdd.numpy(), int(sat.sum())


@pytest.mark.parametrize("nb,topology", CHAINS + TREES, ids=_ids(CHAINS + TREES))
def test_oracle_qdd_matches_lagrangian(oracle, synth_dir, nb, topology):
    """One substep of the oracle's float64 path (qdd = (qd_new - qd) / h) against the Lagrangian on a rotated base."""
    h = 1e-3
    sc, p, _ = make_robot(synth_dir, 0, nb, topology, K=2, T=1, dt=h, substeps=1)
    m = sc.model
    for i in range(0, nb, 2):
        m.effort[i] *= 0.03                     # at h = 1 ms the implicit drive barely needs torque: weaken every other one so it saturates
    assert any(abs(v) > 1e-3 for v in m.base_quat[:3])                        # the base really is rotated
    rng = np.random.default_rng(nb)
    saturated = 0
    for trial in range(2 if nb <= 8 else 1):
        lo = np.maximum(np.array(m.q_lo[:nb]), -2.0) + 0.05
        hi = np.minimum(np.array(m.q_hi[:nb]), 2.0) - 0.05
        q = rng.uniform(lo, hi).astype(np.float32).astype(np.float64)
        qd = rng.uniform(-0.8, 0.8, nb).astype(np.float32).astype(np.float64)
        u = rng.uniform(-0.5, 0.5, sc.nu).astype(np.float32).astype(np.float64)
        qdd_ref, nsat = _qdd_reference(sc, q, qd, u, h)
        saturated += nsat
        actions = np.repeat(u.astype(np.float32)[None, :, None], 2, axis=2)
        st, _ = oracle.rollout(m, p, np.concatenate([q, qd]).astype(np.float32), actions, 0, 1, want_obs=False, use_double=True)
        qdd = (st[nb:2 * nb, 0].astype(np.float64) - qd) / h
        # float32 state / model constants and the float32 step (qd_new is stored in float32: 1 ulp of qd_new / h ~ 1e-4)
        np.testing.assert_allclose(qdd, qdd_ref, rtol=2e-4, atol=2e-3)
    assert saturated > 0                                                       # the re-solve path was part of the comparison


FK_CASES = [(3, "chain"), (8, "chain"), (9, "forest"), (16, "tree"), (16, "deep")]


@pytest.mark.parametrize("nb,topology", FK_CASES, ids=_ids(FK_CASES))
def test_oracle_link_poses_match_forward_kinematics(oracle, synth_dir, nb, topology):
    """Every observed link (the root link, the fixed-joint link, the tip) at every step == host FK of the observed q on the base pose."""
    K, T = 4, 5
    sc, p, s0 = make_robot(synth_dir, 1, nb, topology, K=K, T=T)
    m = sc.model
    actions = np.random.default_rng(nb).uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    _, obs = oracle.rollout(m, p, s0, actions, use_double=True)
    base_pos, base_quat = np.array(m.base_pos[:], np.float64), np.array(m.base_quat[:], np.float64)
    links = [p.obs[j].index for j in range(3)]
    assert [m.link_body[l] for l in links][0] == -1 and sc.robot.link_names[links[1]] == "fx"
    for t in range(T):
        for k in range(K):
            q = obs[39::2, t, k][:nb].astype(np.float64)
            pos, quat = forward_kinematics(sc.robot, q, base_pos, base_quat)
            for j, l in enumerate(links):
                row = obs[13 * j:13 * j + 13, t, k].astype(np.float64)
                np.testing.assert_allclose(row[0:3], pos[l], atol=2e-6, rtol=0)
                qa, qb = row[3:7], quat[l]
                assert min(np.abs(qa - qb).max(), np.abs(qa + qb).max()) <= 2e-6


def _against_oracle(oracle, proto, sc, p, s0, actions):
    st_ref, _ = oracle.rollout(sc.model, p, s0, actions, use_double=True, want_obs=False)
    nb = sc.ndof
    worst_q = worst_qd = 0.0
    for k in range(actions.shape[2]):
        q, qd = proto.rollout(sc.model, p, s0, actions[:, :, k].astype(np.float64))[:2]
        worst_q = max(worst_q, float(np.abs(q - st_ref[:nb, k]).max()))
        worst_qd = max(worst_qd, float(np.abs(qd - st_ref[nb:2 * nb, k]).max()))
    return worst_q, worst_qd


@pytest.mark.parametrize("nb", range(1, 9))
@pytest.mark.parametrize("substeps", [1, 3])
def test_proto_lanes_matches_oracle(oracle, synth_dir, nb, substeps):
    """The float64 restatement of the lanes kernel (frames by scan, composite bodies, distributed LDL^T) == the oracle's ABA."""
    import proto_lanes
    K, T = 4, 6
    sc, p, s0 = make_robot(synth_dir, 2, nb, "chain", K=K, T=T, dt=0.03, substeps=substeps)
    actions = np.random.default_rng(nb).uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    actions[:, :, 0] *= 6.0                                                   # far past the effort limits: the re-solve path
    wq, wqd = _against_oracle(oracle, proto_lanes, sc, p, s0, actions)
    assert wq <= 2e-6 and wqd <= 2e-4, (wq, wqd)


TEAM_CASES = [(4, "star"), (5, "tree"), (9, "forest"), (13, "tree"), (16, "deep")]


@pytest.mark.parametrize("nb,topology", TEAM_CASES, ids=_ids(TEAM_CASES))
def test_proto_team_matches_oracle(oracle, synth_dir, nb, topology):
    """The float64 restatement of the team kernel's articulation phase (pointer jumping, subtree sums) == the oracle's ABA."""
    import proto_team
    K, T = 3, 6
    sc, p, s0 = make_robot(synth_dir, 2, nb, topology, K=K, T=T, dt=0.03, substeps=2)
    actions = np.random.default_rng(nb).uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    actions[:, :, 0] *= 6.0
    wq, wqd = _against_oracle(oracle, proto_team, sc, p, s0, actions)
    assert wq <= 2e-6 and wqd <= 2e-4, (wq, wqd)


def _mapping(model, **env):
    from mppi_isaac_b200 import backend
    lib = backend.load_library()
    old = {k: os.environ.get(k) for k in ("MPPIB_K2_LANES", "MPPIB_K2_TEAM")}
    try:
        for k in old:
            os.environ.pop(k, None)
        os.environ.update(env)
        return backend.CudaBackend.MAPPING_NAMES[lib.mppib_rollout_mapping_for_model(C.byref(model))].split("-")[0]
    finally:
        for k, v in old.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v


@pytest.mark.parametrize("nb,topology", ALL, ids=_ids(ALL))
def test_generated_models_reach_the_intended_kernel(synth_dir, nb, topology):
    """Chains of <= 8 bodies -> lanes kernel, every other generated model -> team kernel (the deep chain is 16 bodies deep, the limit
    of its four pointer-jumping rounds); MPPIB_K2_LANES=0 moves chains to the team kernel, both knobs off -> thread per rollout."""
    sc, _, _ = make_robot(synth_dir, 0, nb, topology, K=8, T=2)
    m = sc.model
    chain = is_chain(m) and nb <= 8
    assert is_chain(m) == (topology in ("chain", "deep"))
    if topology == "forest":
        assert sum(m.parent[i] < 0 for i in range(nb)) >= 2
    if topology == "deep":
        assert depth(m) == 16
    assert _mapping(m) == ("lanes" if chain else "team")
    assert _mapping(m, MPPIB_K2_LANES="0") == "team"
    assert _mapping(m, MPPIB_K2_TEAM="0") == ("lanes" if chain else "thread")
    assert _mapping(m, MPPIB_K2_LANES="0", MPPIB_K2_TEAM="0") == "thread"
