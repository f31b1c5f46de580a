"""-m gpu: every contact-free rollout-kernel instantiation on generated robots (synth_robots.py) against the float64 oracle.

The shipped robots select only a few of the compiled templates; here each case is a generated model whose body count picks a specific
one, and it runs on every mapping that accepts it: lanes (serial chains <= 8 bodies, the default), team (MPPIB_K2_LANES=0) and thread per
rollout (MPPIB_K2_LANES=0 MPPIB_K2_TEAM=0).  The test id names the instantiation:

    lanes <G=4, NB=3>  nb 1..3      lanes <4, 4>   nb 4        lanes <8, 7>  nb 5..7      lanes <8, 8>  nb 8
    team  <8, 4>       nb 1..4      team  <8, 8>   nb 5..8     team <16, 12> nb 9..12     team <16, 16> nb 13..16
    deep16: a 16-body chain, the depth the team kernel's four pointer-jumping rounds reach;  forest: several bodies on the root link

The models have arbitrary joint axes and origins on a rotated, shifted base, rotated inertial frames, off-centre centres of mass, a
fixed-joint link, a 1 g link and saturating drives.  Each test prints its worst errors ("SYNTH ..." lines, visible with -s)."""
import copy

import numpy as np
import pytest
import torch

from synth_robots import make_robot

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

CASES = [(nb, "chain") for nb in range(1, 9)] + [(4, "star"), (5, "tree"), (9, "forest"), (12, "tree"), (13, "tree"), (16, "forest"),
                                                  (16, "tree"), (16, "deep")]
KNOBS = {"lanes": {}, "team": {"MPPIB_K2_LANES": "0"}, "thread": {"MPPIB_K2_LANES": "0", "MPPIB_K2_TEAM": "0"}}


def instantiation(mapping, nb):
    """(name, rollouts per warp) of the template `mapping` launches for nb bodies (launch_rollout_lanes / launch_rollout_team)."""
    if mapping == "lanes":
        G, NB = (4, 3) if nb <= 3 else (4, 4) if nb == 4 else (8, 7) if nb <= 7 else (8, 8)
        return f"lanes_G{G}_NB{NB}", 32 // G
    if mapping == "team":
        G, NB = (8, 4) if nb <= 4 else (8, 8) if nb <= 8 else (16, 12) if nb <= 12 else (16, 16)
        return f"team_G{G}_NB{NB}", 32 // G
    return "thread", 32


def _params():
    out = []
    for nb, topo in CASES:
        for mapping in (("lanes", "team", "thread") if topo == "chain" else ("team", "thread")):
            out.append(pytest.param(nb, topo, mapping, id=f"{topo}{nb}-{instantiation(mapping, nb)[0]}"))
    return out


PARAMS = _params()


@pytest.fixture(scope="module")
def synth_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("synth")


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(DEV)


def backend(monkeypatch, sc, p, mapping, model=None):
    """A handle created under the mapping's knobs; asserts that the library really runs that mapping."""
    from mppi_isaac_b200.backend import CudaBackend
    for k in ("MPPIB_K2_LANES", "MPPIB_K2_TEAM"):
        monkeypatch.delenv(k, raising=False)
    for k, v in KNOBS[mapping].items():
        monkeypatch.setenv(k, v)
    be = CudaBackend(DEV)
    be.create(model if model is not None else sc.model, p)
    assert be.rollout_mapping().startswith(mapping), (mapping, be.rollout_mapping())
    return be


def report(test, **vals):
    print(f"SYNTH {test} " + " ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}" for k, v in vals.items()))


def _random_states(sc, s0, K, rng, spread=0.2):
    """(2 nb, K) per-rollout states around s0, inside the joint limits."""
    m, nb = sc.model, sc.ndof
    st = np.repeat(s0[:, None], K, 1).astype(np.float64)
    st[:nb] += rng.uniform(-spread, spread, (nb, K))
    lo, hi = np.array(m.q_lo[:nb], np.float64)[:, None], np.array(m.q_hi[:nb], np.float64)[:, None]
    st[:nb] = np.clip(st[:nb], lo + 0.02, hi - 0.02)
    st[nb:] += rng.uniform(-0.3, 0.3, (nb, K))
    return st.astype(np.float32)


def _unlimited(model):
    """The model without effort / velocity / position limits: its one-step velocities are the oracle's first (unsaturated) solve."""
    free = copy.deepcopy(model)
    for i in range(model.nb):
        free.effort[i], free.qd_max[i], free.q_lo[i], free.q_hi[i] = 1e30, 1e30, -1e30, 1e30
    return free


def lockstep(oracle, monkeypatch, sc, p, mapping, actions, state, steps):
    """The oracle's state re-injected before every step: the one-step error of the kernel alone.  Rollouts whose unsaturated drive
    torque lies within 1e-3 (relative) of the effort limit may take the other saturation decision in float32 and are left out; returns
    (worst |dq|, worst |dqd|, excluded rollout-steps)."""
    be = backend(monkeypatch, sc, p, mapping)
    m, nb, K = sc.model, sc.ndof, p.K
    a_d = dev(actions)
    free = _unlimited(m)
    eff = np.array(m.effort[:nb], np.float64)[:, None]
    kd = np.array(m.kd[:nb], np.float64)[:, None]
    worst_q = worst_qd = 0.0
    excluded = 0
    for t in range(steps):
        st = dev(state)
        be.rollout(None, st, a_d, t, 1, None)
        ref, _ = oracle.rollout(m, p, None, actions, t, 1, state=state.copy(), want_obs=False, use_double=True)
        near = np.zeros(K, bool)
        if m.drive_mode == 0:
            unsat, _ = oracle.rollout(free, p, None, actions, t, 1, state=state.copy(), want_obs=False, use_double=True)
            tgt = np.array([m.cmd_c0[i] * actions[t, m.cmd_i0[i]] + m.cmd_c1[i] * actions[t, m.cmd_i1[i]] for i in range(nb)], np.float64) * p.u_scale
            td = kd * (tgt - unsat[nb:2 * nb].astype(np.float64))
            near = (np.abs(np.abs(td) / eff - 1.0) <= 1e-3).any(axis=0)
        g = st.cpu().numpy()
        assert np.isfinite(g).all()
        excluded += int(near.sum())
        keep = ~near
        worst_q = max(worst_q, float(np.abs(g[:nb, keep] - ref[:nb, keep]).max()))
        worst_qd = max(worst_qd, float(np.abs(g[nb:2 * nb, keep] - ref[nb:2 * nb, keep]).max()))
        state = ref
    return worst_q, worst_qd, excluded


@pytest.mark.parametrize("nb,topology,mapping", PARAMS)
def test_one_step_lockstep(oracle, monkeypatch, synth_dir, nb, topology, mapping):
    K, T = 128, 6
    sc, p, s0 = make_robot(synth_dir, 0, nb, topology, K=K, T=T)
    rng = np.random.default_rng(nb)
    actions = rng.uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    actions[:, :, : K // 4] *= 0.05                                          # a quarter of the rollouts never saturates
    wq, wqd, excl = lockstep(oracle, monkeypatch, sc, p, mapping, actions, _random_states(sc, s0, K, rng), T)
    report("lockstep", id=f"{topology}{nb}-{mapping}", dq=wq, dqd=wqd, excluded=excl)
    assert wq <= 1e-5                                                        # stated gate
    assert wq <= 2e-6 and wqd <= 1e-4, (wq, wqd)                             # what float32 delivers (measured 5.7e-7 / 2.9e-5, deep16)
    assert excl <= K * T // 50                                               # the exclusion stays a rare edge case (measured <= 3)


def _compare_free_running(sc, o, s, o_ref, st_ref):
    """Per-rollout worst errors of the state and of every observed row over the horizon."""
    nb = sc.ndof
    err = {"q": np.abs(s[:nb] - st_ref[:nb]).max(axis=0), "qd": np.abs(s[nb:2 * nb] - st_ref[nb:2 * nb]).max(axis=0)}
    pos, quat, vel = [], [], []
    for j in range(3):                                                       # root link, fixed-joint link, tip
        r = 13 * j
        pos.append(np.abs(o[r:r + 3] - o_ref[r:r + 3]).max(axis=(0, 1)))
        qa, qb = o[r + 3:r + 7], o_ref[r + 3:r + 7]
        quat.append(np.minimum(np.abs(qa - qb), np.abs(qa + qb)).max(axis=(0, 1)))
        vel.append(np.abs(o[r + 7:r + 13] - o_ref[r + 7:r + 13]).max(axis=(0, 1)))
    err["pos"], err["quat"], err["vel"] = np.max(pos, axis=0), np.max(quat, axis=0), np.max(vel, axis=0)
    err["dof_q"] = np.abs(o[39::2][:nb] - o_ref[39::2][:nb]).max(axis=(0, 1))
    err["dof_qd"] = np.abs(o[40::2][:nb] - o_ref[40::2][:nb]).max(axis=(0, 1))
    return err


# per-rollout worst error over T = 12 steps: (median, 0.97 quantile) gates, and a loose bound on the worst rollout.  A saturation decision
# taken at the threshold can flip between float32 and float64 and changes that joint's torque for one substep, so the tight gates are on
# quantiles over the rollouts.  Measured on an H100 over every case: medians <= 3.6e-6, 0.97 quantiles <= 1.1e-5, worst 2.0e-5 (deep16
# on the team kernel); positions / quaternions are 10x below the velocities.
FREE_GATES = {"q": (2e-6, 1e-5), "qd": (2e-5, 1e-4), "pos": (5e-6, 2e-5), "quat": (2e-6, 1e-5), "vel": (2e-5, 1e-4),
              "dof_q": (2e-6, 1e-5), "dof_qd": (2e-5, 1e-4)}


def check_free_running(err):
    for k, (g_med, g_q97) in FREE_GATES.items():
        assert np.median(err[k]) <= g_med and np.quantile(err[k], 0.97) <= g_q97, (k, np.median(err[k]), np.quantile(err[k], 0.97))
        assert err[k].max() <= 100 * g_q97, (k, err[k].max())


@pytest.mark.parametrize("substeps", [1, 3])
@pytest.mark.parametrize("nb,topology,mapping", PARAMS)
def test_free_running(oracle, monkeypatch, synth_dir, nb, topology, mapping, substeps):
    K, T = 256, 12
    sc, p, s0 = make_robot(synth_dir, 0, nb, topology, K=K, T=T, dt=0.03, substeps=substeps)
    be = backend(monkeypatch, sc, p, mapping)
    rng = np.random.default_rng(100 + nb)
    actions = rng.uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    actions[:, :, : K // 4] *= 0.05
    obs, state = torch.zeros((be.obs_size(), T, K), device=DEV), torch.zeros((be.state_size(), K), device=DEV)
    be.rollout(dev(s0), state, dev(actions), 0, T, obs)
    st_ref, obs_ref = oracle.rollout(sc.model, p, s0, actions, use_double=True, nthreads=8)
    o, s = obs.cpu().numpy(), state.cpu().numpy()
    assert np.isfinite(o).all() and np.isfinite(s).all()
    err = _compare_free_running(sc, o, s, obs_ref, st_ref)
    report("free", id=f"{topology}{nb}-{mapping}-sub{substeps}", **{f"{k}_med": float(np.median(v)) for k, v in err.items()},
           **{f"{k}_q97": float(np.quantile(v, 0.97)) for k, v in err.items()}, **{f"{k}_max": float(v.max()) for k, v in err.items()})
    check_free_running(err)
    assert np.abs(s[:nb] - s0[:nb, None]).max() > 1e-2                       # something actually moved


SENTINEL, GUARD_VALUE, GUARD = float("nan"), -7777.0, 64


def _guarded(n, fill):
    """A view of n floats filled with `fill`, followed by a guard band of GUARD floats."""
    buf = torch.full((n + GUARD,), GUARD_VALUE, device=DEV)
    buf[:n] = fill
    return buf, buf[:n]


@pytest.mark.parametrize("nb,topology,mapping", PARAMS)
def test_ragged_k(monkeypatch, synth_dir, nb, topology, mapping):
    """K that leaves the last warp partly empty: every rollout below K is bit-identical to the same rollout of a launch with K rounded up
    to the rollouts per warp, every output below K is written, and nothing past K is.  Broadcast state0, per-rollout state, and
    nsteps = 0 (observe only)."""
    name, rpw = instantiation(mapping, nb)
    n, T = 3, 5
    Ks = sorted({1, max(1, rpw - 1), rpw * n + 1, rpw * n + rpw - 1})
    K_max = -(-Ks[-1] // rpw) * rpw
    rng = np.random.default_rng(nb)
    sc0, _, s0 = make_robot(synth_dir, 0, nb, topology, K=8, T=T, substeps=2, dt=0.03)
    acts = rng.uniform(-0.5, 0.5, (T, sc0.nu, K_max)).astype(np.float32)
    states = _random_states(sc0, s0, K_max, rng)
    checked = 0
    for K in Ks:
        Kup = -(-K // rpw) * rpw
        assert Kup > K
        outs = {}
        for KK in (K, Kup):
            sc, p, _ = make_robot(synth_dir, 0, nb, topology, K=KK, T=T, substeps=2, dt=0.03)
            be = backend(monkeypatch, sc, p, mapping)
            R, NS = be.obs_size(), be.state_size()
            a_d = dev(acts[:, :, :KK])
            res = {}
            for mode in ("state0", "state", "observe"):
                obuf, obs = _guarded(R * T * KK, SENTINEL)
                if mode == "state0":
                    sbuf, st = _guarded(NS * KK, SENTINEL)
                    be.rollout(dev(s0), st.view(NS, KK), a_d, 0, T, obs.view(R, T, KK))
                else:
                    sbuf, st = _guarded(NS * KK, 0.0)
                    st.copy_(dev(states[:, :KK]).reshape(-1))
                    if mode == "state":
                        be.rollout(None, st.view(NS, KK), a_d, 0, T, obs.view(R, T, KK))
                    else:
                        be.rollout(None, st.view(NS, KK), a_d, 2, 0, obs.view(R, T, KK))
                torch.cuda.synchronize()
                assert bool((obuf[-GUARD:] == GUARD_VALUE).all()) and bool((sbuf[-GUARD:] == GUARD_VALUE).all()), (mode, K, KK)
                res[mode] = (obs.view(R, T, KK)[:, :, :K].cpu().numpy(), st.view(NS, KK)[:, :K].cpu().numpy())
            outs[KK] = res
        for mode in ("state0", "state", "observe"):
            (o, s), (o_up, s_up) = outs[K][mode], outs[Kup][mode]
            written = o if mode != "observe" else o[:, 2]
            assert not np.isnan(written).any() and not np.isnan(s).any(), (mode, K)
            if mode == "observe":
                assert np.isnan(np.delete(o, 2, axis=1)).all()               # observe-only writes its slot and nothing else
            np.testing.assert_array_equal(o, o_up, err_msg=f"{mode} K={K}")
            np.testing.assert_array_equal(s, s_up, err_msg=f"{mode} K={K}")
            checked += 1
    report("ragged", id=f"{topology}{nb}-{mapping}", Ks=",".join(map(str, Ks)), checked=checked)


@pytest.mark.parametrize("nb,topology,mapping", PARAMS)
def test_position_stops_and_velocity_clamp(oracle, monkeypatch, synth_dir, nb, topology, mapping):
    """Joints start within 0.01 of a stop and are driven into it faster than a small qd_max: the kernel matches the oracle's stop and
    clamp per joint -- q stays in [lo, hi], the velocity into a stop is zeroed, |qd| is clamped to qd_max -- and both really happen."""
    K, T = 64, 12
    sc, p, s0 = make_robot(synth_dir, 3, nb, topology, K=K, T=T)
    m = copy.deepcopy(sc.model)
    for i in range(nb):
        m.qd_max[i] = 0.4
    rng = np.random.default_rng(nb)
    lo, hi = np.array(m.q_lo[:nb], np.float64), np.array(m.q_hi[:nb], np.float64)
    side = rng.choice([-1.0, 1.0], (nb, K))
    limited = (hi < 1e29)[:, None]
    q0 = np.where(side > 0, hi[:, None] - rng.uniform(0, 0.01, (nb, K)), lo[:, None] + rng.uniform(0, 0.01, (nb, K)))
    q0 = np.where(limited, q0, rng.uniform(-1, 1, (nb, K)))
    state = np.concatenate([q0, np.zeros((nb, K))]).astype(np.float32)
    actions = (np.repeat(side[None], T, 0) * rng.uniform(0.6, 1.0, (T, nb, K))).astype(np.float32)
    be = backend(monkeypatch, sc, p, mapping, model=m)
    obs, st = torch.zeros((be.obs_size(), T, K), device=DEV), dev(state)
    be.rollout(None, st, dev(actions), 0, T, obs)
    st_ref, obs_ref = oracle.rollout(m, p, None, actions, state=state.copy(), use_double=True)
    o, s = obs.cpu().numpy(), st.cpu().numpy()
    q, qd, q_ref, qd_ref = o[39::2][:nb], o[40::2][:nb], obs_ref[39::2][:nb], obs_ref[40::2][:nb]      # (nb, T, K)
    lo32, hi32 = np.array(m.q_lo[:nb], np.float32)[:, None, None], np.array(m.q_hi[:nb], np.float32)[:, None, None]
    assert (q >= lo32).all() and (q <= hi32).all()
    at_lo, at_hi = q == lo32, q == hi32
    # a step that would cross a stop ends on it with the velocity into it zeroed; a joint left at a stop with velocity into it got there
    # by a step that lands exactly on it (q_prev + h qd == stop after rounding: the stop was not crossed -- the oracle does the same)
    h = p.dt / p.substeps
    q_prev = np.concatenate([state[:nb, None, :], q[:, :-1]], axis=1).astype(np.float64)
    into = (at_lo & (qd < 0)) | (at_hi & (qd > 0))
    landed = np.abs(q_prev + h * qd.astype(np.float64) - q) <= 2 * np.spacing(np.abs(q))
    assert landed[into].all()
    clamp = np.abs(qd) == np.float32(0.4)
    stop_ref = (q_ref == lo32) | (q_ref == hi32)
    clamp_ref = np.abs(qd_ref) == np.float32(0.4)
    same_stop, same_clamp = float(np.mean((at_lo | at_hi) == stop_ref)), float(np.mean(clamp == clamp_ref))
    wq, wqd = float(np.abs(q - q_ref).max()), float(np.abs(qd - qd_ref).max())
    report("limits", id=f"{topology}{nb}-{mapping}", stops=int((at_lo | at_hi).sum()), landed=int(into.sum()), clamps=int(clamp.sum()), same_stop=same_stop,
           same_clamp=same_clamp, dq=wq, dqd=wqd)
    if limited.any():
        assert (at_lo | at_hi)[limited[:, 0]].any(axis=(1, 2)).all()        # every joint with stops reached one
    assert clamp.any()                                                      # the velocity clamp engaged
    assert same_stop >= 0.999 and same_clamp >= 0.999                       # measured: identical in every case
    assert wq <= 1e-5 and wqd <= 1e-4 and np.abs(s[:nb] - st_ref[:nb]).max() <= 1e-5   # measured 1.2e-6 / 4.4e-6 (tree13)


EFFORT_PARAMS = [p for p in PARAMS if p.values[:2] in ((8, "chain"), (16, "tree"))]


@pytest.mark.parametrize("nb,topology,mapping", EFFORT_PARAMS)
def test_effort_mode_gravity_weak_drive(oracle, monkeypatch, synth_dir, nb, topology, mapping):
    """Commands are torques, gravity on, a weak drive (kd 0.5, damping 0.1): M(q), Coriolis and gravity all shape the motion."""
    K, T = 128, 12
    sc, p, s0 = make_robot(synth_dir, 4, nb, topology, K=K, T=T, dt=0.01, substeps=2, dof_mode="effort", gravity=True, u_lim=2.0)
    m = sc.model
    for i in range(nb):
        m.kd[i], m.damping[i] = 0.5, 0.1
    rng = np.random.default_rng(nb)
    actions = rng.uniform(-2.0, 2.0, (T, sc.nu, K)).astype(np.float32)
    wq, wqd, _ = lockstep(oracle, monkeypatch, sc, p, mapping, actions, _random_states(sc, s0, K, rng, spread=0.1), T)
    be = backend(monkeypatch, sc, p, mapping)
    obs, state = torch.zeros((be.obs_size(), T, K), device=DEV), torch.zeros((be.state_size(), K), device=DEV)
    be.rollout(dev(s0), state, dev(actions), 0, T, obs)
    st_ref, obs_ref = oracle.rollout(m, p, s0, actions, use_double=True, nthreads=8)
    s = state.cpu().numpy()
    err = _compare_free_running(sc, obs.cpu().numpy(), s, obs_ref, st_ref)
    report("effort", id=f"{topology}{nb}-{mapping}", dq_lockstep=wq, dqd_lockstep=wqd, **{f"{k}_max": float(v.max()) for k, v in err.items()})
    assert wq <= 1e-5 and wq <= 5e-6 and wqd <= 1e-4, (wq, wqd)              # measured 1.4e-6 / 8.8e-6 (tree16)
    check_free_running(err)
    # gravity matters: the same torques without it end elsewhere
    m0 = copy.deepcopy(m)
    m0.gravity_on = 0
    st0, _ = oracle.rollout(m0, p, s0, actions, use_double=True, want_obs=False, nthreads=8)
    assert np.abs(st0[:nb] - st_ref[:nb]).max() > 1e-3


@pytest.mark.parametrize("nb", range(1, 9))
def test_mappings_agree_on_one_step(monkeypatch, synth_dir, nb):
    """lanes, team and thread per rollout from the same per-rollout state, one model step (3 substeps), no oracle in between: float32
    rounding apart."""
    K, T = 256, 2
    sc, p, s0 = make_robot(synth_dir, 5, nb, "chain", K=K, T=T, dt=0.03, substeps=3)
    rng = np.random.default_rng(nb)
    actions = dev(rng.uniform(-0.5, 0.5, (T, sc.nu, K)) * (rng.uniform(size=K) < 0.75) + 0.02 * rng.uniform(-1, 1, (T, sc.nu, K)))
    state = dev(_random_states(sc, s0, K, rng))
    out = {}
    for mapping in ("lanes", "team", "thread"):
        be = backend(monkeypatch, sc, p, mapping)
        st = state.clone()
        obs = torch.zeros((be.obs_size(), T, K), device=DEV)
        be.rollout(None, st, actions, 0, 1, obs)
        out[mapping] = (st.cpu().numpy(), obs[:, 0].cpu().numpy())
    dq = max(float(np.abs(out[a][0][:nb] - out[b][0][:nb]).max()) for a, b in (("lanes", "team"), ("lanes", "thread"), ("team", "thread")))
    dqd = max(float(np.abs(out[a][0][nb:] - out[b][0][nb:]).max()) for a, b in (("lanes", "team"), ("lanes", "thread"), ("team", "thread")))
    dobs = max(float(np.abs(out[a][1][0:39] - out[b][1][0:39]).max()) for a, b in (("lanes", "team"), ("lanes", "thread"), ("team", "thread")))
    report("cross", id=f"chain{nb}", dq=dq, dqd=dqd, dobs_links=dobs)
    assert dq <= 1e-6 and dqd <= 5e-5 and dobs <= 2e-5, (dq, dqd, dobs)       # measured 2.2e-7 / 9.5e-6 / 4.7e-6 (chain8)
