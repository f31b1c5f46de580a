"""-m gpu: every contact instantiation of the rollout kernels on generated scenes with several free bodies (synth_scenes.py) against the
float64 oracle, on both contact mappings: team of lanes (the default; <G, NB, true, NCS, 8, COMPACT>, the test id names it) and thread
per rollout (MPPIB_K2_TEAM=0).

Contacts switch on margins, face choices and the contact cap, and float32 may take the other branch at a threshold: the lock-step
test runs the float64 oracle also from two copies of the state with every position row moved by +-2e-6 (more than float32 rounding
does) and leaves out the rollout-steps whose result moves by more than a gate under that probe (a threshold was crossed: no
float32 implementation can be held to the float64 branch there); it counts them and bounds them at 2 %.  Each test
prints its worst errors ("SYNTH-CONTACT ..." lines, visible with -s)."""
import copy

import numpy as np
import pytest
import torch

from synth_scenes import CASES, case_id, cube_collision_scene, make_case, stack_scene
from test_gpu_synth import GUARD, GUARD_VALUE, _guarded, backend, dev
from test_oracle_contact_synth import _initial_momenta, free_rows, momenta

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MAPPINGS = ("team", "thread")
PARAMS = [pytest.param(c, mp, id=f"{case_id(c)}-{mp}" if mp == "team" else f"{case_id(c).rsplit('-', 1)[0]}-thread") for c in CASES
          for mp in MAPPINGS]
PROBE = 2e-6


@pytest.fixture(scope="module")
def synth_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("synth_contact_gpu")


def report(test, **vals):
    print(f"SYNTH-CONTACT {test} " + " ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}" for k, v in vals.items()))


def _rows(sc):
    """State rows: positions (joint q, free x and quaternion) and velocities (joint qd, free v and w)."""
    nb, nf = sc.ndof, sc.model.nfree
    pos = list(range(nb)) + [2 * nb + 13 * f + r for f in range(nf) for r in range(7)]
    vel = list(range(nb, 2 * nb)) + [2 * nb + 13 * f + r for f in range(nf) for r in range(7, 13)]
    return np.array(pos), np.array(vel)


def _errors(sc, s, o, s_ref, o_ref):
    """Per-rollout errors of one step: positions, velocities, observed free-body rows, contact forces (relative to max(1, |F|))."""
    nb, nf = sc.ndof, sc.model.nfree
    pos, vel = _rows(sc)
    f0 = 2 * nb + 13 * nf
    F_ref = o_ref[f0:]
    scale = np.maximum(1.0, np.abs(F_ref).max(axis=0)) if len(F_ref) else 1.0
    return {"pos": np.abs(s[pos] - s_ref[pos]).max(axis=0), "vel": np.abs(s[vel] - s_ref[vel]).max(axis=0),
            "obs_free": np.abs(o[2 * nb:f0] - o_ref[2 * nb:f0]).max(axis=0) if nf else np.zeros(s.shape[1]),
            "force": (np.abs(o[f0:] - F_ref).max(axis=0) / scale) if len(F_ref) else np.zeros(s.shape[1])}


def gates(sc):
    """Stated gates of the contact path (test_gpu_parity.py): positions / quaternions 1e-4, velocities 2e-3 (5e-3 with several free
    bodies), net forces 5e-2 max(1, |F|); the observed free-body rows hold both positions and velocities."""
    v = 5e-3 if sc.model.nfree >= 2 else 2e-3
    return {"pos": 1e-4, "vel": v, "obs_free": v, "force": 5e-2}


@pytest.mark.parametrize("case,mapping", PARAMS)
def test_lockstep_against_float64_oracle(oracle, monkeypatch, synth_dir, case, mapping):
    K, T = 128, 8
    sc, p, state, root0 = make_case(synth_dir, case, K=K, T=T)
    m = sc.model
    be = backend(monkeypatch, sc, p, mapping, model=m)
    rng = np.random.default_rng(7)
    actions = rng.uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    a_d, root_d = dev(actions), dev(root0)
    pos, _ = _rows(sc)
    gate = gates(sc)
    worst = {k: 0.0 for k in gate}
    excluded = contact_steps = 0
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    f0 = 2 * sc.ndof + 13 * m.nfree
    for t in range(T):
        st = dev(state)
        be.rollout(None, st, a_d, t, 1, obs, root0=root_d)

        def ref(s):
            return oracle.rollout(m, p, None, actions, t, 1, state=s.copy(), root0=root0, use_double=True, nthreads=8)
        s_ref, o_ref = ref(state)
        sens = {k: np.zeros(K) for k in gate}
        for sign in (1.0, -1.0):
            d = np.zeros_like(state)
            d[pos] = sign * PROBE * rng.choice([-1.0, 1.0], (len(pos), K))
            s_p, o_p = ref(state + d)
            e = _errors(sc, s_p, o_p[:, t], s_ref, o_ref[:, t])
            sens = {k: np.maximum(sens[k], e[k]) for k in gate}
        near = np.zeros(K, bool)
        for k in gate:
            near |= sens[k] > gate[k]
        g, o = st.cpu().numpy(), obs[:, t].cpu().numpy()
        assert np.isfinite(g).all() and np.isfinite(o).all()
        err = _errors(sc, g, o, s_ref, o_ref[:, t])
        keep = ~near
        excluded += int(near.sum())
        contact_steps += int((np.abs(o_ref[f0:, t]).max(axis=0) > 0).sum()) if m.ncontact_slots else 0
        for k in gate:
            if keep.any():
                worst[k] = max(worst[k], float(err[k][keep].max()))
        state = s_ref
    report("lockstep", id=f"{case_id(case)}-{mapping}", excluded=excluded, contact_frac=contact_steps / (K * T), **worst)
    assert excluded <= 0.02 * K * T, excluded                                  # discontinuities stay a rare edge case
    assert contact_steps >= 0.5 * K * T, contact_steps                        # the case really is a contact case
    for k in gate:
        assert worst[k] <= gate[k], (k, worst[k])
    # what float32 delivers on an H100 over every case and both mappings: positions 1.5e-5, velocities 2.7e-3 (forest9, two free
    # bodies), forces 5.0e-3 relative; at most 13 of 1 024 rollout-steps excluded
    assert worst["pos"] <= 3e-5 and worst["force"] <= 1e-2, worst


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("ncubes", [2, 3, 4])
def test_colliding_cubes_conserve_momentum_on_device(oracle, monkeypatch, synth_dir, ncubes, mapping):
    """The known answer of test_oracle_contact_synth.py on the device: free cubes without gravity or ground keep their total linear
    momentum and their angular momentum about the origin on every step."""
    sc, p, st, mass, h = cube_collision_scene(synth_dir, 0, ncubes)
    T, K = p.T, p.K
    be = backend(monkeypatch, sc, p, mapping, model=sc.model)
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    be.rollout(None, dev(st), dev(np.zeros((T, sc.nu, K), np.float32)), 0, T, obs, root0=dev(sc.root_state0))
    rows = free_rows(obs.cpu().numpy(), ncubes)
    P0, L0 = _initial_momenta(st, sc.ndof, mass, h)
    P, L = momenta(rows, mass, h)
    dP = float(np.abs(P - P0[None]).max()) / max(1.0, float(np.abs(P0).max()))
    dL = float(np.abs(L - L0[None]).max()) / max(1.0, float(np.abs(L0).max()))
    report("momentum", id=f"cubes{ncubes}-{mapping}", dP_rel=dP, dL_rel=dL)
    assert dP <= 5e-6 and dL <= 5e-6, (dP, dL)                             # float32: measured 1.0e-6 / 1.8e-6 on an H100
    v0 = st[2 * sc.ndof:].reshape(ncubes, 13, K)[:, 7:10]
    assert np.abs(rows[:, 7:10, -1] - v0).max(axis=(0, 1)).min() > 0.1


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("nboxes", [2, 3])
def test_stack_settles_on_device(monkeypatch, synth_dir, nboxes, mapping):
    """The stack of test_oracle_contact_synth.py on the device: each box's net contact force converges to its weight, the stack rests."""
    from synth_scenes import G
    sc, p, st, mass = stack_scene(synth_dir, 0, nboxes)
    T, K = p.T, p.K
    m = sc.model
    be = backend(monkeypatch, sc, p, mapping, model=m)
    obs = torch.zeros((be.obs_size(), T, K), device=DEV)
    be.rollout(None, dev(st), dev(np.zeros((T, sc.nu, K), np.float32)), 0, T, obs, root0=dev(sc.root_state0))
    o = obs.cpu().numpy()
    rows = free_rows(o, nboxes)
    worst_f = worst_v = 0.0
    for f in range(nboxes):
        s = m.free_slot[f]
        force = o[13 * nboxes + 3 * s: 13 * nboxes + 3 * s + 3, -5:]
        worst_f = max(worst_f, float(np.abs(force[2] - mass[f] * G).max() / max(1.0, mass[f] * G)), float(np.abs(force[0:2]).max()))
        worst_v = max(worst_v, float(np.abs(rows[f, 7:13, -1]).max()))
    report("stack", id=f"stack{nboxes}-{mapping}", dF=worst_f, v=worst_v)
    assert worst_f <= 2e-2 and worst_v <= 2e-3, (worst_f, worst_v)


RAGGED = [c for c in CASES if c[:3] in ((3, "chain", 3), (8, "tree", 4), (9, "forest", 2), (13, "tree", 4))]


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("case", RAGGED, ids=[case_id(c) for c in RAGGED])
def test_ragged_k(monkeypatch, synth_dir, case, mapping):
    """K that leaves the last warp partly empty (4 rollouts per warp in the team kernel's contact phase, 32 in the thread kernel):
    every rollout below K is bit-identical to the same rollout of a launch with K rounded up, every output below K is written and
    nothing past K is.  Broadcast state0, per-rollout state, and observe only."""
    rpw = 4 if mapping == "team" else 32
    Ks = [1, 3, 4 * 3 + 1, 4 * 3 + 3] if mapping == "team" else [31, 33]
    K_max = -(-Ks[-1] // rpw) * rpw
    T = 4
    sc, p0, states, root0 = make_case(synth_dir, case, K=K_max, T=T)
    m = sc.model
    nb = sc.ndof
    s0 = states[:2 * nb, 0].copy()
    acts = np.random.default_rng(3).uniform(-0.5, 0.5, (T, sc.nu, K_max)).astype(np.float32)
    root_d = dev(root0)
    checked = 0
    for K in Ks:
        Kup = -(-K // rpw) * rpw
        assert Kup > K
        outs = {}
        for KK in (K, Kup):
            p = copy.copy(p0)
            p.K = KK
            be = backend(monkeypatch, sc, p, mapping, model=m)
            R, NS = be.obs_size(), be.state_size()
            a_d = dev(acts[:, :, :KK])
            res = {}
            for mode in ("state0", "state", "observe"):
                obuf, obs = _guarded(R * T * KK, float("nan"))
                if mode == "state0":
                    sbuf, st = _guarded(NS * KK, float("nan"))
                    be.rollout(dev(s0), st.view(NS, KK), a_d, 0, T, obs.view(R, T, KK), root0=root_d)
                else:
                    sbuf, st = _guarded(NS * KK, 0.0)
                    st.copy_(dev(states[:, :KK]).reshape(-1))
                    n = T if mode == "state" else 0
                    be.rollout(None, st.view(NS, KK), a_d, 0 if n else 2, n, obs.view(R, T, KK), root0=root_d)
                torch.cuda.synchronize()
                assert bool((obuf[-GUARD:] == GUARD_VALUE).all()) and bool((sbuf[-GUARD:] == GUARD_VALUE).all()), (mode, K, KK)
                res[mode] = (obs.view(R, T, KK)[:, :, :K].cpu().numpy(), st.view(NS, KK)[:, :K].cpu().numpy())
            outs[KK] = res
        for mode in ("state0", "state", "observe"):
            (o, s), (o_up, s_up) = outs[K][mode], outs[Kup][mode]
            written = o if mode != "observe" else o[:, 2]
            assert not np.isnan(written).any() and not np.isnan(s).any(), (mode, K)
            if mode == "observe":
                assert np.isnan(np.delete(o, 2, axis=1)).all()
            np.testing.assert_array_equal(o, o_up, err_msg=f"{mode} K={K}")
            np.testing.assert_array_equal(s, s_up, err_msg=f"{mode} K={K}")
            checked += 1
    report("ragged", id=f"{case_id(case)}-{mapping}", Ks=",".join(map(str, Ks)), checked=checked)


SHARD = [c for c in CASES if c[2] >= 2 and c[7]]


@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("case", SHARD, ids=[case_id(c) for c in SHARD])
def test_shard_offset_with_several_randomised_free_actors(monkeypatch, synth_dir, case, mapping):
    """A k_offset shard reproduces its slice of the whole launch bit for bit: the size / mass / friction draws of every free actor are
    keyed by the global sample index."""
    K, T, KS, off = 64, 4, 16, 24
    sc, p, st, root0 = make_case(synth_dir, case, K=K, T=T)
    m = sc.model
    acts = np.random.default_rng(4).uniform(-0.5, 0.5, (T, sc.nu, K)).astype(np.float32)
    be = backend(monkeypatch, sc, p, mapping, model=m)
    obs, s = torch.zeros((be.obs_size(), T, K), device=DEV), dev(st)
    be.rollout(None, s, dev(acts), 0, T, obs, root0=dev(root0))
    ps = copy.copy(p)
    ps.K, ps.k_offset = KS, off
    bs = backend(monkeypatch, sc, ps, mapping, model=m)
    obs_s, s_s = torch.zeros((bs.obs_size(), T, KS), device=DEV), dev(st[:, off:off + KS])
    bs.rollout(None, s_s, dev(acts[:, :, off:off + KS]), 0, T, obs_s, root0=dev(root0))
    assert torch.isfinite(obs).all()
    assert torch.equal(obs_s, obs[:, :, off:off + KS]) and torch.equal(s_s, s[:, off:off + KS])


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_mappings_agree_on_one_step(monkeypatch, synth_dir, case):
    """Team and thread-per-rollout kernels from the same per-rollout state, one model step, no oracle in between: float32 rounding
    apart, except at the rare contact thresholds (at most 2 % of the rollouts)."""
    K, T = 256, 2
    sc, p, st, root0 = make_case(synth_dir, case, K=K, T=T)
    m = sc.model
    acts = dev(np.random.default_rng(5).uniform(-0.5, 0.5, (T, sc.nu, K)))
    out = {}
    for mapping in MAPPINGS:
        be = backend(monkeypatch, sc, p, mapping, model=m)
        s = dev(st)
        obs = torch.zeros((be.obs_size(), T, K), device=DEV)
        be.rollout(None, s, acts, 0, 1, obs, root0=dev(root0))
        out[mapping] = (s.cpu().numpy(), obs[:, 0].cpu().numpy())
    err = _errors(sc, out["team"][0], out["team"][1], out["thread"][0], out["thread"][1])
    gate = gates(sc)
    q98 = {k: float(np.quantile(v, 0.98)) for k, v in err.items()}
    report("cross", id=case_id(case), **{f"{k}_med": float(np.median(v)) for k, v in err.items()}, **{f"{k}_q98": v for k, v in q98.items()})
    for k in gate:
        assert q98[k] <= gate[k], (k, q98[k])
    # measured on an H100 (0.98 quantiles over every case): positions 6.7e-7, velocities 5.1e-5, forces 9.7e-5 relative
    assert q98["pos"] <= 2e-6 and q98["vel"] <= 2e-4 and q98["obs_free"] <= 2e-4 and q98["force"] <= 5e-4, q98
