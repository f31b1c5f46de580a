"""-m gpu: the peer-window exchange of every reduction rule, with several ranks on one GPU (CUDA IPC between processes), against the
explicit-row K4 and the float64 finalize of the rule's oracle.

``peer_window_worker`` runs the ranks (see its docstring for the cases and protocols); the host orders every step, so no K4 waits
for a flag.  After the workers exit, for every exchange of every case:

(a) every rank holds the same K4 outputs (U, action, stats, the distribution / CEM / smooth state), bit for bit;
(b) ``mppib_finalize`` on one handle here, with the saved shard rows stacked at stride P and the saved state before K4, gives the
    peer K4's outputs bit for bit -- a difference is the window path's own (row offset, stride pcap, parity or counter);
(c) the same rows through the float64 finalize of the rule's oracle pass the gates of the in-process G-row tests
    (test_k4_combines_g_shard_rows, test_hz_k4_combines_g_shard_rows, test_cem_k4_against_float64,
    test_smooth_k4_against_the_oracle, test_risk_k4_shard_rows_against_float64).

What a single GPU cannot show is the timing of an overlapped exchange (K4 spinning on another device's K3); the last test runs the
plain cases that way, one rank per device and without the barrier between K3 and K4, where two or more GPUs are visible."""
import os
import pickle
import subprocess
import sys
import time

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import adaptive_full_oracle as afo  # noqa: E402
import adaptive_horizon_oracle as aho  # noqa: E402
import adaptive_oracle as ada  # noqa: E402
import cem_oracle as ce  # noqa: E402
import peer_window_worker as w  # noqa: E402
from synth_mppi import EPS  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OUTS = ("U", "act", "stats", "st")


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV)


def _exclusive_process():
    """The compute mode of the visible devices, read without changing it: several contexts per device need Default."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=compute_mode", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout
    except (OSError, subprocess.SubprocessError):
        return False
    return "Exclusive_Process" in out


def _spawn(tmp_path, world, names, overlap=False, timeout=900):
    """Run `world` ranks of the worker over `names`; the ranks are joined with a timeout and none outlives this call."""
    out = tmp_path / f"world{world}"
    out.mkdir()
    ctx = mp.spawn(w.run, args=(world, str(tmp_path / f"store{world}"), str(out), names, overlap), nprocs=world, join=False)
    deadline = time.monotonic() + timeout
    try:
        while not ctx.join(timeout=max(1.0, deadline - time.monotonic())):
            if time.monotonic() >= deadline:
                raise TimeoutError(f"world {world}: the ranks did not finish within {timeout} s")
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.terminate()
        for p in ctx.processes:
            p.join(10)
            if p.is_alive():
                p.kill()
                p.join()
    res = {}
    for name in names:
        res[name] = []
        for r in range(world):
            with open(out / f"{name}_{r}.pkl", "rb") as f:
                res[name].append(pickle.load(f))
    return res


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def explicit_k4(spec, world, rec, rows):
    """(b): mppib_finalize of the stacked rows on one handle, from the saved state before K4."""
    from mppi_isaac_b200.backend import CudaBackend
    sh = w.Shard(spec, 0, world, rec["phase"])
    be = CudaBackend(DEV)
    be.create(sh.model, sh.params)
    st = None
    if sh.kind is not None:
        st = dev(rec["st0"])
        (be.set_distribution if sh.kind == "dist" else be.set_smooth_state)(st)
    U, act, stats = dev(rec["U0"]), torch.zeros(sh.nu, device=DEV), torch.zeros(2, device=DEV)
    be.finalize(dev(rows), world, U, act, stats)
    got = dict(U=U.cpu().numpy(), act=act.cpu().numpy(), stats=stats.cpu().numpy(), st=None if st is None else st.cpu().numpy())
    be.destroy()
    return got


def oracle_check(spec, world, rec, rows):
    """(c): the float64 finalize of the rule's oracle on the same rows, with the gates of the in-process G-row tests."""
    from oracle import oracle as orc
    sh = w.Shard(spec, 0, world, rec["phase"])
    p, model, nu, T, G = sh.params, sh.model, sh.nu, sh.T, rows.shape[0]
    U0, st0, Ug, stg, sg = rec["U0"], rec["st0"], rec["U"], rec["st"], rec["stats"]
    if sh.rule == "smooth":
        from test_gpu_smooth import k4_check
        k4_check(p, nu, rows, U0, st0, Ug, stg, rec["act"])
        return
    if sh.rule == "cem":
        E, NR = int(p.n_elites), T * nu
        Uw, _, sw, stw = ce.finalize(p, nu, rows, U0, st0)
        acts = rows[:, 2 * E:2 * E + E * NR]
        amax = float(np.abs(acts).max())
        gate_u = (E + 4) * EPS * amax * (4 if p.filter_u else 1) + 2 * EPS * amax
        assert np.abs(Ug - Uw).max() <= gate_u, f"U {np.abs(Ug - Uw).max():.2e} > {gate_u:.2e}"
        sig_g, sig_w = ce.unpack(stg, T, nu, E)[3], ce.unpack(stw, T, nu, E)[3]
        assert np.abs(sig_g - sig_w).max() <= 4 * amax * np.sqrt((E + 4) * EPS)
        np.testing.assert_array_equal(ce.unpack(stg, T, nu, E)[4], ce.unpack(stw, T, nu, E)[4])
        np.testing.assert_array_equal(stg[:2 + E], stw[:2 + E])
        np.testing.assert_array_equal(sg, sw)
        np.testing.assert_array_equal(rec["act"], Ug[0])
        return
    kind = sh.rkind
    if kind == "W" and sh.kind is None:
        U_ref, _, st_ref = orc.finalize(model, p, rows, U0)
        d_ref = None
    else:
        mod = {"W": ada, "M2": ada, "C": afo, "H": aho}[kind]
        U_ref, _, st_ref, d_ref = mod.finalize(model, p, rows, U0, st0)
    if sh.rule == "risk":                                                      # test_risk_k4_shard_rows_against_float64
        ok = rows[:, 1] > 0
        b = rows[ok, 0].min()
        s = np.exp(-(rows[ok, 0].astype(np.float64) - b) / float(st0[0] if st0 is not None else p.lambda_))
        comb = (s[:, None] * rows[ok].astype(np.float64)).sum(0)
        gate_u = 32 * EPS * (np.abs(U0).max() + np.abs(comb[2:2 + T * nu] / comb[1]).max()) * G
    else:                                                                      # test_k4_combines_g_shard_rows / test_hz_k4_...
        gate_u = 4e-6 * max(1.0, np.abs(U_ref).max())
    err = float(np.abs(Ug - U_ref).max())
    assert err <= gate_u, f"U {err:.2e} > {gate_u:.2e}"
    assert sg[0] == st_ref[0]
    if d_ref is not None:
        if p.update_lambda:
            assert stg[0] == d_ref[0], f"lambda {stg[0]} != {d_ref[0]}"
        if p.update_cov:
            np.testing.assert_allclose(stg[1:], d_ref[1:], rtol=0, atol=2e-5 * np.abs(d_ref[1:]).max())
        else:
            np.testing.assert_array_equal(stg[1:], np.asarray(st0)[1:])


def check_case(spec, world, outs):
    """(a), (b) and (c) on every exchange of a case; the graph replays equal the eager exchanges; returns the failures."""
    fails = []
    name = spec["name"]
    for key in ("ex", "graph"):
        if key not in outs[0]:
            continue
        for j in range(len(outs[0][key])):
            recs = [o[key][j] for o in outs]
            tag = f"{name} world {world} {key}[{j}]"
            for r in range(1, world):
                for k in OUTS + ("U0", "st0"):
                    if not _same(recs[r][k], recs[0][k]):
                        fails.append(f"{tag}: (a) rank {r} {k} differs from rank 0")
            rows = np.stack([rc["row"] for rc in recs])
            got = explicit_k4(spec, world, recs[0], rows)
            for k in OUTS:
                if not _same(got[k], recs[0][k]):
                    fails.append(f"{tag}: (b) the explicit-row K4 differs in {k}")
            try:
                oracle_check(spec, world, recs[0], rows)
            except Exception as e:                                             # noqa: BLE001 -- a wrong state can break the reference too
                fails.append(f"{tag}: (c) {type(e).__name__}: {(str(e).strip().splitlines() or [''])[0]}")
    if "graph" in outs[0]:
        for r, o in enumerate(outs):
            for j, (g, e) in enumerate(zip(o["graph"], o["ex"])):
                for k in OUTS + ("row", "U0", "st0"):
                    if not _same(g[k], e[k]):
                        fails.append(f"{name} world {world} rank {r}: graph replay {j} differs from the eager exchange in {k}")
    if "single" in outs[0]:
        for r, o in enumerate(outs):
            for k in ("row", "U", "act", "stats"):
                if not _same(o["single"][k], o["fresh"][k]):
                    fails.append(f"{name} world {world} rank {r}: after peer_close the fused K3 + K4 differs in {k} from a handle without a window")
    return fails


@pytest.fixture(scope="module", autouse=True)
def _contexts():
    if _exclusive_process():
        pytest.skip("compute mode Exclusive_Process: one context per device, the ranks cannot share a GPU")


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("world", [2, 3, 8, 16])
def test_peer_window_exchange(tmp_path, world):
    names = w.cases(world)
    t0 = time.monotonic()
    res = _spawn(tmp_path, world, names)
    fails = []
    for name in names:
        fails += check_case(w.SPECS[name], world, res[name])
    nex = sum(len(res[n][0]["ex"]) + len(res[n][0].get("graph", [])) for n in names)
    print(f"PEER world {world}: {len(names)} cases, {nex} exchanges per rank, {time.monotonic() - t0:.1f} s")
    assert not fails, "\n".join(fails)


@pytest.mark.timeout(1800)
def test_overlapped_exchange_on_several_gpus(tmp_path):
    """One rank per device, K4 launched right after K3 (no host barrier between them): the real overlapped exchange."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip(f"{n} GPU visible: the overlapped exchange needs one rank per device on two or more")
    world = min(n, 16)
    names = w.plain_cases()
    res = _spawn(tmp_path, world, names, overlap=True)
    fails = []
    for name in names:
        fails += check_case(w.SPECS[name], world, res[name])
    assert not fails, "\n".join(fails)
