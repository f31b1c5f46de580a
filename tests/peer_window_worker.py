"""One rank of the peer-window exchange test (test_gpu_peer_window.py).

Every rank owns a handle for its shard (K samples at k_offset = rank * K) and a peer window; the ranks exchange their shard rows
through the windows (K3 stores its row into every rank's window and release-stores one flag per rank, K4 with partials = NULL
acquires its flags and reads the rows back at the window's stride pcap).  Several processes on one device can do this through CUDA
IPC, and the host orders every step: all ranks finish K3 and meet at a barrier before any rank launches K4, so no K4 ever waits for
a flag of a context that has not run yet.  With ``overlap`` (one rank per device) the barrier between K3 and K4 is left out.

The cases (``SPECS``) cover every row kind ``partial_row_capacity`` distinguishes, at (T, nu) where the row length P takes every
residue mod 4 and the stride pcap exceeds P; ``setup`` / ``inputs`` build a rank's handle and its seeded shard inputs, and the
parent rebuilds the same parameter blocks to check the saved rows.  A case's protocol (``proto``):

* ``plain``  -- ``n`` exchanges (CEM: plans of three iterations, each plan opened by the shift);
* ``ahead``  -- rank 0 runs K4 #1 and K3 #2 before the other ranks run K4 #1, which must still read exchange 1's rows;
* ``graph``  -- the exchanges eagerly, then again from the same state through a captured K3 graph and a captured K4 graph;
* ``shrink`` -- set_params shrinks the row with the windows open (drop update_cov, then a shorter T); a block that would outgrow
  the window is refused;
* ``reopen`` -- peer_close, the single-GPU fused K3 + K4 against a handle that never had a window, a fresh window, one exchange;
* ``refuse`` -- the host refusals of the exchange API, then exchanges on the same windows.

Each rank pickles ``{"ex": [record per exchange], ...}`` to ``<out>/<case>_<rank>.pkl``; a record holds the shard row, the state
before K4 (U and the registered distribution / CEM / smooth state) and every K4 output.
"""
import copy
import os
import pickle
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (HERE, os.path.dirname(HERE)):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def _c(name, rule, T, nu, proto="plain", n=3, K=1024, **kw):
    return dict(name=name, rule=rule, T=T, nu=nu, proto=proto, n=n, K=K, **kw)


MEAN = "halton-spline"
# (P, P mod 4, pcap) in the comments; P = the row K3 writes, pcap = partial_row_capacity rounded up to 4
SPECS = {s["name"]: s for s in [
    _c("W-simple-T16nu9", "W", 16, 9),                                       # 146, 2, 148
    _c("W-mean-filter-T13nu3", "W", 13, 3, mode=MEAN, filter_u=True),        # 41, 1, 44
    _c("W-simple-T10nu1", "W", 10, 1),                                       # 12, 0, 12
    _c("W-simple-T7nu3", "W", 7, 3),                                         # 23, 3, 24
    _c("lambda-mean-T11nu3", "lambda", 11, 3, mode=MEAN),                    # update_lambda alone: 35, 3, 36
    _c("M2-simple-T12nu5", "M2", 12, 5),                                     # 122, 2, 124
    _c("M2-mean-T7nu1", "M2", 7, 1, mode=MEAN),                              # 16, 0, 16
    _c("C-mean-T9nu5", "C", 9, 5, mode=MEAN),                                # 62, 2, 64
    _c("C-simple-T5nu3", "C", 5, 3),                                         # 23, 3, 24
    _c("H-simple-T16nu4", "H", 16, 4),                                       # n 64: 2146, 2, 2148
    _c("H-mean-T64nu4", "H", 64, 4, mode=MEAN),                              # n 256, the largest SYRK row: 33154, 2, 33156
    _c("H-simple-T9nu1", "H", 9, 1),                                         # n 9: 56, 0, 56
    _c("risk-fixed-R2-simple-T8nu3", "risk", 8, 3, kind="fixed", R=2, m=1),  # 26, 2, 28
    _c("risk-diag-R8-mean-T8nu3", "risk", 8, 3, kind="diag", R=8, m=4, mode=MEAN),    # 50, 2, 52
    _c("risk-full-R32-simple-T8nu3", "risk", 8, 3, kind="full", R=32, m=8),            # 32, 0, 32
    _c("risk-full-R8-mean-T5nu2", "risk", 5, 2, kind="full", R=8, m=3, mode=MEAN),     # 15, 3, 16
    _c("risk-diag-R32-simple-T9nu1", "risk", 9, 1, kind="diag", R=32, m=16),            # 20, 0, 20
    _c("risk-fixed-R8-mean-T9nu1", "risk", 9, 1, kind="fixed", R=8, m=8, mode=MEAN),   # 11, 3, 12
    _c("smooth-w0-T9nu7", "smooth", 9, 7, omega=0.0),                       # 65, 1, 68
    _c("smooth-w0.5-T30nu2", "smooth", 30, 2, omega=0.5),                   # 62, 2, 64
    _c("cem-E1-T9nu7", "cem", 9, 7, E=1, n=6),                              # 68
    _c("cem-E10-T12nu5-filter", "cem", 12, 5, E=10, n=6, filter_u=True),    # 620
    _c("cem-E128-T256nu2", "cem", 256, 2, E=128, n=6),                      # T*nu = 512: 65792
    _c("ahead-M2-simple-T12nu5", "M2", 12, 5, proto="ahead"),
    _c("ahead-cem-E10-T12nu5", "cem", 12, 5, E=10, proto="ahead", n=3),
    _c("graph-W-mean-filter-T13nu3", "W", 13, 3, mode=MEAN, filter_u=True, proto="graph"),
    _c("graph-H-simple-T16nu4", "H", 16, 4, proto="graph"),
    _c("graph-cem-E10-T12nu5", "cem", 12, 5, E=10, proto="graph", n=3),
    _c("shrink-M2-simple-T12nu5", "M2", 12, 5, proto="shrink", n=5),
    _c("reopen-W-simple-T16nu9", "W", 16, 9, proto="reopen", n=4),
    _c("refuse-W-simple-T7nu3", "W", 7, 3, proto="refuse", n=2),
]}
# world 8: one case per rule; world 16 (MPPIB_MAX_PEERS): one SIMPLE case
WORLD8 = ["W-simple-T16nu9", "lambda-mean-T11nu3", "M2-simple-T12nu5", "C-mean-T9nu5", "H-simple-T16nu4", "risk-diag-R8-mean-T8nu3",
          "smooth-w0.5-T30nu2", "cem-E10-T12nu5-filter"]
WORLD16 = ["W-simple-T7nu3"]
# the shrink case's phases: the row without update_cov (M2 dropped, the registered (lambda, cov) kept), then at T = 6
SHRINK = [{}, {"no_cov": True}, {"no_cov": True, "T": 6}, {"no_cov": True, "T": 6}, {"no_cov": True, "T": 6}]


def cases(world):
    if world >= 16:
        return list(WORLD16)
    if world >= 8:
        return list(WORLD8)
    return list(SPECS)


def plain_cases():
    return [k for k, s in SPECS.items() if s["proto"] == "plain"]


# -------------------------------------------------------------------------------------------------------------------- cases
class Shard:
    """model, params, the registered state's kind ("dist", "smooth" or None) and its initial value, the synth_mppi case."""

    def __init__(self, spec, rank, world, phase=None):
        from test_gpu_mode_shapes import RISK_KINDS, cem_params, risk_case, smooth_params
        import cem_oracle as ce
        import smooth_oracle as so
        from synth_mppi import make_case, nu_model
        s = dict(spec, **(phase or {}))
        rule, T, nu, K, mode = s["rule"], s["T"], s["nu"], s["K"], s.get("mode", "simple")
        self.spec, self.rule, self.T, self.nu, self.K, self.rank, self.world = s, rule, T, nu, K, rank, world
        self.case, self.kind, self.state = None, None, None
        self.model = nu_model(nu)
        if rule == "smooth":
            self.params = smooth_params(nu, T, K, k_offset=rank * K, smooth_weight=s["omega"], du_min=[-0.3], du_max=[0.3], u_min=[-0.03],
                                        u_max=[0.03])
            self.kind = "smooth"
            self.state = so.make_state(self.params, nu, np.random.default_rng(T + nu).uniform(-0.02, 0.02, nu))
        elif rule == "cem":
            self.params = cem_params(nu, T, K, s["E"], keep=1, alpha=0.3, k_offset=rank * K, k_total=world * K, filter_u=bool(s.get("filter_u")))
            self.kind, self.state = "dist", ce.make_state(np.full(nu, 0.04), T, nu, s["E"])
        else:
            if rule == "risk":
                self.case = risk_case(T, nu, K, s["kind"], s["R"], s["m"], mode)
                self.rkind = RISK_KINDS[s["kind"]]
            else:
                self.case = make_case(T, nu, K, mode=mode, kind="W" if rule in ("W", "lambda") else rule, filter_u=bool(s.get("filter_u")),
                                      update_lambda=rule in ("lambda", "H"))
                self.rkind = "W" if rule in ("W", "lambda") else rule
                if rule == "lambda":                                          # update_lambda alone: (lambda, cov[nu]), row W
                    self.case.dist = np.concatenate([[self.case.lam], np.diag(self.case.sigma)]).astype(np.float32)
            self.params = copy.copy(self.case.params)
            self.params.k_offset = rank * K
            if s.get("no_cov"):
                self.params.update_cov = 0
            if self.case.dist is not None:
                self.kind, self.state = "dist", self.case.dist.copy()

    def inputs(self, j):
        """(cost [T][K], x [T][nu][K], U [T][nu]) of exchange j on this rank: U depends on j alone (every rank holds the same U), the
        samples on (j, rank); each shard has its own beta, a few costs are +inf or NaN, and at j = 1 the last rank's shard has no valid
        sample."""
        T, nu, K, r = self.T, self.nu, self.K, self.rank
        rng = np.random.default_rng(1000 * j + r + 1)
        Ur = np.random.default_rng(1000 * j + 77)
        if self.rule == "cem":
            cost = rng.uniform(0, 1, (T, K)).astype(np.float32)
            x = rng.uniform(-0.2, 0.2, (T, nu, K)).astype(np.float32)
            U = Ur.uniform(-0.1, 0.1, (T, nu)).astype(np.float32)
            lam = 1.0
        elif self.rule == "smooth":
            cost = rng.uniform(0.0, 0.05, (T, K)).astype(np.float32)
            x = rng.normal(0.0, 0.4, (T, nu, K)).astype(np.float32)
            U = Ur.uniform(-0.3, 0.3, (T, nu)).astype(np.float32)
            lam = float(self.params.lambda_)
        else:
            from synth_mppi import k3_inputs
            case = copy.copy(self.case)
            case.kind = self.rkind
            cost, x, _ = k3_inputs(case, seed=1000 * j + r + 1, favour_tail=False)
            U = k3_inputs(case, seed=1000 * j + 77, favour_tail=False)[2]
            lam = case.lam
        cost[0] += np.float32(0.7 * r * lam)                                    # a different beta per shard
        R = int(self.spec.get("R", 1))
        bad = rng.choice(K // R - 1, 2, replace=False) * R
        cost[rng.integers(T), bad[0]] = np.inf                                 # one rollout of one sample / group
        cost[0, bad[1]:bad[1] + R] = np.nan if self.rule == "cem" else np.inf   # a whole group
        if j == 1 and r == self.world - 1:
            cost[:] = np.nan                                                    # no valid sample in this shard
        return np.ascontiguousarray(cost), np.ascontiguousarray(x), np.ascontiguousarray(U)


# -------------------------------------------------------------------------------------------------------------------- a rank
class Rank:
    def __init__(self, spec, rank, world, device, overlap):
        import torch
        from mppi_isaac_b200.backend import CudaBackend
        self.torch, self.spec, self.rank, self.world, self.dev, self.overlap = torch, spec, rank, world, device, overlap
        self.sh = Shard(spec, rank, world)
        self.be = CudaBackend(device)
        self.be.create(self.sh.model, self.sh.params)
        self.st = None
        if self.sh.kind is not None:
            self.st = torch.as_tensor(self.sh.state).to(device)
            (self.be.set_distribution if self.sh.kind == "dist" else self.be.set_smooth_state)(self.st)
        self._buffers()
        self.U.copy_(self._t(self.sh.inputs(0)[2]))
        self.phase = {}
        self.rec = []

    def _t(self, a):
        return self.torch.as_tensor(np.ascontiguousarray(a)).to(self.dev)

    def _buffers(self):
        torch, sh = self.torch, self.sh
        self.U = torch.zeros((sh.T, sh.nu), device=self.dev)
        self.partial = torch.zeros(self.be.partial_row_floats(), device=self.dev)
        self.act, self.stats = torch.zeros(sh.nu, device=self.dev), torch.zeros(2, device=self.dev)

    def barrier(self):
        self.torch.distributed.barrier()

    def sync(self):
        self.torch.cuda.synchronize(self.dev)

    def open(self):
        import torch.distributed as dist
        h = self.be.peer_alloc(self.world, self.rank)
        hs = [None] * self.world
        dist.all_gather_object(hs, h)
        self.handles = hs
        for g in range(self.world):
            if g != self.rank:
                self.be.peer_open(g, hs[g])
        self.barrier()

    def close(self):
        self.sync()
        self.barrier()
        self.be.peer_close()
        self.barrier()

    def host(self, a):
        return a.detach().cpu().numpy().copy()

    def k3(self, j, cost=None, x=None):
        """K3 of exchange j (CEM: a plan of three iterations opens with the shift)."""
        if self.sh.rule == "cem" and j % 3 == 0:
            self.U.copy_(self._t(self.sh.inputs(j)[2]))
            self.be.shift(self.U)
        c, xx, _ = self.sh.inputs(j)
        self.be.reduce(self._t(c) if cost is None else cost, self._t(xx) if x is None else x, self.U, self.partial)

    def pre(self):
        return {"U0": self.host(self.U), "st0": None if self.st is None else self.host(self.st), "phase": dict(self.phase)}

    def k4(self, pre, fn=None):
        (fn or (lambda: self.be.finalize(None, self.world, self.U, self.act, self.stats)))()
        self.sync()
        r = dict(pre, row=self.host(self.partial), U=self.host(self.U), act=self.host(self.act), stats=self.host(self.stats),
                 st=None if self.st is None else self.host(self.st))
        return r

    def exchange(self, j):
        self.k3(j)
        self.sync()
        if not self.overlap:
            self.barrier()
        r = self.k4(self.pre())
        self.barrier()
        return r

    def set_phase(self, phase):
        """set_params with the windows open: the new row must fit the window (the shrink case)."""
        self.phase = phase
        self.sh = Shard(self.spec, self.rank, self.world, phase)
        self.be.set_params(self.sh.params)
        U = self.host(self.U)
        self._buffers()
        if U.shape == tuple(self.U.shape):
            self.U.copy_(self._t(U))
        else:
            self.U.copy_(self._t(self.sh.inputs(0)[2]))


def _refused(fn, what):
    try:
        fn()
    except RuntimeError as e:
        assert what in str(e), f"refused for another reason: {e}"
        return str(e)
    raise AssertionError(f"not refused: {what}")


def _plain(R, out):
    R.open()
    out["ex"] = [R.exchange(j) for j in range(R.spec["n"])]
    R.close()


def _ahead(R, out):
    """Rank 0 one exchange ahead of the others; host barriers between the steps, so that no K4 waits."""
    R.open()
    lead = R.rank == 0
    R.k3(0)
    R.sync()
    R.barrier()
    ex = [None, None]
    if lead:
        ex[0] = R.k4(R.pre())
    R.barrier()
    if lead:
        R.k3(1)                                        # writes exchange 2's rows into every window, parity 0
        R.sync()
    R.barrier()
    if not lead:
        ex[0] = R.k4(R.pre())                          # must still read exchange 1's rows, parity 1
    R.barrier()
    if not lead:
        R.k3(1)
        R.sync()
    R.barrier()
    ex[1] = R.k4(R.pre())
    R.barrier()
    out["ex"] = ex + [R.exchange(j) for j in range(2, R.spec["n"])]
    R.close()


def _graph(R, out):
    """Eager exchanges, then the same ones from the same state through a K3 graph and a K4 graph (the window's exchange number and
    parity are read at run time: the replays run at exchanges n + 1 .. 2n)."""
    torch = R.torch
    U0, st0 = R.host(R.U), None if R.st is None else R.host(R.st)
    R.open()
    out["ex"] = [R.exchange(j) for j in range(R.spec["n"])]
    R.U.copy_(R._t(U0))
    if R.st is not None:
        R.st.copy_(R._t(st0))
    c, x, _ = R.sh.inputs(0)
    cb, xb = R._t(c), R._t(x)
    R.sync()
    s = torch.cuda.Stream(R.dev)
    g3, g4 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g3, stream=s):
        R.be.reduce(cb, xb, R.U, R.partial)
    with torch.cuda.graph(g4, stream=s):
        R.be.finalize(None, R.world, R.U, R.act, R.stats)
    R.sync()
    R.barrier()
    gex = []
    for j in range(R.spec["n"]):
        if R.sh.rule == "cem" and j % 3 == 0:
            R.U.copy_(R._t(R.sh.inputs(j)[2]))
            R.be.shift(R.U)
        c, x, _ = R.sh.inputs(j)
        cb.copy_(R._t(c))
        xb.copy_(R._t(x))
        R.sync()
        g3.replay()
        R.sync()
        R.barrier()
        gex.append(R.k4(R.pre(), g4.replay))
        R.barrier()
    out["graph"] = gex
    del g3, g4
    R.close()


def _shrink(R, out):
    R.open()
    ex = []
    for j, phase in enumerate(SHRINK[:R.spec["n"]]):
        if phase != R.phase:
            R.set_phase(phase)
        if j == 3:                                    # a block that outgrows the window is refused and leaves the handle as it was
            big = Shard(R.spec, R.rank, R.world, {"T": 14})
            before = R.be.params
            out["refused"] = [_refused(lambda: R.be.set_params(big.params), "outgrows the open peer window")]
            assert R.be.params is before
        ex.append(R.exchange(j))
    out["ex"] = ex
    R.close()


def _reopen(R, out):
    from mppi_isaac_b200.backend import CudaBackend
    R.open()
    ex = [R.exchange(j) for j in range(2)]
    R.close()
    # closed: the single-GPU fused tail again, equal to a handle that never had a window
    c, x, _ = R.sh.inputs(2)
    pre = R.pre()
    fresh = CudaBackend(R.dev)
    fresh.create(R.sh.model, R.sh.params)
    Uf, pf, af, sf = R._t(pre["U0"]), R.torch.zeros_like(R.partial), R.torch.zeros_like(R.act), R.torch.zeros_like(R.stats)
    fresh.reduce_finalize(R._t(c), R._t(x), Uf, pf, af, sf)
    R.sync()
    out["single"] = R.k4(pre, lambda: R.be.reduce_finalize(R._t(c), R._t(x), R.U, R.partial, R.act, R.stats))
    out["fresh"] = dict(row=R.host(pf), U=R.host(Uf), act=R.host(af), stats=R.host(sf))
    R.U.copy_(R._t(pre["U0"]))                         # that U moved by this rank's shard alone: every rank starts again from the same U
    # a fresh window starts its exchange counter over
    R.open()
    ex += [R.exchange(j) for j in range(3, R.spec["n"])]
    out["ex"] = ex
    R.close()


def _refuse(R, out):
    from synth_mppi import nu_model
    R.open()
    be, w, r = R.be, R.world, R.rank
    other = (r + 1) % w
    msgs = [
        _refused(lambda: be.finalize(None, w + 1, R.U, R.act, R.stats), "G == world"),
        _refused(lambda: be.finalize(None, w - 1, R.U, R.act, R.stats), "G == world"),
        _refused(lambda: be.reduce_finalize(*[R._t(a) for a in R.sh.inputs(0)[:2]], R.U, R.partial, R.act, R.stats), "open peer window"),
        _refused(lambda: be.peer_open(r, R.handles[r]), "out of range"),
        _refused(lambda: be.peer_open(w, R.handles[other]), "out of range"),
        _refused(lambda: be.peer_open(-1, R.handles[other]), "out of range"),
        _refused(lambda: be.peer_open(other, R.handles[other]), "already open"),
        _refused(lambda: be.peer_alloc(1, 0), "out of range"),
        _refused(lambda: be.peer_alloc(17, 0), "out of range"),
        _refused(lambda: be.set_model(nu_model(R.sh.nu + 1)), "outgrows the open peer window"),
    ]
    assert be.model.nu == R.sh.nu
    out["refused"] = msgs
    R.barrier()
    out["ex"] = [R.exchange(j) for j in range(R.spec["n"])]    # the windows are intact
    R.close()


PROTOS = {"plain": _plain, "ahead": _ahead, "graph": _graph, "shrink": _shrink, "reopen": _reopen, "refuse": _refuse}


def run(rank, world, store, out_dir, names, overlap):
    os.environ["MPPIB_PEER_TIMEOUT_S"] = "10"
    import torch
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="file://" + store, rank=rank, world_size=world)
    device = f"cuda:{rank % torch.cuda.device_count()}"
    torch.cuda.set_device(device)
    for name in names:
        spec = SPECS[name]
        R = Rank(spec, rank, world, device, overlap)
        out = {}
        PROTOS[spec["proto"]](R, out)
        R.be.destroy()
        with open(os.path.join(out_dir, f"{name}_{rank}.pkl"), "wb") as f:
            pickle.dump(out, f)
        dist.barrier()
    dist.destroy_process_group()
