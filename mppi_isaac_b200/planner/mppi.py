"""``MPPIPlanner`` -- host-side mirror of ``mppi_torch.mppi.MPPIPlanner``.

The reference constructs ``MPPIPlanner(cfg.mppi, cfg.nx, dynamics=, running_cost=, prior=)`` and calls
``.command(state)`` (``mppiisaac/planner/mppi_isaac.py:43-49,84,113``); mppi_torch itself
(git dep @75e17e8, ``poetry.lock:1273-1293``) is not vendored, so its behaviour is restated from the
call sites and config keys (SURVEY.md 8(a) rows M1-M6).  Here the class only *sequences* kernels:

    shift U -> K1 sample/clamp -> K2 rollout (+ cost callbacks) -> K3 fused cost/softmax/weighted sum
            -> [all-gather of the (beta, eta, W) shard partials] -> K4 combine + U update (+ savgol)

Two rollout protocols:

* ``batched`` (default when no prior is given): all T steps in one K2 launch, then ONE
  ``running_cost`` call over the (T*K)-row facade views; the whole plan is captured in a CUDA graph.
* ``stepwise``: the reference's protocol -- T x [dynamics(state,u,t); running_cost(state)] -- needed when a
  state-dependent prior overwrites sample row K-2 every step (``mppi_isaac.py:38-41``).

Sample sharding (SURVEY.md 8(e)): rank r of G owns global samples [k_offset, k_offset + K_local); Philox
counters use the global index, so the drawn noise is independent of G.
"""
from __future__ import annotations

from typing import Callable, Optional

import os

import torch

from ..model.blob import MODE_SIMPLE


class _NoRange:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


_NVTX_ON = os.environ.get("MPPIB_NVTX", "0") not in ("", "0")


def _nvtx(name: str):
    """NVTX range around a plan stage (MPPIB_NVTX=1): shows up in an Nsight timeline; off by default (no overhead)."""
    if _NVTX_ON and torch.cuda.is_available():
        return torch.cuda.nvtx.range(name)
    return _NoRange()


def _primes(n: int):
    out, c = [], 2
    while len(out) < n:
        if all(c % q for q in out if q * q <= c):
            out.append(c)
        c += 1
    return out


def halton_table(ndims: int, seed: int):
    """[2][ndims] int32: bases (first primes) and digit multipliers of the scrambled Halton sequence (mult in [1, b-1], seeded).
    ghalton's EA_PERMS table, which mppi_torch uses, is not available offline (SURVEY 8(f) N3): multiplicative scrambling instead."""
    import numpy as np
    bases = np.asarray(_primes(ndims), np.int64)
    rng = np.random.RandomState(int(seed) & 0x7FFFFFFF)
    mult = 1 + rng.randint(0, 1 << 30, size=ndims) % np.maximum(bases - 1, 1)
    return np.stack([bases, mult]).astype(np.int32)


def halton_spline_operator(T: int, n_knots: int):
    """(T, n_knots) float32 matrix of the interpolating degree-2 B-spline (FITPACK splrep s=0 / splev, as mppi_torch's bspline
    helper): the map knots -> horizon points is linear, so it is evaluated once on the host and applied in the kernel."""
    import numpy as np
    from scipy import interpolate as si
    t_arr = np.linspace(0.0, 1.0, n_knots)
    x = np.linspace(0.0, 1.0, T)
    B = np.zeros((T, n_knots))
    for n in range(n_knots):
        e = np.zeros(n_knots); e[n] = 1.0
        B[:, n] = si.splev(x, si.splrep(t_arr, e, k=2, s=0))
    return B.astype(np.float32)


def shard_samples(k_total: int, rank: int, world: int):
    """Split k_total samples over `world` ranks in units of 4 (128-bit loads need K_local % 4 == 0)."""
    if k_total % 4 != 0:
        raise ValueError(f"num_samples={k_total} must be a multiple of 4")
    units = k_total // 4
    base, rem = divmod(units, world)
    mine = base + (1 if rank < rem else 0)
    off = rank * base + min(rank, rem)
    if mine == 0:
        raise ValueError(f"num_samples={k_total} is too small for {world} ranks")
    return 4 * mine, 4 * off


class MPPIPlanner:
    def __init__(self, cfg, nx: int, dynamics: Callable, running_cost: Callable, prior: Optional[Callable] = None, *,
                 sim=None, rollout_mode: str = "auto", use_cuda_graph: bool = True, k_total: Optional[int] = None,
                 k_offset: int = 0, process_group=None, seed: Optional[int] = None):
        if sim is None:
            raise ValueError("MPPIPlanner needs the RolloutSim that owns the kernel handle (sim=...)")
        self.cfg = cfg
        self.nx = nx
        self.sim = sim
        self._dynamics = dynamics
        self._running_cost = running_cost
        self.prior = prior
        self.K = sim.num_envs                     # local samples
        self.K_total = int(k_total) if k_total is not None else self.K
        self.k_offset = int(k_offset)
        self.T = int(cfg.horizon)
        self.nu = sim.scene.nu
        self.lambda_ = float(cfg.lambda_)
        self.u_per_command = int(getattr(cfg, "u_per_command", 1))
        self.seed = int(seed if seed is not None else getattr(cfg, "seed_val", 0))
        self.device = sim.device
        self.pg = process_group
        self.world = 1
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            self.world = torch.distributed.get_world_size(self.pg)
        if str(cfg.sampling_method) not in ("random", "halton"):
            raise ValueError(f"unknown sampling_method {cfg.sampling_method}")
        self.use_library = str(cfg.sampling_method) == "halton"     # Halton-spline noise library, drawn once (SURVEY 8(a) M4)
        # adaptive MPPI (DESIGN.md section 2): the live (lambda, cov) pair is a device buffer that K1 / K3 read and K4 updates, so a
        # captured plan graph follows it without re-capture
        self.update_cov = bool(getattr(cfg, "update_cov", False))
        self.update_lambda = bool(getattr(cfg, "update_lambda", False))
        self.adaptive = self.update_cov or self.update_lambda
        # cov_type chooses the update rule of update_cov: "diag" adapts diag(Sigma), "full" the whole Sigma with its Cholesky factor
        # and inverse (DESIGN.md section 2); make_params rejects other values, full without update_cov and a Sigma that is not SPD
        self.cov_full = self.update_cov and str(getattr(cfg, "cov_type", "diag")) == "full"
        if self.update_cov and not self.cov_full:
            import numpy as np
            sigma = np.asarray(cfg.noise_sigma, np.float64).reshape(self.nu, self.nu)
            if np.any(sigma != np.diag(np.diag(sigma))):
                raise ValueError("update_cov adapts a diagonal covariance: noise_sigma must be diagonal")
        self.backend = sim.backend
        if self.adaptive and not hasattr(self.backend, "set_distribution"):
            raise ValueError(f"update_cov / update_lambda need a backend with set_distribution ({type(self.backend).__name__} has none)")
        self._peer_exchange = False
        self._peer_capable = (self.world > 1 and getattr(self.backend, "name", "") == "cuda"
                              and os.environ.get("MPPIB_EXCHANGE", "peer") == "peer")
        if self._peer_capable:
            self.close_peers()                           # a rebuilt planner re-opens windows sized for the new T * nu
        sim.configure(mppi_cfg=cfg, horizon=self.T)      # (re)bakes Sigma / bounds / lambda into the kernel parameter block
        use_prior = bool(getattr(cfg, "use_priors", False)) and prior is not None
        self.use_priors = use_prior
        if rollout_mode == "auto":
            rollout_mode = "stepwise" if use_prior else "batched"
        if rollout_mode not in ("batched", "stepwise"):
            raise ValueError(rollout_mode)
        self.rollout_mode = rollout_mode
        self.use_cuda_graph = bool(use_cuda_graph) and rollout_mode == "batched" and torch.device(self.device).type == "cuda"
        self._alloc()
        if self._peer_capable:
            self._open_peers()

    # ------------------------------------------------------------------------------------------
    def _open_peers(self):
        """Map every rank's exchange window (include/mppib.h mppib_peer_*): K3 then stores its shard row into all windows
        over NVLink and K4 waits on arrival flags -- the all-gather between them disappears.  Collective; if any rank
        cannot map a peer (no P2P path), every rank falls back to the NCCL all-gather."""
        dist = torch.distributed
        rank = dist.get_rank(self.pg)
        ok, handle = 1, None
        try:
            handle = self.backend.peer_alloc(self.world, rank)
        except RuntimeError as e:
            ok, why = 0, str(e)
        handles = [None] * self.world
        with torch.cuda.device(torch.device(self.device)):     # object collectives stage through the CURRENT device
            dist.all_gather_object(handles, handle, group=self.pg)
        if ok and all(h is not None for h in handles):
            try:
                for g, h in enumerate(handles):
                    if g != rank:
                        self.backend.peer_open(g, h)
            except RuntimeError as e:
                ok, why = 0, str(e)
        else:
            ok, why = 0, "a rank could not allocate its window"
        flag = torch.tensor([ok], dtype=torch.int32, device=self.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.pg)
        self._peer_exchange = bool(int(flag.item()))
        if not self._peer_exchange:
            self.backend.peer_close()
            if rank == 0:
                print(f"[mppi_isaac_b200] peer-memory exchange unavailable ({why if not ok else 'another rank failed'}); using the NCCL all-gather")
        dist.barrier(group=self.pg)

    def close_peers(self):
        """Collective: unmap the exchange windows (call before destroying the process group)."""
        if getattr(self.backend, "name", "") != "cuda" or self.world <= 1:
            return
        if torch.distributed.is_initialized():
            torch.cuda.synchronize(torch.device(self.device))
            torch.distributed.barrier(group=self.pg)     # nobody is still storing into a window that is about to be freed
        self.backend.peer_close()
        self._peer_exchange = False

    def _alloc(self):
        dev, T, nu, K = self.device, self.T, self.nu, self.K
        f32 = dict(dtype=torch.float32, device=dev)
        self.U = torch.zeros((T, nu), **f32)
        U_init = getattr(self.cfg, "U_init", None)
        if U_init is not None:
            self.U.copy_(torch.as_tensor(U_init, dtype=torch.float32).reshape(T, nu))
        else:
            self.U += torch.as_tensor(self.backend.params.u_init[:nu], dtype=torch.float32).to(dev)
        self.actions = torch.zeros((T, nu, K), **f32)       # [T][nu][K]
        self.noise = torch.zeros((T, nu, K), **f32)
        self.cost = torch.zeros((T, K), **f32)
        P = 2 + T * nu * (2 if self.update_cov else 1)      # (beta, eta, W[T*nu]) + M2[T*nu] with update_cov
        if self.cov_full:
            P = 2 + T * nu + nu * (nu + 1) // 2               # (beta, eta, W[T*nu]) + C[lower triangle] with cov_type full
        self.partial = torch.zeros((P,), **f32)
        self.partials = torch.zeros((self.world, P), **f32)
        self._action = torch.zeros((nu,), **f32)
        # host mirror of the action: K4 stores it straight into pinned host memory (include/mppib.h mppib_set_action_mirror), the
        # caller of compute_action* then only waits for the stream -- no device->host copy call
        self._action_host = None
        if torch.device(dev).type == "cuda" and hasattr(self.backend, "set_action_mirror"):
            self._action_host = torch.zeros((nu,), dtype=torch.float32, pin_memory=True)
            self.backend.set_action_mirror(self._action_host)
        self.stats = torch.zeros((2,), **f32)                # (beta, eta)
        self.plan_ctr = torch.zeros((1,), dtype=torch.int32, device=dev)
        self._prior_rows = torch.zeros((T, nu), **f32) if self.use_priors else None
        # adaptive MPPI: dist = (lambda, cov[nu]) from lambda_ and diag(noise_sigma), or with cov_type full (lambda, Sigma, L, Sigma^-1)
        # computed in float64 and rounded; registered before the noise library is built (update_cov makes it white)
        self.dist = None
        if not self.adaptive and hasattr(self.backend, "set_distribution"):
            self.backend.set_distribution(None)          # a planner rebuilt with the flags off must not inherit the previous one's buffer
        if self.adaptive:
            sigma = torch.as_tensor(self.cfg.noise_sigma, dtype=torch.float64).reshape(nu, nu)
            if self.cov_full:
                chol = torch.linalg.cholesky(sigma)
                parts = [sigma.reshape(-1), chol.reshape(-1), torch.cholesky_inverse(chol).reshape(-1)]
            else:
                parts = [torch.diagonal(sigma)]
            self.dist = torch.cat([torch.tensor([self.lambda_], dtype=torch.float64), *parts]).to(**f32)
            self.backend.set_distribution(self.dist)
        self._graph = None
        self._graph_failed = False
        self._graph_epoch = -1
        self._plans = 0
        if self.use_library:
            self._build_library()

    def _build_library(self):
        """Halton-spline perturbations Z[T][nu][K]: scrambled-Halton Gaussian knots (T//4 per control, at least degree+1) interpolated
        by a degree-2 B-spline to the T horizon points and coloured by chol(Sigma); drawn once and reused by every plan."""
        dev, T, nu, K = self.device, self.T, self.nu, self.K
        n_knots = max(T // 4, 3)
        B = halton_spline_operator(T, n_knots)
        tab = halton_table(n_knots * nu, self.seed)
        self.n_knots = n_knots
        self._spline_B = torch.from_numpy(B).to(dev)
        self._halton_tab = torch.from_numpy(tab).to(dev)
        self.Z = torch.zeros((T, nu, K), dtype=torch.float32, device=dev)
        self.backend.noise_library(self.k_offset, self.K_total, self._halton_tab, self._spline_B, n_knots, self.Z)

    def _sample(self):
        be = self.backend
        if self.use_library:
            be.sample_library(self.k_offset, self.K_total, self.U, None, self.Z, self.actions, self.noise)
        else:
            be.sample(self.seed, 0, self.k_offset, self.K_total, self.U, None, self.actions, self.noise, self.plan_ctr)

    @property
    def mean_action(self):
        return self.U

    @property
    def cov_action(self):
        """(nu,) device view of the diagonal sampling covariance of adaptive MPPI: adapted with update_cov, the constant diag(Sigma)
        with update_lambda alone, None with both flags off; with cov_type full the (nu, nu) view of the adapted Sigma.  ``lambda_``
        stays the configured float; the live temperature is ``current_lambda``."""
        if self.dist is None:
            return None
        if self.cov_full:
            return self.dist[1:1 + self.nu * self.nu].view(self.nu, self.nu)
        return self.dist[1:]

    @property
    def current_lambda(self):
        """0-d device view of the live temperature of adaptive MPPI (None without update_cov / update_lambda)."""
        return None if self.dist is None else self.dist[0]

    @property
    def perturbed_action(self):
        """(K, T, nu) view, the layout mppi_torch exposes."""
        return self.actions.permute(2, 0, 1)

    def action_on_host(self):
        """float32 numpy view of the first action of the last plan, after waiting for the plan's stream."""
        if self._action_host is None:
            return self._action.detach().cpu().numpy()
        torch.cuda.current_stream(self._action.device).synchronize()
        return self._action_host.numpy()

    def invalidate_graph(self):
        self._graph = None
        self._graph_failed = False

    # ------------------------------------------------------------------------------------------
    def _cost_batched(self):
        c = self._running_cost(None)
        c = c.reshape(self.T, self.K)
        if c.dtype != torch.float32 or not c.is_contiguous() or c.data_ptr() % 16 != 0:
            self.cost.copy_(c)
            c = self.cost
        return c

    def _exchange(self):
        if self.world == 1:
            return self.partial.view(1, -1), 1
        if self._peer_exchange:
            return None, self.world                      # the rows are already in this rank's window (written by every K3)
        if torch.distributed.get_backend(self.pg) == "nccl":
            torch.distributed.all_gather_into_tensor(self.partials.view(-1), self.partial, group=self.pg)
        else:
            rows = [self.partials[g] for g in range(self.world)]
            torch.distributed.all_gather(rows, self.partial, group=self.pg)
        return self.partials, self.world

    def _plan_batched(self):
        be = self.backend
        with _nvtx("mppi/shift+K1 sample"):
            be.shift(self.U, self.plan_ctr)
            self._sample()
        with _nvtx("mppi/K2 rollout"):
            self.sim.rollout_all(self.actions)
        with _nvtx("mppi/objective cost"):
            cost = self._cost_batched()
        x = self.noise if be.params.mode == MODE_SIMPLE else self.actions
        with _nvtx("mppi/K3 reduce + exchange + K4 update"):
            if self.world == 1 and hasattr(be, "reduce_finalize"):
                be.reduce_finalize(cost, x, self.U, self.partial, self._action, self.stats)      # K3 + K4 in one launch
                return
            be.reduce(cost, x, self.U, self.partial)
            partials, G = self._exchange()
            be.finalize(partials, G, self.U, self._action, self.stats)

    def _plan_stepwise(self, state):
        be, sim, T = self.backend, self.sim, self.T
        be.shift(self.U, self.plan_ctr)
        self._sample()
        sim.begin_step_mode()
        prior_local = self.use_priors and (self.k_offset <= self.K_total - 2 < self.k_offset + self.K)
        for t in range(T):
            u = self.actions[t].t()                                  # (K, nu) view
            if self.use_priors and prior_local:
                row = self.K_total - 2 - self.k_offset
                u[row] = torch.as_tensor(self.prior(state, t), dtype=torch.float32, device=self.device).reshape(-1)
            out = self._dynamics(state, u * be.params.u_scale if be.params.u_scale != 1.0 else u, t)
            if isinstance(out, tuple):
                state, u_out = out
                if u_out is not None and u_out.data_ptr() != u.data_ptr() and be.params.u_scale == 1.0:
                    u.copy_(u_out)                                   # "update action if there were changes"
            c = self._running_cost(state)
            self.cost[t].copy_(c.reshape(-1))
        if self.use_priors and prior_local:
            row = self.K_total - 2 - self.k_offset
            self.noise[:, :, row] = self.actions[:, :, row] - self.U
        x = self.noise if be.params.mode == MODE_SIMPLE else self.actions
        be.reduce(self.cost, x, self.U, self.partial)
        partials, G = self._exchange()
        be.finalize(partials, G, self.U, self._action, self.stats)

    def _try_capture(self):
        dev = torch.device(self.device)
        try:
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            u_keep, ctr_keep = self.U.clone(), self.plan_ctr.clone()
            dist_keep = None if self.dist is None else self.dist.clone()      # the warm-up plans adapt the distribution too
            with torch.cuda.stream(side):
                for _ in range(2):                       # warm-up outside capture (allocator, lazy init)
                    self._plan_batched()
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._plan_batched()
            self.U.copy_(u_keep)
            self.plan_ctr.copy_(ctr_keep)
            if dist_keep is not None:
                self.dist.copy_(dist_keep)
            self._graph = g
            self._graph_epoch = getattr(self.sim, "model_epoch", 0)
        except Exception as e:  # capture is an optimisation; the eager path is the same kernels
            self._graph = None
            self._graph_failed = True
            print(f"[mppi_isaac_b200] CUDA-graph capture failed ({type(e).__name__}: {e}); running the plan eagerly")
            torch.cuda.synchronize(dev)

    # ------------------------------------------------------------------------------------------
    def command(self, state=None):
        """One MPPI plan; returns the first action(s) of the updated control sequence (device tensor)."""
        if self.rollout_mode == "batched":
            # the captured graph bakes in the model block (a by-value kernel parameter: base pose, obstacle poses) and the sim's
            # buffers: any sim-side change of either (setters, set_model, a rebuilt sim) invalidates it
            if self._graph is not None and self._graph_epoch != getattr(self.sim, "model_epoch", 0):
                self.invalidate_graph()
            if self.use_cuda_graph and self._graph is None and not self._graph_failed:
                self._try_capture()
            if self._graph is not None:
                self._graph.replay()
                self.sim.mark_batched()
            else:
                self._plan_batched()
        else:
            self._plan_stepwise(state)
        self._plans += 1
        if self.u_per_command == 1:
            return self._action
        return self.U[: self.u_per_command]
