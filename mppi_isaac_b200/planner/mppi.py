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

from ..backend import shard_row_floats
from ..model.blob import (ANNEAL_MIN_SCALE, ESS_GRID, ESS_ROW_FLOATS, ESS_STATE_FLOATS, MODE_SIMPLE, MODE_SMOOTH, FEATURES, anneal_config,
                          anneal_on, anneal_schedule, constraint_on, ess_grid, ess_on, spline_basis, spline_initial_knots, spline_table)


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


def colored_noise_cov(T: int, beta: float):
    """(T, T) float64 temporal covariance of power-law (1/f^beta) noise, normalised to unit diagonal: the covariance of the
    `powerlaw_psd_gaussian` FFT recipe (iCEM), Sigma[t][t'] = c(|t - t'|) / c(0) with c(tau) = sum_{m=0}^{T//2} a_m s_m^2
    cos(2 pi m tau / T), s_m = max(m, 1)^(-beta/2) (the recipe's fmin = 1/T), a_0 = a_{T/2} (T even) = 1, a_m = 2 otherwise.
    Circulant with eigenvalues proportional to s_m^2 > 0, so positive definite; exactly I at beta = 0."""
    import numpy as np
    if beta == 0.0:
        return np.eye(T)
    m = np.arange(T // 2 + 1)
    a = np.full(m.shape, 2.0)
    a[0] = 1.0
    if T % 2 == 0:
        a[-1] = 1.0
    w = a * np.maximum(m, 1).astype(np.float64) ** (-float(beta))
    ch = w @ np.cos(2.0 * np.pi * np.outer(m, m) / T)               # c(tau), tau = 0 .. T // 2
    lag = np.arange(T)
    c = ch[np.minimum(lag, T - lag)]                                # c(T - tau) = c(tau) exactly: circulant to the bit
    tau = np.abs(lag[:, None] - lag[None, :])
    return c[tau] / c[0]


def colored_noise_chol(T: int, beta: float):
    """(T, T) float32 lower Cholesky factor of ``colored_noise_cov``, computed in float64: the temporal colour of K1's
    ``sampling_method: colored`` (include/mppib.h mppib_sample_colored)."""
    import numpy as np
    return np.linalg.cholesky(colored_noise_cov(T, beta)).astype(np.float32)


def shard_samples(k_total: int, rank: int, world: int, unit: int = 4):
    """Split k_total samples over `world` ranks in units of `unit` samples (128-bit loads need K_local % 4 == 0; risk-aware MPPI
    keeps the n_worlds rollouts of a control sample on one rank with unit = max(4, n_worlds))."""
    if k_total % unit != 0:
        raise ValueError(f"num_samples={k_total} must be a multiple of {unit}")
    units = k_total // unit
    base, rem = divmod(units, world)
    mine = base + (1 if rank < rem else 0)
    off = rank * base + min(rank, rem)
    if mine == 0:
        raise ValueError(f"num_samples={k_total} is too small for {world} ranks")
    return unit * mine, unit * off


def mode_starts(params, nu: int, U0, M: int, seed: int):
    """(M - 1, T, nu) float32 starts of modes 1 .. M-1 of multi-modal MPPI: clamp(U0 + L0 z_m[t], u_min, u_max) with L0 the lower
    Cholesky factor of noise_sigma (the parameter block's float32 copy) and z one (M - 1, T, nu) float64 standard-normal draw of
    numpy.random.default_rng(seed), rounded to float32; the sums in float64, the result rounded once.  Identical modes would stay
    identical under the coupling, so this start breaks the symmetry."""
    import numpy as np
    T = int(params.T)
    z = np.random.default_rng(int(seed)).standard_normal((M - 1, T, nu)).astype(np.float32).astype(np.float64)
    L0 = np.array(params.sigma_chol[:nu * nu], np.float32).astype(np.float64).reshape(nu, nu)
    lo = np.array(params.u_min[:nu], np.float32).astype(np.float64)
    hi = np.array(params.u_max[:nu], np.float32).astype(np.float64)
    U = np.asarray(U0, np.float32).astype(np.float64).reshape(1, T, nu) + np.einsum("ji,mti->mtj", L0, z)
    return np.clip(U, lo, hi).astype(np.float32)


def _randomised(model) -> bool:
    """True when K2 draws something per rollout: a free body's mass, or a shape's friction or size."""
    return (any(model.free_mass_pct[f] != 0.0 for f in range(model.nfree))
            or any(model.shape_fric_pct[s] != 0.0 or any(model.shape_size_sigma[s][i] != 0.0 for i in range(3)) for s in range(model.nshapes)))


class MPPIPlanner:
    def __init__(self, cfg, nx: int, dynamics: Callable, running_cost: Callable, prior: Optional[Callable] = None, *,
                 sim=None, rollout_mode: str = "auto", use_cuda_graph: bool = True, k_total: Optional[int] = None,
                 k_offset: int = 0, process_group=None, seed: Optional[int] = None, running_constraint: Optional[Callable] = None):
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
        if str(cfg.sampling_method) not in ("random", "halton", "colored"):
            raise ValueError(f"unknown sampling_method {cfg.sampling_method}")
        self.use_library = str(cfg.sampling_method) == "halton"     # Halton-spline noise library, drawn once (SURVEY 8(a) M4)
        # power-law noise correlated over the horizon, drawn fresh on every plan (DESIGN.md section 2); make_params checks noise_beta
        self.use_colored = str(cfg.sampling_method) == "colored"
        self.noise_beta = float(getattr(cfg, "noise_beta", 2.0))
        # iCEM (DESIGN.md section 2, "Cross-entropy planning"): the elites of each iteration move the mean U and a per-step sigma,
        # both on the device; make_params checks the keys and refuses the combinations the mode excludes
        self.cem = str(getattr(cfg, "mppi_mode", "")) == "cem"
        self.cem_iterations = int(getattr(cfg, "cem_iterations", 3)) if self.cem else 1
        # annealed MPPI (DESIGN.md section 2, "Annealed MPPI"): N MPPI iterations per plan, the noise of iteration i at step t scaled by
        # s[i][t] = c_i^i c_h^(T-1-t); the schedule is a device buffer K1 / K3 read and K4 / the shift count through.  make_params checks
        # the keys and refuses the combinations the mode excludes; with the defaults nothing is registered and every launch is today's.
        self.annealed = anneal_on(cfg)
        self.anneal_iterations = anneal_config(cfg)[0] if self.annealed else 1
        self.iterations = self.cem_iterations if self.cem else self.anneal_iterations
        # Smooth MPPI (DESIGN.md section 2, "Smooth MPPI"): U is the control derivative; K1 integrates it from the last executed action
        # (the smooth state, a device buffer K4 updates), so the executed command changes by at most du_max * dt per plan
        self.smooth = str(getattr(cfg, "mppi_mode", "")) == "smooth"
        if self.smooth and self.u_per_command > 1:
            raise ValueError("mppi_mode: smooth executes one action per plan (u_per_command = 1): U holds derivatives, not actions")
        # risk-aware MPPI (DESIGN.md section 2, "Risk-aware MPPI"): the K rollouts are K / R control samples, each rolled out in the
        # same R randomised worlds and scored by the CVaR of its R costs; make_params checks the keys against the mode
        self.n_worlds = int(getattr(cfg, "n_worlds", 1))
        self.control_samples = self.K_total // max(1, self.n_worlds)
        if self.n_worlds > 1 and not _randomised(sim.scene.model):
            raise ValueError("n_worlds > 1 needs a scene that randomises its rollouts (noise_percentage_mass, noise_percentage_friction "
                             "or noise_sigma_size on some actor): without it the worlds would be identical copies")
        # multi-modal MPPI (DESIGN.md section 2, "Multi-modal MPPI"): M nominal sequences side by side, each sampled by its block of
        # K_total / M samples and coupled by a Stein-variational step on the device; the mode state (active mode, F[M], U_exec) is a device
        # buffer K4 writes; make_params checks the keys against the mode
        self.n_modes = int(getattr(cfg, "n_modes", 1))
        # adaptive MPPI (DESIGN.md section 2): the live (lambda, cov) pair is a device buffer that K1 / K3 read and K4 updates, so a
        # captured plan graph follows it without re-capture
        self.update_cov = bool(getattr(cfg, "update_cov", False))
        self.update_lambda = bool(getattr(cfg, "update_lambda", False))
        self.adaptive = self.update_cov or self.update_lambda
        # ESS-targeted temperature (DESIGN.md section 2, "ESS-targeted temperature"): every plan chooses lambda on the device so that the
        # Kish ESS of its weights is ess_target of the valid samples; it lives in dist[0] like the adaptive one, so the distribution is
        # registered even with both adaptive flags off; make_params checks the keys against the modes
        self.ess = ess_on(cfg)
        # cov_type chooses the update rule of update_cov: "diag" adapts diag(Sigma), "full" the whole Sigma with its Cholesky factor
        # and inverse (DESIGN.md section 2); make_params rejects other values, full without update_cov and a Sigma that is not SPD
        self.cov_full = self.update_cov and str(getattr(cfg, "cov_type", "diag")) == "full"
        # "horizon" adapts one Sigma_H over the whole control sequence (n = T*nu), started at I_T (x) Sigma
        self.cov_horizon = self.update_cov and str(getattr(cfg, "cov_type", "diag")) == "horizon"
        if self.update_cov and not self.cov_full and not self.cov_horizon:
            import numpy as np
            sigma = np.asarray(cfg.noise_sigma, np.float64).reshape(self.nu, self.nu)
            if np.any(sigma != np.diag(np.diag(sigma))):
                raise ValueError("update_cov adapts a diagonal covariance: noise_sigma must be diagonal")
        # spline MPPI (DESIGN.md section 2, "Spline MPPI"): U is P knots per control of a degree-d B-spline over the horizon; K1 samples
        # the knots and interpolates the actions, K3 / K4 run on the knots; make_params checks the keys against the mode
        self.control_knots = int(getattr(cfg, "control_knots", 0))
        self.spline_degree = int(getattr(cfg, "spline_degree", 1))
        self.backend = sim.backend
        # constrained MPPI (DESIGN.md section 2, "Constrained MPPI"): running_constraint returns a signed margin per row (<= 0 satisfied),
        # written into a (T, K) device buffer K3 reads; make_params checks the keys against the mode
        self.constrained = constraint_on(cfg)
        self._running_constraint = running_constraint
        if self.constrained and running_constraint is None:
            raise ValueError("constraint_mode: feasible_first needs a running_constraint (the Objective's compute_constraint)")
        self._peer_exchange = False
        self._peer_capable = (self.world > 1 and getattr(self.backend, "name", "") == "cuda"
                              and os.environ.get("MPPIB_EXCHANGE", "peer") == "peer")
        if self._peer_capable:
            self.close_peers()                           # a rebuilt planner re-opens windows sized for the new T * nu
        sim.configure(mppi_cfg=cfg, horizon=self.T)      # (re)bakes Sigma / bounds / lambda into the kernel parameter block
        use_prior = bool(getattr(cfg, "use_priors", False)) and prior is not None
        self.use_priors = use_prior
        for f in [f for f in FEATURES if f.on(self.backend.params, cfg)]:    # make_params has refused the modes that exclude each other
            if use_prior and f.no_prior:
                raise ValueError(f"{f.name} does not take a prior: {f.no_prior}")
            if f.setter and not hasattr(self.backend, f.setter):
                raise ValueError(f"{f.name} needs a backend with {f.setter} ({type(self.backend).__name__} has none)")
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
        M = self.n_modes
        Pk, d = self.control_knots, self.spline_degree
        Tc = Pk or T                                         # rows of U: the knots with control_knots > 0, the steps otherwise
        self.U = torch.zeros((Tc, nu), **f32) if M == 1 else torch.zeros((M, T, nu), **f32)
        U0 = self.U if M == 1 else self.U[0]
        U_init = getattr(self.cfg, "U_init", None)
        if U_init is not None and Pk:
            U0.copy_(torch.from_numpy(spline_initial_knots(T, Pk, d, U_init)))
        elif U_init is not None:
            U0.copy_(torch.as_tensor(U_init, dtype=torch.float32).reshape(T, nu))
        else:
            U0 += torch.as_tensor(self.backend.params.u_init[:nu], dtype=torch.float32).to(dev)
        if M > 1:
            self.U[1:].copy_(torch.from_numpy(mode_starts(self.backend.params, nu, U0.cpu().numpy(), M, self.seed)))
        self.actions = torch.zeros((T, nu, K), **f32)       # [T][nu][K]
        self.noise = torch.zeros((T, nu, K), **f32)
        # spline MPPI: the knot samples xk[P][nu][K] K3 weights (theta~ - U in SIMPLE mode, theta~ in MEAN mode) and the table
        # (rows, U_exec) K1 / K4 / the shift read; a planner rebuilt with control_knots = 0 registers none
        self.xk, self.spline_table = None, None
        if Pk:
            self.xk = torch.zeros((Pk, nu, K), **f32)
            self.spline_table = torch.from_numpy(spline_table(T, Pk, d, nu, U0.cpu().numpy())).to(dev)
            self.backend.set_spline(self.spline_table)
        elif hasattr(self.backend, "set_spline"):
            self.backend.set_spline(None)
        self.cost = torch.zeros((T, K), **f32)
        # constrained MPPI: the per-step margins g[T][K] K3 reads and the state (n_feasible as int32 bits, min V) K4 writes; a planner
        # rebuilt with the mode off registers none
        self.viol, self.cstate = None, None
        if self.constrained:
            self.viol = torch.zeros((T, K), **f32)
            self.cstate = torch.zeros((2,), **f32)
            self.backend.set_constraint(self.viol, self.cstate)
        elif hasattr(self.backend, "set_constraint"):
            self.backend.set_constraint(None)
        P = shard_row_floats(self.backend.params, nu)
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
        # (horizon: the same of Sigma_H = I_T (x) Sigma, n = T*nu) computed in float64 and rounded; registered before the noise library is built (update_cov makes it white)
        self.dist = None
        self.mode_state = None
        if self.cem:
            # the CEM state (carry offset, elites valid, S_elite[E], sigma[T][nu], elites[E][T][nu]): sigma starts at sqrt(diag(Sigma))
            E = int(self.backend.params.n_elites)
            sigma0 = torch.sqrt(torch.diagonal(torch.as_tensor(self.cfg.noise_sigma, dtype=torch.float64).reshape(nu, nu)))
            state = torch.zeros((2 + E + T * nu + E * T * nu,), dtype=torch.float64)
            state[2 + E:2 + E + T * nu] = sigma0.repeat(T)
            self.dist = state.to(**f32)
            self.backend.set_distribution(self.dist)
        elif M > 1:
            # the mode state (active mode, F[M], U_exec[T][nu]): mode 0 executed, no free energy yet, U_exec = mode 0
            self.mode_state = torch.cat([torch.zeros(1), torch.full((M,), float("inf")), U0.detach().cpu().reshape(-1)]).to(**f32)
            self.backend.set_distribution(self.mode_state)
        elif not (self.adaptive or self.ess) and hasattr(self.backend, "set_distribution"):
            self.backend.set_distribution(None)          # a planner rebuilt with the flags off must not inherit the previous one's buffer
        if self.adaptive or self.ess:
            sigma = torch.as_tensor(self.cfg.noise_sigma, dtype=torch.float64).reshape(nu, nu)
            if self.cov_horizon:
                sigma = torch.kron(torch.eye(T, dtype=torch.float64), sigma)       # Sigma_H = I_T (x) Sigma
            if self.cov_full or self.cov_horizon:
                chol = torch.linalg.cholesky(sigma)
                parts = [sigma.reshape(-1), chol.reshape(-1), torch.cholesky_inverse(chol).reshape(-1)]
            else:
                parts = [torch.diagonal(sigma)]
            self.dist = torch.cat([torch.tensor([self.lambda_], dtype=torch.float64), *parts]).to(**f32)
            self.backend.set_distribution(self.dist)
        # ESS-targeted temperature: the state (lambda_j, 1/lambda_j, n_valid, lambda, ESS_j) with the grid around lambda_, and the shard rows
        self.temp_state, self.temp_row, self.temp_rows = None, None, None
        if self.ess:
            lam, inv = ess_grid(self.backend.params.lambda_)
            state = torch.zeros((ESS_STATE_FLOATS,), dtype=torch.float32)
            state[:ESS_GRID] = torch.from_numpy(lam)
            state[ESS_GRID:2 * ESS_GRID] = torch.from_numpy(inv)
            state[2 * ESS_GRID + 1] = float(self.dist[0])
            self.temp_state = state.to(dev)
            self.temp_row = torch.zeros((ESS_ROW_FLOATS,), **f32)
            self.temp_rows = torch.zeros((self.world, ESS_ROW_FLOATS), **f32)
            self.backend.set_temperature(self.temp_state)
        elif hasattr(self.backend, "set_temperature"):
            self.backend.set_temperature(None)
        # Smooth MPPI: the state (a_prev[nu], A[T][nu]) starts at a_prev = clamp(0, u_min, u_max), A = a_prev at every step
        self.smooth_state = None
        if self.smooth:
            p = self.backend.params
            a0 = torch.tensor([min(max(0.0, p.u_min[j]), p.u_max[j]) for j in range(nu)], dtype=torch.float32)
            self.smooth_state = a0.repeat(T + 1).to(dev)
            self.backend.set_smooth_state(self.smooth_state)
        elif hasattr(self.backend, "set_smooth_state"):
            self.backend.set_smooth_state(None)          # a rebuilt planner in another mode must not keep the previous one's state
        # annealed MPPI: the schedule (counter, s[N][T], r[N][T]) from float64, each rounded once; a planner rebuilt with the keys at their
        # defaults registers none, as set_distribution(None) above
        self.anneal_state = None
        if self.annealed:
            N, ci, ch = anneal_config(self.cfg)
            s, r = anneal_schedule(N, ci, ch, T)
            self.anneal_state = torch.cat([torch.zeros(1), torch.from_numpy(s.astype("float32")).reshape(-1),
                                           torch.from_numpy(r.astype("float32")).reshape(-1)]).to(**f32)
            self.backend.set_anneal(self.anneal_state, N)
        elif hasattr(self.backend, "set_anneal"):
            self.backend.set_anneal(None)
        self._graph = None
        self._graph_failed = False
        self._graph_epoch = -1
        self._plans = 0
        if self.use_library:
            self._build_library()
        self._noise_Lt = None
        if self.use_colored:                             # the temporal Cholesky factor of the horizon, once per planner
            self._noise_Lt = torch.from_numpy(colored_noise_chol(T, self.noise_beta)).to(dev)
        elif self.cem:                                   # cem with white noise runs the colored K1 with L_b = I
            self._noise_Lt = torch.eye(T, dtype=torch.float32, device=dev)

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

    def refresh_mean_action(self):
        """Spline MPPI: recompute U_exec = B U (float64, rounded once) after U was written from outside a plan (a warm start)."""
        if self.spline_table is not None:
            T, nu = self.T, self.nu
            B, _, _ = spline_basis(T, self.control_knots, self.spline_degree)
            ue = (B @ self.U.detach().cpu().double().numpy()).astype("float32")
            self.mean_action.copy_(torch.from_numpy(ue))

    def _sample(self, iteration=0):
        be = self.backend
        # iteration i of a plan (cem, or annealed MPPI) keys Philox with plan_idx = i << 32: iteration 0 draws what a one-iteration plan draws
        if self.xk is not None:
            be.sample_spline(self.seed, 0, self.k_offset, self.K_total, self.U, self.actions, self.xk, self.plan_ctr)
        elif self.cem:
            be.sample_colored(self.seed, iteration << 32, self.k_offset, self.K_total, self.U, None, self._noise_Lt, self.actions, self.noise,
                              self.plan_ctr)
        elif self.smooth:
            be.sample_smooth(self.seed, 0, self.k_offset, self.K_total, self.U, self.actions, self.noise, self.plan_ctr)
        elif self.use_library:
            be.sample_library(self.k_offset, self.K_total, self.U, None, self.Z, self.actions, self.noise)
        elif self.use_colored:
            be.sample_colored(self.seed, iteration << 32, self.k_offset, self.K_total, self.U, None, self._noise_Lt, self.actions, self.noise,
                              self.plan_ctr)
        else:
            be.sample(self.seed, iteration << 32, self.k_offset, self.K_total, self.U, None, self.actions, self.noise, self.plan_ctr)

    @property
    def noise_schedule(self):
        """(N, T) device view of the noise scales s[i][t] of annealed MPPI (None with the feature off); ``set_noise_schedule`` replaces it."""
        if self.anneal_state is None:
            return None
        n = self.anneal_iterations * self.T
        return self.anneal_state[1:1 + n].view(self.anneal_iterations, self.T)

    def set_noise_schedule(self, s):
        """Annealed MPPI: replace the noise scales by the (N, T) array `s` (each in [2^-20, inf)); s and r = 1 / s^2 are computed in float64
        from the values given and each rounded once, as the planner builds the configured schedule.  Both are written into the registered buffer, so a captured plan graph follows without a re-capture."""
        import numpy as np
        if self.anneal_state is None:
            raise RuntimeError("set_noise_schedule needs annealed MPPI (anneal_iterations > 1 or a decay below 1)")
        s = np.asarray(s.detach().cpu() if isinstance(s, torch.Tensor) else s, np.float64)
        N, T = self.anneal_iterations, self.T
        if s.shape != (N, T):
            raise ValueError(f"set_noise_schedule: s must have shape (anneal_iterations, horizon) = ({N}, {T}), got {s.shape}")
        if not (np.all(np.isfinite(s)) and s.min() >= ANNEAL_MIN_SCALE):
            raise ValueError("set_noise_schedule: every s[i][t] must be finite and at least 2^-20")
        vals = np.concatenate([s.reshape(-1), (1.0 / (s * s)).reshape(-1)]).astype(np.float32)
        self.anneal_state[1:].copy_(torch.from_numpy(vals))

    @property
    def mean_action(self):
        """(T, nu) device view of the nominal sequence U; with mppi_mode smooth that is the mean of the control DERIVATIVE (the
        planned actions are ``action_sequence``); with n_modes > 1 the sequence of the executed mode after the last plan; with
        control_knots > 0 the interpolated sequence U_exec = B U that K4 writes."""
        if self.spline_table is not None:
            return self.spline_table[-self.T * self.nu:].view(self.T, self.nu)
        if self.mode_state is not None:
            return self.mode_state[1 + self.n_modes:].view(self.T, self.nu)
        return self.U

    @property
    def knots(self):
        """(P, nu) device view of the control knots of spline MPPI (U itself; None with control_knots = 0)."""
        return self.U if self.xk is not None else None

    @property
    def knot_samples(self):
        """(P, nu, K) device buffer of the last plan's knot samples of spline MPPI (None with control_knots = 0)."""
        return self.xk

    @property
    def modes(self):
        """(M, T, nu) device view of the nominal sequences of multi-modal MPPI (None unless n_modes > 1)."""
        return self.U if self.n_modes > 1 else None

    @property
    def mode_free_energy(self):
        """(M,) device view of the free energies F_m = beta_m - lambda ln(eta_m / Kc) of the last plan (+inf where a mode had no valid
        sample or before the first plan; None unless n_modes > 1)."""
        return None if self.mode_state is None else self.mode_state[1:1 + self.n_modes]

    @property
    def active_mode(self):
        """Index of the mode the last plan executed (an int, read from the device; None unless n_modes > 1)."""
        return None if self.mode_state is None else int(self.mode_state[0].item())

    @property
    def action_sequence(self):
        """(T, nu) device view of the action sequence A the last smooth plan integrated from ``previous_action`` (None unless
        mppi_mode smooth); its first row is the action that plan returned."""
        return None if self.smooth_state is None else self.smooth_state[self.nu:].view(self.T, self.nu)

    @property
    def previous_action(self):
        """(nu,) device view of the last executed action a_prev that the next smooth plan integrates from (None unless mppi_mode
        smooth).  Every plan sets it to the action it returns."""
        return None if self.smooth_state is None else self.smooth_state[:self.nu]

    def set_previous_action(self, a):
        """mppi_mode smooth: the world executed `a` rather than the planned action (an operator override, a safety stop): the next
        plan integrates from it, so the rate bound holds with respect to what was really executed."""
        if self.smooth_state is None:
            raise RuntimeError("set_previous_action needs mppi_mode: smooth")
        self.smooth_state[:self.nu].copy_(torch.as_tensor(a, dtype=torch.float32).reshape(self.nu))

    @property
    def cov_action(self):
        """(nu,) device view of the diagonal sampling covariance of adaptive MPPI: adapted with update_cov, the constant diag(Sigma)
        with update_lambda alone, None with both flags off; with cov_type full the (nu, nu) view of the adapted Sigma, with
        cov_type horizon the (T*nu, T*nu) view of Sigma_H; with mppi_mode cem the (T, nu) view of the per-step sigma (a standard
        deviation).  ``lambda_`` stays the configured float; the live temperature is ``current_lambda``."""
        if self.dist is None:
            return None
        if self.cem:
            E = int(self.backend.params.n_elites)
            return self.dist[2 + E:2 + E + self.T * self.nu].view(self.T, self.nu)
        if self.cov_horizon:
            n = self.T * self.nu
            return self.dist[1:1 + n * n].view(n, n)
        if self.cov_full:
            return self.dist[1:1 + self.nu * self.nu].view(self.nu, self.nu)
        return self.dist[1:]

    @property
    def current_lambda(self):
        """0-d device view of the live temperature of adaptive MPPI, or the one the last plan chose with lambda_mode ess (None without
        update_cov / update_lambda / lambda_mode ess, and with mppi_mode cem)."""
        return None if self.dist is None or self.cem else self.dist[0]

    @property
    def ess_curve(self):
        """(65,) device view of the Kish ESS of the last plan's weights at each grid temperature, over every rank (None unless lambda_mode
        ess; zeros when no sample was valid)."""
        return None if self.temp_state is None else self.temp_state[2 * ESS_GRID + 2:]

    @property
    def ess_grid(self):
        """(65,) device view of the grid temperatures lambda_j = lambda_ 2^((j - 32)/4) (None unless lambda_mode ess)."""
        return None if self.temp_state is None else self.temp_state[:ESS_GRID]

    @property
    def valid_samples(self):
        """The number of valid samples of the last plan over every rank (an int, read from the device; None unless lambda_mode ess)."""
        return None if self.temp_state is None else int(self.temp_state[2 * ESS_GRID:2 * ESS_GRID + 1].view(torch.int32).item())

    @property
    def elites(self):
        """(E, T, nu) device view of the elites of the last CEM update, best first (None unless mppi_mode cem); ``elite_costs`` holds
        their discounted costs.  Before the first update with E finite samples they are zeros."""
        if not self.cem:
            return None
        E, n = int(self.backend.params.n_elites), self.T * self.nu
        return self.dist[2 + E + n:2 + E + n + E * n].view(E, self.T, self.nu)

    @property
    def elite_costs(self):
        """(E,) device view of the discounted costs S of ``elites`` (None unless mppi_mode cem)."""
        if not self.cem:
            return None
        E = int(self.backend.params.n_elites)
        return self.dist[2:2 + E]

    @property
    def violation(self):
        """(T, K) device view of the last plan's per-step constraint margins g of constrained MPPI, as the Objective returned them (the
        kernels count max(g, 0)); None with constraint_mode none."""
        return self.viol

    @property
    def feasible_samples(self):
        """The number of feasible samples of the last plan over every rank (an int, read from the device; None with constraint_mode
        none)."""
        return None if self.cstate is None else int(self.cstate[0:1].view(torch.int32).item())

    @property
    def min_violation(self):
        """0-d device view of the smallest summed violation V_k of a valid sample in the last plan over every rank (+inf when no sample
        was valid; None with constraint_mode none)."""
        return None if self.cstate is None else self.cstate[1]

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

    def persistent_state(self):
        """{name: device buffer} of the state one plan leaves for the next -- everything the shift or K4 writes and the next plan reads:
        U, the Philox plan counter, the distribution (adaptive, CEM, ESS), the smooth state and the mode state.  The capture restores it
        after its warm-up plans and a keep_U rebuild carries it into the new planner."""
        named = (("U", self.U), ("plan_ctr", self.plan_ctr), ("dist", self.dist), ("smooth_state", self.smooth_state),
                 ("mode_state", self.mode_state))
        return {name: t for name, t in named if t is not None}

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

    def _temperature(self, cost, x):
        """lambda_mode ess: choose this plan's temperature into dist[0] before K3 -- in the pass itself with one rank or the peer window,
        after an all-gather of the shard rows otherwise."""
        be = self.backend
        if self.world == 1 or self._peer_exchange:
            be.temperature(cost, x, self.U, self.temp_row, solve=True)
            return
        be.temperature(cost, x, self.U, self.temp_row, solve=False)
        if torch.distributed.get_backend(self.pg) == "nccl":
            torch.distributed.all_gather_into_tensor(self.temp_rows.view(-1), self.temp_row, group=self.pg)
        else:
            torch.distributed.all_gather([self.temp_rows[g] for g in range(self.world)], self.temp_row, group=self.pg)
        be.temperature_solve(self.temp_rows, self.world)

    def _weighted(self):
        """The samples K3 weights: the knot samples with control_knots > 0, else noise (SIMPLE, smooth) or actions (MEAN)."""
        if self.xk is not None:
            return self.xk
        return self.noise if self.backend.params.mode in (MODE_SIMPLE, MODE_SMOOTH) else self.actions

    def _plan_batched(self):
        be = self.backend
        with _nvtx("mppi/shift"):
            be.shift(self.U, self.plan_ctr)
        for i in range(self.iterations):                 # cem_iterations with mppi_mode cem, anneal_iterations otherwise
            self._iterate_batched(i)

    def _iterate_batched(self, iteration):
        be = self.backend
        with _nvtx("mppi/K1 sample"):
            self._sample(iteration)
        with _nvtx("mppi/K2 rollout"):
            self.sim.rollout_all(self.actions)
        with _nvtx("mppi/objective cost"):
            cost = self._cost_batched()
            if self.viol is not None:
                self.viol.copy_(self._running_constraint(None).reshape(self.T, self.K))
        x = self._weighted()
        if self.ess:
            with _nvtx("mppi/temperature"):
                self._temperature(cost, x)
        with _nvtx("mppi/K3 reduce + exchange + K4 update"):
            if self.world == 1 and hasattr(be, "reduce_finalize"):
                be.reduce_finalize(cost, x, self.U, self.partial, self._action, self.stats)      # K3 + K4 in one launch
                return
            be.reduce(cost, x, self.U, self.partial)
            partials, G = self._exchange()
            be.finalize(partials, G, self.U, self._action, self.stats)

    def _plan_stepwise(self, state):
        self.backend.shift(self.U, self.plan_ctr)
        for i in range(self.iterations):                 # cem_iterations with mppi_mode cem, anneal_iterations otherwise
            state = self._iterate_stepwise(state, i)

    def _iterate_stepwise(self, state, iteration):
        be, sim, T = self.backend, self.sim, self.T
        self._sample(iteration)
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
            if self.viol is not None:
                self.viol[t].copy_(self._running_constraint(state).reshape(-1))
        if self.use_priors and prior_local:
            row = self.K_total - 2 - self.k_offset
            self.noise[:, :, row] = self.actions[:, :, row] - self.U
        x = self._weighted()
        if self.ess:
            self._temperature(self.cost, x)
        be.reduce(self.cost, x, self.U, self.partial)
        partials, G = self._exchange()
        be.finalize(partials, G, self.U, self._action, self.stats)
        return state

    def _try_capture(self):
        dev = torch.device(self.device)
        main = torch.cuda.current_stream(dev)
        # the warm-up plans move the state a plan carries; it is put back whether the capture succeeds or not, so the first plan that
        # follows -- replayed or, after a failed capture, eager -- is the plan an eager planner would run
        keep = {name: t.clone() for name, t in self.persistent_state().items()}
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(main)                           # after the snapshot: the warm-ups must not overwrite what is being copied
        try:
            with torch.cuda.stream(side):
                for _ in range(2):                       # warm-up outside capture (allocator, lazy init)
                    self._plan_batched()
            main.wait_stream(side)
            torch.cuda.synchronize(dev)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._plan_batched()
            self._graph = g
            self._graph_epoch = getattr(self.sim, "model_epoch", 0)
        except Exception as e:  # capture is an optimisation; the eager path is the same kernels
            self._graph = None
            self._graph_failed = True
            print(f"[mppi_isaac_b200] CUDA-graph capture failed ({type(e).__name__}: {e}); running the plan eagerly")
            main.wait_stream(side)
            torch.cuda.synchronize(dev)
        for name, t in self.persistent_state().items():
            t.copy_(keep[name])

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
        return self.mean_action[: self.u_per_command]
