"""ctypes binding of ``libmppib.so`` (the C ABI in ``include/mppib.h``).

This is the only compute backend the package ships.  There is NO CPU fallback: if the CUDA
library is missing or no sm_90a device is visible, construction fails loudly.  Device
memory, streams and ``torch.distributed`` come from PyTorch (plumbing); every kernel on the
hot path is ours.  Tensors are passed as raw ``data_ptr()``s, the stream as
``torch.cuda.current_stream().cuda_stream`` -- no torch types cross the ABI.
"""
from __future__ import annotations

import ctypes as C
import os
import weakref

import torch

from .model.blob import ABI_VERSION, ESS_ROW_FLOATS, ESS_STATE_FLOATS, MODE_CEM, MODE_SIMPLE, MODE_SMOOTH, MppibModel, MppibParams

_LIB_PATH = os.environ.get("MPPIB_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "libmppib.so")   # MPPIB_LIB: tuning builds
_lib = None

SYMBOLS = [
    "mppib_abi_version", "mppib_last_error", "mppib_create", "mppib_destroy", "mppib_set_params",
    "mppib_set_model", "mppib_state_size", "mppib_obs_size", "mppib_sample", "mppib_rollout",
    "mppib_reduce", "mppib_finalize", "mppib_shift", "mppib_noise_library", "mppib_sample_library",
    "mppib_peer_alloc", "mppib_peer_open", "mppib_peer_close", "mppib_cost_pose", "mppib_set_action_mirror", "mppib_reduce_finalize", "mppib_rollout_smem_bytes", "mppib_rollout_mapping", "mppib_rollout_mapping_for_model",
    "mppib_set_distribution", "mppib_sample_colored", "mppib_set_smooth_state", "mppib_sample_smooth", "mppib_set_anneal",
    "mppib_set_spline", "mppib_sample_spline", "mppib_set_constraint", "mppib_set_temperature", "mppib_temperature", "mppib_temperature_solve",
]


def lib_path() -> str:
    return _LIB_PATH


def load_library():
    """dlopen libmppib.so; raises if it was not built (``python -c 'import __graft_entry__ as g; g.build()'``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(
            f"{_LIB_PATH} not found: the CUDA extension is not built. Run `python __graft_entry__.py` "
            "(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU fallback.")
    lib = C.CDLL(_LIB_PATH)
    lib.mppib_last_error.restype = C.c_char_p
    for name in SYMBOLS:
        if name != "mppib_last_error":
            getattr(lib, name).restype = C.c_int64 if name == "mppib_rollout_smem_bytes" else C.c_int32
    if lib.mppib_abi_version() != ABI_VERSION:
        raise RuntimeError(f"libmppib.so ABI {lib.mppib_abi_version()} != python binding {ABI_VERSION}; rebuild")
    _lib = lib
    return lib


def _ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def dist_floats(params, nu):
    """(floats, layout) of the distribution buffer that K1 / K3 / K4 read under `params` with `nu` inputs: 1 + 3 n^2 with cov_horizon
    (n = T*nu), 1 + 3 nu^2 with cov_full, 1 + nu otherwise (update_cov with a diagonal Sigma, or update_lambda alone)."""
    nu = int(nu)
    if params.n_modes > 1:
        M = int(params.n_modes)
        return 1 + M + int(params.T) * nu, f"n_modes > 1 mode state (active mode, F[M], U_exec[T*nu], M = {M})"
    if params.mode == MODE_CEM:
        n, E = int(params.T) * nu, int(params.n_elites)
        return 2 + E + n + E * n, f"mppi_mode cem (carry offset, elites valid, S_elite[E], sigma[T*nu], elites[E][T*nu], E = {E})"
    if params.update_cov and params.cov_horizon:
        n = int(params.T) * nu
        return 1 + 3 * n * n, f"cov_horizon (lambda, Sigma_H, L_H, Sigma_H^-1, n = T*nu = {n})"
    if params.update_cov and params.cov_full:
        return 1 + 3 * nu * nu, "cov_full (lambda, Sigma, L, Sigma^-1)"
    return 1 + nu, "(lambda, cov[nu])"


def shard_row_floats(params, nu):
    """Floats of one shard row that K3 (or the elite kernel of mppi_mode cem) writes under `params` with `nu` inputs once a
    distribution is registered, as the library sizes its buffers (shard_row_floats in csrc/common.cuh): 2 + T*nu, + T*nu with
    update_cov, + nu(nu+1)/2 with cov_full, + n(n+1)/2 with cov_horizon (n = T*nu); n_modes * (2 + T*nu) with n_modes > 1;
    cem_row_floats with mppi_mode cem; 4 + T*nu with constraint_mode (the row adds n_feasible and min V).  With control_knots = P > 0
    the control vector is P*nu long (ctrl_rows in csrc/common.cuh)."""
    T, nu = int(params.T), int(nu)
    n = (int(params.control_knots) or T) * nu
    if params.mode == MODE_CEM:
        return cem_row_floats(T, nu, params.n_elites)
    if params.n_modes > 1:
        return int(params.n_modes) * (2 + n)
    if params.update_cov and params.cov_horizon:
        return 2 + n + n * (n + 1) // 2
    if params.update_cov and params.cov_full:
        return 2 + n + nu * (nu + 1) // 2
    if params.update_cov or params.update_lambda:
        return 2 + n * (2 if params.update_cov else 1)
    return 4 + n if params.constraint_mode else 2 + n


def temperature_row_floats():
    """Floats of one shard row of the temperature pass of lambda_mode ess: (n_valid as int32 bits, (m_j, s1_j, s2_j)[65]).  The library
    sizes its scratch and peer window for the longer of this row and K3's."""
    return ESS_ROW_FLOATS


def smooth_state_floats(T, nu):
    """Floats of the smooth state of mppi_mode smooth: (a_prev[nu], A[T][nu])."""
    return int(nu) + int(T) * int(nu)


def anneal_state_floats(T, n_iterations):
    """Floats of the schedule of annealed MPPI: (counter, s[N][T], r[N][T])."""
    return 1 + 2 * int(n_iterations) * int(T)


def spline_table_floats(T, P, d, nu):
    """Floats of the spline table of spline MPPI: rows[T + P][d + 3], then U_exec[T][nu]."""
    return (int(T) + int(P)) * (int(d) + 3) + int(T) * int(nu)


def cem_row_floats(T, nu, E):
    """Floats of one shard row of mppi_mode cem: (S, index bits)[E], actions[E][T*nu], padded to a multiple of 4."""
    return (2 * int(E) + int(E) * int(T) * int(nu) + 3) & ~3


def _destroy_handle(lib, handle_value):
    """Finalizer of a live MppibHandle (garbage collection or interpreter exit): frees the handle's device scratch."""
    try:
        lib.mppib_destroy(C.c_void_p(handle_value))
    except Exception:  # noqa: BLE001
        pass


class CudaBackend:
    """One handle per GPU (``MppibHandle``).  All tensor arguments must live on ``self.device``."""

    name = "cuda"

    def __init__(self, device):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError(
                f"mppi_isaac_b200 runs its hot path as sm_90a CUDA kernels only; device '{device}' is not a CUDA "
                "device and there is no CPU fallback (the reference's CPU pipeline is reproduced by oracle/ for tests only)")
        if not torch.cuda.is_available():
            raise RuntimeError("no CUDA device visible: mppi_isaac_b200 has no CPU fallback")
        self.lib = load_library()
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self.handle = C.c_void_p(0)
        self.model = None
        self.params = None
        self._mirror_keepalive = None
        self._dist_keepalive = None
        self._smooth_keepalive = None
        self._anneal_keepalive = None     # (state, N)
        self._spline_keepalive = None     # the registered spline table
        self._constraint_keepalive = None  # (viol, cstate) of constrained MPPI
        self._temperature_keepalive = None  # the state of lambda_mode ess
        self.launches = 0   # kernels launched through this handle (bench.py's gpu_launches)

    # -- lifetime -------------------------------------------------------------------------------
    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed ({rc}): {self.lib.mppib_last_error().decode()}")

    def create(self, model: MppibModel, params: MppibParams):
        if self.handle:
            self.destroy()
        self.model, self.params = model, params
        self._check(self.lib.mppib_create(C.byref(model), C.byref(params), C.c_int32(self.device.index), C.byref(self.handle)), "mppib_create")
        self._finalizer = weakref.finalize(self, _destroy_handle, self.lib, self.handle.value)   # also runs at interpreter exit
        if self._mirror_keepalive is not None:           # a re-created handle keeps writing the action to the same pinned mirror
            self.set_action_mirror(self._mirror_keepalive)
        if self._dist_keepalive is not None:             # ... and keeps following the planner's adaptive distribution
            self.set_distribution(self._dist_keepalive)
        if self._smooth_keepalive is not None:           # ... and the planner's smooth state
            self.set_smooth_state(self._smooth_keepalive)
        if self._anneal_keepalive is not None:           # ... and its annealing schedule, while it still fits the horizon (a planner
            state, n = self._anneal_keepalive            # rebuilt for another horizon or mode registers its own)
            if not (state.numel() == anneal_state_floats(params.T, n) and self.lib.mppib_set_anneal(self.handle, _ptr(state), C.c_int32(n)) == 0):
                self._anneal_keepalive = None
        if self._spline_keepalive is not None:           # ... and its spline table, while the block still has the (P, d) it was built for
            table, P, d = self._spline_keepalive
            if not (int(params.control_knots) == P and int(params.spline_degree) == d
                    and table.numel() == spline_table_floats(params.T, P, d, model.nu)
                    and self.lib.mppib_set_spline(self.handle, _ptr(table), C.c_int32(P), C.c_int32(d)) == 0):
                self._spline_keepalive = None
        if self._constraint_keepalive is not None:       # ... and its violation buffer, while the block still plans with it for the same (T, K)
            viol, cstate = self._constraint_keepalive
            if not (params.constraint_mode and viol.numel() == int(params.T) * int(params.K)
                    and self.lib.mppib_set_constraint(self.handle, _ptr(viol), _ptr(cstate)) == 0):
                self._constraint_keepalive = None
        if self._temperature_keepalive is not None:      # ... and its temperature state
            self._check(self.lib.mppib_set_temperature(self.handle, _ptr(self._temperature_keepalive)), "mppib_set_temperature")

    def destroy(self):
        if self.handle:
            fin = getattr(self, "_finalizer", None)
            if fin is not None:
                fin.detach()
            self.lib.mppib_destroy(self.handle)
            self.handle = C.c_void_p(0)

    def set_params(self, params: MppibParams):
        self._check_dist_fits(params, self.model, "mppib_set_params")
        self._check(self.lib.mppib_set_params(self.handle, C.byref(params)), "mppib_set_params")
        self.params = params             # only once the library took it: a refused block leaves the handle as it was

    def set_model(self, model: MppibModel):
        self._check_dist_fits(self.params, model, "mppib_set_model")
        self._check(self.lib.mppib_set_model(self.handle, C.byref(model)), "mppib_set_model")
        self.model = model

    def state_size(self) -> int:
        return int(self.lib.mppib_state_size(self.handle))

    def obs_size(self) -> int:
        return int(self.lib.mppib_obs_size(self.handle))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # -- hot path -------------------------------------------------------------------------------
    def sample(self, seed, plan_idx, k_offset, k_total, U, prior_row, actions, noise, plan_ctr=None):
        self.launches += 1
        self._check(self.lib.mppib_sample(self.handle, C.c_uint64(seed), C.c_uint64(plan_idx), _ptr(plan_ctr), C.c_uint32(k_offset), C.c_uint32(k_total),
                                          _ptr(U), _ptr(prior_row), _ptr(actions), _ptr(noise), self._stream()), "mppib_sample")

    def sample_colored(self, seed, plan_idx, k_offset, k_total, U, prior_row, Lt, actions, noise, plan_ctr=None):
        """K1 with time-correlated noise: the draws of ``sample`` correlated over the horizon by the lower (T, T) float32 device
        tensor ``Lt`` (``planner.mppi.colored_noise_chol``) before the control-space colour."""
        T, n = int(self.params.T), int(self.params.T) * int(self.model.nu) * int(self.params.K)
        if tuple(Lt.shape) != (T, T) or Lt.dtype != torch.float32 or not Lt.is_contiguous():
            raise RuntimeError(f"mppib_sample_colored: Lt must be a contiguous float32 ({T}, {T}) tensor, got {Lt.dtype} {tuple(Lt.shape)}")
        for name, t in (("actions", actions), ("noise", noise)):
            if t is not None and t.numel() != n:
                raise RuntimeError(f"mppib_sample_colored: {name} must hold T*nu*K = {n} floats, got {t.numel()}")
        self.launches += 1
        self._check(self.lib.mppib_sample_colored(self.handle, C.c_uint64(seed), C.c_uint64(plan_idx), _ptr(plan_ctr), C.c_uint32(k_offset),
                                                  C.c_uint32(k_total), _ptr(U), _ptr(prior_row), _ptr(Lt), _ptr(actions), _ptr(noise),
                                                  self._stream()), "mppib_sample_colored")

    def sample_smooth(self, seed, plan_idx, k_offset, k_total, U, actions, noise, plan_ctr=None):
        """K1 of mppi_mode smooth: the draws of ``sample`` are derivatives, integrated from the registered state's last action
        (``set_smooth_state``) into ``actions``; ``noise`` receives the applied derivative minus U."""
        n = int(self.params.T) * int(self.model.nu) * int(self.params.K)
        for name, t in (("actions", actions), ("noise", noise)):
            if t is not None and t.numel() != n:
                raise RuntimeError(f"mppib_sample_smooth: {name} must hold T*nu*K = {n} floats, got {t.numel()}")
        self.launches += 1
        self._check(self.lib.mppib_sample_smooth(self.handle, C.c_uint64(seed), C.c_uint64(plan_idx), _ptr(plan_ctr), C.c_uint32(k_offset),
                                                 C.c_uint32(k_total), _ptr(U), _ptr(actions), _ptr(noise), self._stream()), "mppib_sample_smooth")

    def noise_library(self, k_offset, k_total, halton_tab, B, n_knots, Z):
        self.launches += 1
        self._check(self.lib.mppib_noise_library(self.handle, C.c_uint32(k_offset), C.c_uint32(k_total), _ptr(halton_tab), _ptr(B), C.c_int32(n_knots),
                                                 _ptr(Z), self._stream()), "mppib_noise_library")

    def sample_library(self, k_offset, k_total, U, prior_row, Z, actions, noise):
        self.launches += 1
        self._check(self.lib.mppib_sample_library(self.handle, C.c_uint32(k_offset), C.c_uint32(k_total), _ptr(U), _ptr(prior_row), _ptr(Z),
                                                  _ptr(actions), _ptr(noise), self._stream()), "mppib_sample_library")

    def rollout(self, state0, state, actions, t0, nsteps, obs, act_t0=0, root0=None):
        """``actions`` holds time slices [act_t0, ...) laid out [t][nu][K]; steps t0..t0+nsteps-1 are executed."""
        self.launches += 1
        base = actions.data_ptr() - act_t0 * self.model.nu * self.params.K * 4
        self._check(self.lib.mppib_rollout(self.handle, _ptr(state0), _ptr(root0), _ptr(state), C.c_void_p(base), C.c_int32(t0), C.c_int32(nsteps),
                                           _ptr(obs), self._stream()), "mppib_rollout")

    MAPPING_NAMES = {0: "thread-per-rollout (rollout.cu)", 1: "lanes-per-rollout (rollout_lanes.cu)", 2: "team-of-lanes-per-rollout (rollout_team.cu)"}

    def rollout_mapping(self) -> str:
        """Which K2 kernel this handle launches (include/mppib.h MPPIB_MAPPING_*)."""
        r = self.lib.mppib_rollout_mapping(self.handle)
        self._check(min(r, 0), "mppib_rollout_mapping")
        return self.MAPPING_NAMES[r]

    # -- multi-GPU exchange over peer memory (include/mppib.h: mppib_peer_*) ----------------------
    def peer_alloc(self, world: int, rank: int) -> bytes:
        buf = (C.c_ubyte * 64)()
        self._check(self.lib.mppib_peer_alloc(self.handle, C.c_int32(world), C.c_int32(rank), buf), "mppib_peer_alloc")
        return bytes(buf)

    def peer_open(self, peer: int, ipc_handle: bytes):
        buf = (C.c_ubyte * 64).from_buffer_copy(ipc_handle)
        self._check(self.lib.mppib_peer_open(self.handle, C.c_int32(peer), buf), "mppib_peer_open")

    def peer_close(self):
        if self.handle:
            self.lib.mppib_peer_close(self.handle)

    def set_action_mirror(self, pinned_host_tensor):
        """K4 also stores the action into this PINNED host tensor (None switches it off)."""
        self._mirror_keepalive = pinned_host_tensor
        self._check(self.lib.mppib_set_action_mirror(self.handle, _ptr(pinned_host_tensor)), "mppib_set_action_mirror")

    def _cov_full(self):
        return bool(self.params.update_cov) and bool(self.params.cov_full)

    def _cov_horizon(self):
        return bool(self.params.update_cov) and bool(self.params.cov_horizon)

    def partial_row_floats(self) -> int:
        """Floats of one shard row K3 writes with a registered distribution (``shard_row_floats``)."""
        return shard_row_floats(self.params, self.model.nu)

    def _check_row(self, rows, what):
        if ((self._cov_full() or self._cov_horizon() or self.params.mode == MODE_CEM or self.params.n_modes > 1) and self._dist_keepalive is not None
                and rows is not None and rows.shape[-1] != self.partial_row_floats()):
            kind = "n_modes > 1" if self.params.n_modes > 1 else "mppi_mode cem" if self.params.mode == MODE_CEM else "cov_horizon" if self._cov_horizon() else "cov_full"
            raise RuntimeError(f"{what}: {kind} shard rows hold {self.partial_row_floats()} floats, got {rows.shape[-1]}")

    def _check_dist_fits(self, params, model, what):
        """The library keeps only a pointer to the registered distribution, so every change of (T, nu) or of the update rule is checked
        against its length before the library sees it: a shorter buffer would be read past its end by the next K1, shift or K4.  The
        same holds for the smooth state of mppi_mode smooth."""
        state = getattr(self, "_smooth_keepalive", None)
        if state is not None and params.mode == MODE_SMOOTH:
            need = smooth_state_floats(params.T, model.nu)
            if state.numel() != need:
                raise RuntimeError(f"{what}: the registered smooth state holds {state.numel()} floats, but T = {int(params.T)}, "
                                   f"nu = {int(model.nu)} needs nu + T*nu = {need}; register a new one (set_smooth_state) first")
        if self._dist_keepalive is not None:
            need, layout = dist_floats(params, model.nu)
            if self._dist_keepalive.numel() != need:
                raise RuntimeError(f"{what}: the registered distribution holds {self._dist_keepalive.numel()} floats, but T = {int(params.T)}, "
                                   f"nu = {int(model.nu)} needs {layout} = {need}; register a new one (set_distribution) first")

    def set_distribution(self, dist):
        """Adaptive MPPI: register the device tensor (lambda, cov[nu]) -- with cov_full (lambda, Sigma, L, Sigma^-1), 1 + 3 nu^2
        floats, with cov_horizon (lambda, Sigma_H, L_H, Sigma_H^-1), 1 + 3 n^2 floats, n = T*nu -- that K1 / K3 read and K4 updates
        (None switches it off).  With mppi_mode cem it is the CEM state, with n_modes > 1 the mode state (``dist_floats``)."""
        if dist is not None:
            need, layout = dist_floats(self.params, self.model.nu)
            if dist.numel() != need:
                raise RuntimeError(f"mppib_set_distribution: {layout} = {need} floats, got {dist.numel()}")
        self._dist_keepalive = dist
        self._check(self.lib.mppib_set_distribution(self.handle, _ptr(dist)), "mppib_set_distribution")

    def set_smooth_state(self, state):
        """mppi_mode smooth: register the device tensor (a_prev[nu], A[T][nu]) that K1 reads and K4 updates (None switches it off)."""
        if state is not None:
            need = smooth_state_floats(self.params.T, self.model.nu)
            if state.numel() != need:
                raise RuntimeError(f"mppib_set_smooth_state: (a_prev[nu], A[T][nu]) = nu + T*nu = {need} floats, got {state.numel()}")
        self._smooth_keepalive = state
        self._check(self.lib.mppib_set_smooth_state(self.handle, _ptr(state)), "mppib_set_smooth_state")

    def set_anneal(self, state, n_iterations=0):
        """Annealed MPPI: register the device tensor (counter, s[N][T], r[N][T]) of N = n_iterations MPPI iterations per plan that K1 / K3
        read, K4 advances and the shift resets (None switches it off).  The library records T and refuses launches once it changes."""
        if state is not None:
            need = anneal_state_floats(self.params.T, n_iterations)
            if state.numel() != need or state.dtype != torch.float32 or not state.is_contiguous():
                raise RuntimeError(f"mppib_set_anneal: (counter, s[N][T], r[N][T]) = 1 + 2*N*T = {need} contiguous float32 values, got "
                                   f"{state.dtype} {state.numel()}")
        self._check(self.lib.mppib_set_anneal(self.handle, _ptr(state), C.c_int32(0 if state is None else int(n_iterations))), "mppib_set_anneal")
        self._anneal_keepalive = None if state is None else (state, int(n_iterations))

    def set_spline(self, table):
        """Spline MPPI: register the device tensor (rows[T + P][d + 3], U_exec[T][nu]) of ``blob.spline_table`` for the parameter
        block's (T, control_knots, spline_degree); K1 and the shift read it, K4 writes U_exec (None switches it off)."""
        P, d = int(self.params.control_knots), int(self.params.spline_degree)
        if table is not None:
            need = spline_table_floats(self.params.T, P, d, self.model.nu)
            if table.numel() != need or table.dtype != torch.float32 or not table.is_contiguous():
                raise RuntimeError(f"mppib_set_spline: (rows[T + P][d + 3], U_exec[T][nu]) = {need} contiguous float32 values, got "
                                   f"{table.dtype} {table.numel()}")
        self._check(self.lib.mppib_set_spline(self.handle, _ptr(table), C.c_int32(P), C.c_int32(d)), "mppib_set_spline")
        self._spline_keepalive = None if table is None else (table, P, d)

    def set_constraint(self, viol, cstate=None):
        """Constrained MPPI: register the (T, K) float32 device tensor of per-step constraint margins K3 reads and the (2,) float32
        device tensor (n_feasible as int32 bits, min V) K4 writes (None switches it off).  The library records (T, K)."""
        if viol is not None:
            T, K = int(self.params.T), int(self.params.K)
            if viol.numel() != T * K or viol.dtype != torch.float32 or not viol.is_contiguous():
                raise RuntimeError(f"mppib_set_constraint: viol must be a contiguous float32 (T, K) = ({T}, {K}) tensor, got {viol.dtype} {tuple(viol.shape)}")
            if cstate is None or cstate.numel() != 2 or cstate.dtype != torch.float32:
                raise RuntimeError("mppib_set_constraint: cstate must be a float32 tensor of 2 values")
        self._check(self.lib.mppib_set_constraint(self.handle, _ptr(viol), _ptr(None if viol is None else cstate)), "mppib_set_constraint")
        self._constraint_keepalive = None if viol is None else (viol, cstate)

    def set_temperature(self, state):
        """lambda_mode ess: register the float32 device tensor (lambda_j[65], 1/lambda_j[65], n_valid bits, lambda, ESS_j[65]) whose grid
        the caller filled (``blob.ess_grid``); the solve writes the rest and dist[0] (None switches it off)."""
        if state is not None and (state.numel() != ESS_STATE_FLOATS or state.dtype != torch.float32 or not state.is_contiguous()):
            raise RuntimeError(f"mppib_set_temperature: the state holds {ESS_STATE_FLOATS} contiguous float32 values, got {state.dtype} {state.numel()}")
        self._check(self.lib.mppib_set_temperature(self.handle, _ptr(state)), "mppib_set_temperature")
        self._temperature_keepalive = state

    def temperature(self, cost, x, U, row, solve=True):
        """lambda_mode ess: the temperature pass over this shard's (T, K) cost and, in SIMPLE mode, the noise K3 weights; writes the shard
        row into ``row`` (196 floats).  solve: the last CTA also applies the rule (one rank, or every rank through the open peer window);
        otherwise gather the rows and call ``temperature_solve``."""
        if row is None or row.numel() != ESS_ROW_FLOATS or row.dtype != torch.float32:
            raise RuntimeError(f"mppib_temperature: row must be a float32 tensor of {ESS_ROW_FLOATS} values")
        self.launches += 1
        self._check(self.lib.mppib_temperature(self.handle, _ptr(cost), _ptr(x if self.params.mode == MODE_SIMPLE else None), _ptr(U), _ptr(row),
                                               C.c_int32(1 if solve else 0), self._stream()), "mppib_temperature")

    def temperature_solve(self, rows, G):
        """lambda_mode ess: the rule over the (G, 196) float32 device rows of every rank, in rank order."""
        if rows.dtype != torch.float32 or not rows.is_contiguous() or rows.numel() < int(G) * ESS_ROW_FLOATS:
            raise RuntimeError(f"mppib_temperature_solve: rows must be a contiguous float32 (G, {ESS_ROW_FLOATS}) tensor")
        self.launches += 1
        self._check(self.lib.mppib_temperature_solve(self.handle, _ptr(rows), C.c_int32(int(G)), self._stream()), "mppib_temperature_solve")

    def sample_spline(self, seed, plan_idx, k_offset, k_total, U, actions, xk, plan_ctr=None):
        """K1 of spline MPPI: knots theta~ = clamp(U + L0 z) per sample, xk[P][nu][K] = theta~ - U (SIMPLE) or theta~ (MEAN), and
        actions[T][nu][K] interpolated by the registered table."""
        P, T, nu, K = int(self.params.control_knots), int(self.params.T), int(self.model.nu), int(self.params.K)
        for name, t, n in (("actions", actions, T * nu * K), ("xk", xk, P * nu * K)):
            if t is None or t.numel() != n:
                raise RuntimeError(f"mppib_sample_spline: {name} must hold {n} floats")
        self.launches += 1
        self._check(self.lib.mppib_sample_spline(self.handle, C.c_uint64(seed), C.c_uint64(plan_idx), _ptr(plan_ctr), C.c_uint32(k_offset),
                                                 C.c_uint32(k_total), _ptr(U), _ptr(actions), _ptr(xk), self._stream()), "mppib_sample_spline")

    def reduce(self, cost, x, U, partial):
        self._check_row(partial, "mppib_reduce")
        self.launches += 1
        self._check(self.lib.mppib_reduce(self.handle, _ptr(cost), _ptr(x), _ptr(U), _ptr(partial), self._stream()), "mppib_reduce")

    def reduce_finalize(self, cost, x, U, partial, action_out, stats):
        """K3 + K4 in one launch (single-GPU plans)."""
        self._check_row(partial, "mppib_reduce_finalize")
        self.launches += 1
        self._check(self.lib.mppib_reduce_finalize(self.handle, _ptr(cost), _ptr(x), _ptr(U), _ptr(partial), _ptr(action_out), _ptr(stats), self._stream()),
                    "mppib_reduce_finalize")

    def finalize(self, partials, G, U, action_out, stats):
        self._check_row(partials, "mppib_finalize")
        self.launches += 1
        self._check(self.lib.mppib_finalize(self.handle, _ptr(partials), C.c_int32(G), _ptr(U), _ptr(action_out), _ptr(stats), self._stream()), "mppib_finalize")

    def shift(self, U, plan_ctr=None):
        self.launches += 1
        self._check(self.lib.mppib_shift(self.handle, _ptr(U), _ptr(plan_ctr), self._stream()), "mppib_shift")
