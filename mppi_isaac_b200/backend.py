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

from .model.blob import ABI_VERSION, MppibModel, MppibParams

_LIB_PATH = os.environ.get("MPPIB_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "libmppib.so")   # MPPIB_LIB: tuning builds
_lib = None

SYMBOLS = [
    "mppib_abi_version", "mppib_last_error", "mppib_create", "mppib_destroy", "mppib_set_params",
    "mppib_set_model", "mppib_state_size", "mppib_obs_size", "mppib_sample", "mppib_rollout",
    "mppib_reduce", "mppib_finalize", "mppib_shift", "mppib_noise_library", "mppib_sample_library",
    "mppib_peer_alloc", "mppib_peer_open", "mppib_peer_close", "mppib_cost_pose", "mppib_set_action_mirror", "mppib_reduce_finalize", "mppib_rollout_smem_bytes", "mppib_rollout_mapping", "mppib_rollout_mapping_for_model",
    "mppib_set_distribution",
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

    def destroy(self):
        if self.handle:
            fin = getattr(self, "_finalizer", None)
            if fin is not None:
                fin.detach()
            self.lib.mppib_destroy(self.handle)
            self.handle = C.c_void_p(0)

    def set_params(self, params: MppibParams):
        self.params = params
        self._check(self.lib.mppib_set_params(self.handle, C.byref(params)), "mppib_set_params")

    def set_model(self, model: MppibModel):
        self.model = model
        self._check(self.lib.mppib_set_model(self.handle, C.byref(model)), "mppib_set_model")

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

    def partial_row_floats(self) -> int:
        """Floats of one shard row K3 writes with a registered distribution: 2 + T*nu, + T*nu with update_cov, or + nu(nu+1)/2
        with update_cov and cov_full."""
        T, nu = int(self.params.T), int(self.model.nu)
        if self._cov_full():
            return 2 + T * nu + nu * (nu + 1) // 2
        return 2 + T * nu * (2 if self.params.update_cov else 1)

    def _check_row(self, rows, what):
        if self._cov_full() and self._dist_keepalive is not None and rows is not None and rows.shape[-1] != self.partial_row_floats():
            raise RuntimeError(f"{what}: cov_full shard rows hold {self.partial_row_floats()} floats, got {rows.shape[-1]}")

    def set_distribution(self, dist):
        """Adaptive MPPI: register the device tensor (lambda, cov[nu]) -- with cov_full (lambda, Sigma, L, Sigma^-1), 1 + 3 nu^2
        floats -- that K1 / K3 read and K4 updates (None switches it off)."""
        if dist is not None and self._cov_full() and dist.numel() != 1 + 3 * self.model.nu ** 2:
            raise RuntimeError(f"mppib_set_distribution: cov_full needs (lambda, Sigma, L, Sigma^-1) = {1 + 3 * self.model.nu ** 2} floats, "
                               f"got {dist.numel()}")
        self._dist_keepalive = dist
        self._check(self.lib.mppib_set_distribution(self.handle, _ptr(dist)), "mppib_set_distribution")

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
