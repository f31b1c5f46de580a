"""-m gpu: which K1 entry samples which mode.  Each of the five sampling entries (mppib_sample, _colored, _smooth, mppib_noise_library,
mppib_sample_library) is called on tiny shapes in every handle state: fixed Sigma; the diag, full and horizon rules with a registered
distribution; cem and smooth with and without their state; a registered annealing schedule; n_modes = 2; n_worlds = 4.  An admitted pair
must launch without error, a refused one must raise the library's message before any launch.  A second table pins the shard, size and
schedule refusals that depend on the call's arguments rather than on the mode."""
import copy

import numpy as np
import pytest
import torch

from mppi_isaac_b200.backend import anneal_state_floats, dist_floats, smooth_state_floats
from mppi_isaac_b200.model.blob import MODE_CEM, make_params
from mppi_isaac_b200.planner.mppi import colored_noise_chol, halton_spline_operator, halton_table
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from synth_mppi import nu_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NU, T, K = 3, 8, 256
NK = 3                                                                  # knots of the noise library
ENTRIES = ("sample", "colored", "smooth", "noise_library", "sample_library")

CEM = "samples through mppib_sample_colored"
SMOOTH = "samples through mppib_sample_smooth"
NOT_SMOOTH = "needs mode smooth"
ANNEAL = "noise library"

# state -> (config keys, what is registered, {entry: refusal substring}); an entry not listed is admitted
STATES = {
    "fixed": (dict(), None, {"smooth": NOT_SMOOTH}),
    "diag": (dict(update_cov=True), "dist", {"smooth": NOT_SMOOTH}),
    "full": (dict(update_cov=True, cov_type="full"), "dist", {"smooth": NOT_SMOOTH}),
    "horizon": (dict(update_cov=True, cov_type="horizon"), "dist", {"colored": "cov_horizon", "smooth": NOT_SMOOTH}),
    "horizon_unregistered": (dict(update_cov=True, cov_type="horizon"), None, {"colored": "cov_horizon", "smooth": NOT_SMOOTH}),
    "cem": (dict(mppi_mode="cem"), "dist", {"sample": CEM, "smooth": NOT_SMOOTH, "noise_library": CEM, "sample_library": CEM}),
    "cem_unregistered": (dict(mppi_mode="cem"), None, {"sample": CEM, "colored": "needs its state registered", "smooth": NOT_SMOOTH,
                                                        "noise_library": CEM, "sample_library": CEM}),
    "smooth": (dict(mppi_mode="smooth"), "smooth", {"sample": SMOOTH, "colored": SMOOTH, "noise_library": SMOOTH, "sample_library": SMOOTH}),
    "smooth_unregistered": (dict(mppi_mode="smooth"), None, {"sample": SMOOTH, "colored": SMOOTH, "smooth": "no smooth state",
                                                             "noise_library": SMOOTH, "sample_library": SMOOTH}),
    "anneal": (dict(), "anneal", {"smooth": NOT_SMOOTH, "noise_library": ANNEAL, "sample_library": ANNEAL}),
    "modes": (dict(n_modes=2), "dist", {"smooth": NOT_SMOOTH}),
    "worlds": (dict(n_worlds=4), None, {"smooth": NOT_SMOOTH}),
}


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(DEV)


def handle(keys, registered):
    from mppi_isaac_b200.backend import CudaBackend
    d = dict(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.3 * np.eye(NU)).tolist(), u_min=[-0.6],
             u_max=[0.6], lambda_=0.05, sample_null_action=True)
    d.update(keys)
    p = make_params(MPPIConfig(**d), IsaacGymConfig(), NU, K, [])
    be = CudaBackend(DEV)
    be.create(nu_model(NU), p)
    if registered == "dist":
        n, _ = dist_floats(p, NU)
        buf = np.zeros(n)
        if p.n_modes > 1:
            buf[1:1 + p.n_modes] = np.inf
        elif p.mode == MODE_CEM:                                        # CEM: sigma = 0.3 for every step, no elites yet
            buf[2 + p.n_elites:2 + p.n_elites + T * NU] = 0.3
        else:                                                           # lambda, then Sigma = L = Sigma^-1 = I (or cov = 1)
            m = T * NU if p.cov_horizon else NU
            buf[0] = 0.05
            if p.cov_full or p.cov_horizon:
                buf[1:] = np.tile(np.eye(m).ravel(), 3)
            else:
                buf[1:] = 1.0
        be.set_distribution(dev(buf))
    elif registered == "smooth":
        be.set_smooth_state(torch.zeros(smooth_state_floats(T, NU), device=DEV))
    elif registered == "anneal":
        be.set_anneal(dev(np.concatenate([[0.0], np.full(anneal_state_floats(T, 2) - 1, 1.0)])), 2)
    return be, p


def call(be, p, entry, k_offset=0, k_total=K, n_knots=NK, null=False):
    T_ = int(p.T)
    U = torch.zeros((max(p.n_modes, 1), T_, NU), device=DEV)
    a, n, Z = (torch.zeros((T_, NU, K), device=DEV) for _ in range(3))
    if null:
        a = None
    if entry == "sample":
        be.sample(7, 3, k_offset, k_total, U, None, a, n)
    elif entry == "colored":
        be.sample_colored(7, 3, k_offset, k_total, U, None, dev(colored_noise_chol(T_, 2.0)), a, n)
    elif entry == "smooth":
        be.sample_smooth(7, 3, k_offset, k_total, U, a, n)
    elif entry == "noise_library":
        be.noise_library(k_offset, k_total, torch.from_numpy(halton_table(NK * NU, 5)).to(DEV), dev(halton_spline_operator(T_, NK)), n_knots,
                         None if null else Z)
    else:
        be.sample_library(k_offset, k_total, U, None, Z, a, n)


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("state", list(STATES))
def test_entry_admits_or_refuses_the_handle_state(state, entry):
    keys, registered, refused = STATES[state]
    be, p = handle(keys, registered)
    if entry in refused:
        with pytest.raises(RuntimeError, match=refused[entry]):
            call(be, p, entry)
    else:
        call(be, p, entry)
        torch.cuda.synchronize()
    be.destroy()


# (state, call arguments) -> {entry: refusal substring}; an entry not listed is admitted
ARGUMENT_CASES = [
    ("fixed", dict(null=True), {e: "null argument" for e in ENTRIES}),
    ("fixed", dict(k_total=K - 1), {e: "k_total" for e in ENTRIES}),
    ("fixed", dict(n_knots=33), {"smooth": NOT_SMOOTH, "noise_library": "n_knots = 33"}),
    ("worlds", dict(k_total=K + 2), {"sample": "multiples", "colored": "multiples", "smooth": NOT_SMOOTH, "noise_library": "multiples",
                                     "sample_library": "multiples"}),
    ("modes", dict(k_total=2 * K), {"sample": "k_total", "colored": "k_total", "smooth": NOT_SMOOTH, "sample_library": "k_total"}),
]


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("case", range(len(ARGUMENT_CASES)))
def test_entry_admits_or_refuses_the_call(case, entry):
    state, kw, refused = ARGUMENT_CASES[case]
    be, p = handle(*STATES[state][:2])
    if entry in refused:
        with pytest.raises(RuntimeError, match=refused[entry]):
            call(be, p, entry, **kw)
    else:
        call(be, p, entry, **kw)
        torch.cuda.synchronize()
    be.destroy()


@pytest.mark.parametrize("entry", ENTRIES)
def test_a_schedule_for_another_horizon(entry):
    """The Philox entries check the schedule's T; the library entries refuse any schedule, whatever its T."""
    be, p = handle(*STATES["anneal"][:2])
    q = copy.copy(p)
    q.T = T + 1
    be.set_params(q)
    refused = {"sample": "registered for T", "colored": "registered for T", "smooth": NOT_SMOOTH, "noise_library": ANNEAL,
               "sample_library": ANNEAL}
    with pytest.raises(RuntimeError, match=refused[entry]):
        call(be, q, entry)
    be.destroy()
