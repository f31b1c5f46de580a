"""Which planning modes may run together: make_params refuses the same single features and pairs of features, with the same messages,
as before the exclusions moved into one table (blob.FEATURES / EXCLUSIONS); the table and the library's own (csrc/api.cu) refuse the
same parameter blocks, at and just over every size limit too; and mppib_set_anneal refuses a schedule exactly when the table does."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

from mppi_isaac_b200 import backend
from mppi_isaac_b200.model.blob import make_params, mode_refusal
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from synth_mppi import nu_model

# config keys of each feature, on top of a plain random-sampling config
FEATURES = {
    "cem": dict(mppi_mode="cem"),
    "smooth": dict(mppi_mode="smooth"),
    "halton": dict(sampling_method="halton"),
    "colored": dict(sampling_method="colored"),
    "update_cov": dict(update_cov=True),
    "update_lambda": dict(update_lambda=True),
    "cov_full": dict(update_cov=True, cov_type="full"),
    "cov_horizon": dict(update_cov=True, cov_type="horizon"),
    "filter_u": dict(filter_u=True),
    "n_worlds": dict(n_worlds=2, cvar_alpha=0.5),
    "n_modes": dict(n_modes=2),
    "anneal": dict(anneal_iterations=2, anneal_iter_decay=0.8),
    "knots": dict(control_knots=4),
    "constraint": dict(constraint_mode="feasible_first"),
}

# What make_params refused, and why, before the exclusions moved into the table: every single feature and every pair that sets no
# config key twice, at horizon 12, nu = 3, 256 samples.
REFUSED = {
    (): None,
    ('cem',): None,
    ('smooth',): None,
    ('halton',): None,
    ('colored',): None,
    ('update_cov',): None,
    ('update_lambda',): None,
    ('cov_full',): None,
    ('cov_horizon',): None,
    ('filter_u',): None,
    ('n_worlds',): None,
    ('n_modes',): None,
    ('anneal',): None,
    ('knots',): None,
    ('constraint',): None,
    ('cem', 'halton'): 'mppi_mode: cem samples with sampling_method random or colored, not halton',
    ('cem', 'colored'): None,
    ('cem', 'update_cov'): 'mppi_mode: cem has its own update rule and excludes update_cov and update_lambda',
    ('cem', 'update_lambda'): 'mppi_mode: cem has its own update rule and excludes update_cov and update_lambda',
    ('cem', 'cov_full'): 'mppi_mode: cem has its own update rule and excludes update_cov and update_lambda',
    ('cem', 'cov_horizon'): 'mppi_mode: cem has its own update rule and excludes update_cov and update_lambda',
    ('cem', 'filter_u'): None,
    ('cem', 'n_worlds'): 'n_worlds > 1 excludes mppi_mode cem and smooth',
    ('cem', 'n_modes'): 'n_modes > 1 excludes mppi_mode cem and smooth',
    ('cem', 'anneal'): 'annealed MPPI excludes mppi_mode cem, which has its own sigma',
    ('cem', 'knots'): 'control_knots > 0 excludes mppi_mode cem and smooth',
    ('cem', 'constraint'): 'constraint_mode: feasible_first excludes mppi_mode cem and smooth',
    ('smooth', 'halton'): 'mppi_mode: smooth samples its derivative with sampling_method random, not halton',
    ('smooth', 'colored'): 'mppi_mode: smooth samples its derivative with sampling_method random, not colored',
    ('smooth', 'update_cov'): 'mppi_mode: smooth excludes update_cov and update_lambda',
    ('smooth', 'update_lambda'): 'mppi_mode: smooth excludes update_cov and update_lambda',
    ('smooth', 'cov_full'): 'mppi_mode: smooth excludes update_cov and update_lambda',
    ('smooth', 'cov_horizon'): 'mppi_mode: smooth excludes update_cov and update_lambda',
    ('smooth', 'filter_u'): 'mppi_mode: smooth excludes filter_u: the actions are already smooth, switch filter_u off',
    ('smooth', 'n_worlds'): 'n_worlds > 1 excludes mppi_mode cem and smooth',
    ('smooth', 'n_modes'): 'n_modes > 1 excludes mppi_mode cem and smooth',
    ('smooth', 'anneal'): 'annealed MPPI excludes mppi_mode smooth',
    ('smooth', 'knots'): 'control_knots > 0 excludes mppi_mode cem and smooth',
    ('smooth', 'constraint'): 'constraint_mode: feasible_first excludes mppi_mode cem and smooth',
    ('halton', 'update_cov'): None,
    ('halton', 'update_lambda'): None,
    ('halton', 'cov_full'): None,
    ('halton', 'cov_horizon'): None,
    ('halton', 'filter_u'): None,
    ('halton', 'n_worlds'): None,
    ('halton', 'n_modes'): None,
    ('halton', 'anneal'): 'annealed MPPI excludes sampling_method halton: the library is drawn once, so every iteration would reuse the same directions; use random or colored',
    ('halton', 'knots'): 'control_knots > 0 samples its knots with sampling_method random, not halton',
    ('halton', 'constraint'): None,
    ('colored', 'update_cov'): None,
    ('colored', 'update_lambda'): None,
    ('colored', 'cov_full'): None,
    ('colored', 'cov_horizon'): 'sampling_method: colored excludes cov_type: horizon, whose Sigma_H already models the time correlation',
    ('colored', 'filter_u'): None,
    ('colored', 'n_worlds'): None,
    ('colored', 'n_modes'): None,
    ('colored', 'anneal'): None,
    ('colored', 'knots'): 'control_knots > 0 samples its knots with sampling_method random, not colored',
    ('colored', 'constraint'): None,
    ('update_cov', 'update_lambda'): None,
    ('update_cov', 'cov_full'): None,
    ('update_cov', 'cov_horizon'): None,
    ('update_cov', 'filter_u'): None,
    ('update_cov', 'n_worlds'): None,
    ('update_cov', 'n_modes'): 'n_modes > 1 excludes update_cov and update_lambda: the adapted distribution belongs to one mean',
    ('update_cov', 'anneal'): 'annealed MPPI excludes update_cov and update_lambda (and so every cov_type)',
    ('update_cov', 'knots'): 'control_knots > 0 excludes update_cov and update_lambda',
    ('update_cov', 'constraint'): 'constraint_mode: feasible_first excludes update_cov and update_lambda',
    ('update_lambda', 'cov_full'): None,
    ('update_lambda', 'cov_horizon'): None,
    ('update_lambda', 'filter_u'): None,
    ('update_lambda', 'n_worlds'): None,
    ('update_lambda', 'n_modes'): 'n_modes > 1 excludes update_cov and update_lambda: the adapted distribution belongs to one mean',
    ('update_lambda', 'anneal'): 'annealed MPPI excludes update_cov and update_lambda (and so every cov_type)',
    ('update_lambda', 'knots'): 'control_knots > 0 excludes update_cov and update_lambda',
    ('update_lambda', 'constraint'): 'constraint_mode: feasible_first excludes update_cov and update_lambda',
    ('cov_full', 'filter_u'): None,
    ('cov_full', 'n_worlds'): None,
    ('cov_full', 'n_modes'): 'n_modes > 1 excludes update_cov and update_lambda: the adapted distribution belongs to one mean',
    ('cov_full', 'anneal'): 'annealed MPPI excludes update_cov and update_lambda (and so every cov_type)',
    ('cov_full', 'knots'): 'control_knots > 0 excludes update_cov and update_lambda',
    ('cov_full', 'constraint'): 'constraint_mode: feasible_first excludes update_cov and update_lambda',
    ('cov_horizon', 'filter_u'): None,
    ('cov_horizon', 'n_worlds'): 'n_worlds > 1 excludes cov_type: horizon',
    ('cov_horizon', 'n_modes'): 'n_modes > 1 excludes update_cov and update_lambda: the adapted distribution belongs to one mean',
    ('cov_horizon', 'anneal'): 'annealed MPPI excludes update_cov and update_lambda (and so every cov_type)',
    ('cov_horizon', 'knots'): 'control_knots > 0 excludes update_cov and update_lambda',
    ('cov_horizon', 'constraint'): 'constraint_mode: feasible_first excludes update_cov and update_lambda',
    ('filter_u', 'n_worlds'): None,
    ('filter_u', 'n_modes'): None,
    ('filter_u', 'anneal'): None,
    ('filter_u', 'knots'): 'control_knots > 0 excludes filter_u: the spline is smooth already, switch filter_u off',
    ('filter_u', 'constraint'): None,
    ('n_worlds', 'n_modes'): 'n_modes > 1 excludes n_worlds > 1',
    ('n_worlds', 'anneal'): None,
    ('n_worlds', 'knots'): 'control_knots > 0 excludes n_modes > 1 and n_worlds > 1',
    ('n_worlds', 'constraint'): 'constraint_mode: feasible_first excludes n_worlds > 1',
    ('n_modes', 'anneal'): "annealed MPPI excludes n_modes > 1: the Stein coupling's Sigma^-1 metric would need the schedule",
    ('n_modes', 'knots'): 'control_knots > 0 excludes n_modes > 1 and n_worlds > 1',
    ('n_modes', 'constraint'): 'constraint_mode: feasible_first excludes n_modes > 1',
    ('anneal', 'knots'): 'control_knots > 0 excludes annealed MPPI',
    ('anneal', 'constraint'): 'constraint_mode: feasible_first excludes annealed MPPI',
    ('knots', 'constraint'): 'constraint_mode: feasible_first excludes control_knots > 0',
}

# (feature, horizon, nu, control_knots): refused before the table, at and just over each size limit.  The one change is n_modes > 1 at
# T*nu = 520, which the library has always refused: make_params now refuses it too.
LIMITS = {
    ('cem', 64, 8, None): False,
    ('cem', 65, 8, None): True,
    ('cem', 256, 1, None): False,
    ('cem', 257, 1, None): True,
    ('smooth', 64, 8, None): False,
    ('smooth', 65, 8, None): True,
    ('smooth', 256, 1, None): False,
    ('smooth', 257, 1, None): True,
    ('colored', 64, 8, None): False,
    ('colored', 65, 8, None): True,
    ('colored', 256, 1, None): False,
    ('colored', 257, 1, None): True,
    ('n_modes', 64, 8, None): False,
    ('n_modes', 65, 8, None): False,
    ('n_modes', 256, 1, None): False,
    ('n_modes', 257, 1, None): False,
    ('cov_horizon', 32, 8, None): False,
    ('cov_horizon', 33, 8, None): True,
    ('knots', 64, 16, 32): False,
    ('knots', 64, 16, 33): True,
    ('knots', 256, 1, 4): False,
    ('knots', 257, 1, 4): True,
    # constraint_mode: two ring stages of (T*nu + 2T) * 32 floats fit up to T = 216 at nu = 2 (the library refused T = 217 at the first
    # plan before make_params and mppib_create refused it too)
    ('constraint', 216, 2, None): False,
    ('constraint', 217, 2, None): True,
}
LIMIT_FIXED = {("n_modes", 65, 8, None)}


def config(kw, T=12, nu=3, K=256):
    d = dict(num_samples=K, horizon=T, mppi_mode="simple", sampling_method="random", noise_sigma=(0.1 * np.eye(nu)).tolist(),
             u_min=[-1.0], u_max=[1.0], lambda_=0.1, rollout_var_discount=0.95)
    d.update(kw)
    return MPPIConfig(**d)


def refusal(kw, **shape):
    try:
        make_params(config(kw, **shape), IsaacGymConfig(), shape.get("nu", 3), shape.get("K", 256), [])
        return None
    except ValueError as e:
        return str(e)


def keys(names):
    kw = {}
    for n in names:
        kw.update(FEATURES[n])
    return kw


def test_the_record_covers_every_single_feature_and_every_compatible_pair():
    names = list(FEATURES)
    want = {(), *((n,) for n in names)}
    for a, b in itertools.combinations(names, 2):
        if all(FEATURES[b].get(k, v) == v for k, v in FEATURES[a].items()):
            want.add((a, b))
    assert set(REFUSED) == want


@pytest.mark.parametrize("names", list(REFUSED), ids=lambda n: "+".join(n) or "plain")
def test_make_params_refuses_what_it_refused_before(names):
    assert refusal(keys(names)) == REFUSED[names]


@pytest.mark.parametrize("case", list(LIMITS), ids=lambda c: "-".join(str(x) for x in c))
def test_size_limits(case):
    name, T, nu, P = case
    kw = keys([name])
    if P is not None:
        kw["control_knots"] = P
    why = refusal(kw, T=T, nu=nu)
    assert (why is not None) == (LIMITS[case] or case in LIMIT_FIXED), why
    assert why is None or "<=" in why, why


# ---- the table against the library -----------------------------------------------------------------------------------------------

K = 256
# parameter-block fields of each feature, switched on directly in a valid plain block
BLOCK = {
    "cem": dict(mode=2, n_elites=4, n_keep=1, elite_alpha=0.1),
    "smooth": dict(mode=3),
    "update_cov": dict(update_cov=1),
    "update_lambda": dict(update_lambda=1),
    "cov_full": dict(update_cov=1, cov_full=1),
    "cov_horizon": dict(update_cov=1, cov_horizon=1),
    "filter_u": dict(filter_u=1),
    "n_worlds": dict(n_worlds=2, risk_tail=1),
    "n_modes": dict(n_modes=2, mode_samples=K // 2),
    "control_knots": dict(control_knots=4, spline_degree=1),
    "constraint_mode": dict(constraint_mode=1, constraint_tol=0.0, constraint_lambda=1.0),
}
SAME_KEY = ({"cem", "smooth"}, {"cov_full", "cov_horizon"})       # one config key each: never on together


def block(names, T=12, nu=3, **fields):
    p = make_params(config({}, T=T, nu=nu, K=K), IsaacGymConfig(), nu, K, [])
    for n in names:
        fields = {**BLOCK[n], **fields}
    for k, v in fields.items():
        setattr(p, k, v)
    for j in range(nu):
        p.du_min[j], p.du_max[j] = -1e30, 1e30
    return p


def library():
    if not os.path.exists(backend.lib_path()):
        import __graft_entry__
        __graft_entry__.build()
    return backend.load_library()


def create(lib, p, nu):
    """mppib_create's return code: -1 refused by validate, 0 created (destroyed again), -2 admitted but no CUDA device."""
    h = C.c_void_p()
    rc = lib.mppib_create(C.byref(nu_model(nu)), C.byref(p), C.c_int32(0), C.byref(h))
    if rc == 0:
        lib.mppib_destroy(h)
    return rc


def block_cases():
    names = list(BLOCK)
    cases = [((), {})] + [((n,), {}) for n in names]
    cases += [((a, b), {}) for a, b in itertools.combinations(names, 2) if {a, b} not in SAME_KEY]
    for name, nu in (("cem", 8), ("smooth", 8), ("n_modes", 8)):                 # T*nu = 512 | 520
        cases += [((name,), dict(T=64, nu=nu)), ((name,), dict(T=65, nu=nu))]
    for name in ("cem", "smooth", "control_knots"):                               # T = 256 | 257
        cases += [((name,), dict(T=256, nu=1)), ((name,), dict(T=257, nu=1))]
    cases += [(("control_knots",), dict(T=64, nu=16, control_knots=32)), (("control_knots",), dict(T=64, nu=16, control_knots=33))]
    cases += [(("constraint_mode",), dict(T=216, nu=2)), (("constraint_mode",), dict(T=217, nu=2))]    # two FEASIBLE ring stages | one
    return cases


@pytest.mark.parametrize("names, shape", block_cases(), ids=lambda x: "+".join(x) if isinstance(x, tuple) else
                         "-".join(f"{k}{v}" for k, v in x.items()) or "base")
def test_the_table_and_the_library_refuse_the_same_blocks(names, shape):
    lib = library()
    nu = shape.get("nu", 3)
    p = block(names, **shape)
    why = mode_refusal(p, nu)
    rc = create(lib, p, nu)
    assert rc in (-1, 0, -2), lib.mppib_last_error().decode()
    assert (rc == -1) == (why is not None), (why, lib.mppib_last_error().decode())


def test_constrained_horizons_are_refused_where_the_feasible_ring_holds_one_stage():
    """Every (T, nu) with T <= 256 and T*nu <= 512 under constraint_mode: make_params, mppib_create (-1 refused, else admitted) and the
    restatement of the FEASIBLE K3 layout (synth_mppi.ws_layout) refuse the same shapes, which are nu = 2 with 217 <= T <= 256."""
    from synth_mppi import ws_layout
    lib = library()
    by_params, by_create, by_layout = set(), set(), set()
    for nu in range(1, 17):
        for T in range(1, min(256, 512 // nu) + 1):
            if refusal(FEATURES["constraint"], T=T, nu=nu) is not None:
                by_params.add((T, nu))
            rc = create(lib, block(["constraint_mode"], T=T, nu=nu), nu)
            assert rc in (-1, 0, -2), lib.mppib_last_error().decode()
            if rc == -1:
                by_create.add((T, nu))
                assert "ring stages" in lib.mppib_last_error().decode()
            if ws_layout(T, nu, "W", feasible=True) is None:
                by_layout.add((T, nu))
    assert by_params == by_create == by_layout == {(T, 2) for T in range(217, 257)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", [None, *BLOCK])
def test_set_anneal_refuses_a_schedule_exactly_when_the_table_does(name):
    import torch
    from mppi_isaac_b200.backend import CudaBackend, anneal_state_floats
    nu, T = 3, 12
    p = block([] if name is None else [name])
    be = CudaBackend("cuda:0")
    be.create(nu_model(nu), p)
    state = torch.ones(anneal_state_floats(T, 2), device="cuda:0")
    state[0] = 0.0
    why = mode_refusal(p, nu, anneal=True)
    try:
        if why is None:
            be.set_anneal(state, 2)
        else:
            with pytest.raises(RuntimeError, match="excludes"):
                be.set_anneal(state, 2)
    finally:
        be.destroy()
