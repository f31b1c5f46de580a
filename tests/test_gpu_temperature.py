"""-m gpu: the ESS-targeted temperature (`lambda_mode: ess`) on the device: the shard row and the ESS curve against float64 over T up to 256
and K not a multiple of 32, SIMPLE and MEAN, fixed, diagonal and full Sigma, non-finite tiles; the fused, split and explicit-row solves
agree bit for bit; lambda is the rule applied in float64 to the device's own curve, and the float64 oracle's lambda within the bound the
curve's rounding allows; graph replay; the library's refusals; and whole plans on the point robot and at the C2 shape against
TemperatureOracleBackend."""
import numpy as np
import pytest
import torch

import adaptive_full_oracle as adf
import temperature_oracle as tmo
from mppi_isaac_b200 import MPPIisaacPlanner
from mppi_isaac_b200.backend import CudaBackend
from mppi_isaac_b200.model.blob import ESS_GRID, ESS_ROW_FLOATS, ESS_STATE_FLOATS, ess_grid, make_params
from mppi_isaac_b200.objectives import PandaReachObjective, PointReachObjective
from mppi_isaac_b200.utils.config_store import IsaacGymConfig, MPPIConfig
from scenes import panda_cfg, point_cfg
from synth_mppi import corr_sigma, nu_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = float(np.finfo(np.float32).eps)


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(DEV)


def params(nu, T, K, mode="simple", cov=None, rho=0.05, lam=0.3, sigma=None):
    cfg = dict(num_samples=K, horizon=T, mppi_mode=mode, sampling_method="random", u_min=[-0.6], u_max=[0.6], lambda_=lam,
               rollout_var_discount=0.9, lambda_mode="ess", ess_target=rho,
               noise_sigma=(sigma if sigma is not None else 0.3 * np.eye(nu)).tolist())
    if cov is not None:
        cfg.update(update_cov=True, cov_type=cov)
    return make_params(MPPIConfig(**cfg), IsaacGymConfig(), nu, K, [])


class Case:
    """One handle with a registered distribution and temperature state, and seeded inputs."""

    def __init__(self, T, nu, K, mode="simple", cov=None, seed=0, rho=0.05):
        sigma = corr_sigma(nu) if cov == "full" else None
        self.p = params(nu, T, K, mode, cov, rho, sigma=sigma)
        self.T, self.nu, self.K = T, nu, K
        self.be = CudaBackend(DEV)
        self.be.create(nu_model(nu), self.p)
        rng = np.random.default_rng(seed)
        if cov == "full":
            self.dist_h = adf.make_dist(self.p.lambda_, sigma)
        else:
            d = np.diag(np.asarray(sigma if sigma is not None else 0.3 * np.eye(nu)))
            self.dist_h = np.concatenate([[self.p.lambda_], d * (1.0 + 0.5 * rng.random(nu) if cov == "diag" else 1.0)]).astype(np.float32)
        self.dist = dev(self.dist_h)
        self.be.set_distribution(self.dist)
        lam, inv = ess_grid(self.p.lambda_)
        st = np.zeros(ESS_STATE_FLOATS, np.float32)
        st[:ESS_GRID], st[ESS_GRID:2 * ESS_GRID] = lam, inv
        self.state = dev(st)
        self.be.set_temperature(self.state)
        self.cost_h = (rng.exponential(1.0, size=(T, K)) * (1.0 + 3.0 * rng.random(K))).astype(np.float32)
        self.x_h = rng.normal(scale=0.3, size=(T, nu, K)).astype(np.float32)
        self.U_h = rng.normal(scale=0.3, size=(T, nu)).astype(np.float32)
        self.row = torch.zeros(ESS_ROW_FLOATS, device=DEV)

    def upload(self):
        self.cost, self.x, self.U = dev(self.cost_h), dev(self.x_h), dev(self.U_h)

    def run(self, solve):
        self.upload()
        self.be.temperature(self.cost, self.x, self.U, self.row, solve=solve)
        torch.cuda.synchronize()
        return self.row.cpu().numpy()

    def scores(self):
        return tmo.scores(self.p, self.nu, self.cost_h, self.x_h, self.U_h, self.dist_h)

    def rtol(self):
        """Per grid point: the relative error of ESS_j the float32 sums of C_k and q_k allow (weights move by e^(+-d), ESS by e^(+-4d),
        d = max_k |delta a_jk|, with |delta C_k| <= (T + 2) eps sum_t |gamma^t c_tk| and the same for q over T*nu terms), plus the float32
        sums of the weights."""
        T = self.T
        g = float(self.p.gamma) ** np.arange(T)
        dC = (T + 2) * EPS * (np.abs(self.cost_h.astype(np.float64)) * g[:, None]).sum(0)
        dq = np.zeros(self.K)
        if self.p.mode == 0:
            h = self.U_h.astype(np.float64) @ tmo.sigma_inv(self.p, self.nu, self.dist_h).T
            dq = (T * self.nu + 2) * EPS * (np.abs(h.reshape(-1, 1)) * np.abs(self.x_h.reshape(T * self.nu, -1))).sum(0) + 4 * EPS * np.abs(h).sum()
        inv = ess_grid(self.p.lambda_)[1].astype(np.float64)
        C, q = self.scores()
        ok = np.isfinite(C) & np.isfinite(q)                         # invalid samples carry no weight on either side
        d = (inv[:, None] * dC[None, ok] + dq[None, ok]).max(1)
        return np.expm1(4 * d) + 1e-4

    def close(self):
        self.be.destroy()


SHAPES = [(1, 1, 4), (12, 3, 100), (30, 7, 1000), (64, 8, 4132), (256, 2, 5000), (32, 16, 13001), (16, 8, 65536)]


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("T, nu, K", SHAPES, ids=lambda v: str(v))
def test_row_and_curve_against_float64(T, nu, K, mode):
    c = Case(T, nu, K, mode)
    try:
        row = c.run(solve=False)
        N, ess = tmo.combine([tmo.from_f32(row)])
        C, q = c.scores()
        ref = tmo.shard_row(c.p, nu, c.cost_h, c.x_h, c.U_h, ess_grid(c.p.lambda_)[1], c.dist_h)
        assert N == ref[0] == K
        _, ess_ref = tmo.combine([ref])
        np.testing.assert_array_less(np.abs(ess / ess_ref - 1.0), c.rtol())
    finally:
        c.close()


@pytest.mark.parametrize("cov", [None, "diag", "full"])
@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
def test_sigma_kinds(cov, mode):
    c = Case(20, 4, 3000, mode, cov, seed=5)
    try:
        row = c.run(solve=False)
        _, ess = tmo.combine([tmo.from_f32(row)])
        _, ess_ref = tmo.combine([tmo.shard_row(c.p, 4, c.cost_h, c.x_h, c.U_h, ess_grid(c.p.lambda_)[1], c.dist_h)])
        np.testing.assert_array_less(np.abs(ess / ess_ref - 1.0), c.rtol())
    finally:
        c.close()


def test_non_finite_tiles():
    c = Case(10, 3, 2000, "simple", seed=7)
    try:
        c.cost_h[:, 256:512] = np.nan                                 # a whole tile
        c.cost_h[3, 700] = np.inf
        c.cost_h[5, 701] = -np.inf
        c.x_h[2, 1, 900] = np.nan                                     # q not finite
        c.cost_h[:, 1024:1280] = np.inf                               # another tile, with one valid sample left
        c.cost_h[:, 1100] = 1.0
        row = c.run(solve=True)
        N, ess = tmo.combine([tmo.from_f32(row)])
        ref = tmo.shard_row(c.p, 3, c.cost_h, c.x_h, c.U_h, ess_grid(c.p.lambda_)[1], c.dist_h)
        assert N == ref[0] == 2000 - 256 - 3 - 255
        _, ess_ref = tmo.combine([ref])
        np.testing.assert_array_less(np.abs(ess / ess_ref - 1.0), 1e-3 + c.rtol())
    finally:
        c.close()


def test_no_valid_sample_keeps_lambda():
    c = Case(8, 2, 300, "simple")
    try:
        c.cost_h[:] = np.nan
        c.dist[0] = 0.125
        row = c.run(solve=True)
        assert tmo.from_f32(row)[0] == 0
        assert float(c.dist[0]) == 0.125
        st = c.state.cpu().numpy()
        assert int(st[2 * ESS_GRID:2 * ESS_GRID + 1].view(np.int32)[0]) == 0 and st[2 * ESS_GRID + 1] == np.float32(0.125)
    finally:
        c.close()


def _lam_state(c):
    torch.cuda.synchronize()
    return float(c.dist[0]), c.state.cpu().numpy().copy()


@pytest.mark.parametrize("mode", ["simple", "halton-spline"])
@pytest.mark.parametrize("rho", [0.001, 0.05, 0.5, 1.0])
def test_fused_split_and_explicit_rows_agree_and_follow_the_rule(mode, rho):
    c = Case(24, 5, 7000, mode, seed=11, rho=rho)
    try:
        row = c.run(solve=True)
        lam_f, st_f = _lam_state(c)
        c.dist[0] = -1.0
        c.state[2 * ESS_GRID:] = 0.0
        c.run(solve=False)
        c.be.temperature_solve(c.row.view(1, -1), 1)
        lam_s, st_s = _lam_state(c)
        rows = c.row.clone().view(1, -1)
        c.dist[0] = -1.0
        c.state[2 * ESS_GRID:] = 0.0
        c.be.temperature_solve(rows, 1)
        lam_e, st_e = _lam_state(c)
        assert np.float32(lam_f).tobytes() == np.float32(lam_s).tobytes() == np.float32(lam_e).tobytes()
        np.testing.assert_array_equal(st_f, st_s)
        np.testing.assert_array_equal(st_f, st_e)
        # the rule in float64 on the device's own curve
        lam_grid = ess_grid(c.p.lambda_)[0].astype(np.float64)
        N = int(st_f[2 * ESS_GRID:2 * ESS_GRID + 1].view(np.int32)[0])
        ess_dev = st_f[2 * ESS_GRID + 2:].astype(np.float64)
        assert lam_f == pytest.approx(tmo.rule(ess_dev, N, float(np.float32(rho)), lam_grid, 0.0), rel=2e-6)
        # the float64 oracle: the rule is monotone in the curve, so its lambda lies between the rule of the device curve moved by the bound
        r = c.rtol()
        lo = tmo.rule(ess_dev * (1 + r), N, float(np.float32(rho)), lam_grid, 0.0)
        hi = tmo.rule(ess_dev * (1 - r), N, float(np.float32(rho)), lam_grid, 0.0)
        ref = tmo.rule(tmo.combine([tmo.shard_row(c.p, 5, c.cost_h, c.x_h, c.U_h, ess_grid(c.p.lambda_)[1], c.dist_h)])[1], N,
                       float(np.float32(rho)), lam_grid, 0.0)
        assert lo * (1 - 1e-6) <= ref <= hi * (1 + 1e-6), (lo, ref, hi)
    finally:
        c.close()


def test_explicit_rows_of_several_shards():
    """G rows of three shards combined by the solve entry: the curve of the whole set, in rank order."""
    cs = [Case(16, 3, K, "simple", seed=20) for K in (1000, 804, 1200)]
    try:
        rows = torch.stack([torch.as_tensor(c.run(solve=False)) for c in cs]).to(DEV).contiguous()
        cs[0].be.temperature_solve(rows, 3)
        lam, st = _lam_state(cs[0])
        N, ess = tmo.combine([tmo.from_f32(r) for r in rows.cpu().numpy()])
        assert int(st[2 * ESS_GRID:2 * ESS_GRID + 1].view(np.int32)[0]) == N == 3004
        np.testing.assert_allclose(st[2 * ESS_GRID + 2:], ess, rtol=1e-5)
        lam_grid = ess_grid(cs[0].p.lambda_)[0].astype(np.float64)
        assert lam == pytest.approx(tmo.rule(st[2 * ESS_GRID + 2:].astype(np.float64), N, float(np.float32(0.05)), lam_grid, 0.0), rel=2e-6)
    finally:
        for c in cs:
            c.close()


def test_graph_replay():
    c = Case(20, 4, 3000, "simple", seed=3)
    try:
        c.upload()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            c.be.temperature(c.cost, c.x, c.U, c.row, solve=True)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            c.be.temperature(c.cost, c.x, c.U, c.row, solve=True)
        for seed in (1, 2, 3):
            new = np.random.default_rng(seed).exponential(2.0, size=c.cost_h.shape).astype(np.float32)
            c.cost.copy_(dev(new))
            g.replay()
            lam_g, st_g = _lam_state(c)
            c.be.temperature(c.cost, c.x, c.U, c.row, solve=True)
            lam_e, st_e = _lam_state(c)
            assert lam_g == lam_e
            np.testing.assert_array_equal(st_g, st_e)
    finally:
        c.close()


def test_refusals():
    c = Case(8, 2, 256, "simple")
    try:
        c.upload()
        c.be.set_temperature(None)
        part = torch.zeros(2 + 16, device=DEV)
        with pytest.raises(RuntimeError, match="temperature state"):
            c.be.reduce(c.cost, c.x, c.U, part)
        with pytest.raises(RuntimeError, match="temperature state"):
            c.be.temperature(c.cost, c.x, c.U, c.row)
        c.be.set_temperature(c.state)
        c.be.set_distribution(None)
        with pytest.raises(RuntimeError, match="distribution"):
            c.be.finalize(part.view(1, -1), 1, c.U, torch.zeros(2, device=DEV), torch.zeros(2, device=DEV))
    finally:
        c.close()


# ---- whole plans -----------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode, sampling", [("simple", "random"), ("simple", "halton"), ("halton-spline", "halton")])
def test_point_robot_plans_against_the_oracle(mode, sampling):
    """Five graph-replayed plans.  Every plan re-chooses lambda from a float32 curve on the device and a float64 one in the oracle, so
    the two temperatures differ in the last digits and the difference carries into U from plan to plan: the bound is looser than the
    fixed-lambda plans' 2e-4 and the run shorter."""
    kw = dict(K=256, T=12, mppi_mode=mode, sampling_method=sampling, lambda_mode="ess", ess_target=0.05, filter_u=True)
    gpu = MPPIisaacPlanner(point_cfg(device=DEV, **kw), PointReachObjective())
    cpu = MPPIisaacPlanner(point_cfg(device="cpu", **kw), PointReachObjective(), backend=tmo.TemperatureOracleBackend())
    for _ in range(5):
        a = gpu.compute_action([0.1, 0.0, 0.0], [0.0] * 3).cpu().numpy()
        b = cpu.compute_action([0.1, 0.0, 0.0], [0.0] * 3).numpy()
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-3)
        assert float(gpu.mppi.current_lambda) == pytest.approx(float(cpu.mppi.current_lambda), rel=1e-3)
        assert gpu.mppi.valid_samples == cpu.mppi.valid_samples


def test_c2_shape_plans_against_the_oracle():
    q = [0.0, -0.94, 0.0, -2.8, 0.0, 1.8675, 0.0]
    kw = dict(K=1000, lambda_mode="ess", ess_target=0.05)
    gpu = MPPIisaacPlanner(panda_cfg(device=DEV, **kw), PandaReachObjective())
    cpu = MPPIisaacPlanner(panda_cfg(device="cpu", **kw), PandaReachObjective(), backend=tmo.TemperatureOracleBackend())
    for _ in range(3):
        a = gpu.compute_action(q, [0.0] * 7).cpu().numpy()
        b = cpu.compute_action(q, [0.0] * 7).numpy()
        np.testing.assert_allclose(a, b, rtol=0, atol=2e-4)
        assert float(gpu.mppi.current_lambda) == pytest.approx(float(cpu.mppi.current_lambda), rel=1e-3)
