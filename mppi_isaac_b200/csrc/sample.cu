// sample.cu -- K1: per-sample Gaussian control-noise draw and clamp (north-star item (i)).
// Replaces mppi_torch's `noise_dist.sample((K, T))` + `_bound_action` + null / prior rows
// (external dependency mppi_torch@75e17e8, call site mppiisaac/planner/mppi_isaac.py:43-49,113;
// spec SURVEY.md 8(a) M4/M5).
//
// Counter-based Philox-4x32-10: key = (seed_lo, seed_hi ^ plan_lo), counter = (GLOBAL sample index,
// t, block, plan_hi), so the stream is invariant to how the K samples are sharded over GPUs.
// One thread per (t, k); k is the innermost index of every array, so the nu stores of a warp are
// nu fully coalesced 128-byte lines.  HBM-write bound (2 * 4 * K*T*nu bytes).
#include "common.cuh"

namespace {

// The Philox key of a plan: (seed_lo, seed_hi ^ plan_lo), with plan_hi the last counter word; plan = plan_idx + *plan_ctr (nullable),
// so that a captured graph draws fresh noise on every replay.
struct PhiloxKey { uint32_t k0, k1, plan_hi; };
__device__ __forceinline__ PhiloxKey philox_key(uint32_t key0, uint32_t seed_hi, uint64_t plan_idx, const uint32_t* __restrict__ plan_ctr) {
    const uint64_t plan = plan_idx + (plan_ctr ? (uint64_t)*plan_ctr : 0ull);
    return {key0, seed_hi ^ (uint32_t)plan, (uint32_t)(plan >> 32)};
}
// the white draws z[0..4) of controls 4*blk .. 4*blk + 3 of control sample kc at step t
__device__ __forceinline__ void philox_gauss4(const PhiloxKey& key, uint32_t kc, int t, int blk, float* z) {
    const uint4 r = philox4x32_10<10>(make_uint4(kc, (uint32_t)t, (uint32_t)blk, key.plan_hi), key.k0, key.k1);
    box_muller(r.x, r.y, z[0], z[1]);
    box_muller(r.z, r.w, z[2], z[3]);
}

// The special rows of global sample kg, tested on its control sample (n_worlds keying): the last control sample of the k_total is the
// null action when enabled, the one before it takes prior_row when one is given.
struct SpecialRows { bool null, prior; };
__device__ __forceinline__ SpecialRows special_rows(const MppibParams& p, uint32_t kg, uint32_t k_total, bool has_prior) {
    const uint32_t kc = sample_control(kg, p.n_worlds), kc_total = sample_control(k_total, p.n_worlds);
    return {p.sample_null_action && kc == kc_total - 1, has_prior && kc == kc_total - 2};
}

// The tail of every K1 but smooth at (t, j) of sample k: a = U + noise (0 on the null row) clamped to [u_min, u_max], prior_row on the
// prior row, stored with noise := a - u.
// The clamp of that tail: 0 on the null row, then [u_min, u_max] (spline MPPI applies it to the knots).
__device__ __forceinline__ float clamp_action(const MppibParams& p, int j, float a, SpecialRows rows) {
    if (rows.null) a = 0.f;
    return fminf(fmaxf(a, p.u_min[j]), p.u_max[j]);
}
__device__ __forceinline__ void clamp_store(const MppibParams& p, int nu, int t, int j, int k, float a, float u, SpecialRows rows,
                                            const float* __restrict__ prior_row, float* __restrict__ actions, float* __restrict__ noise) {
    a = clamp_action(p, j, a, rows);
    if (rows.prior) a = prior_row[t * nu + j];
    const size_t idx = ((size_t)t * nu + j) * p.K + k;
    actions[idx] = a;
    if (noise) noise[idx] = a - u;
}

// The control-space colour of one (t, k) in front of clamp_store.  FIXED: noise_j = sum_{i <= j} L0[j][i] z_i with the fixed Sigma's
// Cholesky factor, summed from i = 0 upwards; DIAG (adaptive MPPI with update_cov): sqrt(cov_j) z_j with cov = dist[1..nu], the live
// diagonal covariance; FULL (update_cov with cov_full): the live lower Cholesky factor L = dist[1 + nu*nu ..] in the same order.  LIB: z
// is a column of the noise library, which mppib_noise_library has coloured by L0 already (FIXED) or left white (DIAG / FULL).
// Annealed MPPI (srow = the s row of the iteration, FIXED only): noise_j := s[t] noise_j, one rounded multiplication, so a schedule of
// ones changes no bit.
// The FIXED colour of control j: sum_{i <= j} L0[j][i] z_i, summed from i = 0 upwards.
__device__ __forceinline__ float fixed_colour(const MppibParams& p, int nu, const float (&z)[MPPIB_MAX_NU], int j) {
    float n = 0.f;
#pragma unroll
    for (int i = 0; i < MPPIB_MAX_NU; ++i)
        if (i <= j) n += p.sigma_chol[j * nu + i] * z[i];
    return n;
}

template <Draw D, bool LIB = false>
__device__ __forceinline__ void colour_clamp_store(const MppibParams& p, int nu, const float (&z)[MPPIB_MAX_NU], int t, int k, SpecialRows rows,
                                                   const float* __restrict__ U, const float* __restrict__ prior_row, float* __restrict__ actions,
                                                   float* __restrict__ noise, const float* __restrict__ dist, const float* __restrict__ srow) {
#pragma unroll
    for (int j = 0; j < MPPIB_MAX_NU; ++j) {
        if (j >= nu) break;
        float n = 0.f;
        if constexpr (D == DRAW_DIAG) {
            n = sqrtf(dist[1 + j]) * z[j];
        } else if constexpr (D == DRAW_FULL) {
            const float* Ld = dist + 1 + nu * nu;
#pragma unroll
            for (int i = 0; i < MPPIB_MAX_NU; ++i)
                if (i <= j) n += Ld[j * nu + i] * z[i];
        } else if constexpr (LIB) {
            n = z[j];
        } else {
            n = fixed_colour(p, nu, z, j);
            if (srow) n = __fmul_rn(srow[t], n);
        }
        const float u = U[t * nu + j];
        clamp_store(p, nu, t, j, k, u + n, u, rows, prior_row, actions, noise);
    }
}

// One thread per (t, k) for the per-step colours D = FIXED, DIAG, FULL.  The white draws are the Philox draws of counter (global
// sample, t, block) -- with n_worlds = R > 1 the control sample kg / R replaces the global sample -- or, LIB, column k of the noise
// library Z.  With n_modes > 1 the sample is drawn around its mode's sequence (sample_mode), the counter stays the global sample;
// n_modes > 1 excludes update_cov, so only FIXED carries the mode offset.  anneal (annealed MPPI, FIXED only; nullable): the
// registered schedule of anneal_n iterations, whose s row scales the noise.
template <Draw D, bool LIB>
__global__ void __launch_bounds__(128)
mppib_sample_kernel(const __grid_constant__ MppibParams p, int nu, uint32_t key0, uint32_t seed_hi, uint64_t plan_idx,
                    const uint32_t* __restrict__ plan_ctr, uint32_t k_offset, uint32_t k_total, const float* __restrict__ U,
                    const float* __restrict__ prior_row, const float* __restrict__ Z, float* __restrict__ actions, float* __restrict__ noise,
                    const float* __restrict__ dist, const float* __restrict__ anneal, int anneal_n) {
    const int K = p.K;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int t = blockIdx.y;
    if (k >= K) return;
    const uint32_t kg = k_offset + (uint32_t)k;
    float z[MPPIB_MAX_NU];
    if constexpr (LIB) {
#pragma unroll
        for (int i = 0; i < MPPIB_MAX_NU; ++i) z[i] = i < nu ? Z[((size_t)t * nu + i) * K + k] : 0.f;
    } else {
        const PhiloxKey key = philox_key(key0, seed_hi, plan_idx, plan_ctr);
        const uint32_t kc = sample_control(kg, p.n_worlds);
#pragma unroll
        for (int blk = 0; blk < MPPIB_MAX_NU / 4; ++blk)
            if (blk * 4 < nu) philox_gauss4(key, kc, t, blk, z + 4 * blk);
    }
    const float* Um = U;
    if constexpr (D == DRAW_FIXED) Um += (size_t)sample_mode(kg, p) * (p.T * nu);   // n_modes > 1 (fixed Sigma only)
    const float* srow = (D == DRAW_FIXED && anneal) ? anneal_row(anneal, anneal_n, p.T, false) : nullptr;
    colour_clamp_store<D, LIB>(p, nu, z, t, k, special_rows(p, kg, k_total, prior_row != nullptr), Um, prior_row, actions, noise, dist, srow);
}

// The white Philox draws of a tile of S samples [k0, k0 + S) to shared memory, zs[(t*nu + i) * S + sample]: the draws of the
// fixed-Sigma kernel (counter (control sample of n_worlds = R, t, block)), spread over the CTA.
template <int S>
__device__ __forceinline__ void stage_white_tile(float* zs, int T, int nu, int k0, const PhiloxKey& key, uint32_t k_offset, int R) {
    const int nblk = (nu + 3) / 4;
    for (int idx = threadIdx.x; idx < S * T * nblk; idx += blockDim.x) {
        const int sl = idx % S, rest = idx / S, blk = rest % nblk, t = rest / nblk;
        float z[4];
        philox_gauss4(key, sample_control(k_offset + (uint32_t)(k0 + sl), R), t, blk, z);
#pragma unroll
        for (int e = 0; e < 4; ++e)
            if (4 * blk + e < nu) zs[(t * nu + 4 * blk + e) * S + sl] = z[e];
    }
}

// CEM (mppi_mode: cem): the colour of one (t, k) in front of clamp_store with the per-step diagonal sigma[t][j] of the CEM state
// (include/mppib.h): a = U + sigma (.) w, the product rounded on its own as the FIXED colour rounds L0[j][j] z_j, so a diagonal Sigma
// with sigma = sigma0 draws what FIXED draws, bit for bit.  Once the state holds elites, global rows k_total - 3 - e (e < n_keep) take
// elites[e][t + off] instead, off = the state's carry offset; a row whose t + off = T keeps its draw.
__device__ __forceinline__ void cem_clamp_store(const MppibParams& p, int nu, const float (&w)[MPPIB_MAX_NU], int t, int k, uint32_t kg,
                                                uint32_t k_total, SpecialRows rows, const float* __restrict__ U,
                                                const float* __restrict__ prior_row, float* __restrict__ actions, float* __restrict__ noise,
                                                const float* __restrict__ state) {
    const int NR = p.T * nu;
    const float* sig = state + 2 + p.n_elites;
    const float* el = sig + NR;
    const uint32_t e = k_total - 3u - kg;                                     // carried row e when kg = k_total - 3 - e
    const int ts = t + (int)state[0];
    const bool carried = state[1] != 0.f && kg + 3u <= k_total && e < (uint32_t)p.n_keep && ts < p.T;
#pragma unroll
    for (int j = 0; j < MPPIB_MAX_NU; ++j) {
        if (j >= nu) break;
        const float u = U[t * nu + j];
        const float a = carried ? el[(size_t)e * NR + ts * nu + j] : u + __fmul_rn(sig[t * nu + j], w[j]);
        clamp_store(p, nu, t, j, k, a, u, rows, prior_row, actions, noise);
    }
}

// COLORED (sampling_method: colored): time-correlated noise w[t][i] = sum_{t' <= t} L_b[t][t'] z[t'][i] over the white draws of
// the fixed-Sigma kernel, with L_b = Lt[T][T] the lower Cholesky factor of the power-law temporal covariance, then the colour step
// of D: colour_clamp_store (FIXED L0, or DIAG / FULL the live adaptive ones) or cem_clamp_store (CEM).  A CTA of 128 threads owns a
// tile of CL_S = 32 samples, lane = sample: the tile's white draws go to shared memory, then warp w takes the row pairs (t, T-1-t),
// t = w, w + 4, ..., so that every warp sums about the same number of terms and every shared-memory load of z feeds two rows.  The
// rows of L_b are read with warp-uniform loads (one L1 line per row segment, shared by all CTAs).  Both sums run in a fixed order
// (t' and i from 0 upwards), so a sample's noise depends only on its global index; with L_b = I the temporal sum adds only exact
// zeros before z[t][i] itself, and the result is that of mppib_sample_kernel bit for bit.
constexpr int CL_S = 32;            // samples per CTA
constexpr int CL_MAX_T = 256;
constexpr int CL_MAX_N = 512;       // T*nu: the tile's draws take CL_MAX_N * CL_S * 4 = 64 KB of shared memory

// The FIXED instantiation asks for 8 CTAs per SM: with the annealing scale it takes 64 registers (78 unbounded, 63 without the
// scale) and spills nothing; 0 leaves the other instantiations as the compiler allocates them.
template <Draw D>
__global__ void __launch_bounds__(128, D == DRAW_FIXED ? 8 : 0)
mppib_sample_colored_kernel(const __grid_constant__ MppibParams p, int nu, uint32_t key0, uint32_t seed_hi, uint64_t plan_idx,
                            const uint32_t* __restrict__ plan_ctr, uint32_t k_offset, uint32_t k_total, const float* __restrict__ U,
                            const float* __restrict__ prior_row, const float* __restrict__ Lt, float* __restrict__ actions,
                            float* __restrict__ noise, const float* __restrict__ dist, const float* __restrict__ anneal, int anneal_n) {
    extern __shared__ __align__(16) float cs[];
    const int K = p.K, T = p.T;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int k0 = blockIdx.x * CL_S, k = k0 + lane;
    const uint32_t kg = k_offset + (uint32_t)k;
    const SpecialRows rows = special_rows(p, kg, k_total, prior_row != nullptr);
    stage_white_tile<CL_S>(cs, T, nu, k0, philox_key(key0, seed_hi, plan_idx, plan_ctr), k_offset, p.n_worlds);
    __syncthreads();
    const float* Um = U;
    if constexpr (D == DRAW_FIXED) Um += (size_t)sample_mode(kg, p) * (T * nu);   // n_modes > 1 (fixed Sigma only)
    const float* srow = (D == DRAW_FIXED && anneal) ? anneal_row(anneal, anneal_n, T, false) : nullptr;   // annealed MPPI
    const float* zl = cs + lane;
    for (int tl = warp; tl < (T + 1) / 2; tl += 4) {
        const int th = T - 1 - tl;                                            // th >= tl; th == tl for the middle row of an odd T
        const float* Llo = Lt + (size_t)tl * T;
        const float* Lhi = Lt + (size_t)th * T;
        float wl[MPPIB_MAX_NU], wh[MPPIB_MAX_NU];
#pragma unroll
        for (int i = 0; i < MPPIB_MAX_NU; ++i) { wl[i] = 0.f; wh[i] = 0.f; }
        int tp = 0;
        for (; tp <= tl; ++tp) {
            const float a = __ldg(Llo + tp), b = __ldg(Lhi + tp);
            const float* zr = zl + tp * nu * CL_S;
#pragma unroll
            for (int i = 0; i < MPPIB_MAX_NU; ++i) {
                if (i >= nu) break;
                const float zv = zr[i * CL_S];
                wl[i] = fmaf(a, zv, wl[i]);
                wh[i] = fmaf(b, zv, wh[i]);
            }
        }
        for (; tp <= th; ++tp) {
            const float b = __ldg(Lhi + tp);
            const float* zr = zl + tp * nu * CL_S;
#pragma unroll
            for (int i = 0; i < MPPIB_MAX_NU; ++i) {
                if (i >= nu) break;
                wh[i] = fmaf(b, zr[i * CL_S], wh[i]);
            }
        }
        if (k >= K) continue;
        if constexpr (D == DRAW_CEM) {
            cem_clamp_store(p, nu, wl, tl, k, kg, k_total, rows, U, prior_row, actions, noise, dist);
            if (th != tl) cem_clamp_store(p, nu, wh, th, k, kg, k_total, rows, U, prior_row, actions, noise, dist);
        } else {
            colour_clamp_store<D>(p, nu, wl, tl, k, rows, Um, prior_row, actions, noise, dist, srow);
            if (th != tl) colour_clamp_store<D>(p, nu, wh, th, k, rows, Um, prior_row, actions, noise, dist, srow);
        }
    }
}

template <Draw D>
int launch_sample_colored_t(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                            const float* U, const float* prior_row, const float* Lt, float* actions, float* noise, cudaStream_t s) {
    const int K = c->params.K, T = c->params.T, nu = c->model.nu;
    const int smem = (int)sizeof(float) * T * nu * CL_S;
    if (int rc = ensure_smem<mppib_sample_colored_kernel<D>>(c->device, smem)) return rc;
    mppib_sample_colored_kernel<D><<<(K + CL_S - 1) / CL_S, 128, smem, s>>>(c->params, nu, (uint32_t)seed, (uint32_t)(seed >> 32), plan_idx, plan_ctr,
                                                                            k_offset, k_total, U, prior_row, Lt, actions, noise,
                                                                            D == DRAW_FIXED ? nullptr : c->dist,
                                                                            D == DRAW_FIXED ? c->anneal : nullptr, c->anneal_n);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// SMOOTH (mppi_mode: smooth): the sampled derivative v = clamp(U + L0 z, du_min, du_max) is integrated over the horizon from the last
// executed action a_prev = state[0..nu), a_t = clamp(fmaf(v_t, dt, a_{t-1}), u_min, u_max), and only actions and the applied derivative
// noise = v - U (or (a_t - a_{t-1})/dt - U where the action clamp bound) are stored.  A CTA of 128 threads owns a tile of SM_S = 32
// samples: all threads draw the tile's white draws into shared memory (the counters of the fixed-Sigma kernel), then lane = sample and
// warp w carries the prefix of the controls j = w, w + 4, ... serially in t.  The colour sums i from 0 upwards as colour_clamp_store
// does, so without a binding action clamp the noise is mppib_sample_kernel's bit for bit when that kernel clamps to du_min / du_max.
constexpr int SM_S = 32;            // samples per CTA
constexpr int SM_MAX_N = 512;       // T*nu: the tile's draws take SM_MAX_N * SM_S * 4 = 64 KB of shared memory

__global__ void __launch_bounds__(128)
mppib_sample_smooth_kernel(const __grid_constant__ MppibParams p, int nu, uint32_t key0, uint32_t seed_hi, uint64_t plan_idx,
                           const uint32_t* __restrict__ plan_ctr, uint32_t k_offset, uint32_t k_total, const float* __restrict__ U,
                           float* __restrict__ actions, float* __restrict__ noise, const float* __restrict__ state) {
    extern __shared__ __align__(16) float zs[];
    const int K = p.K, T = p.T;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int k0 = blockIdx.x * SM_S, k = k0 + lane;
    stage_white_tile<SM_S>(zs, T, nu, k0, philox_key(key0, seed_hi, plan_idx, plan_ctr), k_offset, 1);
    __syncthreads();
    if (k >= K) return;
    const bool is_null = special_rows(p, k_offset + (uint32_t)k, k_total, false).null;
    const float dt = p.dt;
    const float* zl = zs + lane;
    for (int j = warp; j < nu; j += 4) {
        const float lo = p.u_min[j], hi = p.u_max[j], dlo = p.du_min[j], dhi = p.du_max[j];
        const float* Lj = p.sigma_chol + j * nu;
        float a = state[j];
        for (int t = 0; t < T; ++t) {
            const float* zr = zl + t * nu * SM_S;
            float n = 0.f;
            for (int i = 0; i <= j; ++i) n += Lj[i] * zr[i * SM_S];
            const float u = U[t * nu + j];
            const float v = is_null ? 0.f : fminf(fmaxf(u + n, dlo), dhi);
            const float ah = fmaf(v, dt, a);
            const float an = fminf(fmaxf(ah, lo), hi);
            const size_t idx = ((size_t)t * nu + j) * K + k;
            actions[idx] = an;
            if (noise) noise[idx] = (an == ah ? v : (an - a) / dt) - u;
            a = an;
        }
    }
}

// SPLINE (control_knots = P > 0, include/mppib.h "Spline MPPI"): K1 over the knots.  A CTA of 128 threads owns a tile of SP_S = 32
// samples, lane = sample: warp w draws knots p = w, w + 4, ... with the Philox counters of mppib_sample (p in the t slot), colours them
// with L0 (fixed_colour), clamps them (clamp_action, the null row included) into the tile's theta~ in shared memory and stores
// xk = theta~ - theta (SIMPLE) or theta~ (MEAN); then warp w interpolates steps t = w, w + 4, ... with the table's row t (spline_apply)
// and clamps the sum to [u_min, u_max].
// With d = 1 and P = T every row is one weight 1.0, and actions / xk equal mppib_sample's actions / noise bit for bit.
constexpr int SP_S = 32;            // samples per CTA
constexpr int SP_MAX_N = 512;       // P*nu: the tile's knots take SP_MAX_N * SP_S * 4 = 64 KB of shared memory

__global__ void __launch_bounds__(128)
mppib_sample_spline_kernel(const __grid_constant__ MppibParams p, int nu, uint32_t key0, uint32_t seed_hi, uint64_t plan_idx,
                           const uint32_t* __restrict__ plan_ctr, uint32_t k_offset, uint32_t k_total, const float* __restrict__ U,
                           const float* __restrict__ spline, float* __restrict__ actions, float* __restrict__ xk) {
    extern __shared__ __align__(16) float ths[];                             // [P*nu][SP_S] theta~ of the tile
    const int K = p.K, T = p.T, P = p.control_knots, S = spline_row_floats(p.spline_degree);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int k = blockIdx.x * SP_S + lane;
    const uint32_t kg = k_offset + (uint32_t)k;
    const PhiloxKey key = philox_key(key0, seed_hi, plan_idx, plan_ctr);
    const SpecialRows rows = special_rows(p, kg, k_total, false);
    const bool mean = p.mode == MPPIB_MODE_MEAN;
    for (int pk = warp; pk < P; pk += 4) {
        float z[MPPIB_MAX_NU];
#pragma unroll
        for (int blk = 0; blk < MPPIB_MAX_NU / 4; ++blk)
            if (blk * 4 < nu) philox_gauss4(key, kg, pk, blk, z + 4 * blk);
#pragma unroll
        for (int j = 0; j < MPPIB_MAX_NU; ++j) {
            if (j >= nu) break;
            const float th = U[pk * nu + j];
            const float a = clamp_action(p, j, th + fixed_colour(p, nu, z, j), rows);
            ths[(pk * nu + j) * SP_S + lane] = a;
            if (k < K) xk[((size_t)pk * nu + j) * K + k] = mean ? a : a - th;
        }
    }
    __syncthreads();
    if (k >= K) return;
    for (int t = warp; t < T; t += 4) {
        const float* row = spline + t * S;
        for (int j = 0; j < nu; ++j)   // the float32 weights sum to 1 only up to rounding: the clamp keeps a_t in the bounds
            actions[((size_t)t * nu + j) * K + k] = fminf(fmaxf(spline_apply(row, ths + j * SP_S + lane, nu * SP_S), p.u_min[j]), p.u_max[j]);
    }
}

// generalised Halton: radical inverse of `index` in base b with multiplicative digit scrambling (digit -> mult * digit mod b)
__device__ __forceinline__ float halton(uint32_t index, uint32_t base, uint32_t mult) {
    const float inv_b = 1.0f / (float)base;
    float f = inv_b, r = 0.f;
    while (index > 0u) {
        const uint32_t digit = index % base;
        r += (float)((digit * mult) % base) * f;
        index /= base;
        f *= inv_b;
    }
    return r;
}

constexpr int MAX_KNOTS = 32;

// one thread per sample k: Gaussian knots (n_knots x nu) -> coloured -> spline-interpolated to T points.  WHITE (draws DIAG, FULL
// and HORIZON of adaptive MPPI with update_cov): identity colour, the library sampler colours by the live distribution on every plan.
template <bool WHITE>
__global__ void __launch_bounds__(128)
mppib_noise_library_kernel(const __grid_constant__ MppibParams p, int nu, uint32_t k_offset, uint32_t k_total,
                           const int32_t* __restrict__ tab, const float* __restrict__ B, int n_knots, float* __restrict__ Z) {
    const int K = p.K, T = p.T;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    const uint32_t kc = sample_control(k_offset + (uint32_t)k, p.n_worlds);
    const bool null_row = special_rows(p, k_offset + (uint32_t)k, k_total, false).null;
    const int nd = n_knots * nu;
    for (int j = 0; j < nu; ++j) {
        // coloured knots of control dimension j:  c[n] = sum_i L[j][i] z[n][i]
        float cn[MAX_KNOTS];
        for (int n = 0; n < n_knots; ++n) {
            float acc = 0.f;
            for (int i = WHITE ? j : 0; i <= j; ++i) {
                const int d = n * nu + i;
                const float u = halton(kc + 1u, (uint32_t)tab[d], (uint32_t)tab[nd + d]);
                const float zn = 1.41421356237f * erfinvf(2.0f * u - 1.0f);
                acc += WHITE ? zn : p.sigma_chol[j * nu + i] * zn;
            }
            cn[n] = acc;
        }
        for (int t = 0; t < T; ++t) {
            float z = 0.f;
            for (int n = 0; n < n_knots; ++n) z += B[t * n_knots + n] * cn[n];
            Z[((size_t)t * nu + j) * K + k] = null_row ? 0.f : z;
        }
    }
}

// HORIZON (update_cov with cov_horizon, n = T*nu <= 256): noise = L_H z over the whole n-vector of a sample, with L_H =
// dist[1 + n*n ..] the live lower Cholesky factor of Sigma_H, rows and columns ordered (t, j) like U.  A CTA of 128 threads owns a
// tile of HZ_S = 64 samples: the white draws of the tile go to shared memory first -- the Philox draws of the fixed-Sigma kernel
// (counter (global sample, t, block)) or, LIB, the white library Z -- then L_H is staged 32 rows at a time, transposed, and every
// warp multiplies 8 of those rows with the tile: lane = samples lane and lane + 32, an 8 x 2 register block, two broadcast LDS.128
// of L_H and two LDS of z per 16 FFMA.  The sum over columns runs from 0 upwards (the zeros above the diagonal add nothing), so a
// sample's noise depends only on its global index.  Then clamp_store, as in the other K1 variants.
constexpr int HZ_S = 64;        // samples per CTA
constexpr int HZ_LP = 36;       // padded row of the transposed L_H panel (16-byte aligned, 4-way store conflicts at most)

__host__ __device__ __forceinline__ int horizon_smem_bytes(int n) { return (int)sizeof(float) * n * (HZ_S + HZ_LP); }

template <bool LIB>
__global__ void __launch_bounds__(128)
mppib_sample_horizon_kernel(const __grid_constant__ MppibParams p, int nu, uint32_t key0, uint32_t seed_hi, uint64_t plan_idx,
                            const uint32_t* __restrict__ plan_ctr, uint32_t k_offset, uint32_t k_total, const float* __restrict__ U,
                            const float* __restrict__ prior_row, const float* __restrict__ Z, float* __restrict__ actions, float* __restrict__ noise,
                            const float* __restrict__ dist) {
    extern __shared__ __align__(16) float hs[];
    const int K = p.K, T = p.T, n = T * nu;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int k0 = blockIdx.x * HZ_S;
    float* zs = hs;                       // [n][HZ_S] white draws of the tile
    float* Lt = hs + n * HZ_S;            // [n][HZ_LP] Lt[c][i] = L_H[r0 + i][c] of the current 32-row panel
    if (LIB) {
        for (int idx = tid; idx < n * HZ_S; idx += blockDim.x) {
            const int r = idx / HZ_S, sl = idx % HZ_S, k = k0 + sl;
            zs[idx] = k < K ? Z[(size_t)r * K + k] : 0.f;
        }
    } else {
        stage_white_tile<HZ_S>(zs, T, nu, k0, philox_key(key0, seed_hi, plan_idx, plan_ctr), k_offset, 1);
    }
    const float* Ld = dist + 1 + (size_t)n * n;
    for (int r0 = 0; r0 < n; r0 += 32) {
        const int cmax = min(n, r0 + 32);                                     // columns of the panel that can be non-zero
        __syncthreads();                                                      // z staged / the previous panel consumed
        for (int idx = tid; idx < 32 * cmax; idx += blockDim.x) {
            const int i = idx / cmax, c = idx % cmax;
            Lt[c * HZ_LP + i] = r0 + i < n ? Ld[(size_t)(r0 + i) * n + c] : 0.f;
        }
        __syncthreads();
        const int rb = r0 + warp * 8;
        if (rb >= n) continue;
        float acc0[8], acc1[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
        const int cend = min(n, rb + 8);
        for (int c = 0; c < cend; ++c) {
            const float za = zs[c * HZ_S + lane], zb = zs[c * HZ_S + 32 + lane];
            const float4 la = *reinterpret_cast<const float4*>(Lt + c * HZ_LP + warp * 8);
            const float4 lb = *reinterpret_cast<const float4*>(Lt + c * HZ_LP + warp * 8 + 4);
            const float lv[8] = {la.x, la.y, la.z, la.w, lb.x, lb.y, lb.z, lb.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) { acc0[i] = fmaf(lv[i], za, acc0[i]); acc1[i] = fmaf(lv[i], zb, acc1[i]); }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = rb + i;
            if (r >= n) break;
            const int t = r / nu, j = r % nu;
            const float u = U[r];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int k = k0 + lane + 32 * h;
                if (k >= K) continue;
                clamp_store(p, nu, t, j, k, u + (h ? acc1[i] : acc0[i]), u, special_rows(p, k_offset + (uint32_t)k, k_total, prior_row != nullptr),
                            prior_row, actions, noise);
            }
        }
    }
}

template <bool LIB>
int launch_sample_horizon_t(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                            const float* U, const float* prior_row, const float* Z, float* actions, float* noise, cudaStream_t s) {
    const int K = c->params.K, n = c->params.T * c->model.nu;
    const int smem = horizon_smem_bytes(n);
    if (int rc = ensure_smem<mppib_sample_horizon_kernel<LIB>>(c->device, smem)) return rc;
    mppib_sample_horizon_kernel<LIB><<<(K + HZ_S - 1) / HZ_S, 128, smem, s>>>(c->params, c->model.nu, (uint32_t)seed, (uint32_t)(seed >> 32), plan_idx,
                                                                              plan_ctr, k_offset, k_total, U, prior_row, Z, actions, noise, c->dist);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// mppib_sample (LIB = false: the Philox draws) and mppib_sample_library (LIB: the draws are the library Z) for the handle's draw;
// k1_admit has refused CEM and SMOOTH.
template <bool LIB>
int launch_sample_t(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                    const float* U, const float* prior_row, const float* Z, float* actions, float* noise, cudaStream_t s) {
    const int nu = c->model.nu;
    const uint32_t key0 = (uint32_t)seed, seed_hi = (uint32_t)(seed >> 32);
    const dim3 grid((c->params.K + 127) / 128, c->params.T);
    switch (draw_rule(c)) {
    case DRAW_HORIZON:
        return launch_sample_horizon_t<LIB>(c, seed, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, Z, actions, noise, s);
    case DRAW_FULL:
        mppib_sample_kernel<DRAW_FULL, LIB><<<grid, 128, 0, s>>>(c->params, nu, key0, seed_hi, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, Z,
                                                                 actions, noise, c->dist, nullptr, 0);
        break;
    case DRAW_DIAG:
        mppib_sample_kernel<DRAW_DIAG, LIB><<<grid, 128, 0, s>>>(c->params, nu, key0, seed_hi, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, Z,
                                                                 actions, noise, c->dist, nullptr, 0);
        break;
    default:
        mppib_sample_kernel<DRAW_FIXED, LIB><<<grid, 128, 0, s>>>(c->params, nu, key0, seed_hi, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, Z,
                                                                  actions, noise, nullptr, c->anneal, c->anneal_n);
    }
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// Risk-aware MPPI: a K1 shard holds whole groups of n_worlds rollouts, so that the R rollouts of a control get the same draw
int check_risk_shard(const MppibContext* c, const char* who, uint32_t k_offset, uint32_t k_total) {
    const int R = c->params.n_worlds;
    if (R <= 1) return 0;
    MPPIB_REQUIRE(c->params.K % R == 0 && k_offset % (uint32_t)R == 0 && k_total % (uint32_t)R == 0,
                  "%s: n_worlds = %d needs K = %d, k_offset = %u and k_total = %u to be multiples of it", who, R, c->params.K, k_offset, k_total);
    return 0;
}

// Multi-modal MPPI: the modes' blocks of Kc samples cover exactly the k_total samples of the plan
int check_modes_total(const MppibContext* c, const char* who, uint32_t k_total) {
    if (!modes_on(c)) return 0;
    MPPIB_REQUIRE((uint64_t)k_total == (uint64_t)c->params.n_modes * (uint64_t)c->params.mode_samples,
                  "%s: n_modes = %d with mode_samples = %d needs k_total = %d, got %u", who, c->params.n_modes, c->params.mode_samples,
                  c->params.n_modes * c->params.mode_samples, k_total);
    return 0;
}

}  // namespace

// Which K1 entry samples which draw (the table of include/mppib.h), checked on the host before any launch:
//   mppib_sample          FIXED, DIAG, FULL, HORIZON
//   mppib_sample_colored  FIXED, DIAG, FULL, CEM (with its state); not cov_horizon, even with no distribution registered
//   mppib_sample_smooth   SMOOTH (with its state); validate excludes n_worlds > 1 and n_modes > 1 from it
//   mppib_noise_library   FIXED, DIAG, FULL, HORIZON: the library is white exactly for DIAG, FULL and HORIZON
//   mppib_sample_library  FIXED, DIAG, FULL, HORIZON
//   mppib_sample_spline   FIXED with control_knots > 0 and a matching spline table; every other entry refuses control_knots > 0
// A registered annealing schedule goes through check_anneal in the two Philox entries; the library entries refuse one whatever its T.
// args: the entry's required pointers are all non-null.
int k1_admit(const MppibContext* c, K1Entry e, bool args, uint32_t k_offset, uint32_t k_total, int n_knots) {
    static const char* const names[] = {"mppib_sample", "mppib_sample_colored", "mppib_sample_smooth", "mppib_noise_library", "mppib_sample_library",
                                        "mppib_sample_spline"};
    const char* who = names[e];
    const bool lib = e == K1_NOISE_LIBRARY || e == K1_SAMPLE_LIBRARY;
    MPPIB_REQUIRE(c && args, "%s: null argument", who);
    if (e == K1_SPLINE) {
        MPPIB_REQUIRE(c->params.control_knots > 0, "%s: needs control_knots > 0 (spline MPPI)", who);
        if (int rc = check_spline(c, who)) return rc;
        MPPIB_REQUIRE((uint64_t)k_offset + (uint64_t)c->params.K <= (uint64_t)k_total, "%s: shard [%u,+%d) exceeds k_total %u", who, k_offset,
                      c->params.K, k_total);
        MPPIB_REQUIRE(c->params.control_knots * c->model.nu <= SP_MAX_N, "%s: needs P*nu <= %d, got %d", who, SP_MAX_N,
                      c->params.control_knots * c->model.nu);
        return 0;
    }
    MPPIB_REQUIRE(c->params.control_knots == 0, "%s: control_knots > 0 samples through mppib_sample_spline", who);
    if (e == K1_SAMPLE || e == K1_COLORED)
        if (int rc = check_anneal(c, who)) return rc;
    const bool in_range = (uint64_t)k_offset + (uint64_t)c->params.K <= (uint64_t)k_total;
    if (lib) MPPIB_REQUIRE(in_range, "%s: shard exceeds k_total", who);
    else MPPIB_REQUIRE(in_range, "%s: shard [%u,+%d) exceeds k_total %u", who, k_offset, c->params.K, k_total);
    const int T = c->params.T, nu = c->model.nu;
    const Draw d = draw_rule(c);
    if (e == K1_SMOOTH) {
        MPPIB_REQUIRE(d == DRAW_SMOOTH, "%s: needs mode smooth (MPPIB_MODE_SMOOTH), the handle has mode %d", who, c->params.mode);
        MPPIB_REQUIRE(c->smooth != nullptr, "%s: no smooth state registered (mppib_set_smooth_state)", who);
        if (int rc = check_exclusions(c->params, c->anneal != nullptr, who)) return rc;
        MPPIB_REQUIRE(T * nu <= SM_MAX_N, "%s: needs T*nu <= %d, got %d", who, SM_MAX_N, T * nu);
        return 0;
    }
    MPPIB_REQUIRE(d != DRAW_CEM || e == K1_COLORED, "%s: mode cem samples through mppib_sample_colored%s", who,
                  e == K1_SAMPLE ? " (white noise: Lt = I)" : "");
    MPPIB_REQUIRE(d != DRAW_SMOOTH, "%s: mode smooth samples through mppib_sample_smooth", who);
    if (lib)
        MPPIB_REQUIRE(c->anneal == nullptr, "%s: annealed MPPI excludes the noise library (every iteration would reuse the same directions); "
                      "register no schedule (mppib_set_anneal(h, NULL, 0))", who);
    if (int rc = check_risk_shard(c, who, k_offset, k_total)) return rc;
    if (e == K1_NOISE_LIBRARY) {
        MPPIB_REQUIRE(n_knots >= 1 && n_knots <= MAX_KNOTS, "%s: n_knots = %d out of range [1, %d]", who, n_knots, MAX_KNOTS);
        return 0;
    }
    if (int rc = check_modes_total(c, who, k_total)) return rc;
    if (e == K1_COLORED) {
        MPPIB_REQUIRE(!c->params.cov_horizon, "%s: cov_horizon already models the time correlation; colored noise excludes it", who);
        MPPIB_REQUIRE(T <= CL_MAX_T && T * nu <= CL_MAX_N, "%s: needs T <= %d and T*nu <= %d, got T = %d, T*nu = %d", who, CL_MAX_T, CL_MAX_N, T,
                      T * nu);
        MPPIB_REQUIRE(d != DRAW_CEM || c->dist != nullptr, "%s: mppi_mode cem needs its state registered with mppib_set_distribution", who);
        return 0;
    }
    MPPIB_REQUIRE(d != DRAW_HORIZON || T * nu <= MPPIB_HZ_MAX_N, "K1: cov_horizon needs n = T*nu <= %d, got %d", MPPIB_HZ_MAX_N, T * nu);
    return 0;
}

int launch_noise_library(MppibContext* c, uint32_t k_offset, uint32_t k_total, const int32_t* halton_tab, const float* B, int n_knots,
                         float* Z, cudaStream_t s) {
    const int K = c->params.K;
    const Draw d = draw_rule(c);
    if (d == DRAW_DIAG || d == DRAW_FULL || d == DRAW_HORIZON)
        mppib_noise_library_kernel<true><<<(K + 127) / 128, 128, 0, s>>>(c->params, c->model.nu, k_offset, k_total, halton_tab, B, n_knots, Z);
    else
        mppib_noise_library_kernel<false><<<(K + 127) / 128, 128, 0, s>>>(c->params, c->model.nu, k_offset, k_total, halton_tab, B, n_knots, Z);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_sample_library(MppibContext* c, uint32_t k_offset, uint32_t k_total, const float* U, const float* prior_row, const float* Z,
                          float* actions, float* noise, cudaStream_t s) {
    return launch_sample_t<true>(c, 0, 0, nullptr, k_offset, k_total, U, prior_row, Z, actions, noise, s);
}

int launch_sample(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                  const float* U, const float* prior_row, float* actions, float* noise, cudaStream_t s) {
    return launch_sample_t<false>(c, seed, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, nullptr, actions, noise, s);
}

int launch_sample_colored(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                          const float* U, const float* prior_row, const float* Lt, float* actions, float* noise, cudaStream_t s) {
    switch (draw_rule(c)) {
    case DRAW_CEM: return launch_sample_colored_t<DRAW_CEM>(c, seed, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, Lt, actions, noise, s);
    case DRAW_FULL: return launch_sample_colored_t<DRAW_FULL>(c, seed, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, Lt, actions, noise, s);
    case DRAW_DIAG: return launch_sample_colored_t<DRAW_DIAG>(c, seed, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, Lt, actions, noise, s);
    default: return launch_sample_colored_t<DRAW_FIXED>(c, seed, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, Lt, actions, noise, s);
    }
}

int launch_sample_smooth(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                         const float* U, float* actions, float* noise, cudaStream_t s) {
    const int K = c->params.K, nu = c->model.nu;
    const int smem = (int)sizeof(float) * c->params.T * nu * SM_S;
    if (int rc = ensure_smem<mppib_sample_smooth_kernel>(c->device, smem)) return rc;
    mppib_sample_smooth_kernel<<<(K + SM_S - 1) / SM_S, 128, smem, s>>>(c->params, nu, (uint32_t)seed, (uint32_t)(seed >> 32), plan_idx, plan_ctr,
                                                                      k_offset, k_total, U, actions, noise, c->smooth);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_sample_spline(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                         const float* U, float* actions, float* xk, cudaStream_t s) {
    const int K = c->params.K, nu = c->model.nu;
    const int smem = (int)sizeof(float) * c->params.control_knots * nu * SP_S;
    if (int rc = ensure_smem<mppib_sample_spline_kernel>(c->device, smem)) return rc;
    mppib_sample_spline_kernel<<<(K + SP_S - 1) / SP_S, 128, smem, s>>>(c->params, nu, (uint32_t)seed, (uint32_t)(seed >> 32), plan_idx, plan_ctr,
                                                                      k_offset, k_total, U, live_spline(c), actions, xk);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
