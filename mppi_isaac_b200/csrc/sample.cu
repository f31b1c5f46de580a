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

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
        uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += W0; k1 += W1;
    }
    return c;
}

__device__ __forceinline__ float u01(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }

__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
    float r = sqrtf(-2.0f * logf(u01(a)));
    float s, c;
    sincospif(2.0f * u01(b), &s, &c);
    z0 = r * c; z1 = r * s;
}

// DIAG (adaptive MPPI with update_cov): noise_j = sqrt(cov_j) z_j with cov = dist[1..nu], the live diagonal covariance; the Philox
// counters, clamping and the null / prior rows are those of the fixed-Sigma kernel.
// FULL (update_cov with cov_full): noise = L z with L = dist[1 + nu*nu ..], the live lower Cholesky factor, summed in the order of the
// fixed-Sigma kernel.
template <bool DIAG, bool FULL = false>
__global__ void __launch_bounds__(128)
mppib_sample_kernel(const __grid_constant__ MppibParams p, int nu, uint32_t key0, uint32_t seed_hi, uint64_t plan_idx,
              const uint32_t* __restrict__ plan_ctr, uint32_t k_offset, uint32_t k_total, const float* __restrict__ U, const float* __restrict__ prior_row,
              float* __restrict__ actions, float* __restrict__ noise, const float* __restrict__ dist) {
    const int K = p.K;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int t = blockIdx.y;
    if (k >= K) return;
    const uint32_t kg = k_offset + (uint32_t)k;
    const uint64_t plan = plan_idx + (plan_ctr ? (uint64_t)*plan_ctr : 0ull);
    const uint32_t key1 = seed_hi ^ (uint32_t)plan, plan_hi = (uint32_t)(plan >> 32);
    float z[MPPIB_MAX_NU];
#pragma unroll
    for (int blk = 0; blk < MPPIB_MAX_NU / 4; ++blk) {
        if (blk * 4 < nu) {
            uint4 r = philox4x32_10(make_uint4(kg, (uint32_t)t, (uint32_t)blk, plan_hi), key0, key1);
            box_muller(r.x, r.y, z[4 * blk], z[4 * blk + 1]);
            box_muller(r.z, r.w, z[4 * blk + 2], z[4 * blk + 3]);
        }
    }
    const bool is_null = p.sample_null_action && kg == k_total - 1;
    const bool is_prior = prior_row != nullptr && kg == k_total - 2;
#pragma unroll
    for (int j = 0; j < MPPIB_MAX_NU; ++j) {
        if (j >= nu) break;
        float n = 0.f;
        if (DIAG) {
            n = sqrtf(dist[1 + j]) * z[j];
        } else if (FULL) {
            const float* Ld = dist + 1 + nu * nu;
#pragma unroll
            for (int i = 0; i < MPPIB_MAX_NU; ++i)
                if (i <= j) n += Ld[j * nu + i] * z[i];
        } else {
#pragma unroll
            for (int i = 0; i < MPPIB_MAX_NU; ++i)
                if (i <= j) n += p.sigma_chol[j * nu + i] * z[i];
        }
        const float u = U[t * nu + j];
        float a = u + n;
        if (is_null) a = 0.f;
        a = fminf(fmaxf(a, p.u_min[j]), p.u_max[j]);
        if (is_prior) a = prior_row[t * nu + j];
        const size_t idx = ((size_t)t * nu + j) * K + k;
        actions[idx] = a;
        if (noise) noise[idx] = a - u;
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

// one thread per sample k: Gaussian knots (n_knots x nu) -> coloured -> spline-interpolated to T points.  WHITE (adaptive MPPI with
// update_cov): identity colour, the library sampler scales by the live sqrt(cov) (or colours by the live L, cov_full) on every plan.
template <bool WHITE>
__global__ void __launch_bounds__(128)
mppib_noise_library_kernel(const __grid_constant__ MppibParams p, int nu, uint32_t k_offset, uint32_t k_total,
                           const int32_t* __restrict__ tab, const float* __restrict__ B, int n_knots, float* __restrict__ Z) {
    const int K = p.K, T = p.T;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    const uint32_t kg = k_offset + (uint32_t)k;
    const bool null_row = p.sample_null_action && kg == k_total - 1;
    const int nd = n_knots * nu;
    for (int j = 0; j < nu; ++j) {
        // coloured knots of control dimension j:  c[n] = sum_i L[j][i] z[n][i]
        float cn[MAX_KNOTS];
        for (int n = 0; n < n_knots; ++n) {
            float acc = 0.f;
            for (int i = WHITE ? j : 0; i <= j; ++i) {
                const int d = n * nu + i;
                const float u = halton(kg + 1u, (uint32_t)tab[d], (uint32_t)tab[nd + d]);
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

// DIAG (adaptive MPPI with update_cov): Z is the white library, scaled by the live sqrt(cov_j) = sqrt(dist[1 + j]).
// FULL (update_cov with cov_full): Z is the white library, coloured by the live L = dist[1 + nu*nu ..]: a = clamp(U + L Z[t][:, k]).
template <bool DIAG, bool FULL = false>
__global__ void __launch_bounds__(128)
mppib_sample_library_kernel(const __grid_constant__ MppibParams p, int nu, uint32_t k_offset, uint32_t k_total, const float* __restrict__ U,
                            const float* __restrict__ prior_row, const float* __restrict__ Z, float* __restrict__ actions,
                            float* __restrict__ noise, const float* __restrict__ dist) {
    const int K = p.K;
    const int k = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y;
    if (k >= K) return;
    const uint32_t kg = k_offset + (uint32_t)k;
    const bool is_null = p.sample_null_action && kg == k_total - 1;
    const bool is_prior = prior_row != nullptr && kg == k_total - 2;
    if constexpr (FULL) {
        const float* Ld = dist + 1 + nu * nu;
        float zc[MPPIB_MAX_NU];
#pragma unroll
        for (int i = 0; i < MPPIB_MAX_NU; ++i) zc[i] = i < nu ? Z[((size_t)t * nu + i) * K + k] : 0.f;
#pragma unroll
        for (int j = 0; j < MPPIB_MAX_NU; ++j) {
            if (j >= nu) break;
            float n = 0.f;
#pragma unroll
            for (int i = 0; i < MPPIB_MAX_NU; ++i)
                if (i <= j) n += Ld[j * nu + i] * zc[i];
            const size_t idx = ((size_t)t * nu + j) * K + k;
            const float u = U[t * nu + j];
            float a = u + n;
            if (is_null) a = 0.f;
            a = fminf(fmaxf(a, p.u_min[j]), p.u_max[j]);
            if (is_prior) a = prior_row[t * nu + j];
            actions[idx] = a;
            if (noise) noise[idx] = a - u;
        }
    } else {
        for (int j = 0; j < nu; ++j) {
            const size_t idx = ((size_t)t * nu + j) * K + k;
            const float u = U[t * nu + j];
            float a = u + (DIAG ? sqrtf(dist[1 + j]) * Z[idx] : Z[idx]);
            if (is_null) a = 0.f;
            a = fminf(fmaxf(a, p.u_min[j]), p.u_max[j]);
            if (is_prior) a = prior_row[t * nu + j];
            actions[idx] = a;
            if (noise) noise[idx] = a - u;
        }
    }
}

}  // namespace

int launch_noise_library(MppibContext* c, uint32_t k_offset, uint32_t k_total, const int32_t* halton_tab, const float* B, int n_knots,
                         float* Z, cudaStream_t s) {
    MPPIB_REQUIRE(n_knots >= 1 && n_knots <= MAX_KNOTS, "mppib_noise_library: n_knots = %d out of range [1, %d]", n_knots, MAX_KNOTS);
    const int K = c->params.K;
    if (adaptive_cov(c))
        mppib_noise_library_kernel<true><<<(K + 127) / 128, 128, 0, s>>>(c->params, c->model.nu, k_offset, k_total, halton_tab, B, n_knots, Z);
    else
        mppib_noise_library_kernel<false><<<(K + 127) / 128, 128, 0, s>>>(c->params, c->model.nu, k_offset, k_total, halton_tab, B, n_knots, Z);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_sample_library(MppibContext* c, uint32_t k_offset, uint32_t k_total, const float* U, const float* prior_row, const float* Z,
                          float* actions, float* noise, cudaStream_t s) {
    const int K = c->params.K, T = c->params.T;
    dim3 block(128), grid((K + 127) / 128, T);
    if (adaptive_full(c))
        mppib_sample_library_kernel<false, true><<<grid, block, 0, s>>>(c->params, c->model.nu, k_offset, k_total, U, prior_row, Z, actions, noise, c->dist);
    else if (adaptive_cov(c))
        mppib_sample_library_kernel<true><<<grid, block, 0, s>>>(c->params, c->model.nu, k_offset, k_total, U, prior_row, Z, actions, noise, c->dist);
    else
        mppib_sample_library_kernel<false><<<grid, block, 0, s>>>(c->params, c->model.nu, k_offset, k_total, U, prior_row, Z, actions, noise, nullptr);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_sample(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                  const float* U, const float* prior_row, float* actions, float* noise, cudaStream_t s) {
    const int K = c->params.K, T = c->params.T;
    dim3 block(128), grid((K + 127) / 128, T);
    if (adaptive_full(c))
        mppib_sample_kernel<false, true><<<grid, block, 0, s>>>(c->params, c->model.nu, (uint32_t)seed, (uint32_t)(seed >> 32), plan_idx, plan_ctr, k_offset,
                                                                k_total, U, prior_row, actions, noise, c->dist);
    else if (adaptive_cov(c))
        mppib_sample_kernel<true><<<grid, block, 0, s>>>(c->params, c->model.nu, (uint32_t)seed, (uint32_t)(seed >> 32), plan_idx, plan_ctr, k_offset, k_total, U,
                                                         prior_row, actions, noise, c->dist);
    else
        mppib_sample_kernel<false><<<grid, block, 0, s>>>(c->params, c->model.nu, (uint32_t)seed, (uint32_t)(seed >> 32), plan_idx, plan_ctr, k_offset, k_total, U,
                                                          prior_row, actions, noise, nullptr);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
