// reduce.cu -- K3: per-step cost accumulation + importance-sampling softmax + weighted control sum over the
// K trajectories as ONE fused single-pass reduction (north-star item (iii)), K4: shard combine + U update,
// and the U shift.  Replaces mppi_torch `_compute_rollout_costs` accumulation, `_exp_util`,
// `_update_distribution` (external dep mppi_torch@75e17e8; call site mppiisaac/planner/mppi_isaac.py:113;
// spec SURVEY.md 8(a) M5/M6 and 8(e)).
//
// K3 data flow (HBM-bound; every input byte is read from HBM exactly once):
//   * persistent CTAs (one per SM), each walks tiles of 32 samples: tile = x[T*nu][32] + cost[T][32]
//   * tiles arrive by TMA (cp.async.bulk.tensor.2d, one elected thread, mbarrier complete_tx) into a shared-memory
//     ring of up to 8 stages, so several tiles are always in flight while the CTA computes
//   * per tile:  S_k = sum_t gamma^t cost[t][k]  (+ sum_r g[r] x[r][k],  g = lambda Sigma^-1 U,  SIMPLE mode)
//                b = min_k S_k ; w_k = exp(-(S_k - b)/lambda) ; eta = sum_k w_k ; W[r] = sum_k w_k x[r][k]
//     and an online log-sum-exp merge into the CTA's running (beta, eta, W) -- no second pass for the minimum
//   * per-CTA partials -> global scratch; the LAST CTA (atomic ticket) folds them in parallel into `partial`
// Algorithmic bytes per launch: 4*K*T*(nu+1) + 4*(T*nu+2)   (BASELINE.md section 3).
#include <cuda.h>

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int NT = 256;         // threads per CTA
constexpr int MAX_GRID = 512;   // persistent CTAs (<= scratch rows)
constexpr int MAX_PAIRS = MPPIB_MAX_NU * (MPPIB_MAX_NU + 1) / 2;   // lower triangle of a full nu x nu covariance

// the rules that read lambda (and Sigma) from a registered distribution and update it in K4
__host__ __device__ constexpr bool rule_adapts(Rule r) { return r == RULE_DIST || r == RULE_FULL || r == RULE_HORIZON; }
// The row a K3 CTA accumulates: the shard row, but one mode's block with MODES and (beta, eta, W[n]) with HORIZON (the SYRK appends C)
__host__ __device__ constexpr Rule k3_row_rule(Rule r) { return r == RULE_MODES || r == RULE_HORIZON ? RULE_PLAIN : r; }
// shared floats finalize_rows<RULE_FULL> needs after un[T*nu] and the G scales: m1[T*nu], d[T*nu], C[nu(nu+1)/2], Sigma, L, L^-1
__host__ __device__ __forceinline__ int full_fin_floats(int T, int nu) { return 2 * T * nu + nu * (nu + 1) / 2 + 3 * nu * nu; }
// cov_horizon, n = T*nu: the shared floats finalize_rows<RULE_HORIZON> needs after un[n] and the G scales: m1[n], d[n], the packed lower
// triangle A[n(n+1)/2] it factors, pivots[n], a column buffer[n]
__host__ __device__ __forceinline__ int hz_fin_floats(int n) { return 4 * n + n * (n + 1) / 2; }
__device__ __forceinline__ int tri(int i) { return i * (i + 1) / 2; }     // offset of row i in a packed lower triangle
// n_modes = M > 1: the shared floats modes_rows needs with G shard rows: d[M*T*nu], Sigma^-1 U then the coupled U [M*T*nu], U[M*T*nu],
// Sigma^-1, the G scales of every mode, (beta, eta, F, sum_j k_ij)[M], D[M][M], k[M][M] and 4 floats
__host__ __device__ __forceinline__ int modes_fin_floats(int NR, int M, int G) {
    return 3 * M * NR + MPPIB_MAX_NU * MPPIB_MAX_NU + M * G + 4 * M + 2 * M * M + 4;
}

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// Risk-aware MPPI: the CVaR score of the aligned group of R lanes (R a power of two <= 32) this lane belongs to.  The group's S (+inf
// for an invalid or padding sample) is sorted in descending order by a bitonic network over __shfl_xor_sync -- every stage but the last
// merges pairs of blocks of opposite order, the last one orders every group the same way -- then lane r = 0 of the group sums its m
// largest values left to right, divides once by m and keeps the result; the other lanes get +inf and so weight 0.
__device__ __forceinline__ float risk_score(float S, int R, int m, int lane) {
    for (int k = 2; k <= R; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            const float o = __shfl_xor_sync(0xffffffffu, S, j);
            const bool desc = k == R || (lane & k) == 0;                      // order of the block of k lanes this lane sorts into
            S = (((lane & j) == 0) == desc) ? fmaxf(S, o) : fminf(S, o);
        }
    }
    const int base = lane & ~(R - 1);
    float acc = S;
    for (int i = 1; i < m; ++i) acc += __shfl_sync(0xffffffffu, S, base + i);
    return lane == base ? __fdiv_rn(acc, (float)m) : INFINITY;
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
// 2-D tiled TMA load: box (W columns x rows) of a row-major [rows][K] float tensor -> dense smem tile
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, int col, int row, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(col), "r"(row), "r"(smem_u32(bar)) : "memory");
}

__constant__ float c_sg_mid[9] = {-21.f, 14.f, 39.f, 54.f, 59.f, 54.f, 39.f, 14.f, -21.f};
__constant__ float c_sg_edge[4][9] = {{763.f, 441.f, 189.f, 7.f, -105.f, -147.f, -119.f, -21.f, 147.f},
                                      {441.f, 322.f, 220.5f, 136.5f, 70.f, 21.f, -10.5f, -24.5f, -21.f},
                                      {189.f, 220.5f, 232.f, 223.5f, 195.f, 146.5f, 78.f, -10.5f, -119.f},
                                      {7.f, 136.5f, 223.5f, 268.f, 270.f, 229.5f, 146.5f, 21.f, -147.f}};
// Savitzky-Golay (window 9, order 2, 'interp' edges) of the [T][nu] sequence u at element r = t*nu + j: the window's products summed
// in window order, then one scaling
__device__ __forceinline__ float savgol(const float* u, int T, int nu, int r) {
    const int t = r / nu, j = r % nu;
    float s = 0.f;
    if (t < 4) {
#pragma unroll
        for (int i = 0; i < 9; ++i) s += c_sg_edge[t][i] * u[i * nu + j];
        s *= (1.0f / 1155.0f);
    } else if (t >= T - 4) {
        const int ee = T - 1 - t;
#pragma unroll
        for (int i = 0; i < 9; ++i) s += c_sg_edge[ee][i] * u[(T - 1 - i) * nu + j];
        s *= (1.0f / 1155.0f);
    } else {
#pragma unroll
        for (int i = 0; i < 9; ++i) s += c_sg_mid[i] * u[(t - 4 + i) * nu + j];
        s *= (1.0f / 231.0f);
    }
    return s;
}

// K4 of cov_horizon (dist = (lambda, Sigma_H, L_H, Sigma_H^-1), n = T*nu, after the U update, e = eta > 0), one CTA:
//   1. Sigma' = shift((1 - s) Sigma_H + s V + kappa I),  V = C/eta - (m1 d^T + d m1^T - d d^T),  C = sum_g scale_g C_g:
//      Sigma'[a][b] = Sigma_new[a + nu][b + nu] for a, b < n - nu; the last block row and column are 0 but for the last diagonal
//      block, sigma0.  Lower triangle, packed into A (shared) and written to both halves of hz_sig (global staging).
//   2. L = chol(Sigma') in place in A, right-looking: pivot k, column k scaled (and kept in `col`), rank-1 update of the trailing
//      triangle; every entry sees its updates in k order, so the result is fixed.  The pivots go to `piv`.
//   3. If every pivot was finite and positive: Sigma' and L to dist, L^-1 in place in A (right-looking forward substitution for all
//      columns at once), Sigma^-1 = L^-T L^-1 to both halves of dist.  Otherwise Sigma_H, L_H and Sigma_H^-1 stay as they were.
// Every rank combines the same rows in the same order and runs the same fixed-order arithmetic, so all write the same bits.
__device__ __noinline__ void horizon_update(const MppibParams& p, int nu, const float* __restrict__ partials, int G, int P, const float* sg, float e,
                                            const float* m1, const float* dd, float* A, float* __restrict__ dist, float* __restrict__ hz_sig) {
    const int n = p.T * nu, m = n - nu, npairs = tri(n);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    float* piv = A + npairs;
    float* col = piv + n;
    const float s = p.step_size_cov;
    float* dS = dist + 1;
    float* dL = dS + (size_t)n * n;
    float* dI = dL + (size_t)n * n;
    for (int i = warp; i < n; i += nw) {
        for (int j = lane; j <= i; j += 32) {
            float v;
            if (i < m) {
                const int a = i + nu, b = j + nu;
                float cq = 0.f;
                for (int g = 0; g < G; ++g) cq += sg[g] * __ldcg(&partials[(size_t)g * P + 2 + n + tri(a) + b]);
                const float vab = cq / e - (m1[a] * dd[b] + dd[a] * m1[b] - dd[a] * dd[b]);
                v = (1.0f - s) * dS[(size_t)a * n + b] + s * vab + (a == b ? p.kappa : 0.f);
            } else {
                v = j >= m ? p.sigma0[(i - m) * nu + (j - m)] : 0.f;
            }
            A[tri(i) + j] = v;
            hz_sig[(size_t)i * n + j] = v;
            hz_sig[(size_t)j * n + i] = v;
        }
    }
    __syncthreads();
    bool ok = true;
    for (int k = 0; k < n; ++k) {
        const float dk = A[tri(k) + k];                                       // the same value in every thread: a uniform branch
        ok = isfinite(dk) && dk > 0.f;
        if (!ok) break;
        const float lkk = sqrtf(dk);
        if (tid == 0) piv[k] = lkk;
        for (int i = k + 1 + tid; i < n; i += blockDim.x) {
            const float l = A[tri(i) + k] / lkk;
            A[tri(i) + k] = l;
            col[i] = l;
        }
        __syncthreads();
        for (int i = k + 1 + warp; i < n; i += nw) {
            const float lik = col[i];
            float* __restrict__ Ai = A + tri(i);
#pragma unroll 4
            for (int j = k + 1 + lane; j <= i; j += 32) Ai[j] -= lik * col[j];
        }
        __syncthreads();
    }
    if (!ok) return;
    for (int i = warp; i < n; i += nw) {
        for (int j = lane; j < n; j += 32) {
            dS[(size_t)i * n + j] = hz_sig[(size_t)i * n + j];
            dL[(size_t)i * n + j] = j < i ? A[tri(i) + j] : j == i ? piv[i] : 0.f;
        }
    }
    __syncthreads();
    // X = L^-1 in place: at step k row k of X is final (X[k][j] = B[k][j] / L[k][k], X[k][k] = 1 / L[k][k]) and the rows below get
    // B[i][j] -= L[i][k] X[k][j] (j <= k; B[i][k] starts at 0, where L[i][k] stood, so column k of L is copied to `col` first)
    for (int k = 0; k < n; ++k) {
        float* Ak = A + tri(k);
        const float pk = piv[k];
        for (int j = tid; j <= k; j += blockDim.x) Ak[j] = j == k ? 1.0f / pk : Ak[j] / pk;
        for (int i = k + 1 + tid; i < n; i += blockDim.x) col[i] = A[tri(i) + k];
        __syncthreads();
        for (int i = k + 1 + warp; i < n; i += nw) {
            const float lik = col[i];
            float* __restrict__ Ai = A + tri(i);
            const float* __restrict__ Xk = Ak;
#pragma unroll 4
            for (int j = lane; j <= k; j += 32) Ai[j] = (j == k ? 0.f : Ai[j]) - lik * Xk[j];
        }
        __syncthreads();
    }
    for (int a = warp; a < n; a += nw) {                                      // Sigma^-1[a][b] = sum_{r >= a} X[r][a] X[r][b], b <= a
        for (int b = lane; b <= a; b += 32) {
            float acc = 0.f;
#pragma unroll 4
            for (int r = a; r < n; ++r) acc += A[tri(r) + a] * A[tri(r) + b];
            dI[(size_t)a * n + b] = acc;
            dI[(size_t)b * n + a] = acc;
        }
    }
}

// K4's merge of G rows (beta_g, eta_g, W_g, ...) of stride P by merge_min / merge_scale (a row with eta_g = 0 is empty): the minimum
// into b, the scale of every row into sg[G], and the return value eta = sum_g sg_g eta_g in g order.  The caller sums W (and what else
// its rows carry) under the same scales.  FEAS: the rows carry (n_feasible bits, min V) after W[NR]; thread 0 writes cstate = (sum
// n_feasible, min V) (nullable).  A CTA-wide call: sg is complete when it returns.
template <bool FEAS>
__device__ __forceinline__ float merge_rows(const MppibParams& p, int NR, const float* __restrict__ partials, int G, int P, float inv_lambda, float* sg,
                                            float& b, float* __restrict__ cstate) {
    auto nf_of = [&](int gidx) { return FEAS ? __float_as_int(__ldcg(&partials[(size_t)gidx * P + 2 + NR])) : 0; };
    int n_all = 0;
    if constexpr (FEAS) {
        float vmin = INFINITY;
        for (int gidx = 0; gidx < G; ++gidx) { n_all += nf_of(gidx); vmin = fminf(vmin, __ldcg(&partials[(size_t)gidx * P + 3 + NR])); }
        if (threadIdx.x == 0 && cstate) { cstate[0] = __int_as_float(n_all); cstate[1] = vmin; }
    }
    const float inv_lc = FEAS ? 1.0f / p.constraint_lambda : inv_lambda;
    b = INFINITY;
    for (int gidx = 0; gidx < G; ++gidx) if (__ldcg(&partials[(size_t)gidx * P + 1]) > 0.f) b = merge_min(nf_of(gidx), __ldcg(&partials[(size_t)gidx * P]), n_all, b);
    for (int gidx = threadIdx.x; gidx < G; gidx += blockDim.x) {
        const float eg = __ldcg(&partials[(size_t)gidx * P + 1]);
        sg[gidx] = eg > 0.f ? merge_scale(nf_of(gidx), __ldcg(&partials[(size_t)gidx * P]), n_all, b, inv_lambda, inv_lc) : 0.f;
    }
    __syncthreads();
    float e = 0.f;
    for (int gidx = 0; gidx < G; ++gidx) e += sg[gidx] * __ldcg(&partials[(size_t)gidx * P + 1]);
    return e;
}

// combine G rows (beta_g, eta_g, W_g) of stride P (merge_rows), update U (+ Savitzky-Golay, clamp), first action, statistics; one CTA of
// 256 threads, `un` = [T*nu + G] floats of shared memory (+ T*nu with update_cov).
// ADAPT (a distribution is registered): lambda comes from dist[0]; after the U update the CTA updates dist in place --
//   update_cov:    the rows carry M2_g after W_g; m1 = W/eta - c, m2 = M2/eta, d = U_new - U_old (before Savitzky-Golay),
//                  var = max(m2 - 2 d m1 + d^2, 0), cov_j <- (1 - s) cov_j + s mean_t var[t][j] + kappa
//   update_lambda: lambda *= 1 - lambda_mult (eta > eta_u_bound) or 1 + lambda_mult (eta < eta_l_bound), kept in [1e-3, 1e3] lambda0
// and leaves it as it is when no sample is valid.  The mean over t runs serially in t order on one thread per j, so every rank of a
// multi-GPU plan, which combines the same rows in the same order, writes bit-identical values.  Every thread reads dist[0] at entry and
// dist[1 + j] is read and written by thread j only; the writes come after the __syncthreads below, so nothing reads a value written here.
// FULL (update_cov with cov_full; dist = (lambda, Sigma, L, Sigma^-1)): the rows carry C_g[nu(nu+1)/2] after W_g.  With m1 = W/eta - c and
// d = U_new - U_old per (t, j):  V = C/eta - sum_t (m1_t d_t^T + d_t m1_t^T - d_t d_t^T),  Sigma <- (1 - s) Sigma + (s/T) V + kappa I,
// one thread per lower-triangle entry (t in order), written to both halves; then warp 0 computes L = chol(Sigma) (left-looking, lane =
// row) and Sigma^-1 = L^-T L^-1 (lane = column of L^-1) in a fixed order.  A pivot that is not finite and positive leaves Sigma, L and
// Sigma^-1 as they were.  The diagonal equals the diagonal rule above without its clamp at 0.
// HZN (update_cov with cov_horizon): the rows carry C_g[n(n+1)/2] over the whole sequence; m1 and d are kept as n-vectors and
// horizon_update does the rest.
// FEAS (constraint_mode): the rows carry (n_feasible bits, min V) after W_g and merge feasibility-first, then the update is today's;
// thread 0 writes cstate = (sum n_feasible, min V) (nullable).
template <Rule R>
__device__ __forceinline__ void finalize_rows(const MppibParams& p, int nu, const float* __restrict__ partials, int G, int P, float* __restrict__ U,
                                              float* __restrict__ action_out, float* __restrict__ stats, float* __restrict__ action_mirror, float* un,
                                              float* __restrict__ dist, float* __restrict__ hz_sig = nullptr, float* __restrict__ cstate = nullptr) {
    constexpr bool ADAPT = rule_adapts(R), FULL = R == RULE_FULL, HZN = R == RULE_HORIZON, FEAS = R == RULE_FEASIBLE;
    const int T = p.T, NR = (R == RULE_PLAIN ? ctrl_rows(p) : T) * nu;   // knots parameterise PLAIN only
    float* sg = un + NR;
    const float lam = ADAPT ? dist[0] : p.lambda_;
    const float inv_lambda = 1.0f / lam;
    const bool cov = ADAPT && !FULL && !HZN && p.update_cov;
    float* var = sg + G;                                                      // [NR] per-element variance (update_cov)
    const int npairs = nu * (nu + 1) / 2;
    float* m1s = sg + G;                                                      // FULL: [NR] m1, [NR] d, [npairs] C, [nu*nu] Sigma, L, L^-1
    float* dds = m1s + NR;
    float* cc = dds + NR;
    float* sn = cc + npairs;
    float* Lm = sn + nu * nu;
    float* Mi = Lm + nu * nu;
    float b;
    const float e = merge_rows<FEAS>(p, NR, partials, G, P, inv_lambda, sg, b, cstate);
    for (int r = threadIdx.x; r < NR; r += blockDim.x) {
        float w = 0.f;
        for (int gidx = 0; gidx < G; ++gidx) w += sg[gidx] * __ldcg(&partials[(size_t)gidx * P + 2 + r]);
        const float wm = e > 0.f ? w / e : (p.mode == MPPIB_MODE_SIMPLE ? 0.f : U[r]);   // no valid sample: keep U
        un[r] = p.mode == MPPIB_MODE_SIMPLE ? U[r] + wm : (1.0f - p.step_size_mean) * U[r] + p.step_size_mean * wm;
        if (cov && e > 0.f) {
            float m2 = 0.f;
            for (int gidx = 0; gidx < G; ++gidx) m2 += sg[gidx] * __ldcg(&partials[(size_t)gidx * P + 2 + NR + r]);
            const float c0 = p.mode == MPPIB_MODE_SIMPLE ? 0.f : U[r];
            const float m1 = w / e - c0, d = un[r] - U[r];
            var[r] = fmaxf(m2 / e - 2.0f * d * m1 + d * d, 0.f);
        }
        if ((FULL || HZN) && e > 0.f) {
            m1s[r] = w / e - (p.mode == MPPIB_MODE_SIMPLE ? 0.f : U[r]);
            dds[r] = un[r] - U[r];
        }
    }
    if (FULL && e > 0.f) {
        for (int q = threadIdx.x; q < npairs; q += blockDim.x) {
            float cq = 0.f;
            for (int gidx = 0; gidx < G; ++gidx) cq += sg[gidx] * __ldcg(&partials[(size_t)gidx * P + 2 + NR + q]);
            cc[q] = cq;
        }
    }
    __syncthreads();
    for (int r = threadIdx.x; r < NR; r += blockDim.x) {
        float out = un[r];
        if (p.filter_u) {
            const int j = r % nu;
            out = fminf(fmaxf(savgol(un, T, nu, r), p.u_min[j]), p.u_max[j]);   // smoothing may overshoot the bounds at the edges
        }
        U[r] = out;
        if (r < nu) { action_out[r] = out; if (action_mirror) action_mirror[r] = out; }
    }
    if (threadIdx.x == 0 && stats) { stats[0] = b; stats[1] = e; }
    if (HZN && e > 0.f) horizon_update(p, nu, partials, G, P, sg, e, m1s, dds, dds + NR, dist, hz_sig);
    if (FULL && e > 0.f) {
        const float* Sig = dist + 1;
        for (int q = threadIdx.x; q < npairs; q += blockDim.x) {
            int i = 0;
            while ((i + 1) * (i + 2) / 2 <= q) ++i;
            const int j = q - i * (i + 1) / 2;
            float acc = 0.f;
            for (int t = 0; t < T; ++t) {
                const float mi = m1s[t * nu + i], mj = m1s[t * nu + j], di = dds[t * nu + i], dj = dds[t * nu + j];
                acc += mi * dj + di * mj - di * dj;
            }
            const float v = cc[q] / e - acc;
            const float sij = (1.0f - p.step_size_cov) * Sig[i * nu + j] + (p.step_size_cov / (float)T) * v + (i == j ? p.kappa : 0.f);
            sn[i * nu + j] = sij;
            sn[j * nu + i] = sij;
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            const int l = threadIdx.x;
            for (int q = l; q < nu * nu; q += 32) { Lm[q] = 0.f; Mi[q] = 0.f; }
            __syncwarp();
            bool ok = true;
            for (int k = 0; k < nu && ok; ++k) {                         // every lane computes the same pivot in the same order
                float dk = sn[k * nu + k];
                for (int m = 0; m < k; ++m) dk -= Lm[k * nu + m] * Lm[k * nu + m];
                ok = isfinite(dk) && dk > 0.f;
                if (ok) {
                    const float lkk = sqrtf(dk);
                    if (l > k && l < nu) {
                        float a = sn[l * nu + k];
                        for (int m = 0; m < k; ++m) a -= Lm[l * nu + m] * Lm[k * nu + m];
                        Lm[l * nu + k] = a / lkk;
                    }
                    if (l == k) Lm[k * nu + k] = lkk;
                }
                __syncwarp();
            }
            if (ok) {
                if (l < nu) {                                             // column l of L^-1 by forward substitution
                    for (int i = l; i < nu; ++i) {
                        float a = i == l ? 1.0f : 0.f;
                        for (int m = l; m < i; ++m) a -= Lm[i * nu + m] * Mi[m * nu + l];
                        Mi[i * nu + l] = a / Lm[i * nu + i];
                    }
                }
                __syncwarp();
                float* dS = dist + 1;
                float* dL = dS + nu * nu;
                float* dI = dL + nu * nu;
                for (int q = l; q < npairs; q += 32) {                   // Sigma^-1 = L^-T L^-1, lower triangle, written to both halves
                    int i = 0;
                    while ((i + 1) * (i + 2) / 2 <= q) ++i;
                    const int j = q - i * (i + 1) / 2;
                    float a = 0.f;
                    for (int m = i; m < nu; ++m) a += Mi[m * nu + i] * Mi[m * nu + j];
                    dI[i * nu + j] = a;
                    dI[j * nu + i] = a;
                }
                for (int q = l; q < nu * nu; q += 32) { dS[q] = sn[q]; dL[q] = Lm[q]; }
            }
        }
    }
    if (ADAPT && e > 0.f) {
        if (cov) {
            for (int j = threadIdx.x; j < nu; j += blockDim.x) {
                float acc = 0.f;
                for (int t = 0; t < T; ++t) acc += var[t * nu + j];
                dist[1 + j] = (1.0f - p.step_size_cov) * dist[1 + j] + p.step_size_cov * (acc / (float)T) + p.kappa;
            }
        }
        if (p.update_lambda && threadIdx.x == 0) {
            float l = lam;
            if (e > p.eta_u_bound) l = lam * (1.0f - p.lambda_mult);
            else if (e < p.eta_l_bound) l = lam * (1.0f + p.lambda_mult);
            dist[0] = fminf(fmaxf(l, 1e-3f * p.lambda_), 1e3f * p.lambda_);
        }
    }
}

// Spline MPPI: after finalize_rows, U_exec[T][nu] = B theta with the table's interpolation rows, theta = un (finalize_rows synchronised
// after writing it; filter_u is refused with knots, so un holds the updated knots as U does).
__device__ __forceinline__ void spline_exec(const MppibParams& p, int nu, const float* un, float* __restrict__ spline) {
    const int T = p.T, S = spline_row_floats(p.spline_degree);
    float* ue = spline + (size_t)(T + p.control_knots) * S;
    for (int r = threadIdx.x; r < T * nu; r += blockDim.x) ue[r] = spline_apply(spline + (r / nu) * S, un + r % nu, nu);
}

// K4 of mode smooth (smooth = (a_prev[nu], A[T][nu])): combine G rows (beta_g, eta_g, W_g) of stride P (merge_rows), the SIMPLE
// update of the derivative U' = U + W/eta (U' = U when eta = 0), clamped to du_min / du_max; then one thread per j integrates it in t
// order from a = a_prev: A_t = clamp(fmaf(U'_t, dt, a), u_min, u_max), U'_t := (A_t - a)/dt where that clamp bound, a = A_t.  U <- U',
// A stored, the action, its mirror and a_prev <- A_0; stats = (beta, eta).  Thread j alone reads and writes column j of the state, and
// every rank combines the same rows in the same order, so all write the same bits.  `un` = [T*nu + G] floats of shared memory.
__device__ __forceinline__ void smooth_rows(const MppibParams& p, int nu, const float* __restrict__ partials, int G, int P, float* __restrict__ U,
                                            float* __restrict__ action_out, float* __restrict__ stats, float* __restrict__ action_mirror, float* un,
                                            float* __restrict__ smooth) {
    const int T = p.T, NR = T * nu;
    float* sg = un + NR;
    float b;
    const float e = merge_rows<false>(p, NR, partials, G, P, 1.0f / p.lambda_, sg, b, nullptr);
    for (int r = threadIdx.x; r < NR; r += blockDim.x) {
        float w = 0.f;
        for (int gidx = 0; gidx < G; ++gidx) w += sg[gidx] * __ldcg(&partials[(size_t)gidx * P + 2 + r]);
        un[r] = U[r] + (e > 0.f ? w / e : 0.f);
    }
    __syncthreads();
    const float dt = p.dt;
    for (int j = threadIdx.x; j < nu; j += blockDim.x) {
        const float lo = p.u_min[j], hi = p.u_max[j], dlo = p.du_min[j], dhi = p.du_max[j];
        float a = smooth[j];
        for (int t = 0; t < T; ++t) {
            const int r = t * nu + j;
            float v = fminf(fmaxf(un[r], dlo), dhi);
            const float ah = fmaf(v, dt, a);
            const float an = fminf(fmaxf(ah, lo), hi);
            if (an != ah) v = (an - a) / dt;
            U[r] = v;
            smooth[nu + r] = an;
            a = an;
        }
        const float first = smooth[nu + j];
        smooth[j] = first;
        action_out[j] = first;
        if (action_mirror) action_mirror[j] = first;
    }
    if (threadIdx.x == 0 && stats) { stats[0] = b; stats[1] = e; }
}

// K4 of multi-modal MPPI (n_modes = M > 1, include/mppib.h "Multi-modal MPPI"; state = (active mode, F[M], U_exec[T][nu])): combine
// the G blocks of every mode as finalize_rows does, form the own steps d_m and free energies F_m, couple the modes (SVGD step with the
// RBF kernel in the Sigma^-1 metric, median bandwidth), Savitzky-Golay and clamp every mode, select the executed mode and write the
// action, stats and state from it.  U[M][T][nu] and Sigma^-1 are staged in shared memory first; D_ij = sum_r (U_i - U_j)_r (V_i - V_j)_r
// with V_m = Sigma^-1 U_m per step, one warp per pair (lane = row, then the warp's butterfly sum); every other sum runs in a fixed
// order on one thread, so every rank, which combines the same rows in the same order, writes the same bits.  `sm` = modes_fin_floats.
__device__ __noinline__ void modes_rows(const MppibParams& p, int nu, const float* __restrict__ partials, int G, int P, float* __restrict__ U,
                                        float* __restrict__ action_out, float* __restrict__ stats, float* __restrict__ action_mirror, float* sm,
                                        float* __restrict__ state) {
    const int T = p.T, NR = T * nu, M = p.n_modes, P1 = 2 + NR, MN = M * NR;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    float* dd = sm;                  // [M*NR] own steps, then the final sequences
    float* un = dd + MN;             // [M*NR] V = Sigma^-1 U per step, then the coupled sequences before Savitzky-Golay
    float* us = un + MN;             // [M*NR] U as it was
    float* si = us + MN;             // [nu*nu] Sigma^-1
    float* sg = si + MPPIB_MAX_NU * MPPIB_MAX_NU;   // [M][G]
    float* bm = sg + M * G;
    float* em = bm + M;
    float* fm = em + M;
    float* ks = fm + M;
    float* Dm = ks + M;              // [M][M]
    float* km = Dm + M * M;          // [M][M]
    float* misc = km + M * M;        // h, executed mode
    const float lam = p.lambda_, inv_lambda = 1.0f / lam;
    const bool simple = p.mode == MPPIB_MODE_SIMPLE;
    for (int q = tid; q < MN; q += nt) us[q] = U[q];
    for (int q = tid; q < nu * nu; q += nt) si[q] = p.sigma_inv[q];
    for (int m = tid; m < M; m += nt) {
        float b = INFINITY;
        for (int g = 0; g < G; ++g) {
            const float* row = partials + (size_t)g * P + (size_t)m * P1;
            if (__ldcg(row + 1) > 0.f) b = merge_min(0, __ldcg(row), 0, b);
        }
        bm[m] = b;
    }
    __syncthreads();
    for (int q = tid; q < M * G; q += nt) {
        const int m = q / G, g = q % G;
        const float* row = partials + (size_t)g * P + (size_t)m * P1;
        const float eg = __ldcg(row + 1);
        sg[q] = eg > 0.f ? merge_scale(0, __ldcg(row), 0, bm[m], inv_lambda, inv_lambda) : 0.f;
    }
    __syncthreads();
    for (int m = tid; m < M; m += nt) {
        float e = 0.f;
        for (int g = 0; g < G; ++g) e += sg[m * G + g] * __ldcg(partials + (size_t)g * P + (size_t)m * P1 + 1);
        em[m] = e;
        fm[m] = e > 0.f ? bm[m] - lam * logf(e / (float)p.mode_samples) : INFINITY;
    }
    __syncthreads();
    for (int q = tid; q < MN; q += nt) {                                      // own MPPI step of every mode
        const int m = q / NR, r = q % NR;
        float w = 0.f;
        for (int g = 0; g < G; ++g) w += sg[m * G + g] * __ldcg(partials + (size_t)g * P + (size_t)m * P1 + 2 + r);
        const float e = em[m], u = us[q];
        float d = 0.f;
        if (e > 0.f) {
            const float wm = w / e;
            d = simple ? wm : (1.0f - p.step_size_mean) * u + p.step_size_mean * wm - u;
        }
        dd[q] = d;
        const int t = r / nu, a = r % nu;
        const float* ut = us + (size_t)m * NR + t * nu;
        float v = 0.f;
        for (int b = 0; b < nu; ++b) v += si[a * nu + b] * ut[b];
        un[q] = v;
    }
    __syncthreads();
    const int npairs = M * (M - 1) / 2;
    for (int q = warp; q < npairs; q += nw) {                                 // D_ij, i < j: one warp per pair
        int i = 0, rem = q;
        while (rem >= M - 1 - i) { rem -= M - 1 - i; ++i; }
        const int j = i + 1 + rem;
        const float* Ui = us + (size_t)i * NR;
        const float* Uj = us + (size_t)j * NR;
        const float* Vi = un + (size_t)i * NR;
        const float* Vj = un + (size_t)j * NR;
        float acc = 0.f;
        for (int r = lane; r < NR; r += 32) acc += (Ui[r] - Uj[r]) * (Vi[r] - Vj[r]);
        acc = warp_sum(acc);
        if (lane == 0) { Dm[i * M + j] = acc; Dm[j * M + i] = acc; }
    }
    for (int i = tid; i < M; i += nt) Dm[i * M + i] = 0.f;
    if (tid == 0) misc[0] = NAN;                                              // no pair of that rank (a NaN distance): k = 1
    __syncthreads();
    for (int q = tid; q < npairs; q += nt) {                                  // the lower median: the pair of rank (npairs - 1) / 2
        int i = 0, rem = q;
        while (rem >= M - 1 - i) { rem -= M - 1 - i; ++i; }
        const float v = Dm[i * M + i + 1 + rem];
        int rank = 0;
        for (int q2 = 0, i2 = 0, j2 = 1; q2 < npairs; ++q2) {
            const float v2 = Dm[i2 * M + j2];
            rank += (v2 < v || (v2 == v && q2 < q)) ? 1 : 0;
            if (++j2 == M) { ++i2; j2 = i2 + 1; }
        }
        if (rank == (npairs - 1) / 2) misc[0] = v / logf((float)(M + 1));
    }
    __syncthreads();
    const float h = misc[0];
    const bool kern = h > 0.f && isfinite(h);
    for (int q = tid; q < M * M; q += nt) km[q] = kern ? expf(-Dm[q] / h) : 1.0f;
    __syncthreads();
    for (int i = tid; i < M; i += nt) {
        float sk = 0.f;
        for (int j = 0; j < M; ++j) sk += km[i * M + j];
        ks[i] = sk;
    }
    __syncthreads();
    const float c2 = kern ? 2.0f / h : 0.f;
    for (int q = tid; q < MN; q += nt) {                                      // the coupled step, j ascending
        const int i = q / NR, r = q % NR;
        const float ui = us[q];
        float a1 = 0.f, a2 = 0.f;
        for (int j = 0; j < M; ++j) {
            const float k = km[i * M + j];
            a1 += k * dd[j * NR + r];
            a2 += k * (ui - us[(size_t)j * NR + r]);
        }
        un[q] = ui + (kern ? a1 + c2 * a2 : a1) / ks[i];
    }
    __syncthreads();
    for (int q = tid; q < MN; q += nt) {                                      // Savitzky-Golay (filter_u) and the clamp, every mode
        const int m = q / NR, r = q % NR, j = r % nu;
        const float* u = un + (size_t)m * NR;
        float out = u[r];
        if (p.filter_u) out = savgol(u, T, nu, r);
        out = fminf(fmaxf(out, p.u_min[j]), p.u_max[j]);
        dd[q] = out;
        U[q] = out;
    }
    if (tid == 0) {                                                           // the executed mode
        int pm = (int)state[0];
        pm = pm < 0 ? 0 : pm >= M ? M - 1 : pm;
        int a = 0;
        for (int m = 1; m < M; ++m) if (fm[m] < fm[a]) a = m;
        if (isfinite(fm[a]) && !(fm[pm] <= fm[a] + p.mode_margin)) pm = a;
        misc[1] = (float)pm;
        state[0] = (float)pm;
        if (stats) { stats[0] = bm[pm]; stats[1] = em[pm]; }
    }
    __syncthreads();
    const int pe = (int)misc[1];
    for (int m = tid; m < M; m += nt) state[1 + m] = fm[m];
    for (int r = tid; r < NR; r += nt) {
        const float v = dd[(size_t)pe * NR + r];
        state[1 + M + r] = v;
        if (r < nu) { action_out[r] = v; if (action_mirror) action_mirror[r] = v; }
    }
}

// n_modes = M > 1, the last CTA of K3: the gridDim.x CTA partials of every mode m (scratch rows m*gx .. m*gx + gx - 1, stride P4 of the
// mode's row P1 = 2 + T*nu) fold into block m of the shard row [M][P1] in CTA order; the row goes into the peer windows as
// fold_and_finish stores it and, for single-GPU plans, modes_rows does K4's work in place.
__device__ __forceinline__ void fold_modes_and_finish(const MppibParams& p, int nu, int P1, float* __restrict__ scratch, unsigned int* __restrict__ ticket,
                                                      float* __restrict__ partial, const PeerArgs& peers, float* __restrict__ fin_U,
                                                      float* __restrict__ fin_action, float* __restrict__ fin_stats, float* __restrict__ fin_mirror,
                                                      float* tiles, float inv_lambda, float* __restrict__ state) {
    const int tid = threadIdx.x, M = (int)gridDim.y, gx = (int)gridDim.x, nrow = M * gx, P = M * P1, P4 = (P1 + 3) & ~3;
    float* sc = tiles;               // [M*gx] CTA beta, then scale
    float* bb = tiles + nrow;        // [M] mode minimum
    for (int q = tid; q < nrow; q += NT) sc[q] = __ldcg(scratch + (size_t)q * P4);
    __syncthreads();
    for (int m = tid; m < M; m += NT) {
        float b = INFINITY;
        for (int g = 0; g < gx; ++g) b = merge_min(0, sc[m * gx + g], 0, b);
        bb[m] = b;
    }
    __syncthreads();
    for (int q = tid; q < nrow; q += NT) {
        const float b = sc[q];
        sc[q] = b == INFINITY ? 0.f : merge_scale(0, b, 0, bb[q / gx], inv_lambda, inv_lambda);
    }
    __syncthreads();
    const PeerRow row = peer_row(peers);
    for (int q = tid; q < P; q += NT) {
        const int m = q / P1, e = q % P1;
        const float* src = scratch + (size_t)m * gx * P4 + e;
        const float* scm = sc + m * gx;
        float v = 0.f;
#pragma unroll 4
        for (int g = 0; g < gx; ++g) v += scm[g] * __ldcg(src + (size_t)g * P4);
        if (e == 0) v = bb[m];
        partial[q] = v;
        peer_store(peers, row, q, v);
    }
    if (peers.world > 1) peer_release(peers, row);
    if (tid == 0) *ticket = 0u;
    if (fin_U != nullptr) {
        __threadfence();
        __syncthreads();
        modes_rows(p, nu, partial, 1, P, fin_U, fin_action, fin_stats, fin_mirror, tiles, state);
    }
}

// The last CTA of a K3 launch: fold the per-CTA partials (128-bit L2 loads, 8 in flight per thread), write the shard row, push it into
// every rank's peer window (multi-GPU) and, for single-GPU plans, do K4's work in place.  `tiles` = the idle ring, WsLayout::fold_floats
// at least, `misc` = 8 floats.  The CTA scales come from merge_min / merge_scale over (beta, and with FEASIBLE n_feasible) of every CTA,
// two CTAs per thread; FEASIBLE's row ends with the summed count and the minimum of min V.
template <Rule R>
__device__ __forceinline__ void fold_and_finish(const MppibParams& p, int nu, int P, float* __restrict__ scratch, unsigned int* __restrict__ ticket,
                                                float* __restrict__ partial, const PeerArgs& peers, float* __restrict__ fin_U, float* __restrict__ fin_action,
                                                float* __restrict__ fin_stats, float* __restrict__ fin_mirror, float* tiles, float* misc, float inv_lambda,
                                                float* __restrict__ dist, float* __restrict__ smooth = nullptr, float* __restrict__ anneal = nullptr,
                                                float* __restrict__ spline = nullptr, float* __restrict__ cstate = nullptr) {
    constexpr bool FEAS = R == RULE_FEASIBLE;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = (int)gridDim.x;
    float* sc = tiles;                   // [MAX_GRID] scale of every CTA partial (the ring is idle now)
    float* fold = tiles + MAX_GRID;      // [4][PP]
    {
        float b = (tid < G) ? __ldcg(scratch + (size_t)tid * ((((P + 3) >> 2) << 2))) : INFINITY;
        const float b2 = (tid + NT < G) ? __ldcg(scratch + (size_t)(tid + NT) * ((((P + 3) >> 2) << 2))) : INFINITY;   // CTAs 256..511
        float bb = INFINITY;
        int n1 = 0, n2 = 0, n_all = 0;
        float vmin = INFINITY;
        if constexpr (FEAS) {
            const size_t PP = ((P + 3) >> 2) << 2;
            n1 = tid < G ? __float_as_int(__ldcg(scratch + (size_t)tid * PP + P - 2)) : 0;
            n2 = tid + NT < G ? __float_as_int(__ldcg(scratch + (size_t)(tid + NT) * PP + P - 2)) : 0;
            const float v1 = tid < G ? __ldcg(scratch + (size_t)tid * PP + P - 1) : INFINITY;
            const float v2 = tid + NT < G ? __ldcg(scratch + (size_t)(tid + NT) * PP + P - 1) : INFINITY;
            int ns = n1 + n2;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) ns += __shfl_xor_sync(0xffffffffu, ns, o);
            const float vm = warp_min(fminf(v1, v2));
            if (lane == 0) { misc[warp] = __int_as_float(ns); tiles[warp] = vm; }
            __syncthreads();
#pragma unroll
            for (int w8 = 0; w8 < 8; ++w8) { n_all += __float_as_int(misc[w8]); vmin = fminf(vmin, tiles[w8]); }
            __syncthreads();
        }
        const float bm = warp_min(merge_min(n2, b2, n_all, merge_min(n1, b, n_all)));
        if (lane == 0) misc[warp] = bm;
        __syncthreads();
#pragma unroll
        for (int w8 = 0; w8 < 8; ++w8) bb = fminf(bb, misc[w8]);
        const float inv_lc = FEAS ? 1.0f / p.constraint_lambda : inv_lambda;
        if (tid < G) sc[tid] = (b == INFINITY) ? 0.f : merge_scale(n1, b, n_all, bb, inv_lambda, inv_lc);
        if (tid + NT < G) sc[tid + NT] = (b2 == INFINITY) ? 0.f : merge_scale(n2, b2, n_all, bb, inv_lambda, inv_lc);
        __syncthreads();
        // parallel fold with deep memory-level parallelism: P4 = ceil(P/4) float4 columns x 4 CTA groups of 64 threads;
        // thread (cg, e4) sums CTAs c = cg, cg+4, ... with 8 independent 128-bit L2 loads in flight
        // (scratch rows are padded to a multiple of 4 floats, so every row is 16-byte aligned)
        const int P4 = (P + 3) >> 2, PP = P4 << 2;
        const int cg = tid >> 6, e4 = tid & 63;
        for (int e = e4; e < P4; e += 64) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            int c = cg;
            for (; c + 60 < G; c += 64) {        // 16 independent 128-bit loads in flight: 132 CTA rows are two to three L2 round trips
                float4 v[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) v[u] = __ldcg(reinterpret_cast<const float4*>(scratch + (size_t)(c + 4 * u) * PP) + e);
#pragma unroll
                for (int u = 0; u < 16; ++u) { const float sc_ = sc[c + 4 * u]; acc.x += sc_ * v[u].x; acc.y += sc_ * v[u].y; acc.z += sc_ * v[u].z; acc.w += sc_ * v[u].w; }
            }
            for (; c + 28 < G; c += 32) {
                float4 v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) v[u] = __ldcg(reinterpret_cast<const float4*>(scratch + (size_t)(c + 4 * u) * PP) + e);
#pragma unroll
                for (int u = 0; u < 8; ++u) { const float sc_ = sc[c + 4 * u]; acc.x += sc_ * v[u].x; acc.y += sc_ * v[u].y; acc.z += sc_ * v[u].z; acc.w += sc_ * v[u].w; }
            }
            for (; c < G; c += 4) {
                const float4 v = __ldcg(reinterpret_cast<const float4*>(scratch + (size_t)c * PP) + e);
                const float sc_ = sc[c];
                acc.x += sc_ * v.x; acc.y += sc_ * v.y; acc.z += sc_ * v.z; acc.w += sc_ * v.w;
            }
            reinterpret_cast<float4*>(fold + (size_t)cg * PP)[e] = acc;
        }
        __syncthreads();
        // fused exchange: this rank's row goes straight into the window of every rank (remote stores over NVLink),
        // then one release-store of the arrival flag per peer; K4 on each rank acquires its own flags
        const PeerRow row = peer_row(peers);
        for (int e = tid; e < P; e += NT) {
            const float v0 = fold[e] + fold[PP + e] + fold[2 * PP + e] + fold[3 * PP + e];
            float v = e == 0 ? bb : v0;
            if constexpr (FEAS) v = e == P - 2 ? __int_as_float(n_all) : e == P - 1 ? vmin : v;
            partial[e] = v;
            peer_store(peers, row, e, v);
        }
        if (peers.world > 1) peer_release(peers, row);
        if (tid == 0) *ticket = 0u;
        if (fin_U != nullptr) {
            // single-GPU plans: this CTA is the last one alive and holds the shard row -> do K4's work here (U update, savgol,
            // first action) instead of launching another kernel.  Every CTA read U -- and, with a registered distribution, lambda and
            // cov -- in its prologue, before it took its ticket, so this CTA is the only reader left when it updates them.
            __threadfence();
            __syncthreads();
            if constexpr (R == RULE_SMOOTH) smooth_rows(p, nu, partial, 1, P, fin_U, fin_action, fin_stats, fin_mirror, tiles, smooth);
            else finalize_rows<R>(p, nu, partial, 1, P, fin_U, fin_action, fin_stats, fin_mirror, tiles, dist, nullptr, cstate);
            if constexpr (R == RULE_PLAIN) if (spline) spline_exec(p, nu, tiles, spline);
            if (tid == 0 && anneal) anneal[0] += 1.0f;                        // annealed MPPI: the next iteration's row (every CTA read it)
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// K3, warp-specialised (the default): ONE producer warp streams 32-sample tiles through an NSTAGE-deep ring with TMA, SEVEN
// consumer warps each own WHOLE tiles end to end -- S_k, minimum, weights, weighted row sums, online merge into the warp's own
// running (beta, eta, W) in registers -- so nothing inside the streaming loop is CTA-wide: no __syncthreads, the only
// synchronisation is the full / empty mbarrier pair of a ring stage.
//   tile i of this CTA -> ring stage i % NSTAGE, consumer i % NCONS;  full[s]: TMA complete_tx;  empty[s]: the consumer's arrive
//   per tile and warp: phase A lane = sample (S_k = sum_t gamma^t c[t][k] + sum_r g[r] x[r][k], conflict-free column reads),
//                      phase B warp shuffles (min, exp, sum), weights to a 32-float per-warp strip,
//                      phase C lane = row (r = lane, lane + 32, ...: W[r] += sum_k w_k x[r][k], rotated LDS.128, conflict-free)
// After the loop the seven warp partials are merged once through shared memory; the per-CTA partial, the ticket (last_cta) and
// the last-CTA fold / exchange / fused K4 follow (fold_and_finish).  Every one of these merges, the per-tile one included, is
// merge_min / merge_scale (common.cuh), with the counts 0 but under FEAS.
constexpr int WS_W = 32;          // samples per tile
constexpr int WS_NCONS = 7;       // consumer warps (warp 0 is the producer)

// Shared-memory layout of the kernel with `nstage` ring stages, used by the host for the size and by the kernel for its pointers.
// Offsets in floats from the base, except `bar` (bytes).  The last CTA reuses the ring for the fold (fold_and_finish), so the ring
// region is at least fold_floats long; for every shape but T*nu + T <= 2 the ring stages alone are longer.  With the C row (RULE_FULL)
// the fused K4 also keeps its covariance scratch there (full_fin_floats), which the ring stages of every accepted shape exceed.
struct WsLayout {
    int g, gp, wk, cpart, misc;   // [NR4] lambda Sigma^-1 U | [T4] gamma^t | [8][32] weights | [nparts][P4] warp partials | [8]
    int us;                       // smooth: [NR4] U for the smoothness cost (no floats otherwise)
    int bar;                      // full[nstage], then empty[nstage] mbarriers
    int bytes;                    // + 128 bytes of headroom: the ring depth of every shape stays what it was tuned at
    // row: the rule whose shard row the warp partials hold; nparts: warp partials stored, by default one per consumer warp
    // (min(nstage, WS_NCONS): the launch rounds the ring depth down to a multiple of the consumer count)
    // T: the cost rows of a tile, Tc: the control rows (ctrl_rows())
    __host__ __device__ WsLayout(int T, int Tc, int nu, int nstage, Rule row, bool update_cov, bool smooth = false, int nparts = -1, int modes = 1) {
        const int NR = Tc * nu, P4 = (shard_row_floats(row, Tc, nu, update_cov, 1, 0) + 3) & ~3;
        if (nparts < 0) nparts = nstage < WS_NCONS ? nstage : WS_NCONS;
        const int ring = nstage * (NR + (row == RULE_FEASIBLE ? 2 * T : T)) * WS_W, fold_floats = MAX_GRID + 4 * P4;   // FEASIBLE: + viol[T]
        g = ring > fold_floats ? ring : fold_floats;
        if (row == RULE_FULL && g < NR + 1 + full_fin_floats(T, nu)) g = NR + 1 + full_fin_floats(T, nu);
        if (modes > 1 && g < modes_fin_floats(NR, modes, 1)) g = modes_fin_floats(NR, modes, 1);   // the fused K4 of n_modes > 1
        gp = g + ((NR + 3) & ~3);
        wk = gp + ((T + 3) & ~3);
        cpart = wk + 8 * WS_W;
        misc = cpart + nparts * P4;
        us = misc + 8;
        bar = ((us + (smooth ? ((NR + 3) & ~3) : 0)) * 4 + 15) & ~15;
        bytes = bar + 2 * 8 * nstage + 128;
    }
};

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// The template is <RPL, rule, RISK>: rows of W per lane (T*nu <= 32 * RPL), the update rule (PLAIN, DIST, FULL, HORIZON, SMOOTH or
// MODES; CEM has the elite kernel) and the risk flag (PLAIN, DIST and FULL only).  The body names what the rule implies:
// ADAPT (DIST, FULL, HORIZON: a distribution is registered): lambda comes from dist[0]; with update_cov the SIMPLE-mode Sigma^-1 is diag(1 / dist[1 + j])
// and phase C keeps a second running sum per row, M2[r] = sum_k w_k (x[r][k] - c[r])^2 with c = U (MEAN) or 0 (SIMPLE), rescaled
// online like W; the shard row becomes (beta, eta, W[T*nu], M2[T*nu]).  The bytes read from HBM are the same.
// FULL (update_cov with cov_full): the SIMPLE-mode Sigma^-1 is the full one of dist, and instead of M2 every consumer lane keeps the
// lower triangle of sum_t w_k (x_tk - c_t)(x_tk - c_t)^T of its own sample k across tiles (lane = sample: column reads of the tile,
// conflict-free like phase A; c = U staged in g in MEAN mode), rescaled online like W and summed over the warp once after the loop;
// the shard row becomes (beta, eta, W[T*nu], C[nu(nu+1)/2]).
// HZN (update_cov with cov_horizon): the SIMPLE-mode g = lambda Sigma_H^-1 U is read from hz_g (mppib_shift computed it), phase B
// stores every S_k (INFINITY for an invalid sample) to hz_S for the SYRK that follows, and the row this kernel writes is
// (beta, eta, W[n]) only; the SYRK appends C.
// SMOOTH (mode smooth, x = the derivative noise): SIMPLE with gamma = 1, plus omega dt^2 sum_r (U_r + x_rk)^2 in phase A (U staged in
// `us`, four chains in r order; with omega = 0 neither the term nor the `us` region exists, so that the ring, the consumers and the row
// are SIMPLE's), and the fused K4 integrates the state `smooth`.
// RISK (n_worlds = R > 1): phase B replaces the S of every aligned group of R samples by its CVaR score on the group's first lane and
// +inf on the others (risk_score); a tile is 32 samples and every shard starts at a multiple of R, so no group straddles two tiles.
// MODES (n_modes = M > 1): the grid is (gx, M) and CTA (x, m) walks only the tiles that hold samples of mode m, with g = lambda Sigma^-1
// U_m; the lanes of a straddling tile that belong to the other mode are masked (weight 0, not in the minimum).  Its partial is scratch
// row m*gx + x, and the last CTA folds every mode into block m of the row [M][2 + T*nu] (fold_modes_and_finish).
// anneal (annealed MPPI, nullable): the registered schedule of anneal_n iterations; SIMPLE mode scales g_r by r[t] = 1 / s[t]^2 of the
// iteration's row after the lambda product (a schedule of ones changes no bit), and the fused K4 advances the counter.
// FEAS (constraint_mode): a third tensor map brings the T violation rows g of the tile (the tile is (NR + 2T)*32 floats); phase A sums
// V_k = sum_t c[t][k] in t order beside S, phase B weights the tile's feasible lanes by S with lambda when the warp ballot finds one and
// its valid lanes by V with lambda_c otherwise, and every fold merges (n_feasible, b, eta, W) feasibility-first; the row is
// (beta, eta, W, n_feasible bits, min V) and the fused K4 writes cstate.
template <int RPL, Rule R, bool RISK>
__global__ void __launch_bounds__(NT, 1)
mppib_reduce_ws_kernel(const __grid_constant__ MppibParams p, const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_c,
                       int nu, int xbox_rows, int nstage, int ncons, const float* __restrict__ U, float* __restrict__ scratch, unsigned int* __restrict__ ticket,
                       float* __restrict__ partial, const __grid_constant__ PeerArgs peers, float* __restrict__ fin_U, float* __restrict__ fin_action,
                       float* __restrict__ fin_stats, float* __restrict__ fin_mirror, float* __restrict__ dist, float* __restrict__ hz_S,
                       const float* __restrict__ hz_g, float* __restrict__ smooth, float* __restrict__ anneal, int anneal_n,
                       float* __restrict__ spline, const __grid_constant__ CUtensorMap tm_v, float* __restrict__ cstate) {
    constexpr bool ADAPT = rule_adapts(R), FULL = R == RULE_FULL, HZN = R == RULE_HORIZON, SMOOTH = R == RULE_SMOOTH, MODES = R == RULE_MODES;
    constexpr bool FEAS = R == RULE_FEASIBLE;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int K = p.K, T = p.T, Tc = R == RULE_PLAIN ? ctrl_rows(p) : T, NR = Tc * nu;   // knots parameterise PLAIN only
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if constexpr (MODES) U += (size_t)blockIdx.y * NR;                       // this CTA's mode
    const float lam = ADAPT ? dist[0] : p.lambda_;
    const float inv_lambda = 1.0f / lam;
    const float inv_lc = FEAS ? 1.0f / p.constraint_lambda : inv_lambda;     // the merge's violation-kind temperature
    const bool simple = SMOOTH || p.mode == MPPIB_MODE_SIMPLE;
    const bool m2 = R == RULE_DIST && p.update_cov;
    const int npairs = FULL ? nu * (nu + 1) / 2 : 0;
    const int P = shard_row_floats(k3_row_rule(R), Tc, nu, m2, 1, 0);

    const int tile_floats = (NR + (FEAS ? 2 * T : T)) * WS_W;                 // a multiple of 32 floats: stages stay 128-B aligned
    const int NR4 = (NR + 3) & ~3, T4 = (T + 3) & ~3, P4 = (P + 3) & ~3;
    const bool smooth_term = SMOOTH && p.smooth_weight != 0.f;
    const WsLayout L(T, Tc, nu, nstage, k3_row_rule(R), m2, smooth_term, -1, MODES ? p.n_modes : 1);
    float* tiles = reinterpret_cast<float*>(smem_raw);                        // [nstage][(NR+T)*32]
    float* g = tiles + L.g;                                                   // [NR4] lambda * Sigma^-1 U (SIMPLE), zero padded; FULL MEAN: U
    float* gp = tiles + L.gp;                                                 // [T4]  gamma^t, zero padded
    float* wk = tiles + L.wk;                                                 // [8][32] weights of the tile a warp is working on
    float* cpart = tiles + L.cpart;                                           // [NCONS][P4] warp partials (after the loop)
    float* misc = tiles + L.misc;                                             // [8]
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + L.bar);           // [nstage]
    uint64_t* empty = full + nstage;                                          // [nstage]

    int ntiles = (K + WS_W - 1) / WS_W, tile0 = 0, lo = 0, hi = K;            // MODES: the local samples [lo, hi) of this CTA's mode
    if constexpr (MODES) {
        const int m = (int)blockIdx.y, kc = p.mode_samples, ko = (int)p.k_offset;
        lo = max(0, m * kc - ko);
        hi = min(K, (m + 1) * kc - ko);
        tile0 = lo / WS_W;
        ntiles = hi > lo ? (hi + WS_W - 1) / WS_W - tile0 : 0;
    }
    const int my_tiles = (int)blockIdx.x < ntiles ? (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const uint32_t tile_bytes = (uint32_t)tile_floats * 4u;

    auto issue_tile = [&](int i) {   // elected producer lane: TMA tile i of this CTA into ring stage i % nstage
        const int s = i % nstage;
        const int k0 = (tile0 + (int)blockIdx.x + i * (int)gridDim.x) * WS_W;
        float* dst = tiles + (size_t)s * tile_floats;
        mbar_expect_tx(&full[s], tile_bytes);
        for (int r0 = 0; r0 < NR; r0 += xbox_rows) tma_load_2d(dst + (size_t)r0 * WS_W, &tm_x, k0, r0, &full[s]);
        tma_load_2d(dst + (size_t)NR * WS_W, &tm_c, k0, 0, &full[s]);
        if constexpr (FEAS) tma_load_2d(dst + (size_t)(NR + T) * WS_W, &tm_v, k0, 0, &full[s]);
    };
    if (tid == 0) {
        for (int s = 0; s < nstage; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        for (int i = 0; i < nstage && i < my_tiles; ++i) issue_tile(i);   // the first ring fill is in flight while the prologue below runs
    }
    const float* rrow = anneal ? anneal_row(anneal, anneal_n, T, true) : nullptr;
    for (int r = tid; r < NR4; r += NT) {
        float acc = 0.f;
        if (HZN && simple && r < NR) {
            acc = hz_g[r];
        } else if (simple && r < NR) {
            const int t = r / nu, i = r % nu;
            if (FULL) {
                const float* sinv = dist + 1 + 2 * nu * nu;
                for (int j = 0; j < nu; ++j) acc += sinv[i * nu + j] * U[t * nu + j];
            } else if (m2) acc = (1.0f / dist[1 + i]) * U[r];
            else
                for (int j = 0; j < nu; ++j) acc += p.sigma_inv[i * nu + j] * U[t * nu + j];
            acc *= lam;
            if (rrow) acc = __fmul_rn(acc, rrow[t]);                          // annealed MPPI: importance term under N(U, s^2 Sigma)
        }
        if (FULL && !simple && r < NR) acc = U[r];                            // phase A reads g in SIMPLE mode only
        g[r] = acc;
        if (smooth_term && r < NR) tiles[L.us + r] = U[r];
    }
    {
        // gamma^0 = 1 for every accepted gamma: log2f(0) * 0 would be NaN (validate refuses a negative or non-finite gamma)
        const float lg = log2f(p.gamma);
        for (int t = tid; t < T4; t += NT) gp[t] = t == 0 ? 1.f : t < T ? (SMOOTH ? 1.f : exp2f(lg * (float)t)) : 0.f;
    }
    __syncthreads();

    if (warp == 0) {
        // ---------------------------------------------------------------- producer: one elected lane keeps the ring full
        if (lane == 0) {
            for (int i = nstage; i < my_tiles; ++i) {
                const int s = i % nstage, n = i / nstage;
                mbar_wait(&empty[s], (uint32_t)((n - 1) & 1));                // the consumer of tile i - nstage is done with the stage
                issue_tile(i);
            }
        }
    } else if (warp <= ncons) {
        // ---------------------------------------------------------------- consumers: whole tiles, no block-wide synchronisation
        // nstage is a multiple of ncons, so ring stage s is always drained by consumer s % ncons: a consumer waits for phase n of
        // full[s] only after it has itself consumed phase n - 1 (the parity test cannot tell phases two apart)
        const int c = warp - 1;
        float* wme = wk + warp * WS_W;
        float b_run = INFINITY, e_run = 0.f, w_run[RPL];
        int nf_run = 0;                                                       // FEAS: feasible samples merged so far
        float v_run = INFINITY;                                               // FEAS: min V over the valid samples seen
        float m2_run[ADAPT ? RPL : 1], c_row[ADAPT ? RPL : 1];               // second moment and its centre per row (update_cov)
        float c_run[FULL ? MAX_PAIRS : 1];                                    // FULL: this lane's lower triangle of C
#pragma unroll
        for (int q = 0; q < (FULL ? MAX_PAIRS : 1); ++q) c_run[q] = 0.f;
#pragma unroll
        for (int i = 0; i < RPL; ++i) w_run[i] = 0.f;
        if (ADAPT) {
#pragma unroll
            for (int i = 0; i < RPL; ++i) {
                const int r = lane + 32 * i;
                m2_run[i] = 0.f;
                c_row[i] = (m2 && !simple && r < NR) ? U[r] : 0.f;
            }
        }
        for (int i = c; i < my_tiles; i += ncons) {
            const int s = i % nstage;
            const int k0 = (tile0 + (int)blockIdx.x + i * (int)gridDim.x) * WS_W;
            const float* xs = tiles + (size_t)s * tile_floats;                // [NR][32]
            const float* cs = xs + (size_t)NR * WS_W;                         // [T][32]
            mbar_wait(&full[s], (uint32_t)((i / nstage) & 1));
            // ---- A: S of sample k0 + lane (four independent accumulation chains; padded g / gp entries are zero and the
            // rows they would multiply are clamped to a valid one)
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
            for (int t = 0; t < T4; t += 4) {
                const float4 g4 = *reinterpret_cast<const float4*>(gp + t);
                a0 = fmaf(g4.x, cs[t * WS_W + lane], a0);
                a1 = fmaf(g4.y, cs[min(t + 1, T - 1) * WS_W + lane], a1);
                a2 = fmaf(g4.z, cs[min(t + 2, T - 1) * WS_W + lane], a2);
                a3 = fmaf(g4.w, cs[min(t + 3, T - 1) * WS_W + lane], a3);
            }
            if (simple) {
                for (int r = 0; r < NR4; r += 4) {
                    const float4 g4 = *reinterpret_cast<const float4*>(g + r);
                    a0 = fmaf(g4.x, xs[r * WS_W + lane], a0);
                    a1 = fmaf(g4.y, xs[min(r + 1, NR - 1) * WS_W + lane], a1);
                    a2 = fmaf(g4.z, xs[min(r + 2, NR - 1) * WS_W + lane], a2);
                    a3 = fmaf(g4.w, xs[min(r + 3, NR - 1) * WS_W + lane], a3);
                }
            }
            float sum = (a0 + a1) + (a2 + a3);
            if constexpr (SMOOTH) {
                if (smooth_term) {                                            // omega dt^2 sum_r (U_r + x_rk)^2
                    const float* us = tiles + L.us;
                    float q0 = 0.f, q1 = 0.f, q2 = 0.f, q3 = 0.f;
                    int r = 0;
                    for (; r + 4 <= NR; r += 4) {
                        const float v0 = us[r] + xs[r * WS_W + lane], v1 = us[r + 1] + xs[(r + 1) * WS_W + lane];
                        const float v2 = us[r + 2] + xs[(r + 2) * WS_W + lane], v3 = us[r + 3] + xs[(r + 3) * WS_W + lane];
                        q0 = fmaf(v0, v0, q0); q1 = fmaf(v1, v1, q1); q2 = fmaf(v2, v2, q2); q3 = fmaf(v3, v3, q3);
                    }
                    for (; r < NR; ++r) { const float v = us[r] + xs[r * WS_W + lane]; q0 = fmaf(v, v, q0); }
                    sum = fmaf(p.smooth_weight * p.dt * p.dt, (q0 + q1) + (q2 + q3), sum);
                }
            }
            // ---- B: tile minimum, weights, their sum
            const bool valid = (k0 + lane < K) && isfinite(sum) && (!MODES || (k0 + lane >= lo && k0 + lane < hi));
            float S = valid ? sum : INFINITY;
            float inv_l = inv_lambda;
            int nf_c = 0;
            if constexpr (FEAS) {
                const float* vs = cs + (size_t)T * WS_W;                      // [T][32] margins g
                float V = 0.f;
                for (int t = 0; t < T; ++t) V += feas_violation(vs[t * WS_W + lane]);
                const bool ok = valid && isfinite(V);
                const unsigned fb = __ballot_sync(0xffffffffu, ok && V <= p.constraint_tol);
                nf_c = __popc(fb);
                S = fb ? (((fb >> lane) & 1u) ? sum : INFINITY) : (ok ? V : INFINITY);
                if (!fb) inv_l = inv_lc;
                v_run = fminf(v_run, warp_min(ok ? V : INFINITY));
            }
            if constexpr (RISK) S = risk_score(S, p.n_worlds, p.risk_tail, lane);
            if (HZN && k0 + lane < K) hz_S[k0 + lane] = S;
            const float b_c = warp_min(S);
            const float w = (S == INFINITY) ? 0.f : expf(-(S - b_c) * inv_l);
            const float e_c = warp_sum(w);
            // FEAS: a tile without a feasible sample adds nothing once the warp holds one (warp-uniform, like b_c)
            if (b_c != INFINITY && (!FEAS || nf_c > 0 || nf_run == 0)) {
                wme[lane] = w;
                __syncwarp();
                const int n_out = nf_run + nf_c;
                const float b_out = merge_min(nf_c, b_c, n_out, merge_min(nf_run, b_run, n_out));
                const float s_old = (b_run == INFINITY) ? 0.f : merge_scale(nf_run, b_run, n_out, b_out, inv_lambda, inv_lc);
                const float s_new = merge_scale(nf_c, b_c, n_out, b_out, inv_lambda, inv_lc);
                nf_run = n_out;
                // ---- C: weighted row sums, lane = row
                const float4* w4 = reinterpret_cast<const float4*>(wme);
#pragma unroll
                for (int rr = 0; rr < RPL; ++rr) {
                    const int r = lane + 32 * rr;
                    if (r < NR) {
                        const float4* xr = reinterpret_cast<const float4*>(xs + (size_t)r * WS_W);
                        float acc = 0.f;
                        if (ADAPT && m2) {
                            const float cr = c_row[ADAPT ? rr : 0];
                            float acc2 = 0.f;
#pragma unroll
                            for (int j = 0; j < WS_W / 4; ++j) {
                                const int jj = (j + lane) & (WS_W / 4 - 1);
                                const float4 a = xr[jj], b = w4[jj];
                                acc += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
                                const float dx = a.x - cr, dy = a.y - cr, dz = a.z - cr, dw = a.w - cr;
                                acc2 += b.x * dx * dx + b.y * dy * dy + b.z * dz * dz + b.w * dw * dw;
                            }
                            m2_run[ADAPT ? rr : 0] = m2_run[ADAPT ? rr : 0] * s_old + acc2 * s_new;
                        } else {
#pragma unroll
                            for (int j = 0; j < WS_W / 4; ++j) {
                                const int jj = (j + lane) & (WS_W / 4 - 1);   // rotation => conflict-free LDS.128
                                const float4 a = xr[jj], b = w4[jj];
                                acc += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
                            }
                        }
                        w_run[rr] = w_run[rr] * s_old + acc * s_new;
                    }
                }
                if constexpr (FULL) {
                    // ---- C of this lane's sample: lane = sample, column reads (conflict-free), weight rescaled to b_out
                    const float ws = w * s_new;
#pragma unroll
                    for (int q = 0; q < MAX_PAIRS; ++q) if (q < npairs) c_run[q] *= s_old;
                    for (int t = 0; t < T; ++t) {
                        float dx[MPPIB_MAX_NU];
#pragma unroll
                        for (int i = 0; i < MPPIB_MAX_NU; ++i) dx[i] = i < nu ? xs[(t * nu + i) * WS_W + lane] - (simple ? 0.f : g[t * nu + i]) : 0.f;
#pragma unroll
                        for (int i = 0; i < MPPIB_MAX_NU; ++i) {
                            if (i >= nu) break;
                            const float wd = ws * dx[i];
#pragma unroll
                            for (int j = 0; j <= i; ++j) c_run[i * (i + 1) / 2 + j] = fmaf(wd, dx[j], c_run[i * (i + 1) / 2 + j]);
                        }
                    }
                }
                e_run = e_run * s_old + e_c * s_new;
                b_run = b_out;
            }
            __syncwarp();                                                     // every lane is done with the stage and with wme
            if (lane == 0) mbar_arrive(&empty[s]);
        }
        // this warp's partial -> shared memory
        float* mine = cpart + (size_t)c * P4;
        if (lane == 0) { mine[0] = b_run; mine[1] = e_run; }
        if (FEAS && lane == 0) { mine[2 + NR] = __int_as_float(nf_run); mine[3 + NR] = v_run; }
#pragma unroll
        for (int rr = 0; rr < RPL; ++rr) { const int r = lane + 32 * rr; if (r < NR) mine[2 + r] = w_run[rr]; }
        if (ADAPT && m2) {
#pragma unroll
            for (int rr = 0; rr < RPL; ++rr) { const int r = lane + 32 * rr; if (r < NR) mine[2 + NR + r] = m2_run[ADAPT ? rr : 0]; }
        }
        if constexpr (FULL) {
#pragma unroll
            for (int q = 0; q < MAX_PAIRS; ++q) {
                if (q >= npairs) break;
                const float v = warp_sum(c_run[q]);
                if (lane == 0) mine[2 + NR + q] = v;
            }
        }
    }
    // (a spare warp -- fewer ring stages than warps -- has no partial: the layout stores the ncons consumers' only)
    __syncthreads();
    // ---- merge the warp partials into the CTA partial (global scratch), then ticket -> the last CTA folds all of them
    {
        float* mine = scratch + (size_t)(blockIdx.x + (MODES ? blockIdx.y * gridDim.x : 0u)) * P4;
        float bb = INFINITY;
        float sc[WS_NCONS];
        int n_all = 0;
        float vmin = INFINITY;
        auto nf_of = [=](int c) { return FEAS && c < ncons ? __float_as_int(cpart[(size_t)c * P4 + 2 + NR]) : 0; };
        if constexpr (FEAS) {
#pragma unroll
            for (int c = 0; c < WS_NCONS; ++c) if (c < ncons) { n_all += nf_of(c); vmin = fminf(vmin, cpart[(size_t)c * P4 + 3 + NR]); }
        }
#pragma unroll
        for (int c = 0; c < WS_NCONS; ++c) if (c < ncons) bb = merge_min(nf_of(c), cpart[(size_t)c * P4], n_all, bb);
#pragma unroll
        for (int c = 0; c < WS_NCONS; ++c) {
            const float bc = c < ncons ? cpart[(size_t)c * P4] : INFINITY;
            sc[c] = (bc == INFINITY) ? 0.f : merge_scale(nf_of(c), bc, n_all, bb, inv_lambda, inv_lc);
        }
        for (int e = tid; e < P; e += NT) {
            float v = 0.f;
#pragma unroll
            for (int c = 0; c < WS_NCONS; ++c) if (c < ncons) v += sc[c] * cpart[(size_t)c * P4 + e];
            if constexpr (FEAS) v = e == 2 + NR ? __int_as_float(n_all) : e == 3 + NR ? vmin : v;
            mine[e] = e == 0 ? bb : v;
        }
    }
    if (!last_cta(ticket, MODES ? gridDim.x * gridDim.y : gridDim.x)) return;
    // the horizon K3 folds as DIST's does; it gets no fin_U and no peers, the SYRK finishes its row
    if constexpr (MODES) fold_modes_and_finish(p, nu, P, scratch, ticket, partial, peers, fin_U, fin_action, fin_stats, fin_mirror, tiles, inv_lambda, dist);
    else fold_and_finish<HZN ? RULE_DIST : R>(p, nu, P, scratch, ticket, partial, peers, fin_U, fin_action, fin_stats, fin_mirror, tiles, misc, inv_lambda,
                                              dist, smooth, anneal, spline, cstate);
}

// K4: combine G shard partials, U update, optional Savitzky-Golay (window 9, order 2, 'interp' edges), action out; DIST / FULL /
// HORIZON: the distribution update of finalize_rows (FULL: of the full covariance, HORIZON: of the covariance over the horizon); SMOOTH:
// smooth_rows; MODES: modes_rows (n_modes > 1, dist = the mode state).  anneal (annealed MPPI, nullable): the counter of the registered
// schedule is advanced by one after the update.
template <Rule R>
__global__ void __launch_bounds__(256)
mppib_finalize_kernel(const __grid_constant__ MppibParams p, int nu, const float* __restrict__ partials_in, int G,
                float* __restrict__ U, float* __restrict__ action_out, float* __restrict__ stats, const __grid_constant__ PeerArgs peers,
                float* __restrict__ action_mirror, float* __restrict__ dist, float* __restrict__ hz_sig, float* __restrict__ smooth,
                float* __restrict__ anneal, float* __restrict__ spline, float* __restrict__ cstate) {
    extern __shared__ float un[];   // [T*nu] then [G] scales (then [T*nu] variances with update_cov, or full_fin_floats with FULL)
    const float* partials = partials_in;
    int P = shard_row_floats(R, p, nu);                                       // row stride of the partials
    uint32_t seq = 0;
    if (partials_in == nullptr) {                                             // rows come from this rank's peer window
        const PeerRows w = peer_acquire(peers, G);
        partials = w.rows;
        P = w.stride;
        seq = w.seq;
    }
    if constexpr (R == RULE_MODES) modes_rows(p, nu, partials, G, P, U, action_out, stats, action_mirror, un, dist);
    else if constexpr (R == RULE_SMOOTH) smooth_rows(p, nu, partials, G, P, U, action_out, stats, action_mirror, un, smooth);
    else finalize_rows<R>(p, nu, partials, G, P, U, action_out, stats, action_mirror, un, dist, hz_sig, cstate);
    if constexpr (R == RULE_PLAIN) if (spline) spline_exec(p, nu, un, spline);
    if (threadIdx.x == 0 && partials_in == nullptr) peer_consume(peers, seq);
    if (threadIdx.x == 0 && anneal) anneal[0] += 1.0f;
}

// ------------------------------------------------------------------------------------------------------------------
// cov_horizon: the weighted SYRK after K3.  C = sum_k w_k (x_k - c)(x_k - c)^T over the n-vectors x_k = x[:, k] (n = T*nu),
// w_k = exp(-(S_k - beta)/lambda) with S_k from K3 (hz_S) and beta = partial[0] from K3's row, c = U (MEAN) or 0 (SIMPLE).
//   grid = lower-triangle 64 x 64 output tiles x ksplit K-chunks; 256 threads, a 4 x 4 register block each; 32 samples at a time
//   are staged to shared memory (weighted, centred rows of the tile's row block, centred rows of its column block; the next 32
//   are loaded into registers meanwhile), FP32 FFMA in sample order.
//   The last CTA of a tile (ticket) folds the ksplit partial tiles in split order and writes its entries of the packed lower
//   triangle into the shard row; the last tile to finish pushes the whole row into the peer windows (multi-GPU) and, for
//   single-GPU plans (fin_U != NULL), does K4's work in place, as K3's last CTA does for the other rules.
constexpr int HZ_KB = 32;   // samples per staged chunk

__global__ void __launch_bounds__(256, 1)
mppib_syrk_kernel(const __grid_constant__ MppibParams p, int nu, int ksplit, int kchunk, const float* __restrict__ x, const float* __restrict__ U,
                  const float* __restrict__ S, float* __restrict__ partial, float* __restrict__ scr, unsigned int* __restrict__ ticket,
                  const __grid_constant__ PeerArgs peers, float* __restrict__ fin_U, float* __restrict__ fin_action, float* __restrict__ fin_stats,
                  float* __restrict__ fin_mirror, float* __restrict__ dist, float* __restrict__ hz_sig) {
    extern __shared__ __align__(16) float hsm[];
    const int n = p.T * nu, K = p.K, P = shard_row_floats(RULE_HORIZON, p, nu);
    const int tid = threadIdx.x;
    const int nb = (n + HZ_TILE - 1) / HZ_TILE, ntiles = nb * (nb + 1) / 2;
    const int tile = (int)blockIdx.x / ksplit, split = (int)blockIdx.x % ksplit;
    int bi = 0;
    while (tri(bi + 1) <= tile) ++bi;
    const int bj = tile - tri(bi);
    const int i0 = bi * HZ_TILE, j0 = bj * HZ_TILE;
    float* As = hsm;                        // [HZ_KB][64] w_k (x[i0 + r][k] - c), sample-major
    float* Bs = hsm + HZ_KB * HZ_TILE;      // [HZ_KB][64] x[j0 + r][k] - c
    const float inv_lambda = 1.0f / dist[0];
    const float beta = __ldcg(&partial[0]);
    const bool simple = p.mode == MPPIB_MODE_SIMPLE;
    // loader: row lr of both blocks, samples lk .. lk + 7 of the chunk
    const int lr = tid & (HZ_TILE - 1), lk = (tid >> 6) * 8;
    const int ra = i0 + lr, rb = j0 + lr;
    const float ca = (!simple && ra < n) ? U[ra] : 0.f, cb = (!simple && rb < n) ? U[rb] : 0.f;
    const int ty = tid >> 4, tx = tid & 15;
    const int kbeg = split * kchunk, kend = min(K, kbeg + kchunk);
    float va[8], vb[8], wv[8];
    auto load = [&](int k0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int k = k0 + lk + 4 * h;                                    // kend is a multiple of 4: a float4 is all in or all out
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a, sv = make_float4(INFINITY, INFINITY, INFINITY, INFINITY);
            if (k < kend) {
                if (ra < n) a = __ldcs(reinterpret_cast<const float4*>(x + (size_t)ra * K + k));
                if (rb < n) b = __ldcs(reinterpret_cast<const float4*>(x + (size_t)rb * K + k));
                sv = __ldg(reinterpret_cast<const float4*>(S + k));
            }
            va[4 * h] = a.x; va[4 * h + 1] = a.y; va[4 * h + 2] = a.z; va[4 * h + 3] = a.w;
            vb[4 * h] = b.x; vb[4 * h + 1] = b.y; vb[4 * h + 2] = b.z; vb[4 * h + 3] = b.w;
            wv[4 * h] = sv.x; wv[4 * h + 1] = sv.y; wv[4 * h + 2] = sv.z; wv[4 * h + 3] = sv.w;
        }
    };
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
    if (kbeg < kend) load(kbeg);
    for (int k0 = kbeg; k0 < kend; k0 += HZ_KB) {
        __syncthreads();                                                      // the previous chunk is consumed
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float w = isfinite(wv[e]) ? expf(-(wv[e] - beta) * inv_lambda) : 0.f;
            As[(lk + e) * HZ_TILE + lr] = ra < n ? w * (va[e] - ca) : 0.f;
            Bs[(lk + e) * HZ_TILE + lr] = rb < n ? vb[e] - cb : 0.f;
        }
        __syncthreads();
        if (k0 + HZ_KB < kend) load(k0 + HZ_KB);                              // in flight while this chunk is multiplied
#pragma unroll 8
        for (int kk = 0; kk < HZ_KB; ++kk) {
            const float4 a4 = *reinterpret_cast<const float4*>(As + kk * HZ_TILE + ty * 4);
            const float4 b4 = *reinterpret_cast<const float4*>(Bs + kk * HZ_TILE + tx * 4);
            const float av[4] = {a4.x, a4.y, a4.z, a4.w}, bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(av[a], bv[b], acc[a][b]);
        }
    }
    float* mine = scr + ((size_t)tile * ksplit + split) * (HZ_TILE * HZ_TILE);
#pragma unroll
    for (int a = 0; a < 4; ++a)
        reinterpret_cast<float4*>(mine + (ty * 4 + a) * HZ_TILE)[tx] = make_float4(acc[a][0], acc[a][1], acc[a][2], acc[a][3]);
    if (!last_cta(&ticket[tile], (unsigned)ksplit)) return;
    // the tile's last CTA: fold the splits in order, write the packed lower-triangle entries of the tile
    const float* base = scr + (size_t)tile * ksplit * (HZ_TILE * HZ_TILE);
    for (int q = tid; q < HZ_TILE * HZ_TILE; q += blockDim.x) {
        const int li = q / HZ_TILE, lj = q % HZ_TILE, gi = i0 + li, gj = j0 + lj;
        if (gi >= n || gj > gi) continue;
        float c = 0.f;
        for (int sp = 0; sp < ksplit; ++sp) c += __ldcg(base + (size_t)sp * (HZ_TILE * HZ_TILE) + q);
        partial[2 + n + tri(gi) + gj] = c;
    }
    if (tid == 0) ticket[tile] = 0u;
    if (!last_cta(&ticket[HZ_MAX_TILES], (unsigned)ntiles)) return;
    if (tid == 0) ticket[HZ_MAX_TILES] = 0u;
    if (peers.world > 1) {
        // the complete row goes into the window of every rank, then one release-store of the arrival flag per peer (as in
        // fold_and_finish)
        const PeerRow row = peer_row(peers);
        for (int e = tid; e < P; e += blockDim.x) peer_store(peers, row, e, __ldcg(&partial[e]));
        peer_release(peers, row);
    }
    if (fin_U != nullptr) {
        // single-GPU plans: every CTA read U and lambda before it took its ticket, so this CTA is the only reader left
        __syncthreads();
        finalize_rows<RULE_HORIZON>(p, nu, partial, 1, P, fin_U, fin_action, fin_stats, fin_mirror, hsm, dist, hz_sig);
    }
}

// hz_g (cov_horizon with a registered distribution, SIMPLE mode): g = lambda Sigma_H^-1 U of the shifted U, once per plan, for K3's
// control cost (a row of Sigma_H^-1 per thread, summed in column order).  anneal (annealed MPPI, nullable): the plan starts at
// iteration 0, so the counter of the registered schedule is reset.
// spline (spline MPPI, nullable): the knots shift by the table's shift rows (count 0: u_init) instead of by one step.
__global__ void mppib_shift_kernel(const __grid_constant__ MppibParams p, int nu, float* __restrict__ U, uint32_t* __restrict__ plan_ctr,
                                   const float* __restrict__ dist, float* __restrict__ hz_g, float* __restrict__ anneal,
                                   const float* __restrict__ spline) {
    extern __shared__ float tmp[];
    const int NR = ctrl_rows(p) * nu;
    for (int r = threadIdx.x; r < NR; r += blockDim.x) {
        if (spline) {
            const float* row = spline + (size_t)(p.T + r / nu) * spline_row_floats(p.spline_degree);
            tmp[r] = row[1] > 0.f ? spline_apply(row, U + r % nu, nu) : p.u_init[r % nu];
        } else {
            tmp[r] = r + nu < NR ? U[r + nu] : p.u_init[r % nu];
        }
    }
    __syncthreads();
    for (int r = threadIdx.x; r < NR; r += blockDim.x) U[r] = tmp[r];
    if (threadIdx.x == 0 && plan_ctr) *plan_ctr += 1u;
    if (threadIdx.x == 0 && anneal) anneal[0] = 0.f;
    if (hz_g != nullptr) {
        const float lam = dist[0];
        const float* sinv = dist + 1 + 2 * (size_t)NR * NR;
        for (int r = threadIdx.x; r < NR; r += blockDim.x) {
            float acc = 0.f;
#pragma unroll 4
            for (int c = 0; c < NR; ++c) acc += sinv[(size_t)r * NR + c] * tmp[c];
            hz_g[r] = lam * acc;
        }
    }
}

// n_modes = M > 1: every mode of U[M][T][nu] shifts as U does (the appended step is u_init)
__global__ void mppib_shift_modes_kernel(const __grid_constant__ MppibParams p, int nu, float* __restrict__ U, uint32_t* __restrict__ plan_ctr) {
    extern __shared__ float tmp[];
    const int NR = p.T * nu, MN = p.n_modes * NR;
    for (int q = threadIdx.x; q < MN; q += blockDim.x) tmp[q] = q % NR + nu < NR ? U[q + nu] : p.u_init[q % nu];
    __syncthreads();
    for (int q = threadIdx.x; q < MN; q += blockDim.x) U[q] = tmp[q];
    if (threadIdx.x == 0 && plan_ctr) *plan_ctr += 1u;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

// row-major [rows][K] float32 tensor, box = box_rows x W columns, zero fill out of bounds, no swizzle
int make_map(CUtensorMap* tm, const float* base, int rows, int K, int box_rows, int W) {
    EncodeTiledFn enc = get_encode();
    MPPIB_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)K * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)W, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MPPIB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d) for rows=%d K=%d box=%dx%d", (int)r, rows, K, box_rows, W);
    return 0;
}

// smooth, anneal: the state of mode smooth and the annealing schedule, for the rules that read them (nullptr otherwise)
template <int RPL, Rule R, bool RISK>
int launch_reduce_ws_t(MppibContext* c, const float* cost, const float* x, const float* U, float* partial, float* fin_U, float* fin_action,
                       float* fin_stats, float* smooth, float* anneal, cudaStream_t s) {
    const int T = c->params.T, Tc = ctrl_rows(c->params), nu = c->model.nu, NR = Tc * nu, K = c->params.K;
    // consumers = min(7, stages that fit); the ring depth is rounded down to a multiple of the consumer count so that a stage always
    // belongs to the same consumer (see the kernel)
    // The horizon K3 sizes its ring for the M2 row of update_cov, which it does not write: its kernel addresses the W layout
    // (DESIGN.md, "The horizon K3's ring is sized for a row it does not write").
    const Rule row = R == RULE_HORIZON ? RULE_DIST : k3_row_rule(R);
    const bool smooth_term = R == RULE_SMOOTH && c->params.smooth_weight != 0.f;   // the `us` region of the kernel's layout
    const int nstage_max = reduce_ws_stages(c->params, nu, row, smooth_term);
    const int ncons = nstage_max < WS_NCONS ? nstage_max : WS_NCONS;
    const int nstage = ncons * (nstage_max / ncons);
    const int modes = R == RULE_MODES ? c->params.n_modes : 1;
    const size_t smem = WsLayout(T, Tc, nu, nstage, row, c->params.update_cov, smooth_term, -1, modes).bytes;
    if (int rc = ensure_smem<mppib_reduce_ws_kernel<RPL, R, RISK>>(c->device, smem)) return rc;
    int xbox_rows = NR < 256 ? NR : 256;
    while (NR % xbox_rows != 0) --xbox_rows;
    // tensor maps are rebuilt only when a buffer, the shape or the device changes (the eager / stepwise path calls this per plan)
    // FEASIBLE: the violation rows get a map of their own (tm_v), built like the cost's; the other rules pass the cost map in its place
    struct MapCache { const void* x; const void* c; const void* v; int K, T, NR, dev; CUtensorMap tm_x, tm_c, tm_v; };
    static thread_local MapCache mc = {nullptr, nullptr, nullptr, 0, 0, 0, -1, {}, {}, {}};
    if (mc.x != x || mc.c != cost || mc.K != K || mc.T != T || mc.NR != NR || mc.dev != c->device) {
        if (int rc = make_map(&mc.tm_x, x, NR, K, xbox_rows, WS_W)) return rc;
        if (int rc = make_map(&mc.tm_c, cost, T, K, T, WS_W)) return rc;
        mc.x = x; mc.c = cost; mc.K = K; mc.T = T; mc.NR = NR; mc.dev = c->device;
        mc.v = nullptr;
    }
    if (R == RULE_FEASIBLE && mc.v != c->viol) {
        if (int rc = make_map(&mc.tm_v, c->viol, T, K, T, WS_W)) return rc;
        mc.v = c->viol;
    }
    const int ntiles = (K + WS_W - 1) / WS_W;
    int grid = ntiles < c->num_sms ? ntiles : c->num_sms;
    if (grid > MAX_GRID) grid = MAX_GRID;
    if (R == RULE_MODES) {
        // gx CTAs per mode, about one per SM over all modes, no more than the tiles of the largest mode's local range
        int tmax = 0;
        for (int m = 0; m < modes; ++m) {
            const long long lo = std::max(0LL, (long long)m * c->params.mode_samples - c->params.k_offset);
            const long long hi = std::min((long long)K, (long long)(m + 1) * c->params.mode_samples - c->params.k_offset);
            if (hi > lo) tmax = std::max(tmax, (int)((hi + WS_W - 1) / WS_W - lo / WS_W));
        }
        grid = std::max(1, std::min(tmax, c->num_sms / modes));
        MPPIB_REQUIRE((long long)grid * modes * ((2 + NR + 3) & ~3) <= (long long)c->reduce_max_ctas * (((long long)partial_row_capacity(c->params, nu) + 3) & ~3LL),
                      "mppib_reduce: scratch too small");
    }
    MPPIB_REQUIRE(grid <= c->reduce_max_ctas, "mppib_reduce: scratch too small");
    PeerArgs peers = reduce_peers(c);
    if (R == RULE_HORIZON) peers.world = 0;                                   // the row is complete only after the SYRK, which stores it
    mppib_reduce_ws_kernel<RPL, R, RISK><<<dim3(grid, modes), NT, smem, s>>>(c->params, mc.tm_x, mc.tm_c, nu, xbox_rows, nstage, ncons, U, c->reduce_scratch,
                                                                             c->reduce_ticket, partial, peers, fin_U, fin_action, fin_stats,
                                                                             fin_U ? c->action_mirror : nullptr, c->dist, c->hz_S, c->hz_g, smooth, anneal,
                                                                             c->anneal_n, R == RULE_PLAIN ? live_spline(c) : nullptr,
                                                                             R == RULE_FEASIBLE ? mc.tm_v : mc.tm_c, R == RULE_FEASIBLE ? c->cstate : nullptr);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// the RPL ladder: T*nu <= 32 * RPL rows of W per lane (the horizon rule's n = T*nu <= 256 stops at 8)
template <Rule R, bool RISK>
int launch_reduce_rule(MppibContext* c, const float* cost, const float* x, const float* U, float* partial, float* fin_U, float* fin_action,
                       float* fin_stats, float* smooth, float* anneal, cudaStream_t s) {
    const int NR = ctrl_rows(c->params) * c->model.nu;
    if (NR <= 32 * 4) return launch_reduce_ws_t<4, R, RISK>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, smooth, anneal, s);
    if constexpr (R != RULE_HORIZON) {
        if (NR > 32 * 8) return launch_reduce_ws_t<16, R, RISK>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, smooth, anneal, s);
    }
    return launch_reduce_ws_t<8, R, RISK>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, smooth, anneal, s);
}

// ksplit x chunk length of the SYRK: about one CTA per SM over the lower-triangle tiles, chunks a multiple of HZ_KB samples
static void syrk_split(const MppibContext* c, int n, int* ntiles, int* ksplit, int* kchunk) {
    const int nb = (n + HZ_TILE - 1) / HZ_TILE, K = c->params.K;
    *ntiles = nb * (nb + 1) / 2;
    int ks = c->num_sms / *ntiles;
    if (ks < 1) ks = 1;
    int kc = (K + ks - 1) / ks;
    kc = (kc + HZ_KB - 1) / HZ_KB * HZ_KB;
    *kchunk = kc;
    *ksplit = (K + kc - 1) / kc;
}

static int hz_fin_smem(int n, int G) { return (int)sizeof(float) * (n + G + hz_fin_floats(n)); }

int launch_syrk(MppibContext* c, const float* x, const float* U, float* partial, float* fin_U, float* fin_action, float* fin_stats, cudaStream_t s) {
    const int n = c->params.T * c->model.nu;
    int ntiles, ksplit, kchunk;
    syrk_split(c, n, &ntiles, &ksplit, &kchunk);
    MPPIB_REQUIRE((size_t)ntiles * ksplit * HZ_TILE * HZ_TILE <= (size_t)c->hz_scr_floats, "mppib_reduce: SYRK scratch too small");
    int smem = (int)sizeof(float) * 2 * HZ_KB * HZ_TILE;
    if (fin_U != nullptr && hz_fin_smem(n, 1) > smem) smem = hz_fin_smem(n, 1);
    if (int rc = ensure_smem<mppib_syrk_kernel>(c->device, smem)) return rc;
    mppib_syrk_kernel<<<ntiles * ksplit, 256, smem, s>>>(c->params, c->model.nu, ksplit, kchunk, x, U, c->hz_S, partial, c->hz_scr, c->hz_ticket,
                                                         reduce_peers(c), fin_U, fin_action, fin_stats, fin_U ? c->action_mirror : nullptr, c->dist,
                                                         c->hz_sig);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

// The ring depth: the deepest ring (<= 8 stages) that fits next to seven warp partials of the rule's row, the depths every shape was
// tuned at.  Where that leaves fewer than two stages (the second-moment row at T = 256, T*nu = 512), two stages fit next to their two
// consumers'.
int reduce_ws_stages(const MppibParams& p, int nu, Rule row, bool smooth) {
    int ns = 8;
    while (ns > 1 && WsLayout(p.T, ctrl_rows(p), nu, ns, row, p.update_cov, smooth, WS_NCONS).bytes > 224 * 1024) --ns;
    if (ns < 2 && WsLayout(p.T, ctrl_rows(p), nu, 2, row, p.update_cov, smooth).bytes <= 224 * 1024) ns = 2;
    return ns;
}

int alloc_horizon(MppibContext* c) {
    const bool on = c->params.update_cov && c->params.cov_horizon;
    const int K = c->params.K, n = c->params.T * c->model.nu;
    if (on && c->hz_S && c->hz_K == K && c->hz_n == n) return 0;
    if (c->hz_S) cudaFree(c->hz_S);
    if (c->hz_g) cudaFree(c->hz_g);
    if (c->hz_sig) cudaFree(c->hz_sig);
    if (c->hz_scr) cudaFree(c->hz_scr);
    if (c->hz_ticket) cudaFree(c->hz_ticket);
    c->hz_S = c->hz_g = c->hz_sig = c->hz_scr = nullptr;
    c->hz_ticket = nullptr;
    c->hz_K = c->hz_n = c->hz_scr_floats = 0;
    if (!on) return 0;
    const int tiles = c->num_sms > HZ_MAX_TILES ? c->num_sms : HZ_MAX_TILES;  // ntiles * ksplit of syrk_split never exceeds this
    c->hz_scr_floats = tiles * HZ_TILE * HZ_TILE;
    MPPIB_CHECK_CUDA(cudaMalloc(&c->hz_S, sizeof(float) * (size_t)((K + 3) & ~3)));
    MPPIB_CHECK_CUDA(cudaMalloc(&c->hz_g, sizeof(float) * (size_t)n));
    MPPIB_CHECK_CUDA(cudaMemset(c->hz_g, 0, sizeof(float) * (size_t)n));
    MPPIB_CHECK_CUDA(cudaMalloc(&c->hz_sig, sizeof(float) * (size_t)n * n));
    MPPIB_CHECK_CUDA(cudaMalloc(&c->hz_scr, sizeof(float) * (size_t)c->hz_scr_floats));
    MPPIB_CHECK_CUDA(cudaMalloc(&c->hz_ticket, sizeof(unsigned int) * (HZ_MAX_TILES + 1)));
    MPPIB_CHECK_CUDA(cudaMemset(c->hz_ticket, 0, sizeof(unsigned int) * (HZ_MAX_TILES + 1)));
    c->hz_K = K;
    c->hz_n = n;
    return 0;
}

int launch_reduce(MppibContext* c, const float* cost, const float* x, const float* U, float* partial, float* fin_U, float* fin_action,
                  float* fin_stats, cudaStream_t s) {
    const Rule rule = update_rule(c);
    if (rule == RULE_CEM) return launch_elite(c, cost, x, partial, fin_U, fin_action, fin_stats, s);   // none of K3's limits apply
    const int T = c->params.T, nu = c->model.nu;
    MPPIB_REQUIRE(c->params.K >= 4 && c->params.K % 4 == 0, "mppib_reduce: K=%d must be a positive multiple of 4 (16-byte rows for TMA / 128-bit loads)", c->params.K);
    MPPIB_REQUIRE(ctrl_rows(c->params) * nu <= 32 * 16, "mppib_reduce: %s = %d exceeds %d", c->params.control_knots > 0 ? "P*nu" : "T*nu",
                  ctrl_rows(c->params) * nu, 32 * 16);
    MPPIB_REQUIRE(T <= 256, "mppib_reduce: T = %d exceeds the 256-row TMA box", T);
    MPPIB_REQUIRE(reduce_ws_stages(c->params, nu, RULE_PLAIN) >= 2, "mppib_reduce: T = %d, nu = %d leaves room for fewer than two ring stages", T, nu);
    MPPIB_REQUIRE(!adaptive_cov(c) || adaptive_full(c) || reduce_ws_stages(c->params, nu, RULE_DIST) >= 2,
                  "mppib_reduce: T = %d, nu = %d leaves room for fewer than two ring stages with the second-moment row of update_cov", T, nu);
    MPPIB_REQUIRE(!adaptive_full(c) || reduce_ws_stages(c->params, nu, RULE_FULL) >= 2,
                  "mppib_reduce: T = %d, nu = %d leaves room for fewer than two ring stages with the covariance row of cov_full", T, nu);
    const int NR = T * nu;
    const bool risk = risk_mode(c);
    if (risk) {
        const int R = c->params.n_worlds;
        MPPIB_REQUIRE(c->params.K % R == 0 && c->params.k_offset % (uint32_t)R == 0, "mppib_reduce: n_worlds = %d needs K = %d and k_offset = %u to be multiples of it",
                      R, c->params.K, c->params.k_offset);
        MPPIB_REQUIRE(rule != RULE_HORIZON, "mppib_reduce: n_worlds > 1 excludes cov_horizon");
    }
    // the annealing schedule is read by the K3 of PLAIN, DIST and FULL, the smooth state by SMOOTH's
    switch (rule) {
    case RULE_MODES:
        MPPIB_REQUIRE(c->dist != nullptr, "mppib_reduce: n_modes > 1 needs its mode state registered with mppib_set_distribution");
        return launch_reduce_rule<RULE_MODES, false>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, nullptr, nullptr, s);
    case RULE_SMOOTH:
        MPPIB_REQUIRE(c->smooth != nullptr, "mppib_reduce: mode smooth needs its state registered with mppib_set_smooth_state");
        MPPIB_REQUIRE(reduce_ws_stages(c->params, nu, RULE_SMOOTH, true) >= 2, "mppib_reduce: T = %d, nu = %d leaves room for fewer than two ring stages in mode smooth", T, nu);
        return launch_reduce_rule<RULE_SMOOTH, false>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, c->smooth, nullptr, s);
    case RULE_HORIZON: {
        MPPIB_REQUIRE(NR <= MPPIB_HZ_MAX_N, "mppib_reduce: cov_horizon needs n = T*nu <= %d, got %d", MPPIB_HZ_MAX_N, NR);
        MPPIB_REQUIRE(c->hz_S != nullptr && c->hz_K == c->params.K && c->hz_n == NR, "mppib_reduce: cov_horizon buffers are not sized for K = %d, n = %d",
                      c->params.K, NR);
        const int rc = launch_reduce_rule<RULE_HORIZON, false>(c, cost, x, U, partial, nullptr, nullptr, nullptr, nullptr, nullptr, s);
        if (rc) return rc;
        return launch_syrk(c, x, U, partial, fin_U, fin_action, fin_stats, s);
    }
    case RULE_FEASIBLE:
        MPPIB_REQUIRE(reduce_ws_stages(c->params, nu, RULE_FEASIBLE) >= 2, "mppib_reduce: T = %d, nu = %d leaves room for fewer than two ring stages with the violation rows of constraint_mode", T, nu);
        return launch_reduce_rule<RULE_FEASIBLE, false>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, nullptr, nullptr, s);
    case RULE_FULL:
        return risk ? launch_reduce_rule<RULE_FULL, true>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, nullptr, c->anneal, s)
                    : launch_reduce_rule<RULE_FULL, false>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, nullptr, c->anneal, s);
    case RULE_DIST:
        return risk ? launch_reduce_rule<RULE_DIST, true>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, nullptr, c->anneal, s)
                    : launch_reduce_rule<RULE_DIST, false>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, nullptr, c->anneal, s);
    default:   // RULE_PLAIN
        return risk ? launch_reduce_rule<RULE_PLAIN, true>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, nullptr, c->anneal, s)
                    : launch_reduce_rule<RULE_PLAIN, false>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, nullptr, c->anneal, s);
    }
}

// one K4 launch; dist, hz_sig, smooth, anneal: the buffers the rule reads (nullptr otherwise)
template <Rule R>
static int launch_finalize_t(MppibContext* c, const float* partials, int G, float* U, float* action_out, float* stats, size_t smem, float* dist,
                             float* hz_sig, float* smooth, float* anneal, cudaStream_t s) {
    mppib_finalize_kernel<R><<<1, 256, smem, s>>>(c->params, c->model.nu, partials, G, U, action_out, stats, peer_args(c), c->action_mirror, dist, hz_sig,
                                                  smooth, anneal, R == RULE_PLAIN ? live_spline(c) : nullptr, R == RULE_FEASIBLE ? c->cstate : nullptr);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_finalize(MppibContext* c, const float* partials, int G, float* U, float* action_out, float* stats, cudaStream_t s) {
    const int NR = ctrl_rows(c->params) * c->model.nu;
    const size_t un = (NR + G) * sizeof(float);                               // U and the G scales, the shared floats of every rule
    switch (update_rule(c)) {
    case RULE_CEM:
        return launch_cem_finalize(c, partials, G, U, action_out, stats, s);
    case RULE_MODES: {
        MPPIB_REQUIRE(c->dist != nullptr, "mppib_finalize: n_modes > 1 needs its mode state registered with mppib_set_distribution");
        const int smem = (int)sizeof(float) * modes_fin_floats(NR, c->params.n_modes, G);
        MPPIB_REQUIRE(smem <= 227 * 1024, "mppib_finalize: n_modes = %d with T*nu = %d and G = %d needs %d bytes of shared memory", c->params.n_modes, NR, G, smem);
        if (int rc = ensure_smem<mppib_finalize_kernel<RULE_MODES>>(c->device, smem)) return rc;
        return launch_finalize_t<RULE_MODES>(c, partials, G, U, action_out, stats, smem, c->dist, nullptr, nullptr, nullptr, s);
    }
    case RULE_SMOOTH:
        MPPIB_REQUIRE(c->smooth != nullptr, "mppib_finalize: mode smooth needs its state registered with mppib_set_smooth_state");
        return launch_finalize_t<RULE_SMOOTH>(c, partials, G, U, action_out, stats, un, nullptr, nullptr, c->smooth, nullptr, s);
    case RULE_HORIZON: {
        MPPIB_REQUIRE(NR <= MPPIB_HZ_MAX_N && c->hz_sig != nullptr && c->hz_n == NR, "mppib_finalize: cov_horizon buffers are not sized for n = %d", NR);
        const int smem = hz_fin_smem(NR, G);
        MPPIB_REQUIRE(smem <= 227 * 1024, "mppib_finalize: cov_horizon with n = %d and G = %d needs %d bytes of shared memory", NR, G, smem);
        if (int rc = ensure_smem<mppib_finalize_kernel<RULE_HORIZON>>(c->device, smem)) return rc;
        return launch_finalize_t<RULE_HORIZON>(c, partials, G, U, action_out, stats, smem, c->dist, c->hz_sig, nullptr, nullptr, s);
    }
    case RULE_FULL:
        return launch_finalize_t<RULE_FULL>(c, partials, G, U, action_out, stats, un + full_fin_floats(c->params.T, c->model.nu) * sizeof(float), c->dist,
                                            nullptr, nullptr, c->anneal, s);
    case RULE_DIST:
        return launch_finalize_t<RULE_DIST>(c, partials, G, U, action_out, stats, un + (adaptive_cov(c) ? NR : 0) * sizeof(float), c->dist, nullptr,
                                            nullptr, c->anneal, s);
    case RULE_FEASIBLE:
        return launch_finalize_t<RULE_FEASIBLE>(c, partials, G, U, action_out, stats, un, nullptr, nullptr, nullptr, nullptr, s);
    default:   // RULE_PLAIN
        return launch_finalize_t<RULE_PLAIN>(c, partials, G, U, action_out, stats, un, nullptr, nullptr, nullptr, c->anneal, s);
    }
}

int launch_shift(MppibContext* c, float* U, uint32_t* plan_ctr, cudaStream_t s) {
    const int NR = ctrl_rows(c->params) * c->model.nu;
    float* hz_g = nullptr;                                                    // lambda Sigma_H^-1 U for K3's control cost
    switch (update_rule(c)) {
    case RULE_CEM:
        return launch_cem_shift(c, U, plan_ctr, s);
    case RULE_MODES:
        mppib_shift_modes_kernel<<<1, 256, c->params.n_modes * NR * sizeof(float), s>>>(c->params, c->model.nu, U, plan_ctr);
        MPPIB_CHECK_CUDA(cudaGetLastError());
        return 0;
    case RULE_HORIZON:
        if (c->params.mode == MPPIB_MODE_SIMPLE) hz_g = c->hz_g;
        break;
    default:
        break;
    }
    mppib_shift_kernel<<<1, 256, NR * sizeof(float), s>>>(c->params, c->model.nu, U, plan_ctr, c->dist, hz_g, c->anneal, live_spline(c));
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
