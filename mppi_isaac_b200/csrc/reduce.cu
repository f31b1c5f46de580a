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

#include "common.cuh"

namespace {

constexpr int NT = 256;         // threads per CTA
constexpr int MAX_GRID = 512;   // persistent CTAs (<= scratch rows)
constexpr int MAX_PAIRS = MPPIB_MAX_NU * (MPPIB_MAX_NU + 1) / 2;   // lower triangle of a full nu x nu covariance

// what a shard row carries after (beta, eta, W[T*nu]): nothing, M2[T*nu] (update_cov) or C[nu(nu+1)/2] (update_cov with cov_full)
enum RowKind { ROW_W = 0, ROW_M2 = 1, ROW_C = 2 };
__host__ __device__ __forceinline__ int row_floats(int T, int nu, int kind) {
    return 2 + T * nu + (kind == ROW_M2 ? T * nu : kind == ROW_C ? nu * (nu + 1) / 2 : 0);
}
// shared floats finalize_rows<true, true> needs after un[T*nu] and the G scales: m1[T*nu], d[T*nu], C[nu(nu+1)/2], Sigma, L, L^-1
__host__ __device__ __forceinline__ int full_fin_floats(int T, int nu) { return 2 * T * nu + nu * (nu + 1) / 2 + 3 * nu * nu; }

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

// combine G rows (beta_g, eta_g, W_g) of stride P, update U (+ Savitzky-Golay, clamp), first action, statistics; one CTA of 256
// threads, `un` = [T*nu + G] floats of shared memory (+ T*nu with update_cov).
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
template <bool ADAPT, bool FULL = false>
__device__ __forceinline__ void finalize_rows(const MppibParams& p, int nu, const float* __restrict__ partials, int G, int P, float* __restrict__ U,
                                              float* __restrict__ action_out, float* __restrict__ stats, float* __restrict__ action_mirror, float* un,
                                              float* __restrict__ dist) {
    const int T = p.T, NR = T * nu;
    float* sg = un + NR;
    const float lam = ADAPT ? dist[0] : p.lambda_;
    const float inv_lambda = 1.0f / lam;
    const bool cov = ADAPT && !FULL && p.update_cov;
    float* var = sg + G;                                                      // [NR] per-element variance (update_cov)
    const int npairs = nu * (nu + 1) / 2;
    float* m1s = sg + G;                                                      // FULL: [NR] m1, [NR] d, [npairs] C, [nu*nu] Sigma, L, L^-1
    float* dds = m1s + NR;
    float* cc = dds + NR;
    float* sn = cc + npairs;
    float* Lm = sn + nu * nu;
    float* Mi = Lm + nu * nu;
    float b = INFINITY;
    for (int gidx = 0; gidx < G; ++gidx) if (__ldcg(&partials[(size_t)gidx * P + 1]) > 0.f) b = fminf(b, __ldcg(&partials[(size_t)gidx * P]));
    for (int gidx = threadIdx.x; gidx < G; gidx += blockDim.x) {
        const float eg = __ldcg(&partials[(size_t)gidx * P + 1]);
        sg[gidx] = eg > 0.f ? expf(-(__ldcg(&partials[(size_t)gidx * P]) - b) * inv_lambda) : 0.f;
    }
    __syncthreads();
    float e = 0.f;
    for (int gidx = 0; gidx < G; ++gidx) e += sg[gidx] * __ldcg(&partials[(size_t)gidx * P + 1]);
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
        if (FULL && e > 0.f) {
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
            const int t = r / nu, j = r % nu;
            float s = 0.f;
            if (t < 4) {
#pragma unroll
                for (int i = 0; i < 9; ++i) s += c_sg_edge[t][i] * un[i * nu + j];
                s *= (1.0f / 1155.0f);
            } else if (t >= T - 4) {
                const int ee = T - 1 - t;
#pragma unroll
                for (int i = 0; i < 9; ++i) s += c_sg_edge[ee][i] * un[(T - 1 - i) * nu + j];
                s *= (1.0f / 1155.0f);
            } else {
#pragma unroll
                for (int i = 0; i < 9; ++i) s += c_sg_mid[i] * un[(t - 4 + i) * nu + j];
                s *= (1.0f / 231.0f);
            }
            out = fminf(fmaxf(s, p.u_min[j]), p.u_max[j]);   // smoothing may overshoot the bounds at the edges
        }
        U[r] = out;
        if (r < nu) { action_out[r] = out; if (action_mirror) action_mirror[r] = out; }
    }
    if (threadIdx.x == 0 && stats) { stats[0] = b; stats[1] = e; }
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

// The last CTA of a K3 launch: fold the per-CTA partials (128-bit L2 loads, 8 in flight per thread), write the shard row, push it into
// every rank's peer window (multi-GPU) and, for single-GPU plans, do K4's work in place.  `tiles` = the idle ring, WsLayout::fold_floats
// at least, `misc` = 8 floats.
template <bool ADAPT, bool FULL = false>
__device__ __forceinline__ void fold_and_finish(const MppibParams& p, int nu, int P, float* __restrict__ scratch, unsigned int* __restrict__ ticket,
                                                float* __restrict__ partial, const PeerArgs& peers, float* __restrict__ fin_U, float* __restrict__ fin_action,
                                                float* __restrict__ fin_stats, float* __restrict__ fin_mirror, float* tiles, float* misc, float inv_lambda,
                                                float* __restrict__ dist) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = (int)gridDim.x;
    float* sc = tiles;                   // [MAX_GRID] scale of every CTA partial (the ring is idle now)
    float* fold = tiles + MAX_GRID;      // [4][PP]
    {
        float b = (tid < G) ? __ldcg(scratch + (size_t)tid * ((((P + 3) >> 2) << 2))) : INFINITY;
        const float b2 = (tid + NT < G) ? __ldcg(scratch + (size_t)(tid + NT) * ((((P + 3) >> 2) << 2))) : INFINITY;   // CTAs 256..511
        float bm = warp_min(fminf(b, b2));
        if (lane == 0) misc[warp] = bm;
        __syncthreads();
        float bb = INFINITY;
#pragma unroll
        for (int w8 = 0; w8 < 8; ++w8) bb = fminf(bb, misc[w8]);
        if (tid < G) sc[tid] = (b == INFINITY) ? 0.f : expf(-(b - bb) * inv_lambda);
        if (tid + NT < G) sc[tid + NT] = (b2 == INFINITY) ? 0.f : expf(-(b2 - bb) * inv_lambda);
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
        uint32_t seq = 0;
        if (peers.world > 1) seq = *reinterpret_cast<const volatile uint32_t*>(peers.win[peers.rank]) + 1u;
        const size_t row_off = MPPIB_WIN_DATA_OFF / sizeof(float) + ((size_t)(seq & 1u) * peers.world + peers.rank) * peers.pcap;
        for (int e = tid; e < P; e += NT) {
            const float v0 = fold[e] + fold[PP + e] + fold[2 * PP + e] + fold[3 * PP + e];
            const float v = e == 0 ? bb : v0;
            partial[e] = v;
            for (int g = 0; g < peers.world; ++g) reinterpret_cast<float*>(peers.win[g])[row_off + e] = v;
        }
        if (peers.world > 1) {
            __threadfence_system();
            __syncthreads();
            if (tid < peers.world) {
                uint32_t* flag = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(peers.win[tid]) + MPPIB_WIN_FLAGS_OFF) + (seq & 1u) * MPPIB_MAX_PEERS + peers.rank;
                asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(seq) : "memory");
            }
        }
        if (tid == 0) *ticket = 0u;
        if (fin_U != nullptr) {
            // single-GPU plans: this CTA is the last one alive and holds the shard row -> do K4's work here (U update, savgol,
            // first action) instead of launching another kernel.  Every CTA read U -- and, with a registered distribution, lambda and
            // cov -- in its prologue, before it took its ticket, so this CTA is the only reader left when it updates them.
            __threadfence();
            __syncthreads();
            finalize_rows<ADAPT, FULL>(p, nu, partial, 1, P, fin_U, fin_action, fin_stats, fin_mirror, tiles, dist);
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
// After the loop the seven warp partials are merged once through shared memory; the per-CTA partial, the ticket and the
// last-CTA fold / exchange / fused K4 follow (fold_and_finish).
constexpr int WS_W = 32;          // samples per tile
constexpr int WS_NCONS = 7;       // consumer warps (warp 0 is the producer)

// Shared-memory layout of the kernel with `nstage` ring stages, used by the host for the size and by the kernel for its pointers.
// Offsets in floats from the base, except `bar` (bytes).  The last CTA reuses the ring for the fold (fold_and_finish), so the ring
// region is at least fold_floats long; for every shape but T*nu + T <= 2 the ring stages alone are longer.  With the C row (ROW_C)
// the fused K4 also keeps its covariance scratch there (full_fin_floats), which the ring stages of every accepted shape exceed.
struct WsLayout {
    int g, gp, wk, cpart, misc;   // [NR4] lambda Sigma^-1 U | [T4] gamma^t | [8][32] weights | [NCONS][P4] warp partials | [8]
    int bar;                      // full[nstage], then empty[nstage] mbarriers
    int bytes;                    // + 128 bytes of headroom: the ring depth of every shape stays what it was tuned at
    __host__ __device__ WsLayout(int T, int nu, int nstage, int kind = ROW_W) {   // kind: what the shard row carries after W (RowKind)
        const int NR = T * nu, P4 = (row_floats(T, nu, kind) + 3) & ~3;
        const int ring = nstage * (NR + T) * WS_W, fold_floats = MAX_GRID + 4 * P4;
        g = ring > fold_floats ? ring : fold_floats;
        if (kind == ROW_C && g < NR + 1 + full_fin_floats(T, nu)) g = NR + 1 + full_fin_floats(T, nu);
        gp = g + ((NR + 3) & ~3);
        wk = gp + ((T + 3) & ~3);
        cpart = wk + 8 * WS_W;
        misc = cpart + WS_NCONS * P4;
        bar = ((misc + 8) * 4 + 15) & ~15;
        bytes = bar + 2 * 8 * nstage + 128;
    }
};

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ADAPT (a distribution is registered): lambda comes from dist[0]; with update_cov the SIMPLE-mode Sigma^-1 is diag(1 / dist[1 + j])
// and phase C keeps a second running sum per row, M2[r] = sum_k w_k (x[r][k] - c[r])^2 with c = U (MEAN) or 0 (SIMPLE), rescaled
// online like W; the shard row becomes (beta, eta, W[T*nu], M2[T*nu]).  The bytes read from HBM are the same.
// FULL (update_cov with cov_full): the SIMPLE-mode Sigma^-1 is the full one of dist, and instead of M2 every consumer lane keeps the
// lower triangle of sum_t w_k (x_tk - c_t)(x_tk - c_t)^T of its own sample k across tiles (lane = sample: column reads of the tile,
// conflict-free like phase A; c = U staged in g in MEAN mode), rescaled online like W and summed over the warp once after the loop;
// the shard row becomes (beta, eta, W[T*nu], C[nu(nu+1)/2]).
template <int RPL, bool ADAPT, bool FULL = false>   // rows of W per lane: T*nu <= 32 * RPL
__global__ void __launch_bounds__(NT, 1)
mppib_reduce_ws_kernel(const __grid_constant__ MppibParams p, const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_c,
                       int nu, int xbox_rows, int nstage, int ncons, const float* __restrict__ U, float* __restrict__ scratch, unsigned int* __restrict__ ticket,
                       float* __restrict__ partial, const __grid_constant__ PeerArgs peers, float* __restrict__ fin_U, float* __restrict__ fin_action,
                       float* __restrict__ fin_stats, float* __restrict__ fin_mirror, float* __restrict__ dist) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int K = p.K, T = p.T, NR = T * nu;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float lam = ADAPT ? dist[0] : p.lambda_;
    const float inv_lambda = 1.0f / lam;
    const bool simple = p.mode == MPPIB_MODE_SIMPLE;
    const bool m2 = ADAPT && !FULL && p.update_cov;
    const int npairs = FULL ? nu * (nu + 1) / 2 : 0;
    const int P = 2 + (m2 ? 2 : 1) * NR + npairs;

    const int tile_floats = (NR + T) * WS_W;                                  // a multiple of 32 floats: stages stay 128-B aligned
    const int NR4 = (NR + 3) & ~3, T4 = (T + 3) & ~3, P4 = (P + 3) & ~3;
    const WsLayout L(T, nu, nstage, FULL ? ROW_C : m2 ? ROW_M2 : ROW_W);
    float* tiles = reinterpret_cast<float*>(smem_raw);                        // [nstage][(NR+T)*32]
    float* g = tiles + L.g;                                                   // [NR4] lambda * Sigma^-1 U (SIMPLE), zero padded; FULL MEAN: U
    float* gp = tiles + L.gp;                                                 // [T4]  gamma^t, zero padded
    float* wk = tiles + L.wk;                                                 // [8][32] weights of the tile a warp is working on
    float* cpart = tiles + L.cpart;                                           // [NCONS][P4] warp partials (after the loop)
    float* misc = tiles + L.misc;                                             // [8]
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + L.bar);           // [nstage]
    uint64_t* empty = full + nstage;                                          // [nstage]

    const int ntiles = (K + WS_W - 1) / WS_W;
    const int my_tiles = (int)blockIdx.x < ntiles ? (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const uint32_t tile_bytes = (uint32_t)tile_floats * 4u;

    auto issue_tile = [&](int i) {   // elected producer lane: TMA tile i of this CTA into ring stage i % nstage
        const int s = i % nstage;
        const int k0 = ((int)blockIdx.x + i * (int)gridDim.x) * WS_W;
        float* dst = tiles + (size_t)s * tile_floats;
        mbar_expect_tx(&full[s], tile_bytes);
        for (int r0 = 0; r0 < NR; r0 += xbox_rows) tma_load_2d(dst + (size_t)r0 * WS_W, &tm_x, k0, r0, &full[s]);
        tma_load_2d(dst + (size_t)NR * WS_W, &tm_c, k0, 0, &full[s]);
    };
    if (tid == 0) {
        for (int s = 0; s < nstage; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        for (int i = 0; i < nstage && i < my_tiles; ++i) issue_tile(i);   // the first ring fill is in flight while the prologue below runs
    }
    for (int r = tid; r < NR4; r += NT) {
        float acc = 0.f;
        if (simple && r < NR) {
            const int t = r / nu, i = r % nu;
            if (FULL) {
                const float* sinv = dist + 1 + 2 * nu * nu;
                for (int j = 0; j < nu; ++j) acc += sinv[i * nu + j] * U[t * nu + j];
            } else if (m2) acc = (1.0f / dist[1 + i]) * U[r];
            else
                for (int j = 0; j < nu; ++j) acc += p.sigma_inv[i * nu + j] * U[t * nu + j];
            acc *= lam;
        }
        if (FULL && !simple && r < NR) acc = U[r];                            // phase A reads g in SIMPLE mode only
        g[r] = acc;
    }
    {
        // gamma^0 = 1 for every accepted gamma: log2f(0) * 0 would be NaN (validate refuses a negative or non-finite gamma)
        const float lg = log2f(p.gamma);
        for (int t = tid; t < T4; t += NT) gp[t] = t == 0 ? 1.f : t < T ? exp2f(lg * (float)t) : 0.f;
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
            const int k0 = ((int)blockIdx.x + i * (int)gridDim.x) * WS_W;
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
            const float sum = (a0 + a1) + (a2 + a3);
            // ---- B: tile minimum, weights, their sum
            const bool valid = (k0 + lane < K) && isfinite(sum);
            const float S = valid ? sum : INFINITY;
            const float b_c = warp_min(S);
            const float w = (S == INFINITY) ? 0.f : expf(-(S - b_c) * inv_lambda);
            const float e_c = warp_sum(w);
            if (b_c != INFINITY) {                                            // warp-uniform
                wme[lane] = w;
                __syncwarp();
                const float b_out = fminf(b_run, b_c);
                const float s_old = (b_run == INFINITY) ? 0.f : expf(-(b_run - b_out) * inv_lambda);
                const float s_new = expf(-(b_c - b_out) * inv_lambda);
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
    } else {
        // spare warp (fewer ring stages than warps): an empty partial
        float* mine = cpart + (size_t)(warp - 1) * P4;
        if (lane == 0) { mine[0] = INFINITY; mine[1] = 0.f; }
        for (int r = lane; r < P - 2; r += 32) mine[2 + r] = 0.f;
    }
    __syncthreads();
    // ---- merge the warp partials into the CTA partial (global scratch), then ticket -> the last CTA folds all of them
    {
        float* mine = scratch + (size_t)blockIdx.x * P4;
        float bb = INFINITY;
#pragma unroll
        for (int c = 0; c < WS_NCONS; ++c) bb = fminf(bb, cpart[(size_t)c * P4]);
        float sc[WS_NCONS];
#pragma unroll
        for (int c = 0; c < WS_NCONS; ++c) { const float bc = cpart[(size_t)c * P4]; sc[c] = (bc == INFINITY) ? 0.f : expf(-(bc - bb) * inv_lambda); }
        for (int e = tid; e < P; e += NT) {
            float v = 0.f;
#pragma unroll
            for (int c = 0; c < WS_NCONS; ++c) v += sc[c] * cpart[(size_t)c * P4 + e];
            mine[e] = e == 0 ? bb : v;
        }
    }
    __threadfence();
    __syncthreads();
    __shared__ unsigned int s_last_ws;
    if (tid == 0) s_last_ws = atomicAdd(ticket, 1u) == gridDim.x - 1 ? 1u : 0u;
    __syncthreads();
    if (!s_last_ws) return;
    __threadfence();
    fold_and_finish<ADAPT, FULL>(p, nu, P, scratch, ticket, partial, peers, fin_U, fin_action, fin_stats, fin_mirror, tiles, misc, inv_lambda, dist);
}

// K4: combine G shard partials, U update, optional Savitzky-Golay (window 9, order 2, 'interp' edges), action out; ADAPT: the
// distribution update of finalize_rows (FULL: of the full covariance).
template <bool ADAPT, bool FULL = false>
__global__ void __launch_bounds__(256)
mppib_finalize_kernel(const __grid_constant__ MppibParams p, int nu, const float* __restrict__ partials_in, int G,
                float* __restrict__ U, float* __restrict__ action_out, float* __restrict__ stats, const __grid_constant__ PeerArgs peers,
                float* __restrict__ action_mirror, float* __restrict__ dist) {
    extern __shared__ float un[];   // [T*nu] then [G] scales (then [T*nu] variances with update_cov, or full_fin_floats with FULL)
    const int T = p.T, NR = T * nu;
    int P = FULL ? row_floats(T, nu, ROW_C) : 2 + ((ADAPT && p.update_cov) ? 2 : 1) * NR;   // row stride of the partials
    const float* partials = partials_in;
    uint32_t seq = 0;
    if (partials_in == nullptr) {
        // rows come from this rank's peer window: wait until every rank's row of exchange `seq` has landed
        char* win = reinterpret_cast<char*>(peers.win[peers.rank]);
        seq = *reinterpret_cast<const volatile uint32_t*>(win) + 1u;
        if ((int)threadIdx.x < G) {
            const uint32_t* flag = reinterpret_cast<const uint32_t*>(win + MPPIB_WIN_FLAGS_OFF) + (seq & 1u) * MPPIB_MAX_PEERS + threadIdx.x;
            unsigned long long t0, now; uint32_t got;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
            while (true) {
                asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(got) : "l"(flag) : "memory");
                if (got == seq) break;
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
                if (now - t0 > peers.timeout_ns) {
                    printf("mppib_finalize: rank %d waited %.1f s for rank %d (exchange %u, flag %u): peer lost\n", peers.rank, (double)peers.timeout_ns * 1e-9, (int)threadIdx.x, seq, got);
                    __trap();
                }
                __nanosleep(64);
            }
        }
        __syncthreads();
        partials = reinterpret_cast<const float*>(win + MPPIB_WIN_DATA_OFF) + (size_t)(seq & 1u) * G * peers.pcap;
        P = peers.pcap;
    }
    finalize_rows<ADAPT, FULL>(p, nu, partials, G, P, U, action_out, stats, action_mirror, un, dist);
    if (threadIdx.x == 0 && partials_in == nullptr) *reinterpret_cast<volatile uint32_t*>(peers.win[peers.rank]) = seq;   // exchange `seq` consumed
}

__global__ void mppib_shift_kernel(const __grid_constant__ MppibParams p, int nu, float* __restrict__ U, uint32_t* __restrict__ plan_ctr) {
    extern __shared__ float tmp[];
    const int NR = p.T * nu;
    for (int r = threadIdx.x; r < NR; r += blockDim.x) tmp[r] = r + nu < NR ? U[r + nu] : p.u_init[r % nu];
    __syncthreads();
    for (int r = threadIdx.x; r < NR; r += blockDim.x) U[r] = tmp[r];
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

// K3 writes into the windows only when every peer is mapped (otherwise: single-GPU behaviour, world = 0)
static PeerArgs reduce_peers(const MppibContext* c) {
    PeerArgs a = peer_args(c);
    for (int g = 0; g < a.world; ++g) if (!a.win[g]) { a.world = 0; break; }
    if (a.world < 2) a.world = 0;
    return a;
}

static int reduce_ws_stages(int T, int nu, int kind) {
    int ns = 8;
    while (ns > 1 && WsLayout(T, nu, ns, kind).bytes > 224 * 1024) --ns;
    return ns;
}

template <int RPL, bool ADAPT, bool FULL = false>
int launch_reduce_ws_t(MppibContext* c, const float* cost, const float* x, const float* U, float* partial, float* fin_U, float* fin_action,
                       float* fin_stats, cudaStream_t s) {
    const int T = c->params.T, nu = c->model.nu, NR = T * nu, K = c->params.K;
    // consumers = min(7, stages that fit); the ring depth is rounded down to a multiple of the consumer count so that a stage always
    // belongs to the same consumer (see the kernel)
    const int kind = FULL ? ROW_C : (ADAPT && c->params.update_cov) ? ROW_M2 : ROW_W;
    const int nstage_max = reduce_ws_stages(T, nu, kind);
    const int ncons = nstage_max < WS_NCONS ? nstage_max : WS_NCONS;
    const int nstage = ncons * (nstage_max / ncons);
    const size_t smem = WsLayout(T, nu, nstage, kind).bytes;
    static size_t smem_attr[64] = {0};
    size_t& attr = smem_attr[c->device & 63];
    if (smem > attr) {
        MPPIB_CHECK_CUDA(cudaFuncSetAttribute(mppib_reduce_ws_kernel<RPL, ADAPT, FULL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    int xbox_rows = NR < 256 ? NR : 256;
    while (NR % xbox_rows != 0) --xbox_rows;
    // tensor maps are rebuilt only when a buffer, the shape or the device changes (the eager / stepwise path calls this per plan)
    struct MapCache { const void* x; const void* c; int K, T, nu, dev; CUtensorMap tm_x, tm_c; };
    static thread_local MapCache mc = {nullptr, nullptr, 0, 0, 0, -1, {}, {}};
    if (mc.x != x || mc.c != cost || mc.K != K || mc.T != T || mc.nu != nu || mc.dev != c->device) {
        if (int rc = make_map(&mc.tm_x, x, NR, K, xbox_rows, WS_W)) return rc;
        if (int rc = make_map(&mc.tm_c, cost, T, K, T, WS_W)) return rc;
        mc.x = x; mc.c = cost; mc.K = K; mc.T = T; mc.nu = nu; mc.dev = c->device;
    }
    const int ntiles = (K + WS_W - 1) / WS_W;
    int grid = ntiles < c->num_sms ? ntiles : c->num_sms;
    if (grid > MAX_GRID) grid = MAX_GRID;
    MPPIB_REQUIRE(grid <= c->reduce_max_ctas, "mppib_reduce: scratch too small");
    mppib_reduce_ws_kernel<RPL, ADAPT, FULL><<<grid, NT, smem, s>>>(c->params, mc.tm_x, mc.tm_c, nu, xbox_rows, nstage, ncons, U, c->reduce_scratch, c->reduce_ticket,
                                                             partial, reduce_peers(c), fin_U, fin_action, fin_stats, fin_U ? c->action_mirror : nullptr, c->dist);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

int launch_reduce(MppibContext* c, const float* cost, const float* x, const float* U, float* partial, float* fin_U, float* fin_action,
                  float* fin_stats, cudaStream_t s) {
    const int T = c->params.T, nu = c->model.nu;
    MPPIB_REQUIRE(c->params.K >= 4 && c->params.K % 4 == 0, "mppib_reduce: K=%d must be a positive multiple of 4 (16-byte rows for TMA / 128-bit loads)", c->params.K);
    MPPIB_REQUIRE(T * nu <= 32 * 16, "mppib_reduce: T*nu = %d exceeds %d", T * nu, 32 * 16);
    MPPIB_REQUIRE(T <= 256, "mppib_reduce: T = %d exceeds the 256-row TMA box", T);
    MPPIB_REQUIRE(reduce_ws_stages(T, nu, ROW_W) >= 2, "mppib_reduce: T = %d, nu = %d leaves room for fewer than two ring stages", T, nu);
    MPPIB_REQUIRE(!adaptive_cov(c) || adaptive_full(c) || reduce_ws_stages(T, nu, ROW_M2) >= 2,
                  "mppib_reduce: T = %d, nu = %d leaves room for fewer than two ring stages with the second-moment row of update_cov", T, nu);
    MPPIB_REQUIRE(!adaptive_full(c) || reduce_ws_stages(T, nu, ROW_C) >= 2,
                  "mppib_reduce: T = %d, nu = %d leaves room for fewer than two ring stages with the covariance row of cov_full", T, nu);
    const int NR = T * nu;
    if (adaptive_full(c)) {
        if (NR <= 32 * 4) return launch_reduce_ws_t<4, true, true>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, s);
        if (NR <= 32 * 8) return launch_reduce_ws_t<8, true, true>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, s);
        return launch_reduce_ws_t<16, true, true>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, s);
    }
    if (c->dist) {
        if (NR <= 32 * 4) return launch_reduce_ws_t<4, true>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, s);
        if (NR <= 32 * 8) return launch_reduce_ws_t<8, true>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, s);
        return launch_reduce_ws_t<16, true>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, s);
    }
    if (NR <= 32 * 4) return launch_reduce_ws_t<4, false>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, s);
    if (NR <= 32 * 8) return launch_reduce_ws_t<8, false>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, s);
    return launch_reduce_ws_t<16, false>(c, cost, x, U, partial, fin_U, fin_action, fin_stats, s);
}

int launch_finalize(MppibContext* c, const float* partials, int G, float* U, float* action_out, float* stats, cudaStream_t s) {
    const int NR = c->params.T * c->model.nu;
    if (adaptive_full(c)) {
        const size_t smem = (NR + G + full_fin_floats(c->params.T, c->model.nu)) * sizeof(float);
        mppib_finalize_kernel<true, true><<<1, 256, smem, s>>>(c->params, c->model.nu, partials, G, U, action_out, stats, peer_args(c), c->action_mirror, c->dist);
    } else if (c->dist) {
        const size_t smem = (NR + G + (adaptive_cov(c) ? NR : 0)) * sizeof(float);
        mppib_finalize_kernel<true><<<1, 256, smem, s>>>(c->params, c->model.nu, partials, G, U, action_out, stats, peer_args(c), c->action_mirror, c->dist);
    } else {
        mppib_finalize_kernel<false><<<1, 256, (NR + G) * sizeof(float), s>>>(c->params, c->model.nu, partials, G, U, action_out, stats, peer_args(c),
                                                                              c->action_mirror, nullptr);
    }
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_shift(MppibContext* c, float* U, uint32_t* plan_ctr, cudaStream_t s) {
    const int NR = c->params.T * c->model.nu;
    mppib_shift_kernel<<<1, 256, NR * sizeof(float), s>>>(c->params, c->model.nu, U, plan_ctr);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
