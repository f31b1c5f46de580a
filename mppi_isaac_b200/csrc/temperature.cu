// temperature.cu -- the ESS-targeted temperature of `lambda_mode: ess` (include/mppib.h "ESS-targeted temperature", DESIGN.md section 2).
//
// Before K3 weights the samples of a plan, one pass over the shard computes, for every sample, the two numbers K3's S is made of,
//   C_k = sum_t gamma^t c[t][k]   and   q_k = sum_r (Sigma^-1 U)_r x[r][k]   (SIMPLE mode; q_k = 0 in MEAN mode),
// so that S_k(lambda) = C_k + lambda q_k, and for each of the 65 grid temperatures lambda_j of the registered state the shifted sums of
// the softmax weights at that temperature, a_jk = C_k / lambda_j + q_k:
//   m_j = min_k a_jk,  s1_j = sum_k exp(-(a_jk - m_j)),  s2_j = sum_k exp(-2 (a_jk - m_j))
// over the valid samples (k < K, C_k and q_k finite).  The Kish effective sample size at lambda_j is s1_j^2 / s2_j whatever the shift.
// A solve (one warp) combines the shard rows of every rank, picks the temperature whose ESS is the target share of the valid samples and
// writes it to dist[0], where K3 and K4 read it.  K1 .. K4 are not changed: with the temperature in dist[0] they run the registered
// distribution's path (RULE_DIST) with both adaptive flags off.
//
// Data flow of the pass (HBM-bound like K3, 4*T*K bytes in MEAN mode, 4*K*T*(nu + 1) in SIMPLE mode):
//   * persistent CTAs of 256 threads (up to two per SM) walk tiles of 64 samples; thread (row group g = warp / 2, sample s) sums the rows
//     r = g, g + 4, ... of sample s, so every row is read coalesced and each thread keeps many independent loads in flight; the four row
//     groups' partial sums of C and q are added in group order
//   * the tile's (C, q) are staged in shared memory; warp w folds the 32 samples of half w % 2 into the running (m, s1, s2) of the grid
//     points j = 17 (w / 2) + lane, lane < 17, that its lanes own -- no warp reduction per grid point
//   * the two warps of a grid point merge into the CTA row, the CTA rows go to the handle's K3 scratch and the last CTA (ticket) folds them
//     in CTA order into the shard row (n_valid as int32 bits, (m_j, s1_j, s2_j)[65]).
// Every fold of several states (warps, CTAs, ranks) is two-pass: m = the minimum of the m's, then s1 = sum_g s1_g e^-(m_g - m) and
// s2 = sum_g s2_g e^-2(m_g - m) in order, so the exponentials are independent of the running sums.
#include "common.cuh"

namespace {

constexpr int TNT = 256;                         // threads per CTA
constexpr int TWARPS = TNT / 32;
constexpr int TS = 64;                           // samples per tile
constexpr int RG = TNT / TS;                     // row groups
constexpr int JG = 17;                           // grid points per warp pair: 4 pairs x 17 >= 65
constexpr int NG = MPPIB_ESS_GRID;               // 65 grid temperatures
constexpr int RF = MPPIB_ESS_ROW_FLOATS;         // 1 + 3 * 65 = 196 floats per shard row (a multiple of 4)

// (m, s1, s2) <- the merge of a tile's shifted sums into a warp's running state; an empty state (m = +inf) adds nothing.  One factor is
// exp(0) = 1 exactly.
__device__ __forceinline__ void ess_merge(float& m, float& s1, float& s2, float mb, float s1b, float s2b) {
    if (mb == INFINITY) return;
    if (m == INFINITY) { m = mb; s1 = s1b; s2 = s2b; return; }
    const float mn = fminf(m, mb);
    const float ra = expf(-(m - mn)), rb = expf(-(mb - mn));
    s1 = s1 * ra + s1b * rb;
    s2 = s2 * (ra * ra) + s2b * (rb * rb);
    m = mn;
}

// (m, s1, s2) of n states at stride `stride` (m at [0], s1 at [1], s2 at [2]), folded in order by the two-pass rule above; empty states
// (m = +inf) add nothing.  GLOBAL: rows other CTAs or ranks wrote, read from L2; otherwise shared memory.
template <bool GLOBAL>
__device__ __forceinline__ void ess_fold(const float* st, int n, size_t stride, float& m, float& s1, float& s2) {
    auto ld = [&](size_t i) { return GLOBAL ? __ldcg(st + i) : st[i]; };
    m = INFINITY;
#pragma unroll 8
    for (int g = 0; g < n; ++g) m = fminf(m, ld((size_t)g * stride));   // unrolled: the loads of eight states are in flight together
    s1 = 0.f; s2 = 0.f;
    if (m == INFINITY) return;
#pragma unroll 8
    for (int g = 0; g < n; ++g) {
        const float mg = ld((size_t)g * stride);
        if (mg == INFINITY) continue;
        const float r = expf(-(mg - m));
        s1 = fmaf(ld((size_t)g * stride + 1), r, s1);
        s2 = fmaf(ld((size_t)g * stride + 2), r * r, s2);
    }
}

// The rule (one warp; the other threads return).  rows[g * stride] is rank g's shard row, combined in rank order.  Writes the curve, the
// valid count and the chosen temperature into the state (lambda_j[65], 1/lambda_j[65], n_valid bits, lambda, ESS[65]) and lambda into
// dist[0]; with no valid sample anywhere dist[0] keeps its value.
__device__ __noinline__ void ess_solve(const MppibParams& p, const float* __restrict__ rows, int G, int stride, float* __restrict__ dist,
                                       float* __restrict__ state) {
    __shared__ float curve[NG];
    const int lane = threadIdx.x;
    if (lane >= 32) return;
    int n = 0;
    for (int g = 0; g < G; ++g) n += __float_as_int(__ldcg(&rows[(size_t)g * stride]));
    const float tau = p.ess_target * (float)n;
    int first = NG;
    for (int j = lane; j < NG; j += 32) {
        float m, s1, s2;
        ess_fold<true>(rows + 1 + 3 * j, G, stride, m, s1, s2);
        const float e = n > 0 ? (s1 * s1) / s2 : 0.f;
        curve[j] = e;
        state[2 * NG + 2 + j] = e;
        if (n > 0 && e >= tau && j < first) first = j;
    }
    first = __reduce_min_sync(0xffffffffu, first);
    __syncwarp();
    if (lane == 0) {
        float lam;
        if (n == 0) lam = dist[0];
        else if (first == NG) lam = state[NG - 1];
        else if (first == 0) lam = state[0];
        else {
            const float lo = logf(curve[first - 1]), hi = logf(curve[first]);
            const float theta = (logf(tau) - lo) / (hi - lo);
            lam = state[first - 1] * exp2f(0.25f * theta);
        }
        dist[0] = lam;
        state[2 * NG] = __int_as_float(n);
        state[2 * NG + 1] = lam;
    }
}

// The pass.  solve: the last CTA also runs the rule -- over its own row (no peers) or, with peers open, over every rank's row once it has
// landed in this rank's window.  Without solve it writes the row only, for a host all-gather and mppib_temperature_solve.
__global__ void __launch_bounds__(TNT, 2) mppib_temperature_kernel(const __grid_constant__ MppibParams p, int nu, const float* __restrict__ cost,
                                                                const float* __restrict__ x, const float* __restrict__ U, float* dist, float* __restrict__ state, float* __restrict__ scratch,
                                                                unsigned int* __restrict__ ticket, float* __restrict__ row, int solve,
                                                                const __grid_constant__ PeerArgs peers) {
    __shared__ float h[512];                     // Sigma^-1 U (SIMPLE), T*nu <= 512
    __shared__ float gp[256];                    // gamma^t, T <= 256
    __shared__ float pC[RG][TS], pq[RG][TS];     // the row groups' partial sums
    __shared__ float sC[TS], sq[TS];             // the tile's C_k (+inf: invalid) and q_k
    __shared__ float wst[TWARPS][3 * JG];        // the warp states after the loop
    const int K = p.K, T = p.T, NR = T * nu;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rg = warp >> 1, half = warp & 1, s_own = half * 32 + lane;   // this thread's row group and sample of the tile
    const int j_own = rg * JG + lane;                                       // the grid point this lane folds (lane < JG, j_own < NG)
    const bool folds = lane < JG && j_own < NG;
    const bool simple = p.mode == MPPIB_MODE_SIMPLE;
    const bool diag = p.update_cov && !p.cov_full, full = p.update_cov && p.cov_full;
    for (int r = tid; r < NR && simple; r += TNT) {                 // the Sigma^-1 of K3: diag(1 / cov), the full one, or the fixed one
        const int t = r / nu, i = r % nu;
        float acc = 0.f;
        if (full) {
            const float* sinv = dist + 1 + 2 * nu * nu;
            for (int j = 0; j < nu; ++j) acc += sinv[i * nu + j] * U[t * nu + j];
        } else if (diag) {
            acc = (1.0f / dist[1 + i]) * U[r];
        } else {
            for (int j = 0; j < nu; ++j) acc += p.sigma_inv[i * nu + j] * U[t * nu + j];
        }
        h[r] = acc;
    }
    {
        const float lg = log2f(p.gamma);                            // gamma^0 = 1 as in K3
        for (int t = tid; t < T; t += TNT) gp[t] = t == 0 ? 1.f : exp2f(lg * (float)t);
    }
    const float inv = folds ? state[NG + j_own] : 1.f;
    float m = INFINITY, s1 = 0.f, s2 = 0.f;
    int n_valid = 0;
    __syncthreads();
    const int ntiles = (K + TS - 1) / TS;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int k = tile * TS + s_own;
        float C = 0.f, q = 0.f;
        if (k < K) {
#pragma unroll 16
            for (int t = rg; t < T; t += RG) C = fmaf(gp[t], __ldg(&cost[(size_t)t * K + k]), C);
            if (simple) {
#pragma unroll 16
                for (int r = rg; r < NR; r += RG) q = fmaf(h[r], __ldg(&x[(size_t)r * K + k]), q);
            }
        }
        pC[rg][s_own] = C;
        pq[rg][s_own] = q;
        __syncthreads();
        bool valid = false;
        if (tid < TS) {
            C = ((pC[0][tid] + pC[1][tid]) + pC[2][tid]) + pC[3][tid];
            q = ((pq[0][tid] + pq[1][tid]) + pq[2][tid]) + pq[3][tid];
            valid = tile * TS + tid < K && isfinite(C) && isfinite(q);
            sC[tid] = valid ? C : INFINITY;
            sq[tid] = valid ? q : 0.f;
        }
        n_valid += __syncthreads_count(valid);
        if (folds) {
            const float* wc = sC + half * 32;
            const float* wq = sq + half * 32;
            float mt = INFINITY;
            for (int i = 0; i < 32; ++i) mt = fminf(mt, fmaf(wc[i], inv, wq[i]));
            if (mt != INFINITY) {                                   // some valid sample in this half of the tile
                float a1 = 0.f, a2 = 0.f;
                for (int i = 0; i < 32; ++i) {
                    const float e = expf(-(fmaf(wc[i], inv, wq[i]) - mt));   // 0 for an invalid sample (a = +inf)
                    a1 += e;
                    a2 = fmaf(e, e, a2);
                }
                ess_merge(m, s1, s2, mt, a1, a2);
            }
        }
        __syncthreads();                                            // the next tile overwrites the partials and sC / sq
    }
    if (folds) { wst[warp][3 * lane] = m; wst[warp][3 * lane + 1] = s1; wst[warp][3 * lane + 2] = s2; }
    __syncthreads();
    float* mine = scratch + (size_t)blockIdx.x * RF;
    if (tid < NG) {                                                 // grid point tid: the warps 2g, 2g + 1 of its group, in order
        const int g = tid / JG, l = tid % JG;
        float mm, a1, a2;
        ess_fold<false>(&wst[2 * g][3 * l], 2, 3 * JG, mm, a1, a2);
        mine[1 + 3 * tid] = mm; mine[2 + 3 * tid] = a1; mine[3 + 3 * tid] = a2;
    }
    if (tid == 0) mine[0] = __int_as_float(n_valid);
    if (!last_cta(ticket, gridDim.x)) return;
    // the last CTA: fold the CTA rows in CTA order into the shard row, publish it with peers open
    const int G = (int)gridDim.x;
    const PeerRow prow = peer_row(peers);
    if (tid < NG) {
        float mm, a1, a2;
        ess_fold<true>(scratch + 1 + 3 * tid, G, RF, mm, a1, a2);
        const float v[3] = {mm, a1, a2};
#pragma unroll
        for (int c = 0; c < 3; ++c) { row[1 + 3 * tid + c] = v[c]; peer_store(peers, prow, 1 + 3 * tid + c, v[c]); }
    }
    if (tid == 32) {
        int n = 0;
        for (int g = 0; g < G; ++g) n += __float_as_int(__ldcg(scratch + (size_t)g * RF));
        row[0] = __int_as_float(n);
        peer_store(peers, prow, 0, __int_as_float(n));
    }
    if (tid == 0) *ticket = 0u;
    if (peers.world > 1) peer_release(peers, prow);
    if (!solve) return;
    if (peers.world > 1) {
        // A second exchange per plan on the window and sequence counter K3 / K4 use: temperature s, then K3's row s + 1.  Two slots are
        // still enough: a rank publishes exchange s + 2 (the next plan's temperature row) only after its K4 acquired every rank's K3 row
        // s + 1, and every rank publishes that row only after its own temperature solve consumed exchange s, so slot s & 1 is free again.
        const PeerRows w = peer_acquire(peers, peers.world);
        ess_solve(p, w.rows, peers.world, w.stride, dist, state);
        __syncthreads();
        if (tid == 0) peer_consume(peers, w.seq);
    } else {
        __threadfence();
        __syncthreads();                                            // the row written above is visible to the solving warp
        ess_solve(p, row, 1, RF, dist, state);
    }
}

__global__ void __launch_bounds__(32) mppib_temperature_solve_kernel(const __grid_constant__ MppibParams p, const float* __restrict__ rows, int G,
                                                                     float* __restrict__ dist, float* __restrict__ state) {
    ess_solve(p, rows, G, RF, dist, state);
}

}  // namespace

int launch_temperature(MppibContext* c, const float* cost, const float* x, const float* U, float* row, bool solve, cudaStream_t s) {
    const int K = c->params.K, T = c->params.T, nu = c->model.nu;
    MPPIB_REQUIRE(T <= 256 && T * nu <= 512, "mppib_temperature: needs T <= 256 and T*nu <= 512, got T = %d, T*nu = %d", T, T * nu);
    const int ntiles = (K + TS - 1) / TS;
    int grid = ntiles < 2 * c->num_sms ? ntiles : 2 * c->num_sms;   // two CTAs per SM keep more loads in flight
    MPPIB_REQUIRE(grid <= c->reduce_max_ctas && partial_row_capacity(c->params, nu) >= RF, "mppib_temperature: scratch too small");
    PeerArgs peers = reduce_peers(c);
    if (!solve) peers.world = 0;                                   // the row goes to the caller's all-gather, not into the windows
    // the K3 scratch and ticket: this pass runs before K3 on the same stream, and its last CTA resets the ticket as K3's does
    mppib_temperature_kernel<<<grid, TNT, 0, s>>>(c->params, nu, cost, x, U, c->dist, c->temp, c->reduce_scratch, c->reduce_ticket, row,
                                                 solve ? 1 : 0, peers);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_temperature_solve(MppibContext* c, const float* rows, int G, cudaStream_t s) {
    mppib_temperature_solve_kernel<<<1, 32, 0, s>>>(c->params, rows, G, c->dist, c->temp);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
