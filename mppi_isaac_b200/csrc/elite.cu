// elite.cu -- cross-entropy planning (MPPIB_MODE_CEM, iCEM): the elite kernel that takes K3's place, its K4 and the shift.
// See include/mppib.h ("Cross-entropy planning") for the shard row and the CEM state.
//
// Elite kernel: every CTA owns chunks of EL_NEW samples.  A thread computes S_k = sum_t gamma^t cost[t][k] of one sample in t order
// (coalesced column reads of cost), turns it into a 64-bit key (order-preserving float bits, then the global index) and the CTA sorts
// its running list of EL_KEEP keys together with the chunk in shared memory (bitonic, ascending); the first EL_KEEP keys stay.  The
// CTA's first E keys go to the handle's scratch; the last CTA (atomic ticket, as in K3) merges those lists the same way, gathers the
// winners' actions into the shard row and, for single-GPU plans, runs K4 in place.  Keys are unique, so every sort order is fixed
// and the shard's elite set is exact.  The kernel reads cost once (4*K*T bytes) and E*T*nu gathered actions.
#include "common.cuh"

namespace {

constexpr int EL_NT = 256;                        // threads per CTA
constexpr int EL_BUF = 1024;                      // keys sorted per pass
constexpr int EL_KEEP = MPPIB_CEM_MAX_ELITES;     // running list (>= E)
constexpr int EL_NEW = EL_BUF - EL_KEEP;          // new samples per pass
constexpr int EL_MAX_NR = 512;                    // T*nu (the limit of the colored K1)
constexpr int FIN_MAX_KEYS = 4096;                // K4 merges at most G*E <= 4096 candidates
constexpr unsigned long long KEY_NONE = ~0ull;

// the Savitzky-Golay coefficients of reduce.cu (window 9, order 2, 'interp' edges)
__constant__ float c_el_sg_mid[9] = {-21.f, 14.f, 39.f, 54.f, 59.f, 54.f, 39.f, 14.f, -21.f};
__constant__ float c_el_sg_edge[4][9] = {{763.f, 441.f, 189.f, 7.f, -105.f, -147.f, -119.f, -21.f, 147.f},
                                         {441.f, 322.f, 220.5f, 136.5f, 70.f, 21.f, -10.5f, -24.5f, -21.f},
                                         {189.f, 220.5f, 232.f, 223.5f, 195.f, 146.5f, 78.f, -10.5f, -119.f},
                                         {7.f, 136.5f, 223.5f, 268.f, 270.f, 229.5f, 146.5f, 21.f, -147.f}};

// order-preserving map of a finite float to uint32 (and back)
__device__ __forceinline__ uint32_t ord_bits(float s) { const uint32_t u = __float_as_uint(s); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ float ord_float(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o); }

// ascending bitonic sort of n (a power of two) keys in shared memory by the whole CTA; ends with a __syncthreads
__device__ void bitonic_sort(unsigned long long* k, int n) {
    for (int size = 2; size <= n; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool asc = (lo & size) == 0;
                const unsigned long long a = k[lo], b = k[hi];
                if ((a > b) == asc) { k[lo] = b; k[hi] = a; }
            }
        }
    }
    __syncthreads();
}

// K4 of MODE_CEM, one CTA: rows[g][P] are G shard rows in the order of their sample ranges.  Candidate (g, e) gets the key
// (S, g, e): within a row the entries are already in (S, global index) order and shard g's samples precede shard g + 1's, so the
// order is that of (S, global index) and the E smallest are the global elites, whatever G is.  `keys` holds >= G*E rounded up to a
// power of two, `un` T*nu floats.
__device__ void cem_update(const MppibParams& p, int nu, const float* __restrict__ rows, int G, int P, float* __restrict__ U,
                           float* __restrict__ action_out, float* __restrict__ stats, float* __restrict__ mirror, float* __restrict__ state,
                           unsigned long long* keys, float* un) {
    const int T = p.T, NR = T * nu, E = p.n_elites, n = G * E, tid = threadIdx.x;
    int npow = 2;
    while (npow < n) npow <<= 1;
    for (int i = tid; i < npow; i += blockDim.x) {
        unsigned long long key = KEY_NONE;
        if (i < n) {
            const int g = i / E, e = i % E;
            const float S = __ldcg(rows + (size_t)g * P + 2 * e);
            const uint32_t idx = __float_as_uint(__ldcg(rows + (size_t)g * P + 2 * e + 1));
            if (idx != 0xFFFFFFFFu && isfinite(S)) key = ((unsigned long long)ord_bits(S) << 32) | ((unsigned long long)g << 8) | (unsigned)e;
        }
        keys[i] = key;
    }
    bitonic_sort(keys, npow);
    const bool ok = keys[E - 1] != KEY_NONE;                                  // E finite elites over all shards
    const float alpha = p.elite_alpha;
    float* sig = state + 2 + E;
    float* elites = sig + NR;
    for (int r = tid; r < NR; r += blockDim.x) {
        if (!ok) { un[r] = U[r]; continue; }
        float acc = 0.f;
        for (int e = 0; e < E; ++e) {
            const unsigned src = (unsigned)(keys[e] & 0xFFFFFFFFull);
            acc += __ldcg(rows + (size_t)(src >> 8) * P + 2 * E + (size_t)(src & 0xFFu) * NR + r);
        }
        const float m = acc / (float)E;
        float v = 0.f;
        for (int e = 0; e < E; ++e) {
            const unsigned src = (unsigned)(keys[e] & 0xFFFFFFFFull);
            const float a = __ldcg(rows + (size_t)(src >> 8) * P + 2 * E + (size_t)(src & 0xFFu) * NR + r);
            const float d = a - m;
            v += d * d;
            elites[(size_t)e * NR + r] = a;
        }
        const float s = sqrtf(v / (float)E);
        un[r] = (1.0f - alpha) * m + alpha * U[r];
        sig[r] = (1.0f - alpha) * s + alpha * sig[r];
    }
    if (ok) {
        for (int e = tid; e < E; e += blockDim.x) state[2 + e] = ord_float((uint32_t)(keys[e] >> 32));
        if (tid == 0) { state[0] = 0.f; state[1] = 1.f; }                        // the next K1 carries these elites unshifted
    }
    __syncthreads();
    for (int r = tid; r < NR; r += blockDim.x) {                              // the tail of every mode: savgol, clamp, first action
        float out = un[r];
        if (p.filter_u) {
            const int t = r / nu, j = r % nu;
            float s = 0.f;
            if (t < 4) {
#pragma unroll
                for (int i = 0; i < 9; ++i) s += c_el_sg_edge[t][i] * un[i * nu + j];
                s *= (1.0f / 1155.0f);
            } else if (t >= T - 4) {
                const int ee = T - 1 - t;
#pragma unroll
                for (int i = 0; i < 9; ++i) s += c_el_sg_edge[ee][i] * un[(T - 1 - i) * nu + j];
                s *= (1.0f / 1155.0f);
            } else {
#pragma unroll
                for (int i = 0; i < 9; ++i) s += c_el_sg_mid[i] * un[(t - 4 + i) * nu + j];
                s *= (1.0f / 231.0f);
            }
            out = fminf(fmaxf(s, p.u_min[j]), p.u_max[j]);
        }
        U[r] = out;
        if (r < nu) { action_out[r] = out; if (mirror) mirror[r] = out; }
    }
    if (tid == 0 && stats) {
        stats[0] = keys[0] == KEY_NONE ? INFINITY : ord_float((uint32_t)(keys[0] >> 32));
        stats[1] = ok ? ord_float((uint32_t)(keys[E - 1] >> 32)) : INFINITY;
    }
}

__global__ void __launch_bounds__(EL_NT)
mppib_elite_kernel(const __grid_constant__ MppibParams p, int nu, const float* __restrict__ cost, const float* __restrict__ x, float* __restrict__ partial,
                   float* __restrict__ scratch, unsigned int* __restrict__ ticket, const __grid_constant__ PeerArgs peers, float* __restrict__ fin_U,
                   float* __restrict__ fin_action, float* __restrict__ fin_stats, float* __restrict__ fin_mirror, float* __restrict__ state) {
    __shared__ unsigned long long keys[EL_BUF];
    __shared__ float gp[256];
    __shared__ float un[EL_MAX_NR];
    const int K = p.K, T = p.T, NR = T * nu, E = p.n_elites, tid = threadIdx.x;
    const int P = shard_row_floats(RULE_CEM, T, nu, false, 0, E);
    {
        const float lg = log2f(p.gamma);                                      // gamma^t as K3 computes it
        for (int t = tid; t < T; t += EL_NT) gp[t] = t == 0 ? 1.f : exp2f(lg * (float)t);
    }
    for (int i = tid; i < EL_KEEP; i += EL_NT) keys[i] = KEY_NONE;
    __syncthreads();
    for (int base = blockIdx.x * EL_NEW; base < K; base += gridDim.x * EL_NEW) {
        for (int i = tid; i < EL_NEW; i += EL_NT) {
            const int k = base + i;
            unsigned long long key = KEY_NONE;
            if (k < K) {
                float S = 0.f;
                for (int t = 0; t < T; ++t) S = fmaf(gp[t], __ldcs(cost + (size_t)t * K + k), S);
                S += 0.0f;                                                    // -0 -> +0: one zero, one key order
                if (isfinite(S)) key = ((unsigned long long)ord_bits(S) << 32) | (p.k_offset + (uint32_t)k);
            }
            keys[EL_KEEP + i] = key;
        }
        bitonic_sort(keys, EL_BUF);
    }
    unsigned long long* mine = reinterpret_cast<unsigned long long*>(scratch + (size_t)blockIdx.x * P);   // P is a multiple of 4
    for (int e = tid; e < E; e += EL_NT) mine[e] = keys[e];
    if (!last_cta(ticket, gridDim.x)) return;
    // the last CTA: merge the per-CTA lists, as many as fit next to the running list per pass
    const int G = (int)gridDim.x, per = EL_NEW / E;
    for (int i = tid; i < EL_KEEP; i += EL_NT) keys[i] = KEY_NONE;
    for (int c0 = 0; c0 < G; c0 += per) {
        __syncthreads();
        for (int i = tid; i < EL_NEW; i += EL_NT) {
            const int c = c0 + i / E, e = i % E;
            keys[EL_KEEP + i] = (i < per * E && c < G) ? __ldcg(reinterpret_cast<const unsigned long long*>(scratch + (size_t)c * P) + e) : KEY_NONE;
        }
        bitonic_sort(keys, EL_BUF);
    }
    if (tid == 0) *ticket = 0u;
    // the shard row: (S, index bits)[E], actions[E][T*nu] gathered from x[T*nu][K]; missing entries (+inf, 0xFFFFFFFF, 0)
    const PeerRow row = peer_row(peers);
    for (int q = tid; q < P; q += EL_NT) {
        float v = 0.f;
        if (q < 2 * E) {
            const unsigned long long key = keys[q >> 1];
            if (q & 1) v = __uint_as_float(key == KEY_NONE ? 0xFFFFFFFFu : (uint32_t)key);
            else v = key == KEY_NONE ? INFINITY : ord_float((uint32_t)(key >> 32));
        } else if (q < 2 * E + E * NR) {
            const int e = (q - 2 * E) / NR, r = (q - 2 * E) % NR;
            const unsigned long long key = keys[e];
            if (key != KEY_NONE) v = __ldg(x + (size_t)r * K + ((uint32_t)key - p.k_offset));
        }
        partial[q] = v;
        peer_store(peers, row, q, v);
    }
    if (peers.world > 1) peer_release(peers, row);
    if (fin_U != nullptr) {
        // single-GPU plans: K4 on the row just written (the same code as mppib_finalize with G = 1, so the same bits); K1 read U and
        // the CEM state before this launch, so nothing else reads them now
        __threadfence();
        __syncthreads();
        cem_update(p, nu, partial, 1, P, fin_U, fin_action, fin_stats, fin_mirror, state, keys, un);
    }
}

__global__ void __launch_bounds__(256)
mppib_cem_finalize_kernel(const __grid_constant__ MppibParams p, int nu, const float* __restrict__ partials_in, int G, float* __restrict__ U,
                          float* __restrict__ action_out, float* __restrict__ stats, const __grid_constant__ PeerArgs peers,
                          float* __restrict__ mirror, float* __restrict__ state) {
    __shared__ unsigned long long keys[FIN_MAX_KEYS];
    __shared__ float un[EL_MAX_NR];
    const float* partials = partials_in;
    int P = shard_row_floats(RULE_CEM, p, nu);
    uint32_t seq = 0;
    if (partials_in == nullptr) {                                             // rows come from this rank's peer window
        const PeerRows w = peer_acquire(peers, G);
        partials = w.rows;
        P = w.stride;
        seq = w.seq;
    }
    cem_update(p, nu, partials, G, P, U, action_out, stats, mirror, state, keys, un);
    if (threadIdx.x == 0 && partials_in == nullptr) peer_consume(peers, seq);
}

// U[t] <- U[t+1], U[T-1] <- u_init; sigma[t][j] <- sigma0_j (the diagonal of sigma_chol); carry offset <- 1; *plan_ctr += 1
__global__ void mppib_cem_shift_kernel(const __grid_constant__ MppibParams p, int nu, float* __restrict__ U, uint32_t* __restrict__ plan_ctr,
                                       float* __restrict__ state) {
    __shared__ float tmp[EL_MAX_NR];
    const int NR = p.T * nu;
    float* sig = state + 2 + p.n_elites;
    for (int r = threadIdx.x; r < NR; r += blockDim.x) tmp[r] = r + nu < NR ? U[r + nu] : p.u_init[r % nu];
    __syncthreads();
    for (int r = threadIdx.x; r < NR; r += blockDim.x) {
        U[r] = tmp[r];
        const int j = r % nu;
        sig[r] = p.sigma_chol[j * nu + j];
    }
    if (threadIdx.x == 0) {
        state[0] = 1.f;
        if (plan_ctr) *plan_ctr += 1u;
    }
}

int cem_checks(const MppibContext* c, const char* what) {
    const int NR = c->params.T * c->model.nu, E = c->params.n_elites;
    MPPIB_REQUIRE(c->dist != nullptr, "%s: mppi_mode cem needs its state registered with mppib_set_distribution", what);
    MPPIB_REQUIRE(NR <= EL_MAX_NR && c->params.T <= 256, "%s: mode cem needs T <= 256 and T*nu <= %d, got T = %d, T*nu = %d", what, EL_MAX_NR,
                  c->params.T, NR);
    MPPIB_REQUIRE(E >= 1 && E <= MPPIB_CEM_MAX_ELITES, "%s: n_elites = %d out of range [1, %d]", what, E, MPPIB_CEM_MAX_ELITES);
    return 0;
}

}  // namespace

int launch_elite(MppibContext* c, const float* cost, const float* x, float* partial, float* fin_U, float* fin_action, float* fin_stats,
                 cudaStream_t s) {
    if (int rc = cem_checks(c, "mppib_reduce")) return rc;
    const int K = c->params.K;
    int grid = (K + EL_NEW - 1) / EL_NEW;
    if (grid > c->num_sms) grid = c->num_sms;
    MPPIB_REQUIRE(grid <= c->reduce_max_ctas, "mppib_reduce: scratch too small");
    mppib_elite_kernel<<<grid, EL_NT, 0, s>>>(c->params, c->model.nu, cost, x, partial, c->reduce_scratch, c->reduce_ticket, reduce_peers(c), fin_U,
                                              fin_action, fin_stats, fin_U ? c->action_mirror : nullptr, c->dist);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_cem_finalize(MppibContext* c, const float* partials, int G, float* U, float* action_out, float* stats, cudaStream_t s) {
    if (int rc = cem_checks(c, "mppib_finalize")) return rc;
    MPPIB_REQUIRE(G <= 255 && G * c->params.n_elites <= FIN_MAX_KEYS, "mppib_finalize: mode cem merges at most %d candidates (G = %d, E = %d)",
                  FIN_MAX_KEYS, G, c->params.n_elites);
    mppib_cem_finalize_kernel<<<1, 256, 0, s>>>(c->params, c->model.nu, partials, G, U, action_out, stats, peer_args(c), c->action_mirror, c->dist);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_cem_shift(MppibContext* c, float* U, uint32_t* plan_ctr, cudaStream_t s) {
    if (int rc = cem_checks(c, "mppib_shift")) return rc;
    mppib_cem_shift_kernel<<<1, 256, 0, s>>>(c->params, c->model.nu, U, plan_ctr, c->dist);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
