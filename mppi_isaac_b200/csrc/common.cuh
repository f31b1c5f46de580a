// common.cuh -- shared declarations of the mppib CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/mppib.h"

// ------------------------------------------------------------------------------------------
// error plumbing: no exceptions cross the C ABI; mppib_last_error() returns the last message
// ------------------------------------------------------------------------------------------
void mppib_set_error(const char* fmt, ...);

#define MPPIB_CHECK_CUDA(expr)                                                              \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            mppib_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return -2;                                                                      \
        }                                                                                   \
    } while (0)

#define MPPIB_REQUIRE(cond, ...)                                                            \
    do {                                                                                    \
        if (!(cond)) {                                                                      \
            mppib_set_error(__VA_ARGS__);                                                   \
            return -1;                                                                      \
        }                                                                                   \
    } while (0)

struct MppibContext {
    int device;
    MppibModel model;
    MppibParams params;
    int obs_rows;            // R
    int state_rows;          // NS
    int num_sms;
    // K3 scratch: per-CTA partials + ticket counter (device memory owned by the handle)
    float* reduce_scratch;   // [max_ctas][partial_row_capacity(), padded to 4]
    unsigned int* reduce_ticket;
    int reduce_max_ctas;
    // peer window (multi-GPU exchange over NVLink peer memory), see include/mppib.h
    int peer_world, peer_rank, peer_pcap;      // pcap: floats per row (>= partial_row_capacity(), multiple of 4)
    void* peer_win[MPPIB_MAX_PEERS];           // window base of every rank (own entry = local allocation)
    unsigned long long peer_timeout_ns;
    float* action_mirror;                      // pinned host mirror of the action written by K4 (nullable)
    float* dist;                               // adaptive MPPI: device (lambda, cov[nu]) or, with cov_full, (lambda, Sigma, L, Sigma^-1)
                                               // read by K1 / K3, updated by K4 (nullable)
    float* smooth;                             // MODE_SMOOTH: device (a_prev[nu], A[T][nu]), read by K1, updated by K4 (nullable)
    float* anneal;                             // annealed MPPI: device (counter, s[N][T], r[N][T]), read by K1 / K3, counter set by K4 / shift (nullable)
    int anneal_n, anneal_T;                    // N iterations and the horizon T the schedule was registered for
    float* spline;                             // spline MPPI: device (rows[T + P][d + 3], U_exec[T][nu]), read by K1 / K4 / shift, U_exec written by K4 (nullable)
    int spline_T, spline_P, spline_d, spline_nu;   // the (T, P, d, nu) the table was registered for
    const float* viol;                         // constrained MPPI: device g[T][K] K3 reads (nullable)
    float* cstate;                             // constrained MPPI: device (n_feasible as int bits, min V), written by K4
    int viol_T, viol_K;                        // the (T, K) the buffer was registered for
    float* temp;                               // ESS-targeted temperature: device (lambda_j, 1/lambda_j, n_valid, lambda, ESS_j), written by the solve (nullable)
    // adaptive MPPI with cov_horizon (update_cov): device buffers owned by the handle, sized for (K, n = T*nu) by alloc_horizon
    float* hz_S;                               // [K] S_k of the last K3, read by the SYRK
    float* hz_g;                               // [n] lambda Sigma_H^-1 U of the last mppib_shift (K3 reads it in SIMPLE mode)
    float* hz_sig;                             // [n*n] the shifted Sigma_H of K4 while it is being factored
    float* hz_scr;                             // SYRK split-K partial tiles
    unsigned int* hz_ticket;                   // [HZ_MAX_TILES + 1] per-tile and final tickets of the SYRK (reset by their last CTA)
    int hz_K, hz_n, hz_scr_floats;
    // K2 mappings the handle may use (rollout_mapping() picks by scene, never by K); both default to true
    bool k2_team;                              // a team of lanes per rollout for trees / contact scenes (rollout_team.cu); MPPIB_K2_TEAM=0 turns it off
    bool k2_lanes;                             // one body per lane for serial chains (rollout_lanes.cu); MPPIB_K2_LANES=0 turns it off
};

// Every C-ABI entry that touches the device runs on the handle's device, whatever the calling thread's current device is (an
// RPC server thread, a caller that switched devices), and leaves the caller's current device as it found it.
struct DeviceGuard {
    int prev = -1;
    bool switched = false;
    cudaError_t err = cudaSuccess;
    explicit DeviceGuard(int device) {
        err = cudaGetDevice(&prev);
        if (err == cudaSuccess && prev != device) { err = cudaSetDevice(device); switched = err == cudaSuccess; }
    }
    ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};
#define MPPIB_ON_DEVICE(h)                                                                   \
    DeviceGuard _guard((h)->device);                                                        \
    MPPIB_CHECK_CUDA(_guard.err)

// Spline MPPI (control_knots = P > 0): the control vector U that K1 samples around, K3 weights and K4 updates is the knot vector
// theta[P][nu], while the cost rows stay T.  Its rows: P, or T with the feature off.  Every length of that vector comes from here.
__host__ __device__ __forceinline__ int ctrl_rows(const MppibParams& p) { return p.control_knots > 0 ? p.control_knots : p.T; }
// The spline table (include/mppib.h "Spline MPPI"): rows[T + P] of (first, count, weights[d + 1]), then U_exec[T][nu]
__host__ __device__ __forceinline__ int spline_row_floats(int d) { return d + 3; }
static inline long long spline_table_floats(int T, int P, int d, int nu) { return (long long)(T + P) * spline_row_floats(d) + (long long)T * nu; }
// sum_q w_q v[(first + q) * stride] over a table row's non-zero weights in index order: the first term a product, the rest fmaf
__device__ __forceinline__ float spline_apply(const float* __restrict__ row, const float* v, int stride) {
    const int first = (int)row[0], n = (int)row[1];
    float a = row[2] * v[first * stride];
    for (int q = 1; q < n; ++q) a = fmaf(row[2 + q], v[(first + q) * stride], a);
    return a;
}
// the launch-time refusals of spline MPPI (api.cu): the registered table must match (T, P, d, nu), and the plan must be plain MPPI
int check_spline(const MppibContext* c, const char* who);
// the table the kernels read: none while the parameter block has control_knots = 0, whatever was registered before
static inline float* live_spline(const MppibContext* c) { return c->params.control_knots > 0 ? c->spline : nullptr; }

// The update rule a plan runs: which K3 (or elite kernel), K4 and shift, and what their shard row carries.  Risk-aware MPPI is not a
// rule but a K3 flag (risk_mode) that combines with PLAIN, DIST and FULL.
enum Rule { RULE_PLAIN, RULE_DIST, RULE_FULL, RULE_HORIZON, RULE_SMOOTH, RULE_MODES, RULE_CEM, RULE_FEASIBLE };
// Floats of one shard row (T: the control rows, ctrl_rows() of the parameter block):
//   PLAIN, SMOOTH  (beta, eta, W[T*nu])
//   DIST           (beta, eta, W[T*nu]), + M2[T*nu] with update_cov
//   FULL           (beta, eta, W[T*nu], C[nu(nu+1)/2])
//   HORIZON        (beta, eta, W[n], C[n(n+1)/2]), n = T*nu
//   MODES          (beta, eta, W[T*nu]) of every mode
//   CEM            (S, index bits)[E] + actions[E][T*nu], padded to 4 floats, E = n_elites
//   FEASIBLE       (beta, eta, W[T*nu], n_feasible as int bits, min V)
// The kernels pass the parts they already hold (T, update_cov, ...); the host passes the parameter block.
__host__ __device__ inline int shard_row_floats(Rule r, int T, int nu, bool update_cov, int n_modes, int E) {
    const int NR = T * nu;
    switch (r) {
    case RULE_DIST: return 2 + NR + (update_cov ? NR : 0);
    case RULE_FULL: return 2 + NR + nu * (nu + 1) / 2;
    case RULE_HORIZON: return 2 + NR + NR * (NR + 1) / 2;
    case RULE_MODES: return n_modes * (2 + NR);
    case RULE_CEM: return (2 * E + E * T * nu + 3) & ~3;
    case RULE_FEASIBLE: return 4 + NR;
    default: return 2 + NR;
    }
}
__host__ __device__ inline int shard_row_floats(Rule r, const MppibParams& p, int nu) {
    return shard_row_floats(r, ctrl_rows(p), nu, p.update_cov, p.n_modes, p.n_elites);
}
static inline bool risk_mode(const MppibContext* c) { return c->params.n_worlds > 1; }
static inline bool modes_on(const MppibContext* c) { return c->params.n_modes > 1; }
static inline bool cem_mode(const MppibContext* c) { return c->params.mode == MPPIB_MODE_CEM; }
static inline bool smooth_mode(const MppibContext* c) { return c->params.mode == MPPIB_MODE_SMOOTH; }
static inline bool adaptive_cov(const MppibContext* c) { return c->dist != nullptr && c->params.update_cov; }
static inline bool adaptive_full(const MppibContext* c) { return adaptive_cov(c) && c->params.cov_full; }
static inline bool adaptive_horizon(const MppibContext* c) { return adaptive_cov(c) && c->params.cov_horizon; }
// the rule of the handle as it stands: the adaptive rules need a registered distribution
static inline Rule update_rule(const MppibContext* c) {
    if (cem_mode(c)) return RULE_CEM;
    if (modes_on(c)) return RULE_MODES;
    if (smooth_mode(c)) return RULE_SMOOTH;
    if (adaptive_horizon(c)) return RULE_HORIZON;
    if (adaptive_full(c)) return RULE_FULL;
    if (c->dist) return RULE_DIST;
    if (c->viol && c->params.constraint_mode) return RULE_FEASIBLE;
    return RULE_PLAIN;
}
// The draw K1 makes for the rule: the colour of the white draws (FIXED L0, DIAG / FULL / HORIZON the live adaptive ones, CEM the
// per-step sigma) or SMOOTH's integrated derivative.  update_lambda alone keeps the fixed Sigma.
enum Draw { DRAW_FIXED, DRAW_DIAG, DRAW_FULL, DRAW_HORIZON, DRAW_CEM, DRAW_SMOOTH };
static inline Draw draw_rule(const MppibContext* c) {
    switch (update_rule(c)) {
    case RULE_CEM: return DRAW_CEM;
    case RULE_SMOOTH: return DRAW_SMOOTH;
    case RULE_HORIZON: return DRAW_HORIZON;
    case RULE_FULL: return DRAW_FULL;
    case RULE_DIST: return c->params.update_cov ? DRAW_DIAG : DRAW_FIXED;
    default: return DRAW_FIXED;
    }
}
// the rule the flags select once a distribution is registered: buffers are sized by it, so that registering a distribution never
// needs a reallocation
static inline Rule configured_rule(const MppibParams& p) {
    if (p.mode == MPPIB_MODE_CEM) return RULE_CEM;
    if (p.n_modes > 1) return RULE_MODES;
    if (p.mode == MPPIB_MODE_SMOOTH) return RULE_SMOOTH;
    if (p.update_cov && p.cov_horizon) return RULE_HORIZON;
    if (p.update_cov && p.cov_full) return RULE_FULL;
    if (p.update_cov || p.update_lambda) return RULE_DIST;
    if (p.constraint_mode) return RULE_FEASIBLE;
    return RULE_PLAIN;
}
// ESS-targeted temperature: its shard row travels through the same scratch and peer window, so they hold the longer of the two rows
static inline int partial_row_capacity(const MppibParams& p, int nu) {
    const int P = shard_row_floats(configured_rule(p), p, nu);
    return p.lambda_ess && P < MPPIB_ESS_ROW_FLOATS ? MPPIB_ESS_ROW_FLOATS : P;
}
// Risk-aware MPPI (n_worlds = R > 1, a power of two): global rollout kg = c*R + r runs control sample c in world r.  K1 keys its draws
// and its null / prior rows by c, K2 keys the per-rollout randomisation by r.  R <= 1 (and a zero-initialised block) keeps kg for both.
__device__ __forceinline__ uint32_t sample_control(uint32_t kg, int R) { return R > 1 ? kg >> (__ffs(R) - 1) : kg; }
__device__ __forceinline__ uint32_t sample_world(uint32_t kg, int R) { return R > 1 ? kg & (uint32_t)(R - 1) : kg; }
// Counter-based Philox-4x32-10, its uniform in (0, 1) and the Box-Muller pair: K1's control noise and K2's per-rollout randomisation.
// UNROLL is the unroll of the ten rounds: K1 unrolls them all (10), K2 draws once per rollout and keeps them rolled (1).
template <int UNROLL>
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll UNROLL
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x, hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += W0; k1 += W1;
    }
    return c;
}
__device__ __forceinline__ float u01(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
    const float r = sqrtf(-2.0f * logf(u01(a)));
    float s, c;
    sincospif(2.0f * u01(b), &s, &c);
    z0 = r * c; z1 = r * s;
}
// Multi-modal MPPI (n_modes = M > 1): global sample kg is drawn around mode kg / Kc of U[M][T][nu], Kc = mode_samples.  M <= 1 (and a
// zero-initialised block) keeps mode 0 for every sample.
__device__ __forceinline__ int sample_mode(uint32_t kg, const MppibParams& p) { return p.n_modes > 1 ? (int)(kg / (uint32_t)p.mode_samples) : 0; }
// Annealed MPPI: the row of the registered schedule a (counter, s[N][T], r[N][T]) that iteration min(counter, N - 1) reads -- the noise
// scale s (recip = false) or r = 1 / s^2 (recip = true).  The counter is a float that K4 advances and the shift resets.
__device__ __forceinline__ const float* anneal_row(const float* __restrict__ a, int n, int T, bool recip) {
    const int i = min(max((int)a[0], 0), n - 1);
    return a + 1 + (size_t)((recip ? n : 0) + i) * T;
}
// the launch-time refusals of a registered schedule (api.cu)
int check_anneal(const MppibContext* c, const char* who);
// the first pair of the exclusion table (api.cu) a block breaks, with a registered schedule counted when anneal is set; who: "" or the
// entry point the message names
int check_exclusions(const MppibParams& p, bool anneal, const char* who);
// The merge of two or more partial states (n_feasible, b, eta, W) that every fold of every rule uses: tile into warp, warps into the
// CTA partial, CTA partials into the shard row, shard rows in K4.  The merged state has n_all = the sum of the counts and b_all =
// merge_min over the states; a state's eta and W enter it times merge_scale.  Constrained MPPI (include/mppib.h "Constrained MPPI") is
// the feasibility-first merge: a state with a feasible sample beats one without, which then weighs 0; states of one kind merge by the
// online-softmax rescale with their temperature (lambda for the feasible kind, lambda_c for the violation kind).  One accumulator
// suffices: once any state holds a feasible sample the violation kind can never win again, so its sums are dropped.  Every other rule
// is the case with every count 0 and lambda in both temperature slots: b_all = min b, scale = exp(-(b - b_all)/lambda).  An empty
// state weighs 0; each level tests for one itself (b = +inf in the kernel's folds, eta = 0 in K4) and does not call merge_scale on it.
// merge_min(nf, b, n_all): the b one state brings into the minimum (+inf when the other kind wins); with b_acc: folded into b_acc
__device__ __forceinline__ float merge_min(int nf, float b, int n_all) { return (nf > 0) == (n_all > 0) ? b : INFINITY; }
__device__ __forceinline__ float merge_min(int nf, float b, int n_all, float b_acc) { return (nf > 0) == (n_all > 0) ? fminf(b_acc, b) : b_acc; }
__device__ __forceinline__ float merge_scale(int nf, float b, int n_all, float b_all, float inv_lambda, float inv_lambda_c) {
    if ((nf > 0) != (n_all > 0)) return 0.f;
    return expf(-(b - b_all) * (n_all > 0 ? inv_lambda : inv_lambda_c));
}
// The election of the CTA that folds a grid's partials: every CTA calls it once its partial is written, and it returns true in the one
// CTA whose atomicAdd takes ticket value count - 1.  The fence before the ticket makes this CTA's partial visible to the others, the
// one after it orders the winner's reads of theirs.  Resetting the ticket is the caller's.  A CTA may call it twice with one flag (the
// SYRK): every thread has read the flag before the second call's first __syncthreads, and thread 0 writes it only after that barrier.
// (A template so that the compiler emits the flag after the calling kernel's own shared arrays: placed before an 8-byte aligned one,
// it would cost 4 bytes of padding.)
template <int = 0>
__device__ __forceinline__ bool last_cta(unsigned int* ticket, unsigned int count) {
    __shared__ unsigned int s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == count - 1u ? 1u : 0u;
    __syncthreads();
    if (!s_last) return false;
    __threadfence();
    return true;
}
// the per-step violation a margin g contributes: g where g > 0, 0 where g <= 0; NaN stays NaN, so the sample becomes invalid
__device__ __forceinline__ float feas_violation(float g) { return g <= 0.f ? 0.f : g; }
// the launch-time refusals of constrained MPPI (api.cu): the mode and the registration must agree, for the registered (T, K)
int check_constraint(const MppibContext* c, const char* who);
// the launch-time refusal of the ESS-targeted temperature (api.cu): lambda_ess needs a registered distribution and state
int check_temperature(const MppibContext* c, const char* who);
#define MPPIB_HZ_MAX_N 256                    // cov_horizon: largest n = T*nu (the packed n x n triangle K4 factors in shared memory)
#define HZ_TILE 64                             // SYRK output tile
#define HZ_MAX_TILES 10                        // lower-triangle tiles of a 256 x 256 C

// device view of the peer windows, passed by value to K3 / K4
struct PeerArgs {
    int world, rank, pcap;
    unsigned long long timeout_ns;
    void* win[MPPIB_MAX_PEERS];
};
// window layout (bytes): [0] uint32 seq | [128] uint32 flags[2][MPPIB_MAX_PEERS] | [256] float rows[2][world][pcap]
#define MPPIB_WIN_FLAGS_OFF 128
#define MPPIB_WIN_DATA_OFF 256
static inline size_t peer_window_bytes(int world, int pcap) { return MPPIB_WIN_DATA_OFF + sizeof(float) * 2 * (size_t)world * pcap; }
static inline PeerArgs peer_args(const MppibContext* c) {
    PeerArgs a; a.world = c->peer_world; a.rank = c->peer_rank; a.pcap = c->peer_pcap; a.timeout_ns = c->peer_timeout_ns;
    for (int g = 0; g < MPPIB_MAX_PEERS; ++g) a.win[g] = c->peer_win[g];
    return a;
}
// the windows K3 (or the elite kernel, or the SYRK) publishes its row into: only when every peer is mapped (otherwise single-GPU
// behaviour, world = 0)
static inline PeerArgs reduce_peers(const MppibContext* c) {
    PeerArgs a = peer_args(c);
    for (int g = 0; g < a.world; ++g) if (!a.win[g]) { a.world = 0; break; }
    if (a.world < 2) a.world = 0;
    return a;
}

// The exchange protocol.  Publish: a rank stores its row of exchange seq = (its own window's consumed counter) + 1 into slot
// (seq & 1, rank) of every window (remote stores over NVLink), then, after a system fence, release-stores seq into flag (seq & 1, rank)
// of every window.  Acquire: K4 waits until the G flags of exchange seq in its own window hold seq, reads the rows and stores seq into
// the counter (consume).  Two slots let the next exchange's rows land while K4 still reads this one's.
struct PeerRow { uint32_t seq; size_t off; };   // off: in floats from the window base
__device__ __forceinline__ PeerRow peer_row(const PeerArgs& peers) {
    uint32_t seq = 0;
    if (peers.world > 1) seq = *reinterpret_cast<const volatile uint32_t*>(peers.win[peers.rank]) + 1u;
    return {seq, MPPIB_WIN_DATA_OFF / sizeof(float) + ((size_t)(seq & 1u) * peers.world + peers.rank) * peers.pcap};
}
// element e of this rank's row into every window (none without peers)
__device__ __forceinline__ void peer_store(const PeerArgs& peers, const PeerRow& row, int e, float v) {
    for (int g = 0; g < peers.world; ++g) reinterpret_cast<float*>(peers.win[g])[row.off + e] = v;
}
// after every thread's peer_store: the row is complete, tell every rank (a CTA-wide call, with peers only: world > 1)
__device__ __forceinline__ void peer_release(const PeerArgs& peers, const PeerRow& row) {
    __threadfence_system();
    __syncthreads();
    const int tid = threadIdx.x;
    if (tid < peers.world) {
        uint32_t* flag = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(peers.win[tid]) + MPPIB_WIN_FLAGS_OFF) + (row.seq & 1u) * MPPIB_MAX_PEERS + peers.rank;
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(row.seq) : "memory");
    }
}
// wait until every rank's row of the next exchange has landed in this rank's window (a CTA-wide call); rows[g * stride] is rank g's
struct PeerRows { const float* rows; int stride; uint32_t seq; };
__device__ __forceinline__ PeerRows peer_acquire(const PeerArgs& peers, int G) {
    char* win = reinterpret_cast<char*>(peers.win[peers.rank]);
    const uint32_t seq = *reinterpret_cast<const volatile uint32_t*>(win) + 1u;
    if ((int)threadIdx.x < G) {
        const uint32_t* flag = reinterpret_cast<const uint32_t*>(win + MPPIB_WIN_FLAGS_OFF) + (seq & 1u) * MPPIB_MAX_PEERS + threadIdx.x;
        unsigned long long t0, now;
        uint32_t got;
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
    return {reinterpret_cast<const float*>(win + MPPIB_WIN_DATA_OFF) + (size_t)(seq & 1u) * G * peers.pcap, peers.pcap, seq};
}
// exchange `seq` is consumed: its slot may take the rows of exchange seq + 2 (one thread)
__device__ __forceinline__ void peer_consume(const PeerArgs& peers, uint32_t seq) {
    *reinterpret_cast<volatile uint32_t*>(peers.win[peers.rank]) = seq;
}

// Raise KERNEL's dynamic shared-memory limit to `bytes` on `device` where it is lower: the attribute belongs to the function on one
// device, so the high-water mark is kept per device.
template <auto KERNEL>
int ensure_smem(int device, size_t bytes) {
    static size_t attr[64] = {0};
    size_t& a = attr[device & 63];
    if (bytes > a) {
        MPPIB_CHECK_CUDA(cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        a = bytes;
    }
    return 0;
}

// The K1 entries of the C ABI.  k1_admit (sample.cu) holds which draw each entry samples and which it refuses: the null arguments
// (args = the entry's pointers are all non-null), the shard range, the annealing schedule, the mode routing, the n_worlds and n_modes
// shards and the size limits.  Returns 0 or the error of the first refusal; nothing is launched.
enum K1Entry { K1_SAMPLE, K1_COLORED, K1_SMOOTH, K1_NOISE_LIBRARY, K1_SAMPLE_LIBRARY, K1_SPLINE };
int k1_admit(const MppibContext* c, K1Entry e, bool args, uint32_t k_offset, uint32_t k_total, int n_knots = 1);

// kernel launchers (defined in the .cu files)
int launch_sample(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                  const float* U, const float* prior_row, float* actions, float* noise, cudaStream_t s);
int launch_sample_colored(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                          const float* U, const float* prior_row, const float* Lt, float* actions, float* noise, cudaStream_t s);
int launch_sample_smooth(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                         const float* U, float* actions, float* noise, cudaStream_t s);
int launch_noise_library(MppibContext* c, uint32_t k_offset, uint32_t k_total, const int32_t* halton_tab, const float* B, int n_knots,
                         float* Z, cudaStream_t s);
int launch_sample_library(MppibContext* c, uint32_t k_offset, uint32_t k_total, const float* U, const float* prior_row, const float* Z,
                          float* actions, float* noise, cudaStream_t s);
int launch_sample_spline(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                         const float* U, float* actions, float* xk, cudaStream_t s);
int launch_rollout(MppibContext* c, const float* state0, const float* root0, float* state, const float* actions, int t0, int nsteps,
                   float* obs, cudaStream_t s);
int launch_reduce(MppibContext* c, const float* cost, const float* x, const float* U, float* partial, float* fin_U, float* fin_action,
                  float* fin_stats, cudaStream_t s);
int launch_finalize(MppibContext* c, const float* partials, int G, float* U, float* action_out, float* stats, cudaStream_t s);
int launch_shift(MppibContext* c, float* U, uint32_t* plan_ctr, cudaStream_t s);
// MODE_CEM (elite.cu): the elite kernel (+ the fused K4 when fin_U != NULL), K4 and the shift
int launch_elite(MppibContext* c, const float* cost, const float* x, float* partial, float* fin_U, float* fin_action, float* fin_stats,
                 cudaStream_t s);
int launch_cem_finalize(MppibContext* c, const float* partials, int G, float* U, float* action_out, float* stats, cudaStream_t s);
int launch_cem_shift(MppibContext* c, float* U, uint32_t* plan_ctr, cudaStream_t s);
// lambda_mode ess (temperature.cu): the temperature pass (+ the solve when `solve`), and the solve over G explicit rows
int launch_temperature(MppibContext* c, const float* cost, const float* x, const float* U, float* row, bool solve, cudaStream_t s);
int launch_temperature_solve(MppibContext* c, const float* rows, int G, cudaStream_t s);
int alloc_horizon(MppibContext* c);           // (re)sizes the hz_* buffers for the handle's K and T*nu (frees them without cov_horizon)
// K3's ring depth for the shard row of `row` (reduce.cu): a launch needs two stages at least, and validate refuses constraint_mode with fewer
int reduce_ws_stages(const MppibParams& p, int nu, Rule row, bool smooth = false);
long long rollout_smem_bytes(const MppibModel& m);
// K2, lanes-per-rollout mapping for serial chains without contacts (rollout_lanes.cu)
bool rollout_lanes_eligible(const MppibModel& m);
// K2, team-of-lanes mapping for trees and scenes with contacts (rollout_team.cu)
bool rollout_team_eligible(const MppibModel& m);
// which kernel mppib_rollout launches for this handle: MPPIB_MAPPING_* (include/mppib.h)
int rollout_mapping(const MppibContext* c);
int launch_rollout_team(MppibContext* c, const float* state0, const float* root0, float* state, const float* actions, int t0, int nsteps,
                        float* obs, cudaStream_t s);
int launch_rollout_lanes(MppibContext* c, const float* state0, float* state, const float* actions, int t0, int nsteps, float* obs,
                         cudaStream_t s);
int launch_cost_pose(long long n, const float* a, long long a_si, long long a_sr, const float* b, long long b_si, long long b_sr, float w_pos,
                     float w_ori, float* cost, int accumulate, cudaStream_t s);

static inline int obs_item_width(const MppibModel& m, int kind) {
    return kind == MPPIB_OBS_DOF_STATE ? 2 * m.nb : (kind == MPPIB_OBS_CONTACT ? 3 : 13);
}
