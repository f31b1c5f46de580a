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
    float* reduce_scratch;   // [max_ctas][partial_row_floats(), padded to 4]
    unsigned int* reduce_ticket;
    int reduce_max_ctas;
    // peer window (multi-GPU exchange over NVLink peer memory), see include/mppib.h
    int peer_world, peer_rank, peer_pcap;      // pcap: floats per row (>= partial_row_floats(), multiple of 4)
    void* peer_win[MPPIB_MAX_PEERS];           // window base of every rank (own entry = local allocation)
    unsigned long long peer_timeout_ns;
    float* action_mirror;                      // pinned host mirror of the action written by K4 (nullable)
    float* dist;                               // adaptive MPPI: device (lambda, cov[nu]) or, with cov_full, (lambda, Sigma, L, Sigma^-1)
                                               // read by K1 / K3, updated by K4 (nullable)
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

// Floats of one shard row (beta, eta, W[T*nu] and, with update_cov, M2[T*nu], or with cov_full too C[nu(nu+1)/2]).  Buffers are
// sized by the flags alone, so that registering a distribution never needs a reallocation; the kernels append M2 / C only when a
// distribution is registered too.
static inline int partial_row_capacity(const MppibParams& p, int nu) {
    if (p.update_cov && p.cov_full) return 2 + p.T * nu + nu * (nu + 1) / 2;
    return 2 + p.T * nu * (p.update_cov ? 2 : 1);
}
static inline bool adaptive_cov(const MppibContext* c) { return c->dist != nullptr && c->params.update_cov; }
static inline bool adaptive_full(const MppibContext* c) { return adaptive_cov(c) && c->params.cov_full; }

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

// kernel launchers (defined in the .cu files)
int launch_sample(MppibContext* c, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                  const float* U, const float* prior_row, float* actions, float* noise, cudaStream_t s);
int launch_noise_library(MppibContext* c, uint32_t k_offset, uint32_t k_total, const int32_t* halton_tab, const float* B, int n_knots,
                         float* Z, cudaStream_t s);
int launch_sample_library(MppibContext* c, uint32_t k_offset, uint32_t k_total, const float* U, const float* prior_row, const float* Z,
                          float* actions, float* noise, cudaStream_t s);
int launch_rollout(MppibContext* c, const float* state0, const float* root0, float* state, const float* actions, int t0, int nsteps,
                   float* obs, cudaStream_t s);
int launch_reduce(MppibContext* c, const float* cost, const float* x, const float* U, float* partial, float* fin_U, float* fin_action,
                  float* fin_stats, cudaStream_t s);
int launch_finalize(MppibContext* c, const float* partials, int G, float* U, float* action_out, float* stats, cudaStream_t s);
int launch_shift(MppibContext* c, float* U, uint32_t* plan_ctr, cudaStream_t s);
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
