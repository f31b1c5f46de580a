/*
 * mppib.h -- C ABI of the H100-native MPPI rollout path ("mppib").
 *
 * This is the drop-in boundary below the Python planner host.  Every entry point
 * replaces one piece of the reference's hot path (tud-airlab/mppi-isaac @ 2e6d5fb,
 * paths relative to the reference tree):
 *
 *   mppib_sample    <- mppi_torch MPPIPlanner sampling + _bound_action (external dep
 *                      pinned in poetry.lock:1273-1293; call site mppi_isaac.py:43-49,113)
 *   mppib_rollout   <- IsaacGymWrapper.apply_robot_cmd + IsaacGymWrapper.step
 *                      (mppiisaac/planner/isaacgym_wrapper.py:524-572, 639-655), i.e.
 *                      gym.simulate/fetch_results/refresh_* for all K envs, T times
 *   mppib_reduce    <- mppi_torch _compute_rollout_costs accumulation + _exp_util
 *                      (softmax over K) + weighted control sum (call site mppi_isaac.py:113)
 *   mppib_finalize  <- mppi_torch _update_distribution / U update / savgol filter_u /
 *                      "return first action" (mppi_isaac.py:84,113)
 *
 * Conventions
 *   - extern "C", plain pointers and sizes only; no torch types.
 *   - Pointers without the _h suffix are DEVICE pointers into caller-owned buffers.
 *   - `stream` is a cudaStream_t passed as void*.
 *   - Every call returns 0 on success, <0 on error; mppib_last_error() gives the text.
 *   - A handle is bound to one device and is not thread-safe (one handle per GPU).
 *   - All floating point data is float32 (the reference path is float32 end to end:
 *     isaacgym_wrapper.py:232,262,612).
 *
 * Device data layouts (sample index k is always the innermost, contiguous dimension):
 *   U        [T][nu]            nominal control sequence (replicated on every GPU)
 *   actions  [T][nu][K]         clamped perturbed controls actually rolled out
 *   noise    [T][nu][K]         actions - U (after clamping / null / prior rows)
 *   state    [NS][K]            per-rollout simulator state, NS = mppib_state_size():
 *                               rows 0..ndof-1 = q, ndof..2ndof-1 = qdot, then free bodies
 *   obs      [R][T][K]          observed rows per step, R = mppib_obs_size()
 *   cost     [T][K]             per-step running cost from Objective.compute_cost
 *   partial  [2 + T*nu]         (beta_g, eta_g, W_g[T][nu]) of one shard
 */
#ifndef MPPIB_H
#define MPPIB_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPPIB_ABI_VERSION 13

#define MPPIB_MAX_BODIES 16   /* moving (1-DoF) bodies of the articulation            */
#define MPPIB_MAX_LINKS  32   /* URDF links whose state can be observed               */
#define MPPIB_MAX_NU     16   /* control dimension                                    */
#define MPPIB_MAX_OBS    64   /* observation items                                    */
#define MPPIB_MAX_FREE   4    /* free rigid bodies (box / sphere actors)              */
#define MPPIB_MAX_SHAPES 24   /* collision primitives                                 */
#define MPPIB_MAX_CONTACTS 24 /* contact points kept per rollout and substep             */
#define MPPIB_MAX_SLOTS  8    /* bodies whose net contact force is tracked            */

/* joint types (body frame is chosen so the joint axis is +z) */
#define MPPIB_JOINT_REVOLUTE  0
#define MPPIB_JOINT_PRISMATIC 1

/* drive modes: isaacgym_wrapper.py:491-507 */
#define MPPIB_DRIVE_VELOCITY 0   /* stiffness 0, damping 600 */
#define MPPIB_DRIVE_EFFORT   1   /* stiffness 0, damping 10, armature 0 */

/* observation item kinds (what Objective getters can read, isaacgym_wrapper.py:292-356) */
#define MPPIB_OBS_LINK_STATE   0  /* 13 floats: pos3 quat_xyzw4 linvel3 angvel3 of link `index`      */
#define MPPIB_OBS_DOF_STATE    1  /* 2*ndof floats interleaved q0,qd0,q1,qd1 (isaacgym_wrapper.py:190) */
#define MPPIB_OBS_FREE_STATE   2  /* 13 floats root state of free body `index`                       */
#define MPPIB_OBS_CONTACT      3  /* 3 floats net contact force on shape-owner `index`               */

/* shape types */
#define MPPIB_SHAPE_BOX    0
#define MPPIB_SHAPE_SPHERE 1

/* shape owner kinds */
#define MPPIB_OWNER_STATIC 0   /* fixed in the world                                   */
#define MPPIB_OWNER_LINK   1   /* attached to robot link owner_index                   */
#define MPPIB_OWNER_FREE   2   /* attached to free body owner_index                    */

/* MPPI update modes (mppi_torch `mppi_mode`, conf/mppi/panda.yaml:4 / omnipanda_effort.yaml:4) */
#define MPPIB_MODE_SIMPLE 0   /* U += sum_k w_k noise_k, cost += lambda U^T Sigma^-1 noise, gamma = 1 */
#define MPPIB_MODE_MEAN   1   /* "halton-spline" rule: mean <- (1-a) mean + a sum_k w_k action_k, discounted cost */

typedef struct MppibModel {
    int32_t abi_version;
    int32_t nb;                 /* moving bodies == ndof                                     */
    int32_t nlinks;             /* observable links (URDF order, depth first)                */
    int32_t nu;                 /* command dimension                                         */
    int32_t drive_mode;
    int32_t gravity_on;         /* ActorWrapper.gravity (isaacgym_utils.py:24)               */
    int32_t nfree;              /* free rigid bodies                                         */
    int32_t nshapes;
    float   gravity[3];         /* world gravity (0,0,-9.8): isaacgym_wrapper.py:29          */
    float   base_pos[3];        /* robot base pose in the world (actor root state)           */
    float   base_quat[4];       /* xyzw                                                      */

    /* articulation, topologically sorted; parent -1 = fixed base */
    int32_t parent[MPPIB_MAX_BODIES];
    int32_t jtype[MPPIB_MAX_BODIES];
    float   tree_R[MPPIB_MAX_BODIES][9];   /* rotation body(q=0) -> parent body coords, row major */
    float   tree_p[MPPIB_MAX_BODIES][3];   /* body origin in parent body coords                   */
    float   tree_quat[MPPIB_MAX_BODIES][4];/* tree_R as a unit quaternion, xyzw                   */
    float   mass[MPPIB_MAX_BODIES];
    float   mcom[MPPIB_MAX_BODIES][3];     /* mass * centre of mass, body coords                  */
    float   inertia[MPPIB_MAX_BODIES][6];  /* about the body origin: xx yy zz xy xz yz            */
    float   q_lo[MPPIB_MAX_BODIES];
    float   q_hi[MPPIB_MAX_BODIES];
    float   qd_max[MPPIB_MAX_BODIES];
    float   effort[MPPIB_MAX_BODIES];
    float   damping[MPPIB_MAX_BODIES];     /* URDF <dynamics damping>                             */
    float   kd[MPPIB_MAX_BODIES];          /* drive damping gain                                  */
    float   armature[MPPIB_MAX_BODIES];

    /* command map, apply_robot_cmd/_ik (isaacgym_wrapper.py:510-572):
       target[i] = cmd_c0[i]*u[cmd_i0[i]] + cmd_c1[i]*u[cmd_i1[i]] */
    int32_t cmd_i0[MPPIB_MAX_BODIES];
    int32_t cmd_i1[MPPIB_MAX_BODIES];
    float   cmd_c0[MPPIB_MAX_BODIES];
    float   cmd_c1[MPPIB_MAX_BODIES];
    /* differential-drive base reduced to a planar chain: bodies 0,1,2 are VIRTUAL joints (world x, world y, yaw) whose
       velocity targets follow the commanded body twist u = (v, omega): (v f(yaw), omega), f = forward axis rotated by yaw */
    int32_t planar_base;
    float   fwd_axis[2];

    /* observable links: pose of the link frame in its owning body's frame */
    int32_t link_body[MPPIB_MAX_LINKS];    /* -1 = rigidly attached to the base                   */
    float   link_R[MPPIB_MAX_LINKS][9];
    float   link_p[MPPIB_MAX_LINKS][3];
    float   link_quat[MPPIB_MAX_LINKS][4]; /* link_R as a unit quaternion, xyzw                   */

    /* free rigid bodies: box actors that are not fixed (isaacgym_utils.py:29-40, isaacgym_wrapper.py:450-456).
       Their initial state is row free_actor[f] of the root-state buffer handed to mppib_rollout.           */
    int32_t free_actor[MPPIB_MAX_FREE];
    float   free_mass[MPPIB_MAX_FREE];
    float   free_mass_pct[MPPIB_MAX_FREE];     /* noise_percentage_mass: mass *= 1 + pct * U(-1,1) per rollout */
    float   free_half[MPPIB_MAX_FREE][3];      /* box half extents (solid-box inertia for the configured mass) */
    int32_t free_gravity[MPPIB_MAX_FREE];
    int32_t free_slot[MPPIB_MAX_FREE];         /* row of the net-contact-force table, -1 none                  */

    /* collision boxes.  owner kind STATIC: pose = root state of actor shape_actor; LINK: rigidly attached to
       articulation body shape_owner (-1 = base) with the local pose below; FREE: free body shape_owner.     */
    int32_t shape_type[MPPIB_MAX_SHAPES];
    int32_t shape_owner_kind[MPPIB_MAX_SHAPES];
    int32_t shape_owner[MPPIB_MAX_SHAPES];
    int32_t shape_actor[MPPIB_MAX_SHAPES];     /* actor index (root-state row) for STATIC / FREE, -1 for LINK  */
    int32_t shape_slot[MPPIB_MAX_SHAPES];      /* row of the net-contact-force table, -1 none                  */
    float   shape_half[MPPIB_MAX_SHAPES][3];   /* box half extents                                             */
    float   shape_pos[MPPIB_MAX_SHAPES][3];    /* pose in the owner frame                                      */
    float   shape_quat[MPPIB_MAX_SHAPES][4];
    float   shape_friction[MPPIB_MAX_SHAPES];
    float   shape_fric_pct[MPPIB_MAX_SHAPES];  /* noise_percentage_friction (isaacgym_wrapper.py:468-475)      */
    float   shape_size_sigma[MPPIB_MAX_SHAPES][3]; /* noise_sigma_size on the FULL box size (isaacgym_utils.py:29-40) */
    int32_t ncontact_slots;
    int32_t ground_plane;                  /* add_ground_plane: z = 0, friction 1 (isaacgym_utils.py:61-68)    */
    float   ground_friction;
    float   contact_kp;                    /* penalty stiffness  [N/m]   (integrated implicitly)               */
    float   contact_kd;                    /* penalty damping    [N s/m]                                       */
    float   max_depen;                     /* cap of the penetration-recovery velocity [m/s]                   */
    float   ground_margin;                 /* speculative-contact distance to the ground plane [m]             */
    float   contact_margin;                /* speculative-contact distance between boxes [m] (PhysX contact_offset 0.01) */
    int32_t contact_iters;                 /* Gauss-Seidel sweeps over the contact set per substep             */
    int32_t nactors;                       /* rows of the root-state buffer                                    */
    int32_t max_contacts;                  /* contact points kept per rollout and substep: 1..MPPIB_MAX_CONTACTS (sized by the host so
                                              that the rollout's working set fits the 227 KB of shared memory of an SM)         */
} MppibModel;

typedef struct MppibObsItem {
    int32_t kind;
    int32_t index;
} MppibObsItem;

typedef struct MppibParams {
    int32_t K;                 /* samples on THIS device; mppib_reduce needs K % 4 == 0 (16-byte rows),
                                  sampling / rollout accept any K >= 1 (a one-env world simulator)        */
    int32_t T;                 /* horizon                                                  */
    int32_t substeps;          /* isaacgym_wrapper.py:24                                   */
    float   dt;                /* model step; substep h = dt/substeps                      */
    int32_t mode;              /* MPPIB_MODE_*                                             */
    float   lambda_;           /* temperature                                              */
    float   gamma;             /* rollout_var_discount (used by MODE_MEAN)                 */
    float   step_size_mean;    /* 0.98 in mppi_torch                                       */
    float   u_scale;
    int32_t sample_null_action;/* global row K-1 := 0                                      */
    int32_t filter_u;          /* Savitzky-Golay window 9 order 2 on U (needs T >= 9)      */
    float   u_min[MPPIB_MAX_NU];
    float   u_max[MPPIB_MAX_NU];
    float   u_init[MPPIB_MAX_NU];
    float   sigma_chol[MPPIB_MAX_NU * MPPIB_MAX_NU]; /* lower Cholesky factor of noise_sigma, row major nu x nu */
    float   sigma_inv[MPPIB_MAX_NU * MPPIB_MAX_NU];  /* inverse of noise_sigma, row major nu x nu               */
    uint32_t k_offset;         /* global index of local sample 0 (keys the per-rollout randomisation) */
    uint32_t rand_seed;        /* seed of the per-rollout size / mass / friction draws              */
    int32_t nobs;
    MppibObsItem obs[MPPIB_MAX_OBS];
} MppibParams;

typedef struct MppibContext* MppibHandle;

/* lifetime ------------------------------------------------------------------------------- */
int32_t mppib_abi_version(void);
const char* mppib_last_error(void);
int32_t mppib_create(const MppibModel* model_h, const MppibParams* params_h, int32_t device, MppibHandle* out);
int32_t mppib_destroy(MppibHandle h);
/* replaces the parameter block (update_mppi_params, mppi_isaac.py:129-138); K, T and obs may change */
int32_t mppib_set_params(MppibHandle h, const MppibParams* params_h);
/* replaces the model block (base pose / obstacle poses change between plans) */
int32_t mppib_set_model(MppibHandle h, const MppibModel* model_h);
int32_t mppib_state_size(MppibHandle h);   /* NS: rows of the state buffer             */
int32_t mppib_obs_size(MppibHandle h);     /* R: rows of the obs buffer                */

/* hot path ------------------------------------------------------------------------------- */
/* K1: Philox-4x32-10 Gaussian draw (key = seed, plan_idx; counter = global sample index
 * k_offset + k, t, block) -> noise = L z, action = clamp(u_scale-free U + noise, u_min, u_max),
 * noise := action - U; global row k_global == K_total-1 is the null action when enabled;
 * row K_total-2 is overwritten with prior_row[T][nu] when prior_row != NULL.  plan_ctr (device,
 * nullable) is added to plan_idx on the device so that a captured CUDA graph draws fresh noise on
 * every replay (mppib_shift increments it).                                                  */
int32_t mppib_sample(MppibHandle h, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr,
                     uint32_t k_offset, uint32_t k_total, const float* U, const float* prior_row,
                     float* actions, float* noise, void* stream);

/* Halton-spline noise library (mppi_torch `sampling_method: halton` / `mppi_mode: halton-spline`, conf/mppi/panda.yaml:4-5;
 * SURVEY.md 8(a) M4, 8(f) N3): Gaussian knots from a scrambled Halton sequence (dimension n*nu + i, bases / digit multipliers
 * in halton_tab[2][n_knots*nu], index = global sample + 1), z = sqrt(2) erfinv(2u - 1), interpolated to T points by the fixed
 * spline operator B[T][n_knots], coloured by the Cholesky factor of Sigma:  Z[t][j][k] = sum_n B[t][n] sum_i L[j][i] z[n][i].
 * Drawn ONCE per planner; global row k_total-1 is the zero-noise sample.                                                   */
int32_t mppib_noise_library(MppibHandle h, uint32_t k_offset, uint32_t k_total, const int32_t* halton_tab,
                            const float* B, int32_t n_knots, float* Z, void* stream);
/* K1 (library variant): action = clamp(U + Z), null / prior rows, noise = action - U.                                      */
int32_t mppib_sample_library(MppibHandle h, uint32_t k_offset, uint32_t k_total, const float* U, const float* prior_row,
                             const float* Z, float* actions, float* noise, void* stream);

/* K2: broadcast initial state state0[2*ndof] (+ free bodies from root0) to all K rollouts, or continue
 * from state[NS][K] when state0 == NULL; root0[nactors][13] holds the world's actor root states (poses of
 * static boxes, initial states of free bodies) and may be NULL for contact-free scenes; apply actions[t0 .. t0+nsteps) ; write obs and the
 * final state.  nsteps == T for a whole plan, 1 for the reference's step-wise protocol,
 * 0 to only write the observation of the current state into slot t0.                        */
int32_t mppib_rollout(MppibHandle h, const float* state0, const float* root0, float* state,
                      const float* actions, int32_t t0, int32_t nsteps, float* obs, void* stream);

/* K3: S_k = sum_t gamma^t cost[t][k] (+ lambda sum_t U_t^T Sigma^-1 noise_k,t in SIMPLE mode),
 * beta_g = min_k S_k, w_k = exp(-(S_k - beta_g)/lambda), eta_g = sum w_k,
 * W_g[t][j] = sum_k w_k x[t][j][k] with x = noise (SIMPLE) or actions (MEAN).
 * Single pass over HBM; the last CTA to finish folds the per-CTA partials.                  */
int32_t mppib_reduce(MppibHandle h, const float* cost, const float* x, const float* U,
                     float* partial, void* stream);

/* K3 + K4 in ONE launch for single-GPU plans (G = 1): the last CTA of the reduction, which holds the shard row, also updates
 * U in place (+ savgol, clamp), writes action_out[nu] and stats[2] -- same results as mppib_reduce followed by
 * mppib_finalize(partial, 1, ...), one kernel launch and one graph node less per plan.                                     */
int32_t mppib_reduce_finalize(MppibHandle h, const float* cost, const float* x, float* U, float* partial,
                              float* action_out, float* stats, void* stream);

/* K4: combine G shard partials, update U in place, optional savgol, write action_out[nu]
 * (= first row of U), and weights statistics stats[2] = (beta, eta).  partials == NULL with an
 * open peer window: take the G = world rows from the window (see mppib_peer_* below).          */
int32_t mppib_finalize(MppibHandle h, const float* partials, int32_t G, float* U,
                       float* action_out, float* stats, void* stream);

/* multi-GPU exchange over peer memory (one process per GPU, one box) -----------------------------
 * Replaces the all-gather between K3 and K4 (the reference has no multi-GPU path; this is the
 * multi-GPU scale-out of its single-GPU mppi_torch reduction, SURVEY.md 8(e)).  Every rank owns a small
 * WINDOW in its HBM: [2 parities][world] rows of 2 + T*nu floats plus one arrival flag per row.
 * With peers open, the last CTA of mppib_reduce stores this rank's (beta, eta, W) row straight
 * into the window of EVERY rank over NVLink (st.global + fence.sys + st.release.sys of the flag),
 * and mppib_finalize (called with partials == NULL) spins on its own window's flags
 * (ld.acquire.sys) before combining -- no host round trip, no NCCL kernel, graph-capturable.
 * Exchanges are numbered by a device-side counter inside the window, so every rank must issue the
 * same sequence of reduce/finalize pairs.  A peer that does not arrive within
 * MPPIB_PEER_TIMEOUT_S seconds (environment, default 20) traps the kernel (loud failure, no hang).
 *   mppib_peer_alloc : allocate + zero the local window, return its 64-byte cudaIpcMemHandle_t
 *   mppib_peer_open  : map the window of rank `peer` from the handle that rank returned
 *   mppib_peer_close : unmap / free; collective-free, the caller synchronises the ranks first    */
#define MPPIB_MAX_PEERS 16
#define MPPIB_IPC_HANDLE_BYTES 64
int32_t mppib_peer_alloc(MppibHandle h, int32_t world, int32_t rank, unsigned char* ipc_handle_out_h);
int32_t mppib_peer_open(MppibHandle h, int32_t peer, const unsigned char* ipc_handle_h);
int32_t mppib_peer_close(MppibHandle h);

/* Fused pose-reach cost term for Objectives (optional helper, no handle needed; the device is the one of the pointers /
 * current context).  cost[i] (+)= w_pos |a[i,0:3] - b[i,0:3]| + w_ori |euler_ZYX(R(a[i,3:7]))[0:2]| for i < n, the
 * quaternion read real-first as the reference's Objectives do (examples/panda/planner.py:22-40).  a and b are strided
 * views: element (i, c) of a lives at a[i*a_si + c*a_sr] (the obs layout gives a_si = 1, a_sr = T*K; a broadcast goal has
 * b_si = 0).  b may be NULL when w_pos == 0.                                                                          */
int32_t mppib_cost_pose(int64_t n, const float* a, int64_t a_si, int64_t a_sr, const float* b, int64_t b_si,
                        int64_t b_sr, float w_pos, float w_ori, float* cost, int32_t accumulate, void* stream);

/* Shared-memory bytes one 32-rollout CTA of mppib_rollout needs for this model (host-side arithmetic, no device access):
 * lets the model compiler size `max_contacts` to what fits an SM (226 KB usable) before a handle exists.                     */
int64_t mppib_rollout_smem_bytes(const MppibModel* model_h);

/* Which rollout kernel mppib_rollout launches for this handle's model (diagnostics / benchmark reporting; the result of the
 * rollout does not depend on it beyond float32 rounding -- every mapping is tested against the same oracle):
 * one thread per rollout, one articulation body per lane (serial chains without contacts), or a team of lanes per rollout
 * (trees; contact scenes of small robots).  The choice depends on the scene, never on K.  Environment MPPIB_K2_LANES=0 /
 * MPPIB_K2_TEAM=0 switch the lanes / team mapping off (the scene then falls to the next one, down to one thread per rollout). */
#define MPPIB_MAPPING_THREAD 0
#define MPPIB_MAPPING_LANES  1
#define MPPIB_MAPPING_TEAM   2
int32_t mppib_rollout_mapping(MppibHandle h);
/* The same decision for a model block before a handle exists (host-side arithmetic, no device access; honours the same environment
 * knobs): lets host code and tests see which scenes each kernel takes -- e.g. a tree whose bodies are not numbered depth first, or one
 * with more than 16 bodies, stays on the thread-per-rollout kernel.  Returns MPPIB_MAPPING_*, negative on a NULL model.        */
int32_t mppib_rollout_mapping_for_model(const MppibModel* model_h);

/* Optional host mirror of the action: when set, mppib_finalize also stores action_out[0..nu) to `mirror` -- a pointer into
 * PINNED host memory (device-addressable under unified addressing), so the caller of the reference's compute_action* only
 * waits for the stream instead of issuing a device->host copy.  NULL switches it off.                                      */
int32_t mppib_set_action_mirror(MppibHandle h, float* mirror);

/* shift U by one step: U[t] <- U[t+1], U[T-1] <- u_init (mppi_torch command() prologue);
 * increments *plan_ctr (device, nullable) by one.                                            */
int32_t mppib_shift(MppibHandle h, float* U, uint32_t* plan_ctr, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MPPIB_H */
