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
 *   partial  [2 + T*nu]         (beta_g, eta_g, W_g[T][nu]) of one shard;
 *            [2 + 2*T*nu]       (beta_g, eta_g, W_g, M2_g[T][nu]) with update_cov and a registered distribution
 *            [2 + T*nu + nu(nu+1)/2]  (beta_g, eta_g, W_g, C_g[lower triangle of nu x nu]) with update_cov, cov_full and a
 *                               registered distribution
 *   dist     [1 + nu]           (lambda, cov[nu]) live sampling distribution of adaptive MPPI (mppib_set_distribution);
 *            [1 + 3*nu*nu]      (lambda, Sigma[nu][nu], L[nu][nu], Sigma^-1[nu][nu]) with cov_full, all row-major, L lower
 *            [1 + 3*n*n]        (lambda, Sigma_H[n][n], L_H[n][n], Sigma_H^-1[n][n]) with cov_horizon, n = T*nu, the same layout
 *                               over the whole control sequence, vectors ordered (t, j) like U
 *   partial  [2 + n + n(n+1)/2] (beta_g, eta_g, W_g, C_g[lower triangle of n x n]) with update_cov, cov_horizon and a registered
 *                               distribution
 *   U, partial, dist with n_modes = M > 1: U[M][T][nu], partial [M][2 + T*nu] (one (beta, eta, W) block per mode), dist = the mode
 *                               state [1 + M + T*nu] (see "Multi-modal MPPI" below)
 */
#ifndef MPPIB_H
#define MPPIB_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPPIB_ABI_VERSION 24

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
#define MPPIB_MODE_CEM    2   /* iCEM rule: the E best samples (elites) by discounted cost; U, sigma <- momentum step towards their mean / std */
#define MPPIB_MODE_SMOOTH 3   /* Smooth MPPI: U is the control DERIVATIVE; actions are integrated from the last executed action (see below) */
#define MPPIB_CEM_MAX_ELITES 128
#define MPPIB_MAX_WORLDS 32   /* risk-aware MPPI: largest n_worlds (a group of worlds never straddles a 32-sample tile) */
#define MPPIB_MAX_MODES 16    /* multi-modal MPPI: largest n_modes */
#define MPPIB_MAX_ANNEAL 16   /* annealed MPPI: largest number of MPPI iterations per plan */
#define MPPIB_MAX_SPLINE_DEGREE 3   /* spline MPPI: largest spline_degree */
#define MPPIB_ESS_GRID 65           /* ESS-targeted temperature: grid temperatures lambda_j = lambda_ 2^((j - 32)/4), j = 0 .. 64 */
#define MPPIB_ESS_ROW_FLOATS 196    /* its shard row: (n_valid as int32 bits, (m_j, s1_j, s2_j)[65]) */
#define MPPIB_ESS_STATE_FLOATS 197  /* its state: (lambda_j[65], 1/lambda_j[65], n_valid as int32 bits, lambda, ESS_j[65]) */

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
    /* adaptive MPPI (mppi_torch update_cov / update_lambda): they act only once a distribution buffer is registered
       (mppib_set_distribution); lambda_ above is then the initial temperature lambda0 and the clamp centre             */
    int32_t update_cov;        /* K1 draws sqrt(cov) z, K3 adds the second-moment row, K4 updates cov (diagonal Sigma)  */
    int32_t update_lambda;     /* K4 adapts lambda to the weight sum eta                                               */
    float   eta_u_bound;       /* eta > bound: lambda *= 1 - lambda_mult                                                */
    float   eta_l_bound;       /* eta < bound: lambda *= 1 + lambda_mult; lambda stays in [1e-3, 1e3] * lambda0      */
    float   step_size_cov;     /* cov <- (1 - s) cov + s mean_t var_t + kappa                                          */
    float   kappa;
    float   lambda_mult;
    int32_t cov_full;          /* with update_cov: adapt a full Sigma (K1 draws L z, K3 appends C, K4 updates Sigma, L, Sigma^-1) */
    int32_t cov_horizon;       /* with update_cov: adapt one Sigma_H over the whole sequence, n = T*nu <= 256 (not with cov_full) */
    float   sigma0[MPPIB_MAX_NU * MPPIB_MAX_NU];    /* cov_horizon: Sigma0 = noise_sigma, row major nu x nu, the block a shift appends */
    /* MODE_CEM (see "Cross-entropy planning" below); sigma_chol must be diagonal, its diagonal is sigma0_j = sqrt(Sigma_jj)      */
    int32_t n_elites;          /* E, 1 .. MPPIB_CEM_MAX_ELITES                                                                   */
    int32_t n_keep;            /* E_keep <= E elites of the last update carried into the next samples (rows K_total - 3 - e)     */
    float   elite_alpha;       /* momentum alpha in [0, 1]: U <- (1 - alpha) mean + alpha U, sigma <- (1 - alpha) std + alpha sigma */
    /* MODE_SMOOTH (see "Smooth MPPI" below); u_min / u_max bound the ACTION, these the derivative                                  */
    float   du_min[MPPIB_MAX_NU];
    float   du_max[MPPIB_MAX_NU];
    float   smooth_weight;     /* omega >= 0: S_k += omega sum_t |a_t - a_{t-1}|^2 (t = 0 against the last executed action)        */
    /* risk-aware MPPI (see "Risk-aware MPPI" below); both are read only when n_worlds > 1, a zero block keeps today's planner      */
    int32_t n_worlds;          /* R: rollouts per control sample, a power of two in 1 .. MPPIB_MAX_WORLDS; K and k_offset are multiples */
    int32_t risk_tail;         /* m in 1 .. R: the score of a control is the mean of its m largest world costs (CVaR)              */
    /* multi-modal MPPI (see "Multi-modal MPPI" below); read only when n_modes > 1, a zero block keeps today's planner               */
    int32_t n_modes;           /* M in 1 .. MPPIB_MAX_MODES nominal sequences planned side by side                                   */
    float   mode_margin;       /* >= 0: the executed mode is kept while its free energy is within this margin of the lowest          */
    int32_t mode_samples;      /* Kc = K_total / M >= 32: global sample kg belongs to mode kg / Kc (the shard alone cannot tell K_total) */
    /* constrained MPPI (see "Constrained MPPI" below); constraint_mode = 0 (and a zero-initialised block) keeps today's planner        */
    int32_t constraint_mode;   /* 1: feasibility-first weighting over the per-step violations registered with mppib_set_constraint      */
    float   constraint_tol;    /* a sample is feasible when its total violation V_k <= tol; finite and >= 0                             */
    float   constraint_lambda; /* lambda_c: the temperature of the violation fallback; finite and > 0                                    */
    int32_t constraint_pad;    /* 0; keeps the spline fields below at the 8-byte alignment they had before the constraint fields       */
    /* ESS-targeted temperature (see "ESS-targeted temperature" below); lambda_ess = 0 (and a zero-initialised block) keeps today's planner;
       the two fields sit before the spline fields, so those keep their 8-byte alignment and stay the last of the block */
    int32_t lambda_ess;        /* 1: every plan chooses lambda on the device so that the weights keep ess_target of the valid samples     */
    float   ess_target;        /* rho in (0, 1], finite, read only when lambda_ess = 1                                                   */
    /* spline MPPI (see "Spline MPPI" below); control_knots = 0 (and a zero-initialised block) keeps today's planner                   */
    int32_t control_knots;     /* P: U, the samples K3 weights and the shard row hold P knots per control instead of T steps            */
    int32_t spline_degree;     /* d in 1 .. MPPIB_MAX_SPLINE_DEGREE, read only when control_knots > 0; P in d + 1 .. T, P*nu <= 512   */
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

/* Which K1 entry samples which mode.  The draw follows the plan's update rule: mode cem, then mode smooth, then, with a registered
 * distribution and update_cov, cov_horizon, cov_full or the diagonal; update_lambda alone, n_modes > 1 and annealing keep the fixed Sigma.
 * A refused pair returns an error before anything is launched.
 *
 *   handle state                    mppib_sample  _colored  _smooth  mppib_noise_library   mppib_sample_library
 *   fixed Sigma                     yes           yes       -        yes (coloured by L0)  yes
 *   update_cov, diagonal            yes           yes       -        yes (white)           yes
 *   update_cov, cov_full            yes           yes       -        yes (white)           yes
 *   update_cov, cov_horizon         yes           - (a)     -        yes (white)           yes
 *   mode cem                        -             yes (b)   -        -                     -
 *   mode smooth                     -             -         yes (c)  -                     -
 *   n_modes > 1                     yes (d)       yes (d)   -        yes                   yes (d)
 *   n_worlds > 1                    yes (e)       yes (e)   -        yes (e)               yes (e)
 *   annealing schedule registered   yes (f)       yes (f)   -        -                     -
 *   control_knots > 0               -             -         -        -                     -          (mppib_sample_spline: yes (g))
 *
 * (a) even with no distribution registered: cov_horizon models the time correlation itself
 * (b) with the CEM state registered (mppib_set_distribution)
 * (c) with the smooth state registered (mppib_set_smooth_state); the parameter block already excludes n_worlds > 1 and n_modes > 1
 * (d) k_total = n_modes * mode_samples
 * (e) K, k_offset and k_total multiples of n_worlds
 * (f) registered for the handle's T; the library entries refuse a schedule whatever its T
 * (g) with a spline table registered for the handle's (T, control_knots, spline_degree) (mppib_set_spline); the parameter block already
 *     excludes every draw but the fixed Sigma
 * Every entry also needs its pointers, k_offset + K <= k_total and its size limits: colored T <= 256 and T*nu <= 512, smooth
 * T*nu <= 512, the noise library 1 <= n_knots <= 32, cov_horizon T*nu <= 256.                                              */

/* K1 (colored variant, `sampling_method: colored`): the white draws z[t][i] of mppib_sample (same counters and transform) are
 * first correlated over the horizon, w[t][i] = sum_{t' <= t} Lt[t][t'] z[t'][i], with Lt[T][T] (caller-owned device memory,
 * row-major, lower) the Cholesky factor of the power-law temporal covariance, then coloured over the controls, clamped and
 * stored as in mppib_sample (the fixed Sigma, or the live diagonal / full one of a registered distribution with update_cov).
 * Both sums run in a fixed order: with Lt = I the result equals mppib_sample's bit for bit.  Needs T <= 256, T*nu <= 512 and
 * no cov_horizon.                                                                                                          */
int32_t mppib_sample_colored(MppibHandle h, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr,
                             uint32_t k_offset, uint32_t k_total, const float* U, const float* prior_row,
                             const float* Lt, float* actions, float* noise, void* stream);

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
 * With a registered distribution lambda (and, with update_cov, Sigma^-1 = diag(1/cov)) come from it, and update_cov appends
 * M2_g[t][j] = sum_k w_k (x[t][j][k] - c[t][j])^2, c = U (MEAN) or 0 (SIMPLE).  With cov_full too, Sigma^-1 is the full one of
 * the buffer and the row carries C_g = sum_t sum_k w_k (x_tk - c_t)(x_tk - c_t)^T instead of M2_g, packed as its lower triangle
 * (i >= j, row-major, nu(nu+1)/2 floats); row length 2 + T*nu + nu(nu+1)/2.
 * With cov_horizon instead, n = T*nu: the SIMPLE-mode term is g^T x_k with g = lambda Sigma_H^-1 U computed by the last
 * mppib_shift, K3 stores every S_k in a handle-owned buffer, and a second kernel of this call (a weighted SYRK, tiled over the
 * lower triangle and split over K, folded in a fixed order) appends C_g = sum_k w_k (x_k - c)(x_k - c)^T over the whole
 * n-vector x_k, packed as its lower triangle; row length 2 + n + n(n+1)/2.
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
 * WINDOW in its HBM: [2 parities][world] rows of 2 + T*nu floats (2 + 2*T*nu with update_cov, 2 + T*nu + nu(nu+1)/2 with
 * update_cov and cov_full, 2 + n + n(n+1)/2 with update_cov and cov_horizon; rounded up to a multiple of 4) plus one arrival flag
 * per row.  With cov_horizon the row is complete only after the SYRK, so its last CTA stores it into the windows.
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

/* Adaptive MPPI: register the device buffer dist[1 + nu] = (lambda, cov[nu]) (float32, caller-owned, initialised by the caller).
 * Once set, K1 draws noise_j = sqrt(cov_j) z_j (update_cov; mppib_noise_library then builds a WHITE library that
 * mppib_sample_library scales per plan), K3 weights with the buffer's lambda (and diag(1/cov)), and K4 updates the buffer in
 * place after the U update: cov (update_cov, needs the [2 + 2*T*nu] partial rows) and lambda (update_lambda); dist is left
 * as it is when no sample is valid.  Because the buffer lives in device memory, a captured plan graph follows it.  NULL
 * switches it off: every launch then runs the fixed-distribution kernels.
 * With update_cov and cov_full the buffer is dist[1 + 3*nu*nu] = (lambda, Sigma[nu][nu], L[nu][nu], Sigma^-1[nu][nu]), row-major,
 * L the lower Cholesky factor of Sigma (zero above the diagonal), all three consistent at registration.  K1 draws noise = L z
 * (the library sampler colours the white library by L), K3 uses the full Sigma^-1 in SIMPLE mode and appends C, and K4 updates
 * Sigma, then L and Sigma^-1 on the device; a non-positive-definite update leaves the three as they were.  The partial rows
 * are [2 + T*nu + nu(nu+1)/2].
 * With update_cov and cov_horizon the buffer is dist[1 + 3*n*n] = (lambda, Sigma_H, L_H, Sigma_H^-1), n = T*nu, the same layout
 * over the whole control sequence.  K1 draws noise = L_H z over the n-vector of a sample, K3 reads lambda Sigma_H^-1 U from
 * mppib_shift in SIMPLE mode, the SYRK appends C, and K4 updates Sigma_H, shifts it by one step like U (the appended block is
 * sigma0), then factors it in one CTA; a non-positive-definite result leaves the three as they were.  The partial rows are
 * [2 + n + n(n+1)/2].                                                                                                       */
int32_t mppib_set_distribution(MppibHandle h, float* dist);

/* shift U by one step: U[t] <- U[t+1], U[T-1] <- u_init (mppi_torch command() prologue);
 * increments *plan_ctr (device, nullable) by one.  With update_cov, cov_horizon and a registered distribution it also computes
 * g = lambda Sigma_H^-1 U of the shifted U once per plan, which K3 reads in SIMPLE mode.                                     */
int32_t mppib_shift(MppibHandle h, float* U, uint32_t* plan_ctr, void* stream);

/* Cross-entropy planning (mode MPPIB_MODE_CEM, `mppi_mode: cem`, iCEM).  The distribution is diagonal and per step: the mean U[T][nu]
 * and sigma[T][nu], both in the CEM state, a device buffer registered with mppib_set_distribution (NR = T*nu, E = n_elites):
 *   state    [2 + E + NR + E*NR]  (carry offset, elites valid, S_elite[E], sigma[T][nu], elites[E][T][nu]); offset and flag are 0.0 / 1.0
 * One plan is mppib_shift, then I iterations of K1 -> K2 -> cost -> mppib_reduce (+ mppib_finalize); nothing on the host changes
 * between iterations but plan_idx, so the whole plan is one CUDA graph.
 *   K1     mppib_sample_colored (white noise: Lt = I): a = clamp(U + sigma (.) w); global rows K_total - 3 - e, e < n_keep, copy
 *          clamp(elites[e][t + off]) with off = the carry offset (the row's own draw where t + off = T) once the elites are valid.
 *   K3     mppib_reduce / mppib_reduce_finalize with x = actions: S_k = sum_t gamma^t cost[t][k] in t order (+0 for -0), key =
 *          (S_k, global index) lexicographically, non-finite S never an elite.  The shard row holds the shard's E smallest keys in
 *          order and their actions:
 *   partial  [4-aligned 2E + E*NR]  (S_e, index bits as float)[E], actions[E][T][nu]; a missing entry is (+inf, 0xFFFFFFFF, zeros)
 *   K4     mppib_finalize (or the last CTA of mppib_reduce_finalize) merges the G*E candidates into the global E smallest keys --
 *          the elite set does not depend on G -- and, with E finite elites, sets m = mean_e a_e, s = sqrt(mean_e (a_e - m)^2) in
 *          elite-rank order, U <- (1 - alpha) m + alpha U, sigma <- (1 - alpha) s + alpha sigma, stores the elites and their S and sets
 *          the carry offset to 0; with fewer it leaves U, sigma, the elites and the offset as they are.  Then Savitzky-Golay, clamp,
 *          first action and mirror as in the other modes; stats = (S of the best elite, S of the E-th).
 *   shift  U as in the other modes, sigma <- sigma0 for every t, carry offset <- 1, *plan_ctr += 1.
 * The other K1 entries refuse this mode (the K1 table at mppib_sample).                                                     */

/* Smooth MPPI (mode MPPIB_MODE_SMOOTH, `mppi_mode: smooth`, after Kim, Kwon, Yoon, RA-L 2022).  U[T][nu] is the mean of the control
 * DERIVATIVE v; the rolled-out and executed actions are its integral from the last executed action, so with derivative bounds the
 * executed command changes by at most du_max * dt per plan.  noise_sigma is the covariance of the derivative noise, u_min / u_max
 * bound the action, du_min / du_max the derivative, dt = MppibParams.dt is the integration step, gamma = 1.  The smooth state is a
 * device buffer registered with mppib_set_smooth_state (caller-owned, initialised by the caller):
 *   state    [nu + T*nu]  (a_prev[nu], A[T][nu]): the last executed action and the planned action sequence; only K4 writes it
 *   K1     mppib_sample_smooth: per sample, t = 0 .. T-1 in order from a = a_prev: the white draws z of mppib_sample (same counters),
 *          n = L0 z (colour_clamp_store's order), v = clamp(U[t] + n, du_min, du_max) (v = 0 on the null row), a_t = clamp(fmaf(v, dt,
 *          a_{t-1}), u_min, u_max); actions = a_t, noise = v - U[t] where the action clamp did not bind, (a_t - a_{t-1})/dt - U[t]
 *          where it did (the derivative actually applied)
 *   K3     mppib_reduce / mppib_reduce_finalize with x = noise, as SIMPLE (gamma = 1, g = lambda Sigma^-1 U) plus the smoothness cost:
 *          S_k = sum_t c[t][k] + sum_r g_r x_rk + omega dt^2 sum_r (U_r + x_rk)^2; the shard row is SIMPLE's [2 + T*nu]
 *   K4     mppib_finalize (or the fused tail): U' = clamp(U + W/eta, du_min, du_max) (U' = U when eta = 0), then per j in t order from
 *          a = a_prev: A_t = clamp(fmaf(U'_t, dt, a), u_min, u_max), U'_t := (A_t - a)/dt where that clamp bound, a = A_t; U <- U',
 *          A stored, action_out and the mirror <- A_0, a_prev <- A_0; stats = (beta, eta).  filter_u is refused in this mode.
 *   shift  U as in the other modes (the appended u_init is a derivative: 0 holds the last action), *plan_ctr += 1; A is not shifted.
 * The other K1 entries refuse this mode (the K1 table at mppib_sample); reduce and finalize refuse it while no state is
 * registered.  A distribution registered with mppib_set_distribution is ignored in this mode.                               */
int32_t mppib_set_smooth_state(MppibHandle h, float* state);

/* Risk-aware MPPI (n_worlds = R > 1, risk_tail = m; modes SIMPLE and MEAN, fixed, diagonal or full Sigma; not cov_horizon).  The K
 * rollouts are Kc = K_total / R control samples of R rollouts each: global rollout kg = c*R + r runs control c in world r.
 *   K1     every variant but smooth / horizon keys its Philox draws (or Halton index) and its null / prior tests by c against Kc
 *          instead of kg against K_total, so the R rollouts of a control carry the same actions: the result is np.repeat of the
 *          K1 at K_total = Kc, R times along k.  The null control is c = Kc - 1.
 *   K2     the per-rollout size / mass / friction draws are keyed by the world r = kg % R instead of kg, so every control faces the
 *          same R worlds (common random numbers), the same on every plan.
 *   K3     S_k as before; then per aligned group of R lanes: a non-finite S_k becomes +inf, the group is sorted in descending order,
 *          rho_c = (s_(0) + ... + s_(m-1)) / m (float32, summed left to right, one division) goes to lane r = 0 and +inf to the
 *          others, and the rest of K3 runs unchanged: the shard row is the control-level row of a Kc-sample MPPI, beta = min rho.
 *   K4, the shift and the peer exchange are unchanged.  The launchers refuse a shard whose K or k_offset is not a multiple of R. */
int32_t mppib_sample_smooth(MppibHandle h, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset,
                            uint32_t k_total, const float* U, float* actions, float* noise, void* stream);

/* Multi-modal MPPI (n_modes = M > 1, mode_samples = Kc; modes SIMPLE and MEAN with the fixed Sigma; no update_cov / update_lambda,
 * n_worlds, cem or smooth).  U is [M][T][nu], mode 0 first; global sample kg belongs to mode m(kg) = kg / Kc, a contiguous block, so a
 * mode may span shards and a shard may hold several modes.  The mode state is a device buffer registered with mppib_set_distribution
 * (caller-owned, initialised by the caller; only K4 writes it):
 *   state    [1 + M + T*nu]  (active mode as a float, F[M], U_exec[T][nu])
 *   K1     mppib_sample, mppib_sample_colored and mppib_sample_library draw sample kg around U + m(kg)*T*nu with the counters of the
 *          global index: the columns of mode m equal today's K1 with U := U_m, bit for bit (entries: the K1 table at mppib_sample)
 *   K3     one launch, CTAs (x, m): the shard row is M blocks of SIMPLE's / MEAN's row, [M][2 + T*nu], block m = (beta_m, eta_m, W_m)
 *          over the shard's samples of mode m only (g_m = lambda Sigma^-1 U_m in SIMPLE mode); a mode without a sample on the shard
 *          writes (+inf, 0, 0); a 32-sample tile straddling two modes is read by both modes' CTAs, each masking the other's lanes
 *   K4     per mode: the G blocks m combined as today -> (beta_m, eta_m, W_m), the own step d_m = W_m/eta_m (SIMPLE) or
 *          (1 - s) U_m + s W_m/eta_m - U_m (MEAN), d_m = 0 when eta_m = 0, F_m = beta_m - lambda ln(eta_m / Kc) (+inf when eta_m = 0);
 *          then, from the U before the update, in float32 with every sum over j in ascending order:
 *            D_ij = sum_t (U_it - U_jt)^T Sigma^-1 (U_it - U_jt),  h = lower median {D_ij : i < j} / ln(M + 1),  k_ij = exp(-D_ij / h),
 *            U_i <- U_i + (sum_j k_ij d_j + (2/h) sum_j k_ij (U_i - U_j)) / sum_j k_ij   (k = 1 and no second term if h is 0 or not finite)
 *          then Savitzky-Golay (filter_u) and the clamp to every mode; the executed mode p is kept while F_p <= min F + mode_margin,
 *          otherwise it becomes argmin F (lowest index; all F infinite keeps p); the action, its mirror and stats = (beta_p, eta_p) come
 *          from mode p, and the state receives (p, F, U_p).
 *   shift  every mode as U is shifted today.
 * Reduce and finalize refuse M > 1 while no mode state is registered.                                                             */

/* Annealed MPPI (N MPPI iterations per plan with a noise schedule over iterations and horizon; modes SIMPLE and MEAN with the fixed
 * Sigma, Gaussian or colored K1, any n_worlds; no update_cov / update_lambda, cem, smooth, n_modes > 1 or Halton library).  The schedule
 * is a device buffer registered with mppib_set_anneal (caller-owned, initialised by the caller; N = n_iterations in 1 .. MPPIB_MAX_ANNEAL):
 *   state    [1 + 2*N*T]  (iteration counter as a float, s[N][T], r[N][T]); the host fills s[i][t] = c_i^i c_h^(T-1-t) and
 *                         r[i][t] = 1 / s[i][t]^2, both from float64 rounded once; iteration i reads row min(counter, N - 1)
 * One plan is mppib_shift, then N times K1 -> K2 -> cost -> K3 -> (exchange) -> K4; nothing on the host changes between iterations but
 * plan_idx = i << 32, so a batched plan is one CUDA graph.
 *   K1     mppib_sample and mppib_sample_colored (fixed Sigma, with their n_worlds keying): the draw and colour of today's K1, then
 *          noise_j = s[i][t] (L z)_j with one float32 multiplication, a = clamp(U + noise) with the null / prior rows, noise := a - U
 *   K3     SIMPLE mode: g_r = (lambda (Sigma^-1 U)_r) r[i][t], the importance-sampling term under N(U, s^2 Sigma), one multiplication
 *          after the lambda product; MEAN mode is unchanged (only its samples are annealed).  Every RPL / RISK instantiation, split or fused.
 *   K4     today's update (Savitzky-Golay, clamp, action, mirror, stats), then counter := counter + 1 (split and fused tail); the action and
 *          stats of a plan are those of its last iteration
 *   shift  as today, then counter := 0
 * With s = 1 every added operation multiplies by 1.0f: a registered schedule of ones with N = 1 reproduces the plain plan bit for bit.
 * Registration refuses N outside 1 .. MPPIB_MAX_ANNEAL and the excluded modes; the library records T there and refuses every launch once
 * mppib_set_params has changed T (or switched to an excluded mode) without a new registration.  The K1 table at mppib_sample lists the
 * entries that refuse a registered schedule.  NULL switches it off: every launch is then today's.                                    */
int32_t mppib_set_anneal(MppibHandle h, float* state, int32_t n_iterations);

/* Spline MPPI (control_knots = P > 0, spline_degree = d; modes SIMPLE and MEAN with the fixed Sigma; no filter_u, update_cov /
 * update_lambda, cem, smooth, n_modes > 1, n_worlds > 1 or annealing).  The planned control sequence is a clamped uniform B-spline of
 * degree d on [0, T-1] with P control knots theta[P][nu]: the action at step t is a_t = sum_p B[t][p] theta_p.  U is theta[P][nu], and
 * the vector K3 weights, K4 updates and the shard row carries is P*nu long (partial [2 + P*nu]); the cost rows stay T.  The table is a
 * device buffer registered with mppib_set_spline (caller-owned, filled by the caller; S = d + 3 floats per row):
 *   table    [(T + P)*S + T*nu]  rows[T + P][S], then U_exec[T][nu].  Row r = (first index, count, weights[count]) of the non-zero
 *            weights in ascending index order: rows 0 .. T-1 interpolate (B[t]), rows T .. T+P-1 shift (theta'_p = sum_q N_q(xi_p + 1)
 *            theta_q at the Greville abscissa xi_p, count 0 = u_init).  Indices and counts are stored as floats.
 *   K1     mppib_sample_spline: for knot p of sample k the white draws of mppib_sample with p in the t slot of the counter,
 *          theta~ = clamp(theta_p + L0 z) (null row: clamp(0)), xk[P][nu][K] = theta~ - theta_p (SIMPLE) or theta~ (MEAN);
 *          actions[T][nu][K] = clamp(sum_q w_q theta~_{first+q}, u_min, u_max) (the first term a product, the rest fmaf in index
 *          order; the clamp only absorbs the rounding of the float32 weights, whose exact values are convex)
 *   K3     mppib_reduce / mppib_reduce_finalize with x = xk: today's K3 over the P*nu rows (g = lambda Sigma^-1 theta per knot)
 *   K4     today's update of theta (split and fused tail); action_out = theta_0 = a_0 (B[0] = e_0); U_exec = B theta by the same sums
 *   shift  theta <- the shift rows applied to theta; *plan_ctr += 1
 * With d = 1 and P = T, B = I and every row holds one weight 1.0: the plan equals today's bit for bit.  Registration records (T, P, d);
 * K1, K3, K4 and the shift refuse a handle with P > 0 while no table or one registered for another (T, P, d) is set, or while a
 * distribution is registered.  NULL switches it off.                                                                              */
int32_t mppib_set_spline(MppibHandle h, float* table, int32_t P, int32_t d);
int32_t mppib_sample_spline(MppibHandle h, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset,
                            uint32_t k_total, const float* U, float* actions, float* xk, void* stream);

/* Constrained MPPI (constraint_mode = 1; modes SIMPLE and MEAN with the fixed Sigma, any K1 that feeds the plain rule -- Gaussian,
 * colored, Halton library -- filter_u, the null / prior rows and any number of ranks; no update_cov / update_lambda, cem, smooth,
 * n_modes > 1, n_worlds > 1, annealing or control_knots > 0).  The Objective returns a signed margin g[t][k] per step (<= 0 satisfied,
 * > 0 the amount of violation) into a device buffer registered with mppib_set_constraint (caller-owned, written by the caller before
 * every K3):
 *   viol     [T][K]  g of the shard's samples, float32
 *   cstate   [2]     (n_feasible as int32 bits, min V) of the last plan, written by K4
 *   K3     per sample V_k = sum_t c[t][k] in t order in float32, c = g where g > 0, 0 where g <= 0 (NaN stays NaN); valid = today's
 *          validity and V_k finite, feasible = valid and V_k <= constraint_tol.  A tile holding a feasible sample weights its feasible
 *          samples by exp(-(S_k - b)/lambda) (S_k as today); one without weights its valid samples by exp(-(V_k - b)/lambda_c) (no
 *          control cost, no gamma^t).  The states (n_feasible, b, eta, W) merge lexicographically: one with n_feasible > 0 beats one
 *          with 0 (which then weighs 0), two of one kind merge by today's rescale with their temperature and add their counts
 *          (merge_scale in csrc/common.cuh, the same function at every fold).  The shard row is
 *   partial  [4 + T*nu]  (beta, eta, W[T*nu], n_feasible as int32 bits, min V over the shard's valid samples (+inf: none))
 *   K4     mppib_finalize (or the fused tail) merges the G rows the same way, then today's update, Savitzky-Golay, clamp, action, mirror;
 *          stats = (beta, eta) of the kind that won, cstate = (sum n_feasible, min V).  No valid sample anywhere: U unchanged.
 *   shift  unchanged.
 * With every g <= 0 each sample is feasible exactly when it is valid today, and every weight, sum and scale is today's: the plan equals
 * today's bit for bit.  Registration records (T, K); reduce and finalize refuse a handle whose constraint_mode and registration disagree
 * or whose T or K changed since, and one with a distribution or annealing schedule registered.  NULL switches it off.             */
int32_t mppib_set_constraint(MppibHandle h, const float* viol, float* cstate);

/* ESS-targeted temperature (lambda_ess = 1, ess_target = rho; modes SIMPLE and MEAN, fixed, diagonal or full Sigma, any K1 but smooth's,
 * filter_u, the null / prior rows and any number of ranks; no update_lambda, cov_horizon, cem, smooth, n_worlds > 1, n_modes > 1,
 * control_knots > 0, constraint_mode or annealing).  Every plan chooses its temperature from its own costs, after the Objective's cost
 * (and the stepwise prior row's noise rewrite) and before K3:
 *   per sample  C_k = sum_t gamma^t c[t][k], q_k = sum_r (Sigma^-1 U)_r x[r][k] in SIMPLE mode (Sigma^-1 = K3's: sigma_inv, diag(1/cov)
 *               with update_cov, dist's full one with cov_full), q_k = 0 in MEAN mode, so S_k(lambda) = C_k + lambda q_k is K3's S; a
 *               sample is valid when k < K and C_k and q_k are finite
 *   grid        lambda_j = lambda_ 2^((j - 32)/4), j = 0 .. 64, and 1/lambda_j, each computed in float64 and rounded once by the caller
 *               into the state
 *   curve       a_jk = C_k / lambda_j + q_k; ESS_j = (sum_k e^-a_jk)^2 / sum_k e^-2a_jk over the valid samples of every rank, shifted by
 *               m_j = min_k a_jk; N = the valid samples of every rank
 *   rule        tau = rho N, j* = the first j with ESS_j >= tau: lambda = lambda_64 if there is none, lambda_0 if j* = 0, otherwise
 *               lambda_{j*-1} 2^(theta/4), theta = (ln tau - ln ESS_{j*-1}) / (ln ESS_{j*} - ln ESS_{j*-1}); N = 0 keeps dist[0]
 *   result      dist[0] <- lambda; K1 .. K4 and the shift then run the registered distribution's path (update_lambda is off, so K4 leaves
 *               dist[0] as it is, and K1 keeps the fixed Sigma unless update_cov is on)
 * The distribution (mppib_set_distribution, (lambda, cov[nu]) or cov_full's layout) is registered even with both adaptive flags off, and
 * the state is a device buffer registered with mppib_set_temperature (caller-owned; the caller fills the grid):
 *   state    [MPPIB_ESS_STATE_FLOATS]  (lambda_j[65], 1/lambda_j[65], n_valid as int32 bits, lambda chosen, ESS_j[65]); the solve writes
 *            the last three
 *   row      [MPPIB_ESS_ROW_FLOATS]    (n_valid as int32 bits, (m_j, s1_j, s2_j)[65]) of one shard; s1 = sum e^-(a - m),
 *            s2 = sum e^-2(a - m)
 * Every rank combines the rows in rank order (CTA partials in CTA order) with the same float32 arithmetic, so all choose the same bits.
 * Reduce and finalize refuse lambda_ess = 1 while no distribution or no state is registered: they would weight with lambda_. */
int32_t mppib_set_temperature(MppibHandle h, float* state);
/* The temperature pass <- the fixed mppi_torch `lambda_` of _exp_util (call site mppi_isaac.py:113): per-CTA curves over the shard, folded
 * by the last CTA into `row` (device, MPPIB_ESS_ROW_FLOATS floats).  solve = 1: the last CTA also applies the rule -- to its own row
 * without peers, or, with the peer window open, after publishing the row into every rank's window and acquiring every rank's row (a second
 * exchange per plan on the window K3 / K4 use).  solve = 0 writes the row only, for an all-gather and mppib_temperature_solve.  x is the
 * noise K3 weights in SIMPLE mode (not read in MEAN mode, may be NULL there).  Needs T <= 256 and T*nu <= 512. */
int32_t mppib_temperature(MppibHandle h, const float* cost, const float* x, const float* U, float* row, int32_t solve, void* stream);
/* The rule over G rows[G][MPPIB_ESS_ROW_FLOATS] (device, rank order) <- the same as above, one warp: the multi-GPU path without peers. */
int32_t mppib_temperature_solve(MppibHandle h, const float* rows, int32_t G, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MPPIB_H */
