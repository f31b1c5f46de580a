// oracle.cpp -- CPU restatement of the MPPI rollout hot path.  TEST INFRASTRUCTURE ONLY.
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
// load this library; the product package never imports it (it fails loudly without CUDA).
//
// PARITY UNPINNED: the arithmetic of this path lives in two third-party engines that are not
// in the reference repository and cannot be installed with it -- mppi_torch @75e17e87 (pyproject.toml:20,
// poetry.lock:1273-1293) and IsaacGym 1.0rc4 / PhysX (pyproject.toml:16, thirdparty/README.md:3).
// The reference ships no golden vectors for them (SURVEY.md section 4).  This file therefore
// restates the *pipeline* the reference source does pin, function by function:
//
//   oracle_sample    : mppi_torch "simple"/"random" Gaussian draw + _bound_action + null/prior rows
//                      (spec: SURVEY.md 8(a) M4/M5; row K-1 null action, row K-2 prior,
//                      mppiisaac/priors/fabrics_point.py:20 env_id=-2)
//   oracle_rollout   : IsaacGymWrapper.apply_robot_cmd + step for K envs, T times
//                      (mppiisaac/planner/isaacgym_wrapper.py:510-572 command map and diff-drive IK,
//                       :639-655 step order command -> simulate -> observe, :21-39 dt/substeps/gravity,
//                       :491-507 drive gains, :186-199 tensor layouts)
//   oracle_reduce    : mppi_torch _compute_rollout_costs accumulation, _exp_util, weighted sum
//                      (SURVEY.md 8(a) M5/M6)
//   oracle_finalize  : shard combine (SURVEY.md 8(e)) + _update_distribution + savgol (Appendix C)
//
// It is written for clarity, not speed: dense 6x6 spatial algebra (Featherstone's ABA), no
// structure exploitation, optional float64 to quantify float32 round-off of the CUDA path.
// What pins it: tests/test_oracle_*.py (FK golden values of SURVEY Appendix B, an independent
// numpy CRBA/RNEA mass-matrix solve, scipy savgol, torch softmax, analytic drive response).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>
#include <algorithm>
#include <limits>

#include "../include/mppib.h"

namespace {

// ------------------------------------------------------------------------------------------
// Philox-4x32-10 (Salmon et al. 2011).  key = (seed_lo, seed_hi ^ plan_lo), counter =
// (global sample index, t, block, plan_hi).
// ------------------------------------------------------------------------------------------
struct U4 { uint32_t x, y, z, w; };

inline U4 philox4x32_10(U4 c, uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)M0 * c.x, p1 = (uint64_t)M1 * c.z;
        U4 n;
        n.x = (uint32_t)(p1 >> 32) ^ c.y ^ k0;
        n.y = (uint32_t)p1;
        n.z = (uint32_t)(p0 >> 32) ^ c.w ^ k1;
        n.w = (uint32_t)p0;
        c = n;
        k0 += W0; k1 += W1;
    }
    return c;
}

inline float u01(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }

// Box-Muller in double, rounded to float: the reference value the CUDA fast path is held to.
inline void box_muller(uint32_t a, uint32_t b, float* z0, float* z1) {
    double u0 = (double)u01(a), u1 = (double)u01(b);
    double r = std::sqrt(-2.0 * std::log(u0));
    double th = 2.0 * M_PI * u1;
    *z0 = (float)(r * std::cos(th));
    *z1 = (float)(r * std::sin(th));
}

// Persistent worker pool (the CPU arm of bench.py times whole plans: spawning and joining a set of std::threads per stage
// cost more than a stage at 128 threads).  parallel_for hands out small index blocks from an atomic counter, so threads
// that finish early (contacts make rollouts unequal) take more blocks.
class Pool {
  public:
    static Pool& get() { static Pool p; return p; }
    void run(int n, int nthreads, int grain, const std::function<void(int, int)>& f) {
        std::unique_lock<std::mutex> user(user_mu_);          // one parallel region at a time
        ensure(nthreads - 1);
        {
            std::lock_guard<std::mutex> lk(mu_);
            job_ = &f; n_ = n; grain_ = grain; next_.store(0); active_ = nthreads - 1; pending_ = nthreads - 1; ++epoch_;
        }
        cv_.notify_all();
        work();
        std::unique_lock<std::mutex> lk(mu_);
        done_cv_.wait(lk, [&] { return pending_ == 0; });
        job_ = nullptr;
    }
  private:
    Pool() = default;
    ~Pool() {
        { std::lock_guard<std::mutex> lk(mu_); stop_ = true; ++epoch_; }
        cv_.notify_all();
        for (auto& t : th_) t.join();
    }
    void ensure(int workers) {
        while ((int)th_.size() < workers) {
            const int id = (int)th_.size();
            th_.emplace_back([this, id] {
                unsigned long long seen = 0;
                for (;;) {
                    std::unique_lock<std::mutex> lk(mu_);
                    cv_.wait(lk, [&] { return stop_ || epoch_ != seen; });
                    if (stop_) return;
                    seen = epoch_;
                    const bool mine = id < active_;
                    lk.unlock();
                    if (mine) {
                        work();
                        std::lock_guard<std::mutex> lk2(mu_);
                        if (--pending_ == 0) done_cv_.notify_all();
                    }
                }
            });
        }
    }
    void work() {
        for (;;) {
            const int a = next_.fetch_add(grain_);
            if (a >= n_) break;
            (*job_)(a, std::min(n_, a + grain_));
        }
    }
    std::mutex mu_, user_mu_;
    std::condition_variable cv_, done_cv_;
    std::vector<std::thread> th_;
    const std::function<void(int, int)>* job_ = nullptr;
    std::atomic<int> next_{0};
    int n_ = 0, grain_ = 1, active_ = 0, pending_ = 0;
    unsigned long long epoch_ = 0;
    bool stop_ = false;
};

template <class F>
void parallel_for(int n, int nthreads, F f) {
    if (nthreads <= 1 || n < 2 * nthreads) { f(0, n); return; }
    // blocks of whole cache lines of the k-innermost arrays (16 floats): neighbouring threads never write the same line
    const int grain = std::max(16, (n / (nthreads * 4)) & ~15);
    Pool::get().run(n, nthreads, grain, std::function<void(int, int)>(f));
}

// ------------------------------------------------------------------------------------------
// dense spatial algebra, motion vectors [w; v], force vectors [n; f]
// ------------------------------------------------------------------------------------------
template <class S> struct M3 { S a[3][3]; };
template <class S> struct V6 { S a[6]; };
template <class S> struct M6 { S a[6][6]; };

template <class S> void cross3(const S* a, const S* b, S* o) {
    o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}

// Pluecker motion transform parent->child coords for a child frame at (R: child axes as columns
// in parent coords, p: child origin in parent coords):  X = [E 0; -E p^x  E],  E = R^T.
template <class S> M6<S> plucker(const M3<S>& R, const S* p) {
    M6<S> X; std::memset(&X, 0, sizeof(X));
    S E[3][3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) E[i][j] = R.a[j][i];
    S px[3][3] = {{0, -p[2], p[1]}, {p[2], 0, -p[0]}, {-p[1], p[0], 0}};
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
        X.a[i][j] = E[i][j]; X.a[i + 3][j + 3] = E[i][j];
        S s = 0; for (int k = 0; k < 3; ++k) s += E[i][k] * px[k][j];
        X.a[i + 3][j] = -s;
    }
    return X;
}
template <class S> V6<S> mulXv(const M6<S>& X, const V6<S>& v) {
    V6<S> o; for (int i = 0; i < 6; ++i) { S s = 0; for (int j = 0; j < 6; ++j) s += X.a[i][j] * v.a[j]; o.a[i] = s; } return o;
}
template <class S> V6<S> mulXTf(const M6<S>& X, const V6<S>& f) {
    V6<S> o; for (int i = 0; i < 6; ++i) { S s = 0; for (int j = 0; j < 6; ++j) s += X.a[j][i] * f.a[j]; o.a[i] = s; } return o;
}
// crm(v) m  (motion cross motion)
template <class S> V6<S> crm(const V6<S>& v, const V6<S>& m) {
    V6<S> o; S t[3];
    cross3(&v.a[0], &m.a[0], &o.a[0]);
    cross3(&v.a[0], &m.a[3], &o.a[3]); cross3(&v.a[3], &m.a[0], t);
    for (int i = 0; i < 3; ++i) o.a[3 + i] += t[i];
    return o;
}
// crf(v) f  (motion cross force)
template <class S> V6<S> crf(const V6<S>& v, const V6<S>& f) {
    V6<S> o; S t[3];
    cross3(&v.a[0], &f.a[0], &o.a[0]); cross3(&v.a[3], &f.a[3], t);
    for (int i = 0; i < 3; ++i) o.a[i] += t[i];
    cross3(&v.a[0], &f.a[3], &o.a[3]);
    return o;
}
template <class S> M6<S> spatial_inertia(S m, const float* h, const float* I6) {
    // [[I_o, h^x], [-(h^x), m 1]] with h = m*com, I_o about the body origin
    M6<S> I; std::memset(&I, 0, sizeof(I));
    S Io[3][3] = {{(S)I6[0], (S)I6[3], (S)I6[4]}, {(S)I6[3], (S)I6[1], (S)I6[5]}, {(S)I6[4], (S)I6[5], (S)I6[2]}};
    S hx[3][3] = {{0, -(S)h[2], (S)h[1]}, {(S)h[2], 0, -(S)h[0]}, {-(S)h[1], (S)h[0], 0}};
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
        I.a[i][j] = Io[i][j]; I.a[i][j + 3] = hx[i][j]; I.a[i + 3][j] = -hx[i][j];
    }
    for (int i = 0; i < 3; ++i) I.a[i + 3][i + 3] = m;
    return I;
}
template <class S> void quat_mul(const S* a, const S* b, S* o) {  // xyzw
    S x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    S y = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
    S z = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
    S w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    o[0] = x; o[1] = y; o[2] = z; o[3] = w;
}
template <class S> M3<S> quat_to_R(const S* q) {
    S x = q[0], y = q[1], z = q[2], w = q[3];
    M3<S> R = {{{1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)},
                {2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)},
                {2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)}}};
    return R;
}

// ------------------------------------------------------------------------------------------
// articulated-body forward dynamics of one substep
// ------------------------------------------------------------------------------------------
template <class S>
struct Articulation {
    const MppibModel* m;
    int nb;
    M3<S> Rl[MPPIB_MAX_BODIES];   // body->parent rotation at the current q
    S pl[MPPIB_MAX_BODIES][3];
    M6<S> X[MPPIB_MAX_BODIES];
    V6<S> v[MPPIB_MAX_BODIES], c[MPPIB_MAX_BODIES], pbias[MPPIB_MAX_BODIES];
    V6<S> a0;                      // base acceleration (= -gravity in base coords)

    void kinematics(const S* q, const S* qd) {
        for (int i = 0; i < nb; ++i) {
            M3<S> Rt; for (int r = 0; r < 3; ++r) for (int cc = 0; cc < 3; ++cc) Rt.a[r][cc] = (S)m->tree_R[i][3 * r + cc];
            if (m->jtype[i] == MPPIB_JOINT_REVOLUTE) {
                S cq = std::cos(q[i]), sq = std::sin(q[i]);
                for (int r = 0; r < 3; ++r) {   // Rt * Rz(q)
                    Rl[i].a[r][0] = Rt.a[r][0] * cq + Rt.a[r][1] * sq;
                    Rl[i].a[r][1] = -Rt.a[r][0] * sq + Rt.a[r][1] * cq;
                    Rl[i].a[r][2] = Rt.a[r][2];
                }
                for (int r = 0; r < 3; ++r) pl[i][r] = (S)m->tree_p[i][r];
            } else {
                Rl[i] = Rt;
                for (int r = 0; r < 3; ++r) pl[i][r] = (S)m->tree_p[i][r] + Rt.a[r][2] * q[i];
            }
            X[i] = plucker(Rl[i], pl[i]);
            V6<S> vp; std::memset(&vp, 0, sizeof(vp));
            if (m->parent[i] >= 0) vp = v[m->parent[i]];
            V6<S> vj; std::memset(&vj, 0, sizeof(vj));
            vj.a[m->jtype[i] == MPPIB_JOINT_REVOLUTE ? 2 : 5] = qd[i];
            v[i] = mulXv(X[i], vp);
            for (int k = 0; k < 6; ++k) v[i].a[k] += vj.a[k];
            c[i] = crm(v[i], vj);
        }
    }

    // world pose / velocity of every body from the last kinematics() call
    M3<S> Rw[MPPIB_MAX_BODIES]; S pw[MPPIB_MAX_BODIES][3], ww[MPPIB_MAX_BODIES][3], vw[MPPIB_MAX_BODIES][3];
    void world_frames(const M3<S>& Rb, const S* pb) {
        for (int i = 0; i < nb; ++i) {
            const M3<S>& Rp = m->parent[i] >= 0 ? Rw[m->parent[i]] : Rb;
            const S* pp = m->parent[i] >= 0 ? pw[m->parent[i]] : pb;
            for (int r = 0; r < 3; ++r) {
                S s = 0; for (int j = 0; j < 3; ++j) s += Rp.a[r][j] * pl[i][j];
                pw[i][r] = pp[r] + s;
                for (int cc = 0; cc < 3; ++cc) { S s2 = 0; for (int j = 0; j < 3; ++j) s2 += Rp.a[r][j] * Rl[i].a[j][cc]; Rw[i].a[r][cc] = s2; }
            }
            for (int r = 0; r < 3; ++r) {   // angular velocity and velocity of the body origin, world coordinates
                S a = 0, b = 0; for (int j = 0; j < 3; ++j) { a += Rw[i].a[r][j] * v[i].a[j]; b += Rw[i].a[r][j] * v[i].a[3 + j]; }
                ww[i][r] = a; vw[i][r] = b;
            }
        }
    }

    // one ABA solve; tau = explicit joint force, dimp = implicit diagonal added to D (h*(kd+damping)+armature)
    // fext[i]: external wrench on body i in BODY coordinates about the body origin (contacts), may be null
    S D[MPPIB_MAX_BODIES];   // joint-space articulated diagonal (incl. the implicit drive term) of the last solve
    void aba(const S* tau, const S* dimp, S* qdd, const V6<S>* fext = nullptr) {
        M6<S> IA[MPPIB_MAX_BODIES]; V6<S> pA[MPPIB_MAX_BODIES];
        V6<S> U[MPPIB_MAX_BODIES]; S u[MPPIB_MAX_BODIES];
        for (int i = 0; i < nb; ++i) {
            IA[i] = spatial_inertia<S>((S)m->mass[i], m->mcom[i], m->inertia[i]);
            V6<S> Iv = mulXv(IA[i], v[i]);
            pA[i] = crf(v[i], Iv);
            if (fext) for (int k = 0; k < 6; ++k) pA[i].a[k] -= fext[i].a[k];
        }
        for (int i = nb - 1; i >= 0; --i) {
            int s = m->jtype[i] == MPPIB_JOINT_REVOLUTE ? 2 : 5;
            for (int k = 0; k < 6; ++k) U[i].a[k] = IA[i].a[k][s];
            D[i] = U[i].a[s] + dimp[i];
            u[i] = tau[i] - pA[i].a[s];
            int p = m->parent[i];
            if (p >= 0) {
                M6<S> Ia; V6<S> pa;
                for (int r = 0; r < 6; ++r) for (int cc = 0; cc < 6; ++cc) Ia.a[r][cc] = IA[i].a[r][cc] - U[i].a[r] * U[i].a[cc] / D[i];
                V6<S> Iac = mulXv(Ia, c[i]);
                for (int k = 0; k < 6; ++k) pa.a[k] = pA[i].a[k] + Iac.a[k] + U[i].a[k] * (u[i] / D[i]);
                // IA[p] += X^T Ia X ; pA[p] += X^T pa
                M6<S> T;
                for (int r = 0; r < 6; ++r) for (int cc = 0; cc < 6; ++cc) { S sum = 0; for (int k = 0; k < 6; ++k) sum += Ia.a[r][k] * X[i].a[k][cc]; T.a[r][cc] = sum; }
                for (int r = 0; r < 6; ++r) for (int cc = 0; cc < 6; ++cc) { S sum = 0; for (int k = 0; k < 6; ++k) sum += X[i].a[k][r] * T.a[k][cc]; IA[p].a[r][cc] += sum; }
                V6<S> pp = mulXTf(X[i], pa);
                for (int k = 0; k < 6; ++k) pA[p].a[k] += pp.a[k];
            }
        }
        V6<S> acc[MPPIB_MAX_BODIES];
        for (int i = 0; i < nb; ++i) {
            int s = m->jtype[i] == MPPIB_JOINT_REVOLUTE ? 2 : 5;
            V6<S> ap = m->parent[i] >= 0 ? acc[m->parent[i]] : a0;
            V6<S> a = mulXv(X[i], ap);
            for (int k = 0; k < 6; ++k) a.a[k] += c[i].a[k];
            S dot = 0; for (int k = 0; k < 6; ++k) dot += U[i].a[k] * a.a[k];
            qdd[i] = (u[i] - dot) / D[i];
            a.a[s] += qdd[i];
            acc[i] = a;
        }
    }
};

// ------------------------------------------------------------------------------------------
// free rigid bodies + contacts (replaces PhysX rigid bodies / contact solve on this path; SURVEY 8(a) G1/G2).
// Spec (DESIGN.md section 2): boxes only; contact points = the 26 surface sample points of one box that lie
// inside the other box (both directions) or below the ground plane; normal = face of least penetration;
// penalty spring-damper (contact_kp, contact_kd) integrated IMPLICITLY as a soft constraint
//     d_lambda = (-v_n + beta d / h - gamma lambda) / (k_n + gamma),  gamma = 1/(h (h kp + kd)),  beta = h kp / (h kp + kd)
// solved by `contact_iters` Gauss-Seidel sweeps with box friction |lambda_t| <= mu lambda_n on the PREDICTED velocities
// (after gravity and the drive have acted for this substep).  Articulation links take part with a DIAGONAL joint-space
// compliance: an impulse P at point x of body b changes the velocity of joint j (ancestors of b) by J_j(x).P / D_j, D_j the
// articulated joint-space diagonal of the ABA solve (inertia + armature + h (k_d + b)); the implicit drive dominates it on
// this path (h k_d = 15..60 kg-equivalent), so the off-diagonal coupling that is dropped is small.
// ------------------------------------------------------------------------------------------
enum { REF_STATIC = -1, REF_FREE0 = 64 };

template <class S> struct FreeBody { S x[3], q[4], v[3], w[3], mass, half[3], Iinv[3]; M3<S> R, IinvW; };
template <class S> struct ShapeW { M3<S> R; S c[3], half[3], mu, rad; int ref, slot, kind, type; };
template <class S> struct Contact { int refA, refB, slotA, slotB, penalty; S p[3], n[3], d, mu, ln, lt1, lt2, t1[3], t2[3], kn, kt1, kt2; };

template <class S> void mat_vec(const M3<S>& R, const S* v, S* o) { for (int r = 0; r < 3; ++r) o[r] = R.a[r][0] * v[0] + R.a[r][1] * v[1] + R.a[r][2] * v[2]; }
template <class S> void matT_vec(const M3<S>& R, const S* v, S* o) { for (int r = 0; r < 3; ++r) o[r] = R.a[0][r] * v[0] + R.a[1][r] * v[1] + R.a[2][r] * v[2]; }

// per-rollout randomisation (isaacgym_utils.py:29-40 size noise, isaacgym_wrapper.py:450-475 mass / friction noise),
// made reproducible: Philox counter (global sample, actor, 0x5EED, draw), key (rand_seed, "MPPI")
inline void actor_noise(const MppibParams* p, uint32_t kg, int actor, float* nsize, float* umass, float* ufric) {
    U4 r0 = philox4x32_10({kg, (uint32_t)actor, 0x5EEDu, 0u}, p->rand_seed, 0x4D505049u);
    U4 r1 = philox4x32_10({kg, (uint32_t)actor, 0x5EEDu, 1u}, p->rand_seed, 0x4D505049u);
    float dummy;
    box_muller(r0.x, r0.y, &nsize[0], &nsize[1]);
    box_muller(r0.z, r0.w, &nsize[2], &dummy);
    *umass = 2.0f * u01(r1.x) - 1.0f;
    *ufric = 2.0f * u01(r1.y) - 1.0f;
}

template <class S>
struct ContactWorld {
    const MppibModel* m; const MppibParams* p;
    FreeBody<S> fb[MPPIB_MAX_FREE];
    S shalf[MPPIB_MAX_SHAPES][3], smu[MPPIB_MAX_SHAPES];     // per-rollout shape parameters
    ShapeW<S> sh[MPPIB_MAX_SHAPES];
    Contact<S> ct[MPPIB_MAX_CONTACTS]; int nc;
    S net[MPPIB_MAX_SLOTS][3];                                // net contact force per slot (last substep)
    S dqv[MPPIB_MAX_BODIES], Dj[MPPIB_MAX_BODIES];            // virtual joint-velocity change inside the solve, joint compliance denominators

    void init_params(uint32_t kg) {
        for (int s = 0; s < m->nshapes; ++s) {
            for (int r = 0; r < 3; ++r) shalf[s][r] = (S)m->shape_half[s][r];
            smu[s] = (S)m->shape_friction[s];
            if (m->shape_actor[s] >= 0) {
                float ns[3], um, uf; actor_noise(p, kg, m->shape_actor[s], ns, &um, &uf);
                for (int r = 0; r < 3; ++r) shalf[s][r] += (S)0.5 * (S)m->shape_size_sigma[s][r] * (S)ns[r];
                smu[s] *= (S)1 + (S)m->shape_fric_pct[s] * (S)uf;
            }
        }
        for (int f = 0; f < m->nfree; ++f) {
            float ns[3], um, uf; actor_noise(p, kg, m->free_actor[f], ns, &um, &uf);
            fb[f].mass = (S)m->free_mass[f] * ((S)1 + (S)m->free_mass_pct[f] * (S)um);
            // size noise of the body = size noise of its (first) shape
            S sg[3] = {0, 0, 0};
            for (int s = 0; s < m->nshapes; ++s) if (m->shape_owner_kind[s] == MPPIB_OWNER_FREE && m->shape_owner[s] == f) { for (int r = 0; r < 3; ++r) sg[r] = (S)m->shape_size_sigma[s][r]; break; }
            for (int r = 0; r < 3; ++r) fb[f].half[r] = (S)m->free_half[f][r] + (S)0.5 * sg[r] * (S)ns[r];
            const S hx = fb[f].half[0], hy = fb[f].half[1], hz = fb[f].half[2], m3 = fb[f].mass / (S)3;
            fb[f].Iinv[0] = (S)1 / (m3 * (hy * hy + hz * hz)); fb[f].Iinv[1] = (S)1 / (m3 * (hx * hx + hz * hz)); fb[f].Iinv[2] = (S)1 / (m3 * (hx * hx + hy * hy));
        }
    }
    void refresh_free(int f) {
        fb[f].R = quat_to_R(fb[f].q);
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { S s = 0; for (int j = 0; j < 3; ++j) s += fb[f].R.a[r][j] * fb[f].Iinv[j] * fb[f].R.a[c][j]; fb[f].IinvW.a[r][c] = s; }
    }
    // velocity of point pt of body b per unit velocity of joint j (world): a_j x (pt - o_j) (revolute) or a_j (prismatic)
    void joint_jac(const Articulation<S>& art, int j, const S* pt, S* J) const {
        S a[3] = {art.Rw[j].a[0][2], art.Rw[j].a[1][2], art.Rw[j].a[2][2]};
        if (m->jtype[j] == MPPIB_JOINT_REVOLUTE) { S r[3] = {pt[0] - art.pw[j][0], pt[1] - art.pw[j][1], pt[2] - art.pw[j][2]}; cross3(a, r, J); }
        else { J[0] = a[0]; J[1] = a[1]; J[2] = a[2]; }
    }
    void point_velocity(int ref, const S* pt, const Articulation<S>& art, S* o) const {
        if (ref == REF_STATIC) { o[0] = o[1] = o[2] = 0; return; }
        S r[3], wxr[3];
        if (ref >= REF_FREE0) { const FreeBody<S>& b = fb[ref - REF_FREE0]; for (int i = 0; i < 3; ++i) r[i] = pt[i] - b.x[i]; cross3(b.w, r, wxr); for (int i = 0; i < 3; ++i) o[i] = b.v[i] + wxr[i]; }
        else {
            for (int i = 0; i < 3; ++i) r[i] = pt[i] - art.pw[ref][i];
            cross3(art.ww[ref], r, wxr);
            for (int i = 0; i < 3; ++i) o[i] = art.vw[ref][i] + wxr[i];
            for (int j = ref; j >= 0; j = m->parent[j]) { S J[3]; joint_jac(art, j, pt, J); for (int i = 0; i < 3; ++i) o[i] += J[i] * dqv[j]; }
        }
    }
    // effective inverse mass of the free bodies of a contact along direction dir at point pt
    S inv_mass(const Contact<S>& c, const S* dir, const Articulation<S>& art) const {
        S k = 0;
        const int refs[2] = {c.refA, c.refB};
        for (int e = 0; e < 2; ++e) if (refs[e] >= 0 && refs[e] < REF_FREE0) {
            for (int j = refs[e]; j >= 0; j = m->parent[j]) { S J[3]; joint_jac(art, j, c.p, J); const S jd = J[0] * dir[0] + J[1] * dir[1] + J[2] * dir[2]; k += jd * jd / Dj[j]; }
        } else if (refs[e] >= REF_FREE0) {
            const FreeBody<S>& b = fb[refs[e] - REF_FREE0];
            S r[3], rxn[3], t[3], u[3];
            for (int i = 0; i < 3; ++i) r[i] = c.p[i] - b.x[i];
            cross3(r, dir, rxn); mat_vec(b.IinvW, rxn, t); cross3(t, r, u);
            k += (S)1 / b.mass + u[0] * dir[0] + u[1] * dir[1] + u[2] * dir[2];
        }
        return k;
    }
    void apply_impulse(const Contact<S>& c, const S* dir, S mag, const Articulation<S>& art) {
        const int refs[2] = {c.refA, c.refB};
        for (int e = 0; e < 2; ++e) if (refs[e] >= 0 && refs[e] < REF_FREE0) {
            const S sgn = e == 0 ? mag : -mag;
            for (int j = refs[e]; j >= 0; j = m->parent[j]) { S J[3]; joint_jac(art, j, c.p, J); dqv[j] += sgn * (J[0] * dir[0] + J[1] * dir[1] + J[2] * dir[2]) / Dj[j]; }
        } else if (refs[e] >= REF_FREE0) {
            FreeBody<S>& b = fb[refs[e] - REF_FREE0];
            const S sgn = e == 0 ? mag : -mag;
            S r[3], rxd[3], dw[3];
            for (int i = 0; i < 3; ++i) { r[i] = c.p[i] - b.x[i]; b.v[i] += sgn * dir[i] / b.mass; }
            cross3(r, dir, rxd); mat_vec(b.IinvW, rxd, dw);
            for (int i = 0; i < 3; ++i) b.w[i] += sgn * dw[i];
        }
    }
    void add_contact(int refA, int refB, int slotA, int slotB, const S* pt, const S* n, S d, S mu, int penalty) {
        if (nc >= m->max_contacts) return;
        Contact<S>& c = ct[nc++];
        c.refA = refA; c.refB = refB; c.slotA = slotA; c.slotB = slotB; c.penalty = penalty; c.d = d; c.mu = mu; c.ln = c.lt1 = c.lt2 = 0;
        for (int i = 0; i < 3; ++i) { c.p[i] = pt[i]; c.n[i] = n[i]; }
        S e[3] = {0, 0, 0}; if (std::fabs(n[0]) < (S)0.9) e[0] = 1; else e[1] = 1;
        cross3(n, e, c.t1); S l = std::sqrt(c.t1[0] * c.t1[0] + c.t1[1] * c.t1[1] + c.t1[2] * c.t1[2]);
        for (int i = 0; i < 3; ++i) c.t1[i] /= l;
        cross3(n, c.t1, c.t2);
    }
    // sample points of box a that are inside box b -> contacts; `flip`: a is the B side of the pair
    void points_in_box(const ShapeW<S>& a, const ShapeW<S>& b, bool flip, int penalty) {
        const S mu = (S)0.5 * (a.mu + b.mu);
        // candidate normal axes: slabs of b that the CENTRE of a lies outside of (a thin box must not push sideways hits
        // up or down); if the centre is inside b, all three axes compete
        S crel[3], cl[3]; for (int i = 0; i < 3; ++i) crel[i] = a.c[i] - b.c[i];
        matT_vec(b.R, crel, cl);
        bool cand[3]; int ncand = 0;
        for (int i = 0; i < 3; ++i) { cand[i] = std::fabs(cl[i]) > b.half[i]; ncand += cand[i]; }
        if (ncand == 0) cand[0] = cand[1] = cand[2] = true;
        for (int ix = -1; ix <= 1; ++ix) for (int iy = -1; iy <= 1; ++iy) for (int iz = -1; iz <= 1; ++iz) {
            if (ix == 0 && iy == 0 && iz == 0) continue;
            S loc[3] = {ix * a.half[0], iy * a.half[1], iz * a.half[2]}, pt[3], rel[3], x[3];
            mat_vec(a.R, loc, pt); for (int i = 0; i < 3; ++i) { pt[i] += a.c[i]; rel[i] = pt[i] - b.c[i]; }
            matT_vec(b.R, rel, x);
            S pen[3]; bool inside = true;
            const S mg = (S)m->contact_margin;                       // speculative margin
            for (int i = 0; i < 3; ++i) { pen[i] = b.half[i] - std::fabs(x[i]); if (!(pen[i] + mg > 0)) inside = false; }
            if (!inside) continue;
            int ax = -1;
            for (int i = 0; i < 3; ++i) if (cand[i] && (ax < 0 || pen[i] < pen[ax])) ax = i;
            S nl[3] = {0, 0, 0}; nl[ax] = x[ax] >= 0 ? (S)1 : (S)-1;
            S n[3]; mat_vec(b.R, nl, n);      // outward normal of b: pushes a out of b
            if (!flip) add_contact(a.ref, b.ref, a.slot, b.slot, pt, n, pen[ax], mu, penalty);
            else { S nn[3] = {-n[0], -n[1], -n[2]}; add_contact(b.ref, a.ref, b.slot, a.slot, pt, nn, pen[ax], mu, penalty); }
        }
    }
    void shapes_world(const Articulation<S>& art, const M3<S>& Rb, const S* pb, const float* root0) {
        for (int s = 0; s < m->nshapes; ++s) {
            ShapeW<S>& w = sh[s];
            S ql[4] = {(S)m->shape_quat[s][0], (S)m->shape_quat[s][1], (S)m->shape_quat[s][2], (S)m->shape_quat[s][3]};
            S pl[3] = {(S)m->shape_pos[s][0], (S)m->shape_pos[s][1], (S)m->shape_pos[s][2]};
            M3<S> Rl = quat_to_R(ql), Ro; S po[3];
            w.kind = m->shape_owner_kind[s]; w.slot = m->shape_slot[s];
            if (w.kind == MPPIB_OWNER_STATIC) {
                const float* rs = root0 + 13 * m->shape_actor[s];
                S q[4] = {(S)rs[3], (S)rs[4], (S)rs[5], (S)rs[6]}; Ro = quat_to_R(q); for (int i = 0; i < 3; ++i) po[i] = (S)rs[i];
                w.ref = REF_STATIC;
            } else if (w.kind == MPPIB_OWNER_LINK) {
                const int b = m->shape_owner[s];
                if (b >= 0) { Ro = art.Rw[b]; for (int i = 0; i < 3; ++i) po[i] = art.pw[b][i]; w.ref = b; }
                else { Ro = Rb; for (int i = 0; i < 3; ++i) po[i] = pb[i]; w.ref = REF_STATIC; }
            } else {
                const FreeBody<S>& b = fb[m->shape_owner[s]]; Ro = b.R; for (int i = 0; i < 3; ++i) po[i] = b.x[i];
                w.ref = REF_FREE0 + m->shape_owner[s];
            }
            for (int r = 0; r < 3; ++r) {
                S acc = 0; for (int j = 0; j < 3; ++j) acc += Ro.a[r][j] * pl[j]; w.c[r] = po[r] + acc;
                for (int c = 0; c < 3; ++c) { S a2 = 0; for (int j = 0; j < 3; ++j) a2 += Ro.a[r][j] * Rl.a[j][c]; w.R.a[r][c] = a2; }
                w.half[r] = shalf[s][r];
            }
            w.mu = smu[s];
            w.type = m->shape_type[s];
            // bounding radius; a sphere shape (isaacgym_utils.py:42-52: gym.create_sphere(radius = size[0])) keeps its radius in half[0]
            w.rad = w.type == MPPIB_SHAPE_SPHERE ? w.half[0] : std::sqrt(w.half[0] * w.half[0] + w.half[1] * w.half[1] + w.half[2] * w.half[2]);
        }
    }
    // ONE contact of a sphere against a box (closest point of the box to the centre; centre inside the box: least-penetration face)
    // or against another sphere.  The normal of a contact pushes side A out of side B.
    void sphere_contact(const ShapeW<S>& a, const ShapeW<S>& b, int penalty) {
        const S mu = (S)0.5 * (a.mu + b.mu), mg = (S)m->contact_margin;
        if (a.type == MPPIB_SHAPE_SPHERE && b.type == MPPIB_SHAPE_SPHERE) {
            S d[3], d2 = 0; for (int i = 0; i < 3; ++i) { d[i] = a.c[i] - b.c[i]; d2 += d[i] * d[i]; }
            const S dist = std::sqrt(d2), rs = a.half[0] + b.half[0];
            if (!(dist < rs + mg) || !(dist > 0)) return;
            S n[3], pt[3]; for (int i = 0; i < 3; ++i) { n[i] = d[i] / dist; pt[i] = b.c[i] + n[i] * b.half[0]; }
            add_contact(a.ref, b.ref, a.slot, b.slot, pt, n, rs - dist, mu, penalty);
            return;
        }
        const bool sphere_is_a = a.type == MPPIB_SHAPE_SPHERE;
        const ShapeW<S>& sp = sphere_is_a ? a : b;
        const ShapeW<S>& bx = sphere_is_a ? b : a;
        const S r = sp.half[0];
        S rel[3], x[3], q[3], d2 = 0;
        for (int i = 0; i < 3; ++i) rel[i] = sp.c[i] - bx.c[i];
        matT_vec(bx.R, rel, x);
        for (int i = 0; i < 3; ++i) { q[i] = std::min(std::max(x[i], -bx.half[i]), bx.half[i]); d2 += (x[i] - q[i]) * (x[i] - q[i]); }
        S nl[3] = {0, 0, 0}, pen;
        if (d2 > 0) {                                  // centre outside the box
            const S dist = std::sqrt(d2);
            if (!(dist < r + mg)) return;
            for (int i = 0; i < 3; ++i) nl[i] = (x[i] - q[i]) / dist;
            pen = r - dist;
        } else {                                       // centre inside: out through the nearest face
            int ax = 0; S best = bx.half[0] - std::fabs(x[0]);
            for (int i = 1; i < 3; ++i) { const S pi = bx.half[i] - std::fabs(x[i]); if (pi < best) { best = pi; ax = i; } }
            nl[ax] = x[ax] >= 0 ? (S)1 : (S)-1;
            q[ax] = nl[ax] * bx.half[ax];
            pen = best + r;
        }
        S n[3], pl[3], pt[3];
        mat_vec(bx.R, nl, n);                          // from the box towards the sphere
        mat_vec(bx.R, q, pl); for (int i = 0; i < 3; ++i) pt[i] = bx.c[i] + pl[i];
        if (sphere_is_a) add_contact(sp.ref, bx.ref, sp.slot, bx.slot, pt, n, pen, mu, penalty);
        else { S nn[3] = {-n[0], -n[1], -n[2]}; add_contact(bx.ref, sp.ref, bx.slot, sp.slot, pt, nn, pen, mu, penalty); }
    }
    // contacts of the ordered pair (a, b): boxes by sample points in both directions, anything with a sphere analytically
    void pair_contacts(const ShapeW<S>& a, const ShapeW<S>& b, int penalty) {
        if (a.type == MPPIB_SHAPE_SPHERE || b.type == MPPIB_SHAPE_SPHERE) { sphere_contact(a, b, penalty); return; }
        points_in_box(a, b, false, penalty);
        points_in_box(b, a, true, penalty);
    }
    // broad phase: bounding spheres, then the 6 face axes of the two boxes (conservative: never rejects boxes closer than the margin)
    bool near(const ShapeW<S>& a, const ShapeW<S>& b) const {
        S d[3], d2 = 0; for (int i = 0; i < 3; ++i) { d[i] = a.c[i] - b.c[i]; d2 += d[i] * d[i]; }
        const S mg = (S)m->contact_margin;
        const bool sph = a.type == MPPIB_SHAPE_SPHERE || b.type == MPPIB_SHAPE_SPHERE;
        const S r = a.rad + b.rad + (sph ? mg : (S)0); if (d2 > r * r) return false;      // (a sphere's bound is exact: the margin counts)
        if (sph) return true;                                                            // the narrow phase is exact and cheap
        S C[3][3];                                   // C = Rb^T Ra
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { S v = 0; for (int k = 0; k < 3; ++k) v += b.R.a[k][i] * a.R.a[k][j]; C[i][j] = v; }
        S tb[3], ta[3]; matT_vec(b.R, d, tb); matT_vec(a.R, d, ta);
        for (int i = 0; i < 3; ++i) {
            const S ra = std::fabs(C[i][0]) * a.half[0] + std::fabs(C[i][1]) * a.half[1] + std::fabs(C[i][2]) * a.half[2];
            if (std::fabs(tb[i]) > b.half[i] + ra + mg) return false;
            const S rb = std::fabs(C[0][i]) * b.half[0] + std::fabs(C[1][i]) * b.half[1] + std::fabs(C[2][i]) * b.half[2];
            if (std::fabs(ta[i]) > a.half[i] + rb + mg) return false;
        }
        return true;
    }
    void detect() {
        nc = 0;
        const int ns = m->nshapes;
        for (int a = 0; a < ns; ++a) {
            if (sh[a].kind != MPPIB_OWNER_FREE) continue;
            if (m->ground_plane) {
                // at most the 4 lowest corners (ties by corner index) are ground points: a box resting flat, on an edge or on a corner
                // is carried by those, the higher ones only have a gap (a speculative row with no impulse) and would use up the cap
                // when the margin 1.5 g h^2 exceeds the box's height (h = 0.1 s: 14.7 cm)
                const S mu = (S)0.5 * (sh[a].mu + (S)m->ground_friction);
                S pts[8][3];
                for (int c = 0; c < 8; ++c) {
                    const int ix = (c >> 2) * 2 - 1, iy = ((c >> 1) & 1) * 2 - 1, iz = (c & 1) * 2 - 1;
                    S loc[3] = {ix * sh[a].half[0], iy * sh[a].half[1], iz * sh[a].half[2]};
                    mat_vec(sh[a].R, loc, pts[c]); for (int i = 0; i < 3; ++i) pts[c][i] += sh[a].c[i];
                }
                for (int c = 0; c < 8; ++c) {
                    int rank = 0;
                    for (int o = 0; o < 8; ++o) rank += pts[o][2] < pts[c][2] || (pts[o][2] == pts[c][2] && o < c);
                    if (rank < 4 && pts[c][2] < (S)m->ground_margin) { S n[3] = {0, 0, 1}; add_contact(sh[a].ref, REF_STATIC, sh[a].slot, -1, pts[c], n, -pts[c][2], mu, 0); }
                }
            }
            for (int b = 0; b < ns; ++b) {
                if (b == a || sh[b].ref == sh[a].ref) continue;
                if (sh[b].kind == MPPIB_OWNER_FREE && b < a) continue;       // free-free pairs once
                if (!near(sh[a], sh[b])) continue;
                pair_contacts(sh[a], sh[b], 0);
            }
        }
        for (int a = 0; a < ns; ++a) {                                        // articulation link vs static box
            if (sh[a].kind != MPPIB_OWNER_LINK || sh[a].ref == REF_STATIC) continue;
            for (int b = 0; b < ns; ++b) {
                if (sh[b].kind != MPPIB_OWNER_STATIC || !near(sh[a], sh[b])) continue;
                pair_contacts(sh[a], sh[b], 1);
            }
        }
    }
    // A contact row whose effective inverse mass is below K_ROW_MIN [1/kg] is dropped: e.g. a ground-parallel base pressed on from
    // above, or the vertical friction direction of a wall contact of a planar robot.  (An exact `> 0` would make the row depend on
    // whether an implementation's rotation arithmetic yields an exact 0 or 1e-9 for such a direction.)
    static constexpr double K_ROW_MIN = 1e-9;
    void solve(const Articulation<S>& art, S h) {
        const S kp = (S)m->contact_kp, kd = (S)m->contact_kd;
        const S gamma = (S)1 / (h * (h * kp + kd)), beta = h * kp / (h * kp + kd);
        for (int j = 0; j < m->nb; ++j) { dqv[j] = 0; Dj[j] = std::max((S)1e-6, art.D[j]); }
        // effective inverse masses along the contact frame are constant during the sweeps (poses are frozen within a substep)
        for (int i = 0; i < nc; ++i) { Contact<S>& c = ct[i]; c.kn = inv_mass(c, c.n, art); c.kt1 = inv_mass(c, c.t1, art); c.kt2 = inv_mass(c, c.t2, art); }
        for (int it = 0; it < m->contact_iters; ++it) for (int i = 0; i < nc; ++i) {
            Contact<S>& c = ct[i];
            if (!(c.kn > (S)K_ROW_MIN)) continue;                     // the bodies cannot move along the normal: no contact row at all
            // one visit = normal row + two friction rows solved from the SAME relative velocity, then one impulse application
            S va[3], vb[3], vr[3];
            point_velocity(c.refA, c.p, art, va); point_velocity(c.refB, c.p, art, vb);
            for (int r = 0; r < 3; ++r) vr[r] = va[r] - vb[r];
            const S vn = vr[0] * c.n[0] + vr[1] * c.n[1] + vr[2] * c.n[2];
            const S vt1 = vr[0] * c.t1[0] + vr[1] * c.t1[1] + vr[2] * c.t1[2], vt2 = vr[0] * c.t2[0] + vr[1] * c.t2[1] + vr[2] * c.t2[2];
            // penetration: push out (at most max_depen m/s, so squeezed bodies are not shot out); gap: may close at most gap / h
            const S bias = c.d > 0 ? std::min(beta * c.d / h, (S)m->max_depen) : c.d / h;
            const S ln_new = std::max((S)0, c.ln + (-vn + bias - gamma * c.ln) / (c.kn + gamma));
            const S lim = c.mu * ln_new;
            const S lt1_new = c.kt1 > (S)K_ROW_MIN ? std::min(std::max(c.lt1 - vt1 / c.kt1, -lim), lim) : c.lt1;
            const S lt2_new = c.kt2 > (S)K_ROW_MIN ? std::min(std::max(c.lt2 - vt2 / c.kt2, -lim), lim) : c.lt2;
            S dP[3];
            for (int r = 0; r < 3; ++r) dP[r] = (ln_new - c.ln) * c.n[r] + (lt1_new - c.lt1) * c.t1[r] + (lt2_new - c.lt2) * c.t2[r];
            c.ln = ln_new; c.lt1 = lt1_new; c.lt2 = lt2_new;
            apply_impulse(c, dP, (S)1, art);
        }
        // totals: net force per slot, reaction wrench on articulation bodies
        for (int s = 0; s < MPPIB_MAX_SLOTS; ++s) net[s][0] = net[s][1] = net[s][2] = 0;
        for (int i = 0; i < nc; ++i) {
            Contact<S>& c = ct[i];
            S F[3];
            for (int r = 0; r < 3; ++r) F[r] = (c.ln * c.n[r] + c.lt1 * c.t1[r] + c.lt2 * c.t2[r]) / h;
            if (c.slotA >= 0) for (int r = 0; r < 3; ++r) net[c.slotA][r] += F[r];
            if (c.slotB >= 0) for (int r = 0; r < 3; ++r) net[c.slotB][r] -= F[r];
        }
    }
    void integrate(S h) {
        for (int f = 0; f < m->nfree; ++f) {
            FreeBody<S>& b = fb[f];
            for (int i = 0; i < 3; ++i) b.x[i] += h * b.v[i];
            S wq[4] = {b.w[0], b.w[1], b.w[2], 0}, dq[4]; quat_mul(wq, b.q, dq);
            S l = 0; for (int i = 0; i < 4; ++i) { b.q[i] += (S)0.5 * h * dq[i]; l += b.q[i] * b.q[i]; }
            l = (S)1 / std::sqrt(l); for (int i = 0; i < 4; ++i) b.q[i] *= l;
            refresh_free(f);
        }
    }
};

template <class S>
void rollout_one(const MppibModel* m, const MppibParams* p, int K, int k, S* q, S* qd, ContactWorld<S>* cw, const float* root0,
                 const float* actions, int t0, int nsteps, float* obs) {
    const int nb = m->nb, nu = m->nu, T = p->T;
    const S h = (S)p->dt / (S)p->substeps;
    const bool contacts = cw != nullptr;
    Articulation<S> art; art.m = m; art.nb = nb;
    // base frame and gravity (Featherstone: a_base = -g expressed in base coordinates)
    S bq[4] = {(S)m->base_quat[0], (S)m->base_quat[1], (S)m->base_quat[2], (S)m->base_quat[3]};
    S bp[3] = {(S)m->base_pos[0], (S)m->base_pos[1], (S)m->base_pos[2]};
    M3<S> Rb = quat_to_R(bq);
    std::memset(&art.a0, 0, sizeof(art.a0));
    if (m->gravity_on) for (int i = 0; i < 3; ++i) { S s = 0; for (int j = 0; j < 3; ++j) s += Rb.a[j][i] * (S)m->gravity[j]; art.a0.a[3 + i] = -s; }

    const int nloop = nsteps > 0 ? nsteps : 1;   // nsteps == 0: observe only
    for (int t = t0; t < t0 + nloop; ++t) {
        // apply_robot_cmd (isaacgym_wrapper.py:524-572): command -> per-DOF targets
        S target[MPPIB_MAX_BODIES];
        for (int i = 0; i < nb && nsteps > 0; ++i) {
            S u0 = (S)p->u_scale * (S)actions[((size_t)t * nu + m->cmd_i0[i]) * K + k];
            S u1 = (S)p->u_scale * (S)actions[((size_t)t * nu + m->cmd_i1[i]) * K + k];
            target[i] = (S)m->cmd_c0[i] * u0 + (S)m->cmd_c1[i] * u1;
        }
        // step (isaacgym_wrapper.py:639-641): `substeps` solver substeps of h = dt/substeps
        for (int s = 0; s < (nsteps > 0 ? p->substeps : 0); ++s) {
            if (m->planar_base) {
                // differential drive reduced to a planar base: body twist (v, omega) -> world-frame velocity targets of the
                // three virtual joints; the forward axis turns with the current yaw (no lateral slip by construction)
                const S v = (S)p->u_scale * (S)actions[((size_t)t * nu + 0) * K + k], w = (S)p->u_scale * (S)actions[((size_t)t * nu + 1) * K + k];
                const S cy = std::cos(q[2]), sy = std::sin(q[2]), fx = (S)m->fwd_axis[0], fy = (S)m->fwd_axis[1];
                target[0] = v * (fx * cy - fy * sy); target[1] = v * (fx * sy + fy * cy); target[2] = w;
            }
            art.kinematics(q, qd);
            S tau[MPPIB_MAX_BODIES], dimp[MPPIB_MAX_BODIES], qdd[MPPIB_MAX_BODIES];
            for (int i = 0; i < nb; ++i) {
                S kd = (S)m->kd[i], b = (S)m->damping[i];
                if (m->drive_mode == MPPIB_DRIVE_VELOCITY) {
                    tau[i] = kd * (target[i] - qd[i]) - b * qd[i];     // implicit in qd_new via dimp
                } else {
                    S e = std::min(std::max(target[i], -(S)m->effort[i]), (S)m->effort[i]);
                    tau[i] = e - (kd + b) * qd[i];
                }
                dimp[i] = (S)m->armature[i] + h * (kd + b);
            }
            art.aba(tau, dimp, qdd);
            if (m->drive_mode == MPPIB_DRIVE_VELOCITY) {
                // drive force limit (URDF <limit effort>): a joint whose implicit drive torque exceeds it is
                // re-solved once with the constant saturated torque
                bool any = false;
                for (int i = 0; i < nb; ++i) {
                    S td = (S)m->kd[i] * (target[i] - (qd[i] + h * qdd[i]));
                    if (std::fabs(td) > (S)m->effort[i]) {
                        any = true;
                        tau[i] = (td > 0 ? (S)m->effort[i] : -(S)m->effort[i]) - (S)m->damping[i] * qd[i];
                        dimp[i] = (S)m->armature[i] + h * (S)m->damping[i];
                    }
                }
                if (any) art.aba(tau, dimp, qdd);
            }
            S qdn[MPPIB_MAX_BODIES];
            for (int i = 0; i < nb; ++i) qdn[i] = qd[i] + h * qdd[i];          // predicted (contact-free) joint velocities
            if (contacts) {
                // contacts act on the predicted velocities: poses of the start of the substep, velocities after gravity / drive
                art.kinematics(q, qdn);
                art.world_frames(Rb, bp);
                cw->shapes_world(art, Rb, bp, root0);
                cw->detect();
                for (int f = 0; f < m->nfree; ++f) if (m->free_gravity[f]) for (int i = 0; i < 3; ++i) cw->fb[f].v[i] += h * (S)m->gravity[i];
                cw->solve(art, h);
                for (int i = 0; i < nb; ++i) qdn[i] += cw->dqv[i];
            }
            for (int i = 0; i < nb; ++i) {           // semi-implicit Euler + velocity / position limits
                S v = std::min(std::max(qdn[i], -(S)m->qd_max[i]), (S)m->qd_max[i]);
                S x = q[i] + h * v;
                if (x < (S)m->q_lo[i]) { x = (S)m->q_lo[i]; if (v < 0) v = 0; }
                if (x > (S)m->q_hi[i]) { x = (S)m->q_hi[i]; if (v > 0) v = 0; }
                q[i] = x; qd[i] = v;
            }
            if (contacts) cw->integrate(h);
        }
        if (!obs) continue;
        // observe (refresh_* tensors, isaacgym_wrapper.py:642-645) -------------------------------------
        art.kinematics(q, qd);
        art.world_frames(Rb, bp);
        S qw[MPPIB_MAX_BODIES][4];
        for (int i = 0; i < nb; ++i) {
            const S* qp = m->parent[i] >= 0 ? qw[m->parent[i]] : bq;
            S qt[4] = {(S)m->tree_quat[i][0], (S)m->tree_quat[i][1], (S)m->tree_quat[i][2], (S)m->tree_quat[i][3]};
            S tmp[4]; quat_mul(qp, qt, tmp);
            if (m->jtype[i] == MPPIB_JOINT_REVOLUTE) {
                S qz[4] = {0, 0, std::sin(q[i] / 2), std::cos(q[i] / 2)};
                quat_mul(tmp, qz, qw[i]);
            } else for (int r = 0; r < 4; ++r) qw[i][r] = tmp[r];
        }
        int row = 0;
        const size_t TK = (size_t)T * K;
        for (int o = 0; o < p->nobs; ++o) {
            float vals[2 * MPPIB_MAX_BODIES > 13 ? 2 * MPPIB_MAX_BODIES : 13]; int w = 0;
            const int kind = p->obs[o].kind, idx = p->obs[o].index;
            if (kind == MPPIB_OBS_LINK_STATE) {
                int l = idx, b = m->link_body[l];
                const M3<S>& R = b >= 0 ? art.Rw[b] : Rb;
                S lp[3] = {(S)m->link_p[l][0], (S)m->link_p[l][1], (S)m->link_p[l][2]};
                S off[3]; mat_vec(R, lp, off);
                S ql[4] = {(S)m->link_quat[l][0], (S)m->link_quat[l][1], (S)m->link_quat[l][2], (S)m->link_quat[l][3]};
                S qo[4]; quat_mul(b >= 0 ? qw[b] : bq, ql, qo);
                S ww[3] = {0, 0, 0}, vw[3] = {0, 0, 0};
                if (b >= 0) for (int r = 0; r < 3; ++r) { ww[r] = art.ww[b][r]; vw[r] = art.vw[b][r]; }
                S wxo[3]; cross3(ww, off, wxo);
                for (int r = 0; r < 3; ++r) vals[r] = (float)((b >= 0 ? art.pw[b][r] : bp[r]) + off[r]);
                for (int r = 0; r < 4; ++r) vals[3 + r] = (float)qo[r];
                for (int r = 0; r < 3; ++r) vals[7 + r] = (float)(vw[r] + wxo[r]);
                for (int r = 0; r < 3; ++r) vals[10 + r] = (float)ww[r];
                w = 13;
            } else if (kind == MPPIB_OBS_DOF_STATE) {
                for (int i = 0; i < nb; ++i) { vals[2 * i] = (float)q[i]; vals[2 * i + 1] = (float)qd[i]; }
                w = 2 * nb;
            } else if (kind == MPPIB_OBS_FREE_STATE) {
                w = 13;
                for (int r = 0; r < 13; ++r) vals[r] = 0.f;
                if (contacts && idx < m->nfree) {
                    const FreeBody<S>& b = cw->fb[idx];
                    for (int r = 0; r < 3; ++r) { vals[r] = (float)b.x[r]; vals[7 + r] = (float)b.v[r]; vals[10 + r] = (float)b.w[r]; }
                    for (int r = 0; r < 4; ++r) vals[3 + r] = (float)b.q[r];
                }
            } else {
                w = 3;
                for (int r = 0; r < 3; ++r) vals[r] = contacts && idx < MPPIB_MAX_SLOTS ? (float)cw->net[idx][r] : 0.f;
            }
            for (int r = 0; r < w; ++r) obs[(size_t)(row + r) * TK + (size_t)t * K + k] = vals[r];
            row += w;
        }
    }
}

template <class S>
void rollout_impl(const MppibModel* m, const MppibParams* p, const float* state0, const float* root0, float* state,
                  const float* actions, int t0, int nsteps, float* obs, int nthreads) {
    const int K = p->K, nb = m->nb;
    const bool contacts = m->nfree > 0 || m->nshapes > 0;
    parallel_for(K, nthreads, [&](int a, int b) {
        std::vector<ContactWorld<S>> cwv(contacts ? 1 : 0);
        for (int k = a; k < b; ++k) {
            S q[MPPIB_MAX_BODIES], qd[MPPIB_MAX_BODIES];
            for (int i = 0; i < nb; ++i) {
                q[i] = state0 ? (S)state0[i] : (S)state[(size_t)i * K + k];
                qd[i] = state0 ? (S)state0[nb + i] : (S)state[(size_t)(nb + i) * K + k];
            }
            ContactWorld<S>* cw = contacts ? &cwv[0] : nullptr;
            if (cw) {
                cw->m = m; cw->p = p; cw->nc = 0;
                for (int s = 0; s < MPPIB_MAX_SLOTS; ++s) cw->net[s][0] = cw->net[s][1] = cw->net[s][2] = 0;
                cw->init_params(p->k_offset + (uint32_t)k);
                for (int f = 0; f < m->nfree; ++f) {
                    FreeBody<S>& fbd = cw->fb[f];
                    for (int r = 0; r < 13; ++r) {
                        const S v = state0 ? (S)root0[13 * m->free_actor[f] + r] : (S)state[(size_t)(2 * nb + 13 * f + r) * K + k];
                        if (r < 3) fbd.x[r] = v; else if (r < 7) fbd.q[r - 3] = v; else if (r < 10) fbd.v[r - 7] = v; else fbd.w[r - 10] = v;
                    }
                    cw->refresh_free(f);
                }
            }
            rollout_one<S>(m, p, K, k, q, qd, cw, root0, actions, t0, nsteps, obs);
            if (state) {
                for (int i = 0; i < nb; ++i) { state[(size_t)i * K + k] = (float)q[i]; state[(size_t)(nb + i) * K + k] = (float)qd[i]; }
                if (cw) for (int f = 0; f < m->nfree; ++f) {
                    const FreeBody<S>& fbd = cw->fb[f];
                    for (int r = 0; r < 13; ++r) {
                        const S v = r < 3 ? fbd.x[r] : (r < 7 ? fbd.q[r - 3] : (r < 10 ? fbd.v[r - 7] : fbd.w[r - 10]));
                        state[(size_t)(2 * nb + 13 * f + r) * K + k] = (float)v;
                    }
                }
            }
        }
    });
}

int obs_rows(const MppibModel* m, const MppibParams* p) {
    int r = 0;
    for (int o = 0; o < p->nobs; ++o) r += p->obs[o].kind == MPPIB_OBS_DOF_STATE ? 2 * m->nb : (p->obs[o].kind == MPPIB_OBS_CONTACT ? 3 : 13);
    return r;
}

}  // namespace

extern "C" {

int32_t oracle_abi_version(void) { return MPPIB_ABI_VERSION; }
int32_t oracle_obs_size(const MppibModel* m, const MppibParams* p) { return obs_rows(m, p); }
int32_t oracle_state_size(const MppibModel* m) { return 2 * m->nb + 13 * m->nfree; }

void oracle_philox(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t* out) {
    U4 r = philox4x32_10({c0, c1, c2, c3}, k0, k1);
    out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}

// inverse of the standard normal CDF (Wichura AS241, PPND16; |rel err| < 1e-16): z = sqrt(2) erfinv(2u - 1)
static double norm_ppf(double pu) {
    const double q = pu - 0.5;
    if (std::fabs(q) <= 0.425) {
        const double r = 0.180625 - q * q;
        return q * (((((((2.5090809287301226727e3 * r + 3.3430575583588128105e4) * r + 6.7265770927008700853e4) * r + 4.5921953931549871457e4) * r +
                         1.3731693765509461125e4) * r + 1.9715909503065514427e3) * r + 1.3314166789178437745e2) * r + 3.3871328727963666080e0) /
               (((((((5.2264952788528545610e3 * r + 2.8729085735721942674e4) * r + 3.9307895800092710610e4) * r + 2.1213794301586595867e4) * r +
                    5.3941960214247511077e3) * r + 6.8718700749205790830e2) * r + 4.2313330701600911252e1) * r + 1.0);
    }
    double r = q < 0 ? pu : 1.0 - pu;
    r = std::sqrt(-std::log(r));
    double val;
    if (r <= 5.0) {
        r -= 1.6;
        val = (((((((7.74545014278341407640e-4 * r + 2.27238449892691845833e-2) * r + 2.41780725177450611770e-1) * r + 1.27045825245236838258e0) * r +
                   3.64784832476320460504e0) * r + 5.76949722146069140550e0) * r + 4.63033784615654529590e0) * r + 1.42343711074968357734e0) /
              (((((((1.05075007164441684324e-9 * r + 5.47593808499534494600e-4) * r + 1.51986665636164571966e-2) * r + 1.48103976427480074590e-1) * r +
                   6.89767334985100004550e-1) * r + 1.67638483018380384940e0) * r + 2.05319162663775882187e0) * r + 1.0);
    } else {
        r -= 5.0;
        val = (((((((2.01033439929228813265e-7 * r + 2.71155556874348757815e-5) * r + 1.24266094738807843860e-3) * r + 2.65321895265761230930e-2) * r +
                   2.96560571828504891230e-1) * r + 1.78482653991729133580e0) * r + 5.46378491116411436990e0) * r + 6.65790464350110377720e0) /
              (((((((2.04426310338993978564e-15 * r + 1.42151175831644588870e-7) * r + 1.84631831751005468180e-5) * r + 7.86869131145613259100e-4) * r +
                   1.48753612908506148525e-2) * r + 1.36929880922735805310e-1) * r + 5.99832206555887937690e-1) * r + 1.0);
    }
    return q < 0 ? -val : val;
}

// generalised Halton point: radical inverse of `index` in base b, digits scrambled by digit -> mult * digit mod b
static double halton_point(uint32_t index, uint32_t base, uint32_t mult) {
    double f = 1.0 / base, r = 0.0;
    while (index > 0) { r += (double)((index % base) * mult % base) * f; index /= base; f /= base; }
    return r;
}
double oracle_halton(uint32_t index, uint32_t base, uint32_t mult) { return halton_point(index, base, mult); }
double oracle_norm_ppf(double u) { return norm_ppf(u); }

// Halton-spline noise library restatement (mppi_torch sampling_method "halton": Gaussian knots -> spline -> scale; SURVEY 8(a) M4)
void oracle_noise_library(const MppibModel* m, const MppibParams* p, uint32_t k_offset, uint32_t k_total, const int32_t* tab,
                          const float* B, int32_t n_knots, float* Z) {
    const int K = p->K, T = p->T, nu = m->nu, nd = n_knots * nu;
    std::vector<double> z((size_t)nd), cn((size_t)n_knots);
    for (int k = 0; k < K; ++k) {
        const uint32_t kg = k_offset + (uint32_t)k;
        const bool null_row = p->sample_null_action && kg == k_total - 1;
        for (int d = 0; d < nd; ++d) z[d] = norm_ppf((double)(float)halton_point(kg + 1u, (uint32_t)tab[d], (uint32_t)tab[nd + d]));
        for (int j = 0; j < nu; ++j) {
            for (int n = 0; n < n_knots; ++n) { double a = 0; for (int i = 0; i <= j; ++i) a += (double)p->sigma_chol[j * nu + i] * z[n * nu + i]; cn[n] = a; }
            for (int t = 0; t < T; ++t) {
                double v = 0; for (int n = 0; n < n_knots; ++n) v += (double)B[t * n_knots + n] * cn[n];
                Z[((size_t)t * nu + j) * K + k] = null_row ? 0.f : (float)v;
            }
        }
    }
}

void oracle_sample_library(const MppibModel* m, const MppibParams* p, uint32_t k_offset, uint32_t k_total, const float* U,
                           const float* prior_row, const float* Z, float* actions, float* noise) {
    const int K = p->K, T = p->T, nu = m->nu;
    for (int k = 0; k < K; ++k) {
        const uint32_t kg = k_offset + (uint32_t)k;
        for (int t = 0; t < T; ++t) for (int j = 0; j < nu; ++j) {
            const size_t idx = ((size_t)t * nu + j) * K + k;
            const float u = U[t * nu + j];
            float a = u + Z[idx];
            if (p->sample_null_action && kg == k_total - 1) a = 0.f;
            a = std::min(std::max(a, p->u_min[j]), p->u_max[j]);
            if (prior_row && kg == k_total - 2) a = prior_row[t * nu + j];
            actions[idx] = a;
            if (noise) noise[idx] = a - u;
        }
    }
}

// K1 restatement.  All buffers are host pointers with the device layouts of include/mppib.h.
void oracle_sample(const MppibModel* m, const MppibParams* p, uint64_t seed, uint64_t plan_idx, uint32_t k_offset,
                   uint32_t k_total, const float* U, const float* prior_row, float* actions, float* noise, int nthreads) {
    const int K = p->K, T = p->T, nu = m->nu;
    const uint32_t key0 = (uint32_t)seed, key1 = (uint32_t)(seed >> 32) ^ (uint32_t)plan_idx;
    parallel_for(K, nthreads, [&](int a, int b) {
        for (int k = a; k < b; ++k) {
            uint32_t kg = k_offset + (uint32_t)k;
            for (int t = 0; t < T; ++t) {
                float z[MPPIB_MAX_NU + 4];
                for (int blk = 0; blk * 4 < nu; ++blk) {
                    U4 r = philox4x32_10({kg, (uint32_t)t, (uint32_t)blk, (uint32_t)(plan_idx >> 32)}, key0, key1);
                    box_muller(r.x, r.y, &z[4 * blk], &z[4 * blk + 1]);
                    box_muller(r.z, r.w, &z[4 * blk + 2], &z[4 * blk + 3]);
                }
                for (int j = 0; j < nu; ++j) {
                    float n = 0.f;
                    for (int i = 0; i <= j; ++i) n += p->sigma_chol[j * nu + i] * z[i];
                    float u = U[t * nu + j];
                    float act = u + n;
                    if (p->sample_null_action && kg == k_total - 1) act = 0.f;
                    act = std::min(std::max(act, p->u_min[j]), p->u_max[j]);
                    if (prior_row && kg == k_total - 2) act = prior_row[t * nu + j];
                    size_t idx = ((size_t)t * nu + j) * K + k;
                    actions[idx] = act;
                    if (noise) noise[idx] = act - u;
                }
            }
        }
    });
}

void oracle_rollout(const MppibModel* m, const MppibParams* p, const float* state0, const float* root0, float* state, const float* actions,
                    int32_t t0, int32_t nsteps, float* obs, int32_t use_double, int32_t nthreads) {
    if (use_double) rollout_impl<double>(m, p, state0, root0, state, actions, t0, nsteps, obs, nthreads);
    else rollout_impl<float>(m, p, state0, root0, state, actions, t0, nsteps, obs, nthreads);
}

// K3 restatement (double accumulation).  partial = (beta, eta, W[T][nu]).
void oracle_reduce(const MppibModel* m, const MppibParams* p, const float* cost, const float* x, const float* U,
                   float* partial, float* S_out) {
    const int K = p->K, T = p->T, nu = m->nu;
    std::vector<double> S(K);
    double beta = std::numeric_limits<double>::infinity();
    for (int k = 0; k < K; ++k) {
        double s = 0, g = 1;
        for (int t = 0; t < T; ++t) { s += g * (double)cost[(size_t)t * K + k]; g *= (double)p->gamma; }
        if (p->mode == MPPIB_MODE_SIMPLE) {
            // perturbation cost  lambda * sum_t U_t^T Sigma^-1 noise_t   (noise @ Sigma^-1, then dot with U)
            double pc = 0;
            for (int t = 0; t < T; ++t) for (int j = 0; j < nu; ++j) {
                double ac = 0;
                for (int i = 0; i < nu; ++i) ac += (double)x[((size_t)t * nu + i) * K + k] * (double)p->sigma_inv[i * nu + j];
                pc += (double)U[t * nu + j] * ac;
            }
            s += (double)p->lambda_ * pc;
        }
        S[k] = s;
        if (std::isfinite(s) && s < beta) beta = s;
    }
    double eta = 0; std::vector<double> W((size_t)T * nu, 0.0);
    for (int k = 0; k < K; ++k) {
        double w = std::isfinite(S[k]) ? std::exp(-(S[k] - beta) / (double)p->lambda_) : 0.0;
        eta += w;
        for (int i = 0; i < T * nu; ++i) W[i] += w * (double)x[(size_t)i * K + k];
        if (S_out) S_out[k] = (float)S[k];
    }
    partial[0] = (float)beta; partial[1] = (float)eta;
    for (int i = 0; i < T * nu; ++i) partial[2 + i] = (float)W[i];
}

// The same reduction on `nthreads` host threads (bench.py's CPU arm): per-thread (beta, eta, W) over blocks of samples,
// merged with the shard-combine rule of oracle_finalize.  The single-threaded oracle_reduce above stays the parity checker.
void oracle_reduce_mt(const MppibModel* m, const MppibParams* p, const float* cost, const float* x, const float* U,
                      float* partial, int32_t nthreads) {
    const int K = p->K, T = p->T, nu = m->nu, NR = T * nu;
    std::vector<double> S(K);
    std::vector<double> g((size_t)NR, 0.0);               // lambda * Sigma^-1 U folded per row
    if (p->mode == MPPIB_MODE_SIMPLE)
        for (int t = 0; t < T; ++t) for (int i = 0; i < nu; ++i) {
            double ac = 0;
            for (int j = 0; j < nu; ++j) ac += (double)p->sigma_inv[i * nu + j] * (double)U[t * nu + j];
            g[(size_t)t * nu + i] = (double)p->lambda_ * ac;
        }
    std::mutex mu;
    double beta = std::numeric_limits<double>::infinity();
    parallel_for(K, nthreads, [&](int a, int b) {
        double bl = std::numeric_limits<double>::infinity();
        std::vector<double> acc(b - a, 0.0);
        double gt = 1;
        for (int t = 0; t < T; ++t) { for (int k = a; k < b; ++k) acc[k - a] += gt * (double)cost[(size_t)t * K + k]; gt *= (double)p->gamma; }
        if (p->mode == MPPIB_MODE_SIMPLE)
            for (int r = 0; r < NR; ++r) { const double gr = g[r]; for (int k = a; k < b; ++k) acc[k - a] += gr * (double)x[(size_t)r * K + k]; }
        for (int k = a; k < b; ++k) { S[k] = acc[k - a]; if (std::isfinite(S[k]) && S[k] < bl) bl = S[k]; }
        std::lock_guard<std::mutex> lk(mu);
        if (bl < beta) beta = bl;
    });
    double eta = 0; std::vector<double> W((size_t)NR, 0.0);
    parallel_for(K, nthreads, [&](int a, int b) {
        std::vector<double> w(b - a), Wl((size_t)NR, 0.0);
        double el = 0;
        for (int k = a; k < b; ++k) { w[k - a] = std::isfinite(S[k]) ? std::exp(-(S[k] - beta) / (double)p->lambda_) : 0.0; el += w[k - a]; }
        for (int r = 0; r < NR; ++r) { double s = 0; for (int k = a; k < b; ++k) s += w[k - a] * (double)x[(size_t)r * K + k]; Wl[r] = s; }
        std::lock_guard<std::mutex> lk(mu);
        eta += el;
        for (int r = 0; r < NR; ++r) W[r] += Wl[r];
    });
    partial[0] = (float)beta; partial[1] = (float)eta;
    for (int i = 0; i < NR; ++i) partial[2 + i] = (float)W[i];
}

// CPU restatement of the pose-reach cost term (examples/panda/planner.py:22-40 as ops.pose_cost / mppib_cost_pose evaluate it):
// cost[i] = w_pos |a[i,0:3] - b[i,0:3]| + w_ori |euler_ZYX(R(a[i,3:7]))[0:2]|, quaternion read real-first; strided views as
// in include/mppib.h.  Threaded over rows so that the CPU arm evaluates its Objective inside the parallel region.
void oracle_cost_pose(int64_t n, const float* a, int64_t a_si, int64_t a_sr, const float* b, int64_t b_si, int64_t b_sr, float w_pos,
                      float w_ori, float* cost, int32_t nthreads) {
    parallel_for((int)n, nthreads, [&](int lo, int hi) {
        for (int i = lo; i < hi; ++i) {
            const float* ai = a + (size_t)i * a_si;
            float c = 0.f;
            if (w_pos != 0.f) {
                const float* bi = b + (size_t)i * b_si;
                const float dx = ai[0] - bi[0], dy = ai[a_sr] - bi[b_sr], dz = ai[2 * a_sr] - bi[2 * b_sr];
                c += w_pos * std::sqrt(dx * dx + dy * dy + dz * dz);
            }
            if (w_ori != 0.f) {
                const float r = ai[3 * a_sr], qi = ai[4 * a_sr], qj = ai[5 * a_sr], qk = ai[6 * a_sr];
                const float two_s = 2.0f / (r * r + qi * qi + qj * qj + qk * qk);
                const float m00 = 1.f - two_s * (qj * qj + qk * qk), m10 = two_s * (qi * qj + qk * r), m20 = two_s * (qi * qk - qj * r);
                const float yaw = std::atan2(m10, m00), pitch = std::asin(-m20);
                c += w_ori * std::sqrt(yaw * yaw + pitch * pitch);
            }
            cost[i] = c;
        }
    });
}

// Savitzky-Golay window 9, polyorder 2, mode='interp' (SURVEY Appendix C), along T for one column.
static void savgol9(const double* y, int T, double* out) {
    static const double mid[9] = {-21, 14, 39, 54, 59, 54, 39, 14, -21};
    static const double edge[4][9] = {{763, 441, 189, 7, -105, -147, -119, -21, 147},
                                      {441, 322, 220.5, 136.5, 70, 21, -10.5, -24.5, -21},
                                      {189, 220.5, 232, 223.5, 195, 146.5, 78, -10.5, -119},
                                      {7, 136.5, 223.5, 268, 270, 229.5, 146.5, 21, -147}};
    for (int t = 0; t < T; ++t) {
        double s = 0;
        if (t < 4) { for (int i = 0; i < 9; ++i) s += edge[t][i] * y[i]; s /= 1155.0; }
        else if (t >= T - 4) { int e = T - 1 - t; for (int i = 0; i < 9; ++i) s += edge[e][i] * y[T - 1 - i]; s /= 1155.0; }
        else { for (int i = 0; i < 9; ++i) s += mid[i] * y[t - 4 + i]; s /= 231.0; }
        out[t] = s;
    }
}

// K4 restatement: combine G partials, update U, optional filter, first action.
void oracle_finalize(const MppibModel* m, const MppibParams* p, const float* partials, int32_t G, float* U,
                     float* action_out, float* stats) {
    const int T = p->T, nu = m->nu, P = 2 + T * nu;
    double beta = std::numeric_limits<double>::infinity();
    for (int g = 0; g < G; ++g) if (partials[(size_t)g * P + 1] > 0) beta = std::min(beta, (double)partials[(size_t)g * P]);
    double eta = 0; std::vector<double> W((size_t)T * nu, 0.0);
    for (int g = 0; g < G; ++g) {
        if (!(partials[(size_t)g * P + 1] > 0)) continue;
        double s = std::exp(-((double)partials[(size_t)g * P] - beta) / (double)p->lambda_);
        eta += s * (double)partials[(size_t)g * P + 1];
        for (int i = 0; i < T * nu; ++i) W[i] += s * (double)partials[(size_t)g * P + 2 + i];
    }
    std::vector<double> Un((size_t)T * nu);
    for (int i = 0; i < T * nu; ++i) {
        double wm = eta > 0 ? W[i] / eta : (p->mode == MPPIB_MODE_SIMPLE ? 0.0 : (double)U[i]);   // no valid sample: keep U
        Un[i] = p->mode == MPPIB_MODE_SIMPLE ? (double)U[i] + wm
                                             : (1.0 - (double)p->step_size_mean) * (double)U[i] + (double)p->step_size_mean * wm;
    }
    if (p->filter_u) {
        std::vector<double> col(T), out(T);
        for (int j = 0; j < nu; ++j) {
            for (int t = 0; t < T; ++t) col[t] = Un[t * nu + j];
            savgol9(col.data(), T, out.data());
            // smoothing may overshoot the control bounds at the horizon edges: clamp back (spec decision, DESIGN.md)
            for (int t = 0; t < T; ++t) Un[t * nu + j] = std::min(std::max(out[t], (double)p->u_min[j]), (double)p->u_max[j]);
        }
    }
    for (int i = 0; i < T * nu; ++i) U[i] = (float)Un[i];
    for (int j = 0; j < nu; ++j) action_out[j] = U[j];
    if (stats) { stats[0] = (float)beta; stats[1] = (float)eta; }
}

void oracle_shift(const MppibModel* m, const MppibParams* p, float* U) {
    const int T = p->T, nu = m->nu;
    for (int t = 0; t + 1 < T; ++t) for (int j = 0; j < nu; ++j) U[t * nu + j] = U[(t + 1) * nu + j];
    for (int j = 0; j < nu; ++j) U[(T - 1) * nu + j] = p->u_init[j];
}

}  // extern "C"
