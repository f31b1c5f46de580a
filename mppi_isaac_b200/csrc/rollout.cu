// rollout.cu -- K2: batched articulated rigid-body rollout (replaces gym.simulate()/IsaacGymWrapper.step
// on the MPPI path: mppiisaac/planner/isaacgym_wrapper.py:524-572 apply_robot_cmd, :639-655 step).
//
// Mapping: ONE THREAD PER ROLLOUT, 32-thread CTAs (<= 1 warp per SM sub-partition up to K = 18 944).  The
// recursion over bodies and over time is strictly serial (SURVEY.md section 5 "T stays sequential"); all
// parallelism is across the K samples.
//   * model / parameter blocks are __grid_constant__ kernel parameters: they live in the constant bank and are
//     read warp-uniformly (every lane needs the same constant at the same time);
//   * per-body working set of a rollout lives in SHARED MEMORY as [slot][lane] (bank = lane: conflict free), so
//     the three ABA sweeps are ROLLED loops over bodies.  The first version of this kernel unrolled everything
//     into registers: 7.6k SASS instructions (122 KB) per substep body, far beyond the 32 KB L1.5 instruction
//     cache, so issue stalled on instruction fetch;
//   * serial chains (point robot, heijn, panda) carry the parent transform / articulated inertia / acceleration
//     in registers from one body to the next (template CHAIN); general trees (gripper fingers) keep them in
//     shared memory and index the parent at run time;
//   * all K-indexed global arrays are [..][K] with k innermost: every global access of a warp is one
//     coalesced 128-byte line.
//
// Dynamics formulation: articulated-body algorithm in WORLD coordinates (spatial vectors taken about the
// world origin), so articulated inertias are summed into the parent without any 6x6 frame transform.
// This is deliberately a different formulation from the CPU oracle (body-coordinate ABA with dense 6x6
// Pluecker transforms); the two must agree to float32 round-off.
//
// Per substep h = dt/substeps:
//   1. kinematics + world spatial inertia + velocity-product terms            (sweep root -> leaves)
//   2. articulated inertias / bias forces with the PD drive and joint damping implicit in the joint-space
//      diagonal (leaves -> root), then accelerations (root -> leaves); one re-solve with constant saturated
//      torques for joints whose drive torque exceeds URDF effort
//   3. semi-implicit Euler, velocity limit, position limits
// After the last substep of a model step the observed rows are written to obs[R][T][K].
#include "common.cuh"

// tuning knobs (A/B builds: tools/tune_rollout.py)
#ifndef ROLL_UNROLL_S1
#define ROLL_UNROLL_S1 1      // unroll factor of sweep 1 (kinematics / inertia: bodies are independent apart from the frame recursion)
#endif
#ifndef ROLL_S1_PIPE
#define ROLL_S1_PIPE 0        // software-pipelined sweep 1 for serial chains (kinematics of body i+1 with the dynamics terms of body i)
#endif
#ifndef ROLL_UNROLL_S2
#define ROLL_UNROLL_S2 1      // unroll factor of sweep 2 (articulated inertias)
#endif
#ifndef ROLL_UNROLL_S3
#define ROLL_UNROLL_S3 2      // unroll factor of sweep 3 (accelerations)
#endif
#define MPPIB_STR2(x) #x
#define MPPIB_STR(x) MPPIB_STR2(x)
#define MPPIB_UNROLL(n) _Pragma(MPPIB_STR(unroll n))

#include "rbd_math.cuh"

namespace {


// spatial (6x6 symmetric) inertia about the world origin: [[A, B], [B^T, C]]
struct SpI { S3 A; M3 B; S3 C; };
struct V6 { V3 n, f; };   // force vectors (n = moment, f = force) and motion vectors (n = angular, f = linear)

__device__ __forceinline__ V6 mul(const SpI& I, const V6& s) {
    V6 o;
    o.n = mul(I.A, s.n) + mul(I.B, s.f);
    o.f = mulT(I.B, s.n) + mul(I.C, s.f);
    return o;
}
__device__ __forceinline__ float dot6(const V6& a, const V6& b) { return dot(a.n, b.n) + dot(a.f, b.f); }
__device__ __forceinline__ void add_to(SpI& p, const SpI& c) {
    p.A.xx += c.A.xx; p.A.yy += c.A.yy; p.A.zz += c.A.zz; p.A.xy += c.A.xy; p.A.xz += c.A.xz; p.A.yz += c.A.yz;
    p.B.m00 += c.B.m00; p.B.m01 += c.B.m01; p.B.m02 += c.B.m02; p.B.m10 += c.B.m10; p.B.m11 += c.B.m11; p.B.m12 += c.B.m12;
    p.B.m20 += c.B.m20; p.B.m21 += c.B.m21; p.B.m22 += c.B.m22;
    p.C.xx += c.C.xx; p.C.yy += c.C.yy; p.C.zz += c.C.zz; p.C.xy += c.C.xy; p.C.xz += c.C.xz; p.C.yz += c.C.yz;
}
// I -= s * U U^T
__device__ __forceinline__ void rank1_sub(SpI& I, const V6& U, float s) {
    V3 a = s * U.n, b = s * U.f;
    I.A.xx -= a.x * U.n.x; I.A.yy -= a.y * U.n.y; I.A.zz -= a.z * U.n.z;
    I.A.xy -= a.x * U.n.y; I.A.xz -= a.x * U.n.z; I.A.yz -= a.y * U.n.z;
    I.B.m00 -= a.x * U.f.x; I.B.m01 -= a.x * U.f.y; I.B.m02 -= a.x * U.f.z;
    I.B.m10 -= a.y * U.f.x; I.B.m11 -= a.y * U.f.y; I.B.m12 -= a.y * U.f.z;
    I.B.m20 -= a.z * U.f.x; I.B.m21 -= a.z * U.f.y; I.B.m22 -= a.z * U.f.z;
    I.C.xx -= b.x * U.f.x; I.C.yy -= b.y * U.f.y; I.C.zz -= b.z * U.f.z;
    I.C.xy -= b.x * U.f.y; I.C.xz -= b.x * U.f.z; I.C.yz -= b.y * U.f.z;
}
__device__ __forceinline__ SpI rigid_inertia(const S3& A, V3 hw, float mass) {
    SpI I;
    I.A = A;
    I.B.m00 = 0; I.B.m01 = -hw.z; I.B.m02 = hw.y; I.B.m10 = hw.z; I.B.m11 = 0; I.B.m12 = -hw.x; I.B.m20 = -hw.y; I.B.m21 = hw.x; I.B.m22 = 0;
    I.C.xx = mass; I.C.yy = mass; I.C.zz = mass; I.C.xy = 0; I.C.xz = 0; I.C.yz = 0;
    return I;
}

// ---- shared-memory slots per body ([slot][lane]) --------------------------------------------------------------
enum : int {
    F_S = 0,      // 6  joint motion subspace (world, about the origin)
    F_C = 6,      // 6  velocity-product acceleration
    F_A = 12,     // 6  rotational inertia about the world origin
    F_HW = 18,    // 3  first moment m * c_world
    F_PB = 21,    // 6  bias force v x* I v
    F_U = 27,     // 6  IA S
    F_INVD = 33, F_UU = 34, F_QDD = 35, F_Q = 36, F_QD = 37, F_TGT = 38, F_SAT = 39,
    // observation scratch: quaternion, world rotation, origin, spatial velocity of the body at the END of a model step.  It is
    // filled by the first sweep 1 of the NEXT step (same state, same kinematics) so that no extra kinematics pass is needed
    F_OQ = 40, F_OR = 44, F_OO = 53, F_OV = 56,
    NSLOT_CHAIN = 62,
    // general trees (and contact scenes) keep every body's world frame for the parent lookup / the shapes: the SAME slots as the
    // observation scratch (when the observation is taken, the frame of the current sweep 1 IS the observed frame)
    F_R = F_OR,   // 9  world rotation of the body
    F_O = F_OO,   // 3
    F_V = F_OV,   // 6  spatial velocity
    F_IA = 62,    // 21 articulated inertia accumulator
    F_PA = 83,    // 6  articulated bias accumulator
    F_ACC = 89,   // 6  spatial acceleration
    NSLOT_TREE = 95,
};

#define SM(i, f) sm[((i) * NSLOT + (f)) * 32 + lane]

__device__ __forceinline__ void st3(float* sm, int base, int lane, V3 v) { sm[(base + 0) * 32 + lane] = v.x; sm[(base + 1) * 32 + lane] = v.y; sm[(base + 2) * 32 + lane] = v.z; }
__device__ __forceinline__ V3 ld3(const float* sm, int base, int lane) { return mk(sm[(base + 0) * 32 + lane], sm[(base + 1) * 32 + lane], sm[(base + 2) * 32 + lane]); }
__device__ __forceinline__ void st6(float* sm, int base, int lane, const V6& v) { st3(sm, base, lane, v.n); st3(sm, base + 3, lane, v.f); }
__device__ __forceinline__ V6 ld6(const float* sm, int base, int lane) { V6 v; v.n = ld3(sm, base, lane); v.f = ld3(sm, base + 3, lane); return v; }
__device__ __forceinline__ void stS3(float* sm, int base, int lane, const S3& s) {
    sm[(base + 0) * 32 + lane] = s.xx; sm[(base + 1) * 32 + lane] = s.yy; sm[(base + 2) * 32 + lane] = s.zz;
    sm[(base + 3) * 32 + lane] = s.xy; sm[(base + 4) * 32 + lane] = s.xz; sm[(base + 5) * 32 + lane] = s.yz;
}
__device__ __forceinline__ S3 ldS3(const float* sm, int base, int lane) {
    S3 s; s.xx = sm[(base + 0) * 32 + lane]; s.yy = sm[(base + 1) * 32 + lane]; s.zz = sm[(base + 2) * 32 + lane];
    s.xy = sm[(base + 3) * 32 + lane]; s.xz = sm[(base + 4) * 32 + lane]; s.yz = sm[(base + 5) * 32 + lane]; return s;
}
__device__ __forceinline__ void stM3(float* sm, int base, int lane, const M3& m) {
    sm[(base + 0) * 32 + lane] = m.m00; sm[(base + 1) * 32 + lane] = m.m01; sm[(base + 2) * 32 + lane] = m.m02;
    sm[(base + 3) * 32 + lane] = m.m10; sm[(base + 4) * 32 + lane] = m.m11; sm[(base + 5) * 32 + lane] = m.m12;
    sm[(base + 6) * 32 + lane] = m.m20; sm[(base + 7) * 32 + lane] = m.m21; sm[(base + 8) * 32 + lane] = m.m22;
}
__device__ __forceinline__ M3 ldM3(const float* sm, int base, int lane) {
    M3 m; m.m00 = sm[(base + 0) * 32 + lane]; m.m01 = sm[(base + 1) * 32 + lane]; m.m02 = sm[(base + 2) * 32 + lane];
    m.m10 = sm[(base + 3) * 32 + lane]; m.m11 = sm[(base + 4) * 32 + lane]; m.m12 = sm[(base + 5) * 32 + lane];
    m.m20 = sm[(base + 6) * 32 + lane]; m.m21 = sm[(base + 7) * 32 + lane]; m.m22 = sm[(base + 8) * 32 + lane]; return m;
}
__device__ __forceinline__ void stSpI(float* sm, int base, int lane, const SpI& I) { stS3(sm, base, lane, I.A); stM3(sm, base + 6, lane, I.B); stS3(sm, base + 15, lane, I.C); }
__device__ __forceinline__ SpI ldSpI(const float* sm, int base, int lane) { SpI I; I.A = ldS3(sm, base, lane); I.B = ldM3(sm, base + 6, lane); I.C = ldS3(sm, base + 15, lane); return I; }

struct Frame { M3 R; V3 o; V6 V; };

// 4-byte asynchronous global -> shared copy (LDGSTS): the warp keeps issuing while the line is in flight
__device__ __forceinline__ void cp_async4(float* dst_smem, const float* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// world kinematics of body i from its parent's frame (R: body axes as columns in the world, o: origin)
__device__ __forceinline__ void body_kinematics(const MppibModel& m, int i, float q, float qd, const Frame& par, Frame& out, V6& S) {
    const float* tr = m.tree_R[i];
    M3 Rt;   // Rp * tree_R
    {
        V3 c0 = mul(par.R, mk(tr[0], tr[3], tr[6])), c1 = mul(par.R, mk(tr[1], tr[4], tr[7])), c2 = mul(par.R, mk(tr[2], tr[5], tr[8]));
        Rt.m00 = c0.x; Rt.m10 = c0.y; Rt.m20 = c0.z; Rt.m01 = c1.x; Rt.m11 = c1.y; Rt.m21 = c1.z; Rt.m02 = c2.x; Rt.m12 = c2.y; Rt.m22 = c2.z;
    }
    V3 oi = par.o + mul(par.R, mk(m.tree_p[i][0], m.tree_p[i][1], m.tree_p[i][2]));
    const V3 axis = mk(Rt.m02, Rt.m12, Rt.m22);
    if (m.jtype[i] == MPPIB_JOINT_REVOLUTE) {
        float sq, cq;
        sincos_cw(q, &sq, &cq);
        out.R = Rt;   // Rt * Rz(q)
        out.R.m00 = Rt.m00 * cq + Rt.m01 * sq; out.R.m01 = Rt.m01 * cq - Rt.m00 * sq;
        out.R.m10 = Rt.m10 * cq + Rt.m11 * sq; out.R.m11 = Rt.m11 * cq - Rt.m10 * sq;
        out.R.m20 = Rt.m20 * cq + Rt.m21 * sq; out.R.m21 = Rt.m21 * cq - Rt.m20 * sq;
        out.o = oi;
        S.n = axis; S.f = cross(oi, axis);
    } else {
        out.R = Rt; out.o = oi + q * axis;
        S.n = mk(0, 0, 0); S.f = axis;
    }
    out.V.n = par.V.n + qd * S.n;
    out.V.f = par.V.f + qd * S.f;
}

// sweep-1 dynamics of body i in its world frame f: rotational inertia about the world origin, first moment, bias force
// V x* (I V) and velocity-product acceleration c = V x (S qd)  ->  slots F_S, F_C, F_A, F_HW, F_PB
template <int NSLOT>
__device__ __forceinline__ void s1_dynamics(const MppibModel& m, float* sm, int lane, int i, const Frame& f, const V6& S, float qdi) {
    const float mass = m.mass[i];
    // centre of mass (world), first moment, inertia about the world origin:
    //   R I_o R^T + m[(|cw|^2 - |cb|^2) 1 - (cw cw^T - cb cb^T)],  cb = R c_body, cw = o + cb
    V3 cb = mk(0, 0, 0);
    if (mass > 0.f) cb = __frcp_rn(mass) * mul(f.R, mk(m.mcom[i][0], m.mcom[i][1], m.mcom[i][2]));
    const V3 cw = f.o + cb;
    const V3 hw = mass * cw;
    const S3 Io = {m.inertia[i][0], m.inertia[i][1], m.inertia[i][2], m.inertia[i][3], m.inertia[i][4], m.inertia[i][5]};
    const V3 r0 = mk(f.R.m00, f.R.m01, f.R.m02), r1 = mk(f.R.m10, f.R.m11, f.R.m12), r2 = mk(f.R.m20, f.R.m21, f.R.m22);
    const V3 t0v = mul(Io, r0), t1v = mul(Io, r1), t2v = mul(Io, r2);
    S3 A;
    A.xx = dot(r0, t0v); A.yy = dot(r1, t1v); A.zz = dot(r2, t2v);
    A.xy = dot(r0, t1v); A.xz = dot(r0, t2v); A.yz = dot(r1, t2v);
    const float d2 = mass * (dot(cw, cw) - dot(cb, cb));
    A.xx += d2 - mass * (cw.x * cw.x - cb.x * cb.x); A.yy += d2 - mass * (cw.y * cw.y - cb.y * cb.y);
    A.zz += d2 - mass * (cw.z * cw.z - cb.z * cb.z);
    A.xy -= mass * (cw.x * cw.y - cb.x * cb.y); A.xz -= mass * (cw.x * cw.z - cb.x * cb.z);
    A.yz -= mass * (cw.y * cw.z - cb.y * cb.z);
    // bias force V x* (I V) and velocity-product acceleration c = V x (S qd)
    const V3 w = f.V.n, v = f.V.f;
    const V3 nn = mul(A, w) + cross(hw, v);
    const V3 ff = mass * v - cross(hw, w);
    V6 pb, c;
    pb.n = cross(w, nn) + cross(v, ff);
    pb.f = cross(w, ff);
    const V3 sw = qdi * S.n, sv = qdi * S.f;
    c.n = cross(w, sw);
    c.f = cross(w, sv) + cross(v, sw);
    st6(sm, i * NSLOT + F_S, lane, S);
    st6(sm, i * NSLOT + F_C, lane, c);
    stS3(sm, i * NSLOT + F_A, lane, A);
    st3(sm, i * NSLOT + F_HW, lane, hw);
    st6(sm, i * NSLOT + F_PB, lane, pb);
}

#include "contact.cuh"

template <bool CHAIN, bool CONTACT>
__global__ void __launch_bounds__(32)
mppib_rollout_kernel(const __grid_constant__ MppibModel m, const __grid_constant__ MppibParams p,
                     const float* __restrict__ state0, const float* __restrict__ root0, float* __restrict__ state,
                     const float* __restrict__ actions, int t0, int nsteps, float* __restrict__ obs) {
    extern __shared__ float sm[];
    constexpr int NSLOT = (CHAIN && !CONTACT) ? NSLOT_CHAIN : NSLOT_TREE;
    constexpr bool STORE_FRAMES = !CHAIN || CONTACT;     // world frame of every body kept in shared memory
    const int K = p.K, T = p.T, nu = m.nu, nb = m.nb;
    const int lane = threadIdx.x;
    const int k = blockIdx.x * 32 + lane;
    __shared__ uint32_t s_bmask[MPPIB_MAX_SHAPES];        // candidate partners of every shape (contact::partner_mask), one table per CTA,
    if (CONTACT) {                                        // filled by all 32 lanes before the lanes of a ragged last CTA leave
        for (int s = lane; s < m.nshapes; s += 32) s_bmask[s] = contact::partner_mask(m, s);
        __syncwarp();
    }
    if (k >= K) return;
    const float h = p.dt / (float)p.substeps;
    const bool vel_mode = m.drive_mode == MPPIB_DRIVE_VELOCITY;

    for (int i = 0; i < nb; ++i) {
        SM(i, F_Q) = state0 ? state0[i] : state[(size_t)i * K + k];
        SM(i, F_QD) = state0 ? state0[nb + i] : state[(size_t)(nb + i) * K + k];
    }
    float* xs = sm + (size_t)nb * NSLOT * 32;             // free bodies / shapes / contacts (CONTACT kernels only)
    const contact::Layout L(nb, m.nfree, m.nshapes, m.max_contacts);
    if (CONTACT) contact::init(m, p, L, xs, lane, p.k_offset + (uint32_t)k, root0, state, state0 != nullptr, K, k);
    Frame base;
    const Quat bq = {m.base_quat[0], m.base_quat[1], m.base_quat[2], m.base_quat[3]};
    base.R = quat_to_R(bq);
    base.o = mk(m.base_pos[0], m.base_pos[1], m.base_pos[2]);
    base.V.n = mk(0, 0, 0); base.V.f = mk(0, 0, 0);
    if (CONTACT) contact::shapes_world<NSLOT>(m, L, sm, xs, lane, base.R, base.o, root0, true);
    // gravity enters as a fictitious base acceleration a0 = [0; -g]
    V6 a0; a0.n = mk(0, 0, 0);
    a0.f = m.gravity_on ? mk(-m.gravity[0], -m.gravity[1], -m.gravity[2]) : mk(0.f, 0.f, 0.f);

    // world frames + quaternions of all bodies at the current (q, qd) -> observation scratch (standalone pass: used once at the end)
    auto observe_pass = [&]() {
    {
        Frame par = base; Quat qp = bq;
#pragma unroll 1
        for (int i = 0; i < nb; ++i) {
            const int pi = CHAIN ? i - 1 : m.parent[i];
            if (!CHAIN) {
                if (pi >= 0) {
                    par.R = ldM3(sm, pi * NSLOT + F_OR, lane); par.o = ld3(sm, pi * NSLOT + F_OO, lane); par.V = ld6(sm, pi * NSLOT + F_OV, lane);
                    qp.x = SM(pi, F_OQ); qp.y = SM(pi, F_OQ + 1); qp.z = SM(pi, F_OQ + 2); qp.w = SM(pi, F_OQ + 3);
                } else { par = base; qp = bq; }
            }
            const float qi = SM(i, F_Q), qdi = SM(i, F_QD);
            Frame f; V6 S;
            body_kinematics(m, i, qi, qdi, par, f, S);
            const Quat qt = {m.tree_quat[i][0], m.tree_quat[i][1], m.tree_quat[i][2], m.tree_quat[i][3]};
            Quat r = qmul(qp, qt);
            if (m.jtype[i] == MPPIB_JOINT_REVOLUTE) {
                float sh, ch; sincos_cw(0.5f * qi, &sh, &ch);
                const Quat qz = {0.f, 0.f, sh, ch};
                r = qmul(r, qz);
            }
            stM3(sm, i * NSLOT + F_OR, lane, f.R); st3(sm, i * NSLOT + F_OO, lane, f.o); st6(sm, i * NSLOT + F_OV, lane, f.V);
            SM(i, F_OQ) = r.x; SM(i, F_OQ + 1) = r.y; SM(i, F_OQ + 2) = r.z; SM(i, F_OQ + 3) = r.w;
            if (CHAIN) { par = f; qp = r; }
        }
    }
    };
    // write the observed rows of model step `t` from the observation scratch / state slots
    auto write_obs = [&](int t) {
    const size_t TK = (size_t)T * K;
    float* dst = obs + (size_t)t * K + k;
    int row = 0;
    for (int oi = 0; oi < p.nobs; ++oi) {
        const int kind = p.obs[oi].kind, idx = p.obs[oi].index;
        if (kind == MPPIB_OBS_LINK_STATE) {
            const int b = m.link_body[idx];
            M3 Rl; V3 ol, w, vO; Quat qb;
            if (b >= 0) {
                Rl = ldM3(sm, b * NSLOT + F_OR, lane); ol = ld3(sm, b * NSLOT + F_OO, lane);
                const V6 Vb = ld6(sm, b * NSLOT + F_OV, lane); w = Vb.n; vO = Vb.f;
                qb.x = SM(b, F_OQ); qb.y = SM(b, F_OQ + 1); qb.z = SM(b, F_OQ + 2); qb.w = SM(b, F_OQ + 3);
            } else { Rl = base.R; ol = base.o; w = mk(0, 0, 0); vO = mk(0, 0, 0); qb = bq; }
            const V3 pos = ol + mul(Rl, mk(m.link_p[idx][0], m.link_p[idx][1], m.link_p[idx][2]));
            const Quat ql = {m.link_quat[idx][0], m.link_quat[idx][1], m.link_quat[idx][2], m.link_quat[idx][3]};
            const Quat qo = qmul(qb, ql);
            const V3 vel = vO + cross(w, pos);   // spatial velocity about the world origin -> velocity of the link origin
            dst[(size_t)(row + 0) * TK] = pos.x; dst[(size_t)(row + 1) * TK] = pos.y; dst[(size_t)(row + 2) * TK] = pos.z;
            dst[(size_t)(row + 3) * TK] = qo.x; dst[(size_t)(row + 4) * TK] = qo.y; dst[(size_t)(row + 5) * TK] = qo.z;
            dst[(size_t)(row + 6) * TK] = qo.w;
            dst[(size_t)(row + 7) * TK] = vel.x; dst[(size_t)(row + 8) * TK] = vel.y; dst[(size_t)(row + 9) * TK] = vel.z;
            dst[(size_t)(row + 10) * TK] = w.x; dst[(size_t)(row + 11) * TK] = w.y; dst[(size_t)(row + 12) * TK] = w.z;
            row += 13;
        } else if (kind == MPPIB_OBS_DOF_STATE) {
            for (int i = 0; i < nb; ++i) {
                dst[(size_t)(row + 2 * i) * TK] = SM(i, F_Q);
                dst[(size_t)(row + 2 * i + 1) * TK] = SM(i, F_QD);
            }
            row += 2 * nb;
        } else if (kind == MPPIB_OBS_FREE_STATE) {
            const int fb = L.fb0 + idx * contact::FBN;
            for (int r = 0; r < 13; ++r) dst[(size_t)(row + r) * TK] = (CONTACT && idx < m.nfree) ? xs[(fb + r) * 32 + lane] : 0.f;
            row += 13;
        } else {
            for (int r = 0; r < 3; ++r) dst[(size_t)(row + r) * TK] = (CONTACT && idx < MPPIB_MAX_SLOTS) ? xs[(L.net0 + 3 * idx + r) * 32 + lane] : 0.f;
            row += 3;
        }
    }
    };
    int pending = (obs != nullptr && nsteps == 0) ? t0 : -1;   // step whose observation is still to be written
    // the nu action rows of step t+1 are fetched (asynchronously, double-buffered [2][nu][lane]) while step t integrates: a
    // plain load at the top of a step left the only resident warp of the SM waiting on HBM for ~9 % of the kernel
    float* ua = xs + (CONTACT ? (size_t)L.total * 32 : 0);
    auto fetch_actions = [&](int t, int buf) {
        for (int j = 0; j < nu; ++j) cp_async4(&ua[(buf * nu + j) * 32 + lane], &actions[((size_t)t * nu + j) * K + k]);
        cp_async_commit();
    };
    if (nsteps > 0) fetch_actions(t0, 0);
    for (int t = t0; t < t0 + nsteps; ++t) {
        const float* ut = ua + (size_t)((t - t0) & 1) * nu * 32;
        cp_async_wait_all();
        if (t + 1 < t0 + nsteps) fetch_actions(t + 1, ((t - t0) & 1) ^ 1);
        {
            // apply_robot_cmd: command -> per-DOF targets (diff-drive IK folded into the cmd map)
            for (int i = 0; i < nb; ++i) {
                const float u0 = p.u_scale * ut[m.cmd_i0[i] * 32 + lane];
                const float u1 = p.u_scale * ut[m.cmd_i1[i] * 32 + lane];
                SM(i, F_TGT) = m.cmd_c0[i] * u0 + m.cmd_c1[i] * u1;
            }
        }
        const int nsub = p.substeps;
#pragma unroll 1
        for (int sub = 0; sub < nsub; ++sub) {
            if (m.planar_base) {
                // differential drive reduced to a planar base: body twist (v, omega) -> world-frame velocity targets of the
                // three virtual joints; the forward axis turns with the current yaw (no lateral slip by construction)
                const float v = p.u_scale * ut[lane], w = p.u_scale * ut[32 + lane];
                float sy, cy; sincos_cw(SM(2, F_Q), &sy, &cy);
                SM(0, F_TGT) = v * (m.fwd_axis[0] * cy - m.fwd_axis[1] * sy);
                SM(1, F_TGT) = v * (m.fwd_axis[0] * sy + m.fwd_axis[1] * cy);
                SM(2, F_TGT) = w;
            }
            // ------------------------------------------------------------------ sweep 1: root -> leaves
            {
                const bool obs_now = sub == 0 && pending >= 0;   // this sweep's kinematics ARE the observation of the previous step
                Frame par = base; Quat qp = bq;
#if ROLL_S1_PIPE
                if (CHAIN && !CONTACT) {
                    // software-pipelined: the kinematics of body i+1 (the frame recursion) and the inertia / bias terms of body i are
                    // independent and sit in ONE basic block, so the scheduler can interleave them (the last iteration recomputes
                    // the kinematics of body nb-1, discarded)
                    auto head = [&](int j, const Frame& pf, Frame& f, V6& S, float& qdj) {
                        const float qj = SM(j, F_Q);
                        qdj = SM(j, F_QD);
                        body_kinematics(m, j, qj, qdj, pf, f, S);
                        return qj;
                    };
                    auto obs_head = [&](int j, float qj, const Frame& f) {
                        const Quat qt = {m.tree_quat[j][0], m.tree_quat[j][1], m.tree_quat[j][2], m.tree_quat[j][3]};
                        Quat r = qmul(qp, qt);
                        if (m.jtype[j] == MPPIB_JOINT_REVOLUTE) {
                            float sh, ch; sincos_cw(0.5f * qj, &sh, &ch);
                            const Quat qz = {0.f, 0.f, sh, ch};
                            r = qmul(r, qz);
                        }
                        stM3(sm, j * NSLOT + F_OR, lane, f.R); st3(sm, j * NSLOT + F_OO, lane, f.o); st6(sm, j * NSLOT + F_OV, lane, f.V);
                        SM(j, F_OQ) = r.x; SM(j, F_OQ + 1) = r.y; SM(j, F_OQ + 2) = r.z; SM(j, F_OQ + 3) = r.w;
                        qp = r;
                    };
                    Frame fc; V6 Sc; float qdc;
                    { const float q0 = head(0, base, fc, Sc, qdc); if (obs_now) obs_head(0, q0, fc); }
#pragma unroll 1
                    for (int i = 0; i < nb; ++i) {
                        const int j = i + 1 < nb ? i + 1 : nb - 1;
                        Frame fn; V6 Sn; float qdn;
                        const float qj = head(j, fc, fn, Sn, qdn);
                        s1_dynamics<NSLOT>(m, sm, lane, i, fc, Sc, qdc);
                        SM(i, F_SAT) = 0.f;
                        if (obs_now && i + 1 < nb) obs_head(j, qj, fn);
                        fc = fn; Sc = Sn; qdc = qdn;
                    }
                } else
#endif
                MPPIB_UNROLL(ROLL_UNROLL_S1)
                for (int i = 0; i < nb; ++i) {
                    if (!CHAIN) {
                        const int pi = m.parent[i];
                        if (pi >= 0) {
                            par.R = ldM3(sm, pi * NSLOT + F_R, lane); par.o = ld3(sm, pi * NSLOT + F_O, lane); par.V = ld6(sm, pi * NSLOT + F_V, lane);
                            if (obs_now) { qp.x = SM(pi, F_OQ); qp.y = SM(pi, F_OQ + 1); qp.z = SM(pi, F_OQ + 2); qp.w = SM(pi, F_OQ + 3); }
                        } else { par = base; qp = bq; }
                    }
                    const float qi = SM(i, F_Q), qdi = SM(i, F_QD);
                    Frame f; V6 S;
                    body_kinematics(m, i, qi, qdi, par, f, S);
                    if (obs_now) {
                        const Quat qt = {m.tree_quat[i][0], m.tree_quat[i][1], m.tree_quat[i][2], m.tree_quat[i][3]};
                        Quat r = qmul(qp, qt);
                        if (m.jtype[i] == MPPIB_JOINT_REVOLUTE) {
                            float sh, ch; sincos_cw(0.5f * qi, &sh, &ch);
                            const Quat qz = {0.f, 0.f, sh, ch};
                            r = qmul(r, qz);
                        }
                        if (!STORE_FRAMES) { stM3(sm, i * NSLOT + F_OR, lane, f.R); st3(sm, i * NSLOT + F_OO, lane, f.o); st6(sm, i * NSLOT + F_OV, lane, f.V); }
                        SM(i, F_OQ) = r.x; SM(i, F_OQ + 1) = r.y; SM(i, F_OQ + 2) = r.z; SM(i, F_OQ + 3) = r.w;
                        qp = r;
                    }
                    s1_dynamics<NSLOT>(m, sm, lane, i, f, S, qdi);
                    SM(i, F_SAT) = 0.f;
                    if (CHAIN) par = f;
                    if (STORE_FRAMES) { stM3(sm, i * NSLOT + F_R, lane, f.R); st3(sm, i * NSLOT + F_O, lane, f.o); st6(sm, i * NSLOT + F_V, lane, f.V); }
                }
                if (obs_now) { write_obs(pending); pending = -1; }
            }
#pragma unroll 1
            for (int solve = 0; solve < 2; ++solve) {
                // -------------------------------------------------------------- sweep 2: leaves -> root
                if (!CHAIN) {
#pragma unroll 1
                    for (int i = 0; i < nb; ++i) {
                        stSpI(sm, i * NSLOT + F_IA, lane, rigid_inertia(ldS3(sm, i * NSLOT + F_A, lane), ld3(sm, i * NSLOT + F_HW, lane), m.mass[i]));
                        st6(sm, i * NSLOT + F_PA, lane, ld6(sm, i * NSLOT + F_PB, lane));
                    }
                }
                SpI Ic; V6 pc;   // contribution of the child (serial chains)
                bool have_child = false;
                MPPIB_UNROLL(ROLL_UNROLL_S2)
                for (int i = nb - 1; i >= 0; --i) {
                    const V6 S = ld6(sm, i * NSLOT + F_S, lane);
                    SpI IA; V6 pA;
                    if (CHAIN) {
                        IA = rigid_inertia(ldS3(sm, i * NSLOT + F_A, lane), ld3(sm, i * NSLOT + F_HW, lane), m.mass[i]);
                        pA = ld6(sm, i * NSLOT + F_PB, lane);
                        if (have_child) { add_to(IA, Ic); pA.n = pA.n + pc.n; pA.f = pA.f + pc.f; }
                    } else {
                        IA = ldSpI(sm, i * NSLOT + F_IA, lane);
                        pA = ld6(sm, i * NSLOT + F_PA, lane);
                    }
                    // joint force and implicit diagonal: velocity drive kd (q* - qd) and damping b qd act on the NEW velocity
                    const float qdi = SM(i, F_QD), tgt = SM(i, F_TGT), sat = SM(i, F_SAT);
                    const float kd = m.kd[i], b = m.damping[i];
                    float tau, dimp;
                    if (sat != 0.f) { tau = sat * m.effort[i] - b * qdi; dimp = m.armature[i] + h * b; }
                    else if (vel_mode) { tau = kd * (tgt - qdi) - b * qdi; dimp = m.armature[i] + h * (kd + b); }
                    else { tau = fminf(fmaxf(tgt, -m.effort[i]), m.effort[i]) - (kd + b) * qdi; dimp = m.armature[i] + h * (kd + b); }
                    const V6 U = mul(IA, S);
                    const float Dj = dot6(S, U) + dimp;
                    const float invD = __frcp_rn(Dj);
                    if (CONTACT) xs[(L.jv0 + nb + i) * 32 + lane] = __frcp_rn(fmaxf(Dj, 1e-6f));   // joint compliance 1 / D_j of the contact solve
                    const float uu = tau - dot6(S, pA);
                    st6(sm, i * NSLOT + F_U, lane, U);
                    SM(i, F_INVD) = invD; SM(i, F_UU) = uu;
                    const int pi = CHAIN ? i - 1 : m.parent[i];
                    if (pi >= 0) {
                        rank1_sub(IA, U, invD);
                        const V6 c = ld6(sm, i * NSLOT + F_C, lane);
                        const V6 Iac = mul(IA, c);
                        const float s = uu * invD;
                        V6 pa;
                        pa.n = pA.n + Iac.n + s * U.n;
                        pa.f = pA.f + Iac.f + s * U.f;
                        if (CHAIN) { Ic = IA; pc = pa; have_child = true; }
                        else {
                            SpI Ip = ldSpI(sm, pi * NSLOT + F_IA, lane); add_to(Ip, IA); stSpI(sm, pi * NSLOT + F_IA, lane, Ip);
                            V6 pp = ld6(sm, pi * NSLOT + F_PA, lane); pp.n = pp.n + pa.n; pp.f = pp.f + pa.f; st6(sm, pi * NSLOT + F_PA, lane, pp);
                        }
                    }
                }
                // -------------------------------------------------------------- sweep 3: root -> leaves
                V6 ap = a0;
                bool any = false;
                MPPIB_UNROLL(ROLL_UNROLL_S3)
                for (int i = 0; i < nb; ++i) {
                    if (!CHAIN) { const int pi = m.parent[i]; ap = pi >= 0 ? ld6(sm, pi * NSLOT + F_ACC, lane) : a0; }
                    const V6 S = ld6(sm, i * NSLOT + F_S, lane), c = ld6(sm, i * NSLOT + F_C, lane), U = ld6(sm, i * NSLOT + F_U, lane);
                    ap.n = ap.n + c.n; ap.f = ap.f + c.f;
                    const float qdd = (SM(i, F_UU) - dot6(U, ap)) * SM(i, F_INVD);
                    ap.n = ap.n + qdd * S.n; ap.f = ap.f + qdd * S.f;
                    if (!CHAIN) st6(sm, i * NSLOT + F_ACC, lane, ap);
                    SM(i, F_QDD) = qdd;
                    if (solve == 0 && vel_mode) {
                        // drive force limit (URDF <limit effort>): saturated joints are re-solved with a constant torque
                        const float td = m.kd[i] * (SM(i, F_TGT) - (SM(i, F_QD) + h * qdd));
                        if (fabsf(td) > m.effort[i]) { SM(i, F_SAT) = td > 0.f ? 1.f : -1.f; any = true; }
                    }
                }
                if (!any) break;
            }
            if (CONTACT) {
                // ------------------------------------------------------------------ contacts on the predicted velocities
                for (int i = 0; i < nb; ++i) { xs[(L.jv0 + 2 * nb + i) * 32 + lane] = SM(i, F_QD) + h * SM(i, F_QDD); xs[(L.jv0 + i) * 32 + lane] = 0.f; }
                contact::shapes_world<NSLOT>(m, L, sm, xs, lane, base.R, base.o, root0, false);
                const int nc = contact::detect(m, L, xs, lane, s_bmask);
                for (int f = 0; f < m.nfree; ++f) if (m.free_gravity[f]) {
                    const int fb = L.fb0 + f * contact::FBN;
                    xs[(fb + contact::FB_V) * 32 + lane] += h * m.gravity[0]; xs[(fb + contact::FB_V + 1) * 32 + lane] += h * m.gravity[1];
                    xs[(fb + contact::FB_V + 2) * 32 + lane] += h * m.gravity[2];
                }
                contact::solve<NSLOT, CHAIN>(m, L, sm, xs, lane, nc, h);
            }
            // ------------------------------------------------------------------ integrate
            for (int i = 0; i < nb; ++i) {
                float v = CONTACT ? xs[(L.jv0 + 2 * nb + i) * 32 + lane] + xs[(L.jv0 + i) * 32 + lane] : SM(i, F_QD) + h * SM(i, F_QDD);
                v = fminf(fmaxf(v, -m.qd_max[i]), m.qd_max[i]);
                float x = SM(i, F_Q) + h * v;
                if (x < m.q_lo[i]) { x = m.q_lo[i]; if (v < 0.f) v = 0.f; }
                if (x > m.q_hi[i]) { x = m.q_hi[i]; if (v > 0.f) v = 0.f; }
                SM(i, F_Q) = x; SM(i, F_QD) = v;
            }
            if (CONTACT) contact::integrate_free(m, L, xs, lane, h);
        }
        if (obs != nullptr) pending = t;       // observed by the next step's first sweep 1, or by observe_pass() after the loop
    }
    if (pending >= 0) { observe_pass(); write_obs(pending); }
    if (state != nullptr) {
        for (int i = 0; i < nb; ++i) {
            state[(size_t)i * K + k] = SM(i, F_Q);
            state[(size_t)(nb + i) * K + k] = SM(i, F_QD);
        }
        if (CONTACT) for (int f = 0; f < m.nfree; ++f)
            for (int r = 0; r < 13; ++r) state[(size_t)(2 * nb + 13 * f + r) * K + k] = xs[(L.fb0 + f * contact::FBN + r) * 32 + lane];
    }
}

static bool is_chain(const MppibModel& m) {
    for (int i = 0; i < m.nb; ++i) if (m.parent[i] != i - 1) return false;
    return true;
}
static size_t smem_bytes_for(const MppibModel& m, bool chain, bool contact) {
    const int nslot = (chain && !contact) ? NSLOT_CHAIN : NSLOT_TREE;
    const contact::Layout L(m.nb, m.nfree, m.nshapes, m.max_contacts);
    return sizeof(float) * 32 * ((size_t)m.nb * nslot + (contact ? (size_t)L.total : 0) + 2 * (size_t)m.nu);
}

template <bool CHAIN, bool CONTACT>
int launch_t(MppibContext* c, const float* state0, const float* root0, float* state, const float* actions, int t0, int nsteps, float* obs, cudaStream_t s) {
    const int K = c->params.K;
    const size_t smem = smem_bytes_for(c->model, CHAIN, CONTACT);
    MPPIB_REQUIRE(smem <= 226 * 1024, "mppib_rollout: %zu bytes of shared memory per CTA exceed the SM (too many bodies / shapes)", smem);
    static size_t smem_attr[64] = {0};              // per device: the attribute belongs to the function on ONE device
    size_t& attr = smem_attr[c->device & 63];
    if (smem > 48 * 1024 && smem > attr) {
        MPPIB_CHECK_CUDA(cudaFuncSetAttribute(mppib_rollout_kernel<CHAIN, CONTACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    dim3 grid((K + 31) / 32), block(32);
    mppib_rollout_kernel<CHAIN, CONTACT><<<grid, block, smem, s>>>(c->model, c->params, state0, root0, state, actions, t0, nsteps, obs);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

// Which kernel runs a scene.  Serial chains without contacts: one body per lane (rollout_lanes.cu).  Everything else the team kernel
// can take (trees of up to 16 bodies in depth-first order, with or without contacts): a team of lanes per rollout (rollout_team.cu),
// which spreads a rollout over many lanes where this kernel gives it one thread.  The choice does not depend on K, so a shard of a
// multi-GPU job runs the same arithmetic as the single-GPU job (bit-identical rollouts, tests/test_gpu_sizes.py).  The
// thread-per-rollout kernel below remains for scenes the team kernel does not take and as the A/B reference:
// MPPIB_K2_LANES=0 / MPPIB_K2_TEAM=0|1 force a mapping.
int rollout_mapping(const MppibContext* c) {
    const MppibModel& m = c->model;
    if (c->k2_lanes && rollout_lanes_eligible(m)) return MPPIB_MAPPING_LANES;
    if (c->k2_team != 0 && rollout_team_eligible(m)) {
        return MPPIB_MAPPING_TEAM;
    }
    return MPPIB_MAPPING_THREAD;
}

int launch_rollout(MppibContext* c, const float* state0, const float* root0, float* state, const float* actions, int t0, int nsteps,
                   float* obs, cudaStream_t s) {
    const MppibModel& m = c->model;
    const bool chain = is_chain(m);
    const bool contact = m.nfree > 0 || m.nshapes > 0;
    const int mapping = rollout_mapping(c);
    if (mapping == MPPIB_MAPPING_LANES) return launch_rollout_lanes(c, state0, state, actions, t0, nsteps, obs, s);
    if (mapping == MPPIB_MAPPING_TEAM) return launch_rollout_team(c, state0, root0, state, actions, t0, nsteps, obs, s);
    if (contact) {
        MPPIB_REQUIRE(root0 != nullptr, "mppib_rollout: root0 is required for scenes with free bodies / collision boxes");
        if (chain) return launch_t<true, true>(c, state0, root0, state, actions, t0, nsteps, obs, s);
        return launch_t<false, true>(c, state0, root0, state, actions, t0, nsteps, obs, s);
    }
    if (chain) return launch_t<true, false>(c, state0, root0, state, actions, t0, nsteps, obs, s);
    return launch_t<false, false>(c, state0, root0, state, actions, t0, nsteps, obs, s);
}

long long rollout_smem_bytes(const MppibModel& m) { return (long long)smem_bytes_for(m, is_chain(m), m.nfree > 0 || m.nshapes > 0); }
