// rollout_lanes.cu -- K2 for serial chains without contacts (BASELINE C2: panda 7-DoF reach): G LANES PER ROLLOUT, one body
// per lane, 32 / G rollout groups per warp.  Replaces gym.simulate() / IsaacGymWrapper.step on the MPPI path
// (mppiisaac/planner/isaacgym_wrapper.py:524-572 apply_robot_cmd, :639-655 step) exactly like rollout.cu; the two kernels
// implement the same substep (same drive model, same saturation re-solve, same integration) and are tested against the same
// oracle.
//
// Why a second mapping.  rollout.cu gives every rollout one thread; at the headline K = 10 000 that is 313 warps for the 528
// warp schedulers of an H100 (132 SMs x 4), each walking a serial recursion of ~5 400 instructions per substep: the kernel
// time is the latency of ONE warp and 41 % of the schedulers have no warp at all.  Here a rollout is spread
// over G = 8 lanes, so K = 10 000 becomes 2 500 warps of ~1 000 instructions per substep, and a shard of a strong-scaled plan
// (K / 8 per GPU) still occupies every scheduler.
//
// Formulation (world coordinates, spatial vectors about the world origin -- as rollout.cu -- but composite-rigid-body +
// joint-space solve instead of the articulated-body recursion, because every stage of it is either lane-local or a
// log2(G)-round warp-shuffle scan):
//   1. frames        T_i = T_0 o ... o T_i           inclusive scan of (unit quaternion, origin) over the chain
//   2. velocities    V_i = sum_{j<=i} S_j qd_j        prefix sum;   c_i = V_i x S_i qd_i ;  a_i = a_0 + sum_{j<=i} c_j   prefix sum
//   3. per body      world rotational inertia A_i about the origin, first moment hw_i, bias force pb_i, f_i = I_i a_i + pb_i
//   4. composites    (A, hw, f) suffix sums: a composite of rigid bodies is a rigid body, 10 numbers, no 6x6 anywhere
//   5. joint space   F_j = Ic_j S_j ;  M_ij = S_i . F_j (i <= j: lane j owns column j) ;  bias_i = S_i . fc_i
//   6. solve         (M + diag(arm + h (kd + b))) qdd = tau - bias by an LDL^T factorisation DISTRIBUTED over the lanes
//                    (lane j holds row j of L and column j of L; pivots and multipliers travel by shuffle), one
//                    re-factorisation when a velocity drive saturates at the URDF effort limit
//   7. integrate     semi-implicit Euler, velocity and position limits (lane-local)
// All exchanges are __shfl_*_sync with width G: no shared memory, no barriers.
//
// Scalar type F (lanes_math.cuh): float = one rollout per lane group; P2 = two rollouts per lane group (two independent fp32
// instruction streams, control / address instructions shared by the pair); opt-in (MPPIB_K2_PAIRS=1), see launch_rollout_lanes.
#include "common.cuh"
#include "lanes_math.cuh"

namespace {

using namespace lm;

#ifndef LANES_MIN_CTAS
#define LANES_MIN_CTAS 19      // resident 1-warp CTAs per SM the register allocation of the float kernel must allow (K = 10 000 -> 19 per SM at G = 8 on 132 SMs)
#endif
#ifndef LANES_MIN_CTAS_P2
#define LANES_MIN_CTAS_P2 10   // the pair kernel: K = 10 000 -> 1 250 warps = 9.5 per SM
#endif

template <class F> __device__ __forceinline__ F dot6(const V6T<F>& a, const V6T<F>& b) {
    return fma_(a.f.z, b.f.z, fma_(a.f.y, b.f.y, fma_(a.f.x, b.f.x, fma_(a.n.z, b.n.z, fma_(a.n.y, b.n.y, a.n.x * b.n.x)))));
}

// inclusive prefix / suffix sums over the G lanes of a rollout (i = lane within the group)
template <int G, class F> __device__ __forceinline__ void prefix_add(F& x, int i) {
#pragma unroll
    for (int d = 1; d < G; d <<= 1) { const F t = shfl_up<G>(x, d); if (i >= d) x = x + t; }
}
template <int G, class F> __device__ __forceinline__ void suffix_add(F& x, int i) {
#pragma unroll
    for (int d = 1; d < G; d <<= 1) { const F t = shfl_dn<G>(x, d); if (i + d < G) x = x + t; }
}
template <int G, class F> __device__ __forceinline__ void prefix_add3(V3T<F>& v, int i) { prefix_add<G>(v.x, i); prefix_add<G>(v.y, i); prefix_add<G>(v.z, i); }
template <int G, class F> __device__ __forceinline__ void suffix_add3(V3T<F>& v, int i) { suffix_add<G>(v.x, i); suffix_add<G>(v.y, i); suffix_add<G>(v.z, i); }

// world frame of the lane's body and the joint's motion subspace / velocity at the current (q, qd)
template <class F> struct Kin {
    QT<F> qw;       // orientation (xyzw), composed along the chain exactly as the observation wants it
    V3T<F> o;       // origin
    M3T<F> R;       // body axes as columns in the world
    V6T<F> S;       // motion subspace (world, about the origin)
    V6T<F> Vl;      // S qd
    V6T<F> V;       // spatial velocity of the body
};

// per-body model constants: the same for every rollout, plain floats
struct BodyConst {
    float tqx, tqy, tqz, tqw;          // parent -> body(q = 0) rotation
    float tpx, tpy, tpz;               // ... and origin
    float tax, tay, taz;               // prismatic axis in parent coordinates (0 for revolute)
    float jrev;                        // 1 revolute, 0 prismatic
    float mass, mc;                    // mass, mass of the sub-chain from this body on
    float cx, cy, cz;                  // centre of mass, body coordinates
    S3T<float> Ic;                     // rotational inertia about the centre of mass, body coordinates
    float q_lo, q_hi, qd_max, effort, damp, kd, dimp_drive, dimp_sat;
};

template <int G, class F>
__device__ __forceinline__ void kinematics(const BodyConst& bc, int i, F q, F qd, Kin<F>& kn) {
    // local transform: tq * Rz(q) for a revolute joint (half-angle quaternion), origin shifted along the axis for a prismatic one
    F sh, ch;
    sincos_cw(q * (0.5f * bc.jrev), &sh, &ch);
    QT<F> ql;
    ql.x = fma_(ch, bc.tqx, sh * bc.tqy);
    ql.y = fma_(ch, bc.tqy, sh * (-bc.tqx));
    ql.z = fma_(ch, bc.tqz, sh * bc.tqw);
    ql.w = fma_(ch, bc.tqw, sh * (-bc.tqz));
    V3T<F> pl = mk3<F>(fma_(q, bc.tax, bc.tpx), fma_(q, bc.tay, bc.tpy), fma_(q, bc.taz, bc.tpz));
    // inclusive scan of rigid transforms over the chain (Kogge-Stone, log2 G rounds): (qa, pa) o (qb, pb) = (qa qb, pa + qa pb qa*)
#pragma unroll
    for (int d = 1; d < G; d <<= 1) {
        QT<F> qp; V3T<F> pp;
        qp.x = shfl_up<G>(ql.x, d); qp.y = shfl_up<G>(ql.y, d); qp.z = shfl_up<G>(ql.z, d); qp.w = shfl_up<G>(ql.w, d);
        pp.x = shfl_up<G>(pl.x, d); pp.y = shfl_up<G>(pl.y, d); pp.z = shfl_up<G>(pl.z, d);
        if (i >= d) {
            pl = qrot_add(pp, qp, pl);
            ql = qmul(qp, ql);
        }
    }
    kn.qw = ql; kn.o = pl;
    kn.R = quat_to_R(ql);
    const V3T<F> axis = mk3<F>(kn.R.m02, kn.R.m12, kn.R.m22);
    const bool rev = bc.jrev != 0.f;
    const V3T<F> oxa = cross(pl, axis);
    const F zero = bcast<F>(0.f);
    kn.S.n = mk3<F>(sel(rev, axis.x, zero), sel(rev, axis.y, zero), sel(rev, axis.z, zero));
    kn.S.f = mk3<F>(sel(rev, oxa.x, axis.x), sel(rev, oxa.y, axis.y), sel(rev, oxa.z, axis.z));
    kn.Vl.n = scale(qd, kn.S.n); kn.Vl.f = scale(qd, kn.S.f);
    kn.V = kn.Vl;
    prefix_add3<G>(kn.V.n, i); prefix_add3<G>(kn.V.f, i);
}

template <class F> struct bounds_of { static constexpr int MIN_CTAS = LANES_MIN_CTAS; };
template <> struct bounds_of<P2> { static constexpr int MIN_CTAS = LANES_MIN_CTAS_P2; };

// G lanes per rollout (power of two), NB >= nb the compile-time number of joint-space rows (loops over bodies are fully unrolled)
template <int G, int NB, class F>
__global__ void __launch_bounds__(32, bounds_of<F>::MIN_CTAS)
mppib_rollout_lanes_kernel(const __grid_constant__ MppibModel m, const __grid_constant__ MppibParams p,
                           const float* __restrict__ state0, float* __restrict__ state, const float* __restrict__ actions,
                           int t0, int nsteps, float* __restrict__ obs) {
    constexpr int N = scalar_traits<F>::N;          // rollouts per lane group
    constexpr int RPW = 32 / G;                     // lane groups per warp
    const int K = p.K, T = p.T, nu = m.nu, nb = m.nb;
    const int lane = threadIdx.x & 31;
    const int i = lane & (G - 1);                   // body of this lane
    const int k_first = ((int)blockIdx.x * ((int)blockDim.x >> 5) + ((int)threadIdx.x >> 5)) * RPW * N;
    if (k_first >= K) return;                       // warp-uniform
    int kc[N]; bool kval[N];
#pragma unroll
    for (int c = 0; c < N; ++c) {
        kc[c] = k_first + c * RPW + lane / G;       // component c of the warp's groups: RPW consecutive rollouts
        kval[c] = kc[c] < K;                        // lanes of a ragged last warp still take part in every shuffle
        if (!kval[c]) kc[c] = K - 1;
    }
    const bool bval = i < nb;
    const int ib = bval ? i : 0;
    const float h = p.dt / (float)p.substeps;
    const bool vel_mode = m.drive_mode == MPPIB_DRIVE_VELOCITY;

    // ---- per-lane model constants (lanes i >= nb: identity transform, no mass -> neutral in every scan)
    BodyConst bc;
    {
        using Vf = V3T<float>; using Qf = QT<float>;
        Qf tq; tq.x = m.tree_quat[ib][0]; tq.y = m.tree_quat[ib][1]; tq.z = m.tree_quat[ib][2]; tq.w = m.tree_quat[ib][3];
        Vf tp = mk3<float>(m.tree_p[ib][0], m.tree_p[ib][1], m.tree_p[ib][2]);
        bc.jrev = m.jtype[ib] == MPPIB_JOINT_REVOLUTE ? 1.f : 0.f;
        Vf tax = bc.jrev != 0.f ? zero3<float>() : mk3<float>(m.tree_R[ib][2], m.tree_R[ib][5], m.tree_R[ib][8]);
        if (i == 0) {                               // the robot base pose is folded into the first body's parent transform
            Qf bq; bq.x = m.base_quat[0]; bq.y = m.base_quat[1]; bq.z = m.base_quat[2]; bq.w = m.base_quat[3];
            tp = qrot_add(mk3<float>(m.base_pos[0], m.base_pos[1], m.base_pos[2]), bq, tp);
            tax = qrot_add(zero3<float>(), bq, tax);
            tq = qmul(bq, tq);
        }
        bc.mass = m.mass[ib];
        const float inv_m = bc.mass > 0.f ? 1.0f / bc.mass : 0.f;
        const Vf c = mk3<float>(inv_m * m.mcom[ib][0], inv_m * m.mcom[ib][1], inv_m * m.mcom[ib][2]);
        const float mm = bc.mass;
        bc.Ic.xx = m.inertia[ib][0] - mm * (c.y * c.y + c.z * c.z);
        bc.Ic.yy = m.inertia[ib][1] - mm * (c.x * c.x + c.z * c.z);
        bc.Ic.zz = m.inertia[ib][2] - mm * (c.x * c.x + c.y * c.y);
        bc.Ic.xy = m.inertia[ib][3] + mm * c.x * c.y;
        bc.Ic.xz = m.inertia[ib][4] + mm * c.x * c.z;
        bc.Ic.yz = m.inertia[ib][5] + mm * c.y * c.z;
        bc.q_lo = m.q_lo[ib]; bc.q_hi = m.q_hi[ib]; bc.qd_max = m.qd_max[ib]; bc.effort = m.effort[ib];
        bc.damp = m.damping[ib]; bc.kd = m.kd[ib];
        bc.dimp_drive = m.armature[ib] + h * (bc.kd + bc.damp);
        bc.dimp_sat = m.armature[ib] + h * bc.damp;
        bc.tqx = tq.x; bc.tqy = tq.y; bc.tqz = tq.z; bc.tqw = tq.w; bc.tpx = tp.x; bc.tpy = tp.y; bc.tpz = tp.z;
        bc.tax = tax.x; bc.tay = tax.y; bc.taz = tax.z; bc.cx = c.x; bc.cy = c.y; bc.cz = c.z;
        if (!bval) {
            bc.tqx = 0.f; bc.tqy = 0.f; bc.tqz = 0.f; bc.tqw = 1.f; bc.tpx = bc.tpy = bc.tpz = 0.f; bc.tax = bc.tay = bc.taz = 0.f; bc.jrev = 0.f;
            bc.mass = 0.f; bc.cx = bc.cy = bc.cz = 0.f;
            bc.Ic.xx = bc.Ic.yy = bc.Ic.zz = bc.Ic.xy = bc.Ic.xz = bc.Ic.yz = 0.f;
            bc.dimp_drive = 1.f; bc.dimp_sat = 1.f; bc.kd = 0.f; bc.damp = 0.f; bc.effort = 3.0e38f; bc.qd_max = 0.f; bc.q_lo = 0.f; bc.q_hi = 0.f;
        }
        bc.mc = bc.mass;
        suffix_add<G>(bc.mc, i);
    }
    const int ci0 = m.cmd_i0[ib], ci1 = m.cmd_i1[ib];
    const float cc0 = bval ? p.u_scale * m.cmd_c0[ib] : 0.f, cc1 = bval ? p.u_scale * m.cmd_c1[ib] : 0.f;
    // gravity enters as a fictitious base acceleration a0 = [0; -g]
    const float a0x = m.gravity_on ? -m.gravity[0] : 0.f, a0y = m.gravity_on ? -m.gravity[1] : 0.f, a0z = m.gravity_on ? -m.gravity[2] : 0.f;

    F q = bcast<F>(0.f), qd = bcast<F>(0.f);
    if (bval) {
#pragma unroll
        for (int c = 0; c < N; ++c) {
            set_comp(q, c, state0 ? state0[i] : state[(size_t)i * K + kc[c]]);
            set_comp(qd, c, state0 ? state0[nb + i] : state[(size_t)(nb + i) * K + kc[c]]);
        }
    }

    // write the observed rows of model step `t` from the frames of the CURRENT state (isaacgym_wrapper.py:186-199 layouts)
    auto write_obs = [&](int t, const Kin<F>& kn) {
        const size_t TK = (size_t)T * K;
        int row = 0;
        for (int oi = 0; oi < p.nobs; ++oi) {
            const int kind = p.obs[oi].kind, idx = p.obs[oi].index;
            if (kind == MPPIB_OBS_LINK_STATE) {
                const int b = m.link_body[idx];
                if (b >= 0 ? i == b : i == 0) {
                    V3T<F> ol, w, vO; QT<F> qb; M3T<F> Rl;
                    if (b >= 0) { Rl = kn.R; ol = kn.o; w = kn.V.n; vO = kn.V.f; qb = kn.qw; }
                    else {
                        qb.x = bcast<F>(m.base_quat[0]); qb.y = bcast<F>(m.base_quat[1]); qb.z = bcast<F>(m.base_quat[2]); qb.w = bcast<F>(m.base_quat[3]);
                        Rl = quat_to_R(qb);
                        ol = mk3<F>(bcast<F>(m.base_pos[0]), bcast<F>(m.base_pos[1]), bcast<F>(m.base_pos[2]));
                        w = zero3<F>(); vO = zero3<F>();
                    }
                    const V3T<F> pos = ol + mulc(Rl, m.link_p[idx][0], m.link_p[idx][1], m.link_p[idx][2]);
                    QT<F> qlk; qlk.x = bcast<F>(m.link_quat[idx][0]); qlk.y = bcast<F>(m.link_quat[idx][1]); qlk.z = bcast<F>(m.link_quat[idx][2]); qlk.w = bcast<F>(m.link_quat[idx][3]);
                    const QT<F> qo = qmul(qb, qlk);
                    const V3T<F> vel = cross_add(vO, w, pos);   // spatial velocity about the world origin -> velocity of the link origin
                    const F vals[13] = {pos.x, pos.y, pos.z, qo.x, qo.y, qo.z, qo.w, vel.x, vel.y, vel.z, w.x, w.y, w.z};
#pragma unroll
                    for (int c = 0; c < N; ++c) {
                        if (!kval[c]) continue;
                        float* dst = obs + (size_t)t * K + kc[c];
#pragma unroll
                        for (int r = 0; r < 13; ++r) dst[(size_t)(row + r) * TK] = comp(vals[r], c);
                    }
                }
                row += 13;
            } else if (kind == MPPIB_OBS_DOF_STATE) {
                if (bval) {
#pragma unroll
                    for (int c = 0; c < N; ++c) {
                        if (!kval[c]) continue;
                        float* dst = obs + (size_t)t * K + kc[c];
                        dst[(size_t)(row + 2 * i) * TK] = comp(q, c);
                        dst[(size_t)(row + 2 * i + 1) * TK] = comp(qd, c);
                    }
                }
                row += 2 * nb;
            } else {
                // free bodies / contact forces do not exist in a contact-free scene: zeros, as rollout.cu writes them
                const int wdt = kind == MPPIB_OBS_FREE_STATE ? 13 : 3;
                if (i == 0) {
#pragma unroll
                    for (int c = 0; c < N; ++c) {
                        if (!kval[c]) continue;
                        float* dst = obs + (size_t)t * K + kc[c];
                        for (int r = 0; r < wdt; ++r) dst[(size_t)(row + r) * TK] = 0.f;
                    }
                }
                row += wdt;
            }
        }
    };

    int pending = (obs != nullptr && nsteps == 0) ? t0 : -1;   // step whose observation is still to be written
    // the two command values of step t + 1 are loaded while step t integrates (the load is consumed one model step later)
    F u0n = bcast<F>(0.f), u1n = bcast<F>(0.f);
    auto load_u = [&](int t) {
#pragma unroll
        for (int c = 0; c < N; ++c) {
            set_comp(u0n, c, __ldg(&actions[((size_t)t * nu + ci0) * K + kc[c]]));
            set_comp(u1n, c, __ldg(&actions[((size_t)t * nu + ci1) * K + kc[c]]));
        }
    };
    if (nsteps > 0) load_u(t0);
    const int nsub = p.substeps;
#pragma unroll 1
    for (int t = t0; t < t0 + nsteps; ++t) {
        // apply_robot_cmd: command -> per-DOF target (the DOF map of isaacgym_wrapper.py:524-572 is a 2-term linear map per DOF)
        const F tgt = fma_(u0n, cc0, u1n * cc1);
        if (t + 1 < t0 + nsteps) load_u(t + 1);
#pragma unroll 1
        for (int sub = 0; sub < nsub; ++sub) {
            Kin<F> kn;
            kinematics<G>(bc, i, q, qd, kn);
            if (sub == 0 && pending >= 0) { write_obs(pending, kn); pending = -1; }   // these frames ARE the observation of the previous step
            // ---- per-body terms about the world origin
            const V3T<F> cw = kn.o + mulc(kn.R, bc.cx, bc.cy, bc.cz);
            const V3T<F> hw = scale(bc.mass, cw);
            S3T<F> A;
            {
                const V3T<F> r0 = mk3<F>(kn.R.m00, kn.R.m01, kn.R.m02), r1 = mk3<F>(kn.R.m10, kn.R.m11, kn.R.m12), r2 = mk3<F>(kn.R.m20, kn.R.m21, kn.R.m22);
                const V3T<F> t0v = mul(bc.Ic, r0), t1v = mul(bc.Ic, r1), t2v = mul(bc.Ic, r2);
                const F d2 = dot(hw, cw);
                A.xx = fma_(-hw.x, cw.x, d2 + dot(r0, t0v)); A.yy = fma_(-hw.y, cw.y, d2 + dot(r1, t1v)); A.zz = fma_(-hw.z, cw.z, d2 + dot(r2, t2v));
                A.xy = fma_(-hw.x, cw.y, dot(r0, t1v)); A.xz = fma_(-hw.x, cw.z, dot(r0, t2v)); A.yz = fma_(-hw.y, cw.z, dot(r1, t2v));
            }
            const V3T<F> w = kn.V.n, v = kn.V.f;
            V6T<F> fb;   // bias force V x* (I V), then + I a
            {
                const V3T<F> nn = cross_add(mul(A, w), hw, v);
                const V3T<F> ff = cross_add(scale(bc.mass, v), w, hw);      // m v - hw x w
                fb.n = cross_add(cross(w, nn), v, ff);
                fb.f = cross(w, ff);
            }
            // velocity-product acceleration c = V x (S qd), accumulated down the chain on top of the gravity term
            V6T<F> a;
            a.n = cross(w, kn.Vl.n);
            a.f = cross_add(cross(w, kn.Vl.f), v, kn.Vl.n);
            prefix_add3<G>(a.n, i); prefix_add3<G>(a.f, i);
            a.f = mk3<F>(a.f.x + a0x, a.f.y + a0y, a.f.z + a0z);
            fb.n = cross_add(mul_add(fb.n, A, a.n), hw, a.f);
            fb.f = cross_add(mk3<F>(fma_(a.f.x, bc.mass, fb.f.x), fma_(a.f.y, bc.mass, fb.f.y), fma_(a.f.z, bc.mass, fb.f.z)), a.n, hw);   // + m a.f - hw x a.n
            // ---- composites: suffix sums of (A, hw, f); the composite mass is a model constant
            suffix_add<G>(A.xx, i); suffix_add<G>(A.yy, i); suffix_add<G>(A.zz, i); suffix_add<G>(A.xy, i); suffix_add<G>(A.xz, i); suffix_add<G>(A.yz, i);
            V3T<F> hc = hw;
            suffix_add3<G>(hc, i);
            suffix_add3<G>(fb.n, i); suffix_add3<G>(fb.f, i);
            V6T<F> Fj;    // Ic S
            Fj.n = cross_add(mul(A, kn.S.n), hc, kn.S.f);
            Fj.f = cross_add(scale(bc.mc, kn.S.f), kn.S.n, hc);              // mc S.f - hc x S.n
            const F bias = dot6(kn.S, fb);
            // ---- joint-space inertia: lane j owns column j (rows i <= j are the valid ones)
            F mcol[NB];
#pragma unroll
            for (int r = 0; r < NB; ++r) {
                V6T<F> Sr;
                Sr.n.x = shfl_at<G>(kn.S.n.x, r); Sr.n.y = shfl_at<G>(kn.S.n.y, r); Sr.n.z = shfl_at<G>(kn.S.n.z, r);
                Sr.f.x = shfl_at<G>(kn.S.f.x, r); Sr.f.y = shfl_at<G>(kn.S.f.y, r); Sr.f.z = shfl_at<G>(kn.S.f.z, r);
                mcol[r] = dot6(Sr, Fj);
            }
            // ---- solve (M + diag(dimp)) qdd = tau - bias ; joint force and implicit diagonal: the velocity drive kd (q* - qd) and
            // the joint damping b qd act on the NEW velocity.  LDL^T, right looking, with the forward substitution folded into
            // the pivot loop: at pivot kk every lane j > kk knows l_jk (its row of L), lane kk collects column kk of L in lcol[]
            // for the backward substitution.  Bodies i >= nb are an identity block (no mass, unit diagonal): no guards needed.
            F sat = bcast<F>(0.f), qdd = bcast<F>(0.f);
#pragma unroll 1
            for (int solve = 0; solve < 2; ++solve) {
                F tau, dimp;
                const F dqd = qd * bc.damp;
                if (vel_mode) tau = fma_(tgt - qd, bc.kd, -dqd);
                else tau = fma_(qd, -bc.kd, clampf(tgt, -bc.effort, bc.effort) - dqd);
                dimp = bcast<F>(bc.dimp_drive);
                if (solve == 1) {
#pragma unroll
                    for (int c = 0; c < N; ++c) {
                        const float s = comp(sat, c);
                        if (s != 0.f) { set_comp(tau, c, s * bc.effort - comp(dqd, c)); set_comp(dimp, c, bc.dimp_sat); }
                    }
                }
                F col[NB], lcol[NB];
#pragma unroll
                for (int r = 0; r < NB; ++r) { col[r] = mcol[r]; lcol[r] = bcast<F>(0.f); }
                F invd = bcast<F>(1.f);
                F y = tau - bias;
#pragma unroll
                for (int kk = 0; kk < NB; ++kk) {
                    const F dk = shfl_at<G>(col[kk] + dimp, kk);         // only lane kk's sum (its diagonal + implicit term) is read
                    const F inv = rcp_approx(dk);
                    const bool own = i == kk;
                    if (own) invd = inv;
                    const F lk = col[kk] * inv;                          // l_jk on lanes j > kk
                    if (kk + 1 < NB) {
                        const F yk = shfl_at<G>(y, kk);                  // y_kk is final
                        if (i > kk) y = fma_(-lk, yk, y);
                    }
#pragma unroll
                    for (int r = kk + 1; r < NB; ++r) {
                        const F lr = shfl_at<G>(lk, r);
                        col[r] = fma_(-lr, col[kk], col[r]);
                        if (own) lcol[r] = lr;
                    }
                }
                y = y * invd;
#pragma unroll
                for (int jj = NB - 1; jj >= 1; --jj) {
                    const F xj = shfl_at<G>(y, jj);
                    if (i < jj) y = fma_(-lcol[jj], xj, y);
                }
                qdd = bval ? y : bcast<F>(0.f);
                bool newly = false;
                if (solve == 0 && vel_mode && bval) {
                    // drive force limit (URDF <limit effort>): saturated joints are re-solved with a constant torque
                    const F td = (tgt - fma_(qdd, h, qd)) * bc.kd;
#pragma unroll
                    for (int c = 0; c < N; ++c) {
                        const float tdc = comp(td, c);
                        if (fabsf(tdc) > bc.effort) { set_comp(sat, c, tdc > 0.f ? 1.f : -1.f); newly = true; }
                    }
                }
                if (!__any_sync(FULL, newly)) break;
            }
            // ---- integrate: semi-implicit Euler, velocity limit, position limits as inelastic stops
            {
                F vn = clampf(fma_(qdd, h, qd), -bc.qd_max, bc.qd_max);
                F x = fma_(vn, h, q);
#pragma unroll
                for (int c = 0; c < N; ++c) {
                    float xc = comp(x, c), vc = comp(vn, c);
                    if (xc < bc.q_lo) { xc = bc.q_lo; if (vc < 0.f) vc = 0.f; }
                    if (xc > bc.q_hi) { xc = bc.q_hi; if (vc > 0.f) vc = 0.f; }
                    set_comp(x, c, xc); set_comp(vn, c, vc);
                }
                if (bval) { q = x; qd = vn; }
            }
        }
        if (obs != nullptr) pending = t;       // observed by the next step's first kinematics pass, or by the pass after the loop
    }
    if (pending >= 0) {
        Kin<F> kn;
        kinematics<G>(bc, i, q, qd, kn);
        write_obs(pending, kn);
    }
    if (state != nullptr && bval) {
#pragma unroll
        for (int c = 0; c < N; ++c) {
            if (!kval[c]) continue;
            state[(size_t)i * K + kc[c]] = comp(q, c);
            state[(size_t)(nb + i) * K + kc[c]] = comp(qd, c);
        }
    }
}

template <int G, int NB, class F>
int launch_lanes_t(MppibContext* c, const float* state0, float* state, const float* actions, int t0, int nsteps, float* obs, cudaStream_t s) {
    const int K = c->params.K;
    constexpr int RPW = (32 / G) * scalar_traits<F>::N;
    const int warps = (K + RPW - 1) / RPW;
    mppib_rollout_lanes_kernel<G, NB, F><<<warps, 32, 0, s>>>(c->model, c->params, state0, state, actions, t0, nsteps, obs);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <class F>
int launch_lanes_f(MppibContext* c, const float* state0, float* state, const float* actions, int t0, int nsteps, float* obs, cudaStream_t s) {
    const int nb = c->model.nb;
    if (nb <= 3) return launch_lanes_t<4, 3, F>(c, state0, state, actions, t0, nsteps, obs, s);
    if (nb <= 4) return launch_lanes_t<4, 4, F>(c, state0, state, actions, t0, nsteps, obs, s);
    if (nb <= 7) return launch_lanes_t<8, 7, F>(c, state0, state, actions, t0, nsteps, obs, s);
    return launch_lanes_t<8, 8, F>(c, state0, state, actions, t0, nsteps, obs, s);
}

}  // namespace

// serial chain on a fixed base, no free bodies / collision shapes, at most 8 bodies
bool rollout_lanes_eligible(const MppibModel& m) {
    if (m.nfree > 0 || m.nshapes > 0 || m.planar_base || m.nb > 8) return false;
    for (int i = 0; i < m.nb; ++i) if (m.parent[i] != i - 1) return false;
    return true;
}

int launch_rollout_lanes(MppibContext* c, const float* state0, float* state, const float* actions, int t0, int nsteps, float* obs, cudaStream_t s) {
    // One rollout per lane group by default.  The pair instantiation (two rollouts per group) shares the control and address
    // instructions of the pair but needs about twice the registers per lane; it stays selectable (MPPIB_K2_PAIRS=1) for A/B runs.
    bool packed = c->k2_pairs > 0;
    if (packed) return launch_lanes_f<lm::P2>(c, state0, state, actions, t0, nsteps, obs, s);
    return launch_lanes_f<float>(c, state0, state, actions, t0, nsteps, obs, s);
}
