// rollout_team.cu -- K2 for TREES and for every scene WITH CONTACTS: a TEAM of lanes per rollout.  Replaces gym.simulate() /
// IsaacGymWrapper.step on the MPPI path (mppiisaac/planner/isaacgym_wrapper.py:524-572, :639-655) for the scenes rollout_lanes.cu does
// not cover: panda + gripper, omnipanda, the planar differential-drive bases (boxer, albert, jackal), and BASELINE C3 / C4 / C5
// (boxer_push, heijn_push, panda_pick).  Same spec as rollout.cu + contact.cuh (the thread-per-rollout kernel, kept for scenes outside
// this kernel's limits and as the A/B reference: MPPIB_K2_TEAM=0) and as oracle/oracle.cpp; tested against the same oracle under
// both mappings (tests/test_gpu_mappings.py).  The contact model (randomisation, shape poses, broad phase, box and sphere contacts,
// tangents, free-body integration) is contact_model.cuh, shared with the thread-per-rollout kernel and compiled here with this
// kernel's algebra (lanes_math.cuh); the lane mapping, the contact records and the Gauss-Seidel solve are this file's own.
//
// Why.  The thread-per-rollout contact kernels are ONE warp per SM walking a data-dependent stream of 23 - 32 k instructions per
// (sub)step: at the BASELINE shard sizes every CTA is resident at once, so their time is the latency of a single warp, and most of
// the machine idles.  Here:
//   * ARTICULATION PHASE, G = 8 / 16 lanes per rollout, one body per lane: the composite-rigid-body / joint-space LDL^T formulation of
//     rollout_lanes.cu generalised to trees (ancestor sums by pointer jumping, subtree sums as differences of suffix sums in depth-first
//     order, leaves-first elimination so that the pivots are the articulated-body diagonals D_j);
//   * CONTACT PHASE, GC = 8 lanes per rollout (4 rollouts per warp): lane = shape / candidate partner / sample point in detection
//     (contacts appended in the oracle's order by ballot + prefix popcount), lane = generalised coordinate in the Gauss-Seidel sweeps
//     (the joints, and per free body 3 linear + 3 body-axis angular velocity components: one scalar inverse inertia each, one number
//     per coordinate and contact row, one butterfly all-reduce per visit).
// Per-rollout data of the contact phase lives in shared memory, one contiguous block per rollout (TLayout: free bodies, world shapes,
// contact records, net forces, contact rows, and the joint block through which the two phases talk): 1.3 - 2 k floats, 7 - 8 one-warp
// CTAs per SM (the thread-per-rollout kernel: 1.3 - 1.8 k slots x 32 lanes = one CTA per SM).  Per-body data of the articulation
// phase (q, qd, frame, motion subspace) stays in the registers of the body's lane.
#include "common.cuh"
#include "lanes_math.cuh"

namespace {

using namespace lm;

__device__ __forceinline__ V3 mk(float x, float y, float z) { return mk3(x, y, z); }
__device__ __forceinline__ float dot6(const V6& a, const V6& b) { return dot(a.n, b.n) + dot(a.f, b.f); }
// the names contact_model.cuh writes its arithmetic with
__device__ __forceinline__ V3 mul(const M3& m, V3 v) { return mulc(m, v.x, v.y, v.z); }
__device__ __forceinline__ V3 mulT(const M3& m, V3 v) {
    return mk(m.m00 * v.x + m.m10 * v.y + m.m20 * v.z, m.m01 * v.x + m.m11 * v.y + m.m21 * v.z, m.m02 * v.x + m.m12 * v.y + m.m22 * v.z);
}

#include "contact_model.cuh"
using namespace contact;

// ---- shared-memory layout of ONE rollout (floats): the free-body and shape records of contact_model.cuh, then
// contact records in 16-byte groups: [ln lt1 lt2 mu] the state of the sweeps | [bias 1/(kn+gamma) 1/kt1 1/kt2] their constants | [p ids]
// [n -] and, in the roomy layout, [t1 -] (compact: the tangents are recomputed from n, tangents()).
// Two layouts of the per-rollout block.  ROOMY (robots of up to 8 joints): 20-float contact records, contact rows as one float4 per
// coordinate -- one LDS.128 per coordinate slot and visit; these kernels run latency-bound with every CTA resident.  COMPACT (9 - 16
// joints, e.g. panda_pick: 15 coordinates x 24 contacts of rows): 16-float records, rows as three planes of floats -- 20 % less shared
// memory per rollout = 7 instead of 5 resident CTAs per SM; the roomy layout is the faster one per CTA for the small robots, which take
// the compact one only where it saves a wave of CTAs (launch_team_contact).
enum : int { CT_LN = 0, CT_LT1 = 1, CT_LT2 = 2, CT_MU = 3, CT_D = 4, CT_KN = 5, CT_KT1 = 6, CT_KT2 = 7, CT_P = 8, CT_IDS = 11, CT_N = 12, CT_T1 = 16 };
enum : int { JB_R = 0, JB_O = 9, JB_SN = 12, JB_SF = 15, JB_VP = 18, JB_INVD = 19, JBN = 20 };
constexpr int MAXS_ALL = 5;                 // generalised coordinates per lane in the contact solve: nb + 6 nfree <= G + 24 over G >= 8 lanes
struct TLayout {
    int fb0, sh0, ct0, net0, rw0, jb0, ncs, ctn, total;
    // rw0: contact rows [contact][n, t1, t2][coordinate];  ncs: coordinate slots per lane = ceil((nb + 6 nfree) / GC);
    // jb0: what the articulation phase hands to the contact phase and back, per body: frame, motion subspace, predicted velocity, 1 / D_j
    __host__ __device__ TLayout(int nb, int nfree, int nshapes, int max_contacts, int GC, bool compact) {
        ctn = compact ? 16 : 20;
        fb0 = 0; sh0 = fb0 + nfree * FBN; ct0 = (sh0 + nshapes * SHN + 3) & ~3; net0 = ct0 + max_contacts * ctn; rw0 = net0 + 3 * MPPIB_MAX_SLOTS;
        ncs = (nb + 6 * nfree + GC - 1) / GC;
        jb0 = (rw0 + max_contacts * (nb + 6 * nfree) * (compact ? 3 : 4) + 3) & ~3;
        total = jb0 + nb * JBN;
    }
};
__host__ __device__ inline int team_stride(int total, int G) { return ((total + 31) & ~31) + G; }   // stride % 32 == G: the teams of a warp start G banks apart

__device__ __forceinline__ V3 ld3(const float* xs, int b) { return mk(xs[b], xs[b + 1], xs[b + 2]); }
__device__ __forceinline__ void st3(float* xs, int b, V3 v) { xs[b] = v.x; xs[b + 1] = v.y; xs[b + 2] = v.z; }
__device__ __forceinline__ M3 ldM3(const float* xs, int b) {
    M3 m; m.m00 = xs[b]; m.m01 = xs[b + 1]; m.m02 = xs[b + 2]; m.m10 = xs[b + 3]; m.m11 = xs[b + 4]; m.m12 = xs[b + 5]; m.m20 = xs[b + 6]; m.m21 = xs[b + 7]; m.m22 = xs[b + 8]; return m;
}
__device__ __forceinline__ void stM3(float* xs, int b, const M3& m) {
    xs[b] = m.m00; xs[b + 1] = m.m01; xs[b + 2] = m.m02; xs[b + 3] = m.m10; xs[b + 4] = m.m11; xs[b + 5] = m.m12; xs[b + 6] = m.m20; xs[b + 7] = m.m21; xs[b + 8] = m.m22;
}

// team-wide helpers: G lanes, lane-in-team i, `tb` = first lane of the team in the warp
// The teams of a warp see different numbers of contacts, but the control flow of the contact phase is kept WARP-UNIFORM: loops run to the
// largest trip count among the teams of the warp and a team past its own count is predicated off.  (The teams of a warp wait for each
// other at the next full-warp shuffle anyway; with team-divergent loops every shuffle would need the team's lane mask in a register,
// which costs a MATCH / REDUX / VOTE convergence check per shuffle group -- 8 of the 83 instructions of a Gauss-Seidel visit.)
template <int G> __device__ __forceinline__ float team_sum(float v) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o, G);
    return v;
}
template <int G> __device__ __forceinline__ uint32_t team_ballot(bool pred, int tb) { return (__ballot_sync(FULL, pred) >> tb) & (G == 32 ? 0xffffffffu : ((1u << G) - 1u)); }
// the team bits of a warp ballot OR-ed over the teams of the warp
template <int G> __device__ __forceinline__ uint32_t union_ballot(bool pred) {
    uint32_t u = __ballot_sync(FULL, pred);
    if (G <= 16) u |= u >> 16;
    if (G <= 8) u |= u >> 8;
    if (G <= 4) u |= u >> 4;
    return u & (G == 32 ? 0xffffffffu : ((1u << G) - 1u));
}

struct BodyConst {
    float tqx, tqy, tqz, tqw, tpx, tpy, tpz, tax, tay, taz, jrev;
    float mass, cx, cy, cz;
    S3 Ic;
    float q_lo, q_hi, qd_max, effort, damp, kd, dimp_drive, dimp_sat;
};

struct Kin { Quat qw; V3 o; M3 R; V6 S, Vl, V; };

// per-lane tree tables
template <int R> struct Tree {
    int jump[R];        // ancestor at distance 2^r (lane in team), -1 none
    uint32_t anc;       // bit j set: body j is this body or an ancestor of it
    uint32_t desc;      // bit j set: body j is this body or a descendant
    int end;            // first body after this body's subtree (depth-first numbering: the subtree is [i, end))
};

template <int G, int R>
__device__ __forceinline__ void anc_add(float& x, const Tree<R>& tr) {
#pragma unroll
    for (int r = 0; r < R; ++r) { const float t = shfl_at<G>(x, tr.jump[r] >= 0 ? tr.jump[r] : 0); if (tr.jump[r] >= 0) x += t; }
}
template <int G, int R> __device__ __forceinline__ void anc_add3(V3& v, const Tree<R>& tr) { anc_add<G, R>(v.x, tr); anc_add<G, R>(v.y, tr); anc_add<G, R>(v.z, tr); }
// sum over the subtree = suffix sum over the depth-first order minus the suffix sum at the subtree's end
template <int G, int R>
__device__ __forceinline__ void subtree_add(float& x, int i, const Tree<R>& tr) {
#pragma unroll
    for (int d = 1; d < G; d <<= 1) { const float t = shfl_dn<G>(x, d); if (i + d < G) x += t; }
    const float e = shfl_at<G>(x, tr.end < G ? tr.end : 0);
    if (tr.end < G) x -= e;
}
template <int G, int R> __device__ __forceinline__ void subtree_add3(V3& v, int i, const Tree<R>& tr) { subtree_add<G, R>(v.x, i, tr); subtree_add<G, R>(v.y, i, tr); subtree_add<G, R>(v.z, i, tr); }

template <int G, int R>
__device__ __forceinline__ void kinematics(const BodyConst& bc, const Tree<R>& tr, float q, float qd, Kin& kn) {
    float sh, ch;
    sincos_cw(q * (0.5f * bc.jrev), &sh, &ch);
    Quat ql;
    ql.x = fmaf(ch, bc.tqx, sh * bc.tqy);
    ql.y = fmaf(ch, bc.tqy, sh * (-bc.tqx));
    ql.z = fmaf(ch, bc.tqz, sh * bc.tqw);
    ql.w = fmaf(ch, bc.tqw, sh * (-bc.tqz));
    V3 pl = mk(fmaf(q, bc.tax, bc.tpx), fmaf(q, bc.tay, bc.tpy), fmaf(q, bc.taz, bc.tpz));
    // world frame = product of the local transforms along the path from the root: pointer jumping over the ancestors
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int src = tr.jump[r] >= 0 ? tr.jump[r] : 0;
        Quat qp; V3 pp;
        qp.x = shfl_at<G>(ql.x, src); qp.y = shfl_at<G>(ql.y, src); qp.z = shfl_at<G>(ql.z, src); qp.w = shfl_at<G>(ql.w, src);
        pp.x = shfl_at<G>(pl.x, src); pp.y = shfl_at<G>(pl.y, src); pp.z = shfl_at<G>(pl.z, src);
        if (tr.jump[r] >= 0) {
            pl = qrot_add(pp, qp, pl);
            ql = qmul(qp, ql);
        }
    }
    kn.qw = ql; kn.o = pl;
    kn.R = quat_to_R(ql);
    const V3 axis = mk(kn.R.m02, kn.R.m12, kn.R.m22);
    const bool rev = bc.jrev != 0.f;
    const V3 oxa = cross(pl, axis);
    kn.S.n = rev ? axis : mk(0.f, 0.f, 0.f);
    kn.S.f = rev ? oxa : axis;
    kn.Vl.n = scale(qd, kn.S.n); kn.Vl.f = scale(qd, kn.S.f);
    kn.V = kn.Vl;
    anc_add3<G, R>(kn.V.n, tr); anc_add3<G, R>(kn.V.f, tr);
}

// G lanes per rollout in the ARTICULATION phase (one body per lane), NB >= nb joint-space rows (compile time); CONTACT: free bodies /
// collision shapes present -> the CONTACT phase runs with GC <= G lanes per rollout over NCS coordinate slots per lane.  A warp owns
// RPW = 32 / GC rollouts; with GC < G (the 9-joint panda_pick scene: G = 16, GC = 8) the articulation runs in G / GC passes over them --
// it is a few per cent of the work -- so that the Gauss-Seidel sweeps, which are 3/4 of the work and whose cost per visit hardly depends
// on the team width, serve four rollouts per warp instead of two.  The two phases talk through the joint block in shared memory.
template <int G, int NB, bool CONTACT, int NCS, int GC, bool COMPACT>
__global__ void __launch_bounds__(32, (CONTACT && G > 8) ? 8 : 12)   // 9 - 16 joint contact kernels: shared memory allows 7 CTAs per SM -> up to 255 registers, no spills
mppib_rollout_team_kernel(const __grid_constant__ MppibModel m, const __grid_constant__ MppibParams p,
                          const float* __restrict__ state0, const float* __restrict__ root0, float* __restrict__ state,
                          const float* __restrict__ actions, int t0, int nsteps, float* __restrict__ obs) {
    constexpr int RPW = 32 / GC;                                 // rollouts per warp
    constexpr int NP = G / GC;                                   // articulation passes
    constexpr int APP = 32 / G;                                  // rollouts per articulation pass
    constexpr int R = (G == 16) ? 4 : ((G == 8) ? 3 : 2);        // rounds of pointer jumping: depth < 2^R
    extern __shared__ float4 sm_all4[];
    float* sm_all = reinterpret_cast<float*>(sm_all4);
    __shared__ uint32_t s_bmask[MPPIB_MAX_SHAPES];               // candidate partners of every shape
    __shared__ uint32_t s_anc[MPPIB_MAX_BODIES];                 // ancestor-or-self mask of every body (the chain of a contact's link)
    __shared__ uint8_t s_link[MPPIB_MAX_SHAPES];                 // the collision shapes of moving links, ascending
    const int K = p.K, T = p.T, nu = m.nu, nb = m.nb;
    const int lane = threadIdx.x & 31;
    const int i = lane & (G - 1);                                // articulation phase: body of this lane
    const int team = lane / G;
    const int k_first = (int)blockIdx.x * RPW;
    if (k_first >= K) return;
    constexpr int CTN = COMPACT ? 16 : 20;
    const TLayout L(nb, m.nfree, m.nshapes, m.max_contacts, GC, COMPACT);
    const int xstride = team_stride(L.total, GC);
    int ka[NP]; bool kvala[NP]; float* xsa[NP];                  // rollout of this lane in articulation pass pp, its shared-memory block
#pragma unroll
    for (int pp = 0; pp < NP; ++pp) {
        const int r = pp * APP + team;
        ka[pp] = k_first + r; kvala[pp] = ka[pp] < K;
        if (!kvala[pp]) ka[pp] = K - 1;
        xsa[pp] = sm_all + (size_t)r * xstride;
    }
    // contact phase: GC lanes per rollout
    const int ic = lane & (GC - 1);
    const int tbc = (lane / GC) * GC;
    int kc = k_first + lane / GC;
    const bool kvalc = kc < K;
    if (!kvalc) kc = K - 1;
    float* xs = sm_all + (size_t)(lane / GC) * xstride;
    const bool bval = i < nb;
    const int ib = bval ? i : 0;
    const float h = p.dt / (float)p.substeps;
    const bool vel_mode = m.drive_mode == MPPIB_DRIVE_VELOCITY;

    // ---- tree tables
    Tree<R> tr;
    {
        const int par = bval ? m.parent[ib] : -1;
        tr.jump[0] = par;
#pragma unroll
        for (int r = 1; r < R; ++r) {
            const int up = __shfl_sync(FULL, tr.jump[r - 1], tr.jump[r - 1] >= 0 ? tr.jump[r - 1] : 0, G);
            tr.jump[r] = tr.jump[r - 1] >= 0 ? up : -1;
        }
        uint32_t anc = bval ? (1u << i) : 0u;
#pragma unroll
        for (int r = 0; r < R; ++r) { const uint32_t t = __shfl_sync(FULL, anc, tr.jump[r] >= 0 ? tr.jump[r] : 0, G); if (tr.jump[r] >= 0) anc |= t; }
        tr.anc = anc;
        uint32_t desc = 0;
#pragma unroll
        for (int j = 0; j < G; ++j) { const uint32_t aj = __shfl_sync(FULL, anc, j, G); if (bval && ((aj >> i) & 1u)) desc |= 1u << j; }
        tr.desc = desc;
        tr.end = bval ? i + __popc(desc) : G;
        if (team == 0 && bval) s_anc[i] = anc;
        if (CONTACT) {
            for (int s = lane; s < m.nshapes; s += 32) s_bmask[s] = partner_mask(m, s);
            if (lane == 0) { int n = 0; for (int s = 0; s < m.nshapes; ++s) if (m.shape_owner_kind[s] == MPPIB_OWNER_LINK && shape_ref(m, s) != REF_STATIC) s_link[n++] = (uint8_t)s; }
        }
        __syncwarp();
    }

    // ---- per-lane model constants (lanes i >= nb: identity transform, no mass)
    BodyConst bc;
    float mc;      // mass of the subtree
    {
        Quat tq; tq.x = m.tree_quat[ib][0]; tq.y = m.tree_quat[ib][1]; tq.z = m.tree_quat[ib][2]; tq.w = m.tree_quat[ib][3];
        V3 tp = mk(m.tree_p[ib][0], m.tree_p[ib][1], m.tree_p[ib][2]);
        bc.jrev = m.jtype[ib] == MPPIB_JOINT_REVOLUTE ? 1.f : 0.f;
        V3 tax = bc.jrev != 0.f ? mk(0.f, 0.f, 0.f) : mk(m.tree_R[ib][2], m.tree_R[ib][5], m.tree_R[ib][8]);
        if (bval && m.parent[ib] < 0) {                 // the robot base pose is folded into a root body's parent transform
            Quat bq; bq.x = m.base_quat[0]; bq.y = m.base_quat[1]; bq.z = m.base_quat[2]; bq.w = m.base_quat[3];
            tp = qrot_add(mk(m.base_pos[0], m.base_pos[1], m.base_pos[2]), bq, tp);
            tax = qrot_add(mk(0.f, 0.f, 0.f), bq, tax);
            tq = qmul(bq, tq);
        }
        bc.mass = m.mass[ib];
        const float inv_m = bc.mass > 0.f ? 1.0f / bc.mass : 0.f;
        const V3 c = mk(inv_m * m.mcom[ib][0], inv_m * m.mcom[ib][1], inv_m * m.mcom[ib][2]);
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
        mc = bc.mass;
        subtree_add<G, R>(mc, i, tr);
    }
    const int ci0 = m.cmd_i0[ib], ci1 = m.cmd_i1[ib];
    const float cc0 = bval ? p.u_scale * m.cmd_c0[ib] : 0.f, cc1 = bval ? p.u_scale * m.cmd_c1[ib] : 0.f;
    const bool planar = m.planar_base != 0;
    const float a0x = m.gravity_on ? -m.gravity[0] : 0.f, a0y = m.gravity_on ? -m.gravity[1] : 0.f, a0z = m.gravity_on ? -m.gravity[2] : 0.f;
    const Quat bq0 = {m.base_quat[0], m.base_quat[1], m.base_quat[2], m.base_quat[3]};
    const M3 Rbase = quat_to_R(bq0);
    const V3 obase = mk(m.base_pos[0], m.base_pos[1], m.base_pos[2]);

    float q[NP], qd[NP];
#pragma unroll
    for (int pp = 0; pp < NP; ++pp) {
        q[pp] = 0.f; qd[pp] = 0.f;
        if (bval) {
            q[pp] = state0 ? state0[i] : state[(size_t)i * K + ka[pp]];
            qd[pp] = state0 ? state0[nb + i] : state[(size_t)(nb + i) * K + ka[pp]];
        }
    }

    // =====================================================================================================================
    // contact pipeline (team-parallel; the oracle's loop orders are kept)
    // =====================================================================================================================
    const uint32_t kg = sample_world(p.k_offset + (uint32_t)kc, p.n_worlds);   // key of the per-rollout randomisation
    // generalised coordinates of the contact solve held by this lane: coordinate sl * GC + ic = joint (< nb), else component of a free body
    constexpr int MAXS = NCS;
    constexpr int ncs = NCS;                                 // (== L.ncs, checked by the launcher)
    int ctype[MAXS], cfb[MAXS], ccomp[MAXS], cref[MAXS];     // 0 none / 1 joint / 2 linear / 3 angular (body axes); free body base, component, ref id
#pragma unroll
    for (int sl = 0; sl < MAXS; ++sl) {
        const int c = sl * GC + ic;
        ctype[sl] = 0; cfb[sl] = 0; ccomp[sl] = 0; cref[sl] = -99;
        if (c < nb) ctype[sl] = 1;
        else if (c - nb < 6 * m.nfree) {
            const int f = (c - nb) / 6, comp = (c - nb) % 6;
            ctype[sl] = comp < 3 ? 2 : 3; ccomp[sl] = comp % 3; cfb[sl] = L.fb0 + f * FBN; cref[sl] = REF_FREE0 + f;
        }
    }
    int nlink = 0; uint32_t static_mask = 0;
    if (CONTACT) for (int s = 0; s < m.nshapes; ++s) {
        if (m.shape_owner_kind[s] == MPPIB_OWNER_STATIC) static_mask |= 1u << s;
        else if (m.shape_owner_kind[s] == MPPIB_OWNER_LINK && shape_ref(m, s) != REF_STATIC) ++nlink;
    }
    auto refresh_free = [&](int fb) {      // all lanes compute, lane 0 writes
        const Quat fq = {xs[fb + FB_Q], xs[fb + FB_Q + 1], xs[fb + FB_Q + 2], xs[fb + FB_Q + 3]};
        const M3 Rf = quat_to_R(fq);
        const V3 iinv = ld3(xs, fb + FB_IINV);
        __syncwarp();
        if (ic == 0) {
            stM3(xs, fb + FB_R, Rf);
            const S3 Iw = world_inv_inertia(Rf, iinv);
            xs[fb + FB_IW + 0] = Iw.xx; xs[fb + FB_IW + 1] = Iw.yy; xs[fb + FB_IW + 2] = Iw.zz;
            xs[fb + FB_IW + 3] = Iw.xy; xs[fb + FB_IW + 4] = Iw.xz; xs[fb + FB_IW + 5] = Iw.yz;
        }
        __syncwarp();
    };
    if (CONTACT) {
        // one-time per rollout: randomised shape / body parameters (lane = shape / free body), initial free-body states
        for (int s = ic; s < m.nshapes; s += GC) {
            V3 half; float mu, rad;
            shape_params(m, p, kg, s, half, mu, rad);
            const int sb = L.sh0 + s * SHN;
            st3(xs, sb + SH_HALF, half);
            xs[sb + SH_MU] = mu;
            xs[sb + SH_RAD] = rad;
        }
        for (int f = ic; f < m.nfree; f += GC) {
            const int fb = L.fb0 + f * FBN;
            float inv_mass; V3 half, iinv;
            free_params(m, p, kg, f, inv_mass, half, iinv);
            xs[fb + FB_MASS] = inv_mass;
            st3(xs, fb + FB_HALF, half);
            st3(xs, fb + FB_IINV, iinv);
            for (int r = 0; r < 13; ++r)
                xs[fb + r] = state0 ? root0[13 * m.free_actor[f] + r] : state[(size_t)(2 * nb + 13 * f + r) * K + kc];
        }
        for (int s = ic; s < 3 * MPPIB_MAX_SLOTS; s += GC) xs[L.net0 + s] = 0.f;
        __syncwarp();
        for (int f = 0; f < m.nfree; ++f) refresh_free(L.fb0 + f * FBN);
    }
    // world poses of the shapes: `statics` once per rollout, links and free bodies in every substep (lane = shape; a link's frame comes
    // from the joint block the articulation phase wrote)
    auto shapes_world = [&](bool statics) {
        const int ns = m.nshapes;
        for (int s = ic; s < ns; s += GC) {
            const int kind = m.shape_owner_kind[s];
            const int own = m.shape_owner[s];
            if ((kind == MPPIB_OWNER_STATIC) != statics) continue;
            M3 Ro; V3 po;
            if (kind == MPPIB_OWNER_STATIC) root_pose(root0, m.shape_actor[s], Ro, po);
            else if (kind == MPPIB_OWNER_LINK) {
                if (own < 0) { Ro = Rbase; po = obase; }
                else { const int jb = L.jb0 + own * JBN; Ro = ldM3(xs, jb + JB_R); po = ld3(xs, jb + JB_O); }
            } else {
                const int fb = L.fb0 + own * FBN;
                Ro = ldM3(xs, fb + FB_R); po = ld3(xs, fb + FB_X);
            }
            M3 R; V3 c; shape_pose(m, s, Ro, po, R, c);
            const int sb = L.sh0 + s * SHN;
            stM3(xs, sb + SH_R, R);
            st3(xs, sb + SH_C, c);
        }
        __syncwarp();
    };
    int nc = 0;
    // append the contacts of the lanes that raise `hit`, in lane order (the oracle's sample-point order)
    auto append = [&](bool hit, int refA, int refB, int slotA, int slotB, V3 pt, V3 n, float d, float mu) {
        const uint32_t bits = team_ballot<GC>(hit, tbc);
        const int slot = nc + __popc(bits & ((1u << ic) - 1u));
        if (hit && slot < m.max_contacts) {
            const int cb = L.ct0 + slot * CTN;
            st3(xs, cb + CT_P, pt); st3(xs, cb + CT_N, n);
            xs[cb + CT_D] = d; xs[cb + CT_MU] = mu; xs[cb + CT_LN] = 0.f; xs[cb + CT_LT1] = 0.f; xs[cb + CT_LT2] = 0.f;
            xs[cb + CT_IDS] = __int_as_float(pack_sides(refA, refB, slotA, slotB));
        }
        nc = min(nc + __popc(bits), (int)m.max_contacts);
    };
    // sample points of box a inside box b (lane = sample point), `flip`: a is the B side of the pair
    // (`on`: this team takes part -- the pair loop runs over the union of the teams' near pairs)
    auto points_in_box = [&](int a, int b, bool flip, bool on) {
        const int sa = L.sh0 + a * SHN, sb = L.sh0 + b * SHN;
        const M3 Ra = ldM3(xs, sa + SH_R), Rb = ldM3(xs, sb + SH_R);
        const V3 ca = ld3(xs, sa + SH_C), cbv = ld3(xs, sb + SH_C);
        const V3 ha = ld3(xs, sa + SH_HALF), hb = ld3(xs, sb + SH_HALF);
        const float mu = 0.5f * (xs[sa + SH_MU] + xs[sb + SH_MU]);
        const int refa = shape_ref(m, a), refb = shape_ref(m, b), slota = m.shape_slot[a], slotb = m.shape_slot[b];
        bool c0, c1, c2; face_axes(Rb, ca, cbv, hb, c0, c1, c2);
        for (int i0 = 0; i0 < 27; i0 += GC) {
            const int idx = i0 + ic;
            V3 pt, n; float pen;
            const bool inside = box_point(idx, Ra, ca, ha, Rb, cbv, hb, c0, c1, c2, m.contact_margin, pt, n, pen);
            const bool hit = on && idx < 27 && idx != 13 && inside;
            if (!flip) append(hit, refa, refb, slota, slotb, pt, n, pen, mu);
            else append(hit, refb, refa, slotb, slota, pt, mk(-n.x, -n.y, -n.z), pen, mu);
        }
    };
    // ONE contact of a sphere against a box or a sphere; all lanes compute, lane 0 appends
    auto sphere_pair = [&](int a, int b, bool on) {
        const int sa = L.sh0 + a * SHN, sb = L.sh0 + b * SHN;
        const float mu = 0.5f * (xs[sa + SH_MU] + xs[sb + SH_MU]);
        const int refa = shape_ref(m, a), refb = shape_ref(m, b), slota = m.shape_slot[a], slotb = m.shape_slot[b];
        const V3 ca = ld3(xs, sa + SH_C), cbv = ld3(xs, sb + SH_C);
        const bool sph_a = m.shape_type[a] == MPPIB_SHAPE_SPHERE;
        V3 pt, n; float pen; bool hit;
        if (sph_a && m.shape_type[b] == MPPIB_SHAPE_SPHERE) hit = sphere_sphere(ca, xs[sa + SH_HALF], cbv, xs[sb + SH_HALF], m.contact_margin, pt, n, pen);
        else {
            const int sx = sph_a ? sb : sa;
            hit = sphere_box(sph_a ? ca : cbv, xs[(sph_a ? sa : sb) + SH_HALF], ldM3(xs, sx + SH_R), sph_a ? cbv : ca, ld3(xs, sx + SH_HALF), m.contact_margin, pt, n, pen);
            if (!sph_a) n = mk(-n.x, -n.y, -n.z);
        }
        append(on && hit && ic == 0, refa, refb, slota, slotb, pt, n, pen, mu);
    };
    auto near_shapes = [&](int a, int b) -> bool {
        const int sa = L.sh0 + a * SHN, sb = L.sh0 + b * SHN;
        const V3 d = ld3(xs, sa + SH_C) - ld3(xs, sb + SH_C);
        const bool sph = m.shape_type[a] == MPPIB_SHAPE_SPHERE || m.shape_type[b] == MPPIB_SHAPE_SPHERE;
        if (!near_bounds(d, xs[sa + SH_RAD], xs[sb + SH_RAD], sph, m.contact_margin)) return false;
        if (sph) return true;
        return near_boxes(d, ldM3(xs, sa + SH_R), ld3(xs, sa + SH_HALF), ldM3(xs, sb + SH_R), ld3(xs, sb + SH_HALF), m.contact_margin);
    };
    // partners of shape a: the broad phase of up to GC partners in parallel (lane = partner), then the near ones in ascending order
    auto pairs_of = [&](int a) {
        uint32_t mask = s_bmask[a];
        while (mask) {                                       // warp-uniform
            uint32_t mine = mask; int b = -1;
            for (int j = 0; j <= ic && mine; ++j) { b = __ffs(mine) - 1; mine &= mine - 1; }     // the (ic+1)-th set bit, if there is one
            const int cnt = __popc(mask);
            const bool have = ic < cnt;
            const bool nearb = have && near_shapes(a, b);
            const uint32_t mybits = team_ballot<GC>(nearb, tbc);
            uint32_t ubits = union_ballot<GC>(nearb);         // near for ANY team of the warp: warp-uniform loop, lanes in ascending partner order
            while (ubits) {
                const int ln = __ffs(ubits) - 1; ubits &= ubits - 1;
                const int bb = __shfl_sync(FULL, b, ln, GC);  // (the same shape for every team: b depends on the lane only)
                const bool on = (mybits >> ln) & 1u;
                if (m.shape_type[a] == MPPIB_SHAPE_SPHERE || m.shape_type[bb] == MPPIB_SHAPE_SPHERE) sphere_pair(a, bb, on);
                else { points_in_box(a, bb, false, on); points_in_box(bb, a, true, on); }
            }
            for (int j = 0; j < GC && mask; ++j) mask &= mask - 1;                               // drop the partners just handled
        }
    };
    auto detect = [&]() {
        nc = 0;
        const int ns = m.nshapes;
        for (int a = 0; a < ns; ++a) {
            if (m.shape_owner_kind[a] != MPPIB_OWNER_FREE) continue;
            const int sa = L.sh0 + a * SHN;
            if (m.ground_plane) {
                const M3 Ra = ldM3(xs, sa + SH_R); const V3 ca = ld3(xs, sa + SH_C), ha = ld3(xs, sa + SH_HALF);
                const float mu = 0.5f * (xs[sa + SH_MU] + m.ground_friction);
                // lane = corner; at most the 4 lowest corners (ties by corner index) are ground points (contact.cuh ground_corner_mask):
                // with more than 4 below the margin (h above ~0.026 s) the lanes rank their heights by shuffles
                static_assert(GC >= 8, "one corner per lane");
                const int idx = ic;
                const int ix = (idx >> 2) * 2 - 1, iy = ((idx >> 1) & 1) * 2 - 1, iz = (idx & 1) * 2 - 1;
                const V3 pt = mul(Ra, mk(ix * ha.x, iy * ha.y, iz * ha.z)) + ca;
                bool hit = idx < 8 && pt.z < m.ground_margin;
                if (__any_sync(FULL, __popc(team_ballot<GC>(hit, tbc)) > 4)) {          // warp-uniform
                    int rank = 0;
                    for (int o = 0; o < 8; ++o) {
                        const float zo = __shfl_sync(FULL, pt.z, o, GC);
                        rank += zo < pt.z || (zo == pt.z && o < idx);
                    }
                    hit = hit && rank < 4;
                }
                append(hit, shape_ref(m, a), REF_STATIC, m.shape_slot[a], -1, pt, mk(0.f, 0.f, 1.f), -pt.z, mu);
            }
            pairs_of(a);
        }
        // articulation link vs static shape.  A link shape has few partners (the static shapes: one table), so the broad phase runs with
        // lane = LINK SHAPE against one static shape at a time; the near pairs are then visited in the oracle's order (link shape
        // ascending, static shape ascending within it)
        for (int l0 = 0; l0 < nlink; l0 += GC) {
            const bool have = l0 + ic < nlink;
            const int a = have ? s_link[l0 + ic] : 0;
            uint32_t mymask = 0;
            for (uint32_t sm = static_mask; sm; sm &= sm - 1) { const int b = __ffs(sm) - 1; if (have && near_shapes(a, b)) mymask |= 1u << b; }
            if (!__any_sync(FULL, mymask != 0u)) continue;                   // (the arm is away from the table: the usual case)
            const int nl = min(GC, nlink - l0);
            for (int ln = 0; ln < nl; ++ln) {
                const int aa = s_link[l0 + ln];
                const uint32_t ma = __shfl_sync(FULL, mymask, ln, GC);       // this team's near static shapes of link shape aa
                uint32_t ub = ma;                                            // ... of any team of the warp: warp-uniform loop
                if (GC <= 16) ub |= __shfl_xor_sync(FULL, ub, 16);
                if (GC <= 8) ub |= __shfl_xor_sync(FULL, ub, 8);
                if (GC <= 4) ub |= __shfl_xor_sync(FULL, ub, 4);
                for (; ub; ub &= ub - 1) {
                    const int b = __ffs(ub) - 1;
                    const bool on = (ma >> b) & 1u;
                    if (m.shape_type[aa] == MPPIB_SHAPE_SPHERE || m.shape_type[b] == MPPIB_SHAPE_SPHERE) sphere_pair(aa, b, on);
                    else { points_in_box(aa, b, false, on); points_in_box(b, aa, true, on); }
                }
            }
        }
        __syncwarp();
    };
    // ---- Gauss-Seidel soft-constraint solve on the predicted velocities (contact.cuh solve, oracle.cpp ContactWorld::solve) over
    // GENERALISED COORDINATES, one (or a few) per lane: the nb joints, then per free body its 3 linear velocity components (world) and its
    // 3 angular velocity components IN BODY AXES -- there the inverse inertia is diagonal like the joints' 1 / D_j, so every coordinate
    // has ONE scalar inverse inertia `minv` and a contact row is one number per coordinate: J_r (kept in shared memory for the
    // sweeps).  A visit is then 3 loads + 3 products per coordinate, ONE butterfly all-reduce of the three row velocities, the row
    // updates (replicated on every lane: no owner lane, no barrier) and 3 FMAs per coordinate.
    auto chain_sign = [&](int joint, int refA, int refB) -> float {      // +1 / -1: the joint moves side A / side B of the contact
        float sg = 0.f;
        if (refA >= 0 && refA < REF_FREE0 && ((s_anc[refA] >> joint) & 1u)) sg = 1.f;
        if (refB >= 0 && refB < REF_FREE0 && ((s_anc[refB] >> joint) & 1u)) sg = -1.f;
        return sg;
    };
    auto solve_contacts = [&](bool last_substep) {
        const float kp = m.contact_kp, kdc = m.contact_kd;
        const float gamma = 1.0f / (h * (h * kp + kdc)), beta = h * kp / (h * kp + kdc), ih = 1.0f / h;
        float vel[MAXS], minv[MAXS];
        float* rows = xs + L.rw0;
        const int ncoord = nb + 6 * m.nfree;
        auto load_row = [&](int c, int sl) -> float4 {       // (n, t1, t2) entries of this lane's coordinate in slot sl; the last slot may be ragged
            if (sl + 1 < MAXS || sl * GC + ic < ncoord) {
                if (!COMPACT) return reinterpret_cast<const float4*>(rows)[c * ncoord + sl * GC + ic];
                const float* rw = rows + c * 3 * ncoord + sl * GC + ic;
                return make_float4(rw[0], rw[ncoord], rw[2 * ncoord], 0.f);
            }
            return make_float4(0.f, 0.f, 0.f, 0.f);
        };
#pragma unroll
        for (int sl = 0; sl < MAXS; ++sl) {
            vel[sl] = 0.f; minv[sl] = 0.f;
            if (sl >= ncs) continue;
            if (ctype[sl] == 1) { const int jb = L.jb0 + (sl * GC + ic) * JBN; vel[sl] = xs[jb + JB_VP]; minv[sl] = xs[jb + JB_INVD]; }
            else if (ctype[sl] == 2) { vel[sl] = xs[cfb[sl] + FB_V + ccomp[sl]]; minv[sl] = xs[cfb[sl] + FB_MASS]; }
            else if (ctype[sl] == 3) {
                const int fb = cfb[sl], cc = ccomp[sl];
                vel[sl] = xs[fb + FB_R + cc] * xs[fb + FB_W] + xs[fb + FB_R + 3 + cc] * xs[fb + FB_W + 1] + xs[fb + FB_R + 6 + cc] * xs[fb + FB_W + 2];
                minv[sl] = xs[fb + FB_IINV + cc];
            }
        }
        const int nc_warp = __reduce_max_sync(FULL, nc);     // contacts of the busiest team of the warp
        for (int c = 0; c < nc_warp; ++c) {                  // per contact, once: tangent frame, rows, inverse effective masses, bias velocity
            const bool act = c < nc;                         // (a team past its own contacts computes on stale records and stores nothing)
            const int cb = L.ct0 + c * CTN;
            const int ids = act ? __float_as_int(xs[cb + CT_IDS]) : 0;
            const int refA = ref_a(ids), refB = ref_b(ids);
            const V3 pt = ld3(xs, cb + CT_P), n = ld3(xs, cb + CT_N);
            V3 t1, t2; tangents(n, t1, t2);
            float kn_ = 0.f, kt1 = 0.f, kt2 = 0.f;
#pragma unroll
            for (int sl = 0; sl < MAXS; ++sl) {
                if (sl >= ncs) continue;
                float jn = 0.f, j1 = 0.f, j2 = 0.f;
                if (ctype[sl] == 1) {
                    const int jb = L.jb0 + (sl * GC + ic) * JBN;
                    const float sg = chain_sign(sl * GC + ic, refA, refB);
                    const V3 Sn = ld3(xs, jb + JB_SN), Sf = ld3(xs, jb + JB_SF);
                    const V3 mn = cross(pt, n), m1 = cross(pt, t1), m2 = cross(pt, t2);
                    jn = sg * (dot(Sf, n) + dot(Sn, mn)); j1 = sg * (dot(Sf, t1) + dot(Sn, m1)); j2 = sg * (dot(Sf, t2) + dot(Sn, m2));
                } else if (ctype[sl] >= 2) {
                    const float sg = refA == cref[sl] ? 1.f : (refB == cref[sl] ? -1.f : 0.f);
                    const int fb = cfb[sl], cc = ccomp[sl];
                    if (ctype[sl] == 2) {
                        jn = sg * (cc == 0 ? n.x : (cc == 1 ? n.y : n.z)); j1 = sg * (cc == 0 ? t1.x : (cc == 1 ? t1.y : t1.z)); j2 = sg * (cc == 0 ? t2.x : (cc == 1 ? t2.y : t2.z));
                    } else {
                        const V3 r = pt - ld3(xs, fb + FB_X);
                        const V3 col = mk(xs[fb + FB_R + cc], xs[fb + FB_R + 3 + cc], xs[fb + FB_R + 6 + cc]);      // body axis cc in the world
                        jn = sg * dot(col, cross(r, n)); j1 = sg * dot(col, cross(r, t1)); j2 = sg * dot(col, cross(r, t2));
                    }
                }
                if (act && sl * GC + ic < ncoord) {
                    if (COMPACT) { float* rw = rows + c * 3 * ncoord + sl * GC + ic; rw[0] = jn; rw[ncoord] = j1; rw[2 * ncoord] = j2; }
                    else reinterpret_cast<float4*>(rows)[c * ncoord + sl * GC + ic] = make_float4(jn, j1, j2, 0.f);
                }
                kn_ = fmaf(jn * jn, minv[sl], kn_); kt1 = fmaf(j1 * j1, minv[sl], kt1); kt2 = fmaf(j2 * j2, minv[sl], kt2);
            }
            kn_ = team_sum<GC>(kn_); kt1 = team_sum<GC>(kt1); kt2 = team_sum<GC>(kt2);
            const float d = xs[cb + CT_D];
            __syncwarp();
            if (ic == 0 && act) {
                xs[cb + CT_KN] = kn_ > K_ROW_MIN ? rcp_approx(kn_ + gamma) : 0.f;
                xs[cb + CT_KT1] = kt1 > K_ROW_MIN ? rcp_approx(kt1) : 0.f;
                xs[cb + CT_KT2] = kt2 > K_ROW_MIN ? rcp_approx(kt2) : 0.f;
                if (!COMPACT) st3(xs, cb + CT_T1, t1);
                xs[cb + CT_D] = d > 0.f ? fminf(beta * d * ih, m.max_depen) : d * ih;
            }
        }
        __syncwarp();
        // the sweeps: contact_iters x nc visits in one flat loop; the constants and rows of the NEXT visit are fetched while this one
        // reduces (they do not change during the sweeps; the multipliers do and are loaded by the visit itself)
        const int nvisit = m.contact_iters * nc;
        const int nvisit_warp = m.contact_iters * nc_warp;
        const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 Bc = zero4, Rc[MAXS];
#pragma unroll
        for (int sl = 0; sl < MAXS; ++sl) Rc[sl] = zero4;
        if (nc > 0) {
            Bc = *reinterpret_cast<const float4*>(xs + L.ct0 + CT_D);
#pragma unroll
            for (int sl = 0; sl < MAXS; ++sl) Rc[sl] = load_row(0, sl);
        }
        int c = 0;
        // one visit: contact c with its constants Bcur / rows Rcur in registers; fetches those of the next visit into Bnxt / Rnxt
        auto visit = [&](int v, const float4& Bcur, const float4 (&Rcur)[MAXS], float4& Bnxt, float4 (&Rnxt)[MAXS]) {
            const int cb = L.ct0 + c * CTN;
            const int cnx = c + 1 >= nc ? 0 : c + 1;
            const bool act_next = v + 1 < nvisit;
            Bnxt = zero4;
            if (act_next) Bnxt = *reinterpret_cast<const float4*>(xs + L.ct0 + cnx * CTN + CT_D);
#pragma unroll
            for (int sl = 0; sl < MAXS; ++sl) { Rnxt[sl] = zero4; if (act_next) Rnxt[sl] = load_row(cnx, sl); }
            const float bias = Bcur.x, ikn = Bcur.y, ikt1 = Bcur.z, ikt2 = Bcur.w;
            const bool upd = ikn > 0.f;                      // (false for a disabled row and for a team past its visits: Bcur = 0)
            float4 A = zero4;                                // ln lt1 lt2 mu
            if (upd) A = *reinterpret_cast<const float4*>(xs + cb);
            float vn = 0.f, v1 = 0.f, v2 = 0.f;
#pragma unroll
            for (int sl = 0; sl < MAXS; ++sl) { vn = fmaf(Rcur[sl].x, vel[sl], vn); v1 = fmaf(Rcur[sl].y, vel[sl], v1); v2 = fmaf(Rcur[sl].z, vel[sl], v2); }
#pragma unroll
            for (int o = GC / 2; o > 0; o >>= 1) {            // relative velocity along the contact frame: one butterfly for the three rows
                vn += __shfl_xor_sync(FULL, vn, o, GC); v1 += __shfl_xor_sync(FULL, v1, o, GC); v2 += __shfl_xor_sync(FULL, v2, o, GC);
            }
            const float ln_new = fmaxf(0.f, A.x + (-vn + bias - gamma * A.x) * ikn);
            const float lim = A.w * ln_new;
            const float lt1_new = ikt1 > 0.f ? fminf(fmaxf(A.y - v1 * ikt1, -lim), lim) : A.y;
            const float lt2_new = ikt2 > 0.f ? fminf(fmaxf(A.z - v2 * ikt2, -lim), lim) : A.z;
            const float dn = upd ? ln_new - A.x : 0.f, d1 = upd ? lt1_new - A.y : 0.f, d2 = upd ? lt2_new - A.z : 0.f;
#pragma unroll
            for (int sl = 0; sl < MAXS; ++sl) vel[sl] = fmaf(minv[sl], fmaf(Rcur[sl].x, dn, fmaf(Rcur[sl].y, d1, Rcur[sl].z * d2)), vel[sl]);
            // every lane stores the same numbers and later reads back what it stored itself: no owner lane.  (The barrier orders this
            // visit's loads of the record before any lane's store for the tools -- compute-sanitizer racecheck -- and costs one issue slot;
            // the shuffles above have already brought the lanes together.)
            __syncwarp();
            if (upd) *reinterpret_cast<float4*>(xs + cb) = make_float4(ln_new, lt1_new, lt2_new, A.w);
            c = cnx;
        };
        float4 Bd, Rd[MAXS];                                 // two register sets, used alternately: no hand-over copies
#pragma unroll 1
        for (int v = 0; v < nvisit_warp; v += 2) {
            visit(v, Bc, Rc, Bd, Rd);
            if (v + 1 < nvisit_warp) visit(v + 1, Bd, Rd, Bc, Rc);
        }
        // ---- back to the bodies: joints keep their lane's value; free bodies: linear components, then omega = R omega_body
        __syncwarp();
#pragma unroll
        for (int sl = 0; sl < MAXS; ++sl) {
            if (sl >= ncs) continue;
            if (ctype[sl] == 1) xs[L.jb0 + (sl * GC + ic) * JBN + JB_VP] = vel[sl];
            else if (ctype[sl] == 2) xs[cfb[sl] + FB_V + ccomp[sl]] = vel[sl];
            else if (ctype[sl] == 3) xs[cfb[sl] + FB_W + ccomp[sl]] = vel[sl];       // (body axes for a moment)
        }
        __syncwarp();
        for (int f = 0; f < m.nfree; ++f) {
            const int fb = L.fb0 + f * FBN;
            const V3 wb = ld3(xs, fb + FB_W);
            const M3 Rf = ldM3(xs, fb + FB_R);
            __syncwarp();
            if (ic == 0) st3(xs, fb + FB_W, mul(Rf, wb));
        }
        __syncwarp();
        if (last_substep) {                                  // net contact force per body = the last substep's impulses / h
            if (ic == 0) {
                for (int s = 0; s < 3 * MPPIB_MAX_SLOTS; ++s) xs[L.net0 + s] = 0.f;
                for (int c = 0; c < nc; ++c) {
                    const int cb = L.ct0 + c * CTN;
                    const int ids = __float_as_int(xs[cb + CT_IDS]);
                    // (slot_a / slot_b written out: with the calls, the roomy <8, 8, true, 1, 8> instantiation spills 8 bytes more)
                    const int slotA = ((ids >> 16) & 0xFF) - 1, slotB = ((ids >> 24) & 0xFF) - 1;
                    if (slotA < 0 && slotB < 0) continue;
                    const V3 n = ld3(xs, cb + CT_N);
                    V3 t1, t2;
                    if (COMPACT) tangents(n, t1, t2);
                    else { t1 = ld3(xs, cb + CT_T1); t2 = cross(n, t1); }
                    const V3 F = scale(ih, scale(xs[cb + CT_LN], n) + scale(xs[cb + CT_LT1], t1) + scale(xs[cb + CT_LT2], t2));
                    if (slotA >= 0) { xs[L.net0 + 3 * slotA] += F.x; xs[L.net0 + 3 * slotA + 1] += F.y; xs[L.net0 + 3 * slotA + 2] += F.z; }
                    if (slotB >= 0) { xs[L.net0 + 3 * slotB] -= F.x; xs[L.net0 + 3 * slotB + 1] -= F.y; xs[L.net0 + 3 * slotB + 2] -= F.z; }
                }
            }
            __syncwarp();
        }
    };
    auto integrate_free = [&]() {
        for (int f = 0; f < m.nfree; ++f) {
            const int fb = L.fb0 + f * FBN;
            V3 x = ld3(xs, fb + FB_X);
            Quat fq = {xs[fb + FB_Q], xs[fb + FB_Q + 1], xs[fb + FB_Q + 2], xs[fb + FB_Q + 3]};
            integrate_pose(x, fq, ld3(xs, fb + FB_V), ld3(xs, fb + FB_W), h);
            __syncwarp();
            if (ic == 0) {
                st3(xs, fb + FB_X, x);
                xs[fb + FB_Q] = fq.x; xs[fb + FB_Q + 1] = fq.y; xs[fb + FB_Q + 2] = fq.z; xs[fb + FB_Q + 3] = fq.w;
            }
            __syncwarp();
            refresh_free(fb);
        }
    };

    // ---- observation rows of model step t from the frames of the CURRENT state
    auto write_obs = [&](int t, const Kin& kn, int pp) {
        const size_t TK = (size_t)T * K;
        const bool kval = kvala[pp];
        const float* xo = xsa[pp];
        float* dst = obs + (size_t)t * K + ka[pp];
        int row = 0;
        for (int oi = 0; oi < p.nobs; ++oi) {
            const int kind = p.obs[oi].kind, idx = p.obs[oi].index;
            if (kind == MPPIB_OBS_LINK_STATE) {
                const int b = m.link_body[idx];
                if (kval && (b >= 0 ? i == b : i == 0)) {
                    V3 ol, w, vO; Quat qb; M3 Rl;
                    if (b >= 0) { Rl = kn.R; ol = kn.o; w = kn.V.n; vO = kn.V.f; qb = kn.qw; }
                    else { qb = bq0; Rl = Rbase; ol = obase; w = mk(0.f, 0.f, 0.f); vO = mk(0.f, 0.f, 0.f); }
                    const V3 pos = ol + mulc(Rl, m.link_p[idx][0], m.link_p[idx][1], m.link_p[idx][2]);
                    const Quat qlk = {m.link_quat[idx][0], m.link_quat[idx][1], m.link_quat[idx][2], m.link_quat[idx][3]};
                    const Quat qo = qmul(qb, qlk);
                    const V3 vel = cross_add(vO, w, pos);
                    dst[(size_t)(row + 0) * TK] = pos.x; dst[(size_t)(row + 1) * TK] = pos.y; dst[(size_t)(row + 2) * TK] = pos.z;
                    dst[(size_t)(row + 3) * TK] = qo.x; dst[(size_t)(row + 4) * TK] = qo.y; dst[(size_t)(row + 5) * TK] = qo.z;
                    dst[(size_t)(row + 6) * TK] = qo.w;
                    dst[(size_t)(row + 7) * TK] = vel.x; dst[(size_t)(row + 8) * TK] = vel.y; dst[(size_t)(row + 9) * TK] = vel.z;
                    dst[(size_t)(row + 10) * TK] = w.x; dst[(size_t)(row + 11) * TK] = w.y; dst[(size_t)(row + 12) * TK] = w.z;
                }
                row += 13;
            } else if (kind == MPPIB_OBS_DOF_STATE) {
                if (kval && bval) {
                    dst[(size_t)(row + 2 * i) * TK] = q[pp];
                    dst[(size_t)(row + 2 * i + 1) * TK] = qd[pp];
                }
                row += 2 * nb;
            } else if (kind == MPPIB_OBS_FREE_STATE) {
                const int fb = L.fb0 + idx * FBN;
                for (int r = i; r < 13; r += G) if (kval) dst[(size_t)(row + r) * TK] = (CONTACT && idx < m.nfree) ? xo[fb + r] : 0.f;
                row += 13;
            } else {
                for (int r = i; r < 3; r += G) if (kval) dst[(size_t)(row + r) * TK] = (CONTACT && idx < MPPIB_MAX_SLOTS) ? xo[L.net0 + 3 * idx + r] : 0.f;
                row += 3;
            }
        }
    };

    // ---- one articulation substep of one rollout: composite-rigid-body terms, joint-space LDL^T; returns the predicted velocity of this
    // lane's joint, `invD_out` = 1 / D_j of the articulated-body recursion (the joint's compliance in the contact solve)
    auto articulation = [&](const Kin& kn, float q, float qd, float tgt, float& invD_out) -> float {
            // ---- per-body terms about the world origin
            const V3 cw = kn.o + mulc(kn.R, bc.cx, bc.cy, bc.cz);
            const V3 hw = scale(bc.mass, cw);
            S3 A;
            {
                const V3 r0 = mk(kn.R.m00, kn.R.m01, kn.R.m02), r1 = mk(kn.R.m10, kn.R.m11, kn.R.m12), r2 = mk(kn.R.m20, kn.R.m21, kn.R.m22);
                const V3 t0v = mul(bc.Ic, r0), t1v = mul(bc.Ic, r1), t2v = mul(bc.Ic, r2);
                const float d2 = dot(hw, cw);
                A.xx = fmaf(-hw.x, cw.x, d2 + dot(r0, t0v)); A.yy = fmaf(-hw.y, cw.y, d2 + dot(r1, t1v)); A.zz = fmaf(-hw.z, cw.z, d2 + dot(r2, t2v));
                A.xy = fmaf(-hw.x, cw.y, dot(r0, t1v)); A.xz = fmaf(-hw.x, cw.z, dot(r0, t2v)); A.yz = fmaf(-hw.y, cw.z, dot(r1, t2v));
            }
            const V3 w = kn.V.n, v = kn.V.f;
            V6 fb6;
            {
                const V3 nn = cross_add(mul(A, w), hw, v);
                const V3 ff = cross_add(scale(bc.mass, v), w, hw);
                fb6.n = cross_add(cross(w, nn), v, ff);
                fb6.f = cross(w, ff);
            }
            V6 a;
            a.n = cross(w, kn.Vl.n);
            a.f = cross_add(cross(w, kn.Vl.f), v, kn.Vl.n);
            anc_add3<G, R>(a.n, tr); anc_add3<G, R>(a.f, tr);
            a.f = mk(a.f.x + a0x, a.f.y + a0y, a.f.z + a0z);
            fb6.n = cross_add(mul_add(fb6.n, A, a.n), hw, a.f);
            fb6.f = cross_add(mk(fmaf(a.f.x, bc.mass, fb6.f.x), fmaf(a.f.y, bc.mass, fb6.f.y), fmaf(a.f.z, bc.mass, fb6.f.z)), a.n, hw);
            // ---- composites: sums over the subtree
            subtree_add<G, R>(A.xx, i, tr); subtree_add<G, R>(A.yy, i, tr); subtree_add<G, R>(A.zz, i, tr);
            subtree_add<G, R>(A.xy, i, tr); subtree_add<G, R>(A.xz, i, tr); subtree_add<G, R>(A.yz, i, tr);
            V3 hc = hw;
            subtree_add3<G, R>(hc, i, tr);
            subtree_add3<G, R>(fb6.n, i, tr); subtree_add3<G, R>(fb6.f, i, tr);
            V6 Fj;
            Fj.n = cross_add(mul(A, kn.S.n), hc, kn.S.f);
            Fj.f = cross_add(scale(mc, kn.S.f), kn.S.n, hc);
            const float bias = dot6(kn.S, fb6);
            // ---- joint-space inertia, LEAF-FIRST elimination order (the pivots are then the articulated-body diagonals D_j the
            // contact solve needs): virtual index v = NB - 1 - body.  Lane j owns column j of the LOWER triangle: M_rj = F_r . S_j for
            // the descendants r of j (0 elsewhere); in virtual indices that is the upper-triangle column the solver below expects.
            constexpr int VB = NB - 1;
            const int vi = VB - i;                                           // virtual index of this lane (negative for lanes >= NB: never a pivot)
            float mcol[NB];
#pragma unroll
            for (int vr = 0; vr < NB; ++vr) {
                const int rb = VB - vr;                                      // body of virtual row vr
                V6 Fr;
                Fr.n.x = shfl_at<G>(Fj.n.x, rb); Fr.n.y = shfl_at<G>(Fj.n.y, rb); Fr.n.z = shfl_at<G>(Fj.n.z, rb);
                Fr.f.x = shfl_at<G>(Fj.f.x, rb); Fr.f.y = shfl_at<G>(Fj.f.y, rb); Fr.f.z = shfl_at<G>(Fj.f.z, rb);
                mcol[vr] = ((tr.desc >> rb) & 1u) ? dot6(Fr, kn.S) : 0.f;
            }
            float sat = 0.f, qdd = 0.f, invD = 1.f;
#pragma unroll 1
            for (int solve = 0; solve < 2; ++solve) {
                float tau, dimp;
                if (sat != 0.f) { tau = sat * bc.effort - bc.damp * qd; dimp = bc.dimp_sat; }
                else if (vel_mode) { tau = bc.kd * (tgt - qd) - bc.damp * qd; dimp = bc.dimp_drive; }
                else { tau = fminf(fmaxf(tgt, -bc.effort), bc.effort) - (bc.kd + bc.damp) * qd; dimp = bc.dimp_drive; }
                float col[NB], lcol[NB];
#pragma unroll
                for (int r = 0; r < NB; ++r) { col[r] = mcol[r]; lcol[r] = 0.f; }
                float invd = 1.f;
                float y = tau - bias;
#pragma unroll
                for (int kk = 0; kk < NB; ++kk) {
                    const int kb = VB - kk;                                  // body of the pivot
                    const float dk = shfl_at<G>(col[kk] + dimp, kb);
                    const float inv = rcp_approx(dk);
                    const bool own = vi == kk;
                    if (own) invd = inv;
                    const float lk = col[kk] * inv;
                    if (kk + 1 < NB) {
                        const float yk = shfl_at<G>(y, kb);
                        if (vi > kk) y = fmaf(-lk, yk, y);
                    }
#pragma unroll
                    for (int r = kk + 1; r < NB; ++r) {
                        const float lr = shfl_at<G>(lk, VB - r);
                        col[r] = fmaf(-lr, col[kk], col[r]);
                        if (own) lcol[r] = lr;
                    }
                }
                y *= invd;
#pragma unroll
                for (int jj = NB - 1; jj >= 1; --jj) {
                    const float xj = shfl_at<G>(y, VB - jj);
                    if (vi >= 0 && vi < jj) y = fmaf(-lcol[jj], xj, y);
                }
                qdd = bval ? y : 0.f;
                invD = invd;                                                 // 1 / D_j of the articulated-body recursion
                bool newly = false;
                if (solve == 0 && vel_mode && bval) {
                    const float td = bc.kd * (tgt - (qd + h * qdd));
                    if (fabsf(td) > bc.effort) { sat = td > 0.f ? 1.f : -1.f; newly = true; }
                }
                if (!__any_sync(FULL, newly)) break;
            }
            invD_out = invD;
            return qd + h * qdd;
    };
    Kin kn;
    if (CONTACT) shapes_world(true);
    int pending = (obs != nullptr && nsteps == 0) ? t0 : -1;
    float u0n[NP], u1n[NP], uv[NP], uw[NP];
#pragma unroll
    for (int pp = 0; pp < NP; ++pp) { u0n[pp] = u1n[pp] = uv[pp] = uw[pp] = 0.f; }
    auto load_u = [&](int t) {
#pragma unroll
        for (int pp = 0; pp < NP; ++pp) {
            u0n[pp] = __ldg(&actions[((size_t)t * nu + ci0) * K + ka[pp]]);
            u1n[pp] = __ldg(&actions[((size_t)t * nu + ci1) * K + ka[pp]]);
            if (planar) { uv[pp] = __ldg(&actions[((size_t)t * nu + 0) * K + ka[pp]]); uw[pp] = __ldg(&actions[((size_t)t * nu + 1) * K + ka[pp]]); }
        }
    };
    if (nsteps > 0) load_u(t0);
    const int nsub = p.substeps;
#pragma unroll 1
    for (int t = t0; t < t0 + nsteps; ++t) {
        float tgt0[NP], pv[NP], pw[NP];
#pragma unroll
        for (int pp = 0; pp < NP; ++pp) { tgt0[pp] = cc0 * u0n[pp] + cc1 * u1n[pp]; pv[pp] = p.u_scale * uv[pp]; pw[pp] = p.u_scale * uw[pp]; }
        if (t + 1 < t0 + nsteps) load_u(t + 1);
#pragma unroll 1
        for (int sub = 0; sub < nsub; ++sub) {
            float vnew[NP];
#pragma unroll
            for (int pp = 0; pp < NP; ++pp) {
                float tgt = tgt0[pp];
                if (planar) {
                    // differential drive reduced to a planar base: body twist (v, omega) -> world-frame velocity targets of the three
                    // virtual joints; the forward axis turns with the current yaw (joint 2)
                    const float yaw = shfl_at<G>(q[pp], 2);
                    float sy, cy; sincos_cw(yaw, &sy, &cy);
                    if (i == 0) tgt = pv[pp] * (m.fwd_axis[0] * cy - m.fwd_axis[1] * sy);
                    if (i == 1) tgt = pv[pp] * (m.fwd_axis[0] * sy + m.fwd_axis[1] * cy);
                    if (i == 2) tgt = pw[pp];
                }
                kinematics<G, R>(bc, tr, q[pp], qd[pp], kn);
                if (sub == 0 && pending >= 0) write_obs(pending, kn, pp);
                float invD;
                vnew[pp] = articulation(kn, q[pp], qd[pp], tgt, invD);
                if (CONTACT && bval) {                       // hand-over to the contact phase
                    float* xa = xsa[pp] + L.jb0 + i * JBN;
                    stM3(xa, JB_R, kn.R); st3(xa, JB_O, kn.o); st3(xa, JB_SN, kn.S.n); st3(xa, JB_SF, kn.S.f);
                    xa[JB_VP] = vnew[pp]; xa[JB_INVD] = fminf(invD, 1.0e6f);       // 1 / max(D_j, 1e-6)
                }
            }
            if (sub == 0) pending = -1;
            if (CONTACT) {
                // ---- contacts on the predicted velocities
                __syncwarp();
                shapes_world(false);
                detect();
                if (ic == 0) for (int f = 0; f < m.nfree; ++f) if (m.free_gravity[f]) {
                    const int fb = L.fb0 + f * FBN;
                    xs[fb + FB_V] += h * m.gravity[0]; xs[fb + FB_V + 1] += h * m.gravity[1]; xs[fb + FB_V + 2] += h * m.gravity[2];
                }
                __syncwarp();
                solve_contacts(sub == nsub - 1);
                __syncwarp();
            }
            // ---- integrate
#pragma unroll
            for (int pp = 0; pp < NP; ++pp) {
                float vj = vnew[pp];
                if (CONTACT && bval) vj = xsa[pp][L.jb0 + i * JBN + JB_VP];
                float vn = fminf(fmaxf(vj, -bc.qd_max), bc.qd_max);
                float x = q[pp] + h * vn;
                if (x < bc.q_lo) { x = bc.q_lo; if (vn < 0.f) vn = 0.f; }
                if (x > bc.q_hi) { x = bc.q_hi; if (vn > 0.f) vn = 0.f; }
                if (bval) { q[pp] = x; qd[pp] = vn; }
            }
            if (CONTACT) integrate_free();
        }
        if (obs != nullptr) pending = t;
    }
    if (pending >= 0) {
#pragma unroll
        for (int pp = 0; pp < NP; ++pp) {
            kinematics<G, R>(bc, tr, q[pp], qd[pp], kn);
            write_obs(pending, kn, pp);
        }
    }
    if (state != nullptr) {
#pragma unroll
        for (int pp = 0; pp < NP; ++pp) if (kvala[pp] && bval) {
            state[(size_t)i * K + ka[pp]] = q[pp];
            state[(size_t)(nb + i) * K + ka[pp]] = qd[pp];
        }
        if (CONTACT && kvalc) for (int f = 0; f < m.nfree; ++f)
            for (int r = ic; r < 13; r += GC) state[(size_t)(2 * nb + 13 * f + r) * K + kc] = xs[L.fb0 + f * FBN + r];
    }
}

// dynamic shared memory of a team CTA; raises the kernel's limit on this device where it needs more than the default 48 KB
template <int G, int NB, bool CONTACT, int NCS, int GC, bool COMPACT>
int team_smem(MppibContext* c, size_t* smem_out) {
    const TLayout L(c->model.nb, c->model.nfree, c->model.nshapes, c->model.max_contacts, GC, COMPACT);
    const size_t smem = CONTACT ? sizeof(float) * (size_t)(32 / GC) * team_stride(L.total, GC) : 0;
    MPPIB_REQUIRE(smem <= 200 * 1024, "mppib_rollout: %zu bytes of shared memory per team CTA", smem);
    static size_t smem_attr[64] = {0};
    size_t& attr = smem_attr[c->device & 63];
    if (smem > 48 * 1024 && smem > attr) {
        MPPIB_CHECK_CUDA(cudaFuncSetAttribute(mppib_rollout_team_kernel<G, NB, CONTACT, NCS, GC, COMPACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    *smem_out = smem;
    return 0;
}

template <int G, int NB, bool CONTACT, int NCS, int GC, bool COMPACT>
int launch_team_t(MppibContext* c, const float* state0, const float* root0, float* state, const float* actions, int t0, int nsteps, float* obs, cudaStream_t s) {
    const int K = c->params.K;
    constexpr int RPW = 32 / GC;
    size_t smem = 0;
    if (int rc = team_smem<G, NB, CONTACT, NCS, GC, COMPACT>(c, &smem)) return rc;
    const int ctas = (K + RPW - 1) / RPW;
    mppib_rollout_team_kernel<G, NB, CONTACT, NCS, GC, COMPACT><<<ctas, 32, smem, s>>>(c->model, c->params, state0, root0, state, actions, t0, nsteps, obs);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// waves of resident CTAs a contact launch of this K needs on this device (CTAs per SM from shared memory and registers)
template <int G, int NB, int NCS, int GC, bool COMPACT>
int team_waves(MppibContext* c, int* waves) {
    size_t smem = 0;
    if (int rc = team_smem<G, NB, true, NCS, GC, COMPACT>(c, &smem)) return rc;
    int per_sm = 0;
    MPPIB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mppib_rollout_team_kernel<G, NB, true, NCS, GC, COMPACT>, 32, smem));
    MPPIB_REQUIRE(per_sm > 0, "mppib_rollout: a team CTA of %zu bytes of shared memory does not fit an SM", smem);
    const long long ctas = (c->params.K + 32 / GC - 1) / (32 / GC), slots = (long long)per_sm * c->num_sms;
    *waves = (int)((ctas + slots - 1) / slots);
    return 0;
}

// Layout of the per-rollout block of a contact scene (see CT_*): 9 - 16 joints always take the compact one.  Up to 8 joints the roomy
// one is faster per CTA, but its CTAs are larger: where it needs more waves of resident CTAs than the compact one at this K (BASELINE
// C3, K = 4 000 on 132 SMs: 1 000 CTAs, 7 per SM roomy, 9 per SM compact), the compact one runs.  Both layouts hold the same values,
// so the choice does not change the arithmetic.
template <int G, int NB, int NCS, int GC>
int launch_team_contact(MppibContext* c, const float* state0, const float* root0, float* state, const float* actions, int t0, int nsteps,
                        float* obs, cudaStream_t s) {
    if constexpr (G > 8) {
        return launch_team_t<G, NB, true, NCS, GC, true>(c, state0, root0, state, actions, t0, nsteps, obs, s);
    } else {
        int w_roomy = 0, w_compact = 0;
        if (int rc = team_waves<G, NB, NCS, GC, false>(c, &w_roomy)) return rc;
        if (int rc = team_waves<G, NB, NCS, GC, true>(c, &w_compact)) return rc;
        if (w_compact < w_roomy) return launch_team_t<G, NB, true, NCS, GC, true>(c, state0, root0, state, actions, t0, nsteps, obs, s);
        return launch_team_t<G, NB, true, NCS, GC, false>(c, state0, root0, state, actions, t0, nsteps, obs, s);
    }
}

// contact scenes: 8 lanes per rollout in the contact phase; coordinate slots per lane (compile time) = ceil((nb + 6 nfree) / 8)
template <int G, int NB>
int launch_team_g(MppibContext* c, bool contact, const float* state0, const float* root0, float* state, const float* actions, int t0, int nsteps, float* obs,
                  cudaStream_t s) {
    if (!contact) return launch_team_t<G, NB, false, 1, G, (G > 8)>(c, state0, root0, state, actions, t0, nsteps, obs, s);
    constexpr int GC = 8;
    const int ncs = (c->model.nb + 6 * c->model.nfree + GC - 1) / GC;
    switch (ncs) {
        case 1: return launch_team_contact<G, NB, 1, GC>(c, state0, root0, state, actions, t0, nsteps, obs, s);
        case 2: return launch_team_contact<G, NB, 2, GC>(c, state0, root0, state, actions, t0, nsteps, obs, s);
        case 3: return launch_team_contact<G, NB, 3, GC>(c, state0, root0, state, actions, t0, nsteps, obs, s);
        case 4: return launch_team_contact<G, NB, 4, GC>(c, state0, root0, state, actions, t0, nsteps, obs, s);
        default: MPPIB_REQUIRE(ncs <= MAXS_ALL, "mppib_rollout: %d coordinate slots per lane", ncs);
                 return launch_team_contact<G, NB, 5, GC>(c, state0, root0, state, actions, t0, nsteps, obs, s);
    }
}

}  // namespace

// trees / contact scenes with at most 16 bodies in depth-first order (every subtree a contiguous index range) and depth < 16
bool rollout_team_eligible(const MppibModel& m) {
    if (m.nb > 16) return false;
    for (int i = 0; i < m.nb; ++i) {
        if (m.parent[i] >= i) return false;
        int depth = 0;
        for (int j = i; j >= 0; j = m.parent[j]) ++depth;
        if (depth > (m.nb <= 8 ? 8 : 16)) return false;
    }
    // contiguity: body j > i is a descendant of i  <=>  j < end_i, where end_i = i + size of the subtree
    for (int i = 0; i < m.nb; ++i) {
        int size = 0, last = i;
        for (int j = i; j < m.nb; ++j) {
            bool desc = false;
            for (int a = j; a >= 0; a = m.parent[a]) if (a == i) { desc = true; break; }
            if (desc) { ++size; last = j; }
        }
        if (last != i + size - 1) return false;
    }
    if (m.planar_base && (m.nb < 3 || m.nu < 2)) return false;
    return true;
}

int launch_rollout_team(MppibContext* c, const float* state0, const float* root0, float* state, const float* actions, int t0, int nsteps,
                        float* obs, cudaStream_t s) {
    const MppibModel& m = c->model;
    const bool contact = m.nfree > 0 || m.nshapes > 0;
    if (contact) MPPIB_REQUIRE(root0 != nullptr, "mppib_rollout: root0 is required for scenes with free bodies / collision shapes");
#define TEAM_CASE(G, NB) return launch_team_g<G, NB>(c, contact, state0, root0, state, actions, t0, nsteps, obs, s)
    if (m.nb <= 4) { TEAM_CASE(8, 4); }
    if (m.nb <= 8) { TEAM_CASE(8, 8); }
    if (m.nb <= 12) { TEAM_CASE(16, 12); }
    TEAM_CASE(16, 16);
#undef TEAM_CASE
}
