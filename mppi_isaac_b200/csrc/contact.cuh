// contact.cuh -- free rigid bodies + contacts of the thread-per-rollout kernel (included by rollout.cu).
//
// Replaces PhysX rigid bodies / contact solve on the MPPI path (SURVEY.md 8(a) G1/G2, configs C3-C5).  The contact model itself
// (randomisation, shape poses, broad phase, box and sphere contacts, tangents, free-body integration) is contact_model.cuh, shared
// with rollout_team.cu.  This file keeps what is this kernel's own:
//   * the per-rollout working set in shared memory as [slot][lane] (same conflict-free layout as the articulation slots) and its
//     contact records (CT_*);
//   * contact detection with one thread per rollout, the oracle's loop orders;
//   * penalty spring-damper (contact_kp, contact_kd) integrated implicitly as a soft constraint on the PREDICTED velocities,
//     `contact_iters` Gauss-Seidel sweeps, box friction, capped recovery velocity; articulation links respond through a diagonal
//     joint-space compliance 1 / D_j (D_j from the ABA sweep), walking the chain of the contact's link.
#pragma once

#include "contact_model.cuh"

namespace contact {

// contact slots
// CT_KN / CT_KT1 / CT_KT2 hold INVERSES: 1 / (k_n + gamma), 1 / k_t1, 1 / k_t2 (0 = row disabled); CT_T1 caches the first tangent
enum : int { CT_P = 0, CT_N = 3, CT_D = 6, CT_MU = 7, CT_LN = 8, CT_LT1 = 9, CT_LT2 = 10, CT_IDS = 11, CT_KN = 12, CT_KT1 = 13, CT_KT2 = 14, CT_T1 = 15, CTN = 18 };

struct Layout {
    int fb0, sh0, ct0, jv0, net0, total;   // offsets in slots
    __host__ __device__ Layout(int nb, int nfree, int nshapes, int max_contacts) {
        fb0 = 0; sh0 = fb0 + nfree * FBN; ct0 = sh0 + nshapes * SHN; jv0 = ct0 + max_contacts * CTN;
        net0 = jv0 + 3 * nb; total = net0 + 3 * MPPIB_MAX_SLOTS;
    }
};

#define XS(i) xs[(i) * 32 + lane]

__device__ __forceinline__ V3 ldx3(const float* xs, int base, int lane) { return mk(XS(base), XS(base + 1), XS(base + 2)); }
__device__ __forceinline__ void stx3(float* xs, int base, int lane, V3 v) { XS(base) = v.x; XS(base + 1) = v.y; XS(base + 2) = v.z; }
__device__ __forceinline__ M3 ldxM3(const float* xs, int b, int lane) {
    M3 m; m.m00 = XS(b); m.m01 = XS(b + 1); m.m02 = XS(b + 2); m.m10 = XS(b + 3); m.m11 = XS(b + 4); m.m12 = XS(b + 5); m.m20 = XS(b + 6); m.m21 = XS(b + 7); m.m22 = XS(b + 8); return m;
}
__device__ __forceinline__ void stxM3(float* xs, int b, int lane, const M3& m) {
    XS(b) = m.m00; XS(b + 1) = m.m01; XS(b + 2) = m.m02; XS(b + 3) = m.m10; XS(b + 4) = m.m11; XS(b + 5) = m.m12; XS(b + 6) = m.m20; XS(b + 7) = m.m21; XS(b + 8) = m.m22;
}
// rotation and world inverse inertia of free body fb from its quaternion
__device__ __forceinline__ void refresh_free(float* xs, int lane, int fb) {
    const Quat q = {XS(fb + FB_Q), XS(fb + FB_Q + 1), XS(fb + FB_Q + 2), XS(fb + FB_Q + 3)};
    const M3 R = quat_to_R(q);
    stxM3(xs, fb + FB_R, lane, R);
    const S3 Iw = world_inv_inertia(R, ldx3(xs, fb + FB_IINV, lane));
    XS(fb + FB_IW + 0) = Iw.xx; XS(fb + FB_IW + 1) = Iw.yy; XS(fb + FB_IW + 2) = Iw.zz;
    XS(fb + FB_IW + 3) = Iw.xy; XS(fb + FB_IW + 4) = Iw.xz; XS(fb + FB_IW + 5) = Iw.yz;
}

// one-time per rollout: randomised shape / body parameters and the free bodies' initial state
__device__ __forceinline__ void init(const MppibModel& m, const MppibParams& p, const Layout& L, float* xs, int lane, uint32_t kg,
                                     const float* __restrict__ root0, const float* __restrict__ state, bool from_root, int K, int k) {
    for (int s = 0; s < m.nshapes; ++s) {
        V3 half; float mu, rad;
        shape_params(m, p, kg, s, half, mu, rad);
        const int sb = L.sh0 + s * SHN;
        stx3(xs, sb + SH_HALF, lane, half);
        XS(sb + SH_MU) = mu;
        XS(sb + SH_RAD) = rad;
    }
    for (int f = 0; f < m.nfree; ++f) {
        const int fb = L.fb0 + f * FBN;
        float inv_mass; V3 half, iinv;
        free_params(m, p, kg, f, inv_mass, half, iinv);
        XS(fb + FB_MASS) = inv_mass;
        stx3(xs, fb + FB_HALF, lane, half);
        stx3(xs, fb + FB_IINV, lane, iinv);
        for (int r = 0; r < 13; ++r)
            XS(fb + r) = from_root ? root0[13 * m.free_actor[f] + r] : state[(size_t)(2 * m.nb + 13 * f + r) * K + k];
        refresh_free(xs, lane, fb);
    }
    for (int s = 0; s < 3 * MPPIB_MAX_SLOTS; ++s) XS(L.net0 + s) = 0.f;
}

// Articulation side of a contact.  The velocity of point pt per unit velocity of joint j is S_j.f + S_j.n x pt (S about the
// world origin), so along a direction d it is  S_j.f . d + S_j.n . (pt x d):  one 6-vector dot per joint and no cross
// product inside the chain walk.  jv0 + j: velocity correction of joint j, jv0 + nb + j: 1 / D_j, jv0 + 2 nb + j: predicted qd.
template <int NSLOT, bool CHAIN>
__device__ __forceinline__ int up(const MppibModel& m, int j) { return CHAIN ? j - 1 : m.parent[j]; }

template <int NSLOT, bool CHAIN>
__device__ __forceinline__ V3 point_velocity(const MppibModel& m, const Layout& L, const float* sm, const float* xs, int lane, int ref, V3 pt) {
    if (ref == REF_STATIC) return mk(0, 0, 0);
    if (ref >= REF_FREE0) {
        const int fb = L.fb0 + (ref - REF_FREE0) * FBN;
        return ldx3(xs, fb + FB_V, lane) + cross(ldx3(xs, fb + FB_W, lane), pt - ldx3(xs, fb + FB_X, lane));
    }
    V3 w = mk(0, 0, 0), v = mk(0, 0, 0);       // spatial velocity of the link = sum over the chain of qd_j S_j
    for (int j = ref; j >= 0; j = up<NSLOT, CHAIN>(m, j)) {
        const float qd = XS(L.jv0 + 2 * m.nb + j) + XS(L.jv0 + j);
        const V6 S = ld6(sm, j * NSLOT + F_S, lane);
        w = w + qd * S.n; v = v + qd * S.f;
    }
    return v + cross(w, pt);
}

template <int NSLOT, bool CHAIN>
__device__ __forceinline__ float inv_mass(const MppibModel& m, const Layout& L, const float* sm, const float* xs, int lane, int refA, int refB, V3 pt, V3 dir) {
    float k = 0.f;
    const V3 mom = cross(pt, dir);
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const int ref = e == 0 ? refA : refB;
        if (ref >= 0 && ref < REF_FREE0) {
            for (int j = ref; j >= 0; j = up<NSLOT, CHAIN>(m, j)) {
                const V6 S = ld6(sm, j * NSLOT + F_S, lane);
                const float jd = dot(S.f, dir) + dot(S.n, mom);
                k += jd * jd * XS(L.jv0 + m.nb + j);
            }
        } else if (ref >= REF_FREE0) {
            const int fb = L.fb0 + (ref - REF_FREE0) * FBN;
            const V3 r = pt - ldx3(xs, fb + FB_X, lane);
            const V3 rxn = cross(r, dir);
            const S3 Iw = {XS(fb + FB_IW), XS(fb + FB_IW + 1), XS(fb + FB_IW + 2), XS(fb + FB_IW + 3), XS(fb + FB_IW + 4), XS(fb + FB_IW + 5)};
            k += XS(fb + FB_MASS) + dot(cross(mul(Iw, rxn), r), dir);
        }
    }
    return k;
}

// impulse vector P at pt: +P on side A, -P on side B
template <int NSLOT, bool CHAIN>
__device__ __forceinline__ void apply_impulse(const MppibModel& m, const Layout& L, const float* sm, float* xs, int lane, int refA, int refB, V3 pt, V3 P) {
    const V3 mom = cross(pt, P);
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const int ref = e == 0 ? refA : refB;
        const float sgn = e == 0 ? 1.0f : -1.0f;
        if (ref >= 0 && ref < REF_FREE0) {
            for (int j = ref; j >= 0; j = up<NSLOT, CHAIN>(m, j)) {
                const V6 S = ld6(sm, j * NSLOT + F_S, lane);
                XS(L.jv0 + j) += sgn * (dot(S.f, P) + dot(S.n, mom)) * XS(L.jv0 + m.nb + j);
            }
        } else if (ref >= REF_FREE0) {
            const int fb = L.fb0 + (ref - REF_FREE0) * FBN;
            const V3 r = pt - ldx3(xs, fb + FB_X, lane);
            const float im = sgn * XS(fb + FB_MASS);
            XS(fb + FB_V) += im * P.x; XS(fb + FB_V + 1) += im * P.y; XS(fb + FB_V + 2) += im * P.z;
            const S3 Iw = {XS(fb + FB_IW), XS(fb + FB_IW + 1), XS(fb + FB_IW + 2), XS(fb + FB_IW + 3), XS(fb + FB_IW + 4), XS(fb + FB_IW + 5)};
            const V3 dw = mul(Iw, cross(r, P));
            XS(fb + FB_W) += sgn * dw.x; XS(fb + FB_W + 1) += sgn * dw.y; XS(fb + FB_W + 2) += sgn * dw.z;
        }
    }
}

__device__ __forceinline__ void add_contact(const MppibModel& m, const Layout& L, float* xs, int lane, int& nc, int refA, int refB, int slotA, int slotB, V3 pt, V3 n, float d, float mu) {
    if (nc >= m.max_contacts) return;
    const int cb = L.ct0 + nc * CTN;
    ++nc;
    stx3(xs, cb + CT_P, lane, pt); stx3(xs, cb + CT_N, lane, n);
    XS(cb + CT_D) = d; XS(cb + CT_MU) = mu; XS(cb + CT_LN) = 0.f; XS(cb + CT_LT1) = 0.f; XS(cb + CT_LT2) = 0.f;
    XS(cb + CT_IDS) = __int_as_float(pack_sides(refA, refB, slotA, slotB));
}

// sample points of box a inside box b -> contacts; flip: a is the B side of the pair
__device__ __forceinline__ void points_in_box(const MppibModel& m, const Layout& L, float* xs, int lane, int& nc, int a, int b, bool flip) {
    const int sa = L.sh0 + a * SHN, sb = L.sh0 + b * SHN;
    const M3 Ra = ldxM3(xs, sa + SH_R, lane), Rb = ldxM3(xs, sb + SH_R, lane);
    const V3 ca = ldx3(xs, sa + SH_C, lane), cbv = ldx3(xs, sb + SH_C, lane);
    const V3 ha = ldx3(xs, sa + SH_HALF, lane), hb = ldx3(xs, sb + SH_HALF, lane);
    const float mu = 0.5f * (XS(sa + SH_MU) + XS(sb + SH_MU));
    const int refa = shape_ref(m, a), refb = shape_ref(m, b), slota = m.shape_slot[a], slotb = m.shape_slot[b];
    bool c0, c1, c2; face_axes(Rb, ca, cbv, hb, c0, c1, c2);
#pragma unroll 1
    for (int idx = 0; idx < 27; ++idx) {
        if (idx == 13) continue;
        V3 pt, n; float pen;
        if (!box_point(idx, Ra, ca, ha, Rb, cbv, hb, c0, c1, c2, m.contact_margin, pt, n, pen)) continue;
        if (!flip) add_contact(m, L, xs, lane, nc, refa, refb, slota, slotb, pt, n, pen, mu);
        else add_contact(m, L, xs, lane, nc, refb, refa, slotb, slota, pt, mk(-n.x, -n.y, -n.z), pen, mu);
    }
}

// ONE contact of a sphere against a box or a sphere.  The normal of a contact pushes side A out of side B.
__device__ __forceinline__ void sphere_pair(const MppibModel& m, const Layout& L, float* xs, int lane, int& nc, int a, int b) {
    const int sa = L.sh0 + a * SHN, sb = L.sh0 + b * SHN;
    const float mu = 0.5f * (XS(sa + SH_MU) + XS(sb + SH_MU));
    const int refa = shape_ref(m, a), refb = shape_ref(m, b), slota = m.shape_slot[a], slotb = m.shape_slot[b];
    const V3 ca = ldx3(xs, sa + SH_C, lane), cbv = ldx3(xs, sb + SH_C, lane);
    const bool sph_a = m.shape_type[a] == MPPIB_SHAPE_SPHERE;
    V3 pt, n; float pen; bool hit;
    if (sph_a && m.shape_type[b] == MPPIB_SHAPE_SPHERE) hit = sphere_sphere(ca, XS(sa + SH_HALF), cbv, XS(sb + SH_HALF), m.contact_margin, pt, n, pen);
    else {
        const int sx = sph_a ? sb : sa;
        hit = sphere_box(sph_a ? ca : cbv, XS((sph_a ? sa : sb) + SH_HALF), ldxM3(xs, sx + SH_R, lane), sph_a ? cbv : ca, ldx3(xs, sx + SH_HALF, lane),
                         m.contact_margin, pt, n, pen);
        if (!sph_a) n = mk(-n.x, -n.y, -n.z);
    }
    if (hit) add_contact(m, L, xs, lane, nc, refa, refb, slota, slotb, pt, n, pen, mu);
}

// contacts of the ordered pair (a, b): boxes by sample points in both directions, anything with a sphere analytically
__device__ __forceinline__ void pair_contacts(const MppibModel& m, const Layout& L, float* xs, int lane, int& nc, int a, int b) {
    if (m.shape_type[a] == MPPIB_SHAPE_SPHERE || m.shape_type[b] == MPPIB_SHAPE_SPHERE) { sphere_pair(m, L, xs, lane, nc, a, b); return; }
    points_in_box(m, L, xs, lane, nc, a, b, false);
    points_in_box(m, L, xs, lane, nc, b, a, true);
}

__device__ __forceinline__ bool near_shapes(const MppibModel& m, const Layout& L, const float* xs, int lane, int a, int b) {
    const int sa = L.sh0 + a * SHN, sb = L.sh0 + b * SHN;
    const V3 d = ldx3(xs, sa + SH_C, lane) - ldx3(xs, sb + SH_C, lane);
    const bool sph = m.shape_type[a] == MPPIB_SHAPE_SPHERE || m.shape_type[b] == MPPIB_SHAPE_SPHERE;
    if (!near_bounds(d, XS(sa + SH_RAD), XS(sb + SH_RAD), sph, m.contact_margin)) return false;
    if (sph) return true;                                                       // the narrow phase is exact and cheap
    return near_boxes(d, ldxM3(xs, sa + SH_R, lane), ldx3(xs, sa + SH_HALF, lane), ldxM3(xs, sb + SH_R, lane), ldx3(xs, sb + SH_HALF, lane),
                      m.contact_margin);
}

// world poses of all shapes (articulation frames from sweep 1, static actors from root0, free bodies from their state)
// `statics`: true once per rollout (static boxes never move inside a rollout), false in every substep (links and free bodies)
template <int NSLOT>
__device__ __forceinline__ void shapes_world(const MppibModel& m, const Layout& L, const float* sm, float* xs, int lane, const M3& Rbase, V3 obase,
                                             const float* __restrict__ root0, bool statics) {
    for (int s = 0; s < m.nshapes; ++s) {
        if ((m.shape_owner_kind[s] == MPPIB_OWNER_STATIC) != statics) continue;
        M3 Ro; V3 po;
        const int kind = m.shape_owner_kind[s];
        if (kind == MPPIB_OWNER_STATIC) root_pose(root0, m.shape_actor[s], Ro, po);
        else if (kind == MPPIB_OWNER_LINK) {
            const int b = m.shape_owner[s];
            if (b >= 0) { Ro = ldM3(sm, b * NSLOT + F_R, lane); po = ld3(sm, b * NSLOT + F_O, lane); }
            else { Ro = Rbase; po = obase; }
        } else {
            const int fb = L.fb0 + m.shape_owner[s] * FBN;
            Ro = ldxM3(xs, fb + FB_R, lane); po = ldx3(xs, fb + FB_X, lane);
        }
        M3 R; V3 c; shape_pose(m, s, Ro, po, R, c);
        const int sb = L.sh0 + s * SHN;
        stxM3(xs, sb + SH_R, lane, R);
        stx3(xs, sb + SH_C, lane, c);
    }
}

// Ground points of a free box (oracle.cpp ContactWorld::detect): bit c is set if corner c is among the 4 lowest of the 8 (ties by
// corner index) and below the ground margin; z[c] is the same expression as the corner's pt.z.  With at most 4 corners below the
// margin those are the answer (a corner below it has only corners below it beneath it): the ranks are needed only above h ~ 0.026 s.
__device__ __forceinline__ uint32_t ground_corner_mask(const float (&z)[8], float margin) {
    uint32_t below = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) below |= (uint32_t)(z[c] < margin) << c;
    if (__popc(below) <= 4) return below;
    uint32_t keep = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        int rank = 0;
#pragma unroll
        for (int o = 0; o < 8; ++o) rank += z[o] < z[c] || (z[o] == z[c] && o < c);
        if (rank < 4) keep |= 1u << c;
    }
    return keep & below;
}

__device__ __forceinline__ int detect(const MppibModel& m, const Layout& L, float* xs, int lane, const uint32_t* __restrict__ bmask) {
    int nc = 0;
    const int ns = m.nshapes;
    for (int a = 0; a < ns; ++a) {
        if (m.shape_owner_kind[a] != MPPIB_OWNER_FREE) continue;
        const int sa = L.sh0 + a * SHN;
        if (m.ground_plane) {
            const M3 Ra = ldxM3(xs, sa + SH_R, lane); const V3 ca = ldx3(xs, sa + SH_C, lane), ha = ldx3(xs, sa + SH_HALF, lane);
            const float mu = 0.5f * (XS(sa + SH_MU) + m.ground_friction);
            float z[8];                                               // at most the 4 lowest corners are ground points
#pragma unroll
            for (int idx = 0; idx < 8; ++idx) {
                const int ix = (idx >> 2) * 2 - 1, iy = ((idx >> 1) & 1) * 2 - 1, iz = (idx & 1) * 2 - 1;
                z[idx] = (mul(Ra, mk(ix * ha.x, iy * ha.y, iz * ha.z)) + ca).z;
            }
            const uint32_t keep = ground_corner_mask(z, m.ground_margin);
#pragma unroll 1
            for (int idx = 0; idx < 8; ++idx) {
                const int ix = (idx >> 2) * 2 - 1, iy = ((idx >> 1) & 1) * 2 - 1, iz = (idx & 1) * 2 - 1;
                const V3 pt = mul(Ra, mk(ix * ha.x, iy * ha.y, iz * ha.z)) + ca;
                if ((keep >> idx) & 1u) add_contact(m, L, xs, lane, nc, shape_ref(m, a), REF_STATIC, m.shape_slot[a], -1, pt, mk(0, 0, 1), -pt.z, mu);
            }
        }
        for (uint32_t mask = bmask[a]; mask; mask &= mask - 1) {          // partners in ascending order, as the oracle's loop visits them
            const int b = __ffs(mask) - 1;
            if (!near_shapes(m, L, xs, lane, a, b)) continue;
            pair_contacts(m, L, xs, lane, nc, a, b);
        }
    }
    for (int a = 0; a < ns; ++a) {   // articulation link vs static shape
        if (m.shape_owner_kind[a] != MPPIB_OWNER_LINK) continue;
        for (uint32_t mask = bmask[a]; mask; mask &= mask - 1) {
            const int b = __ffs(mask) - 1;
            if (!near_shapes(m, L, xs, lane, a, b)) continue;
            pair_contacts(m, L, xs, lane, nc, a, b);
        }
    }
    return nc;
}

// Gauss-Seidel soft-constraint solve on the predicted velocities; fills dqv (joint velocity corrections) and the net forces
template <int NSLOT, bool CHAIN>
__device__ __forceinline__ void solve(const MppibModel& m, const Layout& L, const float* sm, float* xs, int lane, int nc, float h) {
    const float kp = m.contact_kp, kd = m.contact_kd;
    const float gamma = 1.0f / (h * (h * kp + kd)), beta = h * kp / (h * kp + kd), ih = 1.0f / h;
    // per contact, once: tangent frame, effective inverse masses along it (poses are frozen within a substep) -> stored as
    // the reciprocals the sweeps multiply with, and the velocity bias of the normal row
#pragma unroll 1
    for (int c = 0; c < nc; ++c) {
        const int cb = L.ct0 + c * CTN;
        const int ids = __float_as_int(XS(cb + CT_IDS));
        const int refA = ref_a(ids), refB = ref_b(ids);
        const V3 pt = ldx3(xs, cb + CT_P, lane), n = ldx3(xs, cb + CT_N, lane);
        V3 t1, t2; tangents(n, t1, t2);
        const float kn = inv_mass<NSLOT, CHAIN>(m, L, sm, xs, lane, refA, refB, pt, n);
        const float kt1 = inv_mass<NSLOT, CHAIN>(m, L, sm, xs, lane, refA, refB, pt, t1);
        const float kt2 = inv_mass<NSLOT, CHAIN>(m, L, sm, xs, lane, refA, refB, pt, t2);
        XS(cb + CT_KN) = kn > K_ROW_MIN ? 1.0f / (kn + gamma) : 0.f;
        XS(cb + CT_KT1) = kt1 > K_ROW_MIN ? 1.0f / kt1 : 0.f;
        XS(cb + CT_KT2) = kt2 > K_ROW_MIN ? 1.0f / kt2 : 0.f;
        stx3(xs, cb + CT_T1, lane, t1);
        const float d = XS(cb + CT_D);
        XS(cb + CT_D) = d > 0.f ? fminf(beta * d * ih, m.max_depen) : d * ih;      // from here on: the bias velocity
    }
#pragma unroll 1
    for (int it = 0; it < m.contact_iters; ++it) {
#pragma unroll 1
        for (int c = 0; c < nc; ++c) {
            const int cb = L.ct0 + c * CTN;
            const float ikn = XS(cb + CT_KN);
            if (!(ikn > 0.f)) continue;
            const int ids = __float_as_int(XS(cb + CT_IDS));
            const int refA = ref_a(ids), refB = ref_b(ids);
            const V3 pt = ldx3(xs, cb + CT_P, lane), n = ldx3(xs, cb + CT_N, lane), t1 = ldx3(xs, cb + CT_T1, lane);
            const V3 t2 = cross(n, t1);
            const float bias = XS(cb + CT_D), mu = XS(cb + CT_MU), ikt1 = XS(cb + CT_KT1), ikt2 = XS(cb + CT_KT2);
            // one visit = normal row + two friction rows solved from the SAME relative velocity, then one impulse application
            const V3 vr = point_velocity<NSLOT, CHAIN>(m, L, sm, xs, lane, refA, pt) - point_velocity<NSLOT, CHAIN>(m, L, sm, xs, lane, refB, pt);
            const float ln = XS(cb + CT_LN), lt1 = XS(cb + CT_LT1), lt2 = XS(cb + CT_LT2);
            const float ln_new = fmaxf(0.f, ln + (-dot(vr, n) + bias - gamma * ln) * ikn);
            const float lim = mu * ln_new;
            const float lt1_new = ikt1 > 0.f ? fminf(fmaxf(lt1 - dot(vr, t1) * ikt1, -lim), lim) : lt1;
            const float lt2_new = ikt2 > 0.f ? fminf(fmaxf(lt2 - dot(vr, t2) * ikt2, -lim), lim) : lt2;
            const V3 dP = (ln_new - ln) * n + (lt1_new - lt1) * t1 + (lt2_new - lt2) * t2;
            XS(cb + CT_LN) = ln_new; XS(cb + CT_LT1) = lt1_new; XS(cb + CT_LT2) = lt2_new;
            apply_impulse<NSLOT, CHAIN>(m, L, sm, xs, lane, refA, refB, pt, dP);
        }
    }
    for (int s = 0; s < 3 * MPPIB_MAX_SLOTS; ++s) XS(L.net0 + s) = 0.f;
    for (int c = 0; c < nc; ++c) {
        const int cb = L.ct0 + c * CTN;
        const int ids = __float_as_int(XS(cb + CT_IDS));
        const int slotA = slot_a(ids), slotB = slot_b(ids);
        if (slotA < 0 && slotB < 0) continue;
        const V3 n = ldx3(xs, cb + CT_N, lane), t1 = ldx3(xs, cb + CT_T1, lane);
        const V3 t2 = cross(n, t1);
        const V3 F = ih * (XS(cb + CT_LN) * n + XS(cb + CT_LT1) * t1 + XS(cb + CT_LT2) * t2);
        if (slotA >= 0) { XS(L.net0 + 3 * slotA) += F.x; XS(L.net0 + 3 * slotA + 1) += F.y; XS(L.net0 + 3 * slotA + 2) += F.z; }
        if (slotB >= 0) { XS(L.net0 + 3 * slotB) -= F.x; XS(L.net0 + 3 * slotB + 1) -= F.y; XS(L.net0 + 3 * slotB + 2) -= F.z; }
    }
}

__device__ __forceinline__ void integrate_free(const MppibModel& m, const Layout& L, float* xs, int lane, float h) {
    for (int f = 0; f < m.nfree; ++f) {
        const int fb = L.fb0 + f * FBN;
        V3 x = ldx3(xs, fb + FB_X, lane);
        Quat q = {XS(fb + FB_Q), XS(fb + FB_Q + 1), XS(fb + FB_Q + 2), XS(fb + FB_Q + 3)};
        integrate_pose(x, q, ldx3(xs, fb + FB_V, lane), ldx3(xs, fb + FB_W, lane), h);
        stx3(xs, fb + FB_X, lane, x);
        XS(fb + FB_Q) = q.x; XS(fb + FB_Q + 1) = q.y; XS(fb + FB_Q + 2) = q.z; XS(fb + FB_Q + 3) = q.w;
        refresh_free(xs, lane, fb);
    }
}

}  // namespace contact
