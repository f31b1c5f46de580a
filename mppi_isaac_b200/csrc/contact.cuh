// contact.cuh -- free rigid bodies + box contacts of the rollout kernel (included by rollout.cu).
//
// Replaces PhysX rigid bodies / contact solve on the MPPI path (SURVEY.md 8(a) G1/G2, configs C3-C5).  Spec
// (DESIGN.md section 2, restated independently by oracle/oracle.cpp ContactWorld):
//   * boxes only; contact points = the 26 surface sample points of one box inside the other (both directions, with a
//     speculative margin) and the 8 corners against the ground plane; normal = least-penetration face among the slabs
//     the other box's centre lies outside of;
//   * penalty spring-damper (contact_kp, contact_kd) integrated implicitly as a soft constraint on the PREDICTED
//     velocities, `contact_iters` Gauss-Seidel sweeps, box friction, capped recovery velocity;
//   * articulation links respond through a diagonal joint-space compliance 1 / D_j (D_j from the ABA sweep).
// Per-rollout working set in shared memory as [slot][lane] (same conflict-free layout as the articulation slots).
#pragma once

namespace contact {

enum : int { REF_STATIC = -1, REF_FREE0 = 64 };
// free body slots
// FB_MASS holds the INVERSE mass
enum : int { FB_X = 0, FB_Q = 3, FB_V = 7, FB_W = 10, FB_MASS = 13, FB_HALF = 14, FB_IINV = 17, FB_R = 20, FB_IW = 29, FBN = 35 };
// world shape slots
enum : int { SH_R = 0, SH_C = 9, SH_HALF = 12, SH_MU = 15, SH_RAD = 16, SHN = 17 };
// contact slots
// CT_KN / CT_KT1 / CT_KT2 hold INVERSES: 1 / (k_n + gamma), 1 / k_t1, 1 / k_t2 (0 = row disabled); CT_T1 caches the first tangent
// a contact row whose effective inverse mass is below K_ROW_MIN [1/kg] is dropped (bodies that cannot move along that direction; same
// threshold in oracle.cpp -- an exact `> 0` would depend on the rotation arithmetic producing exact zeros)
constexpr float K_ROW_MIN = 1e-9f;
enum : int { CT_P = 0, CT_N = 3, CT_D = 6, CT_MU = 7, CT_LN = 8, CT_LT1 = 9, CT_LT2 = 10, CT_IDS = 11, CT_KN = 12, CT_KT1 = 13, CT_KT2 = 14, CT_T1 = 15, CTN = 18 };

struct Layout {
    int fb0, sh0, ct0, jv0, net0, total;   // offsets in slots
    __host__ __device__ Layout(int nb, int nfree, int nshapes, int max_contacts) {
        fb0 = 0; sh0 = fb0 + nfree * FBN; ct0 = sh0 + nshapes * SHN; jv0 = ct0 + max_contacts * CTN;
        net0 = jv0 + 3 * nb; total = net0 + 3 * MPPIB_MAX_SLOTS;
    }
};

#define XS(i) xs[(i) * 32 + lane]

__device__ __forceinline__ uint4 philox(uint4 c, uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll 1
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
    float s, c; sincospif(2.0f * u01(b), &s, &c);
    z0 = r * c; z1 = r * s;
}
// per-rollout size / mass / friction draws of one actor (same counters as oracle actor_noise)
__device__ __forceinline__ void actor_noise(const MppibParams& p, uint32_t kg, int actor, V3& nsize, float& umass, float& ufric) {
    const uint4 r0 = philox(make_uint4(kg, (uint32_t)actor, 0x5EEDu, 0u), p.rand_seed, 0x4D505049u);
    const uint4 r1 = philox(make_uint4(kg, (uint32_t)actor, 0x5EEDu, 1u), p.rand_seed, 0x4D505049u);
    float dummy;
    box_muller(r0.x, r0.y, nsize.x, nsize.y);
    box_muller(r0.z, r0.w, nsize.z, dummy);
    umass = 2.0f * u01(r1.x) - 1.0f;
    ufric = 2.0f * u01(r1.y) - 1.0f;
}

__device__ __forceinline__ V3 ldx3(const float* xs, int base, int lane) { return mk(XS(base), XS(base + 1), XS(base + 2)); }
__device__ __forceinline__ void stx3(float* xs, int base, int lane, V3 v) { XS(base) = v.x; XS(base + 1) = v.y; XS(base + 2) = v.z; }
__device__ __forceinline__ M3 ldxM3(const float* xs, int b, int lane) {
    M3 m; m.m00 = XS(b); m.m01 = XS(b + 1); m.m02 = XS(b + 2); m.m10 = XS(b + 3); m.m11 = XS(b + 4); m.m12 = XS(b + 5); m.m20 = XS(b + 6); m.m21 = XS(b + 7); m.m22 = XS(b + 8); return m;
}
__device__ __forceinline__ void stxM3(float* xs, int b, int lane, const M3& m) {
    XS(b) = m.m00; XS(b + 1) = m.m01; XS(b + 2) = m.m02; XS(b + 3) = m.m10; XS(b + 4) = m.m11; XS(b + 5) = m.m12; XS(b + 6) = m.m20; XS(b + 7) = m.m21; XS(b + 8) = m.m22;
}
__device__ __forceinline__ M3 mulMM(const M3& a, const M3& b) {
    M3 o;
    o.m00 = a.m00 * b.m00 + a.m01 * b.m10 + a.m02 * b.m20; o.m01 = a.m00 * b.m01 + a.m01 * b.m11 + a.m02 * b.m21; o.m02 = a.m00 * b.m02 + a.m01 * b.m12 + a.m02 * b.m22;
    o.m10 = a.m10 * b.m00 + a.m11 * b.m10 + a.m12 * b.m20; o.m11 = a.m10 * b.m01 + a.m11 * b.m11 + a.m12 * b.m21; o.m12 = a.m10 * b.m02 + a.m11 * b.m12 + a.m12 * b.m22;
    o.m20 = a.m20 * b.m00 + a.m21 * b.m10 + a.m22 * b.m20; o.m21 = a.m20 * b.m01 + a.m21 * b.m11 + a.m22 * b.m21; o.m22 = a.m20 * b.m02 + a.m21 * b.m12 + a.m22 * b.m22;
    return o;
}

// world inverse inertia R diag(Iinv) R^T of free body f, and its rotation, from the quaternion
__device__ __forceinline__ void refresh_free(float* xs, int lane, int fb) {
    const Quat q = {XS(fb + FB_Q), XS(fb + FB_Q + 1), XS(fb + FB_Q + 2), XS(fb + FB_Q + 3)};
    const M3 R = quat_to_R(q);
    stxM3(xs, fb + FB_R, lane, R);
    const float i0 = XS(fb + FB_IINV), i1 = XS(fb + FB_IINV + 1), i2 = XS(fb + FB_IINV + 2);
    XS(fb + FB_IW + 0) = R.m00 * i0 * R.m00 + R.m01 * i1 * R.m01 + R.m02 * i2 * R.m02;
    XS(fb + FB_IW + 1) = R.m10 * i0 * R.m10 + R.m11 * i1 * R.m11 + R.m12 * i2 * R.m12;
    XS(fb + FB_IW + 2) = R.m20 * i0 * R.m20 + R.m21 * i1 * R.m21 + R.m22 * i2 * R.m22;
    XS(fb + FB_IW + 3) = R.m00 * i0 * R.m10 + R.m01 * i1 * R.m11 + R.m02 * i2 * R.m12;
    XS(fb + FB_IW + 4) = R.m00 * i0 * R.m20 + R.m01 * i1 * R.m21 + R.m02 * i2 * R.m22;
    XS(fb + FB_IW + 5) = R.m10 * i0 * R.m20 + R.m11 * i1 * R.m21 + R.m12 * i2 * R.m22;
}

// one-time per rollout: randomised shape / body parameters and the free bodies' initial state
__device__ __forceinline__ void init(const MppibModel& m, const MppibParams& p, const Layout& L, float* xs, int lane, uint32_t kg,
                                     const float* __restrict__ root0, const float* __restrict__ state, bool from_root, int K, int k) {
    for (int s = 0; s < m.nshapes; ++s) {
        V3 half = mk(m.shape_half[s][0], m.shape_half[s][1], m.shape_half[s][2]);
        float mu = m.shape_friction[s];
        if (m.shape_actor[s] >= 0) {
            V3 ns; float um, uf; actor_noise(p, kg, m.shape_actor[s], ns, um, uf);
            half.x += 0.5f * m.shape_size_sigma[s][0] * ns.x; half.y += 0.5f * m.shape_size_sigma[s][1] * ns.y; half.z += 0.5f * m.shape_size_sigma[s][2] * ns.z;
            mu *= 1.0f + m.shape_fric_pct[s] * uf;
        }
        const int sb = L.sh0 + s * SHN;
        stx3(xs, sb + SH_HALF, lane, half);
        XS(sb + SH_MU) = mu;
        // bounding radius; a sphere shape (isaacgym_utils.py:42-52: gym.create_sphere(radius = size[0])) keeps its radius in half.x
        XS(sb + SH_RAD) = m.shape_type[s] == MPPIB_SHAPE_SPHERE ? half.x : sqrtf(dot(half, half));
    }
    for (int f = 0; f < m.nfree; ++f) {
        const int fb = L.fb0 + f * FBN;
        V3 ns; float um, uf; actor_noise(p, kg, m.free_actor[f], ns, um, uf);
        const float mass = m.free_mass[f] * (1.0f + m.free_mass_pct[f] * um);
        V3 sg = mk(0, 0, 0);
        for (int s = 0; s < m.nshapes; ++s)
            if (m.shape_owner_kind[s] == MPPIB_OWNER_FREE && m.shape_owner[s] == f) { sg = mk(m.shape_size_sigma[s][0], m.shape_size_sigma[s][1], m.shape_size_sigma[s][2]); break; }
        const V3 half = mk(m.free_half[f][0] + 0.5f * sg.x * ns.x, m.free_half[f][1] + 0.5f * sg.y * ns.y, m.free_half[f][2] + 0.5f * sg.z * ns.z);
        const float m3 = mass / 3.0f;
        XS(fb + FB_MASS) = 1.0f / mass;
        stx3(xs, fb + FB_HALF, lane, half);
        XS(fb + FB_IINV) = 1.0f / (m3 * (half.y * half.y + half.z * half.z));
        XS(fb + FB_IINV + 1) = 1.0f / (m3 * (half.x * half.x + half.z * half.z));
        XS(fb + FB_IINV + 2) = 1.0f / (m3 * (half.x * half.x + half.y * half.y));
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

__device__ __forceinline__ int shape_ref(const MppibModel& m, int s) {
    const int kind = m.shape_owner_kind[s];
    if (kind == MPPIB_OWNER_FREE) return REF_FREE0 + m.shape_owner[s];
    if (kind == MPPIB_OWNER_LINK && m.shape_owner[s] >= 0) return m.shape_owner[s];
    return REF_STATIC;
}

__device__ __forceinline__ void add_contact(const MppibModel& m, const Layout& L, float* xs, int lane, int& nc, int refA, int refB, int slotA, int slotB, V3 pt, V3 n, float d, float mu) {
    if (nc >= m.max_contacts) return;
    const int cb = L.ct0 + nc * CTN;
    ++nc;
    stx3(xs, cb + CT_P, lane, pt); stx3(xs, cb + CT_N, lane, n);
    XS(cb + CT_D) = d; XS(cb + CT_MU) = mu; XS(cb + CT_LN) = 0.f; XS(cb + CT_LT1) = 0.f; XS(cb + CT_LT2) = 0.f;
    XS(cb + CT_IDS) = __int_as_float((refA + 2) | ((refB + 2) << 8) | ((slotA + 1) << 16) | ((slotB + 1) << 24));
}

__device__ __forceinline__ void tangents(V3 n, V3& t1, V3& t2) {
    const V3 e = fabsf(n.x) < 0.9f ? mk(1, 0, 0) : mk(0, 1, 0);
    t1 = cross(n, e);
    t1 = rsqrtf(dot(t1, t1)) * t1;
    t2 = cross(n, t1);
}

// sample points of box a inside box b -> contacts; flip: a is the B side of the pair
__device__ __forceinline__ void points_in_box(const MppibModel& m, const Layout& L, float* xs, int lane, int& nc, int a, int b, bool flip) {
    const int sa = L.sh0 + a * SHN, sb = L.sh0 + b * SHN;
    const M3 Ra = ldxM3(xs, sa + SH_R, lane), Rb = ldxM3(xs, sb + SH_R, lane);
    const V3 ca = ldx3(xs, sa + SH_C, lane), cbv = ldx3(xs, sb + SH_C, lane);
    const V3 ha = ldx3(xs, sa + SH_HALF, lane), hb = ldx3(xs, sb + SH_HALF, lane);
    const float mu = 0.5f * (XS(sa + SH_MU) + XS(sb + SH_MU));
    const int refa = shape_ref(m, a), refb = shape_ref(m, b), slota = m.shape_slot[a], slotb = m.shape_slot[b];
    const V3 cl = mulT(Rb, ca - cbv);
    bool c0 = fabsf(cl.x) > hb.x, c1 = fabsf(cl.y) > hb.y, c2 = fabsf(cl.z) > hb.z;
    if (!(c0 || c1 || c2)) c0 = c1 = c2 = true;
    const float mg = m.contact_margin;
#pragma unroll 1
    for (int idx = 0; idx < 27; ++idx) {
        if (idx == 13) continue;
        const int ix = idx / 9 - 1, iy = (idx / 3) % 3 - 1, iz = idx % 3 - 1;
        const V3 pt = mul(Ra, mk(ix * ha.x, iy * ha.y, iz * ha.z)) + ca;
        const V3 x = mulT(Rb, pt - cbv);
        const float p0 = hb.x - fabsf(x.x), p1 = hb.y - fabsf(x.y), p2 = hb.z - fabsf(x.z);
        if (!(p0 + mg > 0.f) || !(p1 + mg > 0.f) || !(p2 + mg > 0.f)) continue;
        int ax = -1; float pen = 0.f;
        if (c0) { ax = 0; pen = p0; }
        if (c1 && (ax < 0 || p1 < pen)) { ax = 1; pen = p1; }
        if (c2 && (ax < 0 || p2 < pen)) { ax = 2; pen = p2; }
        const float xa = ax == 0 ? x.x : (ax == 1 ? x.y : x.z);
        const float sg = xa >= 0.f ? 1.f : -1.f;
        const V3 n = ax == 0 ? mk(sg * Rb.m00, sg * Rb.m10, sg * Rb.m20) : (ax == 1 ? mk(sg * Rb.m01, sg * Rb.m11, sg * Rb.m21) : mk(sg * Rb.m02, sg * Rb.m12, sg * Rb.m22));
        if (!flip) add_contact(m, L, xs, lane, nc, refa, refb, slota, slotb, pt, n, pen, mu);
        else add_contact(m, L, xs, lane, nc, refb, refa, slotb, slota, pt, mk(-n.x, -n.y, -n.z), pen, mu);
    }
}

// ONE contact of a sphere against a box (closest point of the box to the centre; centre inside the box: least-penetration face) or
// against another sphere.  The normal of a contact pushes side A out of side B.  Same arithmetic as oracle.cpp sphere_contact.
__device__ __forceinline__ void sphere_contact(const MppibModel& m, const Layout& L, float* xs, int lane, int& nc, int a, int b) {
    const int sa = L.sh0 + a * SHN, sb = L.sh0 + b * SHN;
    const float mu = 0.5f * (XS(sa + SH_MU) + XS(sb + SH_MU)), mg = m.contact_margin;
    const int refa = shape_ref(m, a), refb = shape_ref(m, b), slota = m.shape_slot[a], slotb = m.shape_slot[b];
    const V3 ca = ldx3(xs, sa + SH_C, lane), cbv = ldx3(xs, sb + SH_C, lane);
    if (m.shape_type[a] == MPPIB_SHAPE_SPHERE && m.shape_type[b] == MPPIB_SHAPE_SPHERE) {
        const V3 d = ca - cbv;
        const float dist = sqrtf(dot(d, d)), ra = XS(sa + SH_HALF), rb = XS(sb + SH_HALF), rs = ra + rb;
        if (!(dist < rs + mg) || !(dist > 0.f)) return;
        const V3 n = (1.0f / dist) * d;
        add_contact(m, L, xs, lane, nc, refa, refb, slota, slotb, cbv + rb * n, n, rs - dist, mu);
        return;
    }
    const bool sphere_is_a = m.shape_type[a] == MPPIB_SHAPE_SPHERE;
    const int ss = sphere_is_a ? sa : sb, sx = sphere_is_a ? sb : sa;
    const float r = XS(ss + SH_HALF);
    const V3 cs = sphere_is_a ? ca : cbv, cx = sphere_is_a ? cbv : ca;
    const M3 Rx = ldxM3(xs, sx + SH_R, lane);
    const V3 hx = ldx3(xs, sx + SH_HALF, lane);
    const V3 x = mulT(Rx, cs - cx);
    V3 q = mk(fminf(fmaxf(x.x, -hx.x), hx.x), fminf(fmaxf(x.y, -hx.y), hx.y), fminf(fmaxf(x.z, -hx.z), hx.z));
    const V3 dd = x - q;
    const float d2 = dot(dd, dd);
    V3 nl = mk(0, 0, 0); float pen;
    if (d2 > 0.f) {                                    // centre outside the box
        const float dist = sqrtf(d2);
        if (!(dist < r + mg)) return;
        nl = (1.0f / dist) * dd;
        pen = r - dist;
    } else {                                           // centre inside: out through the nearest face
        int ax = 0; float best = hx.x - fabsf(x.x);
        const float p1 = hx.y - fabsf(x.y), p2 = hx.z - fabsf(x.z);
        if (p1 < best) { best = p1; ax = 1; }
        if (p2 < best) { best = p2; ax = 2; }
        const float xa = ax == 0 ? x.x : (ax == 1 ? x.y : x.z);
        const float sg = xa >= 0.f ? 1.f : -1.f;
        if (ax == 0) { nl.x = sg; q.x = sg * hx.x; } else if (ax == 1) { nl.y = sg; q.y = sg * hx.y; } else { nl.z = sg; q.z = sg * hx.z; }
        pen = best + r;
    }
    const V3 n = mul(Rx, nl);                          // from the box towards the sphere
    const V3 pt = cx + mul(Rx, q);
    if (sphere_is_a) add_contact(m, L, xs, lane, nc, refa, refb, slota, slotb, pt, n, pen, mu);
    else add_contact(m, L, xs, lane, nc, refa, refb, slota, slotb, pt, mk(-n.x, -n.y, -n.z), pen, mu);
}

// contacts of the ordered pair (a, b): boxes by sample points in both directions, anything with a sphere analytically
__device__ __forceinline__ void pair_contacts(const MppibModel& m, const Layout& L, float* xs, int lane, int& nc, int a, int b) {
    if (m.shape_type[a] == MPPIB_SHAPE_SPHERE || m.shape_type[b] == MPPIB_SHAPE_SPHERE) { sphere_contact(m, L, xs, lane, nc, a, b); return; }
    points_in_box(m, L, xs, lane, nc, a, b, false);
    points_in_box(m, L, xs, lane, nc, b, a, true);
}

// broad phase: bounding spheres, then the 6 face axes of the two boxes (conservative: never rejects boxes closer than the margin).
// Without it every articulation link "near" a large static box (table: 1.4 x 2.5 m) paid 52 point-in-box tests per substep.
__device__ __forceinline__ bool near_shapes(const MppibModel& m, const Layout& L, const float* xs, int lane, int a, int b) {
    const int sa = L.sh0 + a * SHN, sb = L.sh0 + b * SHN;
    const V3 d = ldx3(xs, sa + SH_C, lane) - ldx3(xs, sb + SH_C, lane);
    const float mg = m.contact_margin;
    const bool sph = m.shape_type[a] == MPPIB_SHAPE_SPHERE || m.shape_type[b] == MPPIB_SHAPE_SPHERE;
    const float r = XS(sa + SH_RAD) + XS(sb + SH_RAD) + (sph ? mg : 0.f);      // (a sphere's bound is exact: the margin counts)
    if (dot(d, d) > r * r) return false;
    if (sph) return true;                                                       // the narrow phase is exact and cheap
    const M3 Ra = ldxM3(xs, sa + SH_R, lane), Rb = ldxM3(xs, sb + SH_R, lane);
    const V3 ha = ldx3(xs, sa + SH_HALF, lane), hb = ldx3(xs, sb + SH_HALF, lane);
    const V3 tb = mulT(Rb, d), ta = mulT(Ra, d);
    // C = Rb^T Ra, row i = (column i of Rb) . (columns of Ra)
    const V3 b0 = mk(Rb.m00, Rb.m10, Rb.m20), b1 = mk(Rb.m01, Rb.m11, Rb.m21), b2 = mk(Rb.m02, Rb.m12, Rb.m22);
    const V3 a0 = mk(Ra.m00, Ra.m10, Ra.m20), a1 = mk(Ra.m01, Ra.m11, Ra.m21), a2 = mk(Ra.m02, Ra.m12, Ra.m22);
    const float c00 = fabsf(dot(b0, a0)), c01 = fabsf(dot(b0, a1)), c02 = fabsf(dot(b0, a2));
    const float c10 = fabsf(dot(b1, a0)), c11 = fabsf(dot(b1, a1)), c12 = fabsf(dot(b1, a2));
    const float c20 = fabsf(dot(b2, a0)), c21 = fabsf(dot(b2, a1)), c22 = fabsf(dot(b2, a2));
    if (fabsf(tb.x) > hb.x + c00 * ha.x + c01 * ha.y + c02 * ha.z + mg) return false;
    if (fabsf(ta.x) > ha.x + c00 * hb.x + c10 * hb.y + c20 * hb.z + mg) return false;
    if (fabsf(tb.y) > hb.y + c10 * ha.x + c11 * ha.y + c12 * ha.z + mg) return false;
    if (fabsf(ta.y) > ha.y + c01 * hb.x + c11 * hb.y + c21 * hb.z + mg) return false;
    if (fabsf(tb.z) > hb.z + c20 * ha.x + c21 * ha.y + c22 * ha.z + mg) return false;
    if (fabsf(ta.z) > ha.z + c02 * hb.x + c12 * hb.y + c22 * hb.z + mg) return false;
    return true;
}

// world poses of all shapes (articulation frames from sweep 1, static actors from root0, free bodies from their state)
// `statics`: true once per rollout (static boxes never move inside a rollout), false in every substep (links and free bodies)
template <int NSLOT>
__device__ __forceinline__ void shapes_world(const MppibModel& m, const Layout& L, const float* sm, float* xs, int lane, const M3& Rbase, V3 obase,
                                             const float* __restrict__ root0, bool statics) {
    for (int s = 0; s < m.nshapes; ++s) {
        if ((m.shape_owner_kind[s] == MPPIB_OWNER_STATIC) != statics) continue;
        const Quat ql = {m.shape_quat[s][0], m.shape_quat[s][1], m.shape_quat[s][2], m.shape_quat[s][3]};
        const V3 pl = mk(m.shape_pos[s][0], m.shape_pos[s][1], m.shape_pos[s][2]);
        M3 Ro; V3 po;
        const int kind = m.shape_owner_kind[s];
        if (kind == MPPIB_OWNER_STATIC) {
            const float* rs = root0 + 13 * m.shape_actor[s];
            const Quat q = {rs[3], rs[4], rs[5], rs[6]};
            Ro = quat_to_R(q); po = mk(rs[0], rs[1], rs[2]);
        } else if (kind == MPPIB_OWNER_LINK) {
            const int b = m.shape_owner[s];
            if (b >= 0) { Ro = ldM3(sm, b * NSLOT + F_R, lane); po = ld3(sm, b * NSLOT + F_O, lane); }
            else { Ro = Rbase; po = obase; }
        } else {
            const int fb = L.fb0 + m.shape_owner[s] * FBN;
            Ro = ldxM3(xs, fb + FB_R, lane); po = ldx3(xs, fb + FB_X, lane);
        }
        const int sb = L.sh0 + s * SHN;
        stxM3(xs, sb + SH_R, lane, mulMM(Ro, quat_to_R(ql)));
        stx3(xs, sb + SH_C, lane, po + mul(Ro, pl));
    }
}

// Candidate partners of every shape as a bit mask (MPPIB_MAX_SHAPES <= 32), built once per CTA: a FREE shape is tested against every
// shape of another body (free-free pairs once), a LINK shape against the STATIC ones.  The nested shape loops of detect() used to
// re-derive this from the constant bank in every substep, a chain of dependent constant loads.
__device__ __forceinline__ uint32_t partner_mask(const MppibModel& m, int a) {
    const int ns = m.nshapes;
    uint32_t mask = 0;
    if (m.shape_owner_kind[a] == MPPIB_OWNER_FREE) {
        for (int b = 0; b < ns; ++b) {
            if (b == a || shape_ref(m, b) == shape_ref(m, a)) continue;
            if (m.shape_owner_kind[b] == MPPIB_OWNER_FREE && b < a) continue;
            mask |= 1u << b;
        }
    } else if (m.shape_owner_kind[a] == MPPIB_OWNER_LINK && shape_ref(m, a) != REF_STATIC) {
        for (int b = 0; b < ns; ++b) if (m.shape_owner_kind[b] == MPPIB_OWNER_STATIC) mask |= 1u << b;
    }
    return mask;
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
        const int refA = (ids & 0xFF) - 2, refB = ((ids >> 8) & 0xFF) - 2;
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
            const int refA = (ids & 0xFF) - 2, refB = ((ids >> 8) & 0xFF) - 2;
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
        const int slotA = ((ids >> 16) & 0xFF) - 1, slotB = ((ids >> 24) & 0xFF) - 1;
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
        XS(fb + FB_X) += h * XS(fb + FB_V); XS(fb + FB_X + 1) += h * XS(fb + FB_V + 1); XS(fb + FB_X + 2) += h * XS(fb + FB_V + 2);
        const Quat q = {XS(fb + FB_Q), XS(fb + FB_Q + 1), XS(fb + FB_Q + 2), XS(fb + FB_Q + 3)};
        const Quat wq = {XS(fb + FB_W), XS(fb + FB_W + 1), XS(fb + FB_W + 2), 0.f};
        const Quat dq = qmul(wq, q);
        Quat r = {q.x + 0.5f * h * dq.x, q.y + 0.5f * h * dq.y, q.z + 0.5f * h * dq.z, q.w + 0.5f * h * dq.w};
        const float il = rsqrtf(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w);
        XS(fb + FB_Q) = r.x * il; XS(fb + FB_Q + 1) = r.y * il; XS(fb + FB_Q + 2) = r.z * il; XS(fb + FB_Q + 3) = r.w * il;
        refresh_free(xs, lane, fb);
    }
}

}  // namespace contact
