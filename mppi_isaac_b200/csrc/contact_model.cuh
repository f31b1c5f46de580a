// contact_model.cuh -- the contact model of K2, written once for both contact kernels: rollout.cu + contact.cuh (one thread per
// rollout) and rollout_team.cu (a team of lanes per rollout).  Spec: DESIGN.md section 2, restated independently by oracle/oracle.cpp
// ContactWorld.
//
// The functions take values and return values: poses, half extents and indices go in; contact points, normals, depths and a `hit`
// flag come out.  Each kernel keeps what it does differently: where the values live, which lane computes what, how a contact is
// recorded, and the Gauss-Seidel solve.  The header is included inside each kernel's anonymous namespace after that kernel's vector
// algebra (mk, dot, cross, mul / mulT of a 3x3, scale, quat_to_R, qmul): rbd_math.cuh in rollout.cu, lanes_math.cuh in
// rollout_team.cu.  The two round differently on purpose, and each kernel compiles this code with its own.
#pragma once

namespace contact {

// contact sides: static (the world), articulation link j (0 <= j < 64), free body REF_FREE0 + f
enum : int { REF_STATIC = -1, REF_FREE0 = 64 };
// per-rollout record of a free body; FB_MASS holds the INVERSE mass
enum : int { FB_X = 0, FB_Q = 3, FB_V = 7, FB_W = 10, FB_MASS = 13, FB_HALF = 14, FB_IINV = 17, FB_R = 20, FB_IW = 29, FBN = 35 };
// per-rollout record of a world shape
enum : int { SH_R = 0, SH_C = 9, SH_HALF = 12, SH_MU = 15, SH_RAD = 16, SHN = 17 };
// a contact row whose effective inverse mass is below K_ROW_MIN [1/kg] is dropped (bodies that cannot move along that direction; same
// threshold in oracle.cpp -- an exact `> 0` would depend on the rotation arithmetic producing exact zeros)
constexpr float K_ROW_MIN = 1e-9f;

// per-rollout size / mass / friction draws of one actor (the same counters as oracle actor_noise)
__device__ __forceinline__ void actor_noise(const MppibParams& p, uint32_t kg, int actor, V3& nsize, float& umass, float& ufric) {
    const uint4 r0 = philox4x32_10<1>(make_uint4(kg, (uint32_t)actor, 0x5EEDu, 0u), p.rand_seed, 0x4D505049u);
    const uint4 r1 = philox4x32_10<1>(make_uint4(kg, (uint32_t)actor, 0x5EEDu, 1u), p.rand_seed, 0x4D505049u);
    float dummy;
    box_muller(r0.x, r0.y, nsize.x, nsize.y);
    box_muller(r0.z, r0.w, nsize.z, dummy);
    umass = 2.0f * u01(r1.x) - 1.0f;
    ufric = 2.0f * u01(r1.y) - 1.0f;
}

// randomised half extents, friction and bounding radius of shape s in the rollout keyed kg; a sphere shape
// (isaacgym_utils.py:42-52: gym.create_sphere(radius = size[0])) keeps its radius in half.x
__device__ __forceinline__ void shape_params(const MppibModel& m, const MppibParams& p, uint32_t kg, int s, V3& half, float& mu, float& rad) {
    half = mk(m.shape_half[s][0], m.shape_half[s][1], m.shape_half[s][2]);
    mu = m.shape_friction[s];
    if (m.shape_actor[s] >= 0) {
        V3 ns; float um, uf; actor_noise(p, kg, m.shape_actor[s], ns, um, uf);
        half.x += 0.5f * m.shape_size_sigma[s][0] * ns.x; half.y += 0.5f * m.shape_size_sigma[s][1] * ns.y; half.z += 0.5f * m.shape_size_sigma[s][2] * ns.z;
        mu *= 1.0f + m.shape_fric_pct[s] * uf;
    }
    rad = m.shape_type[s] == MPPIB_SHAPE_SPHERE ? half.x : sqrtf(dot(half, half));
}

// randomised inverse mass, half extents and principal inverse inertia of free body f in the rollout keyed kg
__device__ __forceinline__ void free_params(const MppibModel& m, const MppibParams& p, uint32_t kg, int f, float& inv_mass, V3& half, V3& iinv) {
    V3 ns; float um, uf; actor_noise(p, kg, m.free_actor[f], ns, um, uf);
    const float mass = m.free_mass[f] * (1.0f + m.free_mass_pct[f] * um);
    V3 sg = mk(0.f, 0.f, 0.f);
    for (int s = 0; s < m.nshapes; ++s)
        if (m.shape_owner_kind[s] == MPPIB_OWNER_FREE && m.shape_owner[s] == f) { sg = mk(m.shape_size_sigma[s][0], m.shape_size_sigma[s][1], m.shape_size_sigma[s][2]); break; }
    half = mk(m.free_half[f][0] + 0.5f * sg.x * ns.x, m.free_half[f][1] + 0.5f * sg.y * ns.y, m.free_half[f][2] + 0.5f * sg.z * ns.z);
    const float m3 = mass / 3.0f;
    inv_mass = 1.0f / mass;
    iinv = mk(1.0f / (m3 * (half.y * half.y + half.z * half.z)), 1.0f / (m3 * (half.x * half.x + half.z * half.z)),
              1.0f / (m3 * (half.x * half.x + half.y * half.y)));
}

// world inverse inertia R diag(i) R^T of a free body, in the order of FB_IW: xx yy zz xy xz yz
__device__ __forceinline__ S3 world_inv_inertia(const M3& R, V3 i) {
    S3 w;
    w.xx = R.m00 * i.x * R.m00 + R.m01 * i.y * R.m01 + R.m02 * i.z * R.m02;
    w.yy = R.m10 * i.x * R.m10 + R.m11 * i.y * R.m11 + R.m12 * i.z * R.m12;
    w.zz = R.m20 * i.x * R.m20 + R.m21 * i.y * R.m21 + R.m22 * i.z * R.m22;
    w.xy = R.m00 * i.x * R.m10 + R.m01 * i.y * R.m11 + R.m02 * i.z * R.m12;
    w.xz = R.m00 * i.x * R.m20 + R.m01 * i.y * R.m21 + R.m02 * i.z * R.m22;
    w.yz = R.m10 * i.x * R.m20 + R.m11 * i.y * R.m21 + R.m12 * i.z * R.m22;
    return w;
}

// one step of a free body's pose: x += h v, q += h/2 (w, 0) q, renormalised
__device__ __forceinline__ void integrate_pose(V3& x, Quat& q, V3 v, V3 w, float h) {
    x = mk(x.x + h * v.x, x.y + h * v.y, x.z + h * v.z);
    const Quat wq = {w.x, w.y, w.z, 0.f};
    const Quat dq = qmul(wq, q);
    const Quat r = {q.x + 0.5f * h * dq.x, q.y + 0.5f * h * dq.y, q.z + 0.5f * h * dq.z, q.w + 0.5f * h * dq.w};
    const float il = rsqrtf(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w);
    q = {r.x * il, r.y * il, r.z * il, r.w * il};
}

__device__ __forceinline__ M3 mulMM(const M3& a, const M3& b) {
    M3 o;
    o.m00 = a.m00 * b.m00 + a.m01 * b.m10 + a.m02 * b.m20; o.m01 = a.m00 * b.m01 + a.m01 * b.m11 + a.m02 * b.m21; o.m02 = a.m00 * b.m02 + a.m01 * b.m12 + a.m02 * b.m22;
    o.m10 = a.m10 * b.m00 + a.m11 * b.m10 + a.m12 * b.m20; o.m11 = a.m10 * b.m01 + a.m11 * b.m11 + a.m12 * b.m21; o.m12 = a.m10 * b.m02 + a.m11 * b.m12 + a.m12 * b.m22;
    o.m20 = a.m20 * b.m00 + a.m21 * b.m10 + a.m22 * b.m20; o.m21 = a.m20 * b.m01 + a.m21 * b.m11 + a.m22 * b.m21; o.m22 = a.m20 * b.m02 + a.m21 * b.m12 + a.m22 * b.m22;
    return o;
}

// world pose of a static actor from its root state (p, q, v, w)
__device__ __forceinline__ void root_pose(const float* __restrict__ root0, int actor, M3& R, V3& o) {
    const float* rs = root0 + 13 * actor;
    const Quat q = {rs[3], rs[4], rs[5], rs[6]};
    R = quat_to_R(q); o = mk(rs[0], rs[1], rs[2]);
}
// world pose (R, c) of shape s on an owner at (Ro, po)
__device__ __forceinline__ void shape_pose(const MppibModel& m, int s, const M3& Ro, V3 po, M3& R, V3& c) {
    const Quat ql = {m.shape_quat[s][0], m.shape_quat[s][1], m.shape_quat[s][2], m.shape_quat[s][3]};
    R = mulMM(Ro, quat_to_R(ql));
    c = po + mul(Ro, mk(m.shape_pos[s][0], m.shape_pos[s][1], m.shape_pos[s][2]));
}

__device__ __forceinline__ int shape_ref(const MppibModel& m, int s) {
    const int kind = m.shape_owner_kind[s];
    if (kind == MPPIB_OWNER_FREE) return REF_FREE0 + m.shape_owner[s];
    if (kind == MPPIB_OWNER_LINK && m.shape_owner[s] >= 0) return m.shape_owner[s];
    return REF_STATIC;
}

// Candidate partners of shape a as a bit mask (MPPIB_MAX_SHAPES <= 32), built once per CTA: a FREE shape is tested against every shape
// of another body (free-free pairs once), a LINK shape against the STATIC ones.  Ascending bits are the oracle's loop order.
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

// Broad phase, in two steps so that a kernel loads the box poses only for the pairs that pass the first: the bounding spheres of shapes
// at offset d = ca - cb (a sphere's bound is exact, so the margin counts: sph = either is a sphere), then for two boxes the 6 face axes
// (conservative: never rejects boxes closer than the margin).  Without it every articulation link "near" a large static box (table:
// 1.4 x 2.5 m) paid 52 point-in-box tests per substep.
__device__ __forceinline__ bool near_bounds(V3 d, float rad_a, float rad_b, bool sph, float mg) {
    const float r = rad_a + rad_b + (sph ? mg : 0.f);
    return !(dot(d, d) > r * r);
}
__device__ __forceinline__ bool near_boxes(V3 d, const M3& Ra, V3 ha, const M3& Rb, V3 hb, float mg) {
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

// Box a (Ra, ca, ha) against box b (Rb, cb, hb): the 26 surface sample points of a (idx = 0 .. 26 but 13, the centre) that lie inside b
// within the margin are contacts.  face_axes: the face axes of b the normal may take, the slabs of b that a's centre lies outside of
// (all three when it lies inside b).  box_point: sample point idx, its normal (the least-penetration face among those, out of b) and
// depth; returns whether it is a contact.
__device__ __forceinline__ void face_axes(const M3& Rb, V3 ca, V3 cb, V3 hb, bool& c0, bool& c1, bool& c2) {
    const V3 cl = mulT(Rb, ca - cb);
    c0 = fabsf(cl.x) > hb.x; c1 = fabsf(cl.y) > hb.y; c2 = fabsf(cl.z) > hb.z;
    if (!(c0 || c1 || c2)) c0 = c1 = c2 = true;
}
__device__ __forceinline__ bool box_point(int idx, const M3& Ra, V3 ca, V3 ha, const M3& Rb, V3 cb, V3 hb, bool c0, bool c1, bool c2,
                                          float mg, V3& pt, V3& n, float& pen) {
    const int ix = idx / 9 - 1, iy = (idx / 3) % 3 - 1, iz = idx % 3 - 1;
    pt = mul(Ra, mk(ix * ha.x, iy * ha.y, iz * ha.z)) + ca;
    const V3 x = mulT(Rb, pt - cb);
    const float p0 = hb.x - fabsf(x.x), p1 = hb.y - fabsf(x.y), p2 = hb.z - fabsf(x.z);
    int ax = -1; pen = 0.f;
    if (c0) { ax = 0; pen = p0; }
    if (c1 && (ax < 0 || p1 < pen)) { ax = 1; pen = p1; }
    if (c2 && (ax < 0 || p2 < pen)) { ax = 2; pen = p2; }
    const float xa = ax == 0 ? x.x : (ax == 1 ? x.y : x.z);
    const float sg = xa >= 0.f ? 1.f : -1.f;
    n = ax == 0 ? mk(sg * Rb.m00, sg * Rb.m10, sg * Rb.m20) : (ax == 1 ? mk(sg * Rb.m01, sg * Rb.m11, sg * Rb.m21) : mk(sg * Rb.m02, sg * Rb.m12, sg * Rb.m22));
    return p0 + mg > 0.f && p1 + mg > 0.f && p2 + mg > 0.f;
}

// A sphere (centre ca, radius ra) against a sphere (cb, rb): one contact along the line of the centres, the normal pushing a out of b.
__device__ __forceinline__ bool sphere_sphere(V3 ca, float ra, V3 cb, float rb, float mg, V3& pt, V3& n, float& pen) {
    const V3 d = ca - cb;
    const float dist = sqrtf(dot(d, d)), rs = ra + rb;
    n = scale(1.0f / fmaxf(dist, 1e-30f), d);
    pt = cb + scale(rb, n); pen = rs - dist;
    return dist < rs + mg && dist > 0.f;
}
// A sphere (centre cs, radius r) against a box (Rx, cx, hx): one contact at the box's closest point to the centre, or through the
// least-penetration face when the centre is inside; the normal points from the box towards the sphere.  Same arithmetic as oracle.cpp
// sphere_contact.
__device__ __forceinline__ bool sphere_box(V3 cs, float r, const M3& Rx, V3 cx, V3 hx, float mg, V3& pt, V3& n, float& pen) {
    const V3 x = mulT(Rx, cs - cx);
    V3 q = mk(fminf(fmaxf(x.x, -hx.x), hx.x), fminf(fmaxf(x.y, -hx.y), hx.y), fminf(fmaxf(x.z, -hx.z), hx.z));
    const V3 dd = x - q;
    const float d2 = dot(dd, dd);
    V3 nl = mk(0.f, 0.f, 0.f);
    bool hit = true;
    if (d2 > 0.f) {                                    // centre outside the box
        const float dist = sqrtf(d2);
        hit = dist < r + mg;
        nl = scale(1.0f / dist, dd);
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
    n = mul(Rx, nl);
    pt = cx + mul(Rx, q);
    return hit;
}

// tangent frame (t1, t2) of a contact normal n
__device__ __forceinline__ void tangents(V3 n, V3& t1, V3& t2) {
    const V3 e = fabsf(n.x) < 0.9f ? mk(1.f, 0.f, 0.f) : mk(0.f, 1.f, 0.f);
    t1 = cross(n, e);
    t1 = scale(rsqrtf(dot(t1, t1)), t1);
    t2 = cross(n, t1);
}

// the two sides (ref ids) and net-force slots (-1: none) of a contact, packed into one int that a contact record keeps as float bits
__device__ __forceinline__ int pack_sides(int refA, int refB, int slotA, int slotB) {
    return (refA + 2) | ((refB + 2) << 8) | ((slotA + 1) << 16) | ((slotB + 1) << 24);
}
__device__ __forceinline__ int ref_a(int ids) { return (ids & 0xFF) - 2; }
__device__ __forceinline__ int ref_b(int ids) { return ((ids >> 8) & 0xFF) - 2; }
__device__ __forceinline__ int slot_a(int ids) { return ((ids >> 16) & 0xFF) - 1; }
__device__ __forceinline__ int slot_b(int ids) { return ((ids >> 24) & 0xFF) - 1; }

}  // namespace contact
