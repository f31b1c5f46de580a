// lanes_math.cuh -- vector / quaternion algebra of the lanes-per-rollout kernel (rollout_lanes.cu), generic in the scalar type:
//   float : one rollout per lane group
//   P2    : TWO rollouts per lane group.  sm_90 has no packed f32x2 arithmetic, so every P2 operation is two independent
//           scalar fp32 instructions (the same IEEE round-to-nearest results as the float instantiation); what the pair
//           shares is the control, shuffle-index and address instructions, and the two chains give the scheduler ILP 2.
// The formulas are written once against the few primitives below.
#pragma once
#include <cuda_runtime.h>

namespace lm {

struct P2 { float2 v; };
__device__ __forceinline__ P2 mkp(float a, float b) { P2 r; r.v = make_float2(a, b); return r; }

template <class F> struct scalar_traits;
template <> struct scalar_traits<float> { static constexpr int N = 1; };
template <> struct scalar_traits<P2> { static constexpr int N = 2; };

// ---- arithmetic ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ P2 operator+(P2 a, P2 b) { return mkp(__fadd_rn(a.v.x, b.v.x), __fadd_rn(a.v.y, b.v.y)); }
__device__ __forceinline__ P2 operator-(P2 a) { return mkp(-a.v.x, -a.v.y); }                     // folds into the consumer's operand modifier
__device__ __forceinline__ P2 operator-(P2 a, P2 b) { return mkp(__fadd_rn(a.v.x, -b.v.x), __fadd_rn(a.v.y, -b.v.y)); }
__device__ __forceinline__ P2 operator*(P2 a, P2 b) { return mkp(__fmul_rn(a.v.x, b.v.x), __fmul_rn(a.v.y, b.v.y)); }
__device__ __forceinline__ P2 operator*(P2 a, float c) { return mkp(__fmul_rn(a.v.x, c), __fmul_rn(a.v.y, c)); }
__device__ __forceinline__ P2 operator*(float c, P2 a) { return a * c; }
__device__ __forceinline__ P2 operator+(P2 a, float c) { return mkp(__fadd_rn(a.v.x, c), __fadd_rn(a.v.y, c)); }
__device__ __forceinline__ P2 operator+(float c, P2 a) { return a + c; }
__device__ __forceinline__ P2 operator-(P2 a, float c) { return a + (-c); }
__device__ __forceinline__ P2 operator-(float c, P2 a) { return (-a) + c; }
__device__ __forceinline__ P2& operator+=(P2& a, P2 b) { a = a + b; return a; }

// a * b + c
__device__ __forceinline__ float fma_(float a, float b, float c) { return fmaf(a, b, c); }
__device__ __forceinline__ P2 fma_(P2 a, P2 b, P2 c) { return mkp(fmaf(a.v.x, b.v.x, c.v.x), fmaf(a.v.y, b.v.y, c.v.y)); }
__device__ __forceinline__ P2 fma_(P2 a, float b, P2 c) { return mkp(fmaf(a.v.x, b, c.v.x), fmaf(a.v.y, b, c.v.y)); }
__device__ __forceinline__ P2 fma_(float a, P2 b, P2 c) { return fma_(b, a, c); }
__device__ __forceinline__ P2 fma_(P2 a, P2 b, float c) { return mkp(fmaf(a.v.x, b.v.x, c), fmaf(a.v.y, b.v.y, c)); }
__device__ __forceinline__ P2 fma_(P2 a, float b, float c) { return mkp(fmaf(a.v.x, b, c), fmaf(a.v.y, b, c)); }

template <class F> __device__ __forceinline__ F bcast(float c);
template <> __device__ __forceinline__ float bcast<float>(float c) { return c; }
template <> __device__ __forceinline__ P2 bcast<P2>(float c) { return mkp(c, c); }

// component access (i = 0 .. N-1)
__device__ __forceinline__ float comp(float a, int) { return a; }
__device__ __forceinline__ float comp(P2 a, int i) { return i == 0 ? a.v.x : a.v.y; }
__device__ __forceinline__ void set_comp(float& a, int, float v) { a = v; }
__device__ __forceinline__ void set_comp(P2& a, int i, float v) { if (i == 0) a.v.x = v; else a.v.y = v; }

// uniform-condition select, min / max against a per-body constant
__device__ __forceinline__ float sel(bool c, float a, float b) { return c ? a : b; }
__device__ __forceinline__ P2 sel(bool c, P2 a, P2 b) { return mkp(c ? a.v.x : b.v.x, c ? a.v.y : b.v.y); }
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
__device__ __forceinline__ P2 clampf(P2 x, float lo, float hi) { return mkp(fminf(fmaxf(x.v.x, lo), hi), fminf(fmaxf(x.v.y, lo), hi)); }

__device__ __forceinline__ float rcp_approx(float x) {   // MUFU.RCP: 1 ulp, no Newton step on the FP32 pipe
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ P2 rcp_approx(P2 x) { return mkp(rcp_approx(x.v.x), rcp_approx(x.v.y)); }

// sin / cos with a two-term Cody-Waite reduction and the Cephes minimax polynomials on [-pi/4, pi/4] (rbd_math.cuh sincos_cw: max
// error 9e-8 for |x| < 3000 rad, no slow path)
__device__ __forceinline__ void sincos_cw1(float x, float* s_out, float* c_out) {
    const float k = rintf(x * 0.63661975f);
    float r = fmaf(-k, 1.5707964f, x);
    r = fmaf(-k, -4.371139e-08f, r);
    const float r2 = r * r;
    const float s = fmaf(r * r2, fmaf(r2, fmaf(r2, -1.9515295891e-4f, 8.3321608736e-3f), -1.6666654611e-1f), r);
    const float c = fmaf(r2 * r2, fmaf(r2, fmaf(r2, 2.443315711809948e-5f, -1.388731625493765e-3f), 4.166664568298827e-2f), fmaf(-0.5f, r2, 1.0f));
    const int n = (int)k & 3;
    const float ss = (n & 1) ? c : s, cc = (n & 1) ? s : c;
    *s_out = (n & 2) ? -ss : ss;
    *c_out = ((n + 1) & 2) ? -cc : cc;
}
__device__ __forceinline__ void sincos_cw(float x, float* s, float* c) { sincos_cw1(x, s, c); }
__device__ __forceinline__ void sincos_cw(P2 x, P2* s, P2* c) {
    float s0, c0, s1, c1;
    sincos_cw1(x.v.x, &s0, &c0);
    sincos_cw1(x.v.y, &s1, &c1);
    *s = mkp(s0, s1); *c = mkp(c0, c1);
}

// ---- shuffles over the G lanes of a rollout group -----------------------------------------------------------------------
constexpr unsigned FULL = 0xffffffffu;
template <int G> __device__ __forceinline__ float shfl_up(float v, int d) { return __shfl_up_sync(FULL, v, d, G); }
template <int G> __device__ __forceinline__ float shfl_dn(float v, int d) { return __shfl_down_sync(FULL, v, d, G); }
template <int G> __device__ __forceinline__ float shfl_at(float v, int src) { return __shfl_sync(FULL, v, src, G); }
template <int G> __device__ __forceinline__ P2 shfl_up(P2 v, int d) { return mkp(shfl_up<G>(v.v.x, d), shfl_up<G>(v.v.y, d)); }
template <int G> __device__ __forceinline__ P2 shfl_dn(P2 v, int d) { return mkp(shfl_dn<G>(v.v.x, d), shfl_dn<G>(v.v.y, d)); }
template <int G> __device__ __forceinline__ P2 shfl_at(P2 v, int src) { return mkp(shfl_at<G>(v.v.x, src), shfl_at<G>(v.v.y, src)); }

// ---- 3-vectors, symmetric / general 3x3, quaternions ----------------------------------------------------------------------
template <class F> struct V3T { F x, y, z; };
template <class F> struct S3T { F xx, yy, zz, xy, xz, yz; };
template <class F> struct M3T { F m00, m01, m02, m10, m11, m12, m20, m21, m22; };
template <class F> struct QT { F x, y, z, w; };
template <class F> struct V6T { V3T<F> n, f; };

template <class F> __device__ __forceinline__ V3T<F> mk3(F x, F y, F z) { V3T<F> v; v.x = x; v.y = y; v.z = z; return v; }
template <class F> __device__ __forceinline__ V3T<F> zero3() { return mk3<F>(bcast<F>(0.f), bcast<F>(0.f), bcast<F>(0.f)); }
template <class F> __device__ __forceinline__ V3T<F> operator+(V3T<F> a, V3T<F> b) { return mk3<F>(a.x + b.x, a.y + b.y, a.z + b.z); }
template <class F> __device__ __forceinline__ V3T<F> operator-(V3T<F> a, V3T<F> b) { return mk3<F>(a.x - b.x, a.y - b.y, a.z - b.z); }
template <class S, class F> __device__ __forceinline__ V3T<F> scale(S s, V3T<F> a) { return mk3<F>(s * a.x, s * a.y, s * a.z); }   // S = F or float
template <class F> __device__ __forceinline__ F dot(V3T<F> a, V3T<F> b) { return fma_(a.z, b.z, fma_(a.y, b.y, a.x * b.x)); }
template <class F> __device__ __forceinline__ V3T<F> cross(V3T<F> a, V3T<F> b) {
    return mk3<F>(fma_(a.y, b.z, -(a.z * b.y)), fma_(a.z, b.x, -(a.x * b.z)), fma_(a.x, b.y, -(a.y * b.x)));
}
// acc + a x b
template <class F> __device__ __forceinline__ V3T<F> cross_add(V3T<F> acc, V3T<F> a, V3T<F> b) {
    return mk3<F>(fma_(a.y, b.z, fma_(-a.z, b.y, acc.x)), fma_(a.z, b.x, fma_(-a.x, b.z, acc.y)), fma_(a.x, b.y, fma_(-a.y, b.x, acc.z)));
}
// symmetric 3x3 times vector (+ acc)
template <class F, class FM> __device__ __forceinline__ V3T<F> mul(const S3T<FM>& s, V3T<F> v) {
    return mk3<F>(fma_(v.z, s.xz, fma_(v.y, s.xy, v.x * s.xx)), fma_(v.z, s.yz, fma_(v.y, s.yy, v.x * s.xy)), fma_(v.z, s.zz, fma_(v.y, s.yz, v.x * s.xz)));
}
template <class F> __device__ __forceinline__ V3T<F> mul_add(V3T<F> acc, const S3T<F>& s, V3T<F> v) {
    return mk3<F>(fma_(v.z, s.xz, fma_(v.y, s.xy, fma_(v.x, s.xx, acc.x))), fma_(v.z, s.yz, fma_(v.y, s.yy, fma_(v.x, s.xy, acc.y))),
                  fma_(v.z, s.zz, fma_(v.y, s.yz, fma_(v.x, s.xz, acc.z))));
}
// general 3x3 (row major) times a CONSTANT vector (per-body model constant, the same for both rollouts of a pair)
template <class F> __device__ __forceinline__ V3T<F> mulc(const M3T<F>& m, float x, float y, float z) {
    return mk3<F>(fma_(m.m02, z, fma_(m.m01, y, m.m00 * x)), fma_(m.m12, z, fma_(m.m11, y, m.m10 * x)), fma_(m.m22, z, fma_(m.m21, y, m.m20 * x)));
}

template <class F> __device__ __forceinline__ QT<F> qmul(QT<F> a, QT<F> b) {
    QT<F> o;
    o.x = fma_(a.w, b.x, fma_(a.x, b.w, fma_(a.y, b.z, -(a.z * b.y))));
    o.y = fma_(a.w, b.y, fma_(a.y, b.w, fma_(a.z, b.x, -(a.x * b.z))));
    o.z = fma_(a.w, b.z, fma_(a.z, b.w, fma_(a.x, b.y, -(a.y * b.x))));
    o.w = fma_(a.w, b.w, fma_(-a.x, b.x, fma_(-a.y, b.y, -(a.z * b.z))));
    return o;
}
// p + q v q*  =  p + v + 2 w (u x v) + 2 u x (u x v)
template <class F> __device__ __forceinline__ V3T<F> qrot_add(V3T<F> p, QT<F> q, V3T<F> v) {
    const V3T<F> u = mk3<F>(q.x, q.y, q.z);
    V3T<F> c = cross(u, v);
    c = c + c;
    V3T<F> r = p + v;
    r = mk3<F>(fma_(q.w, c.x, r.x), fma_(q.w, c.y, r.y), fma_(q.w, c.z, r.z));
    return cross_add(r, u, c);
}
template <class F> __device__ __forceinline__ M3T<F> quat_to_R(QT<F> q) {
    const F x2 = q.x + q.x, y2 = q.y + q.y, z2 = q.z + q.z;
    const F xx = q.x * x2, yy = q.y * y2, zz = q.z * z2, xy = q.x * y2, xz = q.x * z2, yz = q.y * z2, wx = q.w * x2, wy = q.w * y2, wz = q.w * z2;
    M3T<F> R;
    R.m00 = 1.0f - (yy + zz); R.m01 = xy - wz; R.m02 = xz + wy;
    R.m10 = xy + wz; R.m11 = 1.0f - (xx + zz); R.m12 = yz - wx;
    R.m20 = xz - wy; R.m21 = yz + wx; R.m22 = 1.0f - (xx + yy);
    return R;
}

}  // namespace lm
