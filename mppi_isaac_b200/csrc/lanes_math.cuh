// lanes_math.cuh -- vector / quaternion algebra of the lane-parallel rollout kernels (rollout_lanes.cu, rollout_team.cu).
// Products are written as explicit fma_ / fmaf chains: the order of the fused operations fixes the rounding, which deliberately
// differs from the thread-per-rollout kernel's rbd_math.cuh (a*b + c).
#pragma once
#include <cuda_runtime.h>

namespace lm {

// a * b + c
__device__ __forceinline__ float fma_(float a, float b, float c) { return fmaf(a, b, c); }

// uniform-condition select, clamp against a per-body constant
__device__ __forceinline__ float sel(bool c, float a, float b) { return c ? a : b; }
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }

__device__ __forceinline__ float rcp_approx(float x) {   // MUFU.RCP: 1 ulp, no Newton step on the FP32 pipe
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// sin / cos with a two-term Cody-Waite reduction and the Cephes minimax polynomials on [-pi/4, pi/4] (rbd_math.cuh sincos_cw: max
// error 9e-8 for |x| < 3000 rad, no slow path)
__device__ __forceinline__ void sincos_cw(float x, float* s_out, float* c_out) {
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

// ---- shuffles over the G lanes of a rollout group -----------------------------------------------------------------------
constexpr unsigned FULL = 0xffffffffu;
template <int G> __device__ __forceinline__ float shfl_up(float v, int d) { return __shfl_up_sync(FULL, v, d, G); }
template <int G> __device__ __forceinline__ float shfl_dn(float v, int d) { return __shfl_down_sync(FULL, v, d, G); }
template <int G> __device__ __forceinline__ float shfl_at(float v, int src) { return __shfl_sync(FULL, v, src, G); }

// ---- 3-vectors, symmetric / general 3x3, quaternions ----------------------------------------------------------------------
struct V3 { float x, y, z; };
struct S3 { float xx, yy, zz, xy, xz, yz; };
struct M3 { float m00, m01, m02, m10, m11, m12, m20, m21, m22; };
struct Quat { float x, y, z, w; };
struct V6 { V3 n, f; };

__device__ __forceinline__ V3 mk3(float x, float y, float z) { V3 v; v.x = x; v.y = y; v.z = z; return v; }
__device__ __forceinline__ V3 zero3() { return mk3(0.f, 0.f, 0.f); }
__device__ __forceinline__ V3 operator+(V3 a, V3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ V3 operator-(V3 a, V3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ V3 scale(float s, V3 a) { return mk3(s * a.x, s * a.y, s * a.z); }
__device__ __forceinline__ float dot(V3 a, V3 b) { return fma_(a.z, b.z, fma_(a.y, b.y, a.x * b.x)); }
__device__ __forceinline__ V3 cross(V3 a, V3 b) {
    return mk3(fma_(a.y, b.z, -(a.z * b.y)), fma_(a.z, b.x, -(a.x * b.z)), fma_(a.x, b.y, -(a.y * b.x)));
}
// acc + a x b
__device__ __forceinline__ V3 cross_add(V3 acc, V3 a, V3 b) {
    return mk3(fma_(a.y, b.z, fma_(-a.z, b.y, acc.x)), fma_(a.z, b.x, fma_(-a.x, b.z, acc.y)), fma_(a.x, b.y, fma_(-a.y, b.x, acc.z)));
}
// symmetric 3x3 times vector (+ acc)
__device__ __forceinline__ V3 mul(const S3& s, V3 v) {
    return mk3(fma_(v.z, s.xz, fma_(v.y, s.xy, v.x * s.xx)), fma_(v.z, s.yz, fma_(v.y, s.yy, v.x * s.xy)), fma_(v.z, s.zz, fma_(v.y, s.yz, v.x * s.xz)));
}
__device__ __forceinline__ V3 mul_add(V3 acc, const S3& s, V3 v) {
    return mk3(fma_(v.z, s.xz, fma_(v.y, s.xy, fma_(v.x, s.xx, acc.x))), fma_(v.z, s.yz, fma_(v.y, s.yy, fma_(v.x, s.xy, acc.y))),
               fma_(v.z, s.zz, fma_(v.y, s.yz, fma_(v.x, s.xz, acc.z))));
}
// general 3x3 (row major) times a vector given by its components
__device__ __forceinline__ V3 mulc(const M3& m, float x, float y, float z) {
    return mk3(fma_(m.m02, z, fma_(m.m01, y, m.m00 * x)), fma_(m.m12, z, fma_(m.m11, y, m.m10 * x)), fma_(m.m22, z, fma_(m.m21, y, m.m20 * x)));
}

__device__ __forceinline__ Quat qmul(Quat a, Quat b) {
    Quat o;
    o.x = fma_(a.w, b.x, fma_(a.x, b.w, fma_(a.y, b.z, -(a.z * b.y))));
    o.y = fma_(a.w, b.y, fma_(a.y, b.w, fma_(a.z, b.x, -(a.x * b.z))));
    o.z = fma_(a.w, b.z, fma_(a.z, b.w, fma_(a.x, b.y, -(a.y * b.x))));
    o.w = fma_(a.w, b.w, fma_(-a.x, b.x, fma_(-a.y, b.y, -(a.z * b.z))));
    return o;
}
// p + q v q*  =  p + v + 2 w (u x v) + 2 u x (u x v)
__device__ __forceinline__ V3 qrot_add(V3 p, Quat q, V3 v) {
    const V3 u = mk3(q.x, q.y, q.z);
    V3 c = cross(u, v);
    c = c + c;
    V3 r = p + v;
    r = mk3(fma_(q.w, c.x, r.x), fma_(q.w, c.y, r.y), fma_(q.w, c.z, r.z));
    return cross_add(r, u, c);
}
__device__ __forceinline__ M3 quat_to_R(Quat q) {
    const float x2 = q.x + q.x, y2 = q.y + q.y, z2 = q.z + q.z;
    const float xx = q.x * x2, yy = q.y * y2, zz = q.z * z2, xy = q.x * y2, xz = q.x * z2, yz = q.y * z2, wx = q.w * x2, wy = q.w * y2, wz = q.w * z2;
    M3 R;
    R.m00 = 1.0f - (yy + zz); R.m01 = xy - wz; R.m02 = xz + wy;
    R.m10 = xy + wz; R.m11 = 1.0f - (xx + zz); R.m12 = yz - wx;
    R.m20 = xz - wy; R.m21 = yz + wx; R.m22 = 1.0f - (xx + yy);
    return R;
}

}  // namespace lm
