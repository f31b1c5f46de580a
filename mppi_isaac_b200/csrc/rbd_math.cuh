// rbd_math.cuh -- small vector / quaternion helpers shared by the rollout kernels (rollout.cu: one thread per rollout,
// rollout_lanes.cu: one body per lane).
#pragma once
#include <cuda_runtime.h>

namespace {

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 mk(float x, float y, float z) { V3 v; v.x = x; v.y = y; v.z = z; return v; }
__device__ __forceinline__ V3 operator+(V3 a, V3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ V3 operator-(V3 a, V3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ V3 operator*(float s, V3 a) { return mk(s * a.x, s * a.y, s * a.z); }
__device__ __forceinline__ float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

struct S3 { float xx, yy, zz, xy, xz, yz; };                        // symmetric 3x3
struct M3 { float m00, m01, m02, m10, m11, m12, m20, m21, m22; };   // general 3x3, row major

__device__ __forceinline__ V3 mul(const S3& s, V3 v) {
    return mk(s.xx * v.x + s.xy * v.y + s.xz * v.z, s.xy * v.x + s.yy * v.y + s.yz * v.z, s.xz * v.x + s.yz * v.y + s.zz * v.z);
}
__device__ __forceinline__ V3 mul(const M3& m, V3 v) {
    return mk(m.m00 * v.x + m.m01 * v.y + m.m02 * v.z, m.m10 * v.x + m.m11 * v.y + m.m12 * v.z, m.m20 * v.x + m.m21 * v.y + m.m22 * v.z);
}
__device__ __forceinline__ V3 mulT(const M3& m, V3 v) {
    return mk(m.m00 * v.x + m.m10 * v.y + m.m20 * v.z, m.m01 * v.x + m.m11 * v.y + m.m21 * v.z, m.m02 * v.x + m.m12 * v.y + m.m22 * v.z);
}

// sin / cos with a two-term Cody-Waite reduction and the Cephes minimax polynomials on [-pi/4, pi/4]: max error 9e-8 for
// |x| < 3000 rad (checked against float64), ~25 instructions and NO slow path.  CUDA's sincosf carries a Payne-Hanek
// fallback whose code, registers and convergence barriers this kernel does not need.
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

struct Quat { float x, y, z, w; };
__device__ __forceinline__ Quat qmul(Quat a, Quat b) {
    Quat o;
    o.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
    o.y = a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x;
    o.z = a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w;
    o.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    return o;
}
__device__ __forceinline__ M3 quat_to_R(Quat q) {
    M3 R;
    R.m00 = 1 - 2 * (q.y * q.y + q.z * q.z); R.m01 = 2 * (q.x * q.y - q.z * q.w); R.m02 = 2 * (q.x * q.z + q.y * q.w);
    R.m10 = 2 * (q.x * q.y + q.z * q.w); R.m11 = 1 - 2 * (q.x * q.x + q.z * q.z); R.m12 = 2 * (q.y * q.z - q.x * q.w);
    R.m20 = 2 * (q.x * q.z - q.y * q.w); R.m21 = 2 * (q.y * q.z + q.x * q.w); R.m22 = 1 - 2 * (q.x * q.x + q.y * q.y);
    return R;
}

}  // namespace
