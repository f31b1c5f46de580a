// cost.cu -- fused cost terms callable from a user's Objective (optional: an Objective written with plain torch ops
// on the obs views works unchanged).  One kernel replaces the ~28 element-wise torch launches of the pose-reach cost
// of the reference's panda Objectives (examples/panda/planner.py:22-40, examples/panda_pick/planner.py:24-53):
//     cost[i] (+)= w_pos * | a[i, 0:3] - b[i, 0:3] |  +  w_ori * | euler_ZYX(R(a[i, 3:7]))[0:2] |
// with the quaternion handed REAL-FIRST to the matrix formula exactly as the reference does (SURVEY Appendix A #11).
// HBM-bound: 7 (+3) reads + 1 write of 4 B per element, fully coalesced on the [row][T*K] obs layout.
#include "common.cuh"

namespace {

__global__ void __launch_bounds__(256)
mppib_cost_pose_kernel(long long n, const float* __restrict__ a, long long a_si, long long a_sr, const float* __restrict__ b, long long b_si,
                       long long b_sr, float w_pos, float w_ori, float* __restrict__ cost, int accumulate) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float* ai = a + i * a_si;
        float c = 0.f;
        if (w_pos != 0.f) {
            const float* bi = b + i * b_si;
            const float dx = ai[0] - bi[0], dy = ai[a_sr] - bi[b_sr], dz = ai[2 * a_sr] - bi[2 * b_sr];
            c = w_pos * sqrtf(dx * dx + dy * dy + dz * dz);
        }
        if (w_ori != 0.f) {
            const float r = ai[3 * a_sr], qi = ai[4 * a_sr], qj = ai[5 * a_sr], qk = ai[6 * a_sr];
            const float two_s = 2.0f / (r * r + qi * qi + qj * qj + qk * qk);
            const float m00 = 1.0f - two_s * (qj * qj + qk * qk);
            const float m10 = two_s * (qi * qj + qk * r);
            const float m20 = two_s * (qi * qk - qj * r);
            const float yaw = atan2f(m10, m00), pitch = asinf(-m20);
            c += w_ori * sqrtf(yaw * yaw + pitch * pitch);
        }
        cost[i] = accumulate ? cost[i] + c : c;
    }
}

}  // namespace

int launch_cost_pose(long long n, const float* a, long long a_si, long long a_sr, const float* b, long long b_si, long long b_sr, float w_pos,
                     float w_ori, float* cost, int accumulate, cudaStream_t s) {
    if (n <= 0) return 0;
    // this entry has no handle: run on the device that owns `cost` (the caller's current device may be another one, e.g. a planner
    // on cuda:1 served from a thread whose current device is cuda:0), and give the caller's device back afterwards
    cudaPointerAttributes attr;
    MPPIB_CHECK_CUDA(cudaPointerGetAttributes(&attr, cost));
    MPPIB_REQUIRE(attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged, "mppib_cost_pose: `cost` is not device memory");
    DeviceGuard guard(attr.device);
    MPPIB_CHECK_CUDA(guard.err);
    const int block = 256;
    const long long want = (n + block - 1) / block;
    int sms = 0;
    MPPIB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, attr.device));
    const int grid = (int)(want < 8LL * sms ? want : 8LL * sms);
    mppib_cost_pose_kernel<<<grid, block, 0, s>>>(n, a, a_si, a_sr, b, b_si, b_sr, w_pos, w_ori, cost, accumulate);
    MPPIB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
