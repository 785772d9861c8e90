// gsr_pose.cuh — the pose-gradient hooks of gsr_preprocess.cuh (gsr_pose.cu, libgsr_pose.so).
//
// With T = camera_T_world, W = T[:3, :3] and the camera-frame mean p = W x + t, one visible gaussian contributes
//   dL/dW += g_p x^T + J^T (2 G M Sigma),   dL/dt += g_p
// where g_p is the complete gradient on p (projection, Jacobian, depth, uv, lens), G the symmetric 2x2 gradient on the
// 2-D covariance M Sigma M^T (the packed conic gradient gc after the antialiased rho terms), M = J W, and Sigma the
// (filtered) world covariance.  The camera centre of the SH view direction is held constant, as for xyz.
//
// Each thread holds its gaussian's 12 values (T[:3, :] row-major; NV values with the camera gradient).  After every
// view the CTA adds them up in a fixed order (a shuffle tree per warp, then the 4 warps in order) and writes one partial
// per CTA and view: [C, grid, NV].
// k_pose_finish adds the partials of a view in fp64 in a fixed order and rounds once.  The per-gaussian arithmetic is
// written with explicit rounding intrinsics, so the single-view and the batched kernels give the same bits for the
// same rows.
#pragma once
#include "gsr_common.cuh"

namespace gsr {

constexpr int POSE_VALUES = 12;
constexpr int POSE_CTA_THREADS = 128;  // PRE_THREADS of gsr_preprocess.cuh (checked in gsr_pose.cu)

// acc = this gaussian's contribution; J [6], W [9], S [9] (Sigma, full), gc [3] (packed conic gradient), gp [3]
__device__ __forceinline__ void pose_contribution(const float* __restrict__ J, const float* __restrict__ W,
                                                  const float* __restrict__ S, const float* __restrict__ gc,
                                                  const float* __restrict__ gp, float x, float y, float z,
                                                  float* __restrict__ acc) {
    float M[6], MS[6], P[6];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            M[r * 3 + c] = __fmaf_rn(J[r * 3 + 2], W[6 + c], __fmaf_rn(J[r * 3 + 1], W[3 + c], __fmul_rn(J[r * 3], W[c])));
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            MS[r * 3 + c] =
                __fmaf_rn(M[r * 3 + 2], S[6 + c], __fmaf_rn(M[r * 3 + 1], S[3 + c], __fmul_rn(M[r * 3], S[c])));
    // P = 2 G M Sigma, G = [[gc0, gc1], [gc1, gc2]] (the off-diagonal entries of M Sigma M^T share gc1)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        P[c] = __fmul_rn(2.0f, __fmaf_rn(gc[1], MS[3 + c], __fmul_rn(gc[0], MS[c])));
        P[3 + c] = __fmul_rn(2.0f, __fmaf_rn(gc[2], MS[3 + c], __fmul_rn(gc[1], MS[c])));
    }
    const float xw[3] = {x, y, z};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
            acc[r * 4 + c] = __fmaf_rn(J[3 + r], P[3 + c], __fmaf_rn(J[r], P[c], __fmul_rn(gp[r], xw[c])));
        acc[r * 4 + 3] = gp[r];
    }
}

// Whole CTA: the fixed-order sum of every thread's NV values into out[0..NV-1].  Every thread must call it.  The
// shared scratch may be rewritten by the next call only after a CTA barrier (the batched body has one per view).
template <int NV>
__device__ __forceinline__ void pose_cta_reduce(const float* __restrict__ acc, float* __restrict__ out) {
    static_assert(NV <= POSE_CTA_THREADS, "one thread per value adds the warps' sums");
    __shared__ float s_pose[POSE_CTA_THREADS / 32][NV];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        float v = acc[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v = __fadd_rn(v, __shfl_down_sync(0xffffffffu, v, off));
        if (lane == 0) s_pose[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        float v = s_pose[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < POSE_CTA_THREADS / 32; ++w) v = __fadd_rn(v, s_pose[w][threadIdx.x]);
        out[threadIdx.x] = v;
    }
}

constexpr int POSE_FINISH_THREADS = 256;

// Whole CTA of POSE_FINISH_THREADS, one view: thread t adds the partials t, t + 256, ... of src [nblk, NV] in fp64,
// then a shuffle tree per warp leaves the warps' sums in s_sum; ends with a CTA barrier.  The caller adds the warps in
// order and rounds once.
template <int NV>
__device__ __forceinline__ void finish_partials(int nblk, const float* __restrict__ src, double (*s_sum)[NV]) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    double acc[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = 0.0;
    for (int b = t; b < nblk; b += POSE_FINISH_THREADS) {
        const float4* row = reinterpret_cast<const float4*>(src + (size_t)b * NV);
#pragma unroll
        for (int q = 0; q < NV / 4; ++q) {
            const float4 v = row[q];
            acc[4 * q + 0] += (double)v.x;
            acc[4 * q + 1] += (double)v.y;
            acc[4 * q + 2] += (double)v.z;
            acc[4 * q + 3] += (double)v.w;
        }
    }
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        double v = acc[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
        if (lane == 0) s_sum[warp][k] = v;
    }
    __syncthreads();
}

}  // namespace gsr

// The hooks (gsr_preprocess.cuh): the bodies take the partials [C, grid, NV] as one more trailing parameter.  With
// GSR_POSE_CAMERA (the camera-gradient kernels, gsr_calib.cuh) a row is the 12 pose values followed by
// CAMERA_VALUES - 12 intrinsics and lens values, added by GSR_CAMERA_VIEW.
#define GSR_POSE_HOOKS
#define GSR_POSE_PARAM , float* __restrict__ pose_partials
#ifdef GSR_POSE_CAMERA
#define GSR_POSE_DECL float gpose[CAMERA_VALUES] = {};
#define GSR_POSE_VIEW                                   \
    pose_contribution(J, W, S9, gc, gp, x, y, z, gpose); \
    GSR_CAMERA_VIEW(px, py, pz, guv, gJ, gpose + POSE_VALUES);
#define GSR_POSE_REDUCE(view) \
    pose_cta_reduce<CAMERA_VALUES>(gpose, pose_partials + ((size_t)(view) * gridDim.x + blockIdx.x) * CAMERA_VALUES);
#else
#define GSR_POSE_DECL float gpose[POSE_VALUES] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#define GSR_POSE_VIEW pose_contribution(J, W, S9, gc, gp, x, y, z, gpose);
#define GSR_POSE_REDUCE(view) \
    pose_cta_reduce<POSE_VALUES>(gpose, pose_partials + ((size_t)(view) * gridDim.x + blockIdx.x) * POSE_VALUES);
#endif
