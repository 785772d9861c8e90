// gsr_math_bwd.cuh — analytic VJPs of the per-Gaussian projection chain.
//
// Values follow the reference's backward kernels (file:line per function);
// gradients carry no bit contract (reference accumulates them with fp32
// atomics, SURVEY.md Q18), so ordinary arithmetic is used here.
#pragma once
#include "gsr_math.cuh"

namespace gsr {

template <typename T, int RA, int CA, int CB>
__device__ __forceinline__ void mm(const T* __restrict__ A, const T* __restrict__ B, T* __restrict__ C) {
#pragma unroll
    for (int r = 0; r < RA; ++r)
#pragma unroll
        for (int c = 0; c < CB; ++c) {
            T s = T(0);
#pragma unroll
            for (int k = 0; k < CA; ++k) s += A[r * CA + k] * B[k * CB + c];
            C[r * CB + c] = s;
        }
}

// VJP of u = fx*x/z + cx, v = fy*y/z + cy.  Reference: src/projection_backward.cu:20-35
// (no gradient when z <= 0).  Returns false when the reference leaves the output untouched.
template <typename T>
__device__ __forceinline__ bool project_uv_bwd(T x, T y, T z, T fx, T fy, T gu, T gv, T* __restrict__ g) {
    if (z <= T(0)) return false;
    const T du_dx = fx / z;
    const T dv_dy = fy / z;
    const T du_dz = -fx * x / (z * z);
    const T dv_dz = -fy * y / (z * z);
    g[0] = gu * du_dx;
    g[1] = gv * dv_dy;
    g[2] = gu * du_dz + gv * dv_dz;
    return true;
}

// VJP of the projection Jacobian wrt the camera-frame point.
// Reference: src/projection_backward.cu:105-119.
template <typename T>
__device__ __forceinline__ void proj_jacobian_bwd(T x, T y, T z, T fx, T fy, const T* __restrict__ gJ,
                                                  T* __restrict__ g) {
    const T zz = z * z;
    const T zzz = zz * z;
    g[0] = gJ[2] * -fx / zz;
    g[1] = gJ[5] * -fy / zz;
    g[2] = gJ[0] * -fx / zz + gJ[4] * -fy / zz + gJ[2] * T(2) * x * fx / zzz +
           gJ[5] * T(2) * y * fy / zzz;
}

// VJP of conic = f(Sigma, J, W).  Reference: src/projection_backward.cu:396-470.
// gS: 3x3 (full) grad of Sigma, gJ: 2x3 grad of J.  (grad wrt W is dropped, :461-464)
template <typename T>
__device__ __forceinline__ void conic_bwd(const T* __restrict__ S /*9*/, const T* __restrict__ J /*6*/,
                                          const T* __restrict__ W /*9*/, const T* __restrict__ gc /*3*/,
                                          T* __restrict__ gS /*9*/, T* __restrict__ gJ /*6*/) {
    T JW[6], JWt[6];
    mm<T, 2, 3, 3>(J, W, JW);
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) JWt[c * 2 + r] = JW[r * 3 + c];
    const T G[4] = {gc[0], gc[1], gc[1], gc[2]};  // symmetric 2x2
    T JWtG[6];
    mm<T, 3, 2, 2>(JWt, G, JWtG);
    mm<T, 3, 2, 3>(JWtG, JW, gS);
    T SJWt[6], left[6], St[9], StJWt[6], right[6], gJWt[6], gJt[6];
    mm<T, 3, 3, 2>(S, JWt, SJWt);
    mm<T, 3, 2, 2>(SJWt, G, left);  // G^T == G
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) St[c * 3 + r] = S[r * 3 + c];
    mm<T, 3, 3, 2>(St, JWt, StJWt);
    mm<T, 3, 2, 2>(StJWt, G, right);
#pragma unroll
    for (int i = 0; i < 6; ++i) gJWt[i] = left[i] + right[i];
    mm<T, 3, 3, 2>(W, gJWt, gJt);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 2; ++c) gJ[c * 3 + r] = gJt[r * 2 + c];
}

// VJP of Sigma_world = R diag(e)^2 R^T wrt the quaternion and, through de[k] = d e_k / d s_k, the log-scale s.
// Reference: src/projection_backward.cu:185-314.
template <typename T>
__device__ __forceinline__ void sigma_world_bwd_e(T qw, T qx, T qy, T qz, const T* __restrict__ e /*3*/,
                                                  const T* __restrict__ de /*3*/, const T* __restrict__ G /*9*/,
                                                  T* __restrict__ gq /*4 wxyz*/, T* __restrict__ gs /*3*/) {
    const T nq = Ar<T>::sqrt(qw * qw + qx * qx + qy * qy + qz * qz);
    const T w = qw / nq, x = qx / nq, y = qy / nq, z = qz / nq;
    T R[9];
    R[0] = T(1) - T(2) * y * y - T(2) * z * z;
    R[1] = T(2) * x * y - T(2) * z * w;
    R[2] = T(2) * x * z + T(2) * y * w;
    R[3] = T(2) * x * y + T(2) * z * w;
    R[4] = T(1) - T(2) * x * x - T(2) * z * z;
    R[5] = T(2) * y * z - T(2) * x * w;
    R[6] = T(2) * x * z - T(2) * y * w;
    R[7] = T(2) * y * z + T(2) * x * w;
    R[8] = T(1) - T(2) * x * x - T(2) * y * y;
    T RS[9], RSt[9], Rt[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            RS[r * 3 + c] = R[r * 3 + c] * e[c];
            RSt[c * 3 + r] = RS[r * 3 + c];
            Rt[c * 3 + r] = R[r * 3 + c];
        }
    T gRS[9], gSR[9];
    mm<T, 3, 3, 3>(G, RS, gRS);
    mm<T, 3, 3, 3>(RSt, G, gSR);
    T gR[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) gR[r * 3 + c] = gRS[r * 3 + c] * e[c] + e[c] * gSR[c * 3 + r];
    T gSa[9], gSb[9];
    mm<T, 3, 3, 3>(Rt, gRS, gSa);
    mm<T, 3, 3, 3>(gSR, R, gSb);
#pragma unroll
    for (int k = 0; k < 3; ++k) gs[k] = (gSa[k * 4] + gSb[k * 4]) * de[k];

    T gn[4];
    gn[0] = -T(2) * z * gR[1] + T(2) * y * gR[2] + T(2) * z * gR[3] - T(2) * x * gR[5] -
            T(2) * y * gR[6] + T(2) * x * gR[7];
    gn[1] = T(2) * y * gR[1] + T(2) * z * gR[2] + T(2) * y * gR[3] - T(4) * x * gR[4] -
            T(2) * w * gR[5] + T(2) * z * gR[6] + T(2) * w * gR[7] - T(4) * x * gR[8];
    gn[2] = -T(4) * y * gR[0] + T(2) * x * gR[1] + T(2) * w * gR[2] + T(2) * x * gR[3] +
            T(2) * z * gR[5] - T(2) * w * gR[6] + T(2) * z * gR[7] - T(4) * y * gR[8];
    gn[3] = -T(4) * z * gR[0] - T(2) * w * gR[1] + T(2) * x * gR[2] + T(2) * w * gR[3] -
            T(4) * z * gR[4] + T(2) * y * gR[5] + T(2) * x * gR[6] + T(2) * y * gR[7];
    // through q/|q|: (I/|q| - q q^T/|q|^3) gn
    const T n3 = nq * nq * nq;
    const T q[4] = {qw, qx, qy, qz};
    const T dot = q[0] * gn[0] + q[1] * gn[1] + q[2] * gn[2] + q[3] * gn[3];
#pragma unroll
    for (int i = 0; i < 4; ++i) gq[i] = gn[i] / nq - q[i] * dot / n3;
}

template <typename T>
__device__ __forceinline__ void sigma_world_bwd(T qw, T qx, T qy, T qz, T s0, T s1, T s2,
                                                const T* __restrict__ G /*9*/, T* __restrict__ gq /*4 wxyz*/,
                                                T* __restrict__ gs /*3*/) {
    const T e[3] = {Ar<T>::exp(s0), Ar<T>::exp(s1), Ar<T>::exp(s2)};
    sigma_world_bwd_e<T>(qw, qx, qy, qz, e, e, G, gq, gs);
}

// 3-D filter (Mip-Splatting): Sigma = R diag(v + F) R^T with v_k = e_k^2.  The quaternion gradient is the plain one at
// e'_k = sqrt(v_k + F); the scale chain is d/ds_k (v_k + F) = 2 v_k, i.e. the plain one with de'_k = v_k / e'_k.
// F == 0 selects e' = de' = e, the unfiltered VJP.
template <typename T>
__device__ __forceinline__ void sigma_world_bwd_f3d(T qw, T qx, T qy, T qz, const T* __restrict__ e /*3*/,
                                                    const T* __restrict__ v /*3*/, const T* __restrict__ vp /*3*/,
                                                    T F, const T* __restrict__ G /*9*/, T* __restrict__ gq /*4*/,
                                                    T* __restrict__ gs /*3*/) {
    T ep[3], dep[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const T r = Ar<T>::sqrt(vp[k]);
        ep[k] = F == T(0) ? e[k] : r;
        dep[k] = F == T(0) ? e[k] : v[k] / r;
    }
    sigma_world_bwd_e<T>(qw, qx, qy, qz, ep, dep, G, gq, gs);
}

}  // namespace gsr
