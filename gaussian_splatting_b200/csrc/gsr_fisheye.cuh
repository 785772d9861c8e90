// gsr_fisheye.cuh — COLMAP's OPENCV_FISHEYE (Kannala-Brandt) projection, its Jacobian and their VJPs, fp32.
//
// With p = (x, y, z), rho = |(x, y)|, R = |p|, theta = atan2(rho, z), t = theta^2 and
//   g(theta) = theta P(t),  P = 1 + k1 t + k2 t^2 + k3 t^3 + k4 t^4      (theta_d)
//   s = g / rho,            u = fx s x + cx,  v = fy s y + cy
// the Jacobian is
//   J = [[fx (s + x^2 q), fx x y q, fx x d], [fy x y q, fy (s + y^2 q), fy y d]]
//   q = (ds/drho) / rho = m(theta) / R^3,   m = (g' sin cos - g) / sin^3,   d = ds/dz = -g'(theta) / R^2
// and its derivative needs, besides q and d,
//   q' = (dq/drho) / rho = (m' cot - 3 m) / R^5,   e = dq/dz = -(m' sin + 3 m cos) / R^4,
//   d_z = dd/dz = (g'' sin + 2 g' cos) / R^3.
// s = h(theta) / R with h = g / sin, and h, m, m' / theta are smooth even functions of theta whose closed forms are
// 0/0 at theta = 0: below theta^2 = 1e-4 they come from their Taylor series in t (four terms, truncation t^4).  The
// closed forms lose about eps / theta^2 (m) and eps / theta^4 (m') relatively just above the switch, but they enter
// J and its derivative multiplied by rho^2 and rho^3, which leaves an error of a few eps of J.
#pragma once
#include "gsr_math.cuh"

namespace gsr {

constexpr float FE_SERIES_T = 1e-4f;  // theta^2 below which the series branch is taken

struct FisheyeTerms {
    float s, q, d;      // first order
    float qp, e, dz;    // second order (fisheye_terms<true>)
};

// k: {k1, k2, k3, k4}.  Assumes z > 0 for the Jacobian (every visible gaussian has z >= near > 0).
template <bool SECOND>
__device__ __forceinline__ FisheyeTerms fisheye_terms(float x, float y, float z, const float* k) {
    const float k1 = k[0], k2 = k[1], k3 = k[2], k4 = k[3];
    const float r2 = fmaf(x, x, y * y);
    const float rho = sqrtf(r2);
    const float R2 = fmaf(z, z, r2);
    const float th = atan2f(rho, z);
    const float t = th * th;
    const float P = fmaf(t, fmaf(t, fmaf(t, fmaf(t, k4, k3), k2), k1), 1.0f);
    const float G1 = fmaf(t, fmaf(t, fmaf(t, fmaf(t, 9.0f * k4, 7.0f * k3), 5.0f * k2), 3.0f * k1), 1.0f);  // g'
    FisheyeTerms o;
    o.d = -G1 / R2;
    const float R = sqrtf(R2);
    float m, mc = 0.f, ms = 0.f;  // m, m' cot(theta), m' sin(theta)
    if (t < FE_SERIES_T) {
        const float h = fmaf(t, fmaf(t, fmaf(t, (294.0f * k1 + 2520.0f * k2 + 15120.0f * k3 + 31.0f) / 15120.0f,
                                             k1 / 6.0f + k2 + 7.0f / 360.0f),
                                     k1 + 1.0f / 6.0f),
                             1.0f);
        const float M0 = 2.0f * k1 - 2.0f / 3.0f;
        const float M1 = -(5.0f * k1 - 20.0f * k2 + 1.0f) / 5.0f;
        const float M2 = -(133.0f * k1 + 560.0f * k2 - 2520.0f * k3 + 17.0f) / 420.0f;
        const float M3 = -(2305.0f * k1 + 16380.0f * k2 + 63000.0f * k3 - 302400.0f * k4 + 261.0f) / 37800.0f;
        m = fmaf(t, fmaf(t, fmaf(t, M3, M2), M1), M0);
        o.s = h / R;
        if (SECOND) {
            const float N3 = -(32747.0f * k1 + 271040.0f * k2 + 1829520.0f * k3 + 6652800.0f * k4 + 3543.0f) / 415800.0f;
            const float n = fmaf(t, fmaf(t, fmaf(t, N3, 6.0f * M3), 4.0f * M2), 2.0f * M1);  // m' / theta
            const float tcot = fmaf(t, fmaf(t, -1.0f / 45.0f, -1.0f / 3.0f), 1.0f);          // theta cot(theta)
            mc = n * tcot;
            ms = n * th * (rho / R);
        }
    } else {
        const float g = th * P;
        const float sn = rho / R, cs = z / R;
        const float sn2 = sn * sn, sn3 = sn2 * sn;
        const float num = fmaf(G1 * sn, cs, -g);  // g' sin cos - g
        m = num / sn3;
        o.s = g / rho;
        if (SECOND) {
            const float G2 = fmaf(t, fmaf(t, fmaf(t, 72.0f * k4, 42.0f * k3), 20.0f * k2), 6.0f * k1);  // g'' / theta
            const float mp = (th * G2 * sn2 * cs - 2.0f * G1 * sn3 - 3.0f * cs * num) / (sn2 * sn2);
            mc = mp * cs / sn;
            ms = mp * sn;
        }
    }
    const float R3 = R2 * R;
    o.q = m / R3;
    if (SECOND) {
        const float G2 = fmaf(t, fmaf(t, fmaf(t, 72.0f * k4, 42.0f * k3), 20.0f * k2), 6.0f * k1);
        const float cs = z / R, sn = rho / R;
        o.qp = (mc - 3.0f * m) / (R3 * R2);
        o.e = -(ms + 3.0f * m * cs) / (R2 * R2);
        o.dz = (th * G2 * sn + 2.0f * G1 * cs) / R3;
    } else {
        o.qp = o.e = o.dz = 0.f;
    }
    return o;
}

// projected mean and theta (for the cull).  kc: {k1, k2, k3, k4, theta_max}
__device__ __forceinline__ void fisheye_project(float x, float y, float z, float fx, float cx, float fy, float cy,
                                                const float* kc, float& u, float& v, float& theta) {
    const FisheyeTerms f = fisheye_terms<false>(x, y, z, kc);
    theta = atan2f(sqrtf(fmaf(x, x, y * y)), z);
    u = fmaf(fx, f.s * x, cx);
    v = fmaf(fy, f.s * y, cy);
}

__device__ __forceinline__ void fisheye_jacobian(float x, float y, float z, float fx, float fy, const float* kc,
                                                 float* __restrict__ J) {
    const FisheyeTerms f = fisheye_terms<false>(x, y, z, kc);
    const float xyq = x * y * f.q;
    J[0] = fx * fmaf(x * x, f.q, f.s);
    J[1] = fx * xyq;
    J[2] = fx * x * f.d;
    J[3] = fy * xyq;
    J[4] = fy * fmaf(y * y, f.q, f.s);
    J[5] = fy * y * f.d;
}

// g = sum_ij gJ_ij dJ_ij / dp
__device__ __forceinline__ void fisheye_jacobian_bwd(float x, float y, float z, float fx, float fy, const float* kc,
                                                     const float* __restrict__ gJ, float* __restrict__ g) {
    const FisheyeTerms f = fisheye_terms<true>(x, y, z, kc);
    const float a0 = gJ[0] * fx, a1 = gJ[1] * fx, a2 = gJ[2] * fx;
    const float b0 = gJ[3] * fy, b1 = gJ[4] * fy, b2 = gJ[5] * fy;
    const float xx = x * x, yy = y * y, xy = x * y;
    const float c = a1 + b0;  // J1 and J3 have the same shape
    // d/dx, d/dy, d/dz of (s + x^2 q), x y q, x d, (s + y^2 q), y d
    const float A_x = x * fmaf(xx, f.qp, 3.0f * f.q), A_y = y * fmaf(xx, f.qp, f.q), A_z = fmaf(xx, f.e, f.d);
    const float B_x = y * fmaf(xx, f.qp, f.q), B_y = x * fmaf(yy, f.qp, f.q), B_z = xy * f.e;
    const float C_x = fmaf(xx, f.e, f.d), C_y = xy * f.e, C_z = x * f.dz;
    const float D_x = x * fmaf(yy, f.qp, f.q), D_y = y * fmaf(yy, f.qp, 3.0f * f.q), D_z = fmaf(yy, f.e, f.d);
    const float E_x = xy * f.e, E_y = fmaf(yy, f.e, f.d), E_z = y * f.dz;
    g[0] = a0 * A_x + c * B_x + a2 * C_x + b1 * D_x + b2 * E_x;
    g[1] = a0 * A_y + c * B_y + a2 * C_y + b1 * D_y + b2 * E_y;
    g[2] = a0 * A_z + c * B_z + a2 * C_z + b1 * D_z + b2 * E_z;
}

// g = J^T (gu, gv): J is exactly d(u, v) / dp
__device__ __forceinline__ void fisheye_project_bwd(const float* __restrict__ J, float gu, float gv,
                                                    float* __restrict__ g) {
#pragma unroll
    for (int k = 0; k < 3; ++k) g[k] = J[k] * gu + J[3 + k] * gv;
}

}  // namespace gsr

// The camera-model hooks of gsr_preprocess.cuh for this lens, for a translation unit that defines GSR_FISHEYE_HOOKS
// before including this header and then includes gsr_preprocess.cuh (gsr_lens.cu, gsr_pose.cu).  The lens
// constants of view `view` are read into shared memory next to the view constants.
#ifdef GSR_FISHEYE_HOOKS
#define GSR_PROJECTION_HOOKS
#define GSR_VIEW_PARAM , const float* __restrict__ fisheye
#define GSR_VIEW_DECL __shared__ float vfe[GSR_FISHEYE_CONSTS];
#define GSR_LOAD_VIEW(T, K, cam, view)                                                                          \
    do {                                                                                                        \
        if (threadIdx.x >= 32 && threadIdx.x < 32 + GSR_FISHEYE_CONSTS)                                         \
            vfe[threadIdx.x - 32] = fisheye[GSR_FISHEYE_CONSTS * (view) + threadIdx.x - 32];                     \
        load_view_cta(T, K, cam, vc, HAS_SH); /* ends with a CTA barrier */                                     \
    } while (0)
#define GSR_PROJECT(px, py, pz, u, v) \
    float fe_theta;                   \
    fisheye_project(px, py, pz, vc.K[0], vc.K[2], vc.K[4], vc.K[5], vfe, u, v, fe_theta)
#define GSR_CULL_MORE | (fe_theta >= vfe[4])
#define GSR_JACOBIAN(px, py, pz, J) fisheye_jacobian(px, py, pz, vc.K[0], vc.K[4], vfe, J)
#define GSR_JACOBIAN_BWD(px, py, pz, gJ, g) fisheye_jacobian_bwd(px, py, pz, vc.K[0], vc.K[4], vfe, gJ, g)
#define GSR_PROJECT_BWD(px, py, pz, gu, gv, g) fisheye_project_bwd(J, gu, gv, g)
#endif
