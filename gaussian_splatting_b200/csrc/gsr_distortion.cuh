// gsr_distortion.cuh — COLMAP's OPENCV (radial-tangential, OpenCV's 5-coefficient) projection, its Jacobian and their
// VJPs, fp32.
//
// With p = (x, y, z), iz = 1 / z, a = x iz, b = y iz, s = a^2 + b^2 and the coefficients {k1, k2, p1, p2, k3}:
//   R   = 1 + k1 s + k2 s^2 + k3 s^3,   R' = dR/ds = k1 + 2 k2 s + 3 k3 s^2,   R'' = 2 k2 + 6 k3 s
//   a_d = a R + 2 p1 a b + p2 (s + 2 a^2),   b_d = b R + p1 (s + 2 b^2) + 2 p2 a b
//   u = fx a_d + cx,   v = fy b_d + cy
// The lens Jacobian D = d(a_d, b_d) / d(a, b) is symmetric:
//   D00 = R + 2 a^2 R' + 2 p1 b + 6 p2 a,   D01 = D10 = 2 a b R' + 2 p1 a + 2 p2 b,
//   D11 = R + 2 b^2 R' + 6 p1 b + 2 p2 a
// and with d(a, b) / dp = iz [[1, 0, -a], [0, 1, -b]]
//   J = diag(fx, fy) D d(a, b)/dp = iz [[fx D00, fx D01, -fx (a D00 + b D01)], [fy D01, fy D11, -fy (a D01 + b D11)]].
// Its contraction with a gradient gJ: with (A_i, B_i, C_i) = f_i (gJ_i0, gJ_i1, gJ_i2) (f = fx, fy) and
// E_i0 = A_i - a C_i, E_i1 = B_i - b C_i,  L = sum gJ_ij J_ij = iz M,  M = E00 D00 + (E01 + E10) D01 + E11 D11, so
//   dL/da = iz (dM/da|_E - C0 D00 - C1 D01),   dL/db = iz (dM/db|_E - C0 D01 - C1 D11),   dL/diz = M
//   g = (iz dL/da, iz dL/db, -iz (a dL/da + b dL/db + iz M))
// where dM/d(a, b)|_E takes the second derivatives of a_d and b_d:
//   dD00/da = 6 a R' + 4 a^3 R'' + 6 p2,  dD00/db = dD01/da = 2 b R' + 4 a^2 b R'' + 2 p1,
//   dD01/db = dD11/da = 2 a R' + 4 a b^2 R'' + 2 p2,  dD11/db = 6 b R' + 4 b^3 R'' + 6 p1.
// Everything is a polynomial in (a, b) times powers of iz: unlike the fisheye there is no 0/0 form and no series
// branch.  With all coefficients zero, R = 1 and the tangential terms vanish exactly, so a_d = a and D = I.
#pragma once
#include "gsr_math.cuh"

namespace gsr {

// projected mean and s = (x^2 + y^2) / z^2 (for the fold cull).  kc: {k1, k2, p1, p2, k3, r2_max}
__device__ __forceinline__ void distortion_project(float x, float y, float z, float fx, float cx, float fy, float cy,
                                                   const float* kc, float& u, float& v, float& s) {
    const float iz = 1.0f / z;
    const float a = x * iz, b = y * iz;
    const float aa = a * a, bb = b * b, ab = a * b;
    s = aa + bb;
    const float R = fmaf(s, fmaf(s, fmaf(s, kc[4], kc[1]), kc[0]), 1.0f);
    const float ad = fmaf(a, R, fmaf(2.0f * kc[2], ab, kc[3] * fmaf(2.0f, aa, s)));
    const float bd = fmaf(b, R, fmaf(2.0f * kc[3], ab, kc[2] * fmaf(2.0f, bb, s)));
    u = fmaf(fx, ad, cx);
    v = fmaf(fy, bd, cy);
}

struct DistortionTerms {
    float iz, a, b, R1, R2;  // R1 = R', R2 = R'' (SECOND only)
    float D00, D01, D11;
};

template <bool SECOND>
__device__ __forceinline__ DistortionTerms distortion_terms(float x, float y, float z, const float* kc) {
    const float k1 = kc[0], k2 = kc[1], p1 = kc[2], p2 = kc[3], k3 = kc[4];
    DistortionTerms o;
    o.iz = 1.0f / z;
    o.a = x * o.iz;
    o.b = y * o.iz;
    const float a = o.a, b = o.b;
    const float s = fmaf(a, a, b * b);
    const float R = fmaf(s, fmaf(s, fmaf(s, k3, k2), k1), 1.0f);
    o.R1 = fmaf(s, fmaf(s, 3.0f * k3, 2.0f * k2), k1);
    o.R2 = SECOND ? fmaf(s, 6.0f * k3, 2.0f * k2) : 0.f;
    const float tR1 = 2.0f * o.R1;
    o.D00 = fmaf(a * a, tR1, R) + fmaf(2.0f * p1, b, 6.0f * p2 * a);
    o.D01 = fmaf(a * b, tR1, 2.0f * fmaf(p1, a, p2 * b));
    o.D11 = fmaf(b * b, tR1, R) + fmaf(6.0f * p1, b, 2.0f * p2 * a);
    return o;
}

__device__ __forceinline__ void distortion_jacobian(float x, float y, float z, float fx, float fy, const float* kc,
                                                    float* __restrict__ J) {
    const DistortionTerms t = distortion_terms<false>(x, y, z, kc);
    const float fxz = fx * t.iz, fyz = fy * t.iz;
    J[0] = fxz * t.D00;
    J[1] = fxz * t.D01;
    J[2] = -fxz * fmaf(t.a, t.D00, t.b * t.D01);
    J[3] = fyz * t.D01;
    J[4] = fyz * t.D11;
    J[5] = -fyz * fmaf(t.a, t.D01, t.b * t.D11);
}

// g = sum_ij gJ_ij dJ_ij / dp
__device__ __forceinline__ void distortion_jacobian_bwd(float x, float y, float z, float fx, float fy, const float* kc,
                                                        const float* __restrict__ gJ, float* __restrict__ g) {
    const DistortionTerms t = distortion_terms<true>(x, y, z, kc);
    const float p1 = kc[2], p2 = kc[3];
    const float a = t.a, b = t.b, iz = t.iz;
    const float C0 = gJ[2] * fx, C1 = gJ[5] * fy;
    const float E00 = fmaf(-a, C0, gJ[0] * fx), E01 = fmaf(-b, C0, gJ[1] * fx);
    const float E10 = fmaf(-a, C1, gJ[3] * fy), E11 = fmaf(-b, C1, gJ[4] * fy);
    const float e01 = E01 + E10;  // D01 == D10
    const float M = fmaf(E00, t.D00, fmaf(e01, t.D01, E11 * t.D11));
    const float aR2 = 4.0f * t.R2 * a, bR2 = 4.0f * t.R2 * b;
    const float Daa = fmaf(a * a, aR2, fmaf(6.0f * a, t.R1, 6.0f * p2));  // dD00/da
    const float Dab = fmaf(a * a, bR2, fmaf(2.0f * b, t.R1, 2.0f * p1));  // dD00/db = dD01/da
    const float Dbb = fmaf(b * b, aR2, fmaf(2.0f * a, t.R1, 2.0f * p2));  // dD01/db = dD11/da
    const float Dbbb = fmaf(b * b, bR2, fmaf(6.0f * b, t.R1, 6.0f * p1)); // dD11/db
    const float Ma = fmaf(E00, Daa, fmaf(e01, Dab, E11 * Dbb)) - fmaf(C0, t.D00, C1 * t.D01);
    const float Mb = fmaf(E00, Dab, fmaf(e01, Dbb, E11 * Dbbb)) - fmaf(C0, t.D01, C1 * t.D11);
    const float La = iz * Ma, Lb = iz * Mb;
    g[0] = iz * La;
    g[1] = iz * Lb;
    g[2] = -iz * fmaf(a, La, fmaf(b, Lb, iz * M));
}

// g = J^T (gu, gv): J is exactly d(u, v) / dp
__device__ __forceinline__ void distortion_project_bwd(const float* __restrict__ J, float gu, float gv,
                                                       float* __restrict__ g) {
#pragma unroll
    for (int k = 0; k < 3; ++k) g[k] = J[k] * gu + J[3 + k] * gv;
}

}  // namespace gsr

// The camera-model hooks of gsr_preprocess.cuh for this lens, for a translation unit that defines GSR_DISTORTION_HOOKS
// before including this header and then includes gsr_preprocess.cuh (gsr_lens.cu, gsr_pose.cu).  The lens
// constants of view `view` are read into shared memory next to the view constants.
#ifdef GSR_DISTORTION_HOOKS
#define GSR_PROJECTION_HOOKS
#define GSR_VIEW_PARAM , const float* __restrict__ distortion
#define GSR_VIEW_DECL __shared__ float vdc[GSR_DISTORTION_CONSTS];
#define GSR_LOAD_VIEW(T, K, cam, view)                                                                          \
    do {                                                                                                        \
        if (threadIdx.x >= 32 && threadIdx.x < 32 + GSR_DISTORTION_CONSTS)                                      \
            vdc[threadIdx.x - 32] = distortion[GSR_DISTORTION_CONSTS * (view) + threadIdx.x - 32];              \
        load_view_cta(T, K, cam, vc, HAS_SH); /* ends with a CTA barrier */                                     \
    } while (0)
#define GSR_PROJECT(px, py, pz, u, v) \
    float dt_s;                       \
    distortion_project(px, py, pz, vc.K[0], vc.K[2], vc.K[4], vc.K[5], vdc, u, v, dt_s)
#define GSR_CULL_MORE | (dt_s >= vdc[5])
#define GSR_JACOBIAN(px, py, pz, J) distortion_jacobian(px, py, pz, vc.K[0], vc.K[4], vdc, J)
#define GSR_JACOBIAN_BWD(px, py, pz, gJ, g) distortion_jacobian_bwd(px, py, pz, vc.K[0], vc.K[4], vdc, gJ, g)
#define GSR_PROJECT_BWD(px, py, pz, gu, gv, g) distortion_project_bwd(J, gu, gv, g)
#endif
