// gsr_calib.cuh — the intrinsics and lens-coefficient gradients of one visible gaussian (gsr_pose.cu compiled with
// GSR_POSE_CAMERA, libgsr_calib.so).
//
// Every camera model projects as u = fx a_d(p) + cx, v = fy b_d(p) + cy, so J's rows are fx d a_d / dp and
// fy d b_d / dp.  With g_uv the complete gradient on (u, v) and gJ the gradient on J (conic_bwd's, after the
// antialiased terms):
//   dL/dfx = g_u a_d + sum_j gJ_0j (d a_d / dp_j),   dL/dcx = g_u,   the same for fy, cy with row 1,
//   dL/dk  = g_uv . d(u, v)/dk + sum_ij gJ_ij dJ_ij / dk.
// a_d, b_d and J are affine in the lens coefficients (fisheye: theta_d = theta P(theta^2) is linear in k, and so are
// s, q, d and the near-axis series; distortion: a_d, b_d and D), so d/dk are the coefficient parts of the existing
// expressions, formed directly (never as J(k + e_j) - J(k), which cancels near the optical axis).
//
// out: fx fy cx cy, then the lens's coefficients in the order of its constants.  Written with explicit rounding
// intrinsics, so the single-view and the batched kernels give the same bits.
#pragma once
#include "gsr_distortion.cuh"
#include "gsr_fisheye.cuh"
#include "gsr_math.cuh"

namespace gsr {

#define GSR_FMA __fmaf_rn
#define GSR_MUL __fmul_rn
#define GSR_ADD __fadd_rn

// the intrinsics part shared by every lens: n0, n1 = J's rows divided by fx, fy (the lens's normalised rows)
__device__ __forceinline__ void intrinsics_contribution(float ad, float bd, const float* __restrict__ n0,
                                                        const float* __restrict__ n1, float gu, float gv,
                                                        const float* __restrict__ gJ, float* __restrict__ out) {
    out[0] = GSR_FMA(gJ[2], n0[2], GSR_FMA(gJ[1], n0[1], GSR_FMA(gJ[0], n0[0], GSR_MUL(gu, ad))));
    out[1] = GSR_FMA(gJ[5], n1[2], GSR_FMA(gJ[4], n1[1], GSR_FMA(gJ[3], n1[0], GSR_MUL(gv, bd))));
    out[2] = gu;
    out[3] = gv;
}

// pinhole: a_d = x / z, rows (1/z, 0, -x/z^2), (0, 1/z, -y/z^2).  out [4]
__device__ __forceinline__ void pinhole_calib(float x, float y, float z, float gu, float gv,
                                              const float* __restrict__ gJ, float* __restrict__ out) {
    const float iz = __frcp_rn(z);
    const float a = GSR_MUL(x, iz), b = GSR_MUL(y, iz);
    const float n0[3] = {iz, 0.f, -GSR_MUL(a, iz)}, n1[3] = {0.f, iz, -GSR_MUL(b, iz)};
    intrinsics_contribution(a, b, n0, n1, gu, gv, gJ, out);
}

// fisheye: a_d = s x, rows (s + x^2 q, x y q, x d), (x y q, s + y^2 q, y d) (gsr_fisheye.cuh).  With k_j's parts
// ds_j, dq_j, dd_j of s, q, d:
//   dL/dk_j = A_s ds_j + A_q dq_j + A_d dd_j,  A_s = fx (g_u x + gJ0) + fy (g_v y + gJ4),
//   A_q = fx x (gJ0 x + gJ1 y) + fy y (gJ3 x + gJ4 y),  A_d = fx gJ2 x + fy gJ5 y.
// Closed forms (theta^2 >= FE_SERIES_T): ds_j = theta t^j / rho, dm_j = t^j ((2j+1) sin cos - theta) / sin^3,
// dd_j = -(2j+1) t^j / R^2, dq_j = dm_j / R^3; below, the k_j parts of h and M0..M3.  out [8]
__device__ __forceinline__ void fisheye_calib(float x, float y, float z, float fx, float fy,
                                              const float* __restrict__ kc, float gu, float gv,
                                              const float* __restrict__ gJ, float* __restrict__ out) {
    const FisheyeTerms f = fisheye_terms<false>(x, y, z, kc);
    const float xx = GSR_MUL(x, x), yy = GSR_MUL(y, y), xy = GSR_MUL(x, y);
    const float xyq = GSR_MUL(xy, f.q);
    const float n0[3] = {GSR_FMA(xx, f.q, f.s), xyq, GSR_MUL(x, f.d)};
    const float n1[3] = {xyq, GSR_FMA(yy, f.q, f.s), GSR_MUL(y, f.d)};
    intrinsics_contribution(GSR_MUL(f.s, x), GSR_MUL(f.s, y), n0, n1, gu, gv, gJ, out);

    const float r2 = GSR_FMA(x, x, yy);
    const float rho = __fsqrt_rn(r2);
    const float R2 = GSR_FMA(z, z, r2);
    const float R = __fsqrt_rn(R2);
    const float th = atan2f(rho, z);
    const float t = GSR_MUL(th, th);
    const float tp[4] = {t, GSR_MUL(t, t), GSR_MUL(GSR_MUL(t, t), t), GSR_MUL(GSR_MUL(t, t), GSR_MUL(t, t))};
    const float iR = __frcp_rn(R), iR2 = __frcp_rn(R2);
    const float iR3 = GSR_MUL(iR2, iR);
    float ds[4], dq[4], dd[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) dd[j] = -GSR_MUL(GSR_MUL((float)(2 * j + 3), tp[j]), iR2);
    if (t < FE_SERIES_T) {
        // h = 1 + t (k1 + 1/6) + t^2 (k1/6 + k2 + 7/360) + t^3 (294 k1 + 2520 k2 + 15120 k3 + 31) / 15120, s = h / R
        const float dh[4] = {GSR_FMA(tp[2], 294.0f / 15120.0f, GSR_FMA(tp[1], 1.0f / 6.0f, t)),
                             GSR_FMA(tp[2], 1.0f / 6.0f, tp[1]), tp[2], 0.f};
        // m = M0 + t M1 + t^2 M2 + t^3 M3 (gsr_fisheye.cuh's coefficients)
        const float dm[4] = {
            GSR_FMA(t, GSR_FMA(t, GSR_FMA(t, -2305.0f / 37800.0f, -133.0f / 420.0f), -1.0f), 2.0f),
            GSR_MUL(t, GSR_FMA(t, GSR_FMA(t, -16380.0f / 37800.0f, -4.0f / 3.0f), 4.0f)),
            GSR_MUL(tp[1], GSR_FMA(t, -5.0f / 3.0f, 6.0f)), GSR_MUL(tp[2], 8.0f)};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            ds[j] = GSR_MUL(dh[j], iR);
            dq[j] = GSR_MUL(dm[j], iR3);
        }
    } else {
        const float sn = GSR_MUL(rho, iR), cs = GSR_MUL(z, iR);
        const float isn3 = __frcp_rn(GSR_MUL(GSR_MUL(sn, sn), sn));
        const float snc = GSR_MUL(sn, cs), th_rho = __fdiv_rn(th, rho);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            ds[j] = GSR_MUL(th_rho, tp[j]);
            dq[j] = GSR_MUL(GSR_MUL(GSR_MUL(tp[j], GSR_FMA((float)(2 * j + 3), snc, -th)), isn3), iR3);
        }
    }
    const float As = GSR_FMA(fy, GSR_FMA(gv, y, gJ[4]), GSR_MUL(fx, GSR_FMA(gu, x, gJ[0])));
    const float Aq = GSR_FMA(GSR_MUL(fy, y), GSR_FMA(gJ[3], x, GSR_MUL(gJ[4], y)),
                             GSR_MUL(GSR_MUL(fx, x), GSR_FMA(gJ[0], x, GSR_MUL(gJ[1], y))));
    const float Ad = GSR_FMA(GSR_MUL(fy, gJ[5]), y, GSR_MUL(GSR_MUL(fx, gJ[2]), x));
#pragma unroll
    for (int j = 0; j < 4; ++j) out[4 + j] = GSR_FMA(Ad, dd[j], GSR_FMA(Aq, dq[j], GSR_MUL(As, ds[j])));
}

// distortion {k1, k2, p1, p2, k3}: with a = x/z, b = y/z, s = a^2 + b^2 and (gsr_distortion.cuh)
//   E00 = fx (gJ0 - a gJ2), E01 = fx (gJ1 - b gJ2), E10 = fy (gJ3 - a gJ5), E11 = fy (gJ4 - b gJ5), e01 = E01 + E10,
//   sum_ij gJ_ij dJ_ij = (E00 dD00 + e01 dD01 + E11 dD11) / z.
// The radial k_n (n = 1, 2, 3; dR = s^n, dR' = n s^(n-1)): dD00 = s^n + 2 n a^2 s^(n-1), dD01 = 2 n a b s^(n-1),
// dD11 = s^n + 2 n b^2 s^(n-1), d(a_d, b_d) = (a, b) s^n, so
//   dL/dk_n = (U a + V b + (E00 + E11) / z) s^n + 2 n s^(n-1) (E00 a^2 + e01 a b + E11 b^2) / z,   U = fx g_u, V = fy g_v
// and the tangential p1: d(a_d, b_d) = (2 a b, s + 2 b^2), (dD00, dD01, dD11) = (2 b, 2 a, 6 b);
// p2: d(a_d, b_d) = (s + 2 a^2, 2 a b), (dD00, dD01, dD11) = (6 a, 2 b, 2 a).  out [9]
__device__ __forceinline__ void distortion_calib(float x, float y, float z, float fx, float fy,
                                                 const float* __restrict__ kc, float gu, float gv,
                                                 const float* __restrict__ gJ, float* __restrict__ out) {
    const DistortionTerms d = distortion_terms<false>(x, y, z, kc);
    const float a = d.a, b = d.b, iz = d.iz;
    const float k1 = kc[0], k2 = kc[1], p1 = kc[2], p2 = kc[3], k3 = kc[4];
    const float aa = GSR_MUL(a, a), bb = GSR_MUL(b, b), ab = GSR_MUL(a, b);
    const float s = GSR_ADD(aa, bb);
    const float R = GSR_FMA(s, GSR_FMA(s, GSR_FMA(s, k3, k2), k1), 1.0f);
    const float ta = GSR_FMA(2.0f, aa, s), tb = GSR_FMA(2.0f, bb, s);  // s + 2 a^2, s + 2 b^2
    const float ad = GSR_FMA(a, R, GSR_FMA(GSR_MUL(2.0f, p1), ab, GSR_MUL(p2, ta)));
    const float bd = GSR_FMA(b, R, GSR_FMA(GSR_MUL(2.0f, p2), ab, GSR_MUL(p1, tb)));
    const float n0[3] = {GSR_MUL(iz, d.D00), GSR_MUL(iz, d.D01), -GSR_MUL(iz, GSR_FMA(a, d.D00, GSR_MUL(b, d.D01)))};
    const float n1[3] = {GSR_MUL(iz, d.D01), GSR_MUL(iz, d.D11), -GSR_MUL(iz, GSR_FMA(a, d.D01, GSR_MUL(b, d.D11)))};
    intrinsics_contribution(ad, bd, n0, n1, gu, gv, gJ, out);

    const float C0 = GSR_MUL(gJ[2], fx), C1 = GSR_MUL(gJ[5], fy);
    const float E00 = GSR_FMA(-a, C0, GSR_MUL(gJ[0], fx)), E01 = GSR_FMA(-b, C0, GSR_MUL(gJ[1], fx));
    const float E10 = GSR_FMA(-a, C1, GSR_MUL(gJ[3], fy)), E11 = GSR_FMA(-b, C1, GSR_MUL(gJ[4], fy));
    const float e01 = GSR_ADD(E01, E10);
    const float U = GSR_MUL(fx, gu), V = GSR_MUL(fy, gv);
    const float lin = GSR_FMA(GSR_ADD(E00, E11), iz, GSR_FMA(U, a, GSR_MUL(V, b)));
    const float Q = GSR_MUL(iz, GSR_FMA(E11, bb, GSR_FMA(e01, ab, GSR_MUL(E00, aa))));
    const float s2 = GSR_MUL(s, s);
    out[4] = GSR_FMA(2.0f, Q, GSR_MUL(lin, s));                                   // k1
    out[5] = GSR_FMA(GSR_MUL(4.0f, s), Q, GSR_MUL(lin, s2));                      // k2
    out[6] = GSR_FMA(GSR_MUL(2.0f, ab), U, GSR_MUL(tb, V));                       // p1: uv
    out[6] = GSR_FMA(iz, GSR_FMA(GSR_MUL(2.0f, b), E00, GSR_FMA(GSR_MUL(2.0f, a), e01, GSR_MUL(GSR_MUL(6.0f, b), E11))),
                     out[6]);                                                     // p1: J
    out[7] = GSR_FMA(ta, U, GSR_MUL(GSR_MUL(2.0f, ab), V));                       // p2: uv
    out[7] = GSR_FMA(iz, GSR_FMA(GSR_MUL(6.0f, a), E00, GSR_FMA(GSR_MUL(2.0f, b), e01, GSR_MUL(GSR_MUL(2.0f, a), E11))),
                     out[7]);                                                     // p2: J
    out[8] = GSR_FMA(GSR_MUL(6.0f, s2), Q, GSR_MUL(lin, GSR_MUL(s2, s)));         // k3
}

#undef GSR_FMA
#undef GSR_MUL
#undef GSR_ADD

}  // namespace gsr
