/* calib_oracle.c — CPU oracle of the intrinsics and lens-coefficient gradients of the fused rasterizer's per-gaussian
 * stage, fp64.
 *
 * TEST INFRASTRUCTURE ONLY (tests/calib_oracle.py).  Compiled with -DPOSE_LENS=1 or 2 on top of pose_oracle.c (and so
 * of fisheye_oracle.c or distortion_oracle.c, whose zero coefficients are the pinhole); reuses their projection, their
 * Jacobian and the pose oracle's gradient on J:  gJ = 2 G M Sigma W^T.  Every model projects as u = fx a_d + cx,
 * v = fy b_d + cy, so
 *   dL/dfx = g_u a_d + sum_j gJ_0j J1_0j,   dL/dcx = g_u   (fy, cy with row 1)
 * with a_d, b_d the projection and J1 the Jacobian at fx = fy = 1, cx = cy = 0.  (u, v) and J are affine in every lens
 * coefficient, so d/dk_j = F(k + e_j) - F(k) exactly; in fp64 that difference loses ~1e-16 |F| absolutely, far below
 * the kernels' fp32 tolerances.  (The kernels form the derivatives in closed form instead: in fp32 the difference would
 * cancel near the optical axis.)
 *
 *   calib_vjp_f64   per-gaussian contributions [N, 4 + NK] (fx fy cx cy, then the NK coefficients), 0 when not visible
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mfma -shared -fPIC -I<repo>/oracle -I<repo>/tests -DPOSE_LENS=1|2
 *        calib_oracle.c -lm
 */
#include "pose_oracle.c"

#if POSE_LENS == 1
#define NK 4
/* (u, v) at p for K and the coefficients k */
static void lens_project(const double* p, const double* K, const double* k, double* uv) {
    double f[7];
    fe_terms_f64(p, k, f);
    uv[0] = K[0] * f[0] * p[0] + K[2];
    uv[1] = K[4] * f[0] * p[1] + K[5];
}
#else
#define NK 5
static void lens_project(const double* p, const double* K, const double* k, double* uv) {
    double s;
    dt_project_point_f64(p, K, k, uv, &s);
}
#endif

/* kc: the lens constants (coefficients, then the cull limit); g_uv [N,2], g_conic [N,3] (after the antialiased rho
 * terms); contrib [N, 4 + NK] */
void calib_vjp_f64(int N, const double* xyz, const double* quat, const double* scale, const double* T, const double* K,
                   const double* kc, const unsigned char* visible, const double* g_uv, const double* g_conic,
                   double* contrib) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < N; ++i) {
        double* out = contrib + (size_t)i * (4 + NK);
        for (int k = 0; k < 4 + NK; ++k) out[k] = 0;
        if (!visible[i]) continue;
        double p[3], S[9], J[6], W[9], g[3];
        transform_point_f64(T, xyz[i * 3], xyz[i * 3 + 1], xyz[i * 3 + 2], p);
        sigma_world_f64(quat + i * 4, scale + i * 3, S);
        const int wi[9] = {0, 1, 2, 4, 5, 6, 8, 9, 10};
        for (int k = 0; k < 9; ++k) W[k] = T[wi[k]];
        const double zero_gJ[6] = {0, 0, 0, 0, 0, 0}, zero_uv[2] = {0, 0};
        LENS_JACOBIAN_VJP(p, K[0], K[4], kc, zero_gJ, zero_uv, J, g);
        const double G[4] = {g_conic[i * 3], g_conic[i * 3 + 1], g_conic[i * 3 + 1], g_conic[i * 3 + 2]};
        double M[6], MS[6], GMS[6], P[6], Wt[9], gJ[6];
        mmd_f64(J, W, M, 2, 3, 3);
        mmd_f64(M, S, MS, 2, 3, 3);
        mmd_f64(G, MS, GMS, 2, 2, 3);
        for (int k = 0; k < 6; ++k) P[k] = 2 * GMS[k];
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Wt[c * 3 + r] = W[r * 3 + c];
        mmd_f64(P, Wt, gJ, 2, 3, 3);
        const double gu = g_uv[i * 2], gv = g_uv[i * 2 + 1];

        /* intrinsics: the projection and the Jacobian at unit focal lengths and a zero principal point */
        const double K1[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        double ab[2], J1[6];
        lens_project(p, K1, kc, ab);
        LENS_JACOBIAN_VJP(p, 1.0, 1.0, kc, zero_gJ, zero_uv, J1, g);
        out[0] = gu * ab[0] + gJ[0] * J1[0] + gJ[1] * J1[1] + gJ[2] * J1[2];
        out[1] = gv * ab[1] + gJ[3] * J1[3] + gJ[4] * J1[4] + gJ[5] * J1[5];
        out[2] = gu;
        out[3] = gv;

        /* lens coefficients: the unit steps of an affine function */
        double uv0[2];
        lens_project(p, K, kc, uv0);
        for (int j = 0; j < NK; ++j) {
            double k1[NK + 1], uvj[2], Jj[6];
            for (int m = 0; m <= NK; ++m) k1[m] = kc[m];
            k1[j] += 1;
            lens_project(p, K, k1, uvj);
            LENS_JACOBIAN_VJP(p, K[0], K[4], k1, zero_gJ, zero_uv, Jj, g);
            double a = gu * (uvj[0] - uv0[0]) + gv * (uvj[1] - uv0[1]);
            for (int m = 0; m < 6; ++m) a += gJ[m] * (Jj[m] - J[m]);
            out[4 + j] = a;
        }
    }
}
