/* pose_oracle.c — CPU oracle of the camera pose gradient of the fused rasterizer's per-gaussian stage, fp64.
 *
 * TEST INFRASTRUCTURE ONLY (tests/pose_oracle.py).  Compiled with -DPOSE_LENS=1 on top of fisheye_oracle.c or with
 * -DPOSE_LENS=2 on top of distortion_oracle.c (whose zero coefficients are the pinhole), and reuses their Jacobian and
 * its VJP unchanged.  With T = camera_T_world, W = T[:3, :3], p = W x + t, M = J W, the 2-D covariance M Sigma M^T and
 * its symmetric gradient G (packed conic gradient {g0, g1, g2}: G = [[g0, g1], [g1, g2]]):
 *   P = dL/dM = 2 G M Sigma,   dL/dJ = P W^T,   g_p = J^T g_uv + <dL/dJ, dJ/dp> + g_z e_z,
 *   dL/dW = g_p x^T + J^T P,   dL/dt = g_p.
 *
 *   pose_vjp_f64   per-gaussian contributions [N, 12] (T[:3, :] row-major), 0 for the gaussians not visible
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mfma -shared -fPIC -I<repo>/oracle -I<repo>/tests -DPOSE_LENS=1|2
 *        pose_oracle.c -lm
 */
#if POSE_LENS == 1
#include "fisheye_oracle.c"
#define LENS_JACOBIAN_VJP fe_jacobian_vjp_f64
#else
#include "distortion_oracle.c"
#define LENS_JACOBIAN_VJP dt_jacobian_vjp_f64
#endif

/* scale: the log-scales of the world covariance the forward used (filtered with filter3d); kc: the lens constants;
 * g_uv [N,2], g_conic [N,3] (after the antialiased rho terms), g_z [N] (camera-frame z) */
void pose_vjp_f64(int N, const double* xyz, const double* quat, const double* scale, const double* T, const double* K,
                  const double* kc, const unsigned char* visible, const double* g_uv, const double* g_conic,
                  const double* g_z, double* contrib) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < N; ++i) {
        double* out = contrib + (size_t)i * 12;
        for (int k = 0; k < 12; ++k) out[k] = 0;
        if (!visible[i]) continue;
        double p[3], S[9], J[6], W[9];
        transform_point_f64(T, xyz[i * 3], xyz[i * 3 + 1], xyz[i * 3 + 2], p);
        sigma_world_f64(quat + i * 4, scale + i * 3, S);
        const int wi[9] = {0, 1, 2, 4, 5, 6, 8, 9, 10};
        for (int k = 0; k < 9; ++k) W[k] = T[wi[k]];
        double J0[6], g0[3];
        const double zero_gJ[6] = {0, 0, 0, 0, 0, 0}, zero_uv[2] = {0, 0};
        LENS_JACOBIAN_VJP(p, K[0], K[4], kc, zero_gJ, zero_uv, J0, g0);  /* J at p */
        for (int k = 0; k < 6; ++k) J[k] = J0[k];
        const double G[4] = {g_conic[i * 3], g_conic[i * 3 + 1], g_conic[i * 3 + 1], g_conic[i * 3 + 2]};
        double M[6], MS[6], GMS[6], P[6], Wt[9], gJ[6], gp[3];
        mmd_f64(J, W, M, 2, 3, 3);
        mmd_f64(M, S, MS, 2, 3, 3);
        mmd_f64(G, MS, GMS, 2, 2, 3);
        for (int k = 0; k < 6; ++k) P[k] = 2 * GMS[k];
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Wt[c * 3 + r] = W[r * 3 + c];
        mmd_f64(P, Wt, gJ, 2, 3, 3);
        LENS_JACOBIAN_VJP(p, K[0], K[4], kc, gJ, g_uv + i * 2, J, gp);
        gp[2] += g_z[i];
        const double x[3] = {xyz[i * 3], xyz[i * 3 + 1], xyz[i * 3 + 2]};
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) out[r * 4 + c] = gp[r] * x[c] + J[r] * P[c] + J[3 + r] * P[3 + c];
            out[r * 4 + 3] = gp[r];
        }
    }
}
