/* distortion_oracle.c — CPU oracle of the radial-tangential per-gaussian stage (rasterize(..., distortion=k)) and its
 * VJP, fp64.
 *
 * TEST INFRASTRUCTURE ONLY (tests/distortion_oracle.py).  Compiled together with oracle/gsr_oracle.c, whose helpers
 * (transform_point, sigma_world, conic, mmd, sh_basis, view_dir) it reuses unchanged.
 *
 * COLMAP's OPENCV model, k = {k1, k2, p1, p2, k3}: q = (a, b) = (x / z, y / z), s = a^2 + b^2,
 *   R = 1 + k1 s + k2 s^2 + k3 s^3,  d(q) = q R + t(q),
 *   t = (2 p1 a b + p2 (3 a^2 + b^2), p1 (a^2 + 3 b^2) + 2 p2 a b),   u = fx d_0 + cx,  v = fy d_1 + cy.
 * Written here in tensor form, independently of the kernels' closed forms (gsr_distortion.cuh):
 *   J_ik = f_i sum_m D_im P_mk,   D = dd/dq,  P = dq/dp,
 *   dJ_ik/dp_l = f_i sum_m (sum_n Hd_imn P_nl) P_mk + f_i sum_m D_im dP_mkl,
 * with the Hessians Hd of d (product rule on q_i R(s) plus the constant Hessians of t) and dP of q(p).
 *
 *   dt_project_point_f64     (u, v) and s at one camera-frame point
 *   dt_jacobian_vjp_f64      J at p, and g = J^T g_uv + sum_ij gJ_ij dJ_ij / dp
 *   dt_project_f64           orc_project with the distorted projection, Jacobian and the s >= r2_max cull
 *   dt_project_backward_f64  orc_project_backward with the distorted Jacobian and the camera-frame z gradient
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mfma -shared -fPIC -I<repo>/oracle distortion_oracle.c -lm
 */
#include "gsr_oracle.c"

/* q, s, R, R', R'' at p */
static void dt_radial(const double* p, const double* k, double* q, double* s, double* R, double* R1, double* R2) {
    q[0] = p[0] / p[2];
    q[1] = p[1] / p[2];
    *s = q[0] * q[0] + q[1] * q[1];
    const double S = *s;
    *R = 1 + S * (k[0] + S * (k[1] + S * k[4]));
    *R1 = k[0] + S * (2 * k[1] + S * 3 * k[4]);
    *R2 = 2 * k[1] + S * 6 * k[4];
}

/* K: 3x3 row-major; uv [2]; s_out: (x^2 + y^2) / z^2 */
void dt_project_point_f64(const double* p, const double* K, const double* k, double* uv, double* s_out) {
    double q[2], s, R, R1, R2;
    dt_radial(p, k, q, &s, &R, &R1, &R2);
    const double a = q[0], b = q[1], p1 = k[2], p2 = k[3];
    const double ta = 2 * p1 * a * b + p2 * (3 * a * a + b * b), tb = p1 * (a * a + 3 * b * b) + 2 * p2 * a * b;
    uv[0] = K[0] * (a * R + ta) + K[2];
    uv[1] = K[4] * (b * R + tb) + K[5];
    *s_out = s;
}

/* D [2][2], Hd [2][2][2], P [2][3], dP [2][3][3] */
static void dt_parts(const double* p, const double* k, double D[2][2], double Hd[2][2][2], double P[2][3],
                     double dP[2][3][3]) {
    double q[2], s, R, R1, R2;
    dt_radial(p, k, q, &s, &R, &R1, &R2);
    const double p1 = k[2], p2 = k[3];
    const double gt[2][2] = {{2 * p1 * q[1] + 6 * p2 * q[0], 2 * p1 * q[0] + 2 * p2 * q[1]},
                             {2 * p1 * q[0] + 2 * p2 * q[1], 6 * p1 * q[1] + 2 * p2 * q[0]}};
    const double Ht[2][2][2] = {{{6 * p2, 2 * p1}, {2 * p1, 2 * p2}}, {{2 * p1, 2 * p2}, {2 * p2, 6 * p1}}};
    double dR[2], ddR[2][2];
    for (int m = 0; m < 2; ++m) {
        dR[m] = 2 * q[m] * R1;
        for (int n = 0; n < 2; ++n) ddR[m][n] = (m == n ? 2 * R1 : 0) + 4 * q[m] * q[n] * R2;
    }
    for (int i = 0; i < 2; ++i)
        for (int m = 0; m < 2; ++m) {
            D[i][m] = (i == m ? R : 0) + q[i] * dR[m] + gt[i][m];
            for (int n = 0; n < 2; ++n)
                Hd[i][m][n] = (i == m ? dR[n] : 0) + (i == n ? dR[m] : 0) + q[i] * ddR[m][n] + Ht[i][m][n];
        }
    const double iz = 1 / p[2];
    for (int m = 0; m < 2; ++m) {
        for (int c = 0; c < 3; ++c) {
            P[m][c] = (c == m ? iz : 0) + (c == 2 ? -q[m] * iz : 0);
            for (int l = 0; l < 3; ++l) dP[m][c][l] = 0;
        }
        /* q_m = p_m / z */
        dP[m][m][2] = dP[m][2][m] = -iz * iz;
        dP[m][2][2] = 2 * q[m] * iz * iz;
    }
}

static void dt_jacobian(const double* p, double fx, double fy, const double* k, double* J) {
    double D[2][2], Hd[2][2][2], P[2][3], dP[2][3][3];
    dt_parts(p, k, D, Hd, P, dP);
    const double f[2] = {fx, fy};
    for (int i = 0; i < 2; ++i)
        for (int c = 0; c < 3; ++c) J[i * 3 + c] = f[i] * (D[i][0] * P[0][c] + D[i][1] * P[1][c]);
}

/* J [6], g [3] = J^T g_uv + contraction of dJ/dp with gJ */
void dt_jacobian_vjp_f64(const double* p, double fx, double fy, const double* k, const double* gJ, const double* guv,
                         double* J, double* g) {
    double D[2][2], Hd[2][2][2], P[2][3], dP[2][3][3];
    dt_parts(p, k, D, Hd, P, dP);
    const double f[2] = {fx, fy};
    for (int i = 0; i < 2; ++i)
        for (int c = 0; c < 3; ++c) J[i * 3 + c] = f[i] * (D[i][0] * P[0][c] + D[i][1] * P[1][c]);
    for (int l = 0; l < 3; ++l) {
        double acc = J[l] * guv[0] + J[3 + l] * guv[1];
        for (int i = 0; i < 2; ++i)
            for (int c = 0; c < 3; ++c) {
                double h = 0;
                for (int m = 0; m < 2; ++m) {
                    for (int n = 0; n < 2; ++n) h += Hd[i][m][n] * P[n][l] * P[m][c];
                    h += D[i][m] * dP[m][c][l];
                }
                acc += gJ[i * 3 + c] * f[i] * h;
            }
        g[l] = acc;
    }
}

/* kc: k1 k2 p1 p2 k3 r2_max.  s_out [N] */
void dt_project_f64(int N, int n_sh, const double* xyz, const double* quat, const double* scale,
                    const double* opa_logit, const double* rgb_dc, const double* sh, const double* T, const double* K,
                    const double* cam_centre, const double* kc, double width, double height, double near_t,
                    double far_t, double pad, double* xyz_cam, double* uv, double* conic, double* opa,
                    double* rgb_out, unsigned char* visible, double* s_out) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < N; ++i) {
        double p[3];
        transform_point_f64(T, xyz[i * 3], xyz[i * 3 + 1], xyz[i * 3 + 2], p);
        double uvp[2], s;
        dt_project_point_f64(p, K, kc, uvp, &s);
        const double u = uvp[0], v = uvp[1];
        for (int k = 0; k < 3; ++k) xyz_cam[i * 3 + k] = p[k];
        uv[i * 2] = u; uv[i * 2 + 1] = v;
        s_out[i] = s;
        const int culled = (p[2] < near_t) || (p[2] > far_t) || (u < -pad) || (u > width + pad) || (v < -pad) ||
                           (v > height + pad) || (s >= kc[5]) || u != u || v != v;
        visible[i] = culled ? 0 : 1;
        if (culled) continue;
        double S[9], J[6];
        sigma_world_f64(quat + i * 4, scale + i * 3, S);
        dt_jacobian(p, K[0], K[4], kc, J);
        conic_f64(S, J, T, conic + i * 3);
        opa[i] = 1.0 / (1.0 + exp(-opa_logit[i]));
        if (sh == NULL || n_sh == 1) {
            for (int c = 0; c < 3; ++c) rgb_out[i * 3 + c] = rgb_dc[i * 3 + c];
        } else {
            double d[3], Y[16];
            view_dir_f64(xyz + i * 3, cam_centre, d);
            sh_basis_f64(n_sh, d[0], d[1], d[2], Y);
            const int nr = n_sh - 1;
            for (int c = 0; c < 3; ++c) {
                double acc = Y[0] * rgb_dc[i * 3 + c];
                for (int k = 1; k < n_sh; ++k) acc += Y[k] * sh[((size_t)i * 3 + c) * nr + (k - 1)];
                rgb_out[i * 3 + c] = acc * RSH0F;
            }
        }
    }
}

/* VJP from render-stage rows (all [N, .]): g_opa is the gradient on sigmoid(o), g_z on camera-frame z */
void dt_project_backward_f64(int N, int n_sh, const double* xyz, const double* quat, const double* scale,
                             const double* opa_logit, const double* sh_present, const double* T, const double* K,
                             const double* cam_centre, const double* kc, const unsigned char* visible,
                             const double* g_rgb, const double* g_opa, const double* g_uv, const double* g_conic,
                             const double* g_z, double* d_xyz, double* d_quat, double* d_scale, double* d_opa,
                             double* d_dc, double* d_sh) {
    const int nr = n_sh - 1;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < N; ++i) {
        for (int k = 0; k < 3; ++k) { d_xyz[i * 3 + k] = 0; d_scale[i * 3 + k] = 0; d_dc[i * 3 + k] = 0; }
        for (int k = 0; k < 4; ++k) d_quat[i * 4 + k] = 0;
        d_opa[i] = 0;
        if (sh_present) for (int k = 0; k < 3 * nr; ++k) d_sh[(size_t)i * 3 * nr + k] = 0;
        if (!visible[i]) continue;
        double p[3], S[9], J[6], W[9];
        transform_point_f64(T, xyz[i * 3], xyz[i * 3 + 1], xyz[i * 3 + 2], p);
        sigma_world_f64(quat + i * 4, scale + i * 3, S);
        dt_jacobian(p, K[0], K[4], kc, J);
        const int wi[9] = {0, 1, 2, 4, 5, 6, 8, 9, 10};
        for (int k = 0; k < 9; ++k) W[k] = T[wi[k]];
        /* conic backward: gS = (JW)^T G (JW), gJ = (G JW (S + S^T)) W^T */
        double JW[6], JWt[6], G[4] = {g_conic[i * 3], g_conic[i * 3 + 1], g_conic[i * 3 + 1], g_conic[i * 3 + 2]};
        mmd_f64(J, W, JW, 2, 3, 3);
        for (int r = 0; r < 2; ++r) for (int c = 0; c < 3; ++c) JWt[c * 2 + r] = JW[r * 3 + c];
        double t32[6], gS[9], SJWt[6], left[6], St[9], StJWt[6], right[6], gJWt[6], gJt[6], gJ[6];
        mmd_f64(JWt, G, t32, 3, 2, 2);
        mmd_f64(t32, JW, gS, 3, 2, 3);
        mmd_f64(S, JWt, SJWt, 3, 3, 2);
        mmd_f64(SJWt, G, left, 3, 2, 2);
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) St[c * 3 + r] = S[r * 3 + c];
        mmd_f64(St, JWt, StJWt, 3, 3, 2);
        mmd_f64(StJWt, G, right, 3, 2, 2);
        for (int k = 0; k < 6; ++k) gJWt[k] = left[k] + right[k];
        mmd_f64(W, gJWt, gJt, 3, 3, 2);
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 2; ++c) gJ[c * 3 + r] = gJt[r * 2 + c];
        /* Sigma_world backward */
        const double qw0 = quat[i * 4], qx0 = quat[i * 4 + 1], qy0 = quat[i * 4 + 2], qz0 = quat[i * 4 + 3];
        const double nq = sqrt(qw0 * qw0 + qx0 * qx0 + qy0 * qy0 + qz0 * qz0);
        const double w = qw0 / nq, x = qx0 / nq, y = qy0 / nq, z = qz0 / nq;
        const double e[3] = {exp(scale[i * 3]), exp(scale[i * 3 + 1]), exp(scale[i * 3 + 2])};
        const double R[9] = {1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * z * w, 2 * x * z + 2 * y * w,
                             2 * x * y + 2 * z * w, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * x * w,
                             2 * x * z - 2 * y * w, 2 * y * z + 2 * x * w, 1 - 2 * x * x - 2 * y * y};
        double RS[9], RSt[9], Rt[9], gRS[9], gSR[9], gR[9], gSa[9], gSb[9];
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) {
            RS[r * 3 + c] = R[r * 3 + c] * e[c]; RSt[c * 3 + r] = RS[r * 3 + c]; Rt[c * 3 + r] = R[r * 3 + c];
        }
        mmd_f64(gS, RS, gRS, 3, 3, 3);
        mmd_f64(RSt, gS, gSR, 3, 3, 3);
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) gR[r * 3 + c] = gRS[r * 3 + c] * e[c] + e[c] * gSR[c * 3 + r];
        mmd_f64(Rt, gRS, gSa, 3, 3, 3);
        mmd_f64(gSR, R, gSb, 3, 3, 3);
        for (int k = 0; k < 3; ++k) d_scale[i * 3 + k] = (gSa[k * 4] + gSb[k * 4]) * e[k];
        double gn[4];
        gn[0] = -2 * z * gR[1] + 2 * y * gR[2] + 2 * z * gR[3] - 2 * x * gR[5] - 2 * y * gR[6] + 2 * x * gR[7];
        gn[1] = 2 * y * gR[1] + 2 * z * gR[2] + 2 * y * gR[3] - 4 * x * gR[4] - 2 * w * gR[5] + 2 * z * gR[6] + 2 * w * gR[7] - 4 * x * gR[8];
        gn[2] = -4 * y * gR[0] + 2 * x * gR[1] + 2 * w * gR[2] + 2 * x * gR[3] + 2 * z * gR[5] - 2 * w * gR[6] + 2 * z * gR[7] - 4 * y * gR[8];
        gn[3] = -4 * z * gR[0] - 2 * w * gR[1] + 2 * x * gR[2] + 2 * w * gR[3] - 4 * z * gR[4] + 2 * y * gR[5] + 2 * x * gR[6] + 2 * y * gR[7];
        const double q0[4] = {qw0, qx0, qy0, qz0};
        const double dot = q0[0] * gn[0] + q0[1] * gn[1] + q0[2] * gn[2] + q0[3] * gn[3];
        for (int k = 0; k < 4; ++k) d_quat[i * 4 + k] = gn[k] / nq - q0[k] * dot / (nq * nq * nq);
        /* projection and Jacobian backward, camera-frame z, then xyz = W^T g */
        double Jv[6], gp[3];
        dt_jacobian_vjp_f64(p, K[0], K[4], kc, gJ, g_uv + i * 2, Jv, gp);
        gp[2] += g_z[i];
        for (int k = 0; k < 3; ++k) d_xyz[i * 3 + k] = W[k] * gp[0] + W[3 + k] * gp[1] + W[6 + k] * gp[2];
        const double sg = 1.0 / (1.0 + exp(-opa_logit[i]));
        d_opa[i] = g_opa[i] * sg * (1.0 - sg);
        if (sh_present && n_sh > 1) {
            double d[3], Y[16];
            view_dir_f64(xyz + i * 3, cam_centre, d);
            sh_basis_f64(n_sh, d[0], d[1], d[2], Y);
            for (int c = 0; c < 3; ++c) {
                const double gc = g_rgb[i * 3 + c] * RSH0F;
                d_dc[i * 3 + c] = gc * Y[0];
                for (int k = 1; k < n_sh; ++k) d_sh[((size_t)i * 3 + c) * nr + (k - 1)] = gc * Y[k];
            }
        } else {
            for (int c = 0; c < 3; ++c) d_dc[i * 3 + c] = g_rgb[i * 3 + c];
        }
    }
}
