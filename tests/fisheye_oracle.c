/* fisheye_oracle.c — CPU oracle of the fisheye per-gaussian stage (rasterize(..., fisheye=k)) and its VJP, fp64.
 *
 * TEST INFRASTRUCTURE ONLY (tests/fisheye_oracle.py).  Compiled together with oracle/gsr_oracle.c, whose helpers
 * (transform_point, sigma_world, conic, mmd, sh_basis, view_dir) it reuses unchanged.
 *
 * COLMAP's OPENCV_FISHEYE model: rho = |(x, y)|, R = |p|, theta = atan2(rho, z), t = theta^2,
 *   g = theta P(t), P = 1 + k1 t + k2 t^2 + k3 t^3 + k4 t^4, s = g / rho, u = fx s x + cx, v = fy s y + cy.
 * Every derivative of s is a function of theta over a power of R (polar coordinates rho = R sin, z = R cos):
 *   s = h / R, h = g / sin;   q = (ds/drho) / rho = m / R^3, m = (g' sin cos - g) / sin^3;   d = ds/dz = -g' / R^2
 *   q' = (dq/drho) / rho = (m' cot - 3 m) / R^5;   e = dq/dz = -(m' sin + 3 m cos) / R^4;
 *   dz = dd/dz = (g'' sin + 2 g' cos) / R^3.
 * h, m and m' / theta are 0/0 at theta = 0; below theta^2 = 1e-4 their Taylor series in t replace them (five terms
 * here, truncation t^5).
 *
 *   fe_terms_f64             s, q, d, q', e, dz and theta at one camera-frame point
 *   fe_jacobian_vjp_f64      J at p, and g = J^T g_uv + sum_ij gJ_ij dJ_ij / dp
 *   fe_project_f64           orc_project with the fisheye projection, Jacobian and the theta cull
 *   fe_project_backward_f64  orc_project_backward with the fisheye Jacobian and the camera-frame z gradient
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mfma -shared -fPIC -I<repo>/oracle fisheye_oracle.c -lm
 */
#include "gsr_oracle.c"

/* out: s q d q' e dz theta */
void fe_terms_f64(const double* p, const double* k, double* out) {
    const double x = p[0], y = p[1], z = p[2];
    const double k1 = k[0], k2 = k[1], k3 = k[2], k4 = k[3];
    const double r2 = x * x + y * y, rho = sqrt(r2), R2 = r2 + z * z, R = sqrt(R2);
    const double th = atan2(rho, z), t = th * th;
    const double P = 1 + t * (k1 + t * (k2 + t * (k3 + t * k4)));
    const double G1 = 1 + t * (3 * k1 + t * (5 * k2 + t * (7 * k3 + t * 9 * k4)));
    const double G2 = 6 * k1 + t * (20 * k2 + t * (42 * k3 + t * 72 * k4)); /* g'' / theta */
    const double sn = rho / R, cs = z / R;
    double h, m, mc, ms;
    if (t < 1e-4) {
        const double h_[5] = {1, k1 + 1.0 / 6, k1 / 6 + k2 + 7.0 / 360, (294 * k1 + 2520 * k2 + 15120 * k3 + 31) / 15120,
                              (1240 * k1 + 11760 * k2 + 100800 * k3 + 604800 * k4 + 127) / 604800};
        const double m_[5] = {2 * k1 - 2.0 / 3, -(5 * k1 - 20 * k2 + 1) / 5, -(133 * k1 + 560 * k2 - 2520 * k3 + 17) / 420,
                              -(2305 * k1 + 16380 * k2 + 63000 * k3 - 302400 * k4 + 261) / 37800,
                              -(32747 * k1 + 271040 * k2 + 1829520 * k3 + 6652800 * k4 + 3543) / 3326400};
        h = m = 0;
        double n = 0;
        for (int i = 4; i >= 0; --i) {
            h = h * t + h_[i];
            m = m * t + m_[i];
            if (i >= 1) n = n * t + 2 * i * m_[i];
        }
        /* theta cot theta = 1 - t/3 - t^2/45 - 2 t^3/945 */
        mc = n * (1 - t * (1.0 / 3 + t * (1.0 / 45 + t * 2.0 / 945)));
        ms = n * th * sn;
    } else {
        const double g = th * P;
        h = g / sn;
        const double num = G1 * sn * cs - g;
        m = num / (sn * sn * sn);
        const double mp = (th * G2 * sn * sn * cs - 2 * G1 * sn * sn * sn - 3 * cs * num) / (sn * sn * sn * sn);
        mc = mp * cs / sn;
        ms = mp * sn;
    }
    out[0] = h / R;
    out[1] = m / (R2 * R);
    out[2] = -G1 / R2;
    out[3] = (mc - 3 * m) / (R2 * R2 * R);
    out[4] = -(ms + 3 * m * cs) / (R2 * R2);
    out[5] = (th * G2 * sn + 2 * G1 * cs) / (R2 * R);
    out[6] = th;
}

static void fe_jacobian(const double* p, double fx, double fy, const double* k, double* J, double* f) {
    fe_terms_f64(p, k, f);
    const double x = p[0], y = p[1], s = f[0], q = f[1], d = f[2];
    J[0] = fx * (s + x * x * q); J[1] = fx * x * y * q; J[2] = fx * x * d;
    J[3] = fy * x * y * q;       J[4] = fy * (s + y * y * q); J[5] = fy * y * d;
}

/* J [6], g [3] = J^T g_uv + contraction of dJ/dp with gJ */
void fe_jacobian_vjp_f64(const double* p, double fx, double fy, const double* k, const double* gJ, const double* guv,
                         double* J, double* g) {
    double f[7];
    fe_jacobian(p, fx, fy, k, J, f);
    const double x = p[0], y = p[1], q = f[1], d = f[2], qp = f[3], e = f[4], dz = f[5];
    /* dJ_ij / dp_k, row-major [6][3] */
    const double H[6][3] = {
        {fx * (3 * x * q + x * x * x * qp), fx * (y * q + x * x * y * qp), fx * (d + x * x * e)},
        {fx * (y * q + x * x * y * qp), fx * (x * q + x * y * y * qp), fx * x * y * e},
        {fx * (d + x * x * e), fx * x * y * e, fx * x * dz},
        {fy * (y * q + x * x * y * qp), fy * (x * q + x * y * y * qp), fy * x * y * e},
        {fy * (x * q + x * y * y * qp), fy * (3 * y * q + y * y * y * qp), fy * (d + y * y * e)},
        {fy * x * y * e, fy * (d + y * y * e), fy * y * dz}};
    for (int c = 0; c < 3; ++c) {
        double a = J[c] * guv[0] + J[3 + c] * guv[1];
        for (int r = 0; r < 6; ++r) a += gJ[r] * H[r][c];
        g[c] = a;
    }
}

/* kc: k1 k2 k3 k4 theta_max.  theta_out [N] */
void fe_project_f64(int N, int n_sh, const double* xyz, const double* quat, const double* scale,
                    const double* opa_logit, const double* rgb_dc, const double* sh, const double* T, const double* K,
                    const double* cam_centre, const double* kc, double width, double height, double near_t,
                    double far_t, double pad, double* xyz_cam, double* uv, double* conic, double* opa,
                    double* rgb_out, unsigned char* visible, double* theta_out) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < N; ++i) {
        double p[3];
        transform_point_f64(T, xyz[i * 3], xyz[i * 3 + 1], xyz[i * 3 + 2], p);
        double f[7];
        fe_terms_f64(p, kc, f);
        const double u = K[0] * f[0] * p[0] + K[2], v = K[4] * f[0] * p[1] + K[5];
        for (int k = 0; k < 3; ++k) xyz_cam[i * 3 + k] = p[k];
        uv[i * 2] = u; uv[i * 2 + 1] = v;
        theta_out[i] = f[6];
        const int culled = (p[2] < near_t) || (p[2] > far_t) || (u < -pad) || (u > width + pad) || (v < -pad) ||
                           (v > height + pad) || (f[6] >= kc[4]) || u != u || v != v;
        visible[i] = culled ? 0 : 1;
        if (culled) continue;
        double S[9], J[6];
        sigma_world_f64(quat + i * 4, scale + i * 3, S);
        fe_jacobian(p, K[0], K[4], kc, J, f);
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
void fe_project_backward_f64(int N, int n_sh, const double* xyz, const double* quat, const double* scale,
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
        double p[3], S[9], J[6], f[7], W[9];
        transform_point_f64(T, xyz[i * 3], xyz[i * 3 + 1], xyz[i * 3 + 2], p);
        sigma_world_f64(quat + i * 4, scale + i * 3, S);
        fe_jacobian(p, K[0], K[4], kc, J, f);
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
        fe_jacobian_vjp_f64(p, K[0], K[4], kc, gJ, g_uv + i * 2, Jv, gp);
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
