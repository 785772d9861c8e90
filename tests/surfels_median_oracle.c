/* surfels_median_oracle.c — fp64 oracle of rasterize_surfels(..., median_depth=True) (DESIGN.md 3.28): every pixel's
 * ray against every visible surfel in depth order, with no tiles, and the analytic backward of <G, median>.  TEST
 * INFRASTRUCTURE (tests/surfels_median_oracle.py builds and wraps it).  The surfel set-up, the rays and the intersection
 * are tests/surfels_lens_oracle.c's; zero OPENCV coefficients give the pinhole (rows are then d loss / d M', which the
 * wrapper maps to the pinhole's d loss / d (K M')).
 *
 *   surfel_median_oracle(lens, kc, N, xyz, quat, scale, opl, T, K, H, W, near, far, pad, mh, G_median,
 *                        median, median_id, flag, visible, rows, mass, g_xyz, g_quat, g_scale, g_opl, sort_z, rays)
 *
 * median [H,W], median_id [H,W] (int32, -1 where no surfel contributes); flag [H,W]: the pixel's median may differ in
 * fp32 — a deciding 1 - A within 1e-4 of 0.5, or a surfel the walk meets (the selected one among them) near one of its
 * own thresholds (intersect's near), which fp32 may take the other way.
 * G_median [H,W] (NULL: forward only); rows [N,20] the median loss's gradient rows (only dM' and d p_z), mass [N,20]
 * the same sums of the magnitudes of every term (tests/gradrows.py); g_* the parameter gradients (opacity: exactly 0). */
#include "surfels_lens_oracle.c"

int surfel_median_oracle(int lens, const double* kc, int N, const double* xyz, const double* quat,
                         const double* scale, const double* opl, const double* T, const double* K, int H, int W,
                         double near_t, double far_t, double pad, double mh, const double* G_med, double* median,
                         int* median_id, unsigned char* flag, unsigned char* visible, double* rows, double* mass,
                         double* g_xyz, double* g_quat, double* g_scale, double* g_opl, const double* sort_z,
                         double* rays) {
    g_lens = lens;
    g_kc = kc;
    for (int py = 0; py < H; ++py)
        for (int px = 0; px < W; ++px)
            lens_ray((px - K[2]) / K[0], (py - K[5]) / K[4], rays + ((size_t)py * W + px) * 3);
    Surfel* S = (Surfel*)calloc((size_t)N + 1, sizeof(Surfel));
    int* order = (int*)malloc(sizeof(int) * ((size_t)N + 1));
    double* zs = (double*)malloc(sizeof(double) * ((size_t)N + 1));
    int M = 0;
    for (int i = 0; i < N; ++i) {
        setup(&S[i], xyz + 3 * i, quat + 4 * i, scale + 3 * i, opl[i], T, K, H, W, near_t, far_t, pad, mh);
        visible[i] = (unsigned char)S[i].vis;
        if (S[i].vis) order[M++] = i;
        zs[i] = sort_z != NULL ? sort_z[i] : S[i].p[2];
    }
    g_sort_z = zs;
    qsort(order, (size_t)M, sizeof(int), by_depth);
    const double r2 = mh * mh;
    const int bwd = G_med != NULL;
    if (bwd) {
        memset(rows, 0, sizeof(double) * (size_t)N * SG);
        memset(mass, 0, sizeof(double) * (size_t)N * SG);
    }
    for (int py = 0; py < H; ++py)
        for (int px = 0; px < W; ++px) {
            const size_t pix = (size_t)py * W + px;
            const double* dr = rays + pix * 3;
            double A = 0, med = 0;
            int mid = -1, fl = 0;
            Hit h, hm;
            for (int k = 0; k < M; ++k) {
                const Surfel* s = &S[order[k]];
                if (!intersect(s, px, py, dr, r2, &h, &fl)) continue;
                /* 1 - A > 0.5 in front of this contributor: the median so far */
                med = h.z;
                mid = order[k];
                hm = h;
                A += h.alpha * (1 - A);
                fl |= fabs((1 - A) - 0.5) <= 1e-4;
                if (!(1 - A > 0.5)) break;
            }
            median[pix] = med;
            median_id[pix] = mid;
            flag[pix] = (unsigned char)fl;
            if (!bwd || mid < 0 || G_med[pix] == 0) continue;
            /* z = M'2 . (a, b, 1) where rho3 is used (through (a, b) = (c0, c1) / c2, c = hx x hy), else p_z */
            const double gz = G_med[pix], gzA = fabs(gz);
            const Surfel* s = &S[mid];
            double g[SG], gA[SG];
            memset(g, 0, sizeof(g));
            memset(gA, 0, sizeof(gA));
            if (hm.use3) {
                const double ga = gz * s->M[6], gb = gz * s->M[7];
                const double gaP = gzA * fabs(s->M[6]), gbP = gzA * fabs(s->M[7]);
                g[6] = gz * hm.a;
                g[7] = gz * hm.b;
                g[8] = gz;
                gA[6] = gzA * fabs(hm.a);
                gA[7] = gzA * fabs(hm.b);
                gA[8] = gzA;
                const double gc[3] = {ga / hm.c2, gb / hm.c2, -(ga * hm.a + gb * hm.b) / hm.c2};
                const double ic = 1 / fabs(hm.c2);
                const double gcA[3] = {gaP * ic, gbP * ic, (gaP * fabs(hm.a) + gbP * fabs(hm.b)) * ic};
                const double* X = hm.hx;
                const double* Y = hm.hy;
                const double ghx[3] = {Y[1] * gc[2] - Y[2] * gc[1], Y[2] * gc[0] - Y[0] * gc[2],
                                       Y[0] * gc[1] - Y[1] * gc[0]};
                const double ghy[3] = {gc[1] * X[2] - gc[2] * X[1], gc[2] * X[0] - gc[0] * X[2],
                                       gc[0] * X[1] - gc[1] * X[0]};
                const double ghxA[3] = {fabs(Y[1]) * gcA[2] + fabs(Y[2]) * gcA[1],
                                        fabs(Y[2]) * gcA[0] + fabs(Y[0]) * gcA[2],
                                        fabs(Y[0]) * gcA[1] + fabs(Y[1]) * gcA[0]};
                const double ghyA[3] = {gcA[1] * fabs(X[2]) + gcA[2] * fabs(X[1]),
                                        gcA[2] * fabs(X[0]) + gcA[0] * fabs(X[2]),
                                        gcA[0] * fabs(X[1]) + gcA[1] * fabs(X[0])};
                for (int k = 0; k < 3; ++k) {
                    g[k] = -dr[2] * ghx[k];
                    g[3 + k] = -dr[2] * ghy[k];
                    g[6 + k] += dr[0] * ghx[k] + dr[1] * ghy[k];
                    gA[k] = fabs(dr[2]) * ghxA[k];
                    gA[3 + k] = fabs(dr[2]) * ghyA[k];
                    gA[6 + k] += fabs(dr[0]) * ghxA[k] + fabs(dr[1]) * ghyA[k];
                }
            } else {
                g[18] = gz;
                gA[18] = gzA;
            }
            for (int k = 0; k < SG; ++k) {
                rows[(size_t)mid * SG + k] += g[k];
                mass[(size_t)mid * SG + k] += gA[k];
            }
        }
    if (bwd) {
        for (int i = 0; i < N; ++i) {
            double* gx = g_xyz + 3 * i;
            double* gq = g_quat + 4 * i;
            double* gs = g_scale + 3 * i;
            memset(gx, 0, 3 * sizeof(double));
            memset(gq, 0, 4 * sizeof(double));
            memset(gs, 0, 3 * sizeof(double));
            g_opl[i] = 0;
            const Surfel* s = &S[i];
            if (!s->vis) continue;
            /* M' = [s_u Rc0 | s_v Rc1 | p]: columns j of the rows are d loss / d X_j */
            const double* g = rows + (size_t)i * SG;
            double gX[3][3];
            for (int j = 0; j < 3; ++j) {
                gX[j][0] = g[j];
                gX[j][1] = g[3 + j];
                gX[j][2] = g[6 + j];
            }
            const double gp[3] = {gX[2][0], gX[2][1], gX[2][2] + g[18]};
            double gRc[9];
            for (int r = 0; r < 3; ++r) {
                gRc[r * 3] = s->su * gX[0][r];
                gRc[r * 3 + 1] = s->sv * gX[1][r];
                gRc[r * 3 + 2] = 0;
            }
            gs[0] = (gX[0][0] * s->Rc[0] + gX[0][1] * s->Rc[3] + gX[0][2] * s->Rc[6]) * s->su;
            gs[1] = (gX[1][0] * s->Rc[1] + gX[1][1] * s->Rc[4] + gX[1][2] * s->Rc[7]) * s->sv;
            double gR[9];
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c)
                    gR[r * 3 + c] = T[r] * gRc[c] + T[4 + r] * gRc[3 + c] + T[8 + r] * gRc[6 + c];
            for (int k = 0; k < 3; ++k) gx[k] = T[k] * gp[0] + T[4 + k] * gp[1] + T[8 + k] * gp[2];
            double q[4] = {quat[4 * i], quat[4 * i + 1], quat[4 * i + 2], quat[4 * i + 3]}, R[9], qn[4];
            quat_rot(q, R, qn);
            const double w = qn[0], a = qn[1], b = qn[2], c = qn[3];
            double gn[4];
            gn[0] = -2 * c * gR[1] + 2 * b * gR[2] + 2 * c * gR[3] - 2 * a * gR[5] - 2 * b * gR[6] + 2 * a * gR[7];
            gn[1] = 2 * b * gR[1] + 2 * c * gR[2] + 2 * b * gR[3] - 4 * a * gR[4] - 2 * w * gR[5] + 2 * c * gR[6] +
                    2 * w * gR[7] - 4 * a * gR[8];
            gn[2] = -4 * b * gR[0] + 2 * a * gR[1] + 2 * w * gR[2] + 2 * a * gR[3] + 2 * c * gR[5] - 2 * w * gR[6] +
                    2 * c * gR[7] - 4 * b * gR[8];
            gn[3] = -4 * c * gR[0] - 2 * w * gR[1] + 2 * a * gR[2] + 2 * w * gR[3] - 4 * c * gR[4] + 2 * b * gR[5] +
                    2 * a * gR[6] + 2 * b * gR[7];
            const double nq = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
            const double dot = qn[0] * gn[0] + qn[1] * gn[1] + qn[2] * gn[2] + qn[3] * gn[3];
            for (int k = 0; k < 4; ++k) gq[k] = (gn[k] - qn[k] * dot) / nq;
        }
    }
    free(S);
    free(order);
    free(zs);
    return M;
}
