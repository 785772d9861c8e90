/* surfels_lens_oracle.c — fp64 oracle of rasterize_surfels(..., fisheye=k / distortion=k) (DESIGN.md 3.26): every
 * pixel's ray (the lens inverted by bisection, then Newton for the tangential terms) against every visible surfel in
 * depth order, with no tiles, and the analytic backward.  TEST INFRASTRUCTURE (tests/surfels_lens_oracle.py builds and
 * wraps it).  All inputs are fp64; the lens constants kc are {k1..k4, theta_max} (lens 1) or {k1, k2, p1, p2, k3,
 * r2_max} (lens 2), the limits as the kernels cull with them.  The colour is an input, so its view direction is a
 * constant.
 *
 *   surfel_lens_oracle(lens, kc, N, xyz, quat, scale, opl, colour, T, K, H, W, near, far, pad, mh, bg,
 *                 G_image, G_depth, G_alpha, G_normal, G_dist,          (all NULL: forward only)
 *                 image, depth, alpha, normal, dist, visible, uv,        [H,W,k], [N], [N,2]
 *                 g_xyz, g_quat, g_scale, g_opl, g_colour, rows, uv_grad, mass, near, sort_z)
 *
 *                 ..., rays)                                              rays [H,W,3] out: the oracle's rays
 *
 * rows [N,20]: the render-stage gradient row of every surfel (gsr_surfels_lens.h: dL/dM'), uv_grad [N,2] its uv.grad
 * (J_n^-T g_n + g_c); mass [N,20]
 * (may be NULL) the same sums formed from the magnitudes of every part of every term (tests/gradrows.py's mass);
 * near [H,W] (may be NULL) the pixels where a branch of the blend lies within 1e-4 of its threshold (or the
 * accumulated alpha within 2e-6 of 0.9999 or 1e-5 of 0.999), which fp32 can take the other way; sort_z [N] (may be
 * NULL) the depth the blend order sorts by (ties by index), p_z in fp64 when NULL. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define SG 20

static int g_lens;
static const double* g_kc;

static double fe_td(double th) {
    const double t = th * th;
    return th * (1 + t * (g_kc[0] + t * (g_kc[1] + t * (g_kc[2] + t * g_kc[3]))));
}

static void dt_fwd(double a, double b, double* ad, double* bd) {
    const double k1 = g_kc[0], k2 = g_kc[1], p1 = g_kc[2], p2 = g_kc[3], k3 = g_kc[4];
    const double s = a * a + b * b, R = 1 + s * (k1 + s * (k2 + s * k3));
    *ad = a * R + 2 * p1 * a * b + p2 * (s + 2 * a * a);
    *bd = b * R + p1 * (s + 2 * b * b) + 2 * p2 * a * b;
}

/* the lens projection of p in normalised distorted coordinates, and the fold test (1: beyond the limit) */
static int lens_norm(const double* p, double* xd, double* yd) {
    if (g_lens == 1) {
        const double rho = sqrt(p[0] * p[0] + p[1] * p[1]), th = atan2(rho, p[2]);
        const double s = rho > 0 ? fe_td(th) / rho : 1 / p[2];
        *xd = s * p[0];
        *yd = s * p[1];
        return th >= g_kc[4];
    }
    const double a = p[0] / p[2], b = p[1] / p[2];
    dt_fwd(a, b, xd, yd);
    return a * a + b * b >= g_kc[5];
}

/* J = d(u, v) / dp by Richardson-extrapolated central differences (fp64, relative error ~1e-12) */
static void lens_jac(const double* p, double fx, double fy, double* J) {
    for (int k = 0; k < 3; ++k) {
        double col[2] = {0, 0};
        const double h0 = 1e-4 * (fabs(p[k]) + fabs(p[2]));
        double D[2][2];
        for (int lvl = 0; lvl < 2; ++lvl) {
            const double h = lvl ? h0 / 2 : h0;
            double q[3] = {p[0], p[1], p[2]}, a0, b0, a1, b1;
            q[k] = p[k] + h;
            lens_norm(q, &a0, &b0);
            q[k] = p[k] - h;
            lens_norm(q, &a1, &b1);
            D[lvl][0] = (a0 - a1) / (2 * h);
            D[lvl][1] = (b0 - b1) / (2 * h);
        }
        for (int r = 0; r < 2; ++r) col[r] = (4 * D[1][r] - D[0][r]) / 3;
        J[k] = fx * col[0];
        J[3 + k] = fy * col[1];
    }
}

/* the ray of the distorted normalised point (xd, yd): 0 when it has no preimage on the monotone branch */
static void lens_ray(double xd, double yd, double* d) {
    d[0] = d[1] = d[2] = 0;
    const double rd = sqrt(xd * xd + yd * yd);
    if (g_lens == 1) {
        const double thmax = g_kc[4];
        if (!(rd < fe_td(thmax))) return;
        if (rd == 0) { d[2] = 1; return; }
        double lo = 0, hi = thmax;
        for (int it = 0; it < 200; ++it) {
            const double m = 0.5 * (lo + hi);
            if (fe_td(m) > rd) hi = m; else lo = m;
        }
        const double th = 0.5 * (lo + hi);
        d[0] = sin(th) * xd / rd;
        d[1] = sin(th) * yd / rd;
        d[2] = cos(th);
        return;
    }
    const double r2max = g_kc[5];
    double a = xd, b = yd;
    if (rd > 0) {
        double lo = 0, hi = isfinite(r2max) ? sqrt(r2max) : 1;
        while (!isfinite(r2max) && hi < 1e6 && hi * (1 + hi * hi * (g_kc[0] + hi * hi * (g_kc[1] + hi * hi * g_kc[4]))) < rd)
            hi *= 2;
        for (int it = 0; it < 200; ++it) {
            const double m = 0.5 * (lo + hi);
            const double sm = m * m;  /* the radial part alone, m R(m^2), increasing below r2_max */
            if (m * (1 + sm * (g_kc[0] + sm * (g_kc[1] + sm * g_kc[4]))) > rd) hi = m; else lo = m;
        }
        const double r = 0.5 * (lo + hi);
        a = xd * r / rd;
        b = yd * r / rd;
    }
    for (int it = 0; it < 100; ++it) {
        double ad, bd, a1, b1, a2, b2;
        dt_fwd(a, b, &ad, &bd);
        const double h = 1e-7;
        dt_fwd(a + h, b, &a1, &b1);
        dt_fwd(a - h, b, &a2, &b2);
        const double J00 = (a1 - a2) / (2 * h), J10 = (b1 - b2) / (2 * h);
        dt_fwd(a, b + h, &a1, &b1);
        dt_fwd(a, b - h, &a2, &b2);
        const double J01 = (a1 - a2) / (2 * h), J11 = (b1 - b2) / (2 * h);
        const double det = J00 * J11 - J01 * J10, ex = ad - xd, ey = bd - yd;
        if (det == 0) return;
        a -= (J11 * ex - J01 * ey) / det;
        b -= (J00 * ey - J10 * ex) / det;
    }
    double ad, bd;
    dt_fwd(a, b, &ad, &bd);
    if (!(fabs(ad - xd) + fabs(bd - yd) <= 1e-12 * (1 + rd)) || !(a * a + b * b < r2max)) return;
    const double n = sqrt(a * a + b * b + 1);
    d[0] = a / n;
    d[1] = b / n;
    d[2] = 1 / n;
}

typedef struct {
    double p[3], R[9], Rc[9], su, sv, M[9], u, v, opa, n[3], sgn;
    int vis;
} Surfel;

static void quat_rot(const double* q0, double* R, double* qn) {
    const double nq = sqrt(q0[0] * q0[0] + q0[1] * q0[1] + q0[2] * q0[2] + q0[3] * q0[3]);
    const double w = q0[0] / nq, x = q0[1] / nq, y = q0[2] / nq, z = q0[3] / nq;
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w); R[2] = 2 * (x * z + y * w);
    R[3] = 2 * (x * y + z * w); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
    R[6] = 2 * (x * z - y * w); R[7] = 2 * (y * z + x * w); R[8] = 1 - 2 * (x * x + y * y);
    qn[0] = w; qn[1] = x; qn[2] = y; qn[3] = z;
}

static void setup(Surfel* s, const double* xyz, const double* quat, const double* scale, double opl, const double* T,
                  const double* K, int H, int W, double near_t, double far_t, double pad, double mh) {
    double q[4] = {quat[0], quat[1], quat[2], quat[3]}, qn[4];
    for (int r = 0; r < 3; ++r)
        s->p[r] = T[r * 4] * xyz[0] + T[r * 4 + 1] * xyz[1] + T[r * 4 + 2] * xyz[2] + T[r * 4 + 3];
    quat_rot(q, s->R, qn);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
            s->Rc[r * 3 + c] = T[r * 4] * s->R[c] + T[r * 4 + 1] * s->R[3 + c] + T[r * 4 + 2] * s->R[6 + c];
    s->su = exp(scale[0]);
    s->sv = exp(scale[1]);
    const double fx = K[0], cx = K[2], fy = K[4], cy = K[5];
    const double Tu[3] = {s->su * s->Rc[0], s->su * s->Rc[3], s->su * s->Rc[6]};
    const double Tv[3] = {s->sv * s->Rc[1], s->sv * s->Rc[4], s->sv * s->Rc[7]};
    const double* p = s->p;
    double* M = s->M;
    M[0] = Tu[0]; M[1] = Tv[0]; M[2] = p[0];
    M[3] = Tu[1]; M[4] = Tv[1]; M[5] = p[1];
    M[6] = Tu[2]; M[7] = Tv[2]; M[8] = p[2];
    double xd, yd;
    const int fold = lens_norm(p, &xd, &yd);
    s->u = fx * xd + cx;
    s->v = fy * yd + cy;
    const double r2 = mh * mh;
    const int culled = p[2] < near_t || p[2] > far_t || s->u < -pad || s->u > W + pad || s->v < -pad || s->v > H + pad ||
                       fold;
    const int front = p[2] > 0 && r2 * (M[6] * M[6] + M[7] * M[7]) < p[2] * p[2];
    s->vis = !culled && front;
    s->opa = 1.0 / (1.0 + exp(-opl));
    s->sgn = (s->Rc[2] * p[0] + s->Rc[5] * p[1] + s->Rc[8] * p[2] > 0) ? -1.0 : 1.0;
    for (int r = 0; r < 3; ++r) s->n[r] = s->sgn * s->Rc[r * 3 + 2];
}

typedef struct {
    double hx[3], hy[3], c2, a, b, dx, dy, G, alpha, z;
    int use3, clamped;
} Hit;

/* near (may be NULL): set when a branch of this (pixel, surfel) lies within a relative 1e-4 of its threshold (rho at
 * r^2, the min switch, alpha at 1/255 or at the 0.99 clamp), where fp32 may decide the other way */
static int intersect(const Surfel* s, double x, double y, const double* d, double r2, Hit* h, int* near) {
    const double* M = s->M;
    for (int k = 0; k < 3; ++k) {
        h->hx[k] = d[0] * M[6 + k] - d[2] * M[k];
        h->hy[k] = d[1] * M[6 + k] - d[2] * M[3 + k];
    }
    const double c0 = h->hx[1] * h->hy[2] - h->hx[2] * h->hy[1];
    const double c1 = h->hx[2] * h->hy[0] - h->hx[0] * h->hy[2];
    h->c2 = h->hx[0] * h->hy[1] - h->hx[1] * h->hy[0];
    if (h->c2 == 0) return 0;
    h->a = c0 / h->c2;
    h->b = c1 / h->c2;
    const double rho3 = h->a * h->a + h->b * h->b;
    h->dx = x - s->u;
    h->dy = y - s->v;
    const double rho2 = 2 * (h->dx * h->dx + h->dy * h->dy);
    h->use3 = rho3 <= rho2;
    const double rho = h->use3 ? rho3 : rho2;
    if (near != NULL) {
        /* only branches with a jump: the cutoff where alpha there reaches 1/255, the 1/255 skip, the depth's switch
         * between the intersection and p_z where the surfel contributes, and the clamp (in the gradient) */
        const double ar = s->opa * exp(-0.5 * rho);
        *near |= (fabs(rho - r2) <= 1e-4 * r2 && s->opa * exp(-0.5 * r2) >= 1.0 / 255.0 * (1 - 1e-4)) ||
                 (rho <= r2 && fabs(ar - 1.0 / 255.0) <= 1e-4 / 255.0) ||
                 (rho <= r2 && ar >= 1.0 / 255.0 && (fabs(rho3 - rho2) <= 1e-4 * fmax(rho3, rho2) ||
                                                     fabs(ar - 0.99) <= 1e-4));
    }
    if (!(rho <= r2)) return 0;
    h->G = exp(-0.5 * rho);
    h->clamped = s->opa * h->G >= 0.99;
    h->alpha = h->clamped ? 0.99 : s->opa * h->G;
    if (h->alpha < 1.0 / 255.0) return 0;
    h->z = h->use3 ? M[6] * h->a + M[7] * h->b + M[8] : s->p[2];
    return 1;
}

/* ill (NULL unless surfel_lens_oracle_ill set it; [H,W], zeroed by the caller): the pixels where a contributing surfel's
 * ray-plane intersection is ill-conditioned, |c2| < |hx| |hy| / ILL_KAPPA with a = c0 / c2, b = c1 / c2.  The gradient
 * of (a, b) carries 1 / c2^2: an input rounded to fp32 (eps = 6e-8) moves that pixel's gradient terms by about
 * eps kappa^2 of themselves, 2.4e-4 at kappa = 64.  Such pixels are nearly edge-on surfels whose intersection branch
 * is taken. */
#define ILL_KAPPA 64.0
static unsigned char* g_ill;
void surfel_lens_oracle_ill(unsigned char* ill) { g_ill = ill; }

static int ill_conditioned(const Hit* h) {
    const double nx = sqrt(h->hx[0] * h->hx[0] + h->hx[1] * h->hx[1] + h->hx[2] * h->hx[2]);
    const double ny = sqrt(h->hy[0] * h->hy[0] + h->hy[1] * h->hy[1] + h->hy[2] * h->hy[2]);
    return h->use3 && fabs(h->c2) * ILL_KAPPA < nx * ny;
}

static const double* g_sort_z;
static int by_depth(const void* pa, const void* pb) {
    const int a = *(const int*)pa, b = *(const int*)pb;
    const double za = g_sort_z[a], zb = g_sort_z[b];
    return za < zb ? -1 : za > zb ? 1 : (a < b ? -1 : a > b);
}

int surfel_lens_oracle(int lens, const double* kc, int N, const double* xyz, const double* quat, const double* scale, const double* opl,
                  const double* colour, const double* T, const double* K, int H, int W, double near_t, double far_t,
                  double pad, double mh, const double* bg, const double* G_img, const double* G_dep,
                  const double* G_alp, const double* G_nrm, const double* G_dis, double* image, double* depth,
                  double* alpha, double* normal, double* dist, unsigned char* visible, double* uv, double* g_xyz,
                  double* g_quat, double* g_scale, double* g_opl, double* g_col, double* rows, double* uv_grad,
                  double* mass, unsigned char* near, const double* sort_z, double* rays) {
    g_lens = lens;
    g_kc = kc;
    for (int py = 0; py < H; ++py)
        for (int px = 0; px < W; ++px)
            lens_ray((px - K[2]) / K[0], (py - K[5]) / K[4], rays + ((size_t)py * W + px) * 3);
    Surfel* S = (Surfel*)calloc((size_t)N + 1, sizeof(Surfel));
    int* order = (int*)malloc(sizeof(int) * ((size_t)N + 1));
    int M = 0;
    for (int i = 0; i < N; ++i) {
        setup(&S[i], xyz + 3 * i, quat + 4 * i, scale + 3 * i, opl[i], T, K, H, W, near_t, far_t, pad, mh);
        visible[i] = (unsigned char)S[i].vis;
        uv[2 * i] = S[i].u;
        uv[2 * i + 1] = S[i].v;
        if (S[i].vis) order[M++] = i;
    }
    double* zs = (double*)malloc(sizeof(double) * ((size_t)N + 1));
    for (int i = 0; i < N; ++i) zs[i] = sort_z != NULL ? sort_z[i] : S[i].p[2];
    g_sort_z = zs;
    qsort(order, (size_t)M, sizeof(int), by_depth);
    const double r2 = mh * mh;
    const double ms = isfinite(far_t) ? far_t / (far_t - near_t) : 1.0;
    const int bwd = G_img != NULL;
    if (bwd) memset(rows, 0, sizeof(double) * (size_t)N * SG);
    if (bwd && mass != NULL) memset(mass, 0, sizeof(double) * (size_t)N * SG);
#pragma omp parallel
    {
    int* hit_j = (int*)malloc(sizeof(int) * ((size_t)M + 1));
#pragma omp for schedule(dynamic, 1)
    for (int py = 0; py < H; ++py)
        for (int px = 0; px < W; ++px) {
            const size_t pix = (size_t)py * W + px;
            const double x = px, y = py;
            const double* dr = rays + pix * 3;
            double A = 0, img[3] = {0, 0, 0}, dep = 0, nrm[3] = {0, 0, 0}, wm = 0, wm2 = 0, ds = 0;
            int nh = 0, nr = 0;
            Hit h;
            for (int k = 0; k < M; ++k) {
                nr |= fabs(A - 0.9999) <= 2e-6;
                if (A > 0.9999) break;
                const Surfel* s = &S[order[k]];
                if (!intersect(s, x, y, dr, r2, &h, &nr)) continue;
                if (g_ill != NULL && ill_conditioned(&h)) g_ill[pix] = 1;
                const double w = h.alpha * (1 - A);
                for (int c = 0; c < 3; ++c) {
                    img[c] += w * colour[3 * order[k] + c];
                    nrm[c] += w * s->n[c];
                }
                dep += w * h.z;
                const double m = ms * (1 - near_t / h.z);
                ds += w * (m * m * A - 2 * m * wm + wm2);
                wm += w * m;
                wm2 += w * m * m;
                A += w;
                hit_j[nh++] = k;
            }
            const int with_bg = A < 0.999;
            if (near != NULL) near[pix] = (unsigned char)(nr || fabs(A - 0.999) <= 1e-5);
            for (int c = 0; c < 3; ++c) {
                image[pix * 3 + c] = img[c] + (with_bg ? bg[c] * (1 - A) : 0);
                normal[pix * 3 + c] = nrm[c];
            }
            depth[pix] = dep;
            alpha[pix] = A;
            dist[pix] = ds;
            if (!bwd) continue;
            const double* Gi = G_img + pix * 3;
            const double* Gn = G_nrm + pix * 3;
            const double Gd = G_dep[pix], Ga = G_alp[pix], Gx = G_dis[pix];
            double Tr = 1 - A, Sb = with_bg ? (1 - A) * (Gi[0] * bg[0] + Gi[1] * bg[1] + Gi[2] * bg[2]) : 0;
            double SbA = with_bg ? (1 - A) * (fabs(Gi[0] * bg[0]) + fabs(Gi[1] * bg[1]) + fabs(Gi[2] * bg[2])) : 0;
            for (int q = nh - 1; q >= 0; --q) {
                const int i = order[hit_j[q]];
                const Surfel* s = &S[i];
                intersect(s, x, y, dr, r2, &h, NULL);
                const double om = 1 - h.alpha;
                Tr /= om;
                const double w = Tr * h.alpha;
                const double m = ms * (1 - near_t / h.z);
                const double e = m * m * A - 2 * m * wm + wm2;
                const double* col = colour + 3 * i;
                const double gf = Gi[0] * col[0] + Gi[1] * col[1] + Gi[2] * col[2] + Gn[0] * s->n[0] +
                                  Gn[1] * s->n[1] + Gn[2] * s->n[2] + Gd * h.z + Ga + Gx * e;
                const double ga_ = Tr * gf - Sb / om;
                Sb += w * gf;
                /* the same chain on the magnitudes of every part (mass): |terms| wherever a sum is formed */
                const double gfA = fabs(Gi[0] * col[0]) + fabs(Gi[1] * col[1]) + fabs(Gi[2] * col[2]) +
                                   fabs(Gn[0] * s->n[0]) + fabs(Gn[1] * s->n[1]) + fabs(Gn[2] * s->n[2]) +
                                   fabs(Gd * h.z) + fabs(Ga) + fabs(Gx) * (m * m * A + 2 * fabs(m * wm) + wm2);
                const double gaA = Tr * gfA + SbA / om;
                SbA += w * gfA;
                double g[SG], gA[SG];
                memset(g, 0, sizeof(g));
                memset(gA, 0, sizeof(gA));
                for (int c = 0; c < 3; ++c) {
                    g[10 + c] += w * Gi[c];
                    g[13 + c] += w * Gn[c];
                    gA[10 + c] = fabs(g[10 + c]);
                    gA[13 + c] = fabs(g[13 + c]);
                }
                const double dm = ms * near_t / (h.z * h.z);
                const double gz = w * Gd + Gx * 2 * w * (m * A - wm) * dm;
                const double gzA = fabs(w * Gd) + fabs(Gx) * 2 * w * (fabs(m * A) + fabs(wm)) * dm;
                double grho = 0, grhoA = 0;
                if (!h.clamped) {
                    g[9] += ga_ * h.G;
                    gA[9] = gaA * h.G;
                    grho = -0.5 * h.alpha * ga_;
                    grhoA = 0.5 * h.alpha * gaA;
                }
                if (h.use3) {
                    const double ga = 2 * h.a * grho + gz * s->M[6], gb = 2 * h.b * grho + gz * s->M[7];
                    const double gaP = 2 * fabs(h.a) * grhoA + gzA * fabs(s->M[6]);
                    const double gbP = 2 * fabs(h.b) * grhoA + gzA * fabs(s->M[7]);
                    const double ic = 1 / fabs(h.c2);
                    const double gcA[3] = {gaP * ic, gbP * ic, (gaP * fabs(h.a) + gbP * fabs(h.b)) * ic};
                    const double* X = h.hx;
                    const double* Y = h.hy;
                    const double ghxA[3] = {fabs(Y[1]) * gcA[2] + fabs(Y[2]) * gcA[1],
                                            fabs(Y[2]) * gcA[0] + fabs(Y[0]) * gcA[2],
                                            fabs(Y[0]) * gcA[1] + fabs(Y[1]) * gcA[0]};
                    const double ghyA[3] = {gcA[1] * fabs(X[2]) + gcA[2] * fabs(X[1]),
                                            gcA[2] * fabs(X[0]) + gcA[0] * fabs(X[2]),
                                            gcA[0] * fabs(X[1]) + gcA[1] * fabs(X[0])};
                    for (int k = 0; k < 3; ++k) {
                        gA[k] = fabs(dr[2]) * ghxA[k];
                        gA[3 + k] = fabs(dr[2]) * ghyA[k];
                        gA[6 + k] = fabs(dr[0]) * ghxA[k] + fabs(dr[1]) * ghyA[k];
                    }
                    gA[6] += gzA * fabs(h.a);
                    gA[7] += gzA * fabs(h.b);
                    gA[8] += gzA;
                    g[6] += gz * h.a;
                    g[7] += gz * h.b;
                    g[8] += gz;
                    const double gc[3] = {ga / h.c2, gb / h.c2, -(ga * h.a + gb * h.b) / h.c2};
                    const double ghx[3] = {h.hy[1] * gc[2] - h.hy[2] * gc[1], h.hy[2] * gc[0] - h.hy[0] * gc[2],
                                           h.hy[0] * gc[1] - h.hy[1] * gc[0]};
                    const double ghy[3] = {gc[1] * h.hx[2] - gc[2] * h.hx[1], gc[2] * h.hx[0] - gc[0] * h.hx[2],
                                           gc[0] * h.hx[1] - gc[1] * h.hx[0]};
                    for (int k = 0; k < 3; ++k) {
                        g[k] -= dr[2] * ghx[k];
                        g[3 + k] -= dr[2] * ghy[k];
                        g[6 + k] += dr[0] * ghx[k] + dr[1] * ghy[k];
                    }
                } else {
                    g[16] += -4 * h.dx * grho;
                    g[17] += -4 * h.dy * grho;
                    g[18] += gz;
                    gA[16] = 4 * fabs(h.dx) * grhoA;
                    gA[17] = 4 * fabs(h.dy) * grhoA;
                    gA[18] = gzA;
                }
                double* row = rows + (size_t)i * SG;
                for (int k = 0; k < SG; ++k) {
#pragma omp atomic
                    row[k] += g[k];
                    if (mass != NULL) {
#pragma omp atomic
                        mass[(size_t)i * SG + k] += gA[k];
                    }
                }
            }
        }
    free(hit_j);
    }
    if (bwd) {
        const double fx = K[0], cx = K[2], fy = K[4], cy = K[5];
        for (int i = 0; i < N; ++i) {
            double* gx = g_xyz + 3 * i;
            double* gq = g_quat + 4 * i;
            double* gs = g_scale + 3 * i;
            const Surfel* s = &S[i];
            memset(gx, 0, 3 * sizeof(double));
            memset(gq, 0, 4 * sizeof(double));
            memset(gs, 0, 3 * sizeof(double));
            g_opl[i] = 0;
            uv_grad[2 * i] = uv_grad[2 * i + 1] = 0;
            for (int c = 0; c < 3; ++c) g_col[3 * i + c] = 0;
            if (!s->vis) continue;
            const double* g = rows + (size_t)i * SG;
            for (int c = 0; c < 3; ++c) g_col[3 * i + c] = g[10 + c];
            const double* p = s->p;
            double J[6];
            lens_jac(p, fx, fy, J);
            /* uv.grad = J_n^-T g_n + g_c, J_n = p_z J[:, :2] */
            const double gnx = g[0] * s->M[6] + g[1] * s->M[7] + g[2] * s->M[8];
            const double gny = g[3] * s->M[6] + g[4] * s->M[7] + g[5] * s->M[8];
            const double j00 = p[2] * J[0], j01 = p[2] * J[1], j10 = p[2] * J[3], j11 = p[2] * J[4];
            const double det = j00 * j11 - j01 * j10;
            uv_grad[2 * i] = (j11 * gnx - j10 * gny) / det + g[16];
            uv_grad[2 * i + 1] = (j00 * gny - j01 * gnx) / det + g[17];
            (void)cx; (void)cy;
            double gX[3][3];
            for (int j = 0; j < 3; ++j) {
                gX[j][0] = g[j];
                gX[j][1] = g[3 + j];
                gX[j][2] = g[6 + j];
            }
            double gp[3] = {gX[2][0], gX[2][1], gX[2][2] + g[18]};
            for (int k = 0; k < 3; ++k) gp[k] += J[k] * g[16] + J[3 + k] * g[17];
            double gRc[9];
            for (int r = 0; r < 3; ++r) {
                gRc[r * 3] = s->su * gX[0][r];
                gRc[r * 3 + 1] = s->sv * gX[1][r];
                gRc[r * 3 + 2] = s->sgn * g[13 + r];
            }
            const double gsu = gX[0][0] * s->Rc[0] + gX[0][1] * s->Rc[3] + gX[0][2] * s->Rc[6];
            const double gsv = gX[1][0] * s->Rc[1] + gX[1][1] * s->Rc[4] + gX[1][2] * s->Rc[7];
            gs[0] = gsu * s->su;
            gs[1] = gsv * s->sv;
            double gR[9];
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c)
                    gR[r * 3 + c] = T[r] * gRc[c] + T[4 + r] * gRc[3 + c] + T[8 + r] * gRc[6 + c];
            for (int k = 0; k < 3; ++k) gx[k] = T[k] * gp[0] + T[4 + k] * gp[1] + T[8 + k] * gp[2];
            /* R(q / |q|): d R / d qn, then the normalisation */
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
            g_opl[i] = g[9] * s->opa * (1 - s->opa);
        }
    }
    free(S);
    free(order);
    free(zs);
    return M;
}
