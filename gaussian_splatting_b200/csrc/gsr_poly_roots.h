// gsr_poly_roots.h — real roots of a small polynomial on the host, fp64: the lens cull limits of the fisheye
// (gsr_fisheye_theta_max) and radial-tangential (gsr_distortion_r2_max) libraries.
#pragma once

namespace gsr {

// p(t) = c[0] + c[1] t + ... + c[n] t^n
static inline double poly(const double* c, int n, double t) {
    double r = c[n];
    for (int i = n - 1; i >= 0; --i) r = r * t + c[i];
    return r;
}

// The real roots of p in [lo, hi], ascending (n <= 4): p is monotone between consecutive roots of p' (found the same
// way), so every piece with a sign change holds exactly one root, found by bisection to full precision.
static inline int roots_in(const double* c, int n, double lo, double hi, double* out) {
    while (n > 0 && c[n] == 0.0) --n;
    if (n == 0) return 0;
    double pts[8];
    int np = 0;
    pts[np++] = lo;
    if (n > 1) {
        double dc[4], cr[4];
        for (int i = 1; i <= n; ++i) dc[i - 1] = i * c[i];
        const int m = roots_in(dc, n - 1, lo, hi, cr);
        for (int j = 0; j < m; ++j)
            if (cr[j] > pts[np - 1]) pts[np++] = cr[j];
    }
    if (hi > pts[np - 1]) pts[np++] = hi;
    int r = 0;
    for (int j = 0; j < np; ++j) {
        const double a = pts[j], fa = poly(c, n, a);
        if (fa == 0.0) {
            if (r == 0 || out[r - 1] != a) out[r++] = a;
            continue;
        }
        if (j + 1 == np) break;
        double b = pts[j + 1];
        const double fb = poly(c, n, b);
        if (fb == 0.0 || (fa < 0.0) == (fb < 0.0)) continue;
        double x0 = a, x1 = b;
        // ends when the bracket holds no double between its ends: at most ~2100 halvings over the whole double range
        for (int it = 0; it < 2200 && x1 > x0; ++it) {
            const double mid = 0.5 * (x0 + x1);
            if (mid <= x0 || mid >= x1) break;
            if ((poly(c, n, mid) < 0.0) == (fa < 0.0)) x0 = mid;
            else x1 = mid;
        }
        out[r++] = x0;
    }
    return r;
}

}  // namespace gsr
