// gsr_surfels_lens.cuh — the lens geometry of rasterize_surfels(..., fisheye=k / distortion=k), fp64, for the host
// and the device (DESIGN.md 3.26): each pixel's undistorted ray, and a box in pixels around every pixel whose ray
// meets a surfel's cutoff disk (the binning bound).  Lens constants as in gsr_fisheye.h / gsr_distortion.h:
//   fisheye    {k1, k2, k3, k4, theta_max}      distortion {k1, k2, p1, p2, k3, r2_max}
// A ray exists only on the lens's monotone branch (theta < theta_max, s = r^2 < r2_max); elsewhere it is d = 0.
#pragma once
#include <math.h>

#include "../../include/gsr_surfels_lens.h"

namespace gsr {
namespace surfel {

// theta_d = theta (1 + k1 t + k2 t^2 + k3 t^3 + k4 t^4), t = theta^2, and its derivative
__host__ __device__ __forceinline__ double fe_theta_d(double th, const float* kc) {
    const double t = th * th;
    return th * (1.0 + t * (kc[0] + t * (kc[1] + t * ((double)kc[2] + t * kc[3]))));
}
__host__ __device__ __forceinline__ double fe_theta_d_prime(double th, const float* kc) {
    const double t = th * th;
    return 1.0 + t * (3.0 * kc[0] + t * (5.0 * kc[1] + t * (7.0 * kc[2] + t * 9.0 * kc[3])));
}

// the OPENCV model on the normalised point (a, b): (a_d, b_d) and the symmetric Jacobian (D00, D01, D11)
__host__ __device__ __forceinline__ void dt_model(double a, double b, const float* kc, double& ad, double& bd, double* D) {
    const double k1 = kc[0], k2 = kc[1], p1 = kc[2], p2 = kc[3], k3 = kc[4];
    const double s = a * a + b * b;
    const double R = 1.0 + s * (k1 + s * (k2 + s * k3));
    const double R1 = k1 + s * (2.0 * k2 + s * 3.0 * k3);
    ad = a * R + 2.0 * p1 * a * b + p2 * (s + 2.0 * a * a);
    bd = b * R + p1 * (s + 2.0 * b * b) + 2.0 * p2 * a * b;
    if (D != nullptr) {
        D[0] = R + 2.0 * a * a * R1 + 2.0 * p1 * b + 6.0 * p2 * a;
        D[1] = 2.0 * a * b * R1 + 2.0 * p1 * a + 2.0 * p2 * b;
        D[2] = R + 2.0 * b * b * R1 + 6.0 * p1 * b + 2.0 * p2 * a;
    }
}

// The unit ray d of the distorted normalised point (xd, yd) = ((x - cx) / fx, (y - cy) / fy): the lens inverted on its
// monotone branch.  Returns false (and d = 0) where the point has no preimage there.
__host__ __device__ __forceinline__ bool lens_ray(int lens, double xd, double yd, const float* kc, double* d) {
    d[0] = d[1] = d[2] = 0.0;
    if (!(xd == xd) || !(yd == yd)) return false;
    if (lens == GSR_SURFEL_LENS_FISHEYE) {
        const double td = sqrt(xd * xd + yd * yd);
        const double thmax = kc[4];
        if (!(td < fe_theta_d(thmax, kc))) return false;
        if (td == 0.0) {
            d[2] = 1.0;
            return true;
        }
        // theta_d is increasing on [0, theta_max): Newton inside a shrinking bracket, bisection when it leaves it
        double lo = 0.0, hi = thmax, th = fmin(td, 0.5 * thmax);
        for (int it = 0; it < 100; ++it) {
            const double f = fe_theta_d(th, kc) - td;
            if (f > 0.0) hi = th; else lo = th;
            double nt = th - f / fe_theta_d_prime(th, kc);
            if (!(nt > lo && nt < hi)) nt = 0.5 * (lo + hi);
            if (nt == th || hi - lo <= 1e-17 * hi) { th = nt; break; }
            th = nt;
        }
        if (!(th < thmax)) return false;
        double sn, cs;
#ifdef __CUDA_ARCH__
        sincospi(th * 0.31830988618379067, &sn, &cs);  // theta <= pi / 2: no argument reduction through local memory
#else
        sn = sin(th);
        cs = cos(th);
#endif
        d[0] = sn / td * xd;
        d[1] = sn / td * yd;
        d[2] = cs;
        return true;
    }
    // OPENCV: first the radial part alone (r R(r^2) is increasing for r^2 < r2_max), then Newton on the full model
    const double r2max = kc[5];
    const double rd = sqrt(xd * xd + yd * yd);
    double a = xd, b = yd;
    if (rd > 0.0) {
        auto fr = [&](double r) { const double s = r * r; return r * (1.0 + s * (kc[0] + s * (kc[1] + s * kc[4]))); };
        double lo = 0.0, hi = isfinite(r2max) ? sqrt(r2max) : 1.0;
        if (!isfinite(r2max))
            for (int it = 0; it < 200 && fr(hi) < rd; ++it) hi *= 2.0;
        double r = fmin(rd, 0.5 * hi);
        for (int it = 0; it < 100; ++it) {
            const double f = fr(r) - rd;
            if (f > 0.0) hi = r; else lo = r;
            const double s = r * r;
            double nr = r - f / (1.0 + s * (3.0 * kc[0] + s * (5.0 * kc[1] + s * 7.0 * kc[4])));
            if (!(nr > lo && nr < hi)) nr = 0.5 * (lo + hi);
            if (nr == r || hi - lo <= 1e-17 * hi) { r = nr; break; }
            r = nr;
        }
        a = xd * (r / rd);
        b = yd * (r / rd);
    }
    double ad, bd, D[3];
    for (int it = 0; it < 50; ++it) {
        dt_model(a, b, kc, ad, bd, D);
        const double ex = ad - xd, ey = bd - yd;
        const double det = D[0] * D[2] - D[1] * D[1];
        if (!(det > 0.0)) return false;
        const double da = (D[2] * ex - D[1] * ey) / det, db = (D[0] * ey - D[1] * ex) / det;
        a -= da;
        b -= db;
        if (fabs(da) + fabs(db) <= 1e-16 * (1.0 + fabs(a) + fabs(b))) break;
    }
    dt_model(a, b, kc, ad, bd, nullptr);
    if (!(fabs(ad - xd) + fabs(bd - yd) <= 1e-12 * (1.0 + rd)) || !(a * a + b * b < r2max)) return false;
    const double n = sqrt(a * a + b * b + 1.0);
    d[0] = a / n;
    d[1] = b / n;
    d[2] = 1.0 / n;
    return true;
}

struct Interval {
    double lo, hi;
};
__host__ __device__ __forceinline__ Interval iv_add(Interval x, Interval y) { return {x.lo + y.lo, x.hi + y.hi}; }
__host__ __device__ __forceinline__ Interval iv_scale(Interval x, double c) {
    return c >= 0.0 ? Interval{c * x.lo, c * x.hi} : Interval{c * x.hi, c * x.lo};
}
__host__ __device__ __forceinline__ Interval iv_mul(Interval x, Interval y) {
    const double p0 = x.lo * y.lo, p1 = x.lo * y.hi, p2 = x.hi * y.lo, p3 = x.hi * y.hi;
    return {fmin(fmin(p0, p1), fmin(p2, p3)), fmax(fmax(p0, p1), fmax(p2, p3))};
}
__host__ __device__ __forceinline__ Interval iv_sq(Interval x) {
    const double m = fmax(fabs(x.lo), fabs(x.hi));
    return (x.lo <= 0.0 && x.hi >= 0.0) ? Interval{0.0, m * m} : Interval{fmin(x.lo * x.lo, x.hi * x.hi), m * m};
}

// The binning bound: a box [u0, u1] x [v0, v1] in pixels containing the lens image of every point of the
// cutoff disk a^2 + b^2 <= r2 whose ray is valid.  Mp = M' = [s_u Rc0 | s_v Rc1 | p] (row-major; the disk must lie in
// front of the camera).  1. the disk's bounding box in the normalised plane, from the dual conic of M' (DESIGN.md
// 3.25 with K = I); 2. the lens image of that box: for the fisheye the annular sector of radii theta_d(atan r) over
// the box's range of r (clamped to theta_max) and of the box's angles, for OPENCV interval arithmetic on the model
// with s clamped below r2_max; 3. K.  Returns false when no point of the disk has a valid ray.
__host__ __device__ __forceinline__ bool surfel_lens_box(int lens, const double* Mp, double r2, double fx, double fy, double cx,
                                                double cy, const float* kc, double& u0, double& u1, double& v0,
                                                double& v1) {
    auto Dab = [&](int a, int b) {
        return r2 * (Mp[a * 3] * Mp[b * 3] + Mp[a * 3 + 1] * Mp[b * 3 + 1]) - Mp[a * 3 + 2] * Mp[b * 3 + 2];
    };
    const double D22 = Dab(2, 2);
    Interval A[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const double Dk2 = Dab(k, 2), Dkk = Dab(k, k);
        const double c = Dk2 / D22, half = sqrt(fmax(Dk2 * Dk2 - Dkk * D22, 0.0)) / -D22;
        A[k] = {c - half, c + half};
    }
    double X0, X1, Y0, Y1;  // the box in the distorted normalised plane
    if (lens == GSR_SURFEL_LENS_FISHEYE) {
        const double thmax = kc[4];
        const bool has0 = A[0].lo <= 0.0 && A[0].hi >= 0.0 && A[1].lo <= 0.0 && A[1].hi >= 0.0;
        const double nx = (A[0].lo <= 0.0 && A[0].hi >= 0.0) ? 0.0 : fmin(fabs(A[0].lo), fabs(A[0].hi));
        const double ny = (A[1].lo <= 0.0 && A[1].hi >= 0.0) ? 0.0 : fmin(fabs(A[1].lo), fabs(A[1].hi));
        const double fx_ = fmax(fabs(A[0].lo), fabs(A[0].hi)), fy_ = fmax(fabs(A[1].lo), fabs(A[1].hi));
        const double th0 = atan(sqrt(nx * nx + ny * ny));
        if (!(th0 < thmax)) return false;
        const double R0 = fe_theta_d(th0, kc), R1 = fe_theta_d(fmin(atan(sqrt(fx_ * fx_ + fy_ * fy_)), thmax), kc);
        if (has0) {
            X0 = Y0 = -R1;
            X1 = Y1 = R1;
        } else {
            // the box does not contain the origin: its directions span less than pi around the centre's, from e0 to e1
            // counterclockwise (the corners at the least and the greatest angle from the centre)
            const double ca = 0.5 * (A[0].lo + A[0].hi), cb = 0.5 * (A[1].lo + A[1].hi);
            double p0 = 0.0, p1 = 0.0, e0[2] = {ca, cb}, e1[2] = {ca, cb};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const double x = (j & 1) ? A[0].hi : A[0].lo, y = (j & 2) ? A[1].hi : A[1].lo;
                const double rel = atan2(ca * y - cb * x, ca * x + cb * y);
                if (rel < p0) { p0 = rel; e0[0] = x; e0[1] = y; }
                if (rel > p1) { p1 = rel; e1[0] = x; e1[1] = y; }
            }
            const double n0 = 1.0 / sqrt(e0[0] * e0[0] + e0[1] * e0[1]), n1 = 1.0 / sqrt(e1[0] * e1[0] + e1[1] * e1[1]);
            e0[0] *= n0; e0[1] *= n0; e1[0] *= n1; e1[1] *= n1;
            X0 = fmin(fmin(R0 * e0[0], R1 * e0[0]), fmin(R0 * e1[0], R1 * e1[0]));
            X1 = fmax(fmax(R0 * e0[0], R1 * e0[0]), fmax(R0 * e1[0], R1 * e1[0]));
            Y0 = fmin(fmin(R0 * e0[1], R1 * e0[1]), fmin(R0 * e1[1], R1 * e1[1]));
            Y1 = fmax(fmax(R0 * e0[1], R1 * e0[1]), fmax(R0 * e1[1], R1 * e1[1]));
            // the outer arc's extremes along the axes w between e0 and e1: e0 x w >= 0 and w x e1 >= 0
            if (e0[1] <= 0.0 && e1[1] >= 0.0) X1 = fmax(X1, R1);   // w = (1, 0)
            if (e0[0] >= 0.0 && e1[0] <= 0.0) Y1 = fmax(Y1, R1);   // w = (0, 1)
            if (e0[1] >= 0.0 && e1[1] <= 0.0) X0 = fmin(X0, -R1);  // w = (-1, 0)
            if (e0[0] <= 0.0 && e1[0] >= 0.0) Y0 = fmin(Y0, -R1);  // w = (0, -1)
        }
    } else {
        const double r2max = kc[5];
        if (isfinite(r2max)) {  // points with |a| or |b| >= sqrt(r2_max) have no valid ray
            const double L = sqrt(r2max);
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                A[k].lo = fmax(A[k].lo, -L);
                A[k].hi = fmin(A[k].hi, L);
                if (!(A[k].lo <= A[k].hi)) return false;
            }
        }
        const Interval A2 = iv_sq(A[0]), B2 = iv_sq(A[1]);
        Interval S = iv_add(A2, B2);
        if (!(S.lo < r2max)) return false;
        S.hi = fmin(S.hi, r2max);
        const double k1 = kc[0], k2 = kc[1], p1 = kc[2], p2 = kc[3], k3 = kc[4];
        Interval R = iv_add(iv_scale(S, k3), Interval{k2, k2});
        R = iv_add(iv_mul(S, R), Interval{k1, k1});
        R = iv_add(iv_mul(S, R), Interval{1.0, 1.0});
        const Interval AB = iv_mul(A[0], A[1]);
        const Interval AD = iv_add(iv_add(iv_mul(A[0], R), iv_scale(AB, 2.0 * p1)),
                                   iv_scale(iv_add(S, iv_scale(A2, 2.0)), p2));
        const Interval BD = iv_add(iv_add(iv_mul(A[1], R), iv_scale(iv_add(S, iv_scale(B2, 2.0)), p1)),
                                   iv_scale(AB, 2.0 * p2));
        X0 = AD.lo; X1 = AD.hi; Y0 = BD.lo; Y1 = BD.hi;
    }
    const double ua = fx * X0 + cx, ub = fx * X1 + cx, va = fy * Y0 + cy, vb = fy * Y1 + cy;
    u0 = fmin(ua, ub);
    u1 = fmax(ua, ub);
    v0 = fmin(va, vb);
    v1 = fmax(va, vb);
    return true;
}

}  // namespace surfel
}  // namespace gsr
