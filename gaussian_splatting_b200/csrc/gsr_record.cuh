// gsr_record.cuh — the 48-byte splat record staged by TMA into the tile renderers.
#pragma once
#include "gsr_common.cuh"
#include "gsr_math.cuh"

namespace gsr {

// Culling bound stored in the record: tau' such that a pixel at offset d from the mean with
// d^T Sigma^-1 d > tau' provably has alpha = opacity * exp(-mh/2) below the reference's 1/255 skip
// threshold (alpha < t  <=  mh > 2 ln(opacity / t)).  tau' is the exact bound inflated by 6% plus a
// condition-number term, so that neither the fp32 rounding of mh in the kernels nor the few-ulp error of
// ex2.approx can make a culled pixel pass the reference's test (row_cull adds only margins for its own fp32
// evaluation); culling is therefore invisible in the results (checked bitwise against the reference).
// Returns -1 when the splat can never reach the threshold, +inf when nothing can be proven.
__device__ __forceinline__ float cull_tau(float a, float bh, float c, float det, float opa) {
    if (!(opa > 0.0039137f)) return -1.0f;  // 0.998 / 255: opacity * g <= opacity can never reach 1/255
    if (!(det > 0.0f) || !(a > 0.0f) || !(c > 0.0f)) return __int_as_float(0x7f800000);
    const float hd = 0.5f * (a - c);
    const float lam = 0.5f * (a + c) + sqrtf(hd * hd + bh * bh);  // lambda_max of [[a,b],[b,c]]
    const float tau = fmaxf(2.0f * logf(opa * 255.6f), 0.0f);
    const float t = (1.06f + 4e-6f * (lam * lam / det)) * tau;
    return (t == t) ? t : __int_as_float(0x7f800000);
}

// Necessary conditions for the ellipse {d^T Sigma^-1 d <= tau'} (plus 1 px^2 slack) to reach a pixel
// rectangle whose per-axis distances from the splat centre are (dx, dy): inside the bounding circle of
// radius sqrt(tau' lambda_max) and inside the axis-aligned bounding box sqrt(tau' a) x sqrt(tau' c).
struct FootprintBounds {
    float r2, hx2, hy2;  // squared limits; all negative when the splat can never contribute
};
__device__ __forceinline__ FootprintBounds footprint_bounds(float tau, float a, float b2, float c) {
    FootprintBounds f;
    if (!(tau >= 0.0f)) {
        f.r2 = f.hx2 = f.hy2 = -1.0f;
        return f;
    }
    const float hd = 0.5f * (a - c), bh = 0.5f * b2;
    const float lam = 0.5f * (a + c) + sqrtf(hd * hd + bh * bh);
    f.r2 = fmaf(tau, lam * 1.0001f, 1.0f);
    f.hx2 = fmaf(tau, a, 1.0f);
    f.hy2 = fmaf(tau, c, 1.0f);
    return f;
}
__device__ __forceinline__ bool footprint_hits(const FootprintBounds& f, float dx, float dy) {
    const float dx2 = dx * dx, dy2 = dy * dy;
    return (dx2 + dy2 <= f.r2) && (dx2 <= f.hx2) && (dy2 <= f.hy2);
}

__device__ __forceinline__ float sqrt_approx(float x) {  // MUFU, a few ulps; 0 for x <= 2^-126
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Exact culling of a row band of pixel blocks.  The blocks share the rows y0 .. y0+3 (the slab dv in [lo, hi],
// dv = y - v) and differ only in their columns.  Per record this computes the x-interval of the ellipse
// E = {d^T Sigma^-1 d <= tau'} intersected with the slab; a block of columns x0 .. x0+w is then hit iff
// xlo <= x0 - u <= xhi (row_block_hits: one subtraction and two compares per block).
//
// At fixed dv, E spans du in (bh dv -+ sqrt(det (tau' c - dv^2))) / c.  The right end R(dv) is concave with its
// maximum sqrt(tau' a) at dv* = bh sqrt(tau'/a) (the ellipse's rightmost point), the left end L(dv) = -R(-dv)
// convex with its minimum at -dv*.  So over the slab: max R = sqrt(tau' a) if dv* lies in the slab, else R at
// the slab end nearer dv*; likewise min L.
//
// Conservative by construction, in exact arithmetic and in fp32:
//   * tau' keeps its margin (cull_tau): pixels outside E cannot reach the 1/255 skip threshold.
//   * The interval is evaluated for tau'(1 + 2^-18): the rounding of tau' c and of dv^2 (2^-24 relative each) can
//     then never make tau' c - dv^2 smaller than its exact value, even where it cancels to 0 at the ellipse's top
//     and bottom (where the square root would amplify a rounding error into 2^-12 of the width).
//   * The slab ends carry a rounding error of 2^-24 |lo|, dv* one of a few ulps; e = 2^-18 (|lo| + |hi| + |dv*|)
//     exceeds both.  dv* counts as inside when it is within 2e of the slab; otherwise the end is moved by e
//     TOWARDS dv*, where R (L) is monotone, so the evaluated end is never below (above) the exact one.
//   * The interval is widened by m = 2^-18 sqrt(tau' a) + 2^-12 px: every term of R and L is at most
//     sqrt(tau' a) in size, so the few-ulp errors of the MUFU square roots and reciprocals, the products and
//     x0 - u stay below the relative part; the absolute part covers coordinates' ulps and flushed denormals.
//   * The result is never looser than the previous circle-and-box test (footprint_bounds): the row test is that
//     test's y box intersected with the exact y extent tau'(1 + 2^-18) c, the interval is clipped to that test's
//     x box sqrt(tau' a + 1) shrunk by 2^-19 (its rounding and the square root's), and the few-ulp margins above
//     stay inside the bounding circle's 1.0001 lambda_max + 1 px^2.  Where the 1 px^2 of the box falls below
//     those 2^-19 (sqrt(tau' a) > 512 px) the clip can cut pixels with d^T Sigma^-1 d > tau'(1 - 2^-18), which
//     tau''s 6 % margin covers.
//   * Sentinels need no branch: tau' < 0 fails the row test (its y extent is negative); tau' = +inf (and any
//     overflow) turns the ends into +-inf or NaN, and fminf / fmaxf against the box (then infinite) list the
//     block.
// tests/cull_oracle.c restates this in C; its test checks every culled block against the kernel's per-pixel alpha.
struct RowCull {
    float xlo, xhi;  // x0 - u of a block of columns x0 .. x0+w must lie in [xlo, xhi]
    bool rows;       // the record's ellipse reaches rows y0 .. y0+3 at all
};
__device__ __forceinline__ RowCull row_cull(float v, float tau, float a, float b2, float c, float det, float y0,
                                            float w) {
    constexpr float GROW = 1.0f + 0x1p-18f, EREL = 0x1p-18f, MABS = 0x1p-12f, BOX_SHRINK = 1.0f - 0x1p-19f;
    RowCull r;
    const float bh = 0.5f * b2;
    const float lo = y0 - v, hi = (y0 + 3.0f) - v;
    const float dy = fmaxf(fmaxf(lo, -hi), 0.0f);
    const float te = tau * GROW;
    const float tc = te * c;
    r.rows = dy * dy <= fminf(tc, fmaf(tau, c, 1.0f));
    const float X = sqrt_approx(te * a);
    const float ds = bh * X * rcp_approx(a);
    const float e = (fabsf(lo) + fabsf(hi) + fabsf(ds)) * EREL;
    const float lo1 = lo - e, hi1 = hi + e, lo2 = lo1 - e, hi2 = hi1 + e;
    const float slo = sqrt_approx(det * fmaxf(fmaf(-lo1, lo1, tc), 0.0f));
    const float shi = sqrt_approx(det * fmaxf(fmaf(-hi1, hi1, tc), 0.0f));
    const float rc = rcp_approx(c);
    const bool rup = ds > hi2, lup = -ds > hi2;
    float R = fmaf(bh, rup ? hi1 : lo1, rup ? shi : slo) * rc;
    float L = fmaf(bh, lup ? hi1 : lo1, -(lup ? shi : slo)) * rc;
    R = (ds >= lo2 && !rup) ? X : R;
    L = (-ds >= lo2 && !lup) ? -X : L;
    const float m = fmaf(X, EREL, MABS);
    const float B = sqrt_approx(fmaf(tau, a, 1.0f)) * BOX_SHRINK;
    r.xhi = fminf(R + m, B);
    r.xlo = fmaxf(L - m, -B) - w;
    return r;
}
// NaN-safe: an interval end that is NaN lists the block
__device__ __forceinline__ bool row_block_hits(const RowCull& r, float dx0) {
    return r.rows & !(dx0 > r.xhi) & !(dx0 < r.xlo);
}

// Anti-aliased mode: the opacity factor rho = sqrt(max(det0, 0) / det) that gives the dilated splat the mass of the
// undilated one (det0 = det of the undilated 2-D covariance, det = det of the dilated one, as make_record forms it).
// Pinned operation order; tests/antialiased_oracle.c reproduces it bit for bit:
//   a = c0 + 1/4;  c = c2 + 1/4;  bh = c1 * 1/2;  bb = bh * bh
//   det  = fma(a, c, -bb);  det0 = fma(c0, c2, -bb)
//   rho  = sqrt_rn(div_rn(fmax(det0, 0), det))
// rho == 0 where det0 <= 0 in fp32 (needles seen end-on, underflowing scales): the splat then never contributes.
__device__ __forceinline__ float aa_rho(float c0, float c1, float c2) {
    const float a = __fadd_rn(c0, 0.25f);
    const float c = __fadd_rn(c2, 0.25f);
    const float bh = __fmul_rn(c1, 0.5f);
    const float bb = __fmul_rn(bh, bh);
    const float det = __fmaf_rn(a, c, -bb);
    const float det0 = __fmaf_rn(c0, c2, -bb);
    return __fsqrt_rn(__fdiv_rn(fmaxf(det0, 0.0f), det));
}

// 3-D smoothing filter (Mip-Splatting): Sigma_world = R diag(v + F) R^T with v_k = exp(s_k)^2 and F = f^2, f the
// filter's standard deviation in world units, and the opacity factor coef = sqrt(det Sigma / det(Sigma + F I)) that
// keeps the filtered gaussian's 3-D mass.  Per axis, so that tiny scales do not underflow a product of variances.
// Pinned operation order; tests/filter3d_oracle.c reproduces it bit for bit:
//   v'_k = v_k + F;  t_k = F == 0 ? 1 : v_k / v'_k  (IEEE division);  coef = sqrt_rn((t_0 * t_1) * t_2)
// F == 0 gives v' = v and coef = 1 exactly: the unfiltered record.  coef == 0 where the t_k product underflows (a scale
// far below the filter): the splat then never contributes.
__device__ __forceinline__ float f3d_filter(const float* __restrict__ v, float F, float* __restrict__ vp,
                                            float* __restrict__ t) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        vp[k] = __fadd_rn(v[k], F);
        t[k] = F == 0.0f ? 1.0f : __fdiv_rn(v[k], vp[k]);
    }
    return __fsqrt_rn(__fmul_rn(__fmul_rn(t[0], t[1]), t[2]));
}

__device__ __forceinline__ void make_record(float u, float v, float c0, float c1, float c2, float opa,
                                            float r, float g, float b, float* __restrict__ rec) {
    // a, b, c, det: src/render.cu:117-127 (fp32 branch: +0.25 dilation), rounding order of the reference build
    const float a = __fadd_rn(c0, 0.25f);
    const float c = __fadd_rn(c2, 0.25f);
    const float bh = __fmul_rn(c1, 0.5f);
    const float det = __fmaf_rn(a, c, -__fmul_rn(bh, bh));
    // 1/det, correctly rounded.  The forward uses it for q = num*rcp; q += rcp*fma(-det,q,num), which is the
    // correctly rounded IEEE quotient num/det while det and num stay far from the denormal/overflow range
    // (Markstein); the backward uses it as the reference's `1.0 / det` (src/render_backward.cu:153).
    const float rcp = __frcp_rn(det);
    rec[R_U] = u;
    rec[R_V] = v;
    rec[R_R2] = cull_tau(a, bh, c, det, opa);
    rec[R_OPA] = opa;
    rec[R_A] = a;
    rec[R_B2] = __fadd_rn(bh, bh);
    rec[R_C] = c;
    rec[R_DET] = det;
    rec[R_RCP] = rcp;
    rec[R_CR] = __fmul_rn(r, GSR_SH0);  // sh_to_rgb with N_SH == 1: Y0 * rgb (src/spherical_harmonics.cuh:83)
    rec[R_CG] = __fmul_rn(g, GSR_SH0);
    rec[R_CB] = __fmul_rn(b, GSR_SH0);
}

}  // namespace gsr
