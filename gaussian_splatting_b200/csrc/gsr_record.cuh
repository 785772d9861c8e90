// gsr_record.cuh — the 48-byte splat record staged by TMA into the tile renderers.
#pragma once
#include "gsr_common.cuh"
#include "gsr_math.cuh"

namespace gsr {

// Culling bound stored in the record: tau' such that a pixel at offset d from the mean with
// d^T Sigma^-1 d > tau' provably has alpha = opacity * exp(-mh/2) below the reference's 1/255 skip
// threshold (alpha < t  <=  mh > 2 ln(opacity / t)).  tau' is the exact bound inflated by 6% plus a
// condition-number term, and the footprint tests add 1 px^2 of slack, so that neither the fp32 rounding of
// mh in the kernels nor the few-ulp error of ex2.approx can make a culled pixel pass the reference's test;
// culling is therefore invisible in the results (checked bitwise against the reference).
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
