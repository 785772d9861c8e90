/* cull_oracle.c — CPU restatement of the forward's per-block culling tests (gsr_record.cuh) and of the tile walk's
 * per-pixel alpha, to check that the exact ellipse-vs-block test (row_cull) is conservative and never looser than
 * the bounding circle AND box it replaces (footprint_bounds / footprint_hits).
 *
 * TEST INFRASTRUCTURE ONLY (tests/test_cull_oracle.py).  fp32 throughout, operations in kernel order, no
 * contraction (-ffp-contract=off): every fmaf below is an fma in the kernel.  The kernel's MUFU square roots and
 * reciprocals (a few ulps) are restated as the correctly rounded operations; row_cull's margins are sized for
 * 2^-18 relative, far above either.  ex2.approx (the walk's __expf) is restated pessimistically as exp2f rounded up
 * by 2^-21 relative, so a block the test calls safe stays safe under the approximation's error.
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC cull_oracle.c -lm
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

static float u2f(uint32_t u) {
    float f;
    memcpy(&f, &u, 4);
    return f;
}

/* gsr_record.cuh cull_tau */
static float cull_tau(float a, float bh, float c, float det, float opa) {
    if (!(opa > 0.0039137f)) return -1.0f;
    if (!(det > 0.0f) || !(a > 0.0f) || !(c > 0.0f)) return INFINITY;
    const float hd = 0.5f * (a - c);
    const float lam = 0.5f * (a + c) + sqrtf(hd * hd + bh * bh);
    const float tau = fmaxf(2.0f * logf(opa * 255.6f), 0.0f);
    const float t = (1.06f + 4e-6f * (lam * lam / det)) * tau;
    return (t == t) ? t : INFINITY;
}

/* footprint_bounds + footprint_hits, as build_lists calls them with -DGSR_CULL_BOX=1 */
static int old_hit(float u, float v, float tau, float a, float b2, float c, float x0, float y0, float w) {
    if (!(tau >= 0.0f)) return 0;
    const float hd = 0.5f * (a - c), bh = 0.5f * b2;
    const float lam = 0.5f * (a + c) + sqrtf(hd * hd + bh * bh);
    const float r2 = fmaf(tau, lam * 1.0001f, 1.0f), hx2 = fmaf(tau, a, 1.0f), hy2 = fmaf(tau, c, 1.0f);
    const float dy = fmaxf(fmaxf(y0 - v, v - (y0 + 3.0f)), 0.0f);
    const float dx = fmaxf(fmaxf(x0 - u, u - (x0 + w)), 0.0f);
    const float dx2 = dx * dx, dy2 = dy * dy;
    return (dx2 + dy2 <= r2) && (dx2 <= hx2) && (dy2 <= hy2);
}

/* row_cull + row_block_hits */
static int new_hit(float u, float v, float tau, float a, float b2, float c, float det, float x0, float y0, float w) {
    const float GROW = 1.0f + 0x1p-18f, EREL = 0x1p-18f, MABS = 0x1p-12f, BOX_SHRINK = 1.0f - 0x1p-19f;
    const float bh = 0.5f * b2;
    const float lo = y0 - v, hi = (y0 + 3.0f) - v;
    const float dy = fmaxf(fmaxf(lo, -hi), 0.0f);
    const float te = tau * GROW;
    const float tc = te * c;
    const int rows = dy * dy <= fminf(tc, fmaf(tau, c, 1.0f));
    const float X = sqrtf(te * a);
    const float ds = bh * X * (1.0f / a);
    const float e = (fabsf(lo) + fabsf(hi) + fabsf(ds)) * EREL;
    const float lo1 = lo - e, hi1 = hi + e, lo2 = lo1 - e, hi2 = hi1 + e;
    const float slo = sqrtf(det * fmaxf(fmaf(-lo1, lo1, tc), 0.0f));
    const float shi = sqrtf(det * fmaxf(fmaf(-hi1, hi1, tc), 0.0f));
    const float rc = 1.0f / c;
    const int rup = ds > hi2, lup = -ds > hi2;
    float R = fmaf(bh, rup ? hi1 : lo1, rup ? shi : slo) * rc;
    float L = fmaf(bh, lup ? hi1 : lo1, -(lup ? shi : slo)) * rc;
    R = (ds >= lo2 && !rup) ? X : R;
    L = (-ds >= lo2 && !lup) ? -X : L;
    const float m = fmaf(X, EREL, MABS);
    const float B = sqrtf(fmaf(tau, a, 1.0f)) * BOX_SHRINK;
    const float xhi = fminf(R + m, B);
    const float xlo = fmaxf(L - m, -B) - w;
    const float dx0 = x0 - u;
    return rows && !(dx0 > xhi) && !(dx0 < xlo);
}

/* does pixel (px, py) pass the walk's "mh > 0 and alpha > 1/255" test (fwd_walk; the division is the correctly
 * rounded quotient there, directly or through the exact recompute of a flagged pixel) */
static int pixel_contributes(float u, float v, float opa, float a, float b2, float c, float det, float px, float py) {
    const float du = px - u, dv = py - v;
    const float t1 = du * b2, t2 = du * c;
    const float t4 = fmaf(du, t2, t1 * -dv);
    const float num = fmaf(dv, dv * a, t4);
    const float mh = num / det;
    if (!(mh > 0.0f)) return 0;
    const float xe = (mh * -0.5f) * 1.4426950216293334961f;
    const float g = nextafterf(exp2f(xe) * (1.0f + 0x1p-21f), INFINITY);
    return g * opa > u2f(0x3b808080u);
}

/* Per case k: the record is made from (u, v, a, b2, c, opa) as make_record does (det = fma(a, c, -bh^2)); tau' is
 * cull_tau's unless tau_in[k] is not NaN.  The block is the (w+1) x 4 pixels at (x0, y0).
 * flags[k] bit 0: new test lists, bit 1: old test lists, bit 2: some pixel of the block contributes.
 * Returns the number of cases that break a rule (new culls a contributing block, or lists one the old culls). */
int cull_check(int n, const float* u, const float* v, const float* a, const float* b2, const float* c,
               const float* opa, const float* tau_in, const float* x0, const float* y0, float w, uint8_t* flags) {
    int bad = 0;
    for (int k = 0; k < n; ++k) {
        const float bh = b2[k] * 0.5f;
        const float det = fmaf(a[k], c[k], -(bh * bh));
        const float tau = (tau_in[k] == tau_in[k]) ? tau_in[k] : cull_tau(a[k], bh, c[k], det, opa[k]);
        const int nh = new_hit(u[k], v[k], tau, a[k], b2[k], c[k], det, x0[k], y0[k], w);
        const int oh = old_hit(u[k], v[k], tau, a[k], b2[k], c[k], x0[k], y0[k], w);
        int contrib = 0;
        for (int yy = 0; yy < 4 && !contrib; ++yy)
            for (int xx = 0; xx <= (int)w && !contrib; ++xx)
                contrib = pixel_contributes(u[k], v[k], opa[k], a[k], b2[k], c[k], det, x0[k] + (float)xx,
                                            y0[k] + (float)yy);
        flags[k] = (uint8_t)(nh | (oh << 1) | (contrib << 2));
        bad += (contrib && !nh) || (nh && !oh);
    }
    return bad;
}
