/* antialiased_oracle.c — CPU oracle of the anti-aliased opacity compensation of the fused rasterizer
 * (rasterize(antialiased=True)).  TEST INFRASTRUCTURE ONLY (tests/antialiased_oracle.py).
 *
 *   rho = sqrt(max(det0, 0) / det),  opacity' = opacity * rho
 *
 * with det0 the determinant of the 2-D covariance (c0, c1/2; c1/2, c2) and det that of the covariance + 0.25 I.  The
 * fp32 function performs exactly the operations of gsr_record.cuh aa_rho (fmaf; IEEE division and square root;
 * compiled with -ffp-contract=off), so records can be compared bit for bit.
 * Build: gcc -O2 -ffp-contract=off -mfma -shared -fPIC antialiased_oracle.c -lm
 */
#include <math.h>

void aa_compensate_f32(int n, const float* conic, const float* opacity, float* rho, float* opacity_out) {
    for (int i = 0; i < n; ++i) {
        const float c0 = conic[i * 3], c1 = conic[i * 3 + 1], c2 = conic[i * 3 + 2];
        const float a = c0 + 0.25f;
        const float c = c2 + 0.25f;
        const float bh = c1 * 0.5f;
        const float bb = bh * bh;
        const float det = fmaf(a, c, -bb);
        const float det0 = fmaf(c0, c2, -bb);
        const float r = sqrtf(fmaxf(det0, 0.0f) / det);
        rho[i] = r;
        opacity_out[i] = opacity[i] * r;
    }
}

void aa_compensate_f64(int n, const double* conic, const double* opacity, double* rho, double* opacity_out) {
    for (int i = 0; i < n; ++i) {
        const double c0 = conic[i * 3], c1 = conic[i * 3 + 1], c2 = conic[i * 3 + 2];
        const double bh = c1 * 0.5, bb = bh * bh;
        const double det = fma(c0 + 0.25, c2 + 0.25, -bb);
        const double det0 = fma(c0, c2, -bb);
        const double r = sqrt(fmax(det0, 0.0) / det);
        rho[i] = r;
        opacity_out[i] = opacity[i] * r;
    }
}
