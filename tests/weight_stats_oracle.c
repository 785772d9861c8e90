/* weight_stats_oracle.c — CPU oracle of the blend-weight statistics of the fused rasterizer (weight_stats=...).
 *
 * TEST INFRASTRUCTURE ONLY (tests/weight_stats_oracle.py).  Compiled together with oracle/gsr_oracle.c, whose fp32
 * tile renderer forward (orc_render_forward_f32) it restates per pixel: same 0.25 dilation, fast exp, alpha < 1/255
 * skip and saturation break, and the same blend weight w = (float)((1 - (double)A) * (double)alpha).  For every
 * compact gaussian it accumulates over the pixels where the colour blend uses it
 *   sum[i] += w (double), max[i] = max(max[i], w) (float, exact), count[i] += 1 (exact),
 * and per pixel the accumulated alpha A [H,W] and the number of blends nblend [H,W].
 * uncertain [M] (NULL: not computed): per gaussian, the number of pixels whose walk reaches it at or after an alpha
 * within a relative 3e-5 of the 1/255 skip threshold (the threshold of orc_render_backward's `near`).  There another
 * exp implementation (the GPU's ex2.approx) may decide the skip the other way, and every later splat of that pixel
 * then sees a different accumulated alpha (its weight, and where the pixel saturates, may differ); such a walk is
 * followed to the end of the tile's list, past the saturation break.
 * dilated != 0: conic holds the renderer's (a, 2b, c) with the 0.25 dilation already added (the fused path's records).
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mfma -shared -fPIC -I<repo>/oracle weight_stats_oracle.c -lm
 */
#include "gsr_oracle.c"

void orc_weight_stats_f32(int H, int W, int M, const float* uvs, const float* opacity, const float* conic,
                          const int* ranges, const int* sorted_idx, double* sum, float* wmax, long long* count,
                          float* A_out, int* nblend, int* uncertain, int dilated) {
    const int ntx = (W + 15) / 16;
    for (int i = 0; i < M; ++i) {
        sum[i] = 0.0;
        wmax[i] = 0.0f;
        count[i] = 0;
        if (uncertain != NULL) uncertain[i] = 0;
    }
    /* sequential over pixels: the double sums are then independent of the thread count */
    for (int pix = 0; pix < H * W; ++pix) {
        const int py = pix / W, px = pix % W;
        const int tile = (py / 16) * ntx + (px / 16);
        float A = 0.0f;
        int nb = 0, near = 0, done = 0;
        for (int p = ranges[tile]; p < ranges[tile + 1]; ++p) {
            if ((double)A > 0.9999) done = 1;
            if (done && !near) break;
            const int g = sorted_idx[p];
            const float du = (float)px - uvs[g * 2], dv = (float)py - uvs[g * 2 + 1];
            const float b = conic[g * 3 + 1] * 0.5f;
            const float a = dilated ? conic[g * 3] : conic[g * 3] + 0.25f;
            const float c = dilated ? conic[g * 3 + 2] : conic[g * 3 + 2] + 0.25f;
            const float det = fmaf(a, c, -(b * b));
            const float t3 = dv * (du * (b + b));
            const float t4 = fmaf(du, du * c, -t3);
            const float num = fmaf(dv, dv * a, t4);
            const float mh = num / det;
            float alpha = 0.0f;
            if (mh > 0.0f) alpha = exp2f((-0.5f * mh) * 1.4426950216293334961f) * opacity[g];
            if (uncertain != NULL && fabs((double)alpha - 0.00392156862) <= 3e-5 * 0.00392156862) near = 1;
            if (near && uncertain != NULL) uncertain[g] += 1;
            if (done || (double)alpha < 0.00392156862) continue;
            const float w = (float)((double)alpha * (1.0 - (double)A));
            sum[g] += (double)w;
            if (w > wmax[g]) wmax[g] = w;
            count[g] += 1;
            A = A + w;
            ++nb;
        }
        A_out[pix] = A;
        nblend[pix] = nb;
    }
}
