/* absgrad_oracle.c — CPU oracle of the absolute screen-space gradients of the fused rasterizer (absgrad=True).
 *
 * TEST INFRASTRUCTURE ONLY (tests/absgrad_oracle.py).  Compiled together with oracle/gsr_oracle.c, whose tile
 * renderer's backward recurrence it repeats for precomputed colours (n_sh == 1), with optional upstream gradients on
 * the depth and alpha maps as in tests/depth_alpha_oracle.c.  Per gaussian, next to the signed sums g_uv of the
 * per-pixel gradients on its projected mean, it returns the sums of their absolute values
 *   a_uv = sum_p |d <G_p, out_p> / d uv|   (AbsGS)
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mfma -shared -fPIC -I<repo>/oracle absgrad_oracle.c -lm
 */
#include "gsr_oracle.c"

#define REAL float
#define SUF(x) x##_f32
#define FAST 1
#define FMA(a, b, c) fmaf((a), (b), (c))
#define FASTEXP(a) exp2f((a) * 1.4426950216293334961f)
#include "absgrad_oracle_body.inc"
#undef REAL
#undef SUF
#undef FAST
#undef FMA
#undef FASTEXP

#define REAL double
#define SUF(x) x##_f64
#define FAST 0
#define FMA(a, b, c) fma((a), (b), (c))
#define FASTEXP(a) exp(a)
#include "absgrad_oracle_body.inc"
#undef REAL
#undef SUF
#undef FAST
#undef FMA
#undef FASTEXP
