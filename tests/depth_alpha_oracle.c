/* depth_alpha_oracle.c — CPU oracle of the depth and alpha maps of the fused rasterizer (render_depth_alpha=True).
 *
 * TEST INFRASTRUCTURE ONLY (tests/depth_alpha_oracle.py).  Compiled together with oracle/gsr_oracle.c, whose tile
 * renderer it extends for precomputed colours (n_sh == 1): the same walk, weights, early-out and backward recurrence,
 * with two more outputs per pixel
 *   alpha = A, the accumulated sum of w_i before any background;
 *   depth = D, D <- fma(w_i, z_i, D) front to back (z_i = camera-frame z), no background term;
 * and in the backward two more back-to-front accumulators (no background initialisation)
 *   d_alpha += (z_i*weight - acc_d*r)*dD + (weight - acc_a*r)*dA
 *   g_z_i   += alpha*weight*dD
 *   acc_d   += z_i*alpha*weight ;  acc_a += alpha*weight
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mfma -shared -fPIC -I<repo>/oracle depth_alpha_oracle.c -lm
 */
#include "gsr_oracle.c"

#define REAL float
#define SUF(x) x##_f32
#define FAST 1
#define FMA(a, b, c) fmaf((a), (b), (c))
#define FASTEXP(a) exp2f((a) * 1.4426950216293334961f)
#include "depth_alpha_oracle_body.inc"
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
#include "depth_alpha_oracle_body.inc"
#undef REAL
#undef SUF
#undef FAST
#undef FMA
#undef FASTEXP
