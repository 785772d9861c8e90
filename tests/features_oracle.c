/* features_oracle.c — CPU oracle of the feature maps of the fused rasterizer (rasterize(..., features=F)).
 *
 * TEST INFRASTRUCTURE ONLY (tests/features_oracle.py).  Compiled together with oracle/gsr_oracle.c, whose tile
 * renderer it restates for an arbitrary per-gaussian feature vector F [G,D] in place of the colour: the same walk,
 * weights, early-out and backward recurrence, and no background term.
 *   forward:  fmap[p,c] <- fma(w_i, F[i,c], fmap[p,c]) front to back
 *   backward: d_alpha += sum_c (F[i,c]*weight - acc_c*r) * G[p,c] ;  g_F[i,c] += alpha*weight*G[p,c] ;
 *             acc_c += F[i,c]*alpha*weight
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mfma -shared -fPIC -I<repo>/oracle features_oracle.c -lm
 */
#include <stdlib.h>

#include "gsr_oracle.c"

#define REAL float
#define SUF(x) x##_f32
#define FAST 1
#define FMA(a, b, c) fmaf((a), (b), (c))
#define FASTEXP(a) exp2f((a) * 1.4426950216293334961f)
#include "features_oracle_body.inc"
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
#include "features_oracle_body.inc"
#undef REAL
#undef SUF
#undef FAST
#undef FMA
#undef FASTEXP
