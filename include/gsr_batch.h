/* gsr_batch.h — C ABI of the multi-view per-Gaussian kernels (libgsr_batch.so, csrc/gsr_batch.cu), behind
 * rasterize_batch: C cameras of one scene rendered in one call, with one parameter gradient summed over the views.
 * Conventions of include/gsr_b200.h: device pointers, int status (0 = ok, a cudaError_t value, GSR_ERR_BAD_ARG or
 * GSR_ERR_UNSUPPORTED), `stream` a cudaStream_t.  No entry point synchronises.
 *
 * Per-view arrays are stacked view-major: camera_T_world [C,4,4], K [C,3,3], camera_centre [C,3], visible [C,N],
 * scan [C,N] (view c's packed inclusive scan of gsr_preprocess_forward: (visible rank << 32) | pair count),
 * grad_rows [C,N,12] (view c's interleaved gradient rows of gsr_render_backward_gather).
 *
 * GSR_ERR_BAD_ARG, before any launch, for: C < 1, N < 0, unknown mode bits, a filter3d that is given without
 * GSR_MODE_FILTER3D or missing with it; and, when N > 0, a NULL pointer, a grad_rows that is not 16-byte aligned,
 * grad_uv_compact without scan, and g_sh_rest not given exactly when n_sh_rest > 0.  N == 0 launches nothing. */
#ifndef GSR_BATCH_H
#define GSR_BATCH_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* The per-Gaussian backward of C views in one pass: every gaussian's parameters are read once, view c's VJP
 * (exactly gsr_preprocess_backward's arithmetic on view c's rows, constants and mode) is formed for every view that
 * sees the gaussian, and the views' gradients are added in view order, one rounded fp32 add per view:
 *   g = 0; g += g_0; g += g_1; ...
 * which is bit for bit the sum of C gsr_preprocess_backward outputs added in view order, up to the sign of zero.
 * Outputs (xyz [N,3], quaternion [N,4], scale [N,3], opacity [N], rgb_dc [N,3], sh_rest [N,3,n_sh_rest]) are written
 * once, invisible gaussians get 0.
 * grad_uv_compact [sum_c M_c, 2] (optional): gradient on the compact uv of all views, view c's rows after those of
 * views 0..c-1 (M_c from scan[c, N-1] >> 32); added to the rows' uv gradient, or with use_rows_uv == 0 replacing it. */
int gsr_batch_preprocess_backward(int mode, int C, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                                  const float* scale, const float* opacity_logit, const float* filter3d,
                                  const float* camera_T_world, const float* K, const float* camera_centre,
                                  const uint8_t* visible, const float* grad_rows, int use_rows_uv,
                                  const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                  float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                                  float* g_sh_rest, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GSR_BATCH_H */
