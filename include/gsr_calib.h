/* gsr_calib.h — the per-gaussian backward with the camera pose, intrinsics and lens-coefficient gradients
 * (libgsr_calib.so: csrc/gsr_pose.cu compiled with GSR_POSE_CAMERA).
 *
 * Every entry point does exactly what its pose counterpart in gsr_pose.h does, with the same arguments, the same
 * gaussian gradients and the same g_pose bits, and also writes the gradients on the intrinsics and the lens
 * coefficients.  Every model projects as u = fx a_d(p) + cx, v = fy b_d(p) + cy; with g_uv the complete gradient on
 * (u, v) and gJ the gradient on J = d(u, v)/dp:
 *
 *     dL/dfx = sum_i (g_u a_d + sum_j gJ_0j J_0j / fx),  dL/dcx = sum_i g_u  (fy, cy likewise with row 1)
 *     dL/dk  = sum_i (g_uv . d(u, v)/dk + sum_ij gJ_ij dJ_ij/dk)
 *
 * over the gaussians the view sees.  The reduction is the pose's (fixed order per CTA, fp64 over the partials, one
 * rounding), so the same rows give the same bits and view c of the batched entry point equals the single-view entry
 * point on view c's rows.
 *
 * lens: GSR_LENS_* of gsr_pose.h, lens_consts as there.  g_pose: C * 16 floats as in gsr_pose.h.  g_intrinsics: C * 4
 * floats, view c's (fx, fy, cx, cy).  g_lens: C * n floats (n = 4 fisheye k1..k4, 5 distortion k1 k2 p1 p2 k3, in the
 * order of the lens constants), NULL for the pinhole.  The cull limits and the skew get no gradient.  temp: 16-byte
 * aligned device scratch of at least gsr_camera_temp_bytes(lens, C, N) bytes ([C, ceil(N / 128), 16 | 20 | 24]
 * floats: 12 pose values, 4 intrinsics, n coefficients, zero padding).  GSR_ERR_BAD_ARG as for the pose entry points,
 * and for a NULL g_intrinsics or g_lens not given exactly for a lens.  Return codes are those of gsr_b200.h.
 */
#ifndef GSR_CALIB_H
#define GSR_CALIB_H

#include <stddef.h>
#include <stdint.h>

#include "gsr_pose.h"

#ifdef __cplusplus
extern "C" {
#endif

size_t gsr_camera_temp_bytes(int lens, int C, int N);

int gsr_camera_preprocess_backward(int lens, int mode, int N, int n_sh_rest, const float* xyz,
                                   const float* quaternion, const float* scale, const float* opacity_logit,
                                   const float* filter3d, const float* camera_T_world, const float* K,
                                   const float* camera_centre, const uint8_t* visible, const float* grad_rows,
                                   int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                   float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                                   float* g_sh_rest, const float* lens_consts, float* g_pose, float* g_intrinsics,
                                   float* g_lens, void* temp, size_t temp_bytes, void* stream);

int gsr_camera_batch_preprocess_backward(int lens, int mode, int C, int N, int n_sh_rest, const float* xyz,
                                         const float* quaternion, const float* scale, const float* opacity_logit,
                                         const float* filter3d, const float* camera_T_world, const float* K,
                                         const float* camera_centre, const uint8_t* visible, const float* grad_rows,
                                         int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan,
                                         float* g_xyz, float* g_quaternion, float* g_scale, float* g_opacity_logit,
                                         float* g_rgb_dc, float* g_sh_rest, const float* lens_consts, float* g_pose,
                                         float* g_intrinsics, float* g_lens, void* temp, size_t temp_bytes,
                                         void* stream);

#ifdef __cplusplus
}
#endif

#endif /* GSR_CALIB_H */
