/* gsr_pose.h — the per-gaussian backward with the camera pose gradient (libgsr_pose.so, csrc/gsr_pose.cu).
 *
 * Every entry point does exactly what its counterpart without a pose gradient does — gsr_preprocess_backward
 * (gsr_b200.h), gsr_batch_preprocess_backward (gsr_batch.h) or their fisheye / distortion versions for `lens` — with
 * the same arguments and the same gaussian gradients, and also writes g_pose, the gradient on camera_T_world.
 * With T = camera_T_world, W = T[:3, :3], p = W x + t the camera-frame mean:
 *
 *     dL/dT[:3, :3] = sum_i (g_p,i x_i^T + J_i^T (2 G_i M_i Sigma_i)),   dL/dT[:3, 3] = sum_i g_p,i,   dL/dT[3, :] = 0
 *
 * over the gaussians the view sees; g_p the gradient on p, G the symmetric 2x2 gradient on the 2-D covariance
 * M Sigma M^T (after the antialiased terms), M = J W, Sigma the (filtered) world covariance.  The camera centre of the
 * SH view direction is held constant (no gradient through the view direction, as for xyz).
 *
 * Each CTA writes the fixed-order sum of its 128 gaussians' values into temp ([C, ceil(N / 128), 12] floats); a
 * second kernel adds a view's partials in fp64 in a fixed order and rounds once.  Given the same rows, two calls give
 * the same bits, and view c of the batched entry point equals the single-view entry point on view c's rows.
 *
 * lens: GSR_LENS_PINHOLE (lens_consts NULL), GSR_LENS_FISHEYE (GSR_FISHEYE_CONSTS floats per view, gsr_fisheye.h) or
 * GSR_LENS_DISTORTION (GSR_DISTORTION_CONSTS floats per view, gsr_distortion.h).  g_pose: C * 16 floats, view c's
 * [4, 4] gradient row-major (last row 0); written also when N == 0 (zeros).  temp: 16-byte aligned device scratch of
 * at least gsr_pose_temp_bytes(C, N) bytes.  GSR_ERR_BAD_ARG as for the counterparts, and for an unknown lens,
 * lens_consts not given exactly for a lens, a NULL g_pose or too little temp.  Return codes are those of gsr_b200.h.
 */
#ifndef GSR_POSE_H
#define GSR_POSE_H

#include <stddef.h>
#include <stdint.h>

#define GSR_LENS_PINHOLE 0
#define GSR_LENS_FISHEYE 1
#define GSR_LENS_DISTORTION 2

#ifdef __cplusplus
extern "C" {
#endif

size_t gsr_pose_temp_bytes(int C, int N);

int gsr_pose_preprocess_backward(int lens, int mode, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                                 const float* scale, const float* opacity_logit, const float* filter3d,
                                 const float* camera_T_world, const float* K, const float* camera_centre,
                                 const uint8_t* visible, const float* grad_rows, int use_rows_uv,
                                 const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                 float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                                 float* g_sh_rest, const float* lens_consts, float* g_pose, void* temp,
                                 size_t temp_bytes, void* stream);

int gsr_pose_batch_preprocess_backward(int lens, int mode, int C, int N, int n_sh_rest, const float* xyz,
                                       const float* quaternion, const float* scale, const float* opacity_logit,
                                       const float* filter3d, const float* camera_T_world, const float* K,
                                       const float* camera_centre, const uint8_t* visible, const float* grad_rows,
                                       int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan,
                                       float* g_xyz, float* g_quaternion, float* g_scale, float* g_opacity_logit,
                                       float* g_rgb_dc, float* g_sh_rest, const float* lens_consts, float* g_pose,
                                       void* temp, size_t temp_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* GSR_POSE_H */
