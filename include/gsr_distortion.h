/* gsr_distortion.h — radial-tangential lens distortion in the fused per-gaussian stages (libgsr_distortion.so).
 *
 * COLMAP's OPENCV model (OpenCV's 5-coefficient model; FULL_OPENCV with k4 = k5 = k6 = 0) replaces the pinhole
 * projection of gsr_preprocess_forward / _backward and gsr_batch_preprocess_backward.  With the camera-frame position
 * p = (x, y, z), a = x / z, b = y / z and s = a^2 + b^2:
 *
 *     radial = 1 + k1 s + k2 s^2 + k3 s^3,
 *     a_d = a radial + 2 p1 a b + p2 (s + 2 a^2),   b_d = b radial + p1 (s + 2 b^2) + 2 p2 a b,
 *     u = fx a_d + cx,  v = fy b_d + cy
 *
 * fx fy cx cy come from K as in the pinhole path.  The 2-D covariance uses J = d(u, v) / dp at the mean.  A gaussian
 * with s >= r2_max (gsr_distortion_r2_max), where the radial model folds back, is culled, in addition to the near /
 * far / padding rules.  Depth keys and the depth map keep camera-frame z.
 *
 * Every entry point takes the arguments of its pinhole counterpart (gsr_b200.h, gsr_batch.h) plus `distortion`: device
 * memory holding GSR_DISTORTION_CONSTS fp32 values per view, {k1, k2, p1, p2, k3, r2_max}; C consecutive groups for
 * the batched backward.  Return codes are those of gsr_b200.h.
 */
#ifndef GSR_DISTORTION_H
#define GSR_DISTORTION_H

#include <stddef.h>
#include <stdint.h>

#define GSR_DISTORTION_CONSTS 6

#ifdef __cplusplus
extern "C" {
#endif

/* The smallest positive root s of 1 + 3 k1 s + 5 k2 s^2 + 7 k3 s^3, the derivative of r radial(r^2) in s = r^2, or
 * +inf when there is none: found in fp64 and rounded down to fp32.  k: 5 host floats {k1, k2, p1, p2, k3}; the
 * tangential p1 p2 do not enter the limit (COLMAP's are of order 1e-3).  NaN for a NULL or non-finite k. */
float gsr_distortion_r2_max(const float* k);

int gsr_distortion_preprocess_forward(int mode, int N, int n_sh_rest, const float* xyz, const float* xyz_camera_frame,
                                      int cam_first, const float* quaternion, const float* scale,
                                      const float* opacity_logit, const float* filter3d, const float* rgb_dc,
                                      const float* sh_rest, const float* camera_T_world, const float* K,
                                      const float* camera_centre, int H, int W, float near_thresh, float far_thresh,
                                      float cull_mask_padding, float mh_dist, uint32_t depth_base, float* records,
                                      uint32_t* depth_key, uint8_t* visible, uint64_t* scan, uint64_t* tile_mask,
                                      uint32_t* tile_win, void* temp, size_t temp_bytes, const float* distortion,
                                      void* stream);

int gsr_distortion_preprocess_backward(int mode, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                                       const float* scale, const float* opacity_logit, const float* filter3d,
                                       const float* camera_T_world, const float* K, const float* camera_centre,
                                       const uint8_t* visible, const float* grad_rows, int use_rows_uv,
                                       const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                       float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                                       float* g_sh_rest, const float* distortion, void* stream);

int gsr_distortion_batch_preprocess_backward(int mode, int C, int N, int n_sh_rest, const float* xyz,
                                             const float* quaternion, const float* scale, const float* opacity_logit,
                                             const float* filter3d, const float* camera_T_world, const float* K,
                                             const float* camera_centre, const uint8_t* visible,
                                             const float* grad_rows, int use_rows_uv, const float* grad_uv_compact,
                                             const uint64_t* scan, float* g_xyz, float* g_quaternion, float* g_scale,
                                             float* g_opacity_logit, float* g_rgb_dc, float* g_sh_rest,
                                             const float* distortion, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* GSR_DISTORTION_H */
