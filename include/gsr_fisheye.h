/* gsr_fisheye.h — fisheye cameras in the fused per-gaussian stages (libgsr_fisheye.so).
 *
 * COLMAP's OPENCV_FISHEYE (Kannala-Brandt) model replaces the pinhole projection of gsr_preprocess_forward /
 * _backward and gsr_batch_preprocess_backward.  With the camera-frame position p = (x, y, z):
 *
 *     rho = sqrt(x^2 + y^2),  theta = atan2(rho, z),
 *     theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8),
 *     u = fx (theta_d / rho) x + cx,  v = fy (theta_d / rho) y + cy      (theta_d / rho -> 1 / z as rho -> 0)
 *
 * fx fy cx cy come from K as in the pinhole path.  The 2-D covariance uses J = d(u, v) / dp at the mean.  A gaussian
 * with theta >= theta_max (gsr_fisheye_theta_max) is culled, in addition to the near / far / padding rules.  Depth
 * keys and the depth map keep camera-frame z.
 *
 * Every entry point takes the arguments of its pinhole counterpart (gsr_b200.h, gsr_batch.h) plus `fisheye`: device
 * memory holding GSR_FISHEYE_CONSTS fp32 values per view, {k1, k2, k3, k4, theta_max}; C consecutive groups for the
 * batched backward.  Return codes are those of gsr_b200.h.
 */
#ifndef GSR_FISHEYE_H
#define GSR_FISHEYE_H

#include <stddef.h>
#include <stdint.h>

#define GSR_FISHEYE_CONSTS 5

#ifdef __cplusplus
extern "C" {
#endif

/* The first theta in (0, pi/2) where d theta_d / d theta = 1 + 3 k1 t + 5 k2 t^2 + 7 k3 t^3 + 9 k4 t^4 (t = theta^2)
 * reaches 0, or pi/2 when there is none: found in fp64 and rounded down to fp32.  k: 4 host floats.  NaN for a NULL
 * or non-finite k. */
float gsr_fisheye_theta_max(const float* k);

int gsr_fisheye_preprocess_forward(int mode, int N, int n_sh_rest, const float* xyz, const float* xyz_camera_frame,
                                   int cam_first, const float* quaternion, const float* scale,
                                   const float* opacity_logit, const float* filter3d, const float* rgb_dc,
                                   const float* sh_rest, const float* camera_T_world, const float* K,
                                   const float* camera_centre, int H, int W, float near_thresh, float far_thresh,
                                   float cull_mask_padding, float mh_dist, uint32_t depth_base, float* records,
                                   uint32_t* depth_key, uint8_t* visible, uint64_t* scan, uint64_t* tile_mask,
                                   uint32_t* tile_win, void* temp, size_t temp_bytes, const float* fisheye,
                                   void* stream);

int gsr_fisheye_preprocess_backward(int mode, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                                    const float* scale, const float* opacity_logit, const float* filter3d,
                                    const float* camera_T_world, const float* K, const float* camera_centre,
                                    const uint8_t* visible, const float* grad_rows, int use_rows_uv,
                                    const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                    float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                                    float* g_sh_rest, const float* fisheye, void* stream);

int gsr_fisheye_batch_preprocess_backward(int mode, int C, int N, int n_sh_rest, const float* xyz,
                                          const float* quaternion, const float* scale, const float* opacity_logit,
                                          const float* filter3d, const float* camera_T_world, const float* K,
                                          const float* camera_centre, const uint8_t* visible, const float* grad_rows,
                                          int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan,
                                          float* g_xyz, float* g_quaternion, float* g_scale, float* g_opacity_logit,
                                          float* g_rgb_dc, float* g_sh_rest, const float* fisheye, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* GSR_FISHEYE_H */
