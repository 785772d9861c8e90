/* gsr_shutter.h — rolling-shutter cameras in the fused per-gaussian stages (libgsr_shutter.so, csrc/gsr_shutter.cu).
 *
 * T = camera_T_world is the pose of the image's middle line; shutter_xi holds, per view, a twist xi = (rho, omega)
 * (6 fp32 values, the convention of pose.se3_exp): the camera's motion over the whole readout, applied on the left,
 *
 *     T(tau) = se3_exp((tau - 1/2) xi) T,   tau in [0, 1] the readout time of a line.
 *
 * readout: GSR_READOUT_* below, the line time r(u) of an image point (pixel centres at integer coordinates; H >= 2,
 * or W >= 2 for the horizontal readouts).  Each gaussian is projected at its own line's time tau* = clamp(r(u(tau*)),
 * 0, 1), and its covariance is the local affine map of x -> u at that time, A J W Sigma W^T J^T A^T with
 * A = I + f e^T / (1 - lambda), f = du/dtau, lambda = e^T f (A = I where tau* is clamped).  A gaussian with
 * lambda >= 3/4 or a fixed-point residual above 2^-20 is culled, in addition to the near / far / padding / lens rules.
 * xi = 0 gives the records of gsr_preprocess_forward (or the lens's) bit for bit.  DESIGN.md 3.24.
 *
 * Every entry point takes the arguments of its counterpart without a shutter — gsr_preprocess_forward (gsr_b200.h),
 * gsr_preprocess_backward, gsr_batch_preprocess_backward (gsr_batch.h) or the lens's (gsr_fisheye.h,
 * gsr_distortion.h), with `lens` and lens_consts as in gsr_pose.h — plus the twists, the readout and the image size.
 * The backward entry points take g_pose and g_xi, both NULL or both given: given, they also write view c's gradient
 * on camera_T_world (16 floats, last row 0) and on xi (6 floats), reduced in a fixed order (one partial per CTA in
 * temp, at least gsr_shutter_temp_bytes(C, N) bytes, then an fp64 sum), so the same rows give the same bits and view
 * c of the batched entry point equals the single-view entry point on view c's rows.  Return codes are those of
 * gsr_b200.h; an unknown readout or lens, or H (W) < 2 give GSR_ERR_BAD_ARG.
 */
#ifndef GSR_SHUTTER_H
#define GSR_SHUTTER_H

#include <stddef.h>
#include <stdint.h>

#define GSR_READOUT_TOP_TO_BOTTOM 0 /* r = v / (H - 1) */
#define GSR_READOUT_BOTTOM_TO_TOP 1 /* r = 1 - v / (H - 1) */
#define GSR_READOUT_LEFT_TO_RIGHT 2 /* r = u / (W - 1) */
#define GSR_READOUT_RIGHT_TO_LEFT 3 /* r = 1 - u / (W - 1) */

#ifdef __cplusplus
extern "C" {
#endif

size_t gsr_shutter_temp_bytes(int C, int N);

int gsr_shutter_preprocess_forward(int lens, int mode, int N, int n_sh_rest, const float* xyz,
                                   const float* xyz_camera_frame, int cam_first, const float* quaternion,
                                   const float* scale, const float* opacity_logit, const float* filter3d,
                                   const float* rgb_dc, const float* sh_rest, const float* camera_T_world,
                                   const float* K, const float* camera_centre, int H, int W, float near_thresh,
                                   float far_thresh, float cull_mask_padding, float mh_dist, uint32_t depth_base,
                                   float* records, uint32_t* depth_key, uint8_t* visible, uint64_t* scan,
                                   uint64_t* tile_mask, uint32_t* tile_win, void* temp, size_t temp_bytes,
                                   const float* lens_consts, const float* shutter_xi, int readout, void* stream);

int gsr_shutter_preprocess_backward(int lens, int mode, int N, int n_sh_rest, const float* xyz,
                                    const float* quaternion, const float* scale, const float* opacity_logit,
                                    const float* filter3d, const float* camera_T_world, const float* K,
                                    const float* camera_centre, const uint8_t* visible, const float* grad_rows,
                                    int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                    float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                                    float* g_sh_rest, const float* lens_consts, const float* shutter_xi, int readout,
                                    int H, int W, float* g_pose, float* g_xi, void* temp, size_t temp_bytes,
                                    void* stream);

int gsr_shutter_batch_preprocess_backward(int lens, int mode, int C, int N, int n_sh_rest, const float* xyz,
                                          const float* quaternion, const float* scale, const float* opacity_logit,
                                          const float* filter3d, const float* camera_T_world, const float* K,
                                          const float* camera_centre, const uint8_t* visible, const float* grad_rows,
                                          int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan,
                                          float* g_xyz, float* g_quaternion, float* g_scale, float* g_opacity_logit,
                                          float* g_rgb_dc, float* g_sh_rest, const float* lens_consts,
                                          const float* shutter_xi, int readout, int H, int W, float* g_pose,
                                          float* g_xi, void* temp, size_t temp_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* GSR_SHUTTER_H */
