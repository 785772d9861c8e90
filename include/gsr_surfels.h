/* gsr_surfels.h — 2-D Gaussian surfels (2DGS) in the fused rasterizer (libgsr_surfels.so, csrc/gsr_surfels.cu).
 *
 * Gaussian i is a flat disk: position x, rotation R(q / |q|), tangent scales s_u = exp(scale[0]), s_v = exp(scale[1])
 * (scale[2] is not used).  With camera_T_world = [W | t] and K = [[fx,0,cx],[0,fy,cy],[0,0,1]]:
 *
 *   p = W x + t,  Rc = W R,  M = K [ s_u Rc[:,0] | s_v Rc[:,1] | p ]   (rows M0 M1 M2)
 *
 * and the surfel point (a, b) images at the homogeneous pixel M (a, b, 1)^T.  Per pixel (x, y) (pixel centres at
 * integer coordinates) the ray meets the surfel at (a, b) = (c0, c1) / c2, c = (x M2 - M0) x (y M2 - M1);
 * rho = min(a^2 + b^2, 2 |(x, y) - (u_c, v_c)|^2) (the second term is 2DGS's object-space low-pass filter),
 * alpha = min(0.99, sigmoid(o) exp(-rho / 2)) where rho <= mh_dist^2.  Blending follows the colour renderer (skip
 * alpha < 1/255, stop once the accumulated alpha exceeds 0.9999, background where it ends below 0.999).  DESIGN.md 3.25.
 *
 * All pointers are device pointers, stream is a cudaStream_t, and every entry point returns 0, a cudaError_t, or
 * GSR_ERR_BAD_ARG (gsr_b200.h) before any launch.
 */
#ifndef GSR_SURFELS_H
#define GSR_SURFELS_H

#include <stddef.h>
#include <stdint.h>

/* The surfel record the tile kernels read, one per gaussian, 16-byte aligned:
 *   u_c v_c opacity p_z | M00 M01 M02 M10 | M11 M12 M20 M21 | M22 r g b | n_x n_y n_z 0
 * (u_c, v_c) the pinhole projection of p (the bits gsr_preprocess_forward gives uv), opacity = sigmoid(o), colour the
 * SH colour at the centre's view direction, n = Rc[:,2] turned towards the camera. */
#define GSR_SURFEL_REC_FLOATS 20
/* The gradient row the tile backward accumulates, one per gaussian, 16-byte aligned:
 *   dM00..dM22 (9) | d opacity | d r g b | d n (3) | d u_c d v_c | d p_z | 0
 * d p_z: the depth gradient of the pixels where the fallback (rho = rho2) supplies the depth p_z. */
#define GSR_SURFEL_GRAD_FLOATS 20

#ifdef __cplusplus
extern "C" {
#endif

size_t gsr_surfel_temp_bytes(int N);

/* Per-gaussian forward.  The inputs and the culling follow gsr_preprocess_forward (xyz_camera_frame / cam_first,
 * camera_centre [3] required when n_sh_rest > 0); a surfel is also culled when its cutoff disk a^2 + b^2 <= mh_dist^2
 * does not lie in front of the camera: p_z <= 0 or mh_dist^2 (M20^2 + M21^2) >= M22^2.  Outputs, indexed by gaussian:
 *   surfels [N, GSR_SURFEL_REC_FLOATS], bin_records [N, 12]: the 48-byte record of gsr_b200.h that gsr_emit_keys /
 *   gsr_emit_pairs read, with (R_U, R_V) = (u_c, v_c) and R_A, R_B2 = 0, R_C an axis-aligned ellipse around (u_c, v_c)
 *   that contains every pixel a surfel can reach; depth_key, visible, scan, tile_mask, tile_win as in
 *   gsr_preprocess_forward (tile_mask / tile_win both or neither).  temp: gsr_surfel_temp_bytes(N) bytes.
 *   mh_dist must be > 0. */
int gsr_surfel_preprocess_forward(int N, int n_sh_rest, const float* xyz, const float* xyz_camera_frame, int cam_first,
                                  const float* quaternion, const float* scale, const float* opacity_logit,
                                  const float* rgb_dc, const float* sh_rest, const float* camera_T_world,
                                  const float* K, const float* camera_centre, int H, int W, float near_thresh,
                                  float far_thresh, float cull_mask_padding, float mh_dist, uint32_t depth_base,
                                  float* surfels, float* bin_records, uint32_t* depth_key, uint8_t* visible,
                                  uint64_t* scan, uint64_t* tile_mask, uint32_t* tile_win, void* temp,
                                  size_t temp_bytes, void* stream);

/* Tile forward through the sorted pair list (keys_sorted with the gaussian id in its low id_bits, or ids_sorted;
 * exactly one non-NULL) and tile_ranges [n_tiles + 1].  Outputs [H,W,k]: image (3), depth (1), alpha (1), normal (3),
 * distortion (1); and for the backward last [H,W] (position in the pair list of the pixel's last contributor, -1 for
 * none) and totals [H,W,3] (the final transmittance as the product of the contributors' 1 - alpha, sum w m,
 * sum w m^2).  m = m_scale (1 - near / z), m_scale = far / (far - near) (1 for an infinite far). */
int gsr_surfel_render_forward(const float* surfels, const uint64_t* keys_sorted, int id_bits, const int32_t* ids_sorted,
                              const int32_t* tile_ranges, const float* background_rgb, int H, int W, float near_thresh,
                              float m_scale, float mh_dist, float* image, float* depth, float* alpha, float* normal,
                              float* distortion, int32_t* last, float* totals, void* stream);

/* Tile backward: the upstream gradients of the five maps (each [H,W,k], zeros where a map has no gradient) and the
 * forward's alpha, last and totals -> grad_rows [N, GSR_SURFEL_GRAD_FLOATS], zero-filled by the caller, accumulated
 * into with one atomic per warp and field. */
int gsr_surfel_render_backward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                               const int32_t* ids_sorted, const int32_t* tile_ranges, const float* background_rgb,
                               int H, int W, float near_thresh, float m_scale, float mh_dist, const float* alpha,
                               const int32_t* last, const float* totals, const float* grad_image,
                               const float* grad_depth, const float* grad_alpha, const float* grad_normal,
                               const float* grad_distortion, float* grad_rows, void* stream);

/* uv.grad of the M visible gaussians vis_idx [M]: d loss / d delta, delta a pixel-space translation of the whole
 * footprint (M <- [[1,0,dx],[0,1,dy],[0,0,1]] M): (sum_j dM0j M2j + d u_c, sum_j dM1j M2j + d v_c) -> uv_grad [M,2]. */
int gsr_surfel_uv_grad(int M, const int32_t* vis_idx, const float* surfels, const float* grad_rows, float* uv_grad,
                       void* stream);

/* Per-gaussian backward: grad_rows -> the parameter gradients (g_sh_rest NULL when n_sh_rest == 0; g_scale[:,2] = 0;
 * zero rows for culled gaussians).  grad_uv_compact [M,2] (NULL: none), rank from the forward's scan: a gradient on the
 * returned uv.  When uv_grad_emitted is 1 it holds gsr_surfel_uv_grad's values plus what the caller added, else only
 * what the caller added; the caller's part goes to the centre's projection.  The colour's view direction is held
 * constant, as in gsr_preprocess_backward. */
int gsr_surfel_preprocess_backward(int N, int n_sh_rest, const float* xyz, const float* quaternion, const float* scale,
                                   const float* opacity_logit, const float* camera_T_world, const float* K,
                                   const float* camera_centre, const uint8_t* visible, const float* surfels,
                                   const float* grad_rows, const float* grad_uv_compact, const uint64_t* scan,
                                   int uv_grad_emitted, float* g_xyz, float* g_quaternion, float* g_scale,
                                   float* g_opacity_logit, float* g_rgb_dc, float* g_sh_rest, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* GSR_SURFELS_H */
