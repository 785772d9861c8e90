/* gsr_surfels_lens.h — 2-D Gaussian surfels through a lens (libgsr_surfels_lens.so, csrc/gsr_surfels_lens.cu).
 *
 * rasterize_surfels for COLMAP's OPENCV_FISHEYE (GSR_SURFEL_LENS_FISHEYE) and OPENCV (GSR_SURFEL_LENS_DISTORTION)
 * cameras (DESIGN.md 3.26).  Each pixel (x, y) has its own unit ray d, the lens inverted at the distorted normalised
 * point ((x - cx) / fx, (y - cy) / fy) on the lens's monotone branch (d = 0 where there is no preimage).  With
 * M' = [ s_u Rc[:,0] | s_v Rc[:,1] | p ] (rows M'0 M'1 M'2: gsr_surfels.h's M without K), the pixel meets the surfel at
 * (a, b) = (c0, c1) / c2, c = (d_x M'2 - d_z M'0) x (d_y M'2 - d_z M'1); rho, alpha, the blend, the depth and the
 * distortion term are gsr_surfels.h's.  The centre (u_c, v_c), the depth key and the near / far / padding / fold cull
 * are those of gsr_fisheye_preprocess_forward / gsr_distortion_preprocess_forward, bit for bit.
 *
 * lens_consts: device memory, {k1, k2, k3, k4, theta_max} (GSR_FISHEYE_CONSTS) or {k1, k2, p1, p2, k3, r2_max}
 * (GSR_DISTORTION_CONSTS), the limits from gsr_fisheye_theta_max / gsr_distortion_r2_max.  All pointers are device
 * pointers, stream is a cudaStream_t; every entry point returns 0, a cudaError_t, or GSR_ERR_BAD_ARG before any launch.
 */
#ifndef GSR_SURFELS_LENS_H
#define GSR_SURFELS_LENS_H

#include <stddef.h>
#include <stdint.h>

#define GSR_SURFEL_LENS_FISHEYE 1
#define GSR_SURFEL_LENS_DISTORTION 2

#ifdef __cplusplus
extern "C" {
#endif

/* The ray map rays [H, W, 3] (fp32 unit directions, 0 where the pixel has no ray), formed in fp64.  K [9] row-major. */
int gsr_surfel_rays(int lens, int H, int W, const float* K, const float* lens_consts, float* rays, void* stream);

/* gsr_surfel_preprocess_forward for the lens: the record holds M' in place of M, (u_c, v_c) the lens projection of p;
 * the binning ellipse contains the lens image of the cutoff disk (its points with a valid ray) and the low-pass disk. */
int gsr_surfel_lens_preprocess_forward(int lens, int N, int n_sh_rest, const float* xyz, const float* xyz_camera_frame,
                                       int cam_first, const float* quaternion, const float* scale,
                                       const float* opacity_logit, const float* rgb_dc, const float* sh_rest,
                                       const float* camera_T_world, const float* K, const float* camera_centre, int H,
                                       int W, float near_thresh, float far_thresh, float cull_mask_padding,
                                       float mh_dist, uint32_t depth_base, float* surfels, float* bin_records,
                                       uint32_t* depth_key, uint8_t* visible, uint64_t* scan, uint64_t* tile_mask,
                                       uint32_t* tile_win, void* temp, size_t temp_bytes, const float* lens_consts,
                                       void* stream);

/* gsr_surfel_render_forward / _backward along the ray map rays [H, W, 3]; the gradient rows hold dL/dM'. */
int gsr_surfel_lens_render_forward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                                   const int32_t* ids_sorted, const int32_t* tile_ranges, const float* background_rgb,
                                   int H, int W, float near_thresh, float m_scale, float mh_dist, const float* rays,
                                   float* image, float* depth, float* alpha, float* normal, float* distortion,
                                   int32_t* last, float* totals, void* stream);

int gsr_surfel_lens_render_backward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                                    const int32_t* ids_sorted, const int32_t* tile_ranges, const float* background_rgb,
                                    int H, int W, float near_thresh, float m_scale, float mh_dist, const float* rays,
                                    const float* alpha, const int32_t* last, const float* totals,
                                    const float* grad_image, const float* grad_depth, const float* grad_alpha,
                                    const float* grad_normal, const float* grad_distortion, float* grad_rows,
                                    void* stream);

/* uv.grad = J_n^-T g_n + g_c: g_n = (sum_j dM'0j M'2j, sum_j dM'1j M'2j) the gradient on a translation of the footprint
 * in the normalised plane, J_n = p_z d(u, v) / dp [:, :2] the lens Jacobian with respect to normalised coordinates at
 * the centre, g_c = (d u_c, d v_c) the low-pass filter's centre term. */
int gsr_surfel_lens_uv_grad(int lens, int M, const int32_t* vis_idx, const float* surfels, const float* grad_rows,
                            const float* K, const float* lens_consts, float* uv_grad, void* stream);

/* gsr_surfel_preprocess_backward for the lens: dL/dM' chains to the surfel without K, d(u_c, v_c) through the lens
 * Jacobian's transpose. */
int gsr_surfel_lens_preprocess_backward(int lens, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                                        const float* scale, const float* opacity_logit, const float* camera_T_world,
                                        const float* K, const float* camera_centre, const uint8_t* visible,
                                        const float* surfels, const float* grad_rows, const float* grad_uv_compact,
                                        const uint64_t* scan, int uv_grad_emitted, float* g_xyz, float* g_quaternion,
                                        float* g_scale, float* g_opacity_logit, float* g_rgb_dc, float* g_sh_rest,
                                        const float* lens_consts, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* GSR_SURFELS_LENS_H */
