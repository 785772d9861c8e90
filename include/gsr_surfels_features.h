/* gsr_surfels_features.h — per-gaussian feature channels for 2-D Gaussian surfels (libgsr_surfels_features.so,
 * csrc/gsr_surfels_features.cu, DESIGN.md 3.27).  Conventions of include/gsr_b200.h: device pointers, int status
 * (0 = ok, a cudaError_t value, or GSR_ERR_BAD_ARG), `stream` a cudaStream_t.
 *
 * The kernels blend an arbitrary per-gaussian feature vector with the surfel colour's blend weights:
 *   feature_map[p, c] = sum_i w_i * F[i, c],  w_i = alpha_i (1 - A_i),
 * over exactly the surfels, in exactly the order and with exactly the floats w_i of the surfel colour forward
 * (gsr_surfel_render_forward, or gsr_surfel_lens_render_forward along the same ray map) on the same records and pair
 * list: the same intersections, the 1/255 skip, and the pixel's last contributor `last` of that forward.  There is no
 * background term.
 *
 * rays: NULL for the pinhole (pixel rays (x, y, 1)), else the lens's ray map [H, W, 3] (gsr_surfel_rays); a pixel with
 * d = 0 gets 0 and takes no gradient.
 * features: [N, feature_stride] floats, 16-byte aligned, feature_stride a multiple of 4 with D <= feature_stride <
 * D + 4 (the columns from D on are padding and must be 0).  The channels are processed in chunks of 4, one grid z
 * index per chunk, every chunk walking the tile's pair list again.
 * feature_map / grad_feature_map: [H, W, D].
 *
 * The pair list is given as in gsr_surfel_render_forward: exactly one of keys_sorted (gaussian id in the low id_bits)
 * and ids_sorted.
 *
 * GSR_ERR_BAD_ARG, before any launch, for: H or W < 1, D < 1, a feature_stride that is not such a stride,
 * mh_dist <= 0, a NULL or misaligned pointer, and not exactly one id source. */
#ifndef GSR_SURFELS_FEATURES_H
#define GSR_SURFELS_FEATURES_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* feature_map [H, W, D] = the blend of the features (every pixel written). */
int gsr_surfel_render_features_forward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                                       const int32_t* ids_sorted, const int32_t* tile_ranges, int H, int W,
                                       float mh_dist, const float* rays, const int32_t* last, const float* features,
                                       int feature_stride, int D, float* feature_map, void* stream);

/* Back to front from the colour forward's final transmittance (totals[:, 0]) and last.  Adds
 *   grad_features [N, feature_stride] += sum_p w_ip * G[p, c]          (16-byte aligned; padding columns get 0)
 * and the feature loss's part of d alpha, through the intersection, into the surfel gradient rows
 * grad_rows [N, GSR_SURFEL_GRAD_FLOATS] of gsr_surfel_render_backward: dM (where rho = a^2 + b^2), d opacity and
 * d u_c, d v_c (where the low-pass filter decides); the colour, normal and p_z slots are untouched.  Both are
 * accumulated into, never cleared, and a field whose moment over a warp is zero is not written at all. */
int gsr_surfel_render_features_backward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                                        const int32_t* ids_sorted, const int32_t* tile_ranges, int H, int W,
                                        float mh_dist, const float* rays, const int32_t* last, const float* totals,
                                        const float* features, int feature_stride, int D,
                                        const float* grad_feature_map, float* grad_features, float* grad_rows,
                                        void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GSR_SURFELS_FEATURES_H */
