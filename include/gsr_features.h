/* gsr_features.h — C ABI of the feature-channel tile kernels (libgsr_features.so, csrc/gsr_features.cu).
 * Conventions of include/gsr_b200.h: device pointers, int status (0 = ok, a cudaError_t value, or GSR_ERR_BAD_ARG),
 * `stream` a cudaStream_t.
 *
 * The kernels blend an arbitrary per-gaussian feature vector with the colour's blend weights:
 *   feature_map[p, c] = sum_i w_i * F[i, c],  w_i = T_i * alpha_i,
 * over exactly the splats, in exactly the order and with exactly the floats w_i of the colour forward
 * (gsr_render_forward_gather on the same records and pair list), including the saturation early-out and the pixels
 * the colour forward recomputes exactly.  There is no background term.
 *
 * features: [N, feature_stride] floats, 16-byte aligned, feature_stride a multiple of 4 with D <= feature_stride <
 * D + 4 (the columns from D on are padding and must be 0).  The kernels process the channels in chunks of 4, one
 * grid z index per chunk, every chunk walking the tile's pair list again.
 * feature_map / grad_feature_map: [H, W, D].
 *
 * The pair list is given as in gsr_render_forward_gather: exactly one of keys_sorted (gaussian id in the low id_bits)
 * and ids_sorted.
 *
 * GSR_ERR_BAD_ARG, before any launch, for: H or W < 1, D < 1, a feature_stride that is not such a stride, a NULL or
 * misaligned pointer, and not exactly one id source. */
#ifndef GSR_FEATURES_H
#define GSR_FEATURES_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* feature_map [H, W, D] = the blend of the features (every pixel written). */
int gsr_render_features_forward(const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                                const int32_t* ids_sorted, const int32_t* ranges, int H, int W, const float* features,
                                int feature_stride, int D, float* feature_map, void* stream);

/* Back to front from the colour forward's n_per_pixel (n_in) and final transmittance weight (w_in), with its
 * contribution masks when it recorded them (NULL: the candidate lists are rebuilt from the footprints).  Adds
 *   grad_features [N, feature_stride] += sum_p w_ip * G[p, c]          (16-byte aligned; padding columns get 0)
 * and the feature loss's part of d alpha, through opacity, uv and conic, into the interleaved gradient rows
 * grad_rows [N, 12] (rgb3 opacity | uv2 conic0 conic1 | conic2 ...; slots 3..8 are added to, the others untouched),
 * the rows gsr_render_backward_gather fills.  Both are accumulated into, never cleared. */
int gsr_render_features_backward(const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                                 const int32_t* ids_sorted, const int32_t* ranges, int H, int W, const int32_t* n_in,
                                 const float* w_in, const float* features, int feature_stride, int D,
                                 const float* grad_feature_map, float* grad_features, float* grad_rows,
                                 const uint32_t* contribution_masks, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GSR_FEATURES_H */
