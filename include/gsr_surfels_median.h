/* gsr_surfels_median.h — the median depth of 2-D Gaussian surfels (libgsr_surfels_median.so,
 * csrc/gsr_surfels_median.cu, DESIGN.md 3.28).  Conventions of include/gsr_b200.h: device pointers, int status
 * (0 = ok, a cudaError_t value, or GSR_ERR_BAD_ARG), `stream` a cudaStream_t.
 *
 * The median contributor of a pixel is the last of the surfel colour forward's contributors i (gsr_surfel_render_forward,
 * or gsr_surfel_lens_render_forward along the same ray map, on the same records and pair list: the same intersections,
 * the 1/255 skip, the same order, up to the pixel's last contributor `last`) whose transmittance in front of it,
 * 1 - A_i in fp32 with the colour forward's A (A_1 = 0, A <- A + alpha (1 - A)), is above 0.5.  This is 2DGS's
 * `if (T > 0.5) median = depth`.  Every pixel with a contributor has one.
 *
 *   median [H, W]     the camera z of that contributor's ray-surfel intersection (the z the depth map blends: the
 *                     intersection where rho = a^2 + b^2, else p_z);
 *   median_id [H, W]  its gaussian index.
 * A pixel with no contributor (a fisheye pixel beyond theta_max among them) gets median 0 and id -1.
 *
 * rays: NULL for the pinhole (pixel rays (x, y, 1)), else the lens's ray map [H, W, 3] (gsr_surfel_rays).
 * The pair list is given as in gsr_surfel_render_forward: exactly one of keys_sorted (gaussian id in the low id_bits)
 * and ids_sorted.
 *
 * GSR_ERR_BAD_ARG, before any launch, for: H or W < 1, mh_dist <= 0, a NULL or misaligned pointer, and not exactly
 * one id source. */
#ifndef GSR_SURFELS_MEDIAN_H
#define GSR_SURFELS_MEDIAN_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* median [H, W] and median_id [H, W] (every pixel written); each pixel walks its tile's pair list up to its crossing
 * of 0.5 or its `last`. */
int gsr_surfel_render_median_forward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                                     const int32_t* ids_sorted, const int32_t* tile_ranges, int H, int W,
                                     float mh_dist, const float* rays, const int32_t* last, float* median,
                                     int32_t* median_id, void* stream);

/* Adds d loss / d median[p] of every pixel into the gradient row of its surfel median_id[p] (rows
 * [N, GSR_SURFEL_GRAD_FLOATS] of gsr_surfel_render_backward), through z only: into dM where rho = a^2 + b^2 (through
 * (a, b) and M2 . (a, b, 1)), into d p_z where the low-pass filter decides.  No other slot is written, and a slot whose
 * sum over a warp is zero is not written at all (a zero gradient leaves the rows' bits unchanged).  Accumulated into,
 * never cleared. */
int gsr_surfel_render_median_backward(const float* surfels, int H, int W, float mh_dist, const float* rays,
                                      const int32_t* median_id, const float* grad_median, float* grad_rows,
                                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GSR_SURFELS_MEDIAN_H */
