/* gsr_bilagrid.h — per-image appearance correction with bilateral grids (libgsr_bilagrid.so, csrc/gsr_bilagrid.cu).
 *
 * Grids are G [N, 12, L, GY, GX] fp32, contiguous, one per training image.  For an image rgb [H, W, 3] with id n, pixel
 * (i, j) becomes
 *
 *     fx = (j + 0.5) / W (GX - 1),  fy = (i + 0.5) / H (GY - 1),  fz = clamp(0.299 r + 0.587 g + 0.114 b, 0, 1) (L - 1)
 *     a[12] = trilinear interpolation of G[n] at (fz, fy, fx), node indices clamped to the grid
 *     out = A[:, :3] rgb + A[:, 3],  A = a viewed as 3 x 4 row-major
 *
 * which is F.grid_sample(..., mode="bilinear", padding_mode="border", align_corners=True) followed by the affine.
 * The backward routes the gradient to rgb (directly and through the luminance guidance, zero where the luminance lies
 * outside (0, 1)) and to G.
 *
 * Images are C views rgb [C, H, W, 3] given as a base pointer and four element strides (C, H, W, channel), so any
 * layout is read in place.  ids: C int32 on the device, each in [0, N) (the caller checks them; a view whose id is out
 * of range is skipped).  out and grad_rgb are contiguous [C, H, W, 3].
 *
 * The grid gradient is deterministic: each (view, node, chunk of pixel rows, block of levels) is summed by one CTA in
 * a fixed order into temp; then each grid element forms each view's value as its chunks' sum in order and adds the
 * values of the views that use its grid in fp32 in view order.  Grids no view uses get exact zeros.
 *
 * TV: tv(G) = sum over the L, GY and GX axes of mean((G[..., k + 1, ...] - G[..., k, ...])^2), each mean over all N
 * grids.  The forward reduces in fp64 with a fixed-order finish on the device (no host sync) and writes one float;
 * the backward is one elementwise stencil scaled by the device scalar grad_tv.
 *
 * Every dimension must be >= 2 (C, N >= 1), L <= GSR_BILAGRID_MAX_L.  Return codes are those of gsr_b200.h.
 */
#ifndef GSR_BILAGRID_H
#define GSR_BILAGRID_H

#include <stddef.h>
#include <stdint.h>

#define GSR_BILAGRID_MAX_L 256

#ifdef __cplusplus
extern "C" {
#endif

int gsr_bilagrid_slice_forward(int C, int H, int W, const float* rgb, const int64_t* rgb_strides_host,
                               const float* grids, int N, int L, int GY, int GX, const int32_t* ids, float* out,
                               void* stream);

/* temp: device scratch of at least gsr_bilagrid_slice_backward_temp_bytes(C, H, L, GY, GX) bytes (used only when
 * grad_grids is given).  grad_rgb [C, H, W, 3] and grad_grids [N, 12, L, GY, GX] may each be NULL (not computed);
 * grad_out is read through its four element strides. */
size_t gsr_bilagrid_slice_backward_temp_bytes(int C, int H, int L, int GY, int GX);
int gsr_bilagrid_slice_backward(int C, int H, int W, const float* rgb, const int64_t* rgb_strides_host,
                                const float* grids, int N, int L, int GY, int GX, const int32_t* ids,
                                const float* grad_out, const int64_t* grad_out_strides_host, float* grad_rgb,
                                float* grad_grids, void* temp, size_t temp_bytes, void* stream);

/* temp: device scratch of at least gsr_bilagrid_tv_temp_bytes(N, L, GY, GX) bytes; out: one float on the device. */
size_t gsr_bilagrid_tv_temp_bytes(int N, int L, int GY, int GX);
int gsr_bilagrid_tv_forward(int N, int L, int GY, int GX, const float* grids, float* out, void* temp,
                            size_t temp_bytes, void* stream);
int gsr_bilagrid_tv_backward(int N, int L, int GY, int GX, const float* grids, const float* grad_tv,
                             float* grad_grids, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* GSR_BILAGRID_H */
