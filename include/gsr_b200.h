/* gsr_b200.h — C ABI of the H100-native (sm_90a) Gaussian-splat rasterizer hot path.
 *
 * This is the drop-in boundary: every entry point below is what the reference's
 * pybind module `splat_cuda` (joeyan/gaussian_splatting, src/bindings.cpp:118-159)
 * binds for the rasterization path, restated as plain C: device pointers, sizes,
 * a stream handle, int status (0 = ok, otherwise a cudaError_t value, or
 * GSR_ERR_* below for argument errors).  No torch types cross this line.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host;
 *   - tensors are dense row-major with the shapes the reference uses;
 *   - `dtype` is GSR_F32 or GSR_F64 for the entry points the reference
 *     instantiates for both (its gradcheck tests run in fp64);
 *   - `stream` is a cudaStream_t passed as void*; nothing here synchronizes
 *     (the reference calls cudaDeviceSynchronize() in most wrappers, e.g.
 *     src/render.cu:421 — observationally equivalent for stream-ordered callers);
 *   - outputs are caller-allocated; gradient outputs of the render backward are
 *     ACCUMULATED into (caller zero-fills), exactly like the reference
 *     (splat_py/cuda_autograd_functions.py:195-198).
 */
#ifndef GSR_B200_H
#define GSR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSR_F32 0
#define GSR_F64 1

#define GSR_OK 0
#define GSR_ERR_BAD_ARG (-1)
#define GSR_ERR_UNSUPPORTED (-2)

/* floats per packed splat record consumed by the tile renderers (48 bytes) */
#define GSR_REC_FLOATS 12

/* Modes of the fused rasterizer, a bit mask: the `mode` of gsr_preprocess_forward / gsr_preprocess_backward and of
 * gsr_render_backward_gather, so a caller passes one mode word to every stage; each stage ignores the bits that do not
 * concern it.  The tile renderers run in depth/alpha mode when they are given the depth and alpha maps (forward) or
 * their upstream gradients (backward). */
#define GSR_MODE_DEPTH_ALPHA 1 /* gradient rows carry the render backward's camera-frame z gradient */
#define GSR_MODE_ANTIALIASED 2 /* opacity compensation for the renderer's 0.25 px^2 dilation */
#define GSR_MODE_ABSGRAD 4     /* gradient rows also carry sum over pixels of |d loss_p / d uv| (AbsGS) */
#define GSR_MODE_FILTER3D 8    /* Mip-Splatting's 3-D smoothing filter in the per-gaussian stages (gsr_filter3d) */

/* library identification: returns e.g. "gsr_b200 0.1 sm_90a" */
const char* gsr_version(void);

/* ------------------------------------------------------------------------
 * Per-Gaussian operators (one call == one reference binding)
 * ---------------------------------------------------------------------- */

/* camera_projection_cuda — src/bindings.cpp:35, src/projection.cu:21-54
 * xyz [N,3], K [3,3] -> uv [N,2] */
int gsr_camera_projection(int dtype, int N, const void* xyz, const void* K, void* uv, void* stream);

/* camera_projection_backward_cuda — src/bindings.cpp:37-42, src/projection_backward.cu:38-90
 * writes xyz_grad_in [N,3] (rows with z <= 0 are left untouched) */
int gsr_camera_projection_backward(int dtype, int N, const void* xyz, const void* K,
                                   const void* uv_grad_out, void* xyz_grad_in, void* stream);

/* compute_sigma_world_cuda — src/bindings.cpp:44-48, src/projection.cu:111-152
 * quaternion [N,4] wxyz, scale [N,3] log -> sigma_world [N,3,3] */
int gsr_compute_sigma_world(int dtype, int N, const void* quaternion, const void* scale,
                            void* sigma_world, void* stream);

/* compute_sigma_world_backward_cuda — src/bindings.cpp:50-56, src/projection_backward.cu:317-382 */
int gsr_compute_sigma_world_backward(int dtype, int N, const void* quaternion, const void* scale,
                                     const void* sigma_world_grad_out, void* quaternion_grad_in,
                                     void* scale_grad_in, void* stream);

/* compute_projection_jacobian_cuda — src/bindings.cpp:58, src/projection.cu:177-211
 * xyz [N,3] camera frame, K -> J [N,2,3] */
int gsr_compute_projection_jacobian(int dtype, int N, const void* xyz, const void* K, void* J,
                                    void* stream);

/* compute_projection_jacobian_backward_cuda — src/bindings.cpp:60-65, src/projection_backward.cu:122-166 */
int gsr_compute_projection_jacobian_backward(int dtype, int N, const void* xyz, const void* K,
                                             const void* jac_grad_out, void* xyz_grad_in, void* stream);

/* compute_conic_cuda — src/bindings.cpp:67-72, src/projection.cu:259-311
 * sigma_world [N,3,3], J [N,2,3], camera_T_world [4,4] -> conic [N,3] = [S00, S01+S10, S11] */
int gsr_compute_conic(int dtype, int N, const void* sigma_world, const void* J,
                      const void* camera_T_world, void* conic, void* stream);

/* compute_conic_backward_cuda — src/bindings.cpp:74-81, src/projection_backward.cu:473-550 */
int gsr_compute_conic_backward(int dtype, int N, const void* sigma_world, const void* J,
                               const void* camera_T_world, const void* conic_grad_out,
                               void* sigma_world_grad_in, void* J_grad_in, void* stream);

/* precompute_rgb_from_sh_cuda — src/bindings.cpp:93-98, src/precompute_sh.cu:113-250
 * xyz [N,3] world, sh_coeff [N,3,n_sh] (n_sh in {1,4,9,16}; n_sh==1 may be [N,3]),
 * camera_T_world [4,4] (only the translation column is read; the caller passes the
 * INVERSE pose, splat_py/rasterize.py:91-93) -> rgb [N,3] */
int gsr_precompute_rgb_from_sh(int dtype, int N, int n_sh, const void* xyz, const void* sh_coeff,
                               const void* camera_T_world, void* rgb, void* stream);

/* precompute_rgb_from_sh_backward_cuda — src/bindings.cpp:100-105, src/precompute_sh.cu:252-389
 * grad_rgb [N,3] -> grad_sh [N,3,n_sh] (no gradient to xyz, as in the reference) */
int gsr_precompute_rgb_from_sh_backward(int dtype, int N, int n_sh, const void* xyz,
                                        const void* camera_T_world, const void* grad_rgb,
                                        void* grad_sh, void* stream);

/* ------------------------------------------------------------------------
 * Tile binning: get_sorted_gaussian_list — src/bindings.cpp:83-91,
 * src/tile_culling.cu:244-340.  Split in two because the number of
 * (gaussian, tile) pairs P sizes the outputs: phase 1 counts and scans,
 * the host reads P = offsets[N], phase 2 emits, sorts and builds tile ranges.
 * ---------------------------------------------------------------------- */
size_t gsr_binning_count_temp_bytes(int N);
/* offsets: int32 [N+1], exclusive scan of tiles-per-gaussian (offsets[N] == P) */
int gsr_binning_count(int N, const float* uvs, const float* conic, int n_tiles_x, int n_tiles_y,
                      float mh_dist, int32_t* offsets, void* temp, size_t temp_bytes, void* stream);

size_t gsr_binning_sort_temp_bytes(int P);
/* xyz_camera_frame [N,3] (depth = column 2).  Outputs: sorted_gaussian_idx int32 [P] ordered by
 * (tile, depth, gaussian index); tile_ranges int32 [n_tiles+1] (reference: splat_start_end_idx_by_tile_idx) */
int gsr_binning_emit_sort(int N, int P, const float* uvs, const float* xyz_camera_frame,
                          const float* conic, int n_tiles_x, int n_tiles_y, float mh_dist,
                          const int32_t* offsets, int32_t* sorted_gaussian_idx, int32_t* tile_ranges,
                          void* temp, size_t temp_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Tile renderers, fp32 / precomputed-RGB fast path (N_SH == 1):
 * render_tiles_cuda / render_tiles_backward_cuda — src/bindings.cpp:3-33,
 * src/render.cu:191-422, src/render_backward.cu:287-595.
 *
 * The kernels read one 48-byte splat record per Gaussian (GSR_REC_FLOATS
 * floats) through the depth-sorted pair list of every tile.
 * gsr_preprocess_forward writes these records; gsr_pack_gaussian_records builds them
 * from the reference's per-Gaussian arrays.
 * ---------------------------------------------------------------------- */
/* uvs [N,2], opacity [N] (post-sigmoid), rgb [N,3], conic [N,3] -> records [N,12], row i from Gaussian i.
 * (Earlier releases exported gsr_pack_records, which packed one record per sorted pair; the new name makes a caller
 * built against that argument list fail to resolve instead of passing its pointers into the wrong slots.) */
int gsr_pack_gaussian_records(int N, const float* uvs, const float* opacity, const float* rgb, const float* conic,
                              float* records, void* stream);

/* Number of 32-bit words of the forward -> backward contribution masks for P (gaussian, tile) pairs on an H x W
 * image: per (tile, 128-record batch, warp, lane group) one 128-bit mask whose bit j is set when record j of the
 * batch contributed to at least one pixel of the group's 4x4 pixel block.  Forward and backward must come from the
 * same build. */
size_t gsr_contribution_mask_words(int64_t P, int H, int W);

/* The tile renderers.  They fetch each batch's records themselves from the per-gaussian record array
 * gaussian_records [N,12] through the sorted pair list — keys_sorted (gaussian id in the low id_bits of every key,
 * gsr_sort_keys' output) or ids_sorted (gsr_sort_pairs' id output, or the reference's sorted_gaussian_idx); exactly
 * one of the two is non-NULL.  3 x 16-byte cp.async per record, issued by the warp that recycles a pipeline stage,
 * completion on the stage's mbarrier.  Gradients are indexed by gaussian id.
 *
 * Forward: tile_ranges [n_tiles+1], background [3] ->
 * image [H,W,3], num_splats_per_pixel int32 [H,W], final_weight_per_pixel [H,W].
 * contribution_masks: NULL, or gsr_contribution_mask_words(P, H, W) ZERO-FILLED words the kernel records the
 * contributing (pixel block, record) pairs in, for gsr_render_backward_gather of the same view.  The backward takes
 * NULL (the kernel finds the candidate records of every pixel block with its own conservative footprint test, like
 * the forward), or the masks the forward of this view recorded: it then visits exactly the (pixel block, record)
 * pairs that contributed.
 *
 * Depth and alpha maps from the same walk (precomputed colours), when depth and alpha are non-NULL (both or neither;
 * NULL: colour only, and depth_key / depth_base / depth_bits are not read).  Per pixel, over the splats the colour
 * blend composites (same weights w_i, same saturation early-out):
 *   alpha [H,W] = the accumulated sum of w_i before any background (0 where nothing contributes),
 *   depth [H,W] = D, D <- fma(w_i, z_i, D) front to back, z_i the camera-frame z of gaussian i; no background term
 *                 (un-normalised: expected depth is depth / alpha).
 * z_i is decoded from the depth field of the sorted pair keys — bits(z) - depth_base, or depth_key()'s
 * order-preserving transform when depth_base == 0 (then depth_bits must be 32) — and, with ids_sorted instead of
 * keys_sorted, from the per-gaussian depth keys depth_key [N] (gsr_preprocess_forward's output).
 * Argument errors return GSR_ERR_BAD_ARG. */
int gsr_render_forward_gather(const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                              const int32_t* ids_sorted, const uint32_t* depth_key, uint32_t depth_base, int depth_bits,
                              const int32_t* tile_ranges, const float* background_rgb, int H, int W,
                              int32_t* num_splats_per_pixel, float* final_weight_per_pixel, float* image, float* depth,
                              float* alpha, uint32_t* contribution_masks, void* stream);
/* gsr_render_forward_gather + per-gaussian blend-weight statistics (importance scores for pruning), accumulated into
 * (never cleared) over every pixel p of the view where gaussian i contributes to the colour blend:
 *   weight_sum [N]  f32: += sum_p w_ip, w_ip the blend weight of the colour (T_ip * alpha_ip, the walk's float);
 *   weight_max [N]  f32: max(weight_max, max_p w_ip), taken on the float bits (w >= +0; the array must hold values
 *                   >= +0.0, e.g. zero-filled);
 *   pixel_count [N] i32: += the number of such pixels (wraps past 2^31 - 1).
 * A pixel counts for gaussian i iff the colour blend uses it: the pixel lies in the image and is not yet saturated,
 * the Mahalanobis term is positive and alpha > 1/255.  The image and every other output are bit-identical to
 * gsr_render_forward_gather's.  weight_sum is accumulated with float atomics (determined up to summation order);
 * weight_max and pixel_count are deterministic.  Pixels the walk recomputes exactly contribute the walk's weights.
 * All three NULL: exactly gsr_render_forward_gather; some but not all NULL: GSR_ERR_BAD_ARG.
 * Speculatively sized pair buffers: pair_total (NULL: none) points at the pair scan's total, P in its low 32 bits
 * (the last element of the per-gaussian scan the pair emission reads); when P > pair_capacity (0 <= pair_capacity < 2^32), the pairs the kernel sees
 * are incomplete and NOTHING is accumulated — the caller renders the view again with the exact count. */
int gsr_render_forward_gather_stats(const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                                    const int32_t* ids_sorted, const uint32_t* depth_key, uint32_t depth_base,
                                    int depth_bits, const int32_t* tile_ranges, const float* background_rgb, int H,
                                    int W, int32_t* num_splats_per_pixel, float* final_weight_per_pixel, float* image,
                                    float* depth, float* alpha, uint32_t* contribution_masks, float* weight_sum,
                                    float* weight_max, int32_t* pixel_count, const uint64_t* pair_total,
                                    int64_t pair_capacity, void* stream);
/* + grad_image [H,W,3].  Gradient destination, accumulated into: the four planar arrays grad_rgb [N,3],
 * grad_opacity [N], grad_uv [N,2], grad_conic [N,3] (grad_rows NULL), or grad_rows [N, GSR_GRAD_ROW_FLOATS] (16-byte
 * aligned, zero-filled; then the four planar pointers are ignored): one interleaved row per gaussian,
 * rgb3 opacity | uv2 conic0 conic1 | conic2 pad3, accumulated with 16-byte vector reductions — the nine sums of a pair
 * touch two adjacent 32-byte sectors instead of four arrays.  gsr_preprocess_backward reads the rows.
 * Depth/alpha mode: grad_depth and grad_alpha [H,W] non-NULL (both or neither; zeros where a map has no gradient),
 * the depth descriptor as in the forward, grad_rows required; the rows are then rgb3 opacity | uv2 conic0 conic1 |
 * conic2 z pad2, z being the gradient on the camera-frame z, which gsr_preprocess_backward consumes with
 * GSR_MODE_DEPTH_ALPHA.
 * mode: GSR_MODE_* bits; only GSR_MODE_ABSGRAD changes this stage (other known bits are ignored, unknown ones are
 * GSR_ERR_BAD_ARG).  It requires grad_rows; the rows' last four floats are then conic2 z|0 |u| |v|, flushed as one
 * more 16-byte vector reduction, with
 *   |u| = sum over pixels p of |d <G_p, out_p> / d u|,  |v| likewise,
 * G_p the upstream gradients at pixel p (image, and depth / alpha when given): the absolute value is taken per pixel
 * before summing, so pulls in opposite directions do not cancel (AbsGS).  Units are pixels, like grad_uv.
 * gsr_preprocess_backward does not read slots 10-11. */
#define GSR_GRAD_ROW_FLOATS 12
int gsr_render_backward_gather(int mode, const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                               const int32_t* ids_sorted, const uint32_t* depth_key, uint32_t depth_base,
                               int depth_bits, const int32_t* tile_ranges, const float* background_rgb, int H, int W,
                               const int32_t* num_splats_per_pixel, const float* final_weight_per_pixel,
                               const float* grad_image, const float* grad_depth, const float* grad_alpha,
                               float* grad_rgb, float* grad_opacity, float* grad_uv, float* grad_conic,
                               float* grad_rows, const uint32_t* contribution_masks, void* stream);

/* General renderers: any dtype, any n_sh in {1,4,9,16} (per-pixel SH via view_dir_by_pixel
 * [H,W,3]); same semantics as the reference's template instantiations
 * (fp64: no +0.25 dilation, exp(), no 1/255 skip — src/render.cu:117-148). */
int gsr_render_forward_generic(int dtype, int N, int n_sh, const void* uvs, const void* opacity,
                               const void* rgb, const void* conic, const void* view_dir_by_pixel,
                               const int32_t* tile_ranges, const int32_t* sorted_gaussian_idx,
                               const void* background_rgb, int H, int W,
                               int32_t* num_splats_per_pixel, void* final_weight_per_pixel,
                               void* image, void* stream);
int gsr_render_backward_generic(int dtype, int N, int n_sh, const void* uvs, const void* opacity,
                                const void* rgb, const void* conic, const void* view_dir_by_pixel,
                                const int32_t* tile_ranges, const int32_t* sorted_gaussian_idx,
                                const void* background_rgb, int H, int W,
                                const int32_t* num_splats_per_pixel,
                                const void* final_weight_per_pixel, const void* grad_image,
                                void* grad_rgb, void* grad_opacity, void* grad_uv, void* grad_conic,
                                void* stream);

/* render_depth_cuda — src/bindings.cpp:107-116, src/depth.cu:117-177 (fp32 only) */
int gsr_render_depth(int N, const float* xyz_camera_frame, const float* uvs, const float* opacity,
                     const float* conic, const int32_t* tile_ranges,
                     const int32_t* sorted_gaussian_idx, float alpha_threshold, int H, int W,
                     float* depth_image, void* stream);

/* ------------------------------------------------------------------------
 * Fused path behind splat_py.rasterize.rasterize (splat_py/rasterize.py:18-112):
 * one kernel does world->camera transform, frustum cull, pinhole projection,
 * Sigma_world, Jacobian, 2-D covariance, sigmoid(opacity), SH->RGB and the tile
 * count for every Gaussian; results are bit-identical to running the
 * reference's operator chain on the survivors.
 * ---------------------------------------------------------------------- */
/* centre [3] <- inverse(camera_T_world)[:3, 3]: the camera centre in world coordinates that the SH view
 * directions use (splat_py/rasterize.py:91-93 `torch.inverse(camera_T_world)`, src/precompute_sh.cu:149-151), with the
 * bits torch's LU-based inverse produces for one 4x4 fp32 matrix (one tiny kernel instead of torch's 15). */
int gsr_camera_centre(const float* camera_T_world, float* centre, void* stream);

size_t gsr_preprocess_temp_bytes(int N);
/* inputs: xyz [N,3], quaternion [N,4], scale [N,3], opacity_logit [N], rgb_dc [N,3],
 *         sh_rest [N,3,n_sh_rest] (n_sh_rest in {0,3,8,15}; may be NULL when 0),
 *         camera_T_world [4,4] and K [3,3] ON DEVICE;
 *         xyz_camera_frame [N - cam_first, 3] or NULL: camera-frame positions of gaussians cam_first..N-1
 *         computed by the caller (the reference forms them with torch.matmul, whose rounding order
 *         belongs to cuBLAS); for every other gaussian the kernel applies camera_T_world itself,
 *         reproducing the rounding order of cuBLAS' large-batch kernel (csrc/gsr_math.cuh);
 *         camera_centre [3] or NULL: inverse(camera_T_world)[:3,3] computed by the caller (the reference
 *         uses torch.inverse); when NULL the kernel inverts the pose itself (fp64 Gauss-Jordan).
 * outputs (all indexed by ORIGINAL gaussian index):
 *   records  float [N,12]   packed splat record (undefined for culled rows)
 *   depth_key uint32 [N]    order-preserving key of camera-frame z: float bits of z minus depth_base
 *                           (pass depth_base = float bits of near_thresh when near_thresh > 0 so that only
 *                           bitlength(bits(far) - bits(near)) low bits are significant; 0 otherwise)
 *   visible  uint8 [N]      1 = survives the frustum cull (culling_mask = !visible)
 *   scan     uint64 [N]     INCLUSIVE scan of (visible << 32 | tiles_touched);
 *                           scan[N-1] >> 32 == M, scan[N-1] & 0xffffffff == P
 *   tile_mask uint64 [N], tile_win uint32 [N]  (both or neither; may be NULL): for visible gaussians whose tile
 *                           window has at most 64 tiles, the tiles hit as a bit mask over the window (bit =
 *                           (tx - x0) * height + (ty - y0)) and the window as x0 | y0 << 8 | width << 16 |
 *                           height << 24; tile_win = 0xffffffff for larger windows.  gsr_emit_keys / gsr_emit_pairs
 *                           expand the mask instead of repeating the OBB tests.
 * mode: GSR_MODE_* bits; only GSR_MODE_ANTIALIASED changes this stage (Mip-Splatting's 2-D filter, "antialiased"
 *   rasterize mode): each record's opacity is then sigmoid(opacity_logit) * rho with
 *     rho = sqrt(max(det0, 0) / det),  det0 = det of the 2-D covariance, det = det of the covariance + 0.25 I
 *   (the +0.25 px^2 dilation the tile renderers apply), so the dilated splat carries the mass of the undilated one.
 *   The culling bound is formed from the compensated opacity.  rho == 0 where det0 <= 0 in fp32: the splat then never
 *   contributes.  Operation order: gsr_record.cuh aa_rho.
 * GSR_MODE_FILTER3D (Mip-Splatting's 3-D smoothing filter): filter3d [N] is required with the bit and must be NULL
 *   without it (else GSR_ERR_BAD_ARG).  f = filter3d[i] is a standard deviation in world units, used only squared:
 *   Sigma_world is formed from the variances v_k + f^2 (v_k = exp(scale_k)^2) and the opacity is multiplied by
 *   coef = sqrt(prod_k v_k / (v_k + f^2)), before rho when GSR_MODE_ANTIALIASED is set too; the culling bound is formed
 *   from the final opacity.  f == 0 gives the unfiltered record bit for bit.  Operation order: gsr_record.cuh
 *   f3d_filter.  The render stages ignore the bit. */
int gsr_preprocess_forward(int mode, int N, int n_sh_rest, const float* xyz, const float* xyz_camera_frame,
                           int cam_first, const float* quaternion,
                           const float* scale, const float* opacity_logit, const float* filter3d, const float* rgb_dc,
                           const float* sh_rest, const float* camera_T_world, const float* K,
                           const float* camera_centre, int H, int W, float near_thresh, float far_thresh,
                           float cull_mask_padding, float mh_dist, uint32_t depth_base, float* records,
                           uint32_t* depth_key,
                           uint8_t* visible, uint64_t* scan, uint64_t* tile_mask, uint32_t* tile_win, void* temp,
                           size_t temp_bytes, void* stream);

/* emits the (tile, depth) keys and original-gaussian ids of all P pairs, the compact list of
 * visible gaussian ids vis_idx int32 [M] and the compacted uv [M,2] the reference returns */
/* keys are (tile << depth_bits) | depth_key; depth_bits in 1..32 is the number of significant key bits.
 * capacity: 0 when keys / ids hold exactly P entries (the host has read P = scan[N-1] & 0xffffffff); otherwise the
 * number of entries of SPECULATIVELY sized buffers (the host has not synchronised yet): pairs beyond the capacity
 * are dropped (the caller finds P > capacity when it does read P, and redoes the binning), positions [P, capacity)
 * are filled with the all-ones key, which sorts behind every real pair; gsr_sort_* and gsr_tile_ranges are then
 * called with `capacity` in place of P and ignore the padding. */
int gsr_emit_pairs(int N, const float* records, const uint32_t* depth_key, const uint8_t* visible,
                   const uint64_t* scan, int n_tiles_x, int n_tiles_y, float mh_dist, int depth_bits,
                   uint64_t* keys, uint32_t* ids, int32_t* vis_idx, float* uv_compact, int64_t capacity,
                   const uint64_t* tile_mask, const uint32_t* tile_win, void* stream);

size_t gsr_sort_pairs_temp_bytes(int P);
int gsr_sort_pairs(int P, int n_tiles, int depth_bits, const uint64_t* keys_in, const uint32_t* ids_in,
                   uint64_t* keys_out, uint32_t* ids_out, void* temp, size_t temp_bytes, void* stream);

/* tile_ranges int32 [n_tiles+1] from sorted keys */
int gsr_tile_ranges(int P, int n_tiles, int depth_bits, const uint64_t* keys_sorted, int32_t* tile_ranges,
                    void* stream);

/* Keys-only variant of the three calls above: when tile bits + depth_bits + id bits fit in 64, the gaussian id
 * rides in the low id_bits of the key — (tile | depth | id) — and ONE cub::DeviceRadixSort::SortKeys over bits
 * [id_bits, id_bits + depth_bits + tile bits) replaces SortPairs (8 instead of 12 bytes moved per pair and pass;
 * the id bits are not sorted: the sort is stable and pairs are emitted in gaussian order, so ties resolve as
 * before).  gsr_packed_id_bits returns the id width to use, or 0 when it does not fit (use the pair calls).
 * gsr_tile_ranges takes depth_bits + id_bits as its shift. */
int gsr_packed_id_bits(int N, int n_tiles, int depth_bits);
int gsr_emit_keys(int N, const float* records, const uint32_t* depth_key, const uint8_t* visible,
                  const uint64_t* scan, int n_tiles_x, int n_tiles_y, float mh_dist, int depth_bits, int id_bits,
                  uint64_t* keys, int32_t* vis_idx, float* uv_compact, int64_t capacity, const uint64_t* tile_mask,
                  const uint32_t* tile_win, void* stream);
size_t gsr_sort_keys_temp_bytes(int P);
int gsr_sort_keys(int P, int n_tiles, int depth_bits, int id_bits, const uint64_t* keys_in, uint64_t* keys_out,
                  void* temp, size_t temp_bytes, void* stream);

/* backward of the fused per-Gaussian stage.  grad_rows [N, GSR_GRAD_ROW_FLOATS] (required, 16-byte aligned) are the
 * per-gaussian sums gsr_render_backward_gather accumulated into interleaved rows (indexed by gaussian).  The gradient
 * on a projected mean is the row's uv (skipped when use_rows_uv is 0) PLUS grad_uv_compact[(scan[i] >> 32) - 1]
 * (skipped when NULL): grad_uv_compact [M,2] is a gradient on the compact uv rasterize returned, in its order
 * (scan = the packed inclusive scan of gsr_preprocess_forward) — what a caller added upstream of uv, or the total
 * autograd hands over.
 * mode: the GSR_MODE_* bits of the forward and the render backward.
 *   GSR_MODE_ABSGRAD changes nothing here (the rows' slots 10-11 are not read).
 *   GSR_MODE_DEPTH_ALPHA: the rows of the depth/alpha render backward: row slot 9, the gradient on the camera-frame z,
 *   joins grad_xyz as camera_T_world[2, :3] * g_z.  No gradient goes to the pose.
 *   GSR_MODE_ANTIALIASED: the rows' opacity slot g is the gradient on the compensated opacity sigmoid(o) * rho:
 *   sigmoid(o) receives g * rho and the 2-D covariance g * sigmoid(o) * grad(rho).  Where rho == 0 no gradient goes
 *   through rho (its gradient is infinite there, and g is 0 because the splat never contributed).
 *   GSR_MODE_FILTER3D: filter3d [N] as in gsr_preprocess_forward (required iff the bit is set).  The rows' opacity
 *   slot (times rho with GSR_MODE_ANTIALIASED) is the gradient g on sigmoid(o) * coef: sigmoid(o) receives g * coef and
 *   scale_k additionally g * sigmoid(o) * coef * f^2 / (v_k + f^2).  No gradient goes to filter3d.
 * Writes dense parameter gradients for all N gaussians (zeros for culled ones). */
int gsr_preprocess_backward(int mode, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                            const float* scale, const float* opacity_logit, const float* filter3d,
                            const float* camera_T_world,
                            const float* K, const float* camera_centre, const uint8_t* visible, const float* grad_rows,
                            int use_rows_uv,
                            const float* grad_uv_compact, const uint64_t* scan, float* g_xyz, float* g_quaternion,
                            float* g_scale, float* g_opacity_logit, float* g_rgb_dc, float* g_sh_rest, void* stream);

/* Mip-Splatting's 3-D filter size per gaussian, from C cameras: camera_T_world [C,4,4], K [C,3,3], width / height
 * int32 [C] (all on the device) and xyz [N,3] -> filter3d [N] (standard deviations in world units).
 * Camera c sees gaussian i when, with p = T_c x and (u, v) formed as gsr_preprocess_forward forms them (fp32,
 * csrc/gsr_math.cuh transform_point / project_uv):
 *   p_z > near,  -(m W_c) <= u <= (1 + m) W_c,  -(m H_c) <= v <= (1 + m) H_c    (m = margin; products rounded to fp32)
 * and then samples it at r_c = p_z / max(fx_c, fy_c) world units per pixel (IEEE division).  r_i = min over the
 * cameras that see i; filter3d[i] = sqrtf(variance) * r_i, sqrtf(variance) rounded to float once.  Gaussians no camera
 * sees get the largest r_i of the seen ones; when none is seen at all, every filter3d[i] is 0.  Deterministic.
 * Intrinsics are expected to have positive focal lengths (not checked: no host synchronisation).
 * GSR_ERR_BAD_ARG for C < 1, near < 0, negative (or NaN) margin or variance, or (N > 0) NULL pointers.  N == 0 returns
 * GSR_OK. */
int gsr_filter3d(int N, const float* xyz, int C, const float* camera_T_world, const float* K, const int* width,
                 const int* height, float near, float margin, float variance, float* filter3d, void* stream);

/* ---- optimizer step on the flat parameter buffer (SURVEY.md 8(f) rank 2) ----------------------------
 * Replaces torch.optim.Adam.step() as configured by splat_py/optimizer_manager.py:13-44 (one parameter group
 * per field, betas (0.9, 0.999), eps 1e-8, no weight decay / amsgrad), with the per-element operation order
 * of torch's CUDA implementation.  p, g, m, v: flat fp32 arrays of n elements laid out like the gradients
 * gsr_preprocess_backward produces ([xyz|quaternion|scale|opacity|rgb|sh], sections 16-byte aligned; n and
 * every section_end are multiples of 4).  section_end[k] = exclusive end (in elements) of section k,
 * section_lr[k] its learning rate; step = 1 for the first update. */
int gsr_adam_step(int64_t n, float* p, const float* g, float* m, float* v, int n_sections,
                  const int64_t* section_end, const double* section_lr, double beta1, double beta2, double eps, int step,
                  void* stream);

/* View-parallel form, one process per GPU: this rank owns elements [lo, hi) of the flat buffer.  The gradient
 * of the range is read from every rank's gradient buffer (peer_grads[q], device pointers valid on this device:
 * CUDA IPC / symmetric memory over NVLink), summed in rank order and divided by world; m_shard / v_shard hold
 * only the owned range (hi - lo elements); the updated parameters are stored into every rank's parameter
 * buffer (peer_params[q]).  Reduce-scatter + Adam + all-gather in one kernel.  The caller provides the
 * cross-rank ordering: all gradients complete before the launch, a barrier after it before parameters are read. */
int gsr_adam_step_sharded(int64_t lo, int64_t hi, int world, const float* const* peer_grads,
                          float* const* peer_params, int self_rank, float* m_shard, float* v_shard, int n_sections,
                          const int64_t* section_end, const double* section_lr, double beta1, double beta2, double eps,
                          int step, void* stream);

/* Per-step densification statistics of the reference's trainer (splat_py/trainer.py:376-385), in one pass:
 * uv_grad [M,2] (the gradient of the compact uv rasterize returned, indexed like vis_idx) is scaled IN PLACE by
 * (K[0][0], K[1][1]) and its absolute value added to uv_grad_accum [N,2] at the visible gaussians' rows;
 * grad_accum_count [N] += 1 there; xyz_grad_accum [N,3] += |xyz_grad|.  vis_idx int32 [M] = indices of the
 * gaussians that passed the frustum cull, ascending (gsr_emit_pairs / gsr_emit_keys produce it). */
int gsr_densify_accumulate(int N, int M, const int32_t* vis_idx, float* uv_grad, const float* xyz_grad, const float* K,
                           float* uv_grad_accum, float* xyz_grad_accum, int32_t* grad_accum_count, void* stream);

/* Length (in floats) of the flat parameter / gradient / Adam-moment buffer of n_gaussians gaussians with
 * n_sh_rest higher-order SH coefficients per channel: sections [xyz 3 | quaternion 4 | scale 3 | opacity 1 |
 * rgb 3 | sh 3*n_sh_rest], every section start 16-byte aligned (the layout gsr_preprocess_backward writes). */
int64_t gsr_flat_numel(int64_t n_gaussians, int n_sh_rest);

/* Clone / split / delete of the reference's adaptive density control (splat_py/trainer.py:114-206 with the
 * optimizer surgery of splat_py/optimizer_manager.py:74-172), applied to the flat parameter buffer and both Adam
 * moment buffers in ONE pass.  The plan is per OUTPUT row r (n_out rows):
 *   src[r]        row of the old buffers (n_in rows) it is copied from
 *   clone_row[r]  >= 0: a clone, xyz -= xyz_sub[clone_row[r]][0..2]            (trainer.py:122-126); else -1
 *   split_row[r]  >= 0: a split sample, xyz += xyz_add[...], quaternion = q_set[...], scale = scale_set[...]
 *                 (trainer.py:166-194); else -1
 * Rows with clone_row >= 0 or split_row >= 0 are new: their Adam moments are zero; all others keep their source
 * row's moments.  clone_row / split_row may be NULL (no clones / no splits); m_in, v_in, m_out, v_out may all be
 * NULL (parameters only).  p_out / m_out / v_out: caller-allocated, gsr_flat_numel(n_out, n_sh_rest) floats,
 * must not alias the inputs.  Deletion is expressed by src skipping the deleted rows. */
int gsr_densify_apply(int n_in, int n_out, int n_sh_rest, const float* p_in, const float* m_in, const float* v_in,
                      const int32_t* src, const int32_t* clone_row, const int32_t* split_row, const float* xyz_sub,
                      const float* xyz_add, const float* q_set, const float* scale_set, float* p_out, float* m_out,
                      float* v_out, void* stream);

/* ---- 3DGS-MCMC densification (Kheradmand et al. 2024) on the flat buffers (csrc/gsr_mcmc.cu) -----------------
 * Relocation of n sampled rows: opacity [n] (sigmoid opacity o), scale [n,3] (exp scale), ratio int32 [n] (number
 * of copies, clamped to [1, n_max]) -> new_opacity [n] = clamp(1 - (1 - o)^(1/N), min_opacity, 1 - 2^-23) and
 * new_scale [n,3] = scale * o / sum_{i=1..N} sum_{k=0..i-1} C(i-1,k) (-1)^k o_hat^(k+1) / sqrt(k+1), the sum and the
 * power evaluated in fp64 (the sum alternates in sign; see the kernel).  Outputs must not overlap the inputs or each
 * other; n_max >= 1. */
int gsr_mcmc_relocation(int n, const float* opacity, const float* scale, const int32_t* ratio, int n_max,
                        float min_opacity, float* new_opacity, float* new_scale, void* stream);

/* A relocation or growth plan applied to the flat parameter buffer and both Adam moment buffers in ONE pass
 * (n_out >= n_in; the layout of gsr_flat_numel).  Per OUTPUT row r:
 *   src[r]      row of the old buffers it is copied from
 *   set_row[r]  >= 0: opacity <- logit(new_opacity[set_row[r]]), scale <- log(new_scale[set_row[r]][0..2]), both
 *               formed in the kernel (p / (1 - p), then logf); else -1
 * Moment contract: m and v are ZERO in every row with set_row[r] >= 0 — the rows whose parameters the pass changes:
 * the sampled sources, the relocated dead rows and the appended copies.  Every other row keeps its source row's
 * moments.  A relocated row therefore never inherits a dead row's (or its source's) moments.  Section padding is
 * zero.  set_row, new_opacity and new_scale go together (all NULL: a plain gather); m_in, v_in, m_out, v_out go
 * together.  Outputs must not overlap the inputs or each other.  set_row values index the caller's tables. */
int gsr_mcmc_apply(int n_in, int n_out, int n_sh_rest, const float* p_in, const float* m_in, const float* v_in,
                   const int32_t* src, const int32_t* set_row, const float* new_opacity, const float* new_scale,
                   float* p_out, float* m_out, float* v_out, void* stream);

/* SGLD position noise, in place on the flat parameter buffer p of N gaussians (run after the optimizer step):
 *   xyz_i += scaler * w_i * Sigma_i eps_i,  Sigma_i = R(q_i / |q_i|) diag(exp(2 s_i)) R^T,
 *   w_i = 1 / (1 + exp(-k ((1 - sigmoid(opacity_i)) - x0)))
 * eps_i ~ N(0, I_3) from Philox4x32-10 keyed by (seed, subsequence i, offset): the same (seed, offset) gives the
 * same draws on every device and launch; pass the step as offset.  eps_in [N,3] (optional) replaces the draws;
 * eps_out [N,3] (optional) receives the draws used.  Only the xyz section is written. */
int gsr_mcmc_noise(int N, int n_sh_rest, float* p, double scaler, double k, double x0, uint64_t seed, uint64_t offset,
                   const float* eps_in, float* eps_out, void* stream);

/* ---- photometric loss of the training step (splat_py/trainer.py:363-374) ------------------------------------
 * loss = l1_weight * L1 + ssim_weight * (1 - SSIM), with L1 = mean |pred - target| over all B*C*H*W elements and
 * SSIM the mean over B*C*(H-10)*(W-10) valid window origins of the 11x11 separable Gaussian-window SSIM map
 * S = (2 mu_p mu_t + c1)(2 s_pt + c2) / ((mu_p^2 + mu_t^2 + c1)(s_pp + s_tt + c2)) (no clamping).
 * pred, target, grad_pred: base pointer + element strides (B, C, H, W) in *_strides_host[4], any layout (the
 * [H,W,C] image of the renderer is B = 1 with strides (H*W*C, 1, W*C, C)); window_host [11]: the window taps;
 * c1 = (0.01 * data_range)^2, c2 = (0.03 * data_range)^2.  H and W must be >= 11.  Results do not depend on the
 * strides, bit for bit, and are identical from run to run. */
size_t gsr_photometric_loss_temp_bytes(int B, int C, int H, int W);
/* out [3] (device, dtype) <- {loss, L1, SSIM}; temp: gsr_photometric_loss_temp_bytes(B, C, H, W) bytes. */
int gsr_photometric_loss_forward(int dtype, int B, int C, int H, int W, const void* pred,
                                 const int64_t* pred_strides_host, const void* target,
                                 const int64_t* target_strides_host, const double* window_host, double c1, double c2,
                                 double l1_weight, double ssim_weight, void* out, void* temp, size_t temp_bytes,
                                 void* stream);
/* grad_pred <- grad_loss[0] * d loss / d pred (grad_loss: a device scalar of the same dtype); recomputes the
 * moments, stores no intermediate maps.  No gradient with respect to target. */
int gsr_photometric_loss_backward(int dtype, int B, int C, int H, int W, const void* pred,
                                  const int64_t* pred_strides_host, const void* target,
                                  const int64_t* target_strides_host, const double* window_host, double c1, double c2,
                                  double l1_weight, double ssim_weight, const void* grad_loss, void* grad_pred,
                                  const int64_t* grad_strides_host, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GSR_B200_H */
