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
 * The kernels consume a depth-sorted, tile-contiguous stream of 48-byte splat
 * records (GSR_REC_FLOATS floats per pair) that is staged into shared memory
 * by TMA bulk copies.  gsr_pack_records builds that stream from the
 * reference's per-Gaussian arrays.
 * ---------------------------------------------------------------------- */
/* uvs [N,2], opacity [N] (post-sigmoid), rgb [N,3], conic [N,3], sorted idx [P] -> records [P,12] */
int gsr_pack_records(int P, const int32_t* sorted_gaussian_idx, const float* uvs,
                     const float* opacity, const float* rgb, const float* conic, float* records,
                     void* stream);

/* Number of 32-bit words of the forward -> backward contribution masks for P (gaussian, tile) pairs on an H x W
 * image: per (tile, 128-record batch, warp, lane group) one 128-bit mask whose bit j is set when record j of the
 * batch contributed to at least one pixel of the group's 4x4 pixel block.  Forward and backward must come from the
 * same build. */
size_t gsr_contribution_mask_words(int64_t P, int H, int W);

/* records [P,12], tile_ranges [n_tiles+1], background [3] ->
 * image [H,W,3], num_splats_per_pixel int32 [H,W], final_weight_per_pixel [H,W].
 * contribution_masks: NULL, or gsr_contribution_mask_words(P, H, W) ZERO-FILLED words the kernel records the
 * contributing (pixel block, record) pairs in, for gsr_render_backward of the same view. */
int gsr_render_forward(const float* records, const int32_t* tile_ranges, const float* background_rgb,
                       int H, int W, int32_t* num_splats_per_pixel, float* final_weight_per_pixel,
                       float* image, uint32_t* contribution_masks, void* stream);

/* + grad_image [H,W,3]; accumulates into grad_rgb [N,3], grad_opacity [N], grad_uv [N,2],
 * grad_conic [N,3] at row sorted_gaussian_idx[p].
 * contribution_masks: NULL (the kernel finds the candidate records of every pixel block with its own
 * conservative footprint test, like the forward), or the masks the forward of this view recorded: the backward
 * then visits exactly the (pixel block, record) pairs that contributed. */
int gsr_render_backward(const float* records, const int32_t* sorted_gaussian_idx,
                        const int32_t* tile_ranges, const float* background_rgb, int H, int W,
                        const int32_t* num_splats_per_pixel, const float* final_weight_per_pixel,
                        const float* grad_image, float* grad_rgb, float* grad_opacity,
                        float* grad_uv, float* grad_conic, const uint32_t* contribution_masks, void* stream);

/* The same two kernels WITHOUT a record stream: the tile kernels fetch each batch's records themselves from the
 * per-gaussian record array gaussian_records [N,12] (gsr_preprocess_forward's output), through the sorted pair list
 * — keys_sorted (gaussian id in the low id_bits of every key, gsr_sort_keys' output) or ids_sorted (gsr_sort_pairs'
 * id output); exactly one of the two is non-NULL.  3 x 16-byte cp.async per record, issued by the warp that recycles
 * a pipeline stage, completion on the stage's mbarrier; gsr_gather_records* and the [P,12] stream are not needed.
 * Gradient rows are indexed by gaussian id. */
int gsr_render_forward_gather(const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                              const int32_t* ids_sorted, const int32_t* tile_ranges, const float* background_rgb, int H,
                              int W, int32_t* num_splats_per_pixel, float* final_weight_per_pixel, float* image,
                              uint32_t* contribution_masks, void* stream);
/* Gradient destination: the four planar arrays (grad_rows NULL), or grad_rows [N, GSR_GRAD_ROW_FLOATS] (16-byte
 * aligned, zero-filled; then the four planar pointers are ignored): one interleaved row per gaussian,
 * rgb3 opacity | uv2 conic0 conic1 | conic2 pad3, accumulated with 16-byte vector reductions — the nine sums of a pair
 * touch two adjacent 32-byte sectors instead of four arrays.  gsr_preprocess_backward reads either form. */
#define GSR_GRAD_ROW_FLOATS 12
int gsr_render_backward_gather(const float* gaussian_records, const uint64_t* keys_sorted, int id_bits,
                               const int32_t* ids_sorted, const int32_t* tile_ranges, const float* background_rgb, int H,
                               int W, const int32_t* num_splats_per_pixel, const float* final_weight_per_pixel,
                               const float* grad_image, float* grad_rgb, float* grad_opacity, float* grad_uv,
                               float* grad_conic, float* grad_rows, const uint32_t* contribution_masks, void* stream);

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
 *                           expand the mask instead of repeating the OBB tests. */
int gsr_preprocess_forward(int N, int n_sh_rest, const float* xyz, const float* xyz_camera_frame,
                           int cam_first, const float* quaternion,
                           const float* scale, const float* opacity_logit, const float* rgb_dc,
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
 * are filled with the all-ones key, which sorts behind every real pair; gsr_sort_*, gsr_tile_ranges and
 * gsr_gather_records* are then called with `capacity` in place of P and ignore the padding. */
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

/* records_sorted[p] = records[ids_sorted[p]] (48-byte rows).  scan / ranks_sorted (both or neither): also
 * ranks_sorted[p] = (scan[ids_sorted[p]] >> 32) - 1, the gaussian's rank among the visible ones = its row in
 * compact per-gaussian gradient arrays (see gsr_preprocess_backward). */
int gsr_gather_records(int P, const uint32_t* ids_sorted, const float* records, float* records_sorted,
                       const uint64_t* scan, int32_t* ranks_sorted, void* stream);

/* Keys-only variant of the four calls above: when tile bits + depth_bits + id bits fit in 64, the gaussian id
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
/* ids_sorted[p] = the gaussian id of sorted pair p, or — scan != NULL — its rank among the visible gaussians */
int gsr_gather_records_keys(int P, int id_bits, const uint64_t* keys_sorted, const float* records,
                            float* records_sorted, int32_t* ids_sorted, const uint64_t* scan, void* stream);

/* backward of the fused per-Gaussian stage.  grad_rgb [N,3] / grad_opacity [N] / grad_uv [N,2] / grad_conic [N,3]
 * are the per-gaussian sums the render backward accumulated (indexed by gaussian).  The gradient on a projected
 * mean is grad_uv[i] (skipped when grad_uv is NULL) PLUS grad_uv_compact[(scan[i] >> 32) - 1] (skipped when NULL):
 * grad_uv_compact [M,2] is a gradient on the compact uv rasterize returned, in its order (scan = the packed
 * inclusive scan of gsr_preprocess_forward) — what a caller added upstream of uv, or the total autograd hands over.
 * grad_rows != NULL: the interleaved rows of gsr_render_backward_gather instead of the four planar arrays
 * (grad_uv == NULL then still means "skip the render backward's uv sums").
 * Writes dense parameter gradients for all N gaussians (zeros for culled ones). */
int gsr_preprocess_backward(int N, int n_sh_rest, const float* xyz, const float* quaternion,
                            const float* scale, const float* opacity_logit, const float* camera_T_world,
                            const float* K, const float* camera_centre, const uint8_t* visible, const float* grad_rgb,
                            const float* grad_opacity, const float* grad_uv, const float* grad_conic,
                            const float* grad_rows, int use_rows_uv,
                            const float* grad_uv_compact, const uint64_t* scan, float* g_xyz, float* g_quaternion,
                            float* g_scale, float* g_opacity_logit, float* g_rgb_dc, float* g_sh_rest, void* stream);

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
