// gsr_surfels_lens.cu — 2-D Gaussian surfels through a lens (libgsr_surfels_lens.so, C ABI include/gsr_surfels_lens.h,
// model DESIGN.md 3.26): the ray-map kernel, and the per-gaussian and tile kernels of rasterize_surfels(...,
// fisheye=k / distortion=k).
//
// The bodies are gsr_surfels.cuh's with the lens as a compile-time parameter (GSR_SURFEL_LENS_FISHEYE,
// GSR_SURFEL_LENS_DISTORTION) for the per-gaussian kernels, and the ray map in place of the pinhole's (x, y, 1) for the
// tile kernels.  The lens constants are read into shared memory next to the view constants.  Binning is
// libgsr_b200.so's, unchanged.
#include <cub/cub.cuh>

#include "gsr_surfels.cuh"
#include "../../include/gsr_distortion.h"
#include "../../include/gsr_fisheye.h"
#include "../../include/gsr_surfels_lens.h"

namespace gsr {
namespace surfel {

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

template <int LENS>
constexpr int lens_consts() {
    return LENS == GSR_SURFEL_LENS_FISHEYE ? GSR_FISHEYE_CONSTS : GSR_DISTORTION_CONSTS;
}

// one pixel per thread: the lens inverted at the pixel centre in fp64, the unit ray stored in fp32 (0: no ray)
template <int LENS>
__global__ void __launch_bounds__(256, 1)
    k_surfel_rays(int H, int W, const float* __restrict__ Kdev, const float* __restrict__ lens,
                  float* __restrict__ rays) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const int px = i % W, py = i / W;
    const double fx = Kdev[0], cx = Kdev[2], fy = Kdev[4], cy = Kdev[5];
    double d[3];
    lens_ray(LENS, ((double)px - cx) / fx, ((double)py - cy) / fy, lens, d);
#pragma unroll
    for (int k = 0; k < 3; ++k) rays[(size_t)i * 3 + k] = (float)d[k];
}

template <int N_SH, int LENS>
__global__ void __launch_bounds__(PRE)
    k_surfel_lens_fwd(int N, const float* __restrict__ xyz, const float* __restrict__ xyz_cam, int cam_first,
                      const float* __restrict__ quat, const float* __restrict__ scale,
                      const float* __restrict__ opa_logit, const float* __restrict__ rgb_dc,
                      const float* __restrict__ sh_rest, const float* __restrict__ Tdev, const float* __restrict__ Kdev,
                      const float* __restrict__ camdev, float width, float height, float near_t, float far_t,
                      float pad, float mh, int ntx, int nty, uint32_t depth_base, float* __restrict__ surfels,
                      float* __restrict__ bins, uint32_t* __restrict__ zkey, uint8_t* __restrict__ visible,
                      uint64_t* __restrict__ packed, uint64_t* __restrict__ tile_mask, uint32_t* __restrict__ tile_win,
                      const float* __restrict__ lens) {
    __shared__ float skc[LENS_CONSTS];
    if (threadIdx.x >= 32 && threadIdx.x < 32 + lens_consts<LENS>()) skc[threadIdx.x - 32] = lens[threadIdx.x - 32];
    surfel_fwd<N_SH, LENS>(N, xyz, xyz_cam, cam_first, quat, scale, opa_logit, rgb_dc, sh_rest, Tdev, Kdev, camdev,
                           width, height, near_t, far_t, pad, mh, ntx, nty, depth_base, surfels, bins, zkey, visible,
                           packed, tile_mask, tile_win, skc);
}

__global__ void __launch_bounds__(PIX)
    k_surfel_lens_render_fwd(const float* __restrict__ surfels, const uint64_t* __restrict__ keys, int id_bits,
                             const int32_t* __restrict__ ids, const int32_t* __restrict__ ranges,
                             const float* __restrict__ bg, int H, int W, float near_t, float ms, float r2,
                             const float* __restrict__ rays, float* __restrict__ image, float* __restrict__ depth,
                             float* __restrict__ alpha, float* __restrict__ normal, float* __restrict__ distortion,
                             int32_t* __restrict__ last, float* __restrict__ totals) {
    surfel_render_fwd<true>(surfels, keys, id_bits, ids, ranges, bg, H, W, near_t, ms, r2, rays, image, depth, alpha,
                            normal, distortion, last, totals);
}

__global__ void __launch_bounds__(PIX)
    k_surfel_lens_render_bwd(const float* __restrict__ surfels, const uint64_t* __restrict__ keys, int id_bits,
                             const int32_t* __restrict__ ids, const int32_t* __restrict__ ranges,
                             const float* __restrict__ bg, int H, int W, float near_t, float ms, float r2,
                             const float* __restrict__ rays, const float* __restrict__ alpha,
                             const int32_t* __restrict__ last, const float* __restrict__ totals,
                             const float* __restrict__ g_img, const float* __restrict__ g_dep,
                             const float* __restrict__ g_alp, const float* __restrict__ g_nrm,
                             const float* __restrict__ g_dis, float* __restrict__ rows) {
    surfel_render_bwd_rays(surfels, keys, id_bits, ids, ranges, bg, H, W, near_t, ms, r2, rays, alpha, last, totals,
                           g_img, g_dep, g_alp, g_nrm, g_dis, rows);
}

template <int LENS>
__global__ void k_surfel_lens_uv_grad(int M, const int32_t* __restrict__ vis_idx, const float* __restrict__ surfels,
                                      const float* __restrict__ rows, const float* __restrict__ Kdev,
                                      const float* __restrict__ lens, float* __restrict__ out) {
    __shared__ float sK[9], skc[LENS_CONSTS];
    if (threadIdx.x < 9) sK[threadIdx.x] = Kdev[threadIdx.x];
    else if (threadIdx.x >= 32 && threadIdx.x < 32 + lens_consts<LENS>()) skc[threadIdx.x - 32] = lens[threadIdx.x - 32];
    __syncthreads();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= M) return;
    const size_t i = (size_t)vis_idx[k];
    reinterpret_cast<float2*>(out)[k] = uv_grad_of<LENS>(surfels + i * SF, rows + i * SG, sK, skc);
}

template <int N_SH, int LENS>
__global__ void __launch_bounds__(PRE)
    k_surfel_lens_bwd(int N, const float* __restrict__ xyz, const float* __restrict__ quat,
                      const float* __restrict__ scale, const float* __restrict__ opa_logit,
                      const float* __restrict__ Tdev, const float* __restrict__ Kdev,
                      const float* __restrict__ camdev, const uint8_t* __restrict__ visible,
                      const float* __restrict__ surfels, const float* __restrict__ rows,
                      const float* __restrict__ g_uv_compact, const uint64_t* __restrict__ scan, int uv_emitted,
                      float* __restrict__ o_xyz, float* __restrict__ o_quat, float* __restrict__ o_scale,
                      float* __restrict__ o_opa, float* __restrict__ o_dc, float* __restrict__ o_sh,
                      const float* __restrict__ lens) {
    __shared__ float skc[LENS_CONSTS];
    if (threadIdx.x >= 32 && threadIdx.x < 32 + lens_consts<LENS>()) skc[threadIdx.x - 32] = lens[threadIdx.x - 32];
    surfel_bwd<N_SH, LENS>(N, xyz, quat, scale, opa_logit, Tdev, Kdev, camdev, visible, surfels, rows, g_uv_compact,
                           scan, uv_emitted, o_xyz, o_quat, o_scale, o_opa, o_dc, o_sh, skc);
}

}  // namespace surfel
}  // namespace gsr

using namespace gsr;
using namespace gsr::surfel;

static bool n_sh_ok(int n) { return n == 0 || n == 3 || n == 8 || n == 15; }
static bool lens_ok(int lens) { return lens == GSR_SURFEL_LENS_FISHEYE || lens == GSR_SURFEL_LENS_DISTORTION; }
static bool pairs_ok(const uint64_t* keys, int id_bits, const int32_t* ids) {
    return (keys != nullptr) != (ids != nullptr) && (keys == nullptr || (id_bits >= 1 && id_bits <= 32));
}

// n_sh_rest -> N_SH, then the lens (both checked by the caller)
#define GSR_SURFEL_LENS_SWITCH(LAUNCH)                                                          \
    switch (n_sh_rest) {                                                                         \
        case 0: if (lens == GSR_SURFEL_LENS_FISHEYE) LAUNCH(1, 1); else LAUNCH(1, 2); break;     \
        case 3: if (lens == GSR_SURFEL_LENS_FISHEYE) LAUNCH(4, 1); else LAUNCH(4, 2); break;     \
        case 8: if (lens == GSR_SURFEL_LENS_FISHEYE) LAUNCH(9, 1); else LAUNCH(9, 2); break;     \
        default: if (lens == GSR_SURFEL_LENS_FISHEYE) LAUNCH(16, 1); else LAUNCH(16, 2); break;  \
    }

extern "C" {

int gsr_surfel_rays(int lens, int H, int W, const float* K, const float* lens_consts, float* rays, void* stream) {
    if (!lens_ok(lens) || H <= 0 || W <= 0 || !K || !lens_consts || !rays) return GSR_ERR_BAD_ARG;
    const int n = H * W;
    cudaStream_t st = (cudaStream_t)stream;
    if (lens == GSR_SURFEL_LENS_FISHEYE)
        k_surfel_rays<GSR_SURFEL_LENS_FISHEYE><<<(n + 255) / 256, 256, 0, st>>>(H, W, K, lens_consts, rays);
    else
        k_surfel_rays<GSR_SURFEL_LENS_DISTORTION><<<(n + 255) / 256, 256, 0, st>>>(H, W, K, lens_consts, rays);
    return (int)cudaGetLastError();
}

int gsr_surfel_lens_preprocess_forward(int lens, int N, int n_sh_rest, const float* xyz, const float* xyz_camera_frame,
                                       int cam_first, const float* quaternion, const float* scale,
                                       const float* opacity_logit, const float* rgb_dc, const float* sh_rest,
                                       const float* camera_T_world, const float* K, const float* camera_centre, int H,
                                       int W, float near_thresh, float far_thresh, float cull_mask_padding,
                                       float mh_dist, uint32_t depth_base, float* surfels, float* bin_records,
                                       uint32_t* depth_key, uint8_t* visible, uint64_t* scan, uint64_t* tile_mask,
                                       uint32_t* tile_win, void* temp, size_t temp_bytes, const float* lens_consts,
                                       void* stream) {
    if (!lens_ok(lens) || N < 0 || H <= 0 || W <= 0 || !n_sh_ok(n_sh_rest) || !(mh_dist > 0.0f))
        return GSR_ERR_BAD_ARG;
    if (N == 0) return GSR_OK;
    if (!xyz || !quaternion || !scale || !opacity_logit || !rgb_dc || !camera_T_world || !K || !surfels ||
        !bin_records || !depth_key || !visible || !scan || !temp || !lens_consts)
        return GSR_ERR_BAD_ARG;
    if (n_sh_rest > 0 && (!sh_rest || !camera_centre)) return GSR_ERR_BAD_ARG;
    if ((tile_mask == nullptr) != (tile_win == nullptr)) return GSR_ERR_BAD_ARG;
    if (((uintptr_t)surfels | (uintptr_t)bin_records) & 15u) return GSR_ERR_BAD_ARG;
    size_t scan_bytes = 0;
    cub::DeviceScan::InclusiveSum((void*)nullptr, scan_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, N);
    if (temp_bytes < align256(scan_bytes) + align256(sizeof(uint64_t) * (size_t)N)) return GSR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    uint64_t* packed = reinterpret_cast<uint64_t*>((char*)temp + align256(scan_bytes));
    const int ntx = (W + TILE - 1) / TILE, nty = (H + TILE - 1) / TILE;
    const dim3 grid((N + PRE - 1) / PRE), block(PRE);
#define GSR_SURFEL_LENS_FWD(NS, L)                                                                                     \
    k_surfel_lens_fwd<NS, L><<<grid, block, 0, st>>>(N, xyz, xyz_camera_frame, cam_first, quaternion, scale,          \
                                                     opacity_logit, rgb_dc, sh_rest, camera_T_world, K, camera_centre, \
                                                     (float)W, (float)H, near_thresh, far_thresh, cull_mask_padding,   \
                                                     mh_dist, ntx, nty, depth_base, surfels, bin_records, depth_key,   \
                                                     visible, packed, tile_mask, tile_win, lens_consts)
    GSR_SURFEL_LENS_SWITCH(GSR_SURFEL_LENS_FWD)
#undef GSR_SURFEL_LENS_FWD
    cudaError_t e = cub::DeviceScan::InclusiveSum(temp, scan_bytes, packed, scan, N, st);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

int gsr_surfel_lens_render_forward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                                   const int32_t* ids_sorted, const int32_t* tile_ranges, const float* background_rgb,
                                   int H, int W, float near_thresh, float m_scale, float mh_dist, const float* rays,
                                   float* image, float* depth, float* alpha, float* normal, float* distortion,
                                   int32_t* last, float* totals, void* stream) {
    if (H <= 0 || W <= 0 || !(mh_dist > 0.0f) || !pairs_ok(keys_sorted, id_bits, ids_sorted)) return GSR_ERR_BAD_ARG;
    if (!surfels || !tile_ranges || !background_rgb || !rays || !image || !depth || !alpha || !normal || !distortion ||
        !last || !totals || ((uintptr_t)surfels & 15u))
        return GSR_ERR_BAD_ARG;
    const int n_tiles = ((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE);
    k_surfel_lens_render_fwd<<<n_tiles, PIX, 0, (cudaStream_t)stream>>>(
        surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, background_rgb, H, W, near_thresh, m_scale,
        mh_dist * mh_dist, rays, image, depth, alpha, normal, distortion, last, totals);
    return (int)cudaGetLastError();
}

int gsr_surfel_lens_render_backward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                                    const int32_t* ids_sorted, const int32_t* tile_ranges, const float* background_rgb,
                                    int H, int W, float near_thresh, float m_scale, float mh_dist, const float* rays,
                                    const float* alpha, const int32_t* last, const float* totals,
                                    const float* grad_image, const float* grad_depth, const float* grad_alpha,
                                    const float* grad_normal, const float* grad_distortion, float* grad_rows,
                                    void* stream) {
    if (H <= 0 || W <= 0 || !(mh_dist > 0.0f) || !pairs_ok(keys_sorted, id_bits, ids_sorted)) return GSR_ERR_BAD_ARG;
    if (!surfels || !tile_ranges || !background_rgb || !rays || !alpha || !last || !totals || !grad_image ||
        !grad_depth || !grad_alpha || !grad_normal || !grad_distortion || !grad_rows ||
        (((uintptr_t)surfels | (uintptr_t)grad_rows) & 15u))
        return GSR_ERR_BAD_ARG;
    const int n_tiles = ((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE);
    k_surfel_lens_render_bwd<<<n_tiles, PIX, 0, (cudaStream_t)stream>>>(
        surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, background_rgb, H, W, near_thresh, m_scale,
        mh_dist * mh_dist, rays, alpha, last, totals, grad_image, grad_depth, grad_alpha, grad_normal, grad_distortion,
        grad_rows);
    return (int)cudaGetLastError();
}

int gsr_surfel_lens_uv_grad(int lens, int M, const int32_t* vis_idx, const float* surfels, const float* grad_rows,
                            const float* K, const float* lens_consts, float* uv_grad, void* stream) {
    if (!lens_ok(lens) || M < 0) return GSR_ERR_BAD_ARG;
    if (M == 0) return GSR_OK;
    if (!vis_idx || !surfels || !grad_rows || !K || !lens_consts || !uv_grad || ((uintptr_t)uv_grad & 7u))
        return GSR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (lens == GSR_SURFEL_LENS_FISHEYE)
        k_surfel_lens_uv_grad<GSR_SURFEL_LENS_FISHEYE><<<(M + 255) / 256, 256, 0, st>>>(M, vis_idx, surfels, grad_rows,
                                                                                        K, lens_consts, uv_grad);
    else
        k_surfel_lens_uv_grad<GSR_SURFEL_LENS_DISTORTION><<<(M + 255) / 256, 256, 0, st>>>(
            M, vis_idx, surfels, grad_rows, K, lens_consts, uv_grad);
    return (int)cudaGetLastError();
}

int gsr_surfel_lens_preprocess_backward(int lens, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                                        const float* scale, const float* opacity_logit, const float* camera_T_world,
                                        const float* K, const float* camera_centre, const uint8_t* visible,
                                        const float* surfels, const float* grad_rows, const float* grad_uv_compact,
                                        const uint64_t* scan, int uv_grad_emitted, float* g_xyz, float* g_quaternion,
                                        float* g_scale, float* g_opacity_logit, float* g_rgb_dc, float* g_sh_rest,
                                        const float* lens_consts, void* stream) {
    if (!lens_ok(lens) || N < 0 || !n_sh_ok(n_sh_rest)) return GSR_ERR_BAD_ARG;
    if (N == 0) return GSR_OK;
    if (!xyz || !quaternion || !scale || !opacity_logit || !camera_T_world || !K || !visible || !surfels ||
        !grad_rows || !g_xyz || !g_quaternion || !g_scale || !g_opacity_logit || !g_rgb_dc || !lens_consts)
        return GSR_ERR_BAD_ARG;
    if (n_sh_rest > 0 && (!camera_centre || !g_sh_rest)) return GSR_ERR_BAD_ARG;
    if (grad_uv_compact != nullptr && scan == nullptr) return GSR_ERR_BAD_ARG;
    if (((uintptr_t)surfels | (uintptr_t)grad_rows) & 15u) return GSR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid((N + PRE - 1) / PRE), block(PRE);
#define GSR_SURFEL_LENS_BWD(NS, L)                                                                                    \
    k_surfel_lens_bwd<NS, L><<<grid, block, 0, st>>>(N, xyz, quaternion, scale, opacity_logit, camera_T_world, K,    \
                                                     camera_centre, visible, surfels, grad_rows, grad_uv_compact,    \
                                                     scan, uv_grad_emitted ? 1 : 0, g_xyz, g_quaternion, g_scale,    \
                                                     g_opacity_logit, g_rgb_dc, g_sh_rest, lens_consts)
    GSR_SURFEL_LENS_SWITCH(GSR_SURFEL_LENS_BWD)
#undef GSR_SURFEL_LENS_BWD
    return (int)cudaGetLastError();
}

}  // extern "C"
