// gsr_lens.cu — the fused per-gaussian stages for a lens model, compiled once per lens:
//   GSR_LENS 1: fisheye cameras (rasterize(..., fisheye=k), libgsr_fisheye.so, gsr_fisheye.h)
//   GSR_LENS 2: radial-tangential distortion (rasterize(..., distortion=k), libgsr_distortion.so, gsr_distortion.h)
//
// The bodies are the pinhole ones of gsr_preprocess.cuh — forward, single-view backward and batched backward —
// compiled with the camera-model hooks of COLMAP's OPENCV_FISHEYE model (gsr_fisheye.cuh) or OPENCV model
// (gsr_distortion.cuh).  Each view's lens constants ({k1, k2, k3, k4, theta_max} or {k1, k2, p1, p2, k3, r2_max}) are
// read into shared memory next to the view constants, by threads 32.. while threads 0..27 fetch T, K and the camera
// centre.  The records these kernels write are ordinary records: binning and the tile kernels run unchanged.
#include <cub/cub.cuh>

#include <cmath>

// LENS_NAME(a, b): a<lens>b, so each library keeps its own kernel and C symbol names
#if GSR_LENS == 1
#define GSR_FISHEYE_HOOKS
#include "gsr_fisheye.cuh"
#include "../../include/gsr_fisheye.h"
#define LENS_NAME(a, b) a##fisheye##b
#elif GSR_LENS == 2
#define GSR_DISTORTION_HOOKS
#include "gsr_distortion.cuh"
#include "../../include/gsr_distortion.h"
#define LENS_NAME(a, b) a##distortion##b
#else
#error "GSR_LENS must be 1 (fisheye) or 2 (distortion)"
#endif
#include "gsr_poly_roots.h"

#include "gsr_preprocess.cuh"

namespace gsr {

// CTAs per SM the register budget is sized for (-Xptxas -v: no local memory at these bounds, DESIGN.md 3.19, 3.20)
#ifndef GSR_LENS_FWD_MINB
#define GSR_LENS_FWD_MINB 6
#endif
#ifndef GSR_LENS_BWD_MINB
#define GSR_LENS_BWD_MINB 4
#endif
#ifndef GSR_LENS_BATCH_MINB
#define GSR_LENS_BATCH_MINB 3
#endif

template <int N_SH, bool HAS_SH, bool ANTIALIAS, bool FILTER3D>
__global__ void __launch_bounds__(PRE_THREADS, GSR_LENS_FWD_MINB)
    LENS_NAME(k_, _preprocess_fwd)(GSR_PRE_FWD_PARAMS, const float* __restrict__ filter3d,
                                   const float* __restrict__ lens) {
    preprocess_fwd<N_SH, HAS_SH, ANTIALIAS, FILTER3D>(GSR_PRE_FWD_FORWARD, filter3d, lens);
}

#define GSR_PRE_BWD_PARAMS                                                                                          \
    int N, const float* __restrict__ xyz, const float* __restrict__ quat, const float* __restrict__ scale,          \
        const float* __restrict__ opa_logit, const float* __restrict__ Tdev, const float* __restrict__ Kdev,        \
        const float* __restrict__ camdev, const uint8_t* __restrict__ visible, const float* __restrict__ g_rows,    \
        int rows_uv, const float* __restrict__ g_uv_compact, const uint64_t* __restrict__ scan,                      \
        float* __restrict__ o_xyz, float* __restrict__ o_quat, float* __restrict__ o_scale,                         \
        float* __restrict__ o_opa, float* __restrict__ o_dc, float* __restrict__ o_sh, int use_tma,                 \
        const float* __restrict__ filter3d, const float* __restrict__ lens
template <int N_SH, bool HAS_SH, bool DEPTH, bool ANTIALIAS, bool FILTER3D>
__global__ void __launch_bounds__(PRE_THREADS, GSR_LENS_BWD_MINB) LENS_NAME(k_, _preprocess_bwd)(GSR_PRE_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, DEPTH, ANTIALIAS, FILTER3D>(N, xyz, quat, scale, opa_logit, Tdev, Kdev, camdev,
                                                             visible, g_rows, rows_uv, g_uv_compact, scan, o_xyz,
                                                             o_quat, o_scale, o_opa, o_dc, o_sh, use_tma, filter3d,
                                                             lens);
}
template <int N_SH, bool HAS_SH, bool DEPTH, bool ANTIALIAS, bool FILTER3D>
__global__ void __launch_bounds__(PRE_THREADS, GSR_LENS_BATCH_MINB)
    LENS_NAME(k_, _batch_preprocess_bwd)(int C, GSR_PRE_BWD_PARAMS) {
    batch_preprocess_bwd<N_SH, HAS_SH, DEPTH, ANTIALIAS, FILTER3D>(C, N, xyz, quat, scale, opa_logit, Tdev, Kdev,
                                                                   camdev, visible, g_rows, rows_uv, g_uv_compact,
                                                                   scan, o_xyz, o_quat, o_scale, o_opa, o_dc, o_sh,
                                                                   use_tma, filter3d, lens);
}
#undef GSR_PRE_BWD_PARAMS

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

constexpr int KNOWN_MODES = GSR_MODE_DEPTH_ALPHA | GSR_MODE_ANTIALIASED | GSR_MODE_ABSGRAD | GSR_MODE_FILTER3D;

// n_sh_rest -> the SH template arguments
#define GSR_LENS_SH_SWITCH(LAUNCH)          \
    switch (n_sh_rest) {                    \
        case 0: LAUNCH(1, false); break;    \
        case 3: LAUNCH(4, true); break;     \
        case 8: LAUNCH(9, true); break;     \
        case 15: LAUNCH(16, true); break;   \
        default: return GSR_ERR_UNSUPPORTED; \
    }

template <bool AA, bool F3D>
static int launch_fwd(int n_sh_rest, dim3 grid, cudaStream_t st, int N, const float* xyz, const float* xyz_cam,
                      int cam_first, const float* quat, const float* scale, const float* opa, const float* dc,
                      const float* sh, const float* T, const float* K, const float* cam, float width, float height,
                      float near_t, float far_t, float pad, float mh, int ntx, int nty, uint32_t depth_base,
                      float* records, uint32_t* zkey, uint8_t* visible, uint64_t* packed, uint64_t* tile_mask,
                      uint32_t* tile_win, int use_tma, const float* filter3d, const float* lens) {
#define GSR_LENS_FWD(NSH, HSH)                                                                                      \
    LENS_NAME(k_, _preprocess_fwd)<NSH, HSH, AA, F3D><<<grid, PRE_THREADS, 0, st>>>(                                \
        N, xyz, xyz_cam, cam_first, quat, scale, opa, dc, sh, T, K, cam, width, height, near_t, far_t, pad, mh, ntx, \
        nty, depth_base, records, zkey, visible, packed, tile_mask, tile_win, use_tma, filter3d, lens)
    GSR_LENS_SH_SWITCH(GSR_LENS_FWD)
#undef GSR_LENS_FWD
    return GSR_OK;
}

#define GSR_LENS_BWD_ARGS_DECL                                                                                     \
    int n_sh_rest, dim3 grid, cudaStream_t st, int N, const float *xyz, const float *quat, const float *scale,     \
        const float *opa, const float *T, const float *K, const float *cam, const uint8_t *visible,                \
        const float *rows, int rows_uv, const float *g_uv, const uint64_t *scan, float *o_xyz, float *o_quat,      \
        float *o_scale, float *o_opa, float *o_dc, float *o_sh, int use_tma, const float *filter3d,                \
        const float *lens
#define GSR_LENS_BWD_ARGS                                                                                           \
    N, xyz, quat, scale, opa, T, K, cam, visible, rows, rows_uv, g_uv, scan, o_xyz, o_quat, o_scale, o_opa, o_dc,    \
        o_sh, use_tma, filter3d, lens

template <bool DEPTH, bool AA, bool F3D>
static int launch_bwd(GSR_LENS_BWD_ARGS_DECL) {
#define GSR_LENS_BWD(NSH, HSH) \
    LENS_NAME(k_, _preprocess_bwd)<NSH, HSH, DEPTH, AA, F3D><<<grid, PRE_THREADS, 0, st>>>(GSR_LENS_BWD_ARGS)
    GSR_LENS_SH_SWITCH(GSR_LENS_BWD)
#undef GSR_LENS_BWD
    return GSR_OK;
}

template <bool DEPTH, bool AA, bool F3D>
static int launch_batch_bwd(int C, GSR_LENS_BWD_ARGS_DECL) {
#define GSR_LENS_BWD(NSH, HSH) \
    LENS_NAME(k_, _batch_preprocess_bwd)<NSH, HSH, DEPTH, AA, F3D><<<grid, PRE_THREADS, 0, st>>>(C, GSR_LENS_BWD_ARGS)
    GSR_LENS_SH_SWITCH(GSR_LENS_BWD)
#undef GSR_LENS_BWD
    return GSR_OK;
}

// the 8 (depth, antialiased, filter3d) instantiations of a backward launcher, selected by the mode bits
#define GSR_LENS_MODE_DISPATCH(launcher, ...)                                                           \
    (f3d ? (aa ? (depth ? launcher<true, true, true>(__VA_ARGS__) : launcher<false, true, true>(__VA_ARGS__))   \
               : (depth ? launcher<true, false, true>(__VA_ARGS__) : launcher<false, false, true>(__VA_ARGS__))) \
         : (aa ? (depth ? launcher<true, true, false>(__VA_ARGS__) : launcher<false, true, false>(__VA_ARGS__))  \
               : (depth ? launcher<true, false, false>(__VA_ARGS__) : launcher<false, false, false>(__VA_ARGS__))))

}  // namespace gsr

using namespace gsr;

extern "C" {

// The cull limit of the lens's constants (the last value of each view's group)
#if GSR_LENS == 1
float gsr_fisheye_theta_max(const float* k) {
    if (k == nullptr) return NAN;
    for (int i = 0; i < 4; ++i)
        if (!std::isfinite(k[i])) return NAN;
    const double half_pi = 1.5707963267948966;
    // d theta_d / d theta as a polynomial in t = theta^2
    const double c[5] = {1.0, 3.0 * k[0], 5.0 * k[1], 7.0 * k[2], 9.0 * k[3]};
    double roots[4];
    const int n = roots_in(c, 4, 0.0, half_pi * half_pi, roots);
    double th = half_pi;
    for (int i = 0; i < n; ++i)
        if (roots[i] > 0.0) { th = std::sqrt(roots[i]); break; }
    float f = (float)th;
    if ((double)f > th) f = std::nextafter(f, 0.0f);  // round down: the cull never admits a folded theta
    return f;
}
#elif GSR_LENS == 2
float gsr_distortion_r2_max(const float* k) {
    if (k == nullptr) return NAN;
    for (int i = 0; i < 5; ++i)
        if (!std::isfinite(k[i])) return NAN;
    // d (r radial(r^2)) / dr as a polynomial in s = r^2; c[0] = 1 > 0, so every positive root is below the Cauchy bound
    const double c[4] = {1.0, 3.0 * k[0], 5.0 * k[1], 7.0 * k[4]};
    int n = 3;
    while (n > 0 && c[n] == 0.0) --n;
    if (n == 0) return INFINITY;
    double bound = 0.0;
    for (int i = 0; i < n; ++i) bound = std::fmax(bound, std::fabs(c[i] / c[n]));
    double roots[3];
    const int m = roots_in(c, n, 0.0, 1.0 + bound, roots);
    for (int i = 0; i < m; ++i)
        if (roots[i] > 0.0) {
            float f = (float)roots[i];
            if ((double)f > roots[i]) f = std::nextafter(f, 0.0f);  // round down: the cull never admits a folded s
            return f;
        }
    return INFINITY;
}
#endif

int LENS_NAME(gsr_, _preprocess_forward)(int mode, int N, int n_sh_rest, const float* xyz,
                                         const float* xyz_camera_frame, int cam_first, const float* quaternion,
                                         const float* scale, const float* opacity_logit, const float* filter3d,
                                         const float* rgb_dc, const float* sh_rest, const float* camera_T_world,
                                         const float* K, const float* camera_centre, int H, int W, float near_thresh,
                                         float far_thresh, float cull_mask_padding, float mh_dist,
                                         uint32_t depth_base, float* records, uint32_t* depth_key, uint8_t* visible,
                                         uint64_t* scan, uint64_t* tile_mask, uint32_t* tile_win, void* temp,
                                         size_t temp_bytes, const float* lens, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if ((mode & ~KNOWN_MODES) != 0) return GSR_ERR_BAD_ARG;
    if (((mode & GSR_MODE_FILTER3D) != 0) != (filter3d != nullptr)) return GSR_ERR_BAD_ARG;
    if (N < 0 || lens == nullptr) return GSR_ERR_BAD_ARG;
    if (N == 0) return GSR_OK;
    size_t scan_bytes = 0;
    cub::DeviceScan::InclusiveSum((void*)nullptr, scan_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, N);
    if (temp == nullptr || temp_bytes < align256(scan_bytes) + align256(sizeof(uint64_t) * (size_t)N))
        return GSR_ERR_BAD_ARG;
    if ((tile_mask == nullptr) != (tile_win == nullptr)) return GSR_ERR_BAD_ARG;
    uint64_t* packed = reinterpret_cast<uint64_t*>((char*)temp + align256(scan_bytes));
    const int ntx = (W + TILE - 1) / TILE, nty = (H + TILE - 1) / TILE;
    const dim3 grid((N + PRE_THREADS - 1) / PRE_THREADS);
    const int use_tma = (aligned16(records) && (sh_rest == nullptr || aligned16(sh_rest))) ? 1 : 0;
    const bool aa = (mode & GSR_MODE_ANTIALIASED) != 0, f3d = (mode & GSR_MODE_FILTER3D) != 0;
#define GSR_FWD_ARGS                                                                                                \
    n_sh_rest, grid, st, N, xyz, xyz_camera_frame, cam_first, quaternion, scale, opacity_logit, rgb_dc, sh_rest,     \
        camera_T_world, K, camera_centre, (float)W, (float)H, near_thresh, far_thresh, cull_mask_padding, mh_dist,   \
        ntx, nty, depth_base, records, depth_key, visible, packed, tile_mask, tile_win, use_tma, filter3d, lens
    const int rc = f3d ? (aa ? launch_fwd<true, true>(GSR_FWD_ARGS) : launch_fwd<false, true>(GSR_FWD_ARGS))
                       : (aa ? launch_fwd<true, false>(GSR_FWD_ARGS) : launch_fwd<false, false>(GSR_FWD_ARGS));
#undef GSR_FWD_ARGS
    if (rc != GSR_OK) return rc;
    cudaError_t e = cub::DeviceScan::InclusiveSum(temp, scan_bytes, packed, scan, N, st);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

}  // extern "C"

// single: the single-view kernels (C is 1, no running sums); else the batched ones over C views
static int lens_backward(bool single, int mode, int C, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                         const float* scale, const float* opacity_logit, const float* filter3d,
                         const float* camera_T_world, const float* K, const float* camera_centre,
                         const uint8_t* visible, const float* grad_rows, int use_rows_uv, const float* grad_uv_compact,
                         const uint64_t* scan, float* g_xyz, float* g_quaternion, float* g_scale,
                         float* g_opacity_logit, float* g_rgb_dc, float* g_sh_rest, const float* lens, void* stream) {
    if (C < 1 || N < 0 || (mode & ~KNOWN_MODES) != 0) return GSR_ERR_BAD_ARG;
    if (((mode & GSR_MODE_FILTER3D) != 0) != (filter3d != nullptr)) return GSR_ERR_BAD_ARG;
    if (N == 0) return GSR_OK;  // nothing to launch (the arrays of an empty scene may be NULL)
    if (xyz == nullptr || quaternion == nullptr || scale == nullptr || opacity_logit == nullptr ||
        camera_T_world == nullptr || K == nullptr || visible == nullptr || grad_rows == nullptr || g_xyz == nullptr ||
        g_quaternion == nullptr || g_scale == nullptr || g_opacity_logit == nullptr || g_rgb_dc == nullptr ||
        lens == nullptr)
        return GSR_ERR_BAD_ARG;
    if ((n_sh_rest > 0) != (g_sh_rest != nullptr)) return GSR_ERR_BAD_ARG;
    if (!aligned16(grad_rows)) return GSR_ERR_BAD_ARG;
    if (grad_uv_compact != nullptr && scan == nullptr) return GSR_ERR_BAD_ARG;
    if (n_sh_rest != 0 && n_sh_rest != 3 && n_sh_rest != 8 && n_sh_rest != 15) return GSR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid((N + PRE_THREADS - 1) / PRE_THREADS);
    const int use_tma = (aligned16(g_xyz) && aligned16(g_quaternion) && aligned16(g_scale) &&
                         aligned16(g_opacity_logit) && aligned16(g_rgb_dc) &&
                         (g_sh_rest == nullptr || aligned16(g_sh_rest)))
                            ? 1
                            : 0;
    const bool depth = (mode & GSR_MODE_DEPTH_ALPHA) != 0, aa = (mode & GSR_MODE_ANTIALIASED) != 0,
               f3d = (mode & GSR_MODE_FILTER3D) != 0;
#define GSR_LENS_ARGS                                                                                              \
    n_sh_rest, grid, st, N, xyz, quaternion, scale, opacity_logit, camera_T_world, K, camera_centre, visible,        \
        grad_rows, use_rows_uv, grad_uv_compact, scan, g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc,      \
        g_sh_rest, use_tma, filter3d, lens
    const int rc = single ? GSR_LENS_MODE_DISPATCH(launch_bwd, GSR_LENS_ARGS)
                          : GSR_LENS_MODE_DISPATCH(launch_batch_bwd, C, GSR_LENS_ARGS);
#undef GSR_LENS_ARGS
    if (rc != GSR_OK) return rc;
    return (int)cudaGetLastError();
}

extern "C" {

int LENS_NAME(gsr_, _preprocess_backward)(int mode, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                                          const float* scale, const float* opacity_logit, const float* filter3d,
                                          const float* camera_T_world, const float* K, const float* camera_centre,
                                          const uint8_t* visible, const float* grad_rows, int use_rows_uv,
                                          const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                          float* g_quaternion, float* g_scale, float* g_opacity_logit,
                                          float* g_rgb_dc, float* g_sh_rest, const float* lens, void* stream) {
    return lens_backward(true, mode, 1, N, n_sh_rest, xyz, quaternion, scale, opacity_logit, filter3d, camera_T_world,
                         K, camera_centre, visible, grad_rows, use_rows_uv, grad_uv_compact, scan, g_xyz,
                         g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, lens, stream);
}

int LENS_NAME(gsr_, _batch_preprocess_backward)(int mode, int C, int N, int n_sh_rest, const float* xyz,
                                                const float* quaternion, const float* scale,
                                                const float* opacity_logit, const float* filter3d,
                                                const float* camera_T_world, const float* K,
                                                const float* camera_centre, const uint8_t* visible,
                                                const float* grad_rows, int use_rows_uv,
                                                const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                                float* g_quaternion, float* g_scale, float* g_opacity_logit,
                                                float* g_rgb_dc, float* g_sh_rest, const float* lens, void* stream) {
    return lens_backward(false, mode, C, N, n_sh_rest, xyz, quaternion, scale, opacity_logit, filter3d,
                         camera_T_world, K, camera_centre, visible, grad_rows, use_rows_uv, grad_uv_compact, scan,
                         g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, lens, stream);
}

}  // extern "C"
