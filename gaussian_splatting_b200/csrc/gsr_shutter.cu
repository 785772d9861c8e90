// gsr_shutter.cu — the fused per-gaussian stages for rolling-shutter cameras (libgsr_shutter.so, gsr_shutter.h):
// rasterize(..., rolling_shutter=xi) and rasterize_batch(..., rolling_shutter=xi).
//
// The bodies are those of gsr_preprocess.cuh — forward, single-view backward and batched backward — compiled with the
// shutter hooks of gsr_shutter.cuh, which also carry the camera row (pose and twist gradients) through the pose
// hooks' slots.  The records are ordinary records: binning and the tile kernels run unchanged.  This file is compiled
// once per camera model, GSR_SHUTTER_LENS 0 (pinhole), 1 (gsr_fisheye.cuh's hooks) or 2 (gsr_distortion.cuh's hooks);
// each compile puts its kernels in a namespace of its own and exports hidden launchers, and the compile with
// GSR_SHUTTER_LENS == 0 also holds the fp64 finishing kernel and the C ABI, which dispatch on the lens.
#include <cub/cub.cuh>

#include <cstdint>

#include "../../include/gsr_distortion.h"
#include "../../include/gsr_fisheye.h"
#include "../../include/gsr_pose.h"
#include "../../include/gsr_shutter.h"

#ifndef GSR_SHUTTER_LENS
#define GSR_SHUTTER_LENS 0
#endif

#if GSR_SHUTTER_LENS == 1
#define GSR_FISHEYE_HOOKS
#include "gsr_fisheye.cuh"
#define GSR_SH_LENS_ARG , lens
#define GSR_SH_NS shutter_fisheye
#define GSR_SH_LAUNCH_FWD gsr_shutter_launch_fwd_fisheye
#define GSR_SH_LAUNCH_BWD gsr_shutter_launch_bwd_fisheye
#define camera_centre camera_centre_shutter_fisheye
#elif GSR_SHUTTER_LENS == 2
#define GSR_DISTORTION_HOOKS
#include "gsr_distortion.cuh"
#define GSR_SH_LENS_ARG , lens
#define GSR_SH_NS shutter_distortion
#define GSR_SH_LAUNCH_FWD gsr_shutter_launch_fwd_distortion
#define GSR_SH_LAUNCH_BWD gsr_shutter_launch_bwd_distortion
#define camera_centre camera_centre_shutter_distortion
#else
#define GSR_SH_LENS_ARG
#define GSR_SH_NS shutter_pinhole
#define GSR_SH_LAUNCH_FWD gsr_shutter_launch_fwd_pinhole
#define GSR_SH_LAUNCH_BWD gsr_shutter_launch_bwd_pinhole
#define camera_centre camera_centre_shutter_pinhole
#endif

#include "gsr_common.cuh"
#include "gsr_pose.cuh"  // pose_cta_reduce, finish_partials; its hooks are replaced by gsr_shutter.cuh's
#undef GSR_POSE_HOOKS
#undef GSR_POSE_PARAM
#undef GSR_POSE_DECL
#undef GSR_POSE_VIEW
#undef GSR_POSE_REDUCE
#include "gsr_shutter.cuh"
#include "gsr_preprocess.cuh"

// CTAs per SM the register budget is sized for (-Xptxas -v: no local memory at these bounds, DESIGN.md 3.24)
#ifndef GSR_SHUTTER_FWD_MINB
#define GSR_SHUTTER_FWD_MINB 6
#endif
#ifndef GSR_SHUTTER_BWD_MINB
#define GSR_SHUTTER_BWD_MINB 3
#endif
#ifndef GSR_SHUTTER_BATCH_MINB
#define GSR_SHUTTER_BATCH_MINB 2
#endif

#define GSR_SH_FWD_DECL(name)                                                                                        \
    __attribute__((visibility("hidden"))) int name(                                                                 \
        int mode, int n_sh_rest, int N, const float* xyz, const float* xyz_cam, int cam_first, const float* quat,    \
        const float* scale, const float* opa, const float* dc, const float* sh, const float* T, const float* K,       \
        const float* cam, float width, float height, float near_t, float far_t, float pad, float mh, int ntx,        \
        int nty, uint32_t depth_base, float* records, uint32_t* zkey, uint8_t* visible, uint64_t* packed,            \
        uint64_t* tile_mask, uint32_t* tile_win, int use_tma, const float* filter3d, const float* lens,              \
        const float* xi, float r0, float e0, float e1, cudaStream_t st)
#define GSR_SH_BWD_DECL(name)                                                                                        \
    __attribute__((visibility("hidden"))) int name(                                                                 \
        bool single, int mode, int C, int N, int n_sh_rest, const float* xyz, const float* quat, const float* scale, \
        const float* opa, const float* filter3d, const float* T, const float* K, const float* cam,                  \
        const uint8_t* visible, const float* rows, int rows_uv, const float* g_uv, const uint64_t* scan,            \
        float* o_xyz, float* o_quat, float* o_scale, float* o_opa, float* o_dc, float* o_sh, int use_tma,           \
        const float* lens, const float* xi, float r0, float e0, float e1, float* partials, cudaStream_t st)

namespace gsr {
static_assert(POSE_CTA_THREADS == PRE_THREADS, "pose_cta_reduce sums one CTA of the bodies");
namespace GSR_SH_NS {

#define GSR_SH_SHUTTER_PARAMS \
    const float* __restrict__ shutter_xi, float sh_r0, float sh_e0, float sh_e1
template <int N_SH, bool HAS_SH, bool ANTIALIAS, bool FILTER3D>
__global__ void __launch_bounds__(PRE_THREADS, GSR_SHUTTER_FWD_MINB)
    k_shutter_preprocess_fwd(GSR_PRE_FWD_PARAMS, const float* __restrict__ filter3d, const float* __restrict__ lens,
                             GSR_SH_SHUTTER_PARAMS) {
    preprocess_fwd<N_SH, HAS_SH, ANTIALIAS, FILTER3D>(GSR_PRE_FWD_FORWARD, filter3d GSR_SH_LENS_ARG, shutter_xi, sh_r0,
                                                      sh_e0, sh_e1);
}

#define GSR_SH_BWD_PARAMS                                                                                           \
    int N, const float* __restrict__ xyz, const float* __restrict__ quat, const float* __restrict__ scale,          \
        const float* __restrict__ opa_logit, const float* __restrict__ Tdev, const float* __restrict__ Kdev,        \
        const float* __restrict__ camdev, const uint8_t* __restrict__ visible, const float* __restrict__ g_rows,    \
        int rows_uv, const float* __restrict__ g_uv_compact, const uint64_t* __restrict__ scan,                      \
        float* __restrict__ o_xyz, float* __restrict__ o_quat, float* __restrict__ o_scale,                         \
        float* __restrict__ o_opa, float* __restrict__ o_dc, float* __restrict__ o_sh, int use_tma,                 \
        const float* __restrict__ filter3d, const float* __restrict__ lens, GSR_SH_SHUTTER_PARAMS,                  \
        float* __restrict__ partials
#define GSR_SH_BWD_FORWARD                                                                                          \
    N, xyz, quat, scale, opa_logit, Tdev, Kdev, camdev, visible, g_rows, rows_uv, g_uv_compact, scan, o_xyz, o_quat, \
        o_scale, o_opa, o_dc, o_sh, use_tma, filter3d GSR_SH_LENS_ARG, shutter_xi, sh_r0, sh_e0, sh_e1, partials
template <int N_SH, bool HAS_SH, bool DEPTH, bool ANTIALIAS, bool FILTER3D>
__global__ void __launch_bounds__(PRE_THREADS, GSR_SHUTTER_BWD_MINB) k_shutter_preprocess_bwd(GSR_SH_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, DEPTH, ANTIALIAS, FILTER3D>(GSR_SH_BWD_FORWARD);
}
template <int N_SH, bool HAS_SH, bool DEPTH, bool ANTIALIAS, bool FILTER3D>
__global__ void __launch_bounds__(PRE_THREADS, GSR_SHUTTER_BATCH_MINB)
    k_shutter_batch_preprocess_bwd(int C, GSR_SH_BWD_PARAMS) {
    batch_preprocess_bwd<N_SH, HAS_SH, DEPTH, ANTIALIAS, FILTER3D>(C, GSR_SH_BWD_FORWARD);
}
#undef GSR_SH_BWD_PARAMS
#undef GSR_SH_BWD_FORWARD
#undef GSR_SH_SHUTTER_PARAMS

#define GSR_SH_SWITCH(LAUNCH)                 \
    switch (n_sh_rest) {                      \
        case 0: LAUNCH(1, false); break;      \
        case 3: LAUNCH(4, true); break;       \
        case 8: LAUNCH(9, true); break;       \
        case 15: LAUNCH(16, true); break;     \
        default: return GSR_ERR_UNSUPPORTED;  \
    }

template <bool AA, bool F3D>
static int launch_fwd(int n_sh_rest, dim3 grid, cudaStream_t st, int N, const float* xyz, const float* xyz_cam,
                      int cam_first, const float* quat, const float* scale, const float* opa, const float* dc,
                      const float* sh, const float* T, const float* K, const float* cam, float width, float height,
                      float near_t, float far_t, float pad, float mh, int ntx, int nty, uint32_t depth_base,
                      float* records, uint32_t* zkey, uint8_t* visible, uint64_t* packed, uint64_t* tile_mask,
                      uint32_t* tile_win, int use_tma, const float* filter3d, const float* lens, const float* xi,
                      float r0, float e0, float e1) {
#define GSR_SH_FWD(NSH, HSH)                                                                                       \
    k_shutter_preprocess_fwd<NSH, HSH, AA, F3D><<<grid, PRE_THREADS, 0, st>>>(                                     \
        N, xyz, xyz_cam, cam_first, quat, scale, opa, dc, sh, T, K, cam, width, height, near_t, far_t, pad, mh, ntx, \
        nty, depth_base, records, zkey, visible, packed, tile_mask, tile_win, use_tma, filter3d, lens, xi, r0, e0, e1)
    GSR_SH_SWITCH(GSR_SH_FWD)
#undef GSR_SH_FWD
    return GSR_OK;
}

template <bool DEPTH, bool AA, bool F3D>
static int launch_bwd(bool single, int n_sh_rest, dim3 grid, cudaStream_t st, int C, int N, const float* xyz,
                      const float* quat, const float* scale, const float* opa, const float* T, const float* K,
                      const float* cam, const uint8_t* visible, const float* rows, int rows_uv, const float* g_uv,
                      const uint64_t* scan, float* o_xyz, float* o_quat, float* o_scale, float* o_opa, float* o_dc,
                      float* o_sh, int use_tma, const float* filter3d, const float* lens, const float* xi, float r0,
                      float e0, float e1, float* partials) {
#define GSR_SH_ARGS                                                                                                  \
    N, xyz, quat, scale, opa, T, K, cam, visible, rows, rows_uv, g_uv, scan, o_xyz, o_quat, o_scale, o_opa, o_dc,    \
        o_sh, use_tma, filter3d, lens, xi, r0, e0, e1, partials
#define GSR_SH_BWD(NSH, HSH)                                                                                         \
    if (single)                                                                                                      \
        k_shutter_preprocess_bwd<NSH, HSH, DEPTH, AA, F3D><<<grid, PRE_THREADS, 0, st>>>(GSR_SH_ARGS);               \
    else                                                                                                             \
        k_shutter_batch_preprocess_bwd<NSH, HSH, DEPTH, AA, F3D><<<grid, PRE_THREADS, 0, st>>>(C, GSR_SH_ARGS)
    GSR_SH_SWITCH(GSR_SH_BWD)
#undef GSR_SH_BWD
#undef GSR_SH_ARGS
    return GSR_OK;
}

}  // namespace GSR_SH_NS
}  // namespace gsr

GSR_SH_FWD_DECL(GSR_SH_LAUNCH_FWD) {
    using namespace gsr::GSR_SH_NS;
    const dim3 grid((N + gsr::PRE_THREADS - 1) / gsr::PRE_THREADS);
    const bool aa = (mode & GSR_MODE_ANTIALIASED) != 0, f3d = (mode & GSR_MODE_FILTER3D) != 0;
#define GSR_SH_ARGS                                                                                                  \
    n_sh_rest, grid, st, N, xyz, xyz_cam, cam_first, quat, scale, opa, dc, sh, T, K, cam, width, height, near_t,     \
        far_t, pad, mh, ntx, nty, depth_base, records, zkey, visible, packed, tile_mask, tile_win, use_tma, filter3d, \
        lens, xi, r0, e0, e1
    return f3d ? (aa ? launch_fwd<true, true>(GSR_SH_ARGS) : launch_fwd<false, true>(GSR_SH_ARGS))
               : (aa ? launch_fwd<true, false>(GSR_SH_ARGS) : launch_fwd<false, false>(GSR_SH_ARGS));
#undef GSR_SH_ARGS
}

GSR_SH_BWD_DECL(GSR_SH_LAUNCH_BWD) {
    using namespace gsr::GSR_SH_NS;
    const dim3 grid((N + gsr::PRE_THREADS - 1) / gsr::PRE_THREADS);
    const bool depth = (mode & GSR_MODE_DEPTH_ALPHA) != 0, aa = (mode & GSR_MODE_ANTIALIASED) != 0,
               f3d = (mode & GSR_MODE_FILTER3D) != 0;
#define GSR_SH_ARGS                                                                                                  \
    single, n_sh_rest, grid, st, C, N, xyz, quat, scale, opa, T, K, cam, visible, rows, rows_uv, g_uv, scan, o_xyz,  \
        o_quat, o_scale, o_opa, o_dc, o_sh, use_tma, filter3d, lens, xi, r0, e0, e1, partials
    return f3d ? (aa ? (depth ? launch_bwd<true, true, true>(GSR_SH_ARGS) : launch_bwd<false, true, true>(GSR_SH_ARGS))
                     : (depth ? launch_bwd<true, false, true>(GSR_SH_ARGS) : launch_bwd<false, false, true>(GSR_SH_ARGS)))
               : (aa ? (depth ? launch_bwd<true, true, false>(GSR_SH_ARGS) : launch_bwd<false, true, false>(GSR_SH_ARGS))
                     : (depth ? launch_bwd<true, false, false>(GSR_SH_ARGS)
                              : launch_bwd<false, false, false>(GSR_SH_ARGS)));
#undef GSR_SH_ARGS
}

#if GSR_SHUTTER_LENS == 0

GSR_SH_FWD_DECL(gsr_shutter_launch_fwd_fisheye);
GSR_SH_FWD_DECL(gsr_shutter_launch_fwd_distortion);
GSR_SH_BWD_DECL(gsr_shutter_launch_bwd_fisheye);
GSR_SH_BWD_DECL(gsr_shutter_launch_bwd_distortion);

namespace gsr {

// one CTA per view: the fixed-order fp64 sum of the view's partials, rounded once: g_pose [C, 4, 4] (last row 0) and
// g_xi [C, 6]
__global__ void __launch_bounds__(POSE_FINISH_THREADS)
    k_shutter_finish(int nblk, const float* __restrict__ partials, float* __restrict__ g_pose,
                     float* __restrict__ g_xi) {
    __shared__ double s_sum[POSE_FINISH_THREADS / 32][SHUTTER_VALUES];
    const int c = blockIdx.x, t = threadIdx.x;
    finish_partials<SHUTTER_VALUES>(nblk, partials + (size_t)c * nblk * SHUTTER_VALUES, s_sum);
    if (t < 18) {
        double v = s_sum[0][t];
        for (int w = 1; w < POSE_FINISH_THREADS / 32; ++w) v += s_sum[w][t];
        const float out = (float)v;
        if (t < 12) {
            g_pose[(size_t)c * 16 + t] = out;
        } else {
            if (t < 16) g_pose[(size_t)c * 16 + t] = 0.f;  // the last row
            g_xi[(size_t)c * 6 + t - 12] = out;
        }
    }
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

constexpr int KNOWN_MODES = GSR_MODE_DEPTH_ALPHA | GSR_MODE_ANTIALIASED | GSR_MODE_ABSGRAD | GSR_MODE_FILTER3D;

// the readout line r(u) = r0 + e0 u + e1 v of an H x W image; false for an unknown readout or a 1-pixel extent
static bool readout_line(int readout, int H, int W, float& r0, float& e0, float& e1) {
    const bool vertical = readout == GSR_READOUT_TOP_TO_BOTTOM || readout == GSR_READOUT_BOTTOM_TO_TOP;
    if (!vertical && readout != GSR_READOUT_LEFT_TO_RIGHT && readout != GSR_READOUT_RIGHT_TO_LEFT) return false;
    const int n = vertical ? H : W;
    if (n < 2) return false;
    const bool reverse = readout == GSR_READOUT_BOTTOM_TO_TOP || readout == GSR_READOUT_RIGHT_TO_LEFT;
    const float e = (float)((reverse ? -1.0 : 1.0) / (double)(n - 1));
    r0 = reverse ? 1.0f : 0.0f;
    e0 = vertical ? 0.0f : e;
    e1 = vertical ? e : 0.0f;
    return true;
}

static bool known_lens(int lens, const float* lens_consts) {
    if (lens != GSR_LENS_PINHOLE && lens != GSR_LENS_FISHEYE && lens != GSR_LENS_DISTORTION) return false;
    return (lens != GSR_LENS_PINHOLE) == (lens_consts != nullptr);
}

static size_t partial_bytes(int C, int N) {
    const size_t nblk = (size_t)((N > 0 ? N : 0) + PRE_THREADS - 1) / PRE_THREADS;
    return align256(sizeof(float) * (size_t)SHUTTER_VALUES * nblk * (size_t)(C > 0 ? C : 0));
}

}  // namespace gsr

using namespace gsr;

static int shutter_backward(bool single, int lens, int mode, int C, int N, int n_sh_rest, const float* xyz,
                            const float* quaternion, const float* scale, const float* opacity_logit,
                            const float* filter3d, const float* camera_T_world, const float* K,
                            const float* camera_centre_, const uint8_t* visible, const float* grad_rows,
                            int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                            float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                            float* g_sh_rest, const float* lens_consts, const float* shutter_xi, int readout, int H,
                            int W, float* g_pose, float* g_xi, void* temp, size_t temp_bytes, void* stream) {
    float r0, e0, e1;
    if (C < 1 || N < 0 || (mode & ~KNOWN_MODES) != 0 || !known_lens(lens, lens_consts)) return GSR_ERR_BAD_ARG;
    if (!readout_line(readout, H, W, r0, e0, e1) || shutter_xi == nullptr) return GSR_ERR_BAD_ARG;
    if (((mode & GSR_MODE_FILTER3D) != 0) != (filter3d != nullptr)) return GSR_ERR_BAD_ARG;
    if ((g_pose == nullptr) != (g_xi == nullptr)) return GSR_ERR_BAD_ARG;
    const bool camera = g_pose != nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    const int nblk = (N + PRE_THREADS - 1) / PRE_THREADS;
    float* partials = camera ? reinterpret_cast<float*>(temp) : nullptr;
    if (N > 0) {
        if (xyz == nullptr || quaternion == nullptr || scale == nullptr || opacity_logit == nullptr ||
            camera_T_world == nullptr || K == nullptr || visible == nullptr || grad_rows == nullptr ||
            g_xyz == nullptr || g_quaternion == nullptr || g_scale == nullptr || g_opacity_logit == nullptr ||
            g_rgb_dc == nullptr)
            return GSR_ERR_BAD_ARG;
        if ((n_sh_rest > 0) != (g_sh_rest != nullptr)) return GSR_ERR_BAD_ARG;
        if (!aligned16(grad_rows)) return GSR_ERR_BAD_ARG;
        if (grad_uv_compact != nullptr && scan == nullptr) return GSR_ERR_BAD_ARG;
        if (n_sh_rest != 0 && n_sh_rest != 3 && n_sh_rest != 8 && n_sh_rest != 15) return GSR_ERR_UNSUPPORTED;
        if (camera && (temp == nullptr || !aligned16(temp) || temp_bytes < partial_bytes(C, N))) return GSR_ERR_BAD_ARG;
        const int use_tma = (aligned16(g_xyz) && aligned16(g_quaternion) && aligned16(g_scale) &&
                             aligned16(g_opacity_logit) && aligned16(g_rgb_dc) &&
                             (g_sh_rest == nullptr || aligned16(g_sh_rest)))
                                ? 1
                                : 0;
        const auto launcher = lens == GSR_LENS_FISHEYE      ? gsr_shutter_launch_bwd_fisheye
                              : lens == GSR_LENS_DISTORTION ? gsr_shutter_launch_bwd_distortion
                                                            : gsr_shutter_launch_bwd_pinhole;
        const int rc = launcher(single, mode, C, N, n_sh_rest, xyz, quaternion, scale, opacity_logit, filter3d,
                                camera_T_world, K, camera_centre_, visible, grad_rows, use_rows_uv, grad_uv_compact,
                                scan, g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, use_tma,
                                lens_consts, shutter_xi, r0, e0, e1, partials, st);
        if (rc != GSR_OK) return rc;
    }
    if (camera) k_shutter_finish<<<C, POSE_FINISH_THREADS, 0, st>>>(nblk, partials, g_pose, g_xi);
    return (int)cudaGetLastError();
}

extern "C" {

size_t gsr_shutter_temp_bytes(int C, int N) { return partial_bytes(C, N); }

int gsr_shutter_preprocess_forward(int lens, int mode, int N, int n_sh_rest, const float* xyz,
                                   const float* xyz_camera_frame, int cam_first, const float* quaternion,
                                   const float* scale, const float* opacity_logit, const float* filter3d,
                                   const float* rgb_dc, const float* sh_rest, const float* camera_T_world,
                                   const float* K, const float* camera_centre_, int H, int W, float near_thresh,
                                   float far_thresh, float cull_mask_padding, float mh_dist, uint32_t depth_base,
                                   float* records, uint32_t* depth_key, uint8_t* visible, uint64_t* scan,
                                   uint64_t* tile_mask, uint32_t* tile_win, void* temp, size_t temp_bytes,
                                   const float* lens_consts, const float* shutter_xi, int readout, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    float r0, e0, e1;
    if ((mode & ~KNOWN_MODES) != 0 || !known_lens(lens, lens_consts)) return GSR_ERR_BAD_ARG;
    if (!readout_line(readout, H, W, r0, e0, e1) || shutter_xi == nullptr) return GSR_ERR_BAD_ARG;
    if (((mode & GSR_MODE_FILTER3D) != 0) != (filter3d != nullptr)) return GSR_ERR_BAD_ARG;
    if (N < 0) return GSR_ERR_BAD_ARG;
    if (N == 0) return GSR_OK;
    size_t scan_bytes = 0;
    cub::DeviceScan::InclusiveSum((void*)nullptr, scan_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, N);
    if (temp == nullptr || temp_bytes < align256(scan_bytes) + align256(sizeof(uint64_t) * (size_t)N))
        return GSR_ERR_BAD_ARG;
    if ((tile_mask == nullptr) != (tile_win == nullptr)) return GSR_ERR_BAD_ARG;
    uint64_t* packed = reinterpret_cast<uint64_t*>((char*)temp + align256(scan_bytes));
    const int ntx = (W + TILE - 1) / TILE, nty = (H + TILE - 1) / TILE;
    const int use_tma = (aligned16(records) && (sh_rest == nullptr || aligned16(sh_rest))) ? 1 : 0;
    const auto launcher = lens == GSR_LENS_FISHEYE      ? gsr_shutter_launch_fwd_fisheye
                          : lens == GSR_LENS_DISTORTION ? gsr_shutter_launch_fwd_distortion
                                                        : gsr_shutter_launch_fwd_pinhole;
    const int rc = launcher(mode, n_sh_rest, N, xyz, xyz_camera_frame, cam_first, quaternion, scale, opacity_logit,
                            rgb_dc, sh_rest, camera_T_world, K, camera_centre_, (float)W, (float)H, near_thresh,
                            far_thresh, cull_mask_padding, mh_dist, ntx, nty, depth_base, records, depth_key, visible,
                            packed, tile_mask, tile_win, use_tma, filter3d, lens_consts, shutter_xi, r0, e0, e1, st);
    if (rc != GSR_OK) return rc;
    cudaError_t e = cub::DeviceScan::InclusiveSum(temp, scan_bytes, packed, scan, N, st);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

int gsr_shutter_preprocess_backward(int lens, int mode, int N, int n_sh_rest, const float* xyz,
                                    const float* quaternion, const float* scale, const float* opacity_logit,
                                    const float* filter3d, const float* camera_T_world, const float* K,
                                    const float* camera_centre_, const uint8_t* visible, const float* grad_rows,
                                    int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                    float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                                    float* g_sh_rest, const float* lens_consts, const float* shutter_xi, int readout,
                                    int H, int W, float* g_pose, float* g_xi, void* temp, size_t temp_bytes,
                                    void* stream) {
    return shutter_backward(true, lens, mode, 1, N, n_sh_rest, xyz, quaternion, scale, opacity_logit, filter3d,
                            camera_T_world, K, camera_centre_, visible, grad_rows, use_rows_uv, grad_uv_compact, scan,
                            g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, lens_consts,
                            shutter_xi, readout, H, W, g_pose, g_xi, temp, temp_bytes, stream);
}

int gsr_shutter_batch_preprocess_backward(int lens, int mode, int C, int N, int n_sh_rest, const float* xyz,
                                          const float* quaternion, const float* scale, const float* opacity_logit,
                                          const float* filter3d, const float* camera_T_world, const float* K,
                                          const float* camera_centre_, const uint8_t* visible, const float* grad_rows,
                                          int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan,
                                          float* g_xyz, float* g_quaternion, float* g_scale, float* g_opacity_logit,
                                          float* g_rgb_dc, float* g_sh_rest, const float* lens_consts,
                                          const float* shutter_xi, int readout, int H, int W, float* g_pose,
                                          float* g_xi, void* temp, size_t temp_bytes, void* stream) {
    return shutter_backward(false, lens, mode, C, N, n_sh_rest, xyz, quaternion, scale, opacity_logit, filter3d,
                            camera_T_world, K, camera_centre_, visible, grad_rows, use_rows_uv, grad_uv_compact, scan,
                            g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, lens_consts,
                            shutter_xi, readout, H, W, g_pose, g_xi, temp, temp_bytes, stream);
}

}  // extern "C"

#endif  // GSR_SHUTTER_LENS == 0
