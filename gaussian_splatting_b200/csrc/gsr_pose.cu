// gsr_pose.cu — the per-gaussian backward with the camera pose gradient (libgsr_pose.so): rasterize(...) and
// rasterize_batch(...) when camera_T_world requires grad.
//
// The bodies are those of gsr_preprocess.cuh — single-view and batched backward, so the gaussian gradients are the
// existing arithmetic — compiled with the pose hooks of gsr_pose.cuh.  This file is compiled once per camera model:
// GSR_POSE_LENS 0 (pinhole, the default hooks), 1 (gsr_fisheye.cuh's hooks) or 2 (gsr_distortion.cuh's hooks).  Each
// compile puts its kernels in a namespace of its own and exports one hidden launcher; the compile with
// GSR_POSE_LENS == 0 also holds the fp64 finishing kernel and the C ABI of include/gsr_pose.h, which dispatch on the
// lens.  With GSR_POSE_CAMERA the same three compiles make libgsr_calib.so: the same bodies, whose rows also carry the
// intrinsics and lens-coefficient gradients of gsr_calib.cuh, with the C ABI of include/gsr_calib.h.
#include <cstdint>

#include "../../include/gsr_distortion.h"
#include "../../include/gsr_fisheye.h"

#ifndef GSR_POSE_LENS
#define GSR_POSE_LENS 0
#endif

#if GSR_POSE_LENS == 1
#define GSR_FISHEYE_HOOKS
#include "gsr_fisheye.cuh"
#define GSR_POSE_LENS_ARG , lens
#elif GSR_POSE_LENS == 2
#define GSR_DISTORTION_HOOKS
#include "gsr_distortion.cuh"
#define GSR_POSE_LENS_ARG , lens
#else
#define GSR_POSE_LENS_ARG
#endif

// one namespace, launcher and name of gsr_preprocess.cuh's one non-inline device function (it has a host-side symbol)
// per compile, so that the three objects of a library (and the two libraries) link side by side
#ifdef GSR_POSE_CAMERA
#if GSR_POSE_LENS == 1
#define GSR_POSE_NS camera_fisheye
#define GSR_POSE_LAUNCH gsr_camera_launch_fisheye
#define camera_centre camera_centre_camera_fisheye
#elif GSR_POSE_LENS == 2
#define GSR_POSE_NS camera_distortion
#define GSR_POSE_LAUNCH gsr_camera_launch_distortion
#define camera_centre camera_centre_camera_distortion
#else
#define GSR_POSE_NS camera_pinhole
#define GSR_POSE_LAUNCH gsr_camera_launch_pinhole
#define camera_centre camera_centre_camera_pinhole
#endif
#else
#if GSR_POSE_LENS == 1
#define GSR_POSE_NS pose_fisheye
#define GSR_POSE_LAUNCH gsr_pose_launch_fisheye
#define camera_centre camera_centre_pose_fisheye
#elif GSR_POSE_LENS == 2
#define GSR_POSE_NS pose_distortion
#define GSR_POSE_LAUNCH gsr_pose_launch_distortion
#define camera_centre camera_centre_pose_distortion
#else
#define GSR_POSE_NS pose_pinhole
#define GSR_POSE_LAUNCH gsr_pose_launch_pinhole
#endif
#endif
#include "gsr_common.cuh"
#ifdef GSR_POSE_CAMERA
#include "gsr_calib.cuh"
namespace gsr {
// a row: 12 pose values, fx fy cx cy, the lens's coefficients, zero padding to a multiple of 4 (float4 loads)
#if GSR_POSE_LENS == 1
constexpr int CAMERA_VALUES = 20;
#define GSR_CAMERA_VIEW(px, py, pz, guv, gJ, out) \
    fisheye_calib(px, py, pz, vc.K[0], vc.K[4], vfe, guv[0], guv[1], gJ, out)
#elif GSR_POSE_LENS == 2
constexpr int CAMERA_VALUES = 24;
#define GSR_CAMERA_VIEW(px, py, pz, guv, gJ, out) \
    distortion_calib(px, py, pz, vc.K[0], vc.K[4], vdc, guv[0], guv[1], gJ, out)
#else
constexpr int CAMERA_VALUES = 16;
#define GSR_CAMERA_VIEW(px, py, pz, guv, gJ, out) pinhole_calib(px, py, pz, guv[0], guv[1], gJ, out)
#endif
}  // namespace gsr
#endif
#include "gsr_pose.cuh"
#include "gsr_preprocess.cuh"

#include "../../include/gsr_pose.h"
#ifdef GSR_POSE_CAMERA
#include "../../include/gsr_calib.h"
#endif

// CTAs per SM the register budget is sized for (-Xptxas -v: no local memory at these bounds, DESIGN.md 3.21, 3.23)
#ifndef GSR_POSE_BWD_MINB
#define GSR_POSE_BWD_MINB 4
#endif
#ifndef GSR_POSE_BATCH_MINB
#define GSR_POSE_BATCH_MINB 3
#endif
#ifdef GSR_POSE_CAMERA
#define k_pose_preprocess_bwd k_camera_preprocess_bwd
#define k_pose_batch_preprocess_bwd k_camera_batch_preprocess_bwd
#endif

// the launcher of one camera model: the per-gaussian kernel of `single` (C == 1) or of C views, writing the
// partials [C, grid, 12] (the camera-gradient kernels: [C, grid, CAMERA_VALUES])
#define GSR_POSE_LAUNCH_DECL(name)                                                                                   \
    __attribute__((visibility("hidden"))) int name(                                                                 \
        bool single, int mode, int C, int N, int n_sh_rest, const float* xyz, const float* quat, const float* scale, \
        const float* opa, const float* filter3d, const float* T, const float* K, const float* cam,                  \
        const uint8_t* visible, const float* rows, int rows_uv, const float* g_uv, const uint64_t* scan,            \
        float* o_xyz, float* o_quat, float* o_scale, float* o_opa, float* o_dc, float* o_sh, int use_tma,           \
        const float* lens, float* partials, cudaStream_t st)

namespace gsr {
static_assert(POSE_CTA_THREADS == PRE_THREADS, "pose_cta_reduce sums one CTA of the bodies");
namespace GSR_POSE_NS {

#define GSR_POSE_BWD_PARAMS                                                                                         \
    int N, const float* __restrict__ xyz, const float* __restrict__ quat, const float* __restrict__ scale,          \
        const float* __restrict__ opa_logit, const float* __restrict__ Tdev, const float* __restrict__ Kdev,        \
        const float* __restrict__ camdev, const uint8_t* __restrict__ visible, const float* __restrict__ g_rows,    \
        int rows_uv, const float* __restrict__ g_uv_compact, const uint64_t* __restrict__ scan,                      \
        float* __restrict__ o_xyz, float* __restrict__ o_quat, float* __restrict__ o_scale,                         \
        float* __restrict__ o_opa, float* __restrict__ o_dc, float* __restrict__ o_sh, int use_tma,                 \
        const float* __restrict__ filter3d, const float* __restrict__ lens, float* __restrict__ partials
#define GSR_POSE_BWD_FORWARD                                                                                        \
    N, xyz, quat, scale, opa_logit, Tdev, Kdev, camdev, visible, g_rows, rows_uv, g_uv_compact, scan, o_xyz, o_quat, \
        o_scale, o_opa, o_dc, o_sh, use_tma, filter3d GSR_POSE_LENS_ARG, partials
template <int N_SH, bool HAS_SH, bool DEPTH, bool ANTIALIAS, bool FILTER3D>
__global__ void __launch_bounds__(PRE_THREADS, GSR_POSE_BWD_MINB) k_pose_preprocess_bwd(GSR_POSE_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, DEPTH, ANTIALIAS, FILTER3D>(GSR_POSE_BWD_FORWARD);
}
template <int N_SH, bool HAS_SH, bool DEPTH, bool ANTIALIAS, bool FILTER3D>
__global__ void __launch_bounds__(PRE_THREADS, GSR_POSE_BATCH_MINB)
    k_pose_batch_preprocess_bwd(int C, GSR_POSE_BWD_PARAMS) {
    batch_preprocess_bwd<N_SH, HAS_SH, DEPTH, ANTIALIAS, FILTER3D>(C, GSR_POSE_BWD_FORWARD);
}
#undef GSR_POSE_BWD_PARAMS
#undef GSR_POSE_BWD_FORWARD

template <bool DEPTH, bool AA, bool F3D>
static int launch(bool single, int n_sh_rest, dim3 grid, cudaStream_t st, int C, int N, const float* xyz,
                  const float* quat, const float* scale, const float* opa, const float* T, const float* K,
                  const float* cam, const uint8_t* visible, const float* rows, int rows_uv, const float* g_uv,
                  const uint64_t* scan, float* o_xyz, float* o_quat, float* o_scale, float* o_opa, float* o_dc,
                  float* o_sh, int use_tma, const float* filter3d, const float* lens, float* partials) {
#define GSR_POSE_ARGS                                                                                                \
    N, xyz, quat, scale, opa, T, K, cam, visible, rows, rows_uv, g_uv, scan, o_xyz, o_quat, o_scale, o_opa, o_dc,    \
        o_sh, use_tma, filter3d, lens, partials
#define GSR_POSE_SH(NSH, HSH)                                                                                        \
    if (single)                                                                                                      \
        k_pose_preprocess_bwd<NSH, HSH, DEPTH, AA, F3D><<<grid, PRE_THREADS, 0, st>>>(GSR_POSE_ARGS);                \
    else                                                                                                             \
        k_pose_batch_preprocess_bwd<NSH, HSH, DEPTH, AA, F3D><<<grid, PRE_THREADS, 0, st>>>(C, GSR_POSE_ARGS);
    switch (n_sh_rest) {
        case 0: GSR_POSE_SH(1, false) break;
        case 3: GSR_POSE_SH(4, true) break;
        case 8: GSR_POSE_SH(9, true) break;
        case 15: GSR_POSE_SH(16, true) break;
        default: return GSR_ERR_UNSUPPORTED;
    }
#undef GSR_POSE_SH
#undef GSR_POSE_ARGS
    return GSR_OK;
}

}  // namespace GSR_POSE_NS
}  // namespace gsr

GSR_POSE_LAUNCH_DECL(GSR_POSE_LAUNCH) {
    using namespace gsr::GSR_POSE_NS;
    const dim3 grid((N + gsr::PRE_THREADS - 1) / gsr::PRE_THREADS);
    const bool depth = (mode & GSR_MODE_DEPTH_ALPHA) != 0, aa = (mode & GSR_MODE_ANTIALIASED) != 0,
               f3d = (mode & GSR_MODE_FILTER3D) != 0;
#define GSR_POSE_ARGS                                                                                                \
    single, n_sh_rest, grid, st, C, N, xyz, quat, scale, opa, T, K, cam, visible, rows, rows_uv, g_uv, scan, o_xyz,  \
        o_quat, o_scale, o_opa, o_dc, o_sh, use_tma, filter3d, lens, partials
    return f3d ? (aa ? (depth ? launch<true, true, true>(GSR_POSE_ARGS) : launch<false, true, true>(GSR_POSE_ARGS))
                     : (depth ? launch<true, false, true>(GSR_POSE_ARGS) : launch<false, false, true>(GSR_POSE_ARGS)))
               : (aa ? (depth ? launch<true, true, false>(GSR_POSE_ARGS) : launch<false, true, false>(GSR_POSE_ARGS))
                     : (depth ? launch<true, false, false>(GSR_POSE_ARGS)
                              : launch<false, false, false>(GSR_POSE_ARGS)));
#undef GSR_POSE_ARGS
}

#if GSR_POSE_LENS == 0

// the launchers of the other two lenses, compiled in the same library
#ifdef GSR_POSE_CAMERA
#define GSR_LAUNCH_FISHEYE gsr_camera_launch_fisheye
#define GSR_LAUNCH_DISTORTION gsr_camera_launch_distortion
#else
#define GSR_LAUNCH_FISHEYE gsr_pose_launch_fisheye
#define GSR_LAUNCH_DISTORTION gsr_pose_launch_distortion
#endif
GSR_POSE_LAUNCH_DECL(GSR_LAUNCH_FISHEYE);
GSR_POSE_LAUNCH_DECL(GSR_LAUNCH_DISTORTION);

namespace gsr {

#ifndef GSR_POSE_CAMERA
// one CTA per view: the fixed-order fp64 sum of the view's partials, rounded once.  Writes the view's [4, 4] gradient,
// the last row 0.
__global__ void __launch_bounds__(POSE_FINISH_THREADS) k_pose_finish(int nblk, const float* __restrict__ partials,
                                                                    float* __restrict__ g_pose) {
    __shared__ double s_sum[POSE_FINISH_THREADS / 32][POSE_VALUES];
    const int c = blockIdx.x, t = threadIdx.x;
    finish_partials<POSE_VALUES>(nblk, partials + (size_t)c * nblk * POSE_VALUES, s_sum);
    if (t < 16) {
        float out = 0.f;
        if (t < POSE_VALUES) {
            double v = s_sum[0][t];
            for (int w = 1; w < POSE_FINISH_THREADS / 32; ++w) v += s_sum[w][t];
            out = (float)v;
        }
        g_pose[(size_t)c * 16 + t] = out;
    }
}
#else
// the same for rows of NV camera values: g_pose [C, 4, 4] (last row 0), g_intrinsics [C, 4] (fx fy cx cy) and
// g_lens [C, n_lens]
template <int NV>
__global__ void __launch_bounds__(POSE_FINISH_THREADS)
    k_camera_finish(int nblk, int n_lens, const float* __restrict__ partials, float* __restrict__ g_pose,
                    float* __restrict__ g_intrinsics, float* __restrict__ g_lens) {
    __shared__ double s_sum[POSE_FINISH_THREADS / 32][NV];
    const int c = blockIdx.x, t = threadIdx.x;
    finish_partials<NV>(nblk, partials + (size_t)c * nblk * NV, s_sum);
    if (t < POSE_VALUES + 4 + n_lens) {
        double v = s_sum[0][t];
        for (int w = 1; w < POSE_FINISH_THREADS / 32; ++w) v += s_sum[w][t];
        const float out = (float)v;
        if (t < POSE_VALUES) {
            g_pose[(size_t)c * 16 + t] = out;
        } else if (t < POSE_VALUES + 4) {
            g_pose[(size_t)c * 16 + t] = 0.f;
            g_intrinsics[(size_t)c * 4 + t - POSE_VALUES] = out;
        } else {
            g_lens[(size_t)c * n_lens + t - POSE_VALUES - 4] = out;
        }
    }
}
#endif

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

constexpr int KNOWN_MODES = GSR_MODE_DEPTH_ALPHA | GSR_MODE_ANTIALIASED | GSR_MODE_ABSGRAD | GSR_MODE_FILTER3D;

}  // namespace gsr

using namespace gsr;

// the values per row of the camera-gradient kernels of a lens (12 pose, 4 intrinsics, the coefficients, padding)
static int camera_values(int lens) { return lens == GSR_LENS_FISHEYE ? 20 : lens == GSR_LENS_DISTORTION ? 24 : 16; }

static size_t partial_bytes(int values, int C, int N) {
    const size_t nblk = (size_t)((N > 0 ? N : 0) + PRE_THREADS - 1) / PRE_THREADS;
    return align256(sizeof(float) * (size_t)values * nblk * (size_t)(C > 0 ? C : 0));
}

#ifdef GSR_POSE_CAMERA
constexpr bool CAMERA = true;
#else
constexpr bool CAMERA = false;
#endif

// The entry points of this library (libgsr_pose.so; with GSR_POSE_CAMERA libgsr_calib.so, which also writes the
// intrinsics and lens-coefficient gradients g_intrinsics [C, 4] and g_lens [C, n], NULL for the pinhole)
static int pose_backward(bool single, int lens, int mode, int C, int N, int n_sh_rest, const float* xyz,
                         const float* quaternion, const float* scale, const float* opacity_logit, const float* filter3d,
                         const float* camera_T_world, const float* K, const float* camera_centre,
                         const uint8_t* visible, const float* grad_rows, int use_rows_uv,
                         const float* grad_uv_compact, const uint64_t* scan, float* g_xyz, float* g_quaternion,
                         float* g_scale, float* g_opacity_logit, float* g_rgb_dc, float* g_sh_rest,
                         const float* lens_consts, float* g_pose, float* g_intrinsics, float* g_lens, void* temp,
                         size_t temp_bytes, void* stream) {
    if (C < 1 || N < 0 || (mode & ~KNOWN_MODES) != 0 || g_pose == nullptr) return GSR_ERR_BAD_ARG;
    if (lens != GSR_LENS_PINHOLE && lens != GSR_LENS_FISHEYE && lens != GSR_LENS_DISTORTION) return GSR_ERR_BAD_ARG;
    if ((lens != GSR_LENS_PINHOLE) != (lens_consts != nullptr)) return GSR_ERR_BAD_ARG;
    if (CAMERA && (g_intrinsics == nullptr || (lens != GSR_LENS_PINHOLE) != (g_lens != nullptr))) return GSR_ERR_BAD_ARG;
    const int values = CAMERA ? camera_values(lens) : POSE_VALUES;
    if (((mode & GSR_MODE_FILTER3D) != 0) != (filter3d != nullptr)) return GSR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int nblk = (N + PRE_THREADS - 1) / PRE_THREADS;
    float* partials = reinterpret_cast<float*>(temp);
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
        if (temp == nullptr || !aligned16(temp) || temp_bytes < partial_bytes(values, C, N)) return GSR_ERR_BAD_ARG;
        const int use_tma = (aligned16(g_xyz) && aligned16(g_quaternion) && aligned16(g_scale) &&
                             aligned16(g_opacity_logit) && aligned16(g_rgb_dc) &&
                             (g_sh_rest == nullptr || aligned16(g_sh_rest)))
                                ? 1
                                : 0;
        const auto launcher = lens == GSR_LENS_FISHEYE      ? GSR_LAUNCH_FISHEYE
                              : lens == GSR_LENS_DISTORTION ? GSR_LAUNCH_DISTORTION
                                                            : GSR_POSE_LAUNCH;
        const int rc = launcher(single, mode, C, N, n_sh_rest, xyz, quaternion, scale, opacity_logit, filter3d,
                                camera_T_world, K, camera_centre, visible, grad_rows, use_rows_uv, grad_uv_compact,
                                scan, g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, use_tma,
                                lens_consts, partials, st);
        if (rc != GSR_OK) return rc;
    }
#ifdef GSR_POSE_CAMERA
    if (values == 20)
        k_camera_finish<20><<<C, POSE_FINISH_THREADS, 0, st>>>(nblk, 4, partials, g_pose, g_intrinsics, g_lens);
    else if (values == 24)
        k_camera_finish<24><<<C, POSE_FINISH_THREADS, 0, st>>>(nblk, 5, partials, g_pose, g_intrinsics, g_lens);
    else
        k_camera_finish<16><<<C, POSE_FINISH_THREADS, 0, st>>>(nblk, 0, partials, g_pose, g_intrinsics, g_lens);
#else
    k_pose_finish<<<C, POSE_FINISH_THREADS, 0, st>>>(nblk, partials, g_pose);
#endif
    return (int)cudaGetLastError();
}

extern "C" {

#ifdef GSR_POSE_CAMERA

size_t gsr_camera_temp_bytes(int lens, int C, int N) { return partial_bytes(camera_values(lens), C, N); }

int gsr_camera_preprocess_backward(int lens, int mode, int N, int n_sh_rest, const float* xyz,
                                   const float* quaternion, const float* scale, const float* opacity_logit,
                                   const float* filter3d, const float* camera_T_world, const float* K,
                                   const float* camera_centre, const uint8_t* visible, const float* grad_rows,
                                   int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                   float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                                   float* g_sh_rest, const float* lens_consts, float* g_pose, float* g_intrinsics,
                                   float* g_lens, void* temp, size_t temp_bytes, void* stream) {
    return pose_backward(true, lens, mode, 1, N, n_sh_rest, xyz, quaternion, scale, opacity_logit, filter3d,
                         camera_T_world, K, camera_centre, visible, grad_rows, use_rows_uv, grad_uv_compact, scan,
                         g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, lens_consts, g_pose,
                         g_intrinsics, g_lens, temp, temp_bytes, stream);
}

int gsr_camera_batch_preprocess_backward(int lens, int mode, int C, int N, int n_sh_rest, const float* xyz,
                                         const float* quaternion, const float* scale, const float* opacity_logit,
                                         const float* filter3d, const float* camera_T_world, const float* K,
                                         const float* camera_centre, const uint8_t* visible, const float* grad_rows,
                                         int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan,
                                         float* g_xyz, float* g_quaternion, float* g_scale, float* g_opacity_logit,
                                         float* g_rgb_dc, float* g_sh_rest, const float* lens_consts, float* g_pose,
                                         float* g_intrinsics, float* g_lens, void* temp, size_t temp_bytes,
                                         void* stream) {
    return pose_backward(false, lens, mode, C, N, n_sh_rest, xyz, quaternion, scale, opacity_logit, filter3d,
                         camera_T_world, K, camera_centre, visible, grad_rows, use_rows_uv, grad_uv_compact, scan,
                         g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, lens_consts, g_pose,
                         g_intrinsics, g_lens, temp, temp_bytes, stream);
}

#else

size_t gsr_pose_temp_bytes(int C, int N) { return partial_bytes(POSE_VALUES, C, N); }

int gsr_pose_preprocess_backward(int lens, int mode, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                                 const float* scale, const float* opacity_logit, const float* filter3d,
                                 const float* camera_T_world, const float* K, const float* camera_centre,
                                 const uint8_t* visible, const float* grad_rows, int use_rows_uv,
                                 const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                 float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                                 float* g_sh_rest, const float* lens_consts, float* g_pose, void* temp,
                                 size_t temp_bytes, void* stream) {
    return pose_backward(true, lens, mode, 1, N, n_sh_rest, xyz, quaternion, scale, opacity_logit, filter3d,
                         camera_T_world, K, camera_centre, visible, grad_rows, use_rows_uv, grad_uv_compact, scan,
                         g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, lens_consts, g_pose,
                         nullptr, nullptr, temp, temp_bytes, stream);
}

int gsr_pose_batch_preprocess_backward(int lens, int mode, int C, int N, int n_sh_rest, const float* xyz,
                                       const float* quaternion, const float* scale, const float* opacity_logit,
                                       const float* filter3d, const float* camera_T_world, const float* K,
                                       const float* camera_centre, const uint8_t* visible, const float* grad_rows,
                                       int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan,
                                       float* g_xyz, float* g_quaternion, float* g_scale, float* g_opacity_logit,
                                       float* g_rgb_dc, float* g_sh_rest, const float* lens_consts, float* g_pose,
                                       void* temp, size_t temp_bytes, void* stream) {
    return pose_backward(false, lens, mode, C, N, n_sh_rest, xyz, quaternion, scale, opacity_logit, filter3d,
                         camera_T_world, K, camera_centre, visible, grad_rows, use_rows_uv, grad_uv_compact, scan,
                         g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, lens_consts, g_pose,
                         nullptr, nullptr, temp, temp_bytes, stream);
}

#endif  // GSR_POSE_CAMERA

}  // extern "C"

#endif  // GSR_POSE_LENS == 0
