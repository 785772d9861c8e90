// gsr_batch.cu — the per-Gaussian backward of C views of one scene in one pass (rasterize_batch).
//
// The body, batch_preprocess_bwd, lives in gsr_preprocess.cuh next to the single-view VJP it repeats per view.
#include "gsr_preprocess.cuh"

#include "../../include/gsr_batch.h"

namespace gsr {

// the running sums (14 floats) come on top of the single-view kernel's registers: 4 CTAs per SM (128 registers)
// keep every variant out of local memory
#ifndef GSR_BATCH_BWD_MINB
#define GSR_BATCH_BWD_MINB 4
#endif
#define GSR_BATCH_BWD_PARAMS                                                                                        \
    int C, int N, const float* __restrict__ xyz, const float* __restrict__ quat, const float* __restrict__ scale,   \
        const float* __restrict__ opa_logit, const float* __restrict__ Tdev, const float* __restrict__ Kdev,        \
        const float* __restrict__ camdev, const uint8_t* __restrict__ visible, const float* __restrict__ g_rows,    \
        int rows_uv, const float* __restrict__ g_uv_compact, const uint64_t* __restrict__ scan,                      \
        float* __restrict__ o_xyz, float* __restrict__ o_quat, float* __restrict__ o_scale,                         \
        float* __restrict__ o_opa, float* __restrict__ o_dc, float* __restrict__ o_sh, int use_tma,                 \
        const float* __restrict__ filter3d
#define GSR_BATCH_BWD_FORWARD                                                                                       \
    C, N, xyz, quat, scale, opa_logit, Tdev, Kdev, camdev, visible, g_rows, rows_uv, g_uv_compact, scan, o_xyz,      \
        o_quat, o_scale, o_opa, o_dc, o_sh, use_tma, filter3d
template <int N_SH, bool HAS_SH, bool DEPTH, bool ANTIALIAS, bool FILTER3D>
__global__ void __launch_bounds__(PRE_THREADS, GSR_BATCH_BWD_MINB) k_batch_preprocess_bwd(GSR_BATCH_BWD_PARAMS) {
    batch_preprocess_bwd<N_SH, HAS_SH, DEPTH, ANTIALIAS, FILTER3D>(GSR_BATCH_BWD_FORWARD);
}
#undef GSR_BATCH_BWD_PARAMS
#undef GSR_BATCH_BWD_FORWARD

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// GSR_MODE_ABSGRAD only changes the render backward (row slots 10-11, which the per-gaussian backward does not read)
constexpr int KNOWN_MODES = GSR_MODE_DEPTH_ALPHA | GSR_MODE_ANTIALIASED | GSR_MODE_ABSGRAD | GSR_MODE_FILTER3D;

template <bool DEPTH, bool ANTIALIAS, bool FILTER3D>
static int launch_batch_bwd(int n_sh_rest, dim3 grid, cudaStream_t st, int C, int N, const float* xyz,
                            const float* quat, const float* scale, const float* opa, const float* T, const float* K,
                            const float* cam, const uint8_t* visible, const float* rows, int rows_uv,
                            const float* g_uv, const uint64_t* scan, float* o_xyz, float* o_quat, float* o_scale,
                            float* o_opa, float* o_dc, float* o_sh, int use_tma, const float* filter3d) {
#define GSR_BATCH_ARGS                                                                                              \
    C, N, xyz, quat, scale, opa, T, K, cam, visible, rows, rows_uv, g_uv, scan, o_xyz, o_quat, o_scale, o_opa, o_dc, \
        o_sh, use_tma, filter3d
    switch (n_sh_rest) {
        case 0: k_batch_preprocess_bwd<1, false, DEPTH, ANTIALIAS, FILTER3D><<<grid, PRE_THREADS, 0, st>>>(GSR_BATCH_ARGS); break;
        case 3: k_batch_preprocess_bwd<4, true, DEPTH, ANTIALIAS, FILTER3D><<<grid, PRE_THREADS, 0, st>>>(GSR_BATCH_ARGS); break;
        case 8: k_batch_preprocess_bwd<9, true, DEPTH, ANTIALIAS, FILTER3D><<<grid, PRE_THREADS, 0, st>>>(GSR_BATCH_ARGS); break;
        case 15: k_batch_preprocess_bwd<16, true, DEPTH, ANTIALIAS, FILTER3D><<<grid, PRE_THREADS, 0, st>>>(GSR_BATCH_ARGS); break;
        default: return GSR_ERR_UNSUPPORTED;
    }
#undef GSR_BATCH_ARGS
    return (int)cudaGetLastError();
}

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_batch_preprocess_backward(int mode, int C, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                                  const float* scale, const float* opacity_logit, const float* filter3d,
                                  const float* camera_T_world, const float* K, const float* camera_centre,
                                  const uint8_t* visible, const float* grad_rows, int use_rows_uv,
                                  const float* grad_uv_compact, const uint64_t* scan, float* g_xyz,
                                  float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                                  float* g_sh_rest, void* stream) {
    if (C < 1 || N < 0 || (mode & ~KNOWN_MODES) != 0) return GSR_ERR_BAD_ARG;
    if (((mode & GSR_MODE_FILTER3D) != 0) != (filter3d != nullptr)) return GSR_ERR_BAD_ARG;
    if (N == 0) return GSR_OK;  // nothing to launch (the arrays of an empty scene may be NULL)
    if (xyz == nullptr || quaternion == nullptr || scale == nullptr || opacity_logit == nullptr ||
        camera_T_world == nullptr || K == nullptr || visible == nullptr || grad_rows == nullptr || g_xyz == nullptr ||
        g_quaternion == nullptr || g_scale == nullptr || g_opacity_logit == nullptr || g_rgb_dc == nullptr)
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
#define GSR_BATCH_ARGS                                                                                              \
    n_sh_rest, grid, st, C, N, xyz, quaternion, scale, opacity_logit, camera_T_world, K, camera_centre, visible,     \
        grad_rows, use_rows_uv, grad_uv_compact, scan, g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc,       \
        g_sh_rest, use_tma, filter3d
    const bool depth = (mode & GSR_MODE_DEPTH_ALPHA) != 0, aa = (mode & GSR_MODE_ANTIALIASED) != 0,
               f3d = (mode & GSR_MODE_FILTER3D) != 0;
    int rc;
    if (f3d) {
        if (aa && depth) rc = launch_batch_bwd<true, true, true>(GSR_BATCH_ARGS);
        else if (aa) rc = launch_batch_bwd<false, true, true>(GSR_BATCH_ARGS);
        else if (depth) rc = launch_batch_bwd<true, false, true>(GSR_BATCH_ARGS);
        else rc = launch_batch_bwd<false, false, true>(GSR_BATCH_ARGS);
    } else {
        if (aa && depth) rc = launch_batch_bwd<true, true, false>(GSR_BATCH_ARGS);
        else if (aa) rc = launch_batch_bwd<false, true, false>(GSR_BATCH_ARGS);
        else if (depth) rc = launch_batch_bwd<true, false, false>(GSR_BATCH_ARGS);
        else rc = launch_batch_bwd<false, false, false>(GSR_BATCH_ARGS);
    }
#undef GSR_BATCH_ARGS
    return rc;
}

}  // extern "C"
