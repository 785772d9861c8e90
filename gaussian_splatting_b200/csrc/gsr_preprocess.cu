// gsr_preprocess.cu — the fused per-Gaussian stage behind rasterize().
//
// One kernel replaces, for every Gaussian of the scene, the reference's chain
//   transform_points_torch        splat_py/utils.py:60-72
//   CameraPointProjection         src/projection.cu:8-19
//   frustum cull + 8 mask gathers splat_py/rasterize.py:33-75
//   sigmoid(opacity)              splat_py/rasterize.py:60-62
//   ComputeSigmaWorld             src/projection.cu:56-109
//   ComputeProjectionJacobian     src/projection.cu:154-175
//   ComputeConic                  src/projection.cu:213-257
//   cat(rgb, sh) + PrecomputeRGBFromSH   splat_py/rasterize.py:89-93, src/precompute_sh.cu:7-58
//   compute_num_splats_kernel     src/tile_culling.cu:124-177
// and writes one 48-byte splat record, a depth key, a visibility flag and the
// tiles-touched count per Gaussian.  No Sigma_world / J intermediates reach HBM.
// The backward kernel is the fused VJP of the same chain (SURVEY.md Appendix A).
#include <cub/cub.cuh>

#include "gsr_preprocess.cuh"

namespace gsr {

__global__ void k_camera_centre(const float* __restrict__ T, float* __restrict__ cam) {
    if (threadIdx.x == 0 && blockIdx.x == 0) camera_centre(T, cam);
}

template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, 7) k_preprocess_fwd(GSR_PRE_FWD_PARAMS) {
    preprocess_fwd<N_SH, HAS_SH, false, false>(GSR_PRE_FWD_FORWARD, nullptr);
}
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, 7) k_preprocess_fwd_aa(GSR_PRE_FWD_PARAMS) {
    preprocess_fwd<N_SH, HAS_SH, true, false>(GSR_PRE_FWD_FORWARD, nullptr);
}
#ifndef GSR_PRE_FWD_F3D_MINB
#define GSR_PRE_FWD_F3D_MINB 7
#endif
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_FWD_F3D_MINB)
    k_preprocess_fwd_f3d(GSR_PRE_FWD_PARAMS, const float* __restrict__ filter3d) {
    preprocess_fwd<N_SH, HAS_SH, false, true>(GSR_PRE_FWD_FORWARD, filter3d);
}
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_FWD_F3D_MINB)
    k_preprocess_fwd_aa_f3d(GSR_PRE_FWD_PARAMS, const float* __restrict__ filter3d) {
    preprocess_fwd<N_SH, HAS_SH, true, true>(GSR_PRE_FWD_FORWARD, filter3d);
}
#undef GSR_PRE_FWD_PARAMS
#undef GSR_PRE_FWD_FORWARD

// Fused VJP (preprocess_bwd, gsr_preprocess.cuh).  g_rows are the per-Gaussian sums produced by the render
// backward, one interleaved row per original gaussian.
#ifndef GSR_PRE_BWD_MINB
#define GSR_PRE_BWD_MINB 6
#endif
// the anti-aliased backward re-forms the conic for rho's gradient: at 6 CTAs per SM (80 registers) that spills, at 5
// it does not
#ifndef GSR_PRE_BWD_AA_MINB
#define GSR_PRE_BWD_AA_MINB 5
#endif

#define GSR_PRE_BWD_PARAMS                                                                                          \
    int N, const float* __restrict__ xyz, const float* __restrict__ quat, const float* __restrict__ scale,          \
        const float* __restrict__ opa_logit, const float* __restrict__ Tdev, const float* __restrict__ Kdev,        \
        const float* __restrict__ camdev, const uint8_t* __restrict__ visible, const float* __restrict__ g_rows,    \
        int rows_uv, const float* __restrict__ g_uv_compact,                                                         \
        const uint64_t* __restrict__ scan, float* __restrict__ o_xyz, float* __restrict__ o_quat,                   \
        float* __restrict__ o_scale, float* __restrict__ o_opa, float* __restrict__ o_dc, float* __restrict__ o_sh, \
        int use_tma
#define GSR_PRE_BWD_FORWARD                                                                                      \
    N, xyz, quat, scale, opa_logit, Tdev, Kdev, camdev, visible, g_rows, rows_uv, g_uv_compact, scan, o_xyz, o_quat, \
        o_scale, o_opa, o_dc, o_sh, use_tma
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_BWD_MINB) k_preprocess_bwd(GSR_PRE_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, false, false, false>(GSR_PRE_BWD_FORWARD, nullptr);
}
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_BWD_MINB) k_preprocess_bwd_depth(GSR_PRE_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, true, false, false>(GSR_PRE_BWD_FORWARD, nullptr);
}
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_BWD_AA_MINB) k_preprocess_bwd_aa(GSR_PRE_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, false, true, false>(GSR_PRE_BWD_FORWARD, nullptr);
}
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_BWD_AA_MINB) k_preprocess_bwd_depth_aa(GSR_PRE_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, true, true, false>(GSR_PRE_BWD_FORWARD, nullptr);
}
#ifndef GSR_PRE_BWD_F3D_MINB
#define GSR_PRE_BWD_F3D_MINB 5
#endif
#define GSR_PRE_BWD_F3D_KERNEL(name, depth, aa)                                                                    \
    template <int N_SH, bool HAS_SH>                                                                             \
    __global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_BWD_F3D_MINB)                                         \
        name(GSR_PRE_BWD_PARAMS, const float* __restrict__ filter3d) {                                           \
        preprocess_bwd<N_SH, HAS_SH, depth, aa, true>(GSR_PRE_BWD_FORWARD, filter3d);                            \
    }
GSR_PRE_BWD_F3D_KERNEL(k_preprocess_bwd_f3d, false, false)
GSR_PRE_BWD_F3D_KERNEL(k_preprocess_bwd_depth_f3d, true, false)
GSR_PRE_BWD_F3D_KERNEL(k_preprocess_bwd_aa_f3d, false, true)
GSR_PRE_BWD_F3D_KERNEL(k_preprocess_bwd_depth_aa_f3d, true, true)
#undef GSR_PRE_BWD_F3D_KERNEL
#undef GSR_PRE_BWD_PARAMS
#undef GSR_PRE_BWD_FORWARD

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// GSR_MODE_ABSGRAD only changes the render backward (row slots 10-11, which the per-gaussian backward does not read)
constexpr int KNOWN_MODES = GSR_MODE_DEPTH_ALPHA | GSR_MODE_ANTIALIASED | GSR_MODE_ABSGRAD | GSR_MODE_FILTER3D;

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_camera_centre(const float* camera_T_world, float* centre, void* stream) {
    if (camera_T_world == nullptr || centre == nullptr) return GSR_ERR_BAD_ARG;
    k_camera_centre<<<1, 32, 0, (cudaStream_t)stream>>>(camera_T_world, centre);
    return (int)cudaGetLastError();
}

size_t gsr_preprocess_temp_bytes(int N) {
    size_t b = 0;
    cub::DeviceScan::InclusiveSum((void*)nullptr, b, (uint64_t*)nullptr, (uint64_t*)nullptr, N > 0 ? N : 1);
    return align256(b) + align256(sizeof(uint64_t) * (size_t)(N > 0 ? N : 1));
}

int gsr_preprocess_forward(int mode, int N, int n_sh_rest, const float* xyz, const float* xyz_camera_frame,
                           int cam_first, const float* quaternion, const float* scale, const float* opacity_logit,
                           const float* filter3d, const float* rgb_dc, const float* sh_rest,
                           const float* camera_T_world, const float* K,
                           const float* camera_centre, int H, int W, float near_thresh, float far_thresh,
                           float cull_mask_padding, float mh_dist, uint32_t depth_base, float* records,
                           uint32_t* depth_key, uint8_t* visible, uint64_t* scan, uint64_t* tile_mask,
                           uint32_t* tile_win, void* temp, size_t temp_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if ((mode & ~KNOWN_MODES) != 0) return GSR_ERR_BAD_ARG;
    if (((mode & GSR_MODE_FILTER3D) != 0) != (filter3d != nullptr)) return GSR_ERR_BAD_ARG;
    if (N <= 0) return GSR_OK;
    if (temp_bytes < gsr_preprocess_temp_bytes(N)) return GSR_ERR_BAD_ARG;
    if ((tile_mask == nullptr) != (tile_win == nullptr)) return GSR_ERR_BAD_ARG;
    size_t scan_bytes = 0;
    cub::DeviceScan::InclusiveSum((void*)nullptr, scan_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, N);
    uint64_t* packed = reinterpret_cast<uint64_t*>((char*)temp + align256(scan_bytes));
    const int ntx = (W + TILE - 1) / TILE, nty = (H + TILE - 1) / TILE;
    const dim3 grid((N + PRE_THREADS - 1) / PRE_THREADS), block(PRE_THREADS);
    const int use_tma = (aligned16(records) && (sh_rest == nullptr || aligned16(sh_rest))) ? 1 : 0;
#define GSR_PRE_ARGS                                                                              \
    N, xyz, xyz_camera_frame, cam_first, quaternion, scale, opacity_logit, rgb_dc, sh_rest, camera_T_world, K, \
        camera_centre, (float)W, (float)H,                                                                 \
        near_thresh, far_thresh, cull_mask_padding, mh_dist, ntx, nty, depth_base, records, depth_key, visible, \
        packed, tile_mask, tile_win, use_tma
#define GSR_PRE_FWD_F3D_SWITCH(kernel)                                                                  \
    switch (n_sh_rest) {                                                                                \
        case 0: kernel<1, false><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;                \
        case 3: kernel<4, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;                 \
        case 8: kernel<9, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;                 \
        case 15: kernel<16, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;               \
        default: return GSR_ERR_UNSUPPORTED;                                                            \
    }
    if ((mode & GSR_MODE_FILTER3D) && (mode & GSR_MODE_ANTIALIASED)) {
        GSR_PRE_FWD_F3D_SWITCH(k_preprocess_fwd_aa_f3d)
    } else if (mode & GSR_MODE_FILTER3D) {
        GSR_PRE_FWD_F3D_SWITCH(k_preprocess_fwd_f3d)
    } else if (mode & GSR_MODE_ANTIALIASED) {
        switch (n_sh_rest) {
            case 0: k_preprocess_fwd_aa<1, false><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 3: k_preprocess_fwd_aa<4, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 8: k_preprocess_fwd_aa<9, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 15: k_preprocess_fwd_aa<16, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            default: return GSR_ERR_UNSUPPORTED;
        }
    } else {
        switch (n_sh_rest) {
            case 0: k_preprocess_fwd<1, false><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 3: k_preprocess_fwd<4, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 8: k_preprocess_fwd<9, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 15: k_preprocess_fwd<16, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            default: return GSR_ERR_UNSUPPORTED;
        }
    }
#undef GSR_PRE_FWD_F3D_SWITCH
#undef GSR_PRE_ARGS
    cudaError_t e = cub::DeviceScan::InclusiveSum(temp, scan_bytes, packed, scan, N, st);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

int gsr_preprocess_backward(int mode, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                            const float* scale, const float* opacity_logit, const float* filter3d,
                            const float* camera_T_world,
                            const float* K, const float* camera_centre, const uint8_t* visible,
                            const float* grad_rows, int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan,
                            float* g_xyz, float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                            float* g_sh_rest, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if ((mode & ~KNOWN_MODES) != 0) return GSR_ERR_BAD_ARG;
    if (((mode & GSR_MODE_FILTER3D) != 0) != (filter3d != nullptr)) return GSR_ERR_BAD_ARG;
    if (N <= 0) return GSR_OK;
    if (grad_rows == nullptr || !aligned16(grad_rows)) return GSR_ERR_BAD_ARG;
    if (grad_uv_compact != nullptr && scan == nullptr) return GSR_ERR_BAD_ARG;
    const dim3 grid((N + PRE_THREADS - 1) / PRE_THREADS), block(PRE_THREADS);
    const int use_tma = (aligned16(g_xyz) && aligned16(g_quaternion) && aligned16(g_scale) &&
                         aligned16(g_opacity_logit) && aligned16(g_rgb_dc) &&
                         (g_sh_rest == nullptr || aligned16(g_sh_rest)))
                            ? 1
                            : 0;
#define GSR_PRE_ARGS                                                                                   \
    N, xyz, quaternion, scale, opacity_logit, camera_T_world, K, camera_centre, visible, grad_rows, use_rows_uv, \
        grad_uv_compact, scan, g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, use_tma
#define GSR_PRE_BWD_SWITCH(kernel)                                                      \
    switch (n_sh_rest) {                                                                \
        case 0: kernel<1, false><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;          \
        case 3: kernel<4, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;           \
        case 8: kernel<9, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;           \
        case 15: kernel<16, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;         \
        default: return GSR_ERR_UNSUPPORTED;                                            \
    }
    const bool depth = (mode & GSR_MODE_DEPTH_ALPHA) != 0, antialiased = (mode & GSR_MODE_ANTIALIASED) != 0;
    if (mode & GSR_MODE_FILTER3D) {
#define GSR_PRE_BWD_F3D_SWITCH(kernel)                                                      \
    switch (n_sh_rest) {                                                                    \
        case 0: kernel<1, false><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;    \
        case 3: kernel<4, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;     \
        case 8: kernel<9, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;     \
        case 15: kernel<16, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;   \
        default: return GSR_ERR_UNSUPPORTED;                                                \
    }
        if (antialiased && depth) {
            GSR_PRE_BWD_F3D_SWITCH(k_preprocess_bwd_depth_aa_f3d)
        } else if (antialiased) {
            GSR_PRE_BWD_F3D_SWITCH(k_preprocess_bwd_aa_f3d)
        } else if (depth) {
            GSR_PRE_BWD_F3D_SWITCH(k_preprocess_bwd_depth_f3d)
        } else {
            GSR_PRE_BWD_F3D_SWITCH(k_preprocess_bwd_f3d)
        }
#undef GSR_PRE_BWD_F3D_SWITCH
    } else if (antialiased && depth) {
        GSR_PRE_BWD_SWITCH(k_preprocess_bwd_depth_aa)
    } else if (antialiased) {
        GSR_PRE_BWD_SWITCH(k_preprocess_bwd_aa)
    } else if (depth) {
        GSR_PRE_BWD_SWITCH(k_preprocess_bwd_depth)
    } else {
        GSR_PRE_BWD_SWITCH(k_preprocess_bwd)
    }
#undef GSR_PRE_BWD_SWITCH
#undef GSR_PRE_ARGS
    return (int)cudaGetLastError();
}

}  // extern "C"
