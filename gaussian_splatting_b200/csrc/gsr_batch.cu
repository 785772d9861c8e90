// gsr_batch.cu — the per-Gaussian backward of C views of one scene in one pass (rasterize_batch).
//
// A CTA takes 128 gaussians, reads their parameters once and walks the views in order.  For every view that sees a
// gaussian it forms that view's VJP with the single-view kernel's own statement block (GSR_PRE_BWD_VIEW,
// gsr_preprocess.cuh) and adds it to the running sums with one rounded fp32 add, so the result is the view-order
// sum of the single-view gradients bit for bit (up to the sign of zero).  The sums of the SH rest coefficients live
// in the shared-memory staging the single-view kernel stores from; everything leaves once, by the same bulk stores.
#include "gsr_preprocess.cuh"

#include "../../include/gsr_batch.h"

namespace gsr {

template <int N_SH, bool HAS_SH, bool DEPTH, bool ANTIALIAS, bool FILTER3D>
__device__ __forceinline__ void batch_preprocess_bwd(
    int C, int N, const float* __restrict__ xyz, const float* __restrict__ quat, const float* __restrict__ scale,
    const float* __restrict__ opa_logit, const float* __restrict__ Tdev, const float* __restrict__ Kdev,
    const float* __restrict__ camdev, const uint8_t* __restrict__ visible, const float* __restrict__ g_rows,
    int rows_uv, const float* __restrict__ g_uv_compact, const uint64_t* __restrict__ scan, float* __restrict__ o_xyz,
    float* __restrict__ o_quat, float* __restrict__ o_scale, float* __restrict__ o_opa, float* __restrict__ o_dc,
    float* __restrict__ o_sh, int use_tma, const float* __restrict__ filter3d) {
    constexpr int NR = N_SH - 1;
    constexpr int NR3 = HAS_SH ? 3 * NR : 1;
    __shared__ ViewConsts vc;
    __shared__ __align__(128) float s_sh[PRE_THREADS * NR3];
    __shared__ __align__(128) float s_xyz[PRE_THREADS * 3];
    __shared__ __align__(128) float s_quat[PRE_THREADS * 4];
    __shared__ __align__(128) float s_scale[PRE_THREADS * 3];
    __shared__ __align__(128) float s_opa[PRE_THREADS];
    __shared__ __align__(128) float s_dc[PRE_THREADS * 3];
    const int tid = threadIdx.x;
    const int i0 = blockIdx.x * PRE_THREADS;
    const int cnt = min(PRE_THREADS, N - i0);
    const bool tma = use_tma && cnt == PRE_THREADS;
    const int i = i0 + tid;
    // running sums over the views
    float ax[3] = {0.f, 0.f, 0.f}, aq[4] = {0.f, 0.f, 0.f, 0.f}, as[3] = {0.f, 0.f, 0.f}, ao = 0.f,
          adc[3] = {0.f, 0.f, 0.f};
    float* acc_sh = s_sh + tid * NR3;
    if (HAS_SH) {
#pragma unroll
        for (int k = 0; k < NR3; ++k) acc_sh[k] = 0.f;
    }
    bool any = false;
    if (i < N)
        for (int c = 0; c < C; ++c) any |= visible[(size_t)c * N + i] != 0;
    float x = 0.f, y = 0.f, z = 0.f, qw = 1.f, qx = 0.f, qy = 0.f, qz = 0.f, s0 = 0.f, s1 = 0.f, s2 = 0.f, opl = 0.f,
          f = 0.f;
    if (any) {
        if (FILTER3D) f = filter3d[i];
        x = xyz[i * 3 + 0]; y = xyz[i * 3 + 1]; z = xyz[i * 3 + 2];
        qw = quat[i * 4 + 0]; qx = quat[i * 4 + 1]; qy = quat[i * 4 + 2]; qz = quat[i * 4 + 3];
        s0 = scale[i * 3 + 0]; s1 = scale[i * 3 + 1]; s2 = scale[i * 3 + 2];
        opl = opa_logit[i];
    }
    size_t uv_base = 0;  // first compact uv row of view c
    for (int c = 0; c < C; ++c) {
        const size_t ci = (size_t)c * N + i;
        const bool vis = any && visible[ci] != 0;
        float gcv[3] = {0.f, 0.f, 0.f}, guv[2] = {0.f, 0.f}, gov = 0.f, grv[3] = {0.f, 0.f, 0.f}, gzc = 0.f;
        if (vis) {
            // view c's row, read exactly as the single-view kernel reads it
            const float4* row = reinterpret_cast<const float4*>(g_rows + ci * GSR_GRAD_ROW_FLOATS);
            const float4 r0 = row[0], r1 = row[1];
            grv[0] = r0.x; grv[1] = r0.y; grv[2] = r0.z; gov = r0.w;
            if (rows_uv) { guv[0] = r1.x; guv[1] = r1.y; }
            gcv[0] = r1.z; gcv[1] = r1.w;
            if (DEPTH) {
                const float2 r2 = *reinterpret_cast<const float2*>(g_rows + ci * GSR_GRAD_ROW_FLOATS + 8);
                gcv[2] = r2.x;
                gzc = r2.y;
            } else {
                gcv[2] = g_rows[ci * GSR_GRAD_ROW_FLOATS + 8];
            }
            if (g_uv_compact != nullptr) {
                const size_t r = uv_base + (size_t)(scan[ci] >> 32) - 1;
                const float2 t = *reinterpret_cast<const float2*>(g_uv_compact + r * 2);
                guv[0] = __fadd_rn(guv[0], t.x);
                guv[1] = __fadd_rn(guv[1], t.y);
            }
        }
        if (g_uv_compact != nullptr) uv_base += (size_t)(scan[(size_t)c * N + N - 1] >> 32);
        if (c > 0) __syncthreads();  // every thread is done with the previous view's constants
        load_view_cta(Tdev + 16 * c, Kdev + 9 * c, camdev != nullptr ? camdev + 3 * c : nullptr, vc, HAS_SH);
        if (vis) {
            float gx[3], gq[4], gs[3], go, gdc[3], v_sh[NR3];
            float* my_sh = v_sh;
            GSR_PRE_BWD_VIEW
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                ax[k] = __fadd_rn(ax[k], gx[k]);
                as[k] = __fadd_rn(as[k], gs[k]);
                adc[k] = __fadd_rn(adc[k], gdc[k]);
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) aq[k] = __fadd_rn(aq[k], gq[k]);
            ao = __fadd_rn(ao, go);
            if (HAS_SH) {
#pragma unroll
                for (int k = 0; k < NR3; ++k) acc_sh[k] = __fadd_rn(acc_sh[k], v_sh[k]);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) { s_xyz[tid * 3 + k] = ax[k]; s_scale[tid * 3 + k] = as[k]; s_dc[tid * 3 + k] = adc[k]; }
    *reinterpret_cast<float4*>(s_quat + tid * 4) = make_float4(aq[0], aq[1], aq[2], aq[3]);
    s_opa[tid] = ao;
    if (tma) {
        fence_proxy_async_smem();
        __syncthreads();
        if (tid == 0) {
            tma_store_1d(o_xyz + (size_t)i0 * 3, s_xyz, PRE_THREADS * 3 * 4);
            tma_store_1d(o_quat + (size_t)i0 * 4, s_quat, PRE_THREADS * 4 * 4);
            tma_store_1d(o_scale + (size_t)i0 * 3, s_scale, PRE_THREADS * 3 * 4);
            tma_store_1d(o_opa + (size_t)i0, s_opa, PRE_THREADS * 4);
            tma_store_1d(o_dc + (size_t)i0 * 3, s_dc, PRE_THREADS * 3 * 4);
            if (HAS_SH) tma_store_1d(o_sh + (size_t)i0 * NR3, s_sh, PRE_THREADS * NR3 * 4);
            tma_store_commit_and_wait();
        }
    } else {
        __syncthreads();
        coop_copy(o_xyz + (size_t)i0 * 3, s_xyz, cnt * 3);
        coop_copy(o_quat + (size_t)i0 * 4, s_quat, cnt * 4);
        coop_copy(o_scale + (size_t)i0 * 3, s_scale, cnt * 3);
        coop_copy(o_opa + (size_t)i0, s_opa, cnt);
        coop_copy(o_dc + (size_t)i0 * 3, s_dc, cnt * 3);
        if (HAS_SH) coop_copy(o_sh + (size_t)i0 * NR3, s_sh, cnt * NR3);
    }
}

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
