// gsr_surfels.cu — 2-D Gaussian surfels (2DGS): the per-gaussian stages and the tile kernels of rasterize_surfels
// (libgsr_surfels.so, C ABI include/gsr_surfels.h, model DESIGN.md 3.25).  The kernel bodies are gsr_surfels.cuh's,
// shared with the lens kernels of gsr_surfels_lens.cu.
//
// Binning is libgsr_b200.so's (gsr_emit_keys / gsr_sort_keys / gsr_tile_ranges) on a 48-byte binning record written
// here; the tile kernels are a plain design of their own (one CTA per 16x16 tile, one pixel per thread, batches of
// surfel records staged in shared memory) because the tuned walk of gsr_tile_walk.cuh is pinned to the conic record.
#include <cub/cub.cuh>

#include "gsr_surfels.cuh"

namespace gsr {
namespace surfel {

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// ---- per-gaussian forward ---------------------------------------------------------------------------------------------
template <int N_SH>
__global__ void __launch_bounds__(PRE)
    k_surfel_fwd(int N, const float* __restrict__ xyz, const float* __restrict__ xyz_cam, int cam_first,
                 const float* __restrict__ quat, const float* __restrict__ scale, const float* __restrict__ opa_logit,
                 const float* __restrict__ rgb_dc, const float* __restrict__ sh_rest, const float* __restrict__ Tdev,
                 const float* __restrict__ Kdev, const float* __restrict__ camdev, float width, float height,
                 float near_t, float far_t, float pad, float mh, int ntx, int nty, uint32_t depth_base,
                 float* __restrict__ surfels, float* __restrict__ bins, uint32_t* __restrict__ zkey,
                 uint8_t* __restrict__ visible, uint64_t* __restrict__ packed, uint64_t* __restrict__ tile_mask,
                 uint32_t* __restrict__ tile_win) {
    surfel_fwd<N_SH, 0>(N, xyz, xyz_cam, cam_first, quat, scale, opa_logit, rgb_dc, sh_rest, Tdev, Kdev, camdev, width,
                        height, near_t, far_t, pad, mh, ntx, nty, depth_base, surfels, bins, zkey, visible, packed,
                        tile_mask, tile_win, nullptr);
}

// ---- tile forward -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PIX)
    k_surfel_render_fwd(const float* __restrict__ surfels, const uint64_t* __restrict__ keys, int id_bits,
                        const int32_t* __restrict__ ids, const int32_t* __restrict__ ranges,
                        const float* __restrict__ bg, int H, int W, float near_t, float ms, float r2,
                        float* __restrict__ image, float* __restrict__ depth, float* __restrict__ alpha,
                        float* __restrict__ normal, float* __restrict__ distortion, int32_t* __restrict__ last,
                        float* __restrict__ totals) {
    surfel_render_fwd<false>(surfels, keys, id_bits, ids, ranges, bg, H, W, near_t, ms, r2, nullptr, image, depth, alpha,
                             normal, distortion, last, totals);
}

// ---- tile backward ----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PIX)
    k_surfel_render_bwd(const float* __restrict__ surfels, const uint64_t* __restrict__ keys, int id_bits,
                        const int32_t* __restrict__ ids, const int32_t* __restrict__ ranges,
                        const float* __restrict__ bg, int H, int W, float near_t, float ms, float r2,
                        const float* __restrict__ alpha, const int32_t* __restrict__ last,
                        const float* __restrict__ totals, const float* __restrict__ g_img,
                        const float* __restrict__ g_dep, const float* __restrict__ g_alp,
                        const float* __restrict__ g_nrm, const float* __restrict__ g_dis, float* __restrict__ rows) {
    __shared__ float4 s_rec[BATCH * 5];
    __shared__ int s_id[BATCH];
    const int ntx = (W + TILE - 1) / TILE;
    const int tile = blockIdx.x, tx = tile % ntx, ty = tile / ntx;
    const int px = tx * TILE + (threadIdx.x & 15), py = ty * TILE + (threadIdx.x >> 4);
    const bool inside = px < W && py < H;
    const float x = (float)px, y = (float)py;
    const int start = ranges[tile], end = ranges[tile + 1];
    const int lane = threadIdx.x & 31;
    int lst = -1;
    float Wt = 0.f, WM = 0.f, WM2 = 0.f, T = 1.f, S = 0.f, Gi[3] = {0.f, 0.f, 0.f}, Gn[3] = {0.f, 0.f, 0.f}, Gd = 0.f,
          Ga = 0.f, Gx = 0.f;
    if (inside) {
        const size_t pix = (size_t)py * W + px;
        lst = last[pix];
        Wt = alpha[pix];
        T = totals[pix * 3];
        WM = totals[pix * 3 + 1];
        WM2 = totals[pix * 3 + 2];
#pragma unroll
        for (int c = 0; c < 3; ++c) { Gi[c] = g_img[pix * 3 + c]; Gn[c] = g_nrm[pix * 3 + c]; }
        Gd = g_dep[pix];
        Ga = g_alp[pix];
        Gx = g_dis[pix];
        // d image / d alpha_i of the background term T_final bg (where it was added)
        if (Wt < 0.999f) S = T * (Gi[0] * bg[0] + Gi[1] * bg[1] + Gi[2] * bg[2]);
    }
    const int nb = (end - start + BATCH - 1) / BATCH;
    for (int bi = nb - 1; bi >= 0; --bi) {
        const int p0 = start + bi * BATCH;
        if (!__syncthreads_or(lst >= p0)) continue;
        const int n = min(BATCH, end - p0);
        stage_batch(s_rec, surfels, keys, id_bits, ids, p0, n);
        for (int k = threadIdx.x; k < n; k += PIX) s_id[k] = pair_id(keys, id_bits, ids, p0 + k);
        __syncthreads();
        for (int j = n - 1; j >= 0; --j) {
            const float* r = reinterpret_cast<const float*>(s_rec + j * 5);
            float g[SG - 1];
#pragma unroll
            for (int k = 0; k < SG - 1; ++k) g[k] = 0.f;
            Hit h;
            const bool on = p0 + j <= lst && intersect<false>(r, x, y, nullptr, r2, h);
            if (on) {
                const float* M = r + S_M;
                const float om = 1.0f - h.alpha;
                T = T / om;  // T_i, the transmittance in front of this surfel
                const float w = T * h.alpha;
                const float m = ndc_depth(h.z, near_t, ms);
                const float e = fmaf(m, fmaf(m, Wt, -2.0f * WM), WM2);  // d distortion / d w_i
                const float gf = Gi[0] * r[S_C] + Gi[1] * r[S_C + 1] + Gi[2] * r[S_C + 2] + Gn[0] * r[S_N] +
                                 Gn[1] * r[S_N + 1] + Gn[2] * r[S_N + 2] + Gd * h.z + Ga + Gx * e;
                const float g_alpha = T * gf - S / om;
                S = fmaf(w, gf, S);
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    g[G_C + c] = w * Gi[c];
                    g[G_N + c] = w * Gn[c];
                }
                // depth and distortion through z: dm/dz = m_scale near / z^2
                const float gz = w * Gd + Gx * 2.0f * w * (m * Wt - WM) * (ms * near_t / (h.z * h.z));
                float grho = 0.f;
                if (__fmul_rn(r[S_OPA], h.G) < 0.99f) {  // not clamped
                    g[G_OPA] = g_alpha * h.G;
                    grho = -0.5f * h.alpha * g_alpha;
                }
                if (h.use3) {
                    const float ga = 2.0f * h.a * grho + gz * M[6], gb = 2.0f * h.b * grho + gz * M[7];
                    g[G_M + 6] += gz * h.a;
                    g[G_M + 7] += gz * h.b;
                    g[G_M + 8] += gz;
                    const float ic = 1.0f / h.c2;
                    const float gc[3] = {ga * ic, gb * ic, -(ga * h.a + gb * h.b) * ic};
                    // c = hx x hy: d/dhx = hy x gc, d/dhy = gc x hx
                    const float ghx[3] = {h.hy[1] * gc[2] - h.hy[2] * gc[1], h.hy[2] * gc[0] - h.hy[0] * gc[2],
                                          h.hy[0] * gc[1] - h.hy[1] * gc[0]};
                    const float ghy[3] = {gc[1] * h.hx[2] - gc[2] * h.hx[1], gc[2] * h.hx[0] - gc[0] * h.hx[2],
                                          gc[0] * h.hx[1] - gc[1] * h.hx[0]};
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        g[G_M + k] = -ghx[k];
                        g[G_M + 3 + k] = -ghy[k];
                        g[G_M + 6 + k] += x * ghx[k] + y * ghy[k];
                    }
                } else {
                    // rho2 = 2 |(x, y) - (u_c, v_c)|^2
                    g[G_UC] = -4.0f * h.dx * grho;
                    g[G_UC + 1] = -4.0f * h.dy * grho;
                    g[G_PZ] = gz;
                }
            }
            // one atomic per warp and field
            if (__any_sync(0xffffffffu, on)) {
#pragma unroll
                for (int k = 0; k < SG - 1; ++k) {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) g[k] += __shfl_xor_sync(0xffffffffu, g[k], o);
                }
                if (lane == 0) {
                    float4* dst = reinterpret_cast<float4*>(rows + (size_t)s_id[j] * SG);
                    atomicAdd(dst + 0, make_float4(g[0], g[1], g[2], g[3]));
                    atomicAdd(dst + 1, make_float4(g[4], g[5], g[6], g[7]));
                    atomicAdd(dst + 2, make_float4(g[8], g[9], g[10], g[11]));
                    atomicAdd(dst + 3, make_float4(g[12], g[13], g[14], g[15]));
                    atomicAdd(dst + 4, make_float4(g[16], g[17], g[18], 0.f));
                }
            }
        }
        __syncthreads();
    }
}

// ---- per-gaussian backward --------------------------------------------------------------------------------------------
__global__ void k_surfel_uv_grad(int M, const int32_t* __restrict__ vis_idx, const float* __restrict__ surfels,
                                 const float* __restrict__ rows, float* __restrict__ out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= M) return;
    const size_t i = (size_t)vis_idx[k];
    reinterpret_cast<float2*>(out)[k] = uv_grad_of<0>(surfels + i * SF, rows + i * SG, nullptr, nullptr);
}

template <int N_SH>
__global__ void __launch_bounds__(PRE)
    k_surfel_bwd(int N, const float* __restrict__ xyz, const float* __restrict__ quat,
                 const float* __restrict__ scale, const float* __restrict__ opa_logit, const float* __restrict__ Tdev,
                 const float* __restrict__ Kdev, const float* __restrict__ camdev, const uint8_t* __restrict__ visible,
                 const float* __restrict__ surfels, const float* __restrict__ rows,
                 const float* __restrict__ g_uv_compact, const uint64_t* __restrict__ scan, int uv_emitted,
                 float* __restrict__ o_xyz, float* __restrict__ o_quat, float* __restrict__ o_scale,
                 float* __restrict__ o_opa, float* __restrict__ o_dc, float* __restrict__ o_sh) {
    surfel_bwd<N_SH, 0>(N, xyz, quat, scale, opa_logit, Tdev, Kdev, camdev, visible, surfels, rows, g_uv_compact, scan,
                        uv_emitted, o_xyz, o_quat, o_scale, o_opa, o_dc, o_sh, nullptr);
}

}  // namespace surfel
}  // namespace gsr

using namespace gsr;
using namespace gsr::surfel;

static bool n_sh_ok(int n) { return n == 0 || n == 3 || n == 8 || n == 15; }

extern "C" {

size_t gsr_surfel_temp_bytes(int N) {
    size_t b = 0;
    cub::DeviceScan::InclusiveSum((void*)nullptr, b, (uint64_t*)nullptr, (uint64_t*)nullptr, N > 0 ? N : 1);
    return align256(b) + align256(sizeof(uint64_t) * (size_t)(N > 0 ? N : 1));
}

int gsr_surfel_preprocess_forward(int N, int n_sh_rest, const float* xyz, const float* xyz_camera_frame, int cam_first,
                                  const float* quaternion, const float* scale, const float* opacity_logit,
                                  const float* rgb_dc, const float* sh_rest, const float* camera_T_world,
                                  const float* K, const float* camera_centre, int H, int W, float near_thresh,
                                  float far_thresh, float cull_mask_padding, float mh_dist, uint32_t depth_base,
                                  float* surfels, float* bin_records, uint32_t* depth_key, uint8_t* visible,
                                  uint64_t* scan, uint64_t* tile_mask, uint32_t* tile_win, void* temp,
                                  size_t temp_bytes, void* stream) {
    if (N < 0 || H <= 0 || W <= 0 || !n_sh_ok(n_sh_rest) || !(mh_dist > 0.0f)) return GSR_ERR_BAD_ARG;
    if (N == 0) return GSR_OK;
    if (!xyz || !quaternion || !scale || !opacity_logit || !rgb_dc || !camera_T_world || !K || !surfels ||
        !bin_records || !depth_key || !visible || !scan || !temp)
        return GSR_ERR_BAD_ARG;
    if (n_sh_rest > 0 && (!sh_rest || !camera_centre)) return GSR_ERR_BAD_ARG;
    if ((tile_mask == nullptr) != (tile_win == nullptr)) return GSR_ERR_BAD_ARG;
    if (((uintptr_t)surfels | (uintptr_t)bin_records) & 15u) return GSR_ERR_BAD_ARG;
    if (temp_bytes < gsr_surfel_temp_bytes(N)) return GSR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    size_t scan_bytes = 0;
    cub::DeviceScan::InclusiveSum((void*)nullptr, scan_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, N);
    uint64_t* packed = reinterpret_cast<uint64_t*>((char*)temp + align256(scan_bytes));
    const int ntx = (W + TILE - 1) / TILE, nty = (H + TILE - 1) / TILE;
    const dim3 grid((N + PRE - 1) / PRE), block(PRE);
#define GSR_SURFEL_FWD(NS)                                                                                          \
    k_surfel_fwd<NS><<<grid, block, 0, st>>>(N, xyz, xyz_camera_frame, cam_first, quaternion, scale, opacity_logit, \
                                             rgb_dc, sh_rest, camera_T_world, K, camera_centre, (float)W, (float)H,  \
                                             near_thresh, far_thresh, cull_mask_padding, mh_dist, ntx, nty,          \
                                             depth_base, surfels, bin_records, depth_key, visible, packed,           \
                                             tile_mask, tile_win)
    switch (n_sh_rest) {
        case 0: GSR_SURFEL_FWD(1); break;
        case 3: GSR_SURFEL_FWD(4); break;
        case 8: GSR_SURFEL_FWD(9); break;
        default: GSR_SURFEL_FWD(16); break;
    }
#undef GSR_SURFEL_FWD
    cudaError_t e = cub::DeviceScan::InclusiveSum(temp, scan_bytes, packed, scan, N, st);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

static bool pairs_ok(const uint64_t* keys, int id_bits, const int32_t* ids) {
    return (keys != nullptr) != (ids != nullptr) && (keys == nullptr || (id_bits >= 1 && id_bits <= 32));
}

int gsr_surfel_render_forward(const float* surfels, const uint64_t* keys_sorted, int id_bits, const int32_t* ids_sorted,
                              const int32_t* tile_ranges, const float* background_rgb, int H, int W, float near_thresh,
                              float m_scale, float mh_dist, float* image, float* depth, float* alpha, float* normal,
                              float* distortion, int32_t* last, float* totals, void* stream) {
    if (H <= 0 || W <= 0 || !(mh_dist > 0.0f) || !pairs_ok(keys_sorted, id_bits, ids_sorted)) return GSR_ERR_BAD_ARG;
    if (!surfels || !tile_ranges || !background_rgb || !image || !depth || !alpha || !normal || !distortion || !last ||
        !totals || ((uintptr_t)surfels & 15u))
        return GSR_ERR_BAD_ARG;
    const int n_tiles = ((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE);
    k_surfel_render_fwd<<<n_tiles, PIX, 0, (cudaStream_t)stream>>>(
        surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, background_rgb, H, W, near_thresh, m_scale,
        mh_dist * mh_dist, image, depth, alpha, normal, distortion, last, totals);
    return (int)cudaGetLastError();
}

int gsr_surfel_render_backward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                               const int32_t* ids_sorted, const int32_t* tile_ranges, const float* background_rgb,
                               int H, int W, float near_thresh, float m_scale, float mh_dist, const float* alpha,
                               const int32_t* last, const float* totals, const float* grad_image,
                               const float* grad_depth, const float* grad_alpha, const float* grad_normal,
                               const float* grad_distortion, float* grad_rows, void* stream) {
    if (H <= 0 || W <= 0 || !(mh_dist > 0.0f) || !pairs_ok(keys_sorted, id_bits, ids_sorted)) return GSR_ERR_BAD_ARG;
    if (!surfels || !tile_ranges || !background_rgb || !alpha || !last || !totals || !grad_image || !grad_depth ||
        !grad_alpha || !grad_normal || !grad_distortion || !grad_rows ||
        (((uintptr_t)surfels | (uintptr_t)grad_rows) & 15u))
        return GSR_ERR_BAD_ARG;
    const int n_tiles = ((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE);
    k_surfel_render_bwd<<<n_tiles, PIX, 0, (cudaStream_t)stream>>>(
        surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, background_rgb, H, W, near_thresh, m_scale,
        mh_dist * mh_dist, alpha, last, totals, grad_image, grad_depth, grad_alpha, grad_normal, grad_distortion,
        grad_rows);
    return (int)cudaGetLastError();
}

int gsr_surfel_uv_grad(int M, const int32_t* vis_idx, const float* surfels, const float* grad_rows, float* uv_grad,
                       void* stream) {
    if (M < 0) return GSR_ERR_BAD_ARG;
    if (M == 0) return GSR_OK;
    if (!vis_idx || !surfels || !grad_rows || !uv_grad || ((uintptr_t)uv_grad & 7u)) return GSR_ERR_BAD_ARG;
    k_surfel_uv_grad<<<(M + 255) / 256, 256, 0, (cudaStream_t)stream>>>(M, vis_idx, surfels, grad_rows, uv_grad);
    return (int)cudaGetLastError();
}

int gsr_surfel_preprocess_backward(int N, int n_sh_rest, const float* xyz, const float* quaternion, const float* scale,
                                   const float* opacity_logit, const float* camera_T_world, const float* K,
                                   const float* camera_centre, const uint8_t* visible, const float* surfels,
                                   const float* grad_rows, const float* grad_uv_compact, const uint64_t* scan,
                                   int uv_grad_emitted, float* g_xyz, float* g_quaternion, float* g_scale,
                                   float* g_opacity_logit, float* g_rgb_dc, float* g_sh_rest, void* stream) {
    if (N < 0 || !n_sh_ok(n_sh_rest)) return GSR_ERR_BAD_ARG;
    if (N == 0) return GSR_OK;
    if (!xyz || !quaternion || !scale || !opacity_logit || !camera_T_world || !K || !visible || !surfels ||
        !grad_rows || !g_xyz || !g_quaternion || !g_scale || !g_opacity_logit || !g_rgb_dc)
        return GSR_ERR_BAD_ARG;
    if (n_sh_rest > 0 && (!camera_centre || !g_sh_rest)) return GSR_ERR_BAD_ARG;
    if (grad_uv_compact != nullptr && scan == nullptr) return GSR_ERR_BAD_ARG;
    if (((uintptr_t)surfels | (uintptr_t)grad_rows) & 15u) return GSR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid((N + PRE - 1) / PRE), block(PRE);
#define GSR_SURFEL_BWD(NS)                                                                                            \
    k_surfel_bwd<NS><<<grid, block, 0, st>>>(N, xyz, quaternion, scale, opacity_logit, camera_T_world, K,             \
                                             camera_centre, visible, surfels, grad_rows, grad_uv_compact, scan,       \
                                             uv_grad_emitted ? 1 : 0, g_xyz, g_quaternion, g_scale, g_opacity_logit, \
                                             g_rgb_dc, g_sh_rest)
    switch (n_sh_rest) {
        case 0: GSR_SURFEL_BWD(1); break;
        case 3: GSR_SURFEL_BWD(4); break;
        case 8: GSR_SURFEL_BWD(9); break;
        default: GSR_SURFEL_BWD(16); break;
    }
#undef GSR_SURFEL_BWD
    return (int)cudaGetLastError();
}

}  // extern "C"
