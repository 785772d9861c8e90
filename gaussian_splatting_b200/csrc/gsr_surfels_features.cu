// gsr_surfels_features.cu — per-gaussian feature channels blended with the surfel colour's weights (DESIGN.md 3.27),
// forward and backward (libgsr_surfels_features.so, C ABI include/gsr_surfels_features.h).
//
// The tile kernels of gsr_surfels.cuh's design: one CTA per 16x16 tile and chunk of FCH channels (grid z), one pixel
// per thread, batches of surfel records staged in shared memory with the chunk's FCH feature floats beside them.
// RAYS: each pixel's ray from the ray map (the lens kernels), else (x, y, 1) (the pinhole).
//
// Forward: intersect<RAYS> on the same records gives every (pixel, surfel) the colour forward's decision and alpha, and
// the walk stops at the pixel's last contributor (the colour forward's `last`), so A and w_i = alpha_i (1 - A_i) are
// the colour's floats, bit for bit.
//
// Backward: the colour backward's recurrence (T back from the final transmittance totals[0], T_i = T / (1 - alpha_i),
// the 0.99 clamp) with the colour replaced by the chunk's features and no background.  Each (pixel, surfel) gives 16
// moments (the FCH feature gradients, dM, d opacity, d u_c, d v_c); a butterfly over the warp leaves moment k's warp
// sum in lanes 2k and 2k + 1, and the even lanes add the non-zero ones into grad_features and the gradient rows.
#include "gsr_surfels.cuh"
#include "../../include/gsr_surfels_features.h"

namespace gsr {
namespace surfel {

constexpr int FCH = 4;   // feature channels per CTA: one 16-byte copy per record
constexpr int NMOM = 16; // backward moments per (pixel, surfel): dM (9), d opacity, d u_c, d v_c, FCH feature gradients
static_assert(NMOM == 12 + FCH && NMOM * 2 == 32, "the butterfly leaves one moment per lane pair");

// the chunk's FCH floats of the n records stage_batch staged (fsrc: the chunk's first column)
__device__ __forceinline__ void stage_features(float4* __restrict__ s_feat, const float* __restrict__ fsrc, int stride,
                                               const uint64_t* __restrict__ keys, int id_bits,
                                               const int32_t* __restrict__ ids, int p0, int n) {
    for (int k = threadIdx.x; k < n; k += PIX)
        s_feat[k] = *reinterpret_cast<const float4*>(fsrc + (size_t)pair_id(keys, id_bits, ids, p0 + k) * stride);
}

template <bool RAYS>
__global__ void __launch_bounds__(PIX)
    k_surfel_features_fwd(const float* __restrict__ surfels, const uint64_t* __restrict__ keys, int id_bits,
                          const int32_t* __restrict__ ids, const int32_t* __restrict__ ranges, int H, int W, float r2,
                          const float* __restrict__ rays, const int32_t* __restrict__ last,
                          const float* __restrict__ features, int stride, int D, float* __restrict__ feature_map) {
    __shared__ float4 s_rec[BATCH * 5];
    __shared__ float4 s_feat[BATCH];
    const int ntx = (W + TILE - 1) / TILE;
    const int tile = blockIdx.x, tx = tile % ntx, ty = tile / ntx;
    const int c0 = blockIdx.z * FCH;
    const float* fsrc = features + c0;
    const int px = tx * TILE + (threadIdx.x & 15), py = ty * TILE + (threadIdx.x >> 4);
    const bool inside = px < W && py < H;
    const size_t pix = (size_t)py * W + px;
    const float x = (float)px, y = (float)py;
    float d[3] = {0.f, 0.f, 0.f};
    int lst = -1;
    if (inside) {
        if constexpr (RAYS) {
            d[0] = rays[pix * 3]; d[1] = rays[pix * 3 + 1]; d[2] = rays[pix * 3 + 2];
        }
        lst = last[pix];
    }
    const int start = ranges[tile], end = ranges[tile + 1];
    float A = 0.f, f[FCH];
#pragma unroll
    for (int c = 0; c < FCH; ++c) f[c] = 0.f;
    for (int p0 = start; p0 < end; p0 += BATCH) {
        if (!__syncthreads_or(lst >= p0)) break;
        const int n = min(BATCH, end - p0);
        stage_batch(s_rec, surfels, keys, id_bits, ids, p0, n);
        stage_features(s_feat, fsrc, stride, keys, id_bits, ids, p0, n);
        __syncthreads();
        const int m = min(n, lst - p0 + 1);  // up to the colour forward's last contributor
        for (int j = 0; j < m; ++j) {
            const float* r = reinterpret_cast<const float*>(s_rec + j * 5);
            Hit h;
            if (!intersect<RAYS>(r, x, y, d, r2, h)) continue;
            // the colour forward's weight and accumulated alpha, operation for operation
            const float w = __fmul_rn(h.alpha, __fsub_rn(1.0f, A));
            const float4 q = s_feat[j];
            f[0] = __fmaf_rn(w, q.x, f[0]);
            f[1] = __fmaf_rn(w, q.y, f[1]);
            f[2] = __fmaf_rn(w, q.z, f[2]);
            f[3] = __fmaf_rn(w, q.w, f[3]);
            A = __fadd_rn(A, w);
        }
    }
    if (!inside) return;
    const int nc = min(FCH, D - c0);
    float* o = feature_map + pix * D + c0;
#pragma unroll
    for (int c = 0; c < FCH; ++c)
        if (c < nc) o[c] = f[c];
}

// v[0..NMOM) of every lane -> the warp sum of moment (lane >> 1) in v[0]: each step halves the moments a lane keeps
// and trades the other half with its partner (16 shuffles in all)
__device__ __forceinline__ float warp_moments(float (&v)[NMOM], int lane) {
#pragma unroll
    for (int h = NMOM / 2, o = 16; h >= 1; h >>= 1, o >>= 1) {
        const bool upper = (lane & o) != 0;
#pragma unroll
        for (int k = 0; k < h; ++k) {
            const float send = upper ? v[k] : v[k + h];
            const float keep = upper ? v[k + h] : v[k];
            v[k] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
    }
    return v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
}

template <bool RAYS>
__global__ void __launch_bounds__(PIX)
    k_surfel_features_bwd(const float* __restrict__ surfels, const uint64_t* __restrict__ keys, int id_bits,
                          const int32_t* __restrict__ ids, const int32_t* __restrict__ ranges, int H, int W, float r2,
                          const float* __restrict__ rays, const int32_t* __restrict__ last,
                          const float* __restrict__ totals, const float* __restrict__ features, int stride, int D,
                          const float* __restrict__ grad_map, float* __restrict__ grad_features,
                          float* __restrict__ rows) {
    __shared__ float4 s_rec[BATCH * 5];
    __shared__ float4 s_feat[BATCH];
    __shared__ int s_id[BATCH];
    const int ntx = (W + TILE - 1) / TILE;
    const int tile = blockIdx.x, tx = tile % ntx, ty = tile / ntx;
    const int c0 = blockIdx.z * FCH;
    const float* fsrc = features + c0;
    const int px = tx * TILE + (threadIdx.x & 15), py = ty * TILE + (threadIdx.x >> 4);
    const bool inside = px < W && py < H;
    const float x = (float)px, y = (float)py;
    const int start = ranges[tile], end = ranges[tile + 1];
    const int lane = threadIdx.x & 31;
    const int nc = min(FCH, D - c0);
    int lst = -1;
    float T = 1.f, S = 0.f, Gf[FCH];
    float d[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < FCH; ++c) Gf[c] = 0.f;
    if (inside) {
        const size_t pix = (size_t)py * W + px;
        if constexpr (RAYS) {
            d[0] = rays[pix * 3]; d[1] = rays[pix * 3 + 1]; d[2] = rays[pix * 3 + 2];
        }
        lst = last[pix];
        T = totals[pix * 3];
#pragma unroll
        for (int c = 0; c < FCH; ++c)
            if (c < nc) Gf[c] = grad_map[pix * D + c0 + c];
    }
    // the moment lane pair (2q, 2q + 1) reduces, and where its even lane adds it
    const int q = lane >> 1;
    float* const dst_base = q < FCH ? grad_features + c0 + q : rows + (q < FCH + 10 ? q - FCH : G_UC + (q - FCH - 10));
    const int dst_stride = q < FCH ? stride : SG;
    const int nb = (end - start + BATCH - 1) / BATCH;
    for (int bi = nb - 1; bi >= 0; --bi) {
        const int p0 = start + bi * BATCH;
        if (!__syncthreads_or(lst >= p0)) continue;
        const int n = min(BATCH, end - p0);
        stage_batch(s_rec, surfels, keys, id_bits, ids, p0, n);
        stage_features(s_feat, fsrc, stride, keys, id_bits, ids, p0, n);
        for (int k = threadIdx.x; k < n; k += PIX) s_id[k] = pair_id(keys, id_bits, ids, p0 + k);
        __syncthreads();
        for (int j = n - 1; j >= 0; --j) {
            const float* r = reinterpret_cast<const float*>(s_rec + j * 5);
            // moments: [0, FCH) feature gradients, then dM (9), d opacity, d u_c, d v_c
            float g[NMOM];
#pragma unroll
            for (int k = 0; k < NMOM; ++k) g[k] = 0.f;
            Hit h;
            const bool on = p0 + j <= lst && intersect<RAYS>(r, x, y, d, r2, h);
            if (on) {
                const float om = 1.0f - h.alpha;
                T = T / om;  // T_i, the transmittance in front of this surfel
                const float w = T * h.alpha;
                const float4 fq = s_feat[j];
                const float gf = Gf[0] * fq.x + Gf[1] * fq.y + Gf[2] * fq.z + Gf[3] * fq.w;
                const float g_alpha = T * gf - S / om;
                S = fmaf(w, gf, S);
#pragma unroll
                for (int c = 0; c < FCH; ++c) g[c] = w * Gf[c];
                float* gm = g + FCH;
                float grho = 0.f;
                if (__fmul_rn(r[S_OPA], h.G) < 0.99f) {  // not clamped
                    gm[9] = g_alpha * h.G;
                    grho = -0.5f * h.alpha * g_alpha;
                }
                if (h.use3) {
                    const float ga = 2.0f * h.a * grho, gb = 2.0f * h.b * grho;
                    const float ic = 1.0f / h.c2;
                    const float gc[3] = {ga * ic, gb * ic, -(ga * h.a + gb * h.b) * ic};
                    // c = hx x hy: d/dhx = hy x gc, d/dhy = gc x hx
                    const float ghx[3] = {h.hy[1] * gc[2] - h.hy[2] * gc[1], h.hy[2] * gc[0] - h.hy[0] * gc[2],
                                          h.hy[0] * gc[1] - h.hy[1] * gc[0]};
                    const float ghy[3] = {gc[1] * h.hx[2] - gc[2] * h.hx[1], gc[2] * h.hx[0] - gc[0] * h.hx[2],
                                          gc[0] * h.hx[1] - gc[1] * h.hx[0]};
                    // hx = d_x M2 - d_z M0, hy = d_y M2 - d_z M1 (pinhole: d = (x, y, 1))
                    const float dx = RAYS ? d[0] : x, dy = RAYS ? d[1] : y, dz = RAYS ? d[2] : 1.0f;
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        gm[k] = -dz * ghx[k];
                        gm[3 + k] = -dz * ghy[k];
                        gm[6 + k] = dx * ghx[k] + dy * ghy[k];
                    }
                } else {
                    // rho2 = 2 |(x, y) - (u_c, v_c)|^2
                    gm[10] = -4.0f * h.dx * grho;
                    gm[11] = -4.0f * h.dy * grho;
                }
            }
            if (__any_sync(0xffffffffu, on)) {
                const float s = warp_moments(g, lane);
                if ((lane & 1) == 0 && s != 0.0f) atomicAdd(dst_base + (size_t)s_id[j] * dst_stride, s);
            }
        }
        __syncthreads();
    }
}

}  // namespace surfel
}  // namespace gsr

using namespace gsr;
using namespace gsr::surfel;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// the arguments both entry points share
static bool args_ok(const float* surfels, const uint64_t* keys, int id_bits, const int32_t* ids, const int32_t* ranges,
                    int H, int W, float mh_dist, const int32_t* last, const float* features, int stride, int D) {
    if ((keys == nullptr) == (ids == nullptr)) return false;  // exactly one id source
    if (keys != nullptr && (id_bits < 1 || id_bits > 32)) return false;
    if (surfels == nullptr || !aligned16(surfels) || ranges == nullptr || last == nullptr || features == nullptr ||
        !aligned16(features))
        return false;
    if (H <= 0 || W <= 0 || D <= 0 || !(mh_dist > 0.0f)) return false;
    if (stride % FCH != 0 || stride < D || stride >= D + FCH || stride / FCH > 65535) return false;
    return true;
}

extern "C" {

int gsr_surfel_render_features_forward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                                       const int32_t* ids_sorted, const int32_t* tile_ranges, int H, int W,
                                       float mh_dist, const float* rays, const int32_t* last, const float* features,
                                       int feature_stride, int D, float* feature_map, void* stream) {
    if (!args_ok(surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, H, W, mh_dist, last, features,
                 feature_stride, D) ||
        feature_map == nullptr)
        return GSR_ERR_BAD_ARG;
    const dim3 grid(((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE), 1, feature_stride / FCH);
    cudaStream_t st = (cudaStream_t)stream;
    const float r2 = mh_dist * mh_dist;
    if (rays != nullptr)
        k_surfel_features_fwd<true><<<grid, PIX, 0, st>>>(surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, H,
                                                          W, r2, rays, last, features, feature_stride, D, feature_map);
    else
        k_surfel_features_fwd<false><<<grid, PIX, 0, st>>>(surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, H,
                                                           W, r2, nullptr, last, features, feature_stride, D,
                                                           feature_map);
    return (int)cudaGetLastError();
}

int gsr_surfel_render_features_backward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                                        const int32_t* ids_sorted, const int32_t* tile_ranges, int H, int W,
                                        float mh_dist, const float* rays, const int32_t* last, const float* totals,
                                        const float* features, int feature_stride, int D,
                                        const float* grad_feature_map, float* grad_features, float* grad_rows,
                                        void* stream) {
    if (!args_ok(surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, H, W, mh_dist, last, features,
                 feature_stride, D))
        return GSR_ERR_BAD_ARG;
    if (totals == nullptr || grad_feature_map == nullptr || grad_features == nullptr || grad_rows == nullptr ||
        !aligned16(grad_features) || !aligned16(grad_rows))
        return GSR_ERR_BAD_ARG;
    const dim3 grid(((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE), 1, feature_stride / FCH);
    cudaStream_t st = (cudaStream_t)stream;
    const float r2 = mh_dist * mh_dist;
    if (rays != nullptr)
        k_surfel_features_bwd<true><<<grid, PIX, 0, st>>>(surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, H,
                                                          W, r2, rays, last, totals, features, feature_stride, D,
                                                          grad_feature_map, grad_features, grad_rows);
    else
        k_surfel_features_bwd<false><<<grid, PIX, 0, st>>>(surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, H,
                                                           W, r2, nullptr, last, totals, features, feature_stride, D,
                                                           grad_feature_map, grad_features, grad_rows);
    return (int)cudaGetLastError();
}

}  // extern "C"
