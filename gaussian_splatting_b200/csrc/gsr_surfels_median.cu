// gsr_surfels_median.cu — the median depth of the surfel blend (DESIGN.md 3.28), forward and backward
// (libgsr_surfels_median.so, C ABI include/gsr_surfels_median.h).
//
// Forward: the tile kernels' design of gsr_surfels.cuh, one CTA per 16x16 tile, one pixel per thread, batches of surfel
// records staged in shared memory with their gaussian ids.  intersect<RAYS> on the same records gives every (pixel,
// surfel) the colour forward's decision and z, and A is formed with the colour forward's rounded operations, so the
// median contributor is decided on the colour's floats.  A pixel stops at its first contributor with 1 - A <= 0.5 or at
// its `last`; the CTA leaves once no pixel is still walking.
//
// Backward: no walk.  One thread per pixel reads its median surfel's record, recomputes intersect<RAYS> (the pinned
// operations give the forward's hit and z) and chains d loss / d median through z into dM (9) or d p_z.  The warp's
// pixels with the same median surfel are summed in shared memory and one lane adds each non-zero sum.
#include "gsr_surfels.cuh"
#include "../../include/gsr_surfels_median.h"

namespace gsr {
namespace surfel {

constexpr int NMED = 10;  // row slots the median writes: dM (9), then d p_z

template <bool RAYS>
__global__ void __launch_bounds__(PIX)
    k_surfel_median_fwd(const float* __restrict__ surfels, const uint64_t* __restrict__ keys, int id_bits,
                        const int32_t* __restrict__ ids, const int32_t* __restrict__ ranges, int H, int W, float r2,
                        const float* __restrict__ rays, const int32_t* __restrict__ last, float* __restrict__ median,
                        int32_t* __restrict__ median_id) {
    __shared__ float4 s_rec[BATCH * 5];
    __shared__ int s_id[BATCH];
    const int ntx = (W + TILE - 1) / TILE;
    const int tile = blockIdx.x, tx = tile % ntx, ty = tile / ntx;
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
    float A = 0.f, med = 0.f;
    int mid = -1;
    bool walking = inside;
    for (int p0 = start; p0 < end; p0 += BATCH) {
        if (!__syncthreads_or(walking && lst >= p0)) break;
        const int n = min(BATCH, end - p0);
        stage_batch(s_rec, surfels, keys, id_bits, ids, p0, n);
        for (int k = threadIdx.x; k < n; k += PIX) s_id[k] = pair_id(keys, id_bits, ids, p0 + k);
        __syncthreads();
        const int m = walking ? min(n, lst - p0 + 1) : 0;  // up to the colour forward's last contributor
        for (int j = 0; j < m; ++j) {
            const float* r = reinterpret_cast<const float*>(s_rec + j * 5);
            Hit h;
            if (!intersect<RAYS>(r, x, y, d, r2, h)) continue;
            // 1 - A > 0.5 in front of this contributor (checked after the previous one): it is the median so far
            med = h.z;
            mid = s_id[j];
            // the colour forward's accumulated alpha, operation for operation
            A = __fadd_rn(A, __fmul_rn(h.alpha, __fsub_rn(1.0f, A)));
            if (!(__fsub_rn(1.0f, A) > 0.5f)) {
                walking = false;  // no later contributor has 1 - A > 0.5
                break;
            }
        }
    }
    if (!inside) return;
    median[pix] = med;
    median_id[pix] = mid;
}

template <bool RAYS>
__global__ void __launch_bounds__(PIX)
    k_surfel_median_bwd(const float* __restrict__ surfels, int H, int W, float r2, const float* __restrict__ rays,
                        const int32_t* __restrict__ median_id, const float* __restrict__ grad_median,
                        float* __restrict__ rows) {
    const int ntx = (W + TILE - 1) / TILE;
    const int tile = blockIdx.x, tx = tile % ntx, ty = tile / ntx;
    const int px = tx * TILE + (threadIdx.x & 15), py = ty * TILE + (threadIdx.x >> 4);
    const bool inside = px < W && py < H;
    const size_t pix = (size_t)py * W + px;
    const float x = (float)px, y = (float)py;
    int id = -1;
    float gz = 0.f;
    if (inside) {
        id = median_id[pix];
        gz = grad_median[pix];
    }
    float g[NMED];
#pragma unroll
    for (int k = 0; k < NMED; ++k) g[k] = 0.f;
    bool on = id >= 0 && gz != 0.0f;
    if (on) {
        float r[SF];
        const float4* rec = reinterpret_cast<const float4*>(surfels + (size_t)id * SF);
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const float4 q = rec[k];
            r[4 * k] = q.x; r[4 * k + 1] = q.y; r[4 * k + 2] = q.z; r[4 * k + 3] = q.w;
        }
        float d[3] = {0.f, 0.f, 0.f};
        if constexpr (RAYS) {
            d[0] = rays[pix * 3]; d[1] = rays[pix * 3 + 1]; d[2] = rays[pix * 3 + 2];
        }
        Hit h;
        on = intersect<RAYS>(r, x, y, d, r2, h);  // the forward's hit: always taken for a pixel's median surfel
        if (on) {
            if (h.use3) {
                // z = M2 . (a, b, 1): the colour backward's z chain with no rho gradient
                const float* M = r + S_M;
                const float ga = gz * M[6], gb = gz * M[7];
                g[6] = gz * h.a;
                g[7] = gz * h.b;
                g[8] = gz;
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
                    g[k] = -dz * ghx[k];
                    g[3 + k] = -dz * ghy[k];
                    g[6 + k] += dx * ghx[k] + dy * ghy[k];
                }
            } else {
                g[9] = gz;  // z = p_z where the low-pass filter decides
            }
        }
    }
    // the warp's lanes with the same median surfel: the lowest one sums their slots and adds the non-zero sums
    __shared__ float s_g[NMED][PIX];
    const int lane = threadIdx.x & 31;
    const unsigned peers = __match_any_sync(0xffffffffu, on ? id : -1);
#pragma unroll
    for (int k = 0; k < NMED; ++k) s_g[k][threadIdx.x] = g[k];
    __syncwarp();
    if (on && (peers & ((1u << lane) - 1u)) == 0u) {
        const int base = threadIdx.x - lane;
        float* dst = rows + (size_t)id * SG;
#pragma unroll
        for (int k = 0; k < NMED; ++k) {
            float s = 0.f;
            for (unsigned b = peers; b != 0u; b &= b - 1u) s += s_g[k][base + __ffs(b) - 1];
            if (s != 0.0f) atomicAdd(dst + (k < 9 ? G_M + k : G_PZ), s);
        }
    }
}

}  // namespace surfel
}  // namespace gsr

using namespace gsr;
using namespace gsr::surfel;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }

extern "C" {

int gsr_surfel_render_median_forward(const float* surfels, const uint64_t* keys_sorted, int id_bits,
                                     const int32_t* ids_sorted, const int32_t* tile_ranges, int H, int W,
                                     float mh_dist, const float* rays, const int32_t* last, float* median,
                                     int32_t* median_id, void* stream) {
    if ((keys_sorted == nullptr) == (ids_sorted == nullptr)) return GSR_ERR_BAD_ARG;  // exactly one id source
    if (keys_sorted != nullptr && (id_bits < 1 || id_bits > 32 || (reinterpret_cast<uintptr_t>(keys_sorted) & 7u)))
        return GSR_ERR_BAD_ARG;
    if (ids_sorted != nullptr && !aligned4(ids_sorted)) return GSR_ERR_BAD_ARG;
    if (surfels == nullptr || !aligned16(surfels) || tile_ranges == nullptr || !aligned4(tile_ranges) ||
        last == nullptr || !aligned4(last) || median == nullptr || !aligned4(median) || median_id == nullptr ||
        !aligned4(median_id) || (rays != nullptr && !aligned4(rays)))
        return GSR_ERR_BAD_ARG;
    if (H <= 0 || W <= 0 || !(mh_dist > 0.0f)) return GSR_ERR_BAD_ARG;
    const int tiles = ((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE);
    cudaStream_t st = (cudaStream_t)stream;
    const float r2 = mh_dist * mh_dist;
    if (rays != nullptr)
        k_surfel_median_fwd<true><<<tiles, PIX, 0, st>>>(surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, H, W,
                                                         r2, rays, last, median, median_id);
    else
        k_surfel_median_fwd<false><<<tiles, PIX, 0, st>>>(surfels, keys_sorted, id_bits, ids_sorted, tile_ranges, H,
                                                          W, r2, nullptr, last, median, median_id);
    return (int)cudaGetLastError();
}

int gsr_surfel_render_median_backward(const float* surfels, int H, int W, float mh_dist, const float* rays,
                                      const int32_t* median_id, const float* grad_median, float* grad_rows,
                                      void* stream) {
    if (surfels == nullptr || !aligned16(surfels) || median_id == nullptr || !aligned4(median_id) ||
        grad_median == nullptr || !aligned4(grad_median) || grad_rows == nullptr || !aligned16(grad_rows) ||
        (rays != nullptr && !aligned4(rays)))
        return GSR_ERR_BAD_ARG;
    if (H <= 0 || W <= 0 || !(mh_dist > 0.0f)) return GSR_ERR_BAD_ARG;
    const int tiles = ((W + TILE - 1) / TILE) * ((H + TILE - 1) / TILE);
    cudaStream_t st = (cudaStream_t)stream;
    const float r2 = mh_dist * mh_dist;
    if (rays != nullptr)
        k_surfel_median_bwd<true><<<tiles, PIX, 0, st>>>(surfels, H, W, r2, rays, median_id, grad_median, grad_rows);
    else
        k_surfel_median_bwd<false><<<tiles, PIX, 0, st>>>(surfels, H, W, r2, nullptr, median_id, grad_median,
                                                          grad_rows);
    return (int)cudaGetLastError();
}

}  // extern "C"
