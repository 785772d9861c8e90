// gsr_bilagrid.cu — bilateral-grid appearance correction: slice forward / backward and the grids' total variation.
//
// Contract: include/gsr_bilagrid.h.
//
// Slice (forward and the rgb gradient): one CTA per grid cell (cx, cy), chunk of SLICE_RB pixel rows and view.  The
// cell's 2 x 2 x L x 12 node values are staged in shared memory as [corner][coefficient][level], so for a given
// coefficient the lanes of a warp, whose levels differ, read distinct banks.  A CTA walks a slightly wider pixel
// window than its cell and keeps the pixels whose own (fp32) cell index is its cell, so every pixel is handled by
// exactly one CTA and the fp32 cell arithmetic alone decides which.  The backward recomputes a and da/dfz from the
// same loads instead of storing 48 B per pixel.
//
// Grid gradient, gathered: one CTA per (node (x, y), chunk of GRAD_RB pixel rows, view, block of SLICE_LB levels)
// walks its rows of the pixels of the up to 2 x 2 cells around its node.  Each thread keeps SLICE_LB x 12
// accumulators (the level weight is predicated, so there is no indexing by a runtime level), then the CTA reduces
// them in a fixed order (shuffle tree, then the warps in order) into a per-(view, chunk) buffer.  A last pass forms
// each view's value as the sum of its chunks in order and writes every grid element as 0 + the values of the views
// that use that grid, in view order.  No float atomics anywhere: results repeat bit for bit, and a view's values do
// not depend on the other views of the batch.
//
// TV: one grid-stride pass accumulates the three axes' sums of squares in fp64; each CTA writes its partial and the
// last CTA to finish (an atomic ticket) adds them in a fixed order and writes the result on the device.  The backward
// is one elementwise stencil.
#include <cmath>
#include <cstdint>

#include "gsr_common.cuh"
#include "../../include/gsr_bilagrid.h"

namespace gsr {

constexpr int SLICE_THREADS = 256;
constexpr int SLICE_RB = 8;          // pixel rows per slice CTA
constexpr int SLICE_MARGIN = 2;      // extra pixels walked on each side of a cell's nominal pixel window
constexpr int GRAD_THREADS = 128;
constexpr int GRAD_RB = 16;          // pixel rows per grid-gradient CTA
constexpr int SLICE_LB = 8;          // grid levels per grid-gradient CTA
constexpr int TV_THREADS = 256;
constexpr int TV_MAX_BLOCKS = 1024;

struct SliceGeom {
    int C, H, W, N, L, GY, GX;
    long long rs[4];  // rgb element strides (view, row, column, channel)
};

// pixel -> (cell, fraction) along one axis: f = (p + 0.5) / n (G - 1), cell = floor(f) kept inside [0, G - 2]
__device__ __forceinline__ void axis_cell(int p, int n, int G, int& c, float& t) {
    const float f = (p + 0.5f) / (float)n * (float)(G - 1);
    c = min(max((int)floorf(f), 0), G - 2);
    t = f - (float)c;
}

// nominal pixel window [lo, hi) of cell c along an axis of n pixels and G nodes, widened by SLICE_MARGIN
__device__ __forceinline__ void cell_window(int c, int n, int G, int& lo, int& hi) {
    const float s = (float)n / (float)(G - 1);
    lo = max(0, (int)floorf((float)c * s) - SLICE_MARGIN);
    hi = min(n, (int)ceilf((float)(c + 1) * s) + SLICE_MARGIN);
}

struct Guide {
    float lum, tz;
    int z0;
};

__device__ __forceinline__ Guide guide(float r, float g, float b, int L) {
    Guide q;
    q.lum = 0.299f * r + 0.587f * g + 0.114f * b;
    const float fz = fminf(fmaxf(q.lum, 0.f), 1.f) * (float)(L - 1);
    q.z0 = min((int)floorf(fz), L - 2);
    q.tz = fz - (float)q.z0;
    return q;
}

template <bool BWD>
__global__ void __launch_bounds__(SLICE_THREADS)
    k_bilagrid_slice(SliceGeom S, int n_chunks, const float* __restrict__ rgb, const float* __restrict__ grids,
                     const int32_t* __restrict__ ids, float* __restrict__ out, const float* __restrict__ grad_out,
                     long long gs0, long long gs1, long long gs2, long long gs3) {
    extern __shared__ float sg[];  // [4 corners][12][L]
    const int cx = blockIdx.x, cy = blockIdx.y / n_chunks, chunk = blockIdx.y % n_chunks, c = blockIdx.z;
    const int L = S.L, GY = S.GY, GX = S.GX;
    const int n = ids[c];
    if (n < 0 || n >= S.N) return;

    int i_lo, i_hi, j_lo, j_hi;
    cell_window(cy, S.H, GY, i_lo, i_hi);
    cell_window(cx, S.W, GX, j_lo, j_hi);
    i_lo += chunk * SLICE_RB;
    i_hi = min(i_hi, i_lo + SLICE_RB);
    if (i_lo >= i_hi) return;

    const long long plane = (long long)GY * GX;
    const float* g = grids + (long long)n * 12 * L * plane;
    for (int e = threadIdx.x; e < 4 * 12 * L; e += SLICE_THREADS) {
        const int l = e % L, k = (e / L) % 12, corner = e / (12 * L);
        sg[e] = g[(long long)(k * L + l) * plane + (cy + (corner >> 1)) * GX + cx + (corner & 1)];
    }
    __syncthreads();

    const int ncols = j_hi - j_lo, npix = (i_hi - i_lo) * ncols;
    const float lw = (float)(L - 1);
    for (int e = threadIdx.x; e < npix; e += SLICE_THREADS) {
        const int i = i_lo + e / ncols, j = j_lo + e % ncols;
        int pcx, pcy;
        float tx, ty;
        axis_cell(j, S.W, GX, pcx, tx);
        axis_cell(i, S.H, GY, pcy, ty);
        if (pcx != cx || pcy != cy) continue;
        const long long src = (long long)c * S.rs[0] + (long long)i * S.rs[1] + (long long)j * S.rs[2];
        const float v[3] = {rgb[src], rgb[src + S.rs[3]], rgb[src + 2 * S.rs[3]]};
        const Guide q = guide(v[0], v[1], v[2], L);
        const float w[4] = {(1.f - ty) * (1.f - tx), (1.f - ty) * tx, ty * (1.f - tx), ty * tx};
        float a[12], da[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) {
            float s = 0.f, d = 0.f;
#pragma unroll
            for (int corner = 0; corner < 4; ++corner) {
                const float g0 = sg[(corner * 12 + k) * L + q.z0], g1 = sg[(corner * 12 + k) * L + q.z0 + 1];
                s = fmaf(w[corner], fmaf(q.tz, g1 - g0, g0), s);
                if (BWD) d = fmaf(w[corner], g1 - g0, d);
            }
            a[k] = s;
            da[k] = d;
        }
        const long long dst = (((long long)c * S.H + i) * S.W + j) * 3;
        if (!BWD) {
#pragma unroll
            for (int r = 0; r < 3; ++r)
                out[dst + r] = fmaf(a[4 * r], v[0], fmaf(a[4 * r + 1], v[1], fmaf(a[4 * r + 2], v[2], a[4 * r + 3])));
        } else {
            const long long go = (long long)c * gs0 + (long long)i * gs1 + (long long)j * gs2;
            const float gr[3] = {grad_out[go], grad_out[go + gs3], grad_out[go + 2 * gs3]};
            float dfz = 0.f;
#pragma unroll
            for (int r = 0; r < 3; ++r)
                dfz = fmaf(gr[r], fmaf(da[4 * r], v[0], fmaf(da[4 * r + 1], v[1], fmaf(da[4 * r + 2], v[2],
                                                                                        da[4 * r + 3]))),
                           dfz);
            const bool inside = q.lum > 0.f && q.lum < 1.f;
            dfz = inside ? dfz * lw : 0.f;
            const float lc[3] = {0.299f, 0.587f, 0.114f};
#pragma unroll
            for (int ch = 0; ch < 3; ++ch)
                out[dst + ch] = fmaf(dfz, lc[ch], fmaf(a[ch], gr[0], fmaf(a[4 + ch], gr[1], a[8 + ch] * gr[2])));
        }
    }
}

// Deterministic CTA sum of NV floats per thread (butterfly within each warp, then the warps in order); the result
// for value v is left in red[(THREADS / 32) * NV + v] (valid after the trailing __syncthreads).
template <int NV, int THREADS>
__device__ __forceinline__ void block_sum_n(float (&acc)[NV], float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[v] += __shfl_xor_sync(0xffffffffu, acc[v], o);
    }
    if (lane == 0) {
#pragma unroll
        for (int v = 0; v < NV; ++v) red[warp * NV + v] = acc[v];
    }
    __syncthreads();
    for (int v = threadIdx.x; v < NV; v += THREADS) {
        float s = red[v];
        for (int q = 1; q < THREADS / 32; ++q) s += red[q * NV + v];
        red[(THREADS / 32) * NV + v] = s;
    }
    __syncthreads();
}

// per-(view, row chunk) grid gradient: part [C][n_chunks][12][L][GY][GX]
__global__ void __launch_bounds__(GRAD_THREADS)
    k_bilagrid_grid_grad(SliceGeom S, int n_chunks, int n_lblocks, const float* __restrict__ rgb, const int32_t* __restrict__ ids,
                         const float* __restrict__ grad_out, long long gs0, long long gs1, long long gs2,
                         long long gs3, float* __restrict__ part) {
    __shared__ float red[(GRAD_THREADS / 32 + 1) * SLICE_LB * 12];
    const int x = blockIdx.x, y = blockIdx.y / n_chunks, chunk = blockIdx.y % n_chunks, c = blockIdx.z / n_lblocks, l0 = (blockIdx.z % n_lblocks) * SLICE_LB;
    const int L = S.L, GY = S.GY, GX = S.GX;
    const int n = ids[c];
    if (n < 0 || n >= S.N) return;

    // pixels of the cells (x - 1 .. x) x (y - 1 .. y) inside the grid
    int i_lo, i_hi, j_lo, j_hi, t0, t1;
    cell_window(max(y - 1, 0), S.H, GY, i_lo, t0);
    cell_window(min(y, GY - 2), S.H, GY, t1, i_hi);
    cell_window(max(x - 1, 0), S.W, GX, j_lo, t0);
    cell_window(min(x, GX - 2), S.W, GX, t1, j_hi);
    i_lo += chunk * GRAD_RB;
    i_hi = min(i_hi, i_lo + GRAD_RB);

    float acc[SLICE_LB * 12];
#pragma unroll
    for (int v = 0; v < SLICE_LB * 12; ++v) acc[v] = 0.f;
    const int ncols = j_hi - j_lo, npix = max(i_hi - i_lo, 0) * ncols;
    for (int e = threadIdx.x; e < npix; e += GRAD_THREADS) {
        const int i = i_lo + e / ncols, j = j_lo + e % ncols;
        int pcx, pcy;
        float tx, ty;
        axis_cell(j, S.W, GX, pcx, tx);
        axis_cell(i, S.H, GY, pcy, ty);
        if ((pcx != x && pcx != x - 1) || (pcy != y && pcy != y - 1)) continue;
        const float wxy = (pcx == x ? 1.f - tx : tx) * (pcy == y ? 1.f - ty : ty);
        const long long src = (long long)c * S.rs[0] + (long long)i * S.rs[1] + (long long)j * S.rs[2];
        const float v[3] = {rgb[src], rgb[src + S.rs[3]], rgb[src + 2 * S.rs[3]]};
        const Guide q = guide(v[0], v[1], v[2], L);
        const long long go = (long long)c * gs0 + (long long)i * gs1 + (long long)j * gs2;
        const float gr[3] = {grad_out[go], grad_out[go + gs3], grad_out[go + 2 * gs3]};
        float gA[12];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            gA[4 * r] = gr[r] * v[0];
            gA[4 * r + 1] = gr[r] * v[1];
            gA[4 * r + 2] = gr[r] * v[2];
            gA[4 * r + 3] = gr[r];
        }
#pragma unroll
        for (int l = 0; l < SLICE_LB; ++l) {
            const int lv = l0 + l;
            const float wz = lv == q.z0 ? 1.f - q.tz : (lv == q.z0 + 1 ? q.tz : 0.f);
            const float w = wxy * wz;
#pragma unroll
            for (int k = 0; k < 12; ++k) acc[l * 12 + k] = fmaf(w, gA[k], acc[l * 12 + k]);
        }
    }

    block_sum_n<SLICE_LB * 12, GRAD_THREADS>(acc, red);
    const long long plane = (long long)GY * GX;
    for (int v = threadIdx.x; v < SLICE_LB * 12; v += GRAD_THREADS) {
        const int l = v / 12, k = v % 12, lv = l0 + l;
        if (lv < L)
            part[(((long long)c * n_chunks + chunk) * 12 * L + k * L + lv) * plane + y * GX + x] =
                red[(GRAD_THREADS / 32) * SLICE_LB * 12 + v];
    }
}

// grad_grids[n] = 0 + the values of the views whose id is n, in view order; a view's value is the sum of its row
// chunks in order
__global__ void __launch_bounds__(256)
    k_bilagrid_grid_grad_finish(long long per_grid, long long total, int C, int n_chunks,
                                const int32_t* __restrict__ ids, const float* __restrict__ part,
                                float* __restrict__ grad_grids) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int n = (int)(e / per_grid);
    const long long off = e - (long long)n * per_grid;
    float s = 0.f;
    for (int c = 0; c < C; ++c) {
        if (ids[c] != n) continue;
        const float* p = part + (long long)c * n_chunks * per_grid + off;
        float v = p[0];
        for (int q = 1; q < n_chunks; ++q) v += p[(long long)q * per_grid];
        s += v;
    }
    grad_grids[e] = s;
}

// ---- total variation --------------------------------------------------------------------------------------------------
__device__ __forceinline__ void block_sum3(double& a, double& b, double& c, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
        c += __shfl_xor_sync(0xffffffffu, c, o);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();  // red may still be read by a previous call
    if (lane == 0) {
        red[3 * warp] = a;
        red[3 * warp + 1] = b;
        red[3 * warp + 2] = c;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        a = red[0];
        b = red[1];
        c = red[2];
        for (int q = 1; q < TV_THREADS / 32; ++q) {
            a += red[3 * q];
            b += red[3 * q + 1];
            c += red[3 * q + 2];
        }
    }
}

__global__ void __launch_bounds__(TV_THREADS)
    k_bilagrid_tv_fwd(long long total, int L, int GY, int GX, const float* __restrict__ g, double* __restrict__ partials,
                      unsigned int* __restrict__ ticket, float* __restrict__ out, double inv_z, double inv_y,
                      double inv_x) {
    __shared__ double red[3 * TV_THREADS / 32];
    __shared__ bool is_last;
    const long long plane = (long long)GY * GX;
    double sz = 0.0, sy = 0.0, sx = 0.0;
    for (long long e = (long long)blockIdx.x * TV_THREADS + threadIdx.x; e < total;
         e += (long long)gridDim.x * TV_THREADS) {
        const int x = (int)(e % GX), y = (int)((e / GX) % GY), z = (int)((e / plane) % L);
        const float v = g[e];
        if (z < L - 1) {
            const float d = g[e + plane] - v;
            sz += (double)(d * d);
        }
        if (y < GY - 1) {
            const float d = g[e + GX] - v;
            sy += (double)(d * d);
        }
        if (x < GX - 1) {
            const float d = g[e + 1] - v;
            sx += (double)(d * d);
        }
    }
    block_sum3(sz, sy, sx, red);
    if (threadIdx.x == 0) {
        partials[3 * blockIdx.x] = sz;
        partials[3 * blockIdx.x + 1] = sy;
        partials[3 * blockIdx.x + 2] = sx;
        __threadfence();
        is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    sz = sy = sx = 0.0;
    for (unsigned int q = threadIdx.x; q < gridDim.x; q += TV_THREADS) {
        sz += __ldcg(partials + 3 * q);
        sy += __ldcg(partials + 3 * q + 1);
        sx += __ldcg(partials + 3 * q + 2);
    }
    block_sum3(sz, sy, sx, red);
    if (threadIdx.x == 0) {
        *out = (float)(sz * inv_z + sy * inv_y + sx * inv_x);
        *ticket = 0u;  // ready for the next launch on the same buffer
    }
}

__global__ void __launch_bounds__(TV_THREADS)
    k_bilagrid_tv_bwd(long long total, int L, int GY, int GX, const float* __restrict__ g,
                      const float* __restrict__ grad_tv, float* __restrict__ grad, float sz, float sy, float sx) {
    const long long e = (long long)blockIdx.x * TV_THREADS + threadIdx.x;
    if (e >= total) return;
    const long long plane = (long long)GY * GX;
    const int x = (int)(e % GX), y = (int)((e / GX) % GY), z = (int)((e / plane) % L);
    const float v = g[e];
    float dz = 0.f, dy = 0.f, dx = 0.f;  // d/dv of the axis's sum of squares, halved
    if (z > 0) dz += v - g[e - plane];
    if (z < L - 1) dz -= g[e + plane] - v;
    if (y > 0) dy += v - g[e - GX];
    if (y < GY - 1) dy -= g[e + GX] - v;
    if (x > 0) dx += v - g[e - 1];
    if (x < GX - 1) dx -= g[e + 1] - v;
    grad[e] = *grad_tv * fmaf(sz, dz, fmaf(sy, dy, sx * dx));
}

static bool grid_ok(int N, int L, int GY, int GX) {
    return N >= 1 && L >= 2 && GY >= 2 && GX >= 2 && L <= GSR_BILAGRID_MAX_L && GY <= 65535 && GX <= 65535 &&
           (long long)N * 12 * L * GY * GX < (1LL << 40);
}

static bool slice_ok(int C, int H, int W, int N, int L, int GY, int GX) {
    return grid_ok(N, L, GY, GX) && C >= 1 && C <= 65535 && H >= 1 && W >= 1 && H <= (1 << 20) && W <= (1 << 20);
}

// row chunks of a cell's pixel window (slice) and of a node's two cells (grid gradient): the window of cell c spans
// at most ceil(H / (GY - 1)) + 2 + 2 SLICE_MARGIN rows
static int cell_rows(int H, int GY) { return (H + GY - 2) / (GY - 1) + 2 + 2 * SLICE_MARGIN; }
static int slice_chunks(int H, int GY) { return (cell_rows(H, GY) + SLICE_RB - 1) / SLICE_RB; }
static int grad_chunks(int H, int GY) { return (2 * cell_rows(H, GY) + GRAD_RB - 1) / GRAD_RB; }

static SliceGeom slice_geom(int C, int H, int W, int N, int L, int GY, int GX, const int64_t* rs) {
    SliceGeom S;
    S.C = C;
    S.H = H;
    S.W = W;
    S.N = N;
    S.L = L;
    S.GY = GY;
    S.GX = GX;
    for (int k = 0; k < 4; ++k) S.rs[k] = rs[k];
    return S;
}

template <bool BWD>
static int launch_slice(const SliceGeom& S, const float* rgb, const float* grids, const int32_t* ids, float* out,
                        const float* grad_out, const int64_t* gs, cudaStream_t stream) {
    const int chunks = slice_chunks(S.H, S.GY);
    if ((long long)chunks * (S.GY - 1) > 65535) return GSR_ERR_BAD_ARG;
    const size_t smem = sizeof(float) * 4 * 12 * S.L;
    const dim3 grid((unsigned)(S.GX - 1), (unsigned)((S.GY - 1) * chunks), (unsigned)S.C);
    k_bilagrid_slice<BWD><<<grid, SLICE_THREADS, smem, stream>>>(S, chunks, rgb, grids, ids, out, grad_out,
                                                                 gs ? gs[0] : 0, gs ? gs[1] : 0, gs ? gs[2] : 0,
                                                                 gs ? gs[3] : 0);
    return (int)cudaGetLastError();
}

static bool tv_grid_ok(int N, int L, int GY, int GX) { return grid_ok(N, L, GY, GX); }

static unsigned int tv_blocks(long long total) {
    return (unsigned int)std::min<long long>(TV_MAX_BLOCKS, (total + 4 * TV_THREADS - 1) / (4 * TV_THREADS));
}

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_bilagrid_slice_forward(int C, int H, int W, const float* rgb, const int64_t* rgb_strides_host,
                               const float* grids, int N, int L, int GY, int GX, const int32_t* ids, float* out,
                               void* stream) {
    if (!slice_ok(C, H, W, N, L, GY, GX) || !rgb || !rgb_strides_host || !grids || !ids || !out) return GSR_ERR_BAD_ARG;
    return launch_slice<false>(slice_geom(C, H, W, N, L, GY, GX, rgb_strides_host), rgb, grids, ids, out, nullptr,
                               nullptr, (cudaStream_t)stream);
}

size_t gsr_bilagrid_slice_backward_temp_bytes(int C, int H, int L, int GY, int GX) {
    if (C < 1 || H < 1 || L < 2 || GY < 2 || GX < 2) return 0;
    return sizeof(float) * (size_t)C * grad_chunks(H, GY) * 12 * L * GY * GX;
}

int gsr_bilagrid_slice_backward(int C, int H, int W, const float* rgb, const int64_t* rgb_strides_host,
                                const float* grids, int N, int L, int GY, int GX, const int32_t* ids,
                                const float* grad_out, const int64_t* grad_out_strides_host, float* grad_rgb,
                                float* grad_grids, void* temp, size_t temp_bytes, void* stream) {
    if (!slice_ok(C, H, W, N, L, GY, GX) || !rgb || !rgb_strides_host || !grids || !ids || !grad_out ||
        !grad_out_strides_host)
        return GSR_ERR_BAD_ARG;
    if (grad_grids && (!temp || temp_bytes < gsr_bilagrid_slice_backward_temp_bytes(C, H, L, GY, GX)))
        return GSR_ERR_BAD_ARG;
    const SliceGeom S = slice_geom(C, H, W, N, L, GY, GX, rgb_strides_host);
    const int64_t* gs = grad_out_strides_host;
    cudaStream_t st = (cudaStream_t)stream;
    if (grad_rgb) {
        const int rc = launch_slice<true>(S, rgb, grids, ids, grad_rgb, grad_out, gs, st);
        if (rc != 0) return rc;
    }
    if (grad_grids) {
        const int lblocks = (L + SLICE_LB - 1) / SLICE_LB, chunks = grad_chunks(H, GY);
        if ((long long)C * lblocks > 65535 || (long long)GY * chunks > 65535) return GSR_ERR_BAD_ARG;
        float* part = static_cast<float*>(temp);
        k_bilagrid_grid_grad<<<dim3((unsigned)GX, (unsigned)(GY * chunks), (unsigned)(C * lblocks)), GRAD_THREADS, 0,
                               st>>>(S, chunks, lblocks, rgb, ids, grad_out, gs[0], gs[1], gs[2], gs[3], part);
        const long long per = 12LL * L * GY * GX, total = per * N;
        k_bilagrid_grid_grad_finish<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(per, total, C, chunks, ids, part,
                                                                                    grad_grids);
        const int rc = (int)cudaGetLastError();
        if (rc != 0) return rc;
    }
    return GSR_OK;
}

size_t gsr_bilagrid_tv_temp_bytes(int N, int L, int GY, int GX) {
    if (!tv_grid_ok(N, L, GY, GX)) return 16;
    return 16 + 3 * sizeof(double) * tv_blocks(12LL * N * L * GY * GX);
}

int gsr_bilagrid_tv_forward(int N, int L, int GY, int GX, const float* grids, float* out, void* temp,
                            size_t temp_bytes, void* stream) {
    if (!tv_grid_ok(N, L, GY, GX) || !grids || !out || !temp) return GSR_ERR_BAD_ARG;
    if (temp_bytes < gsr_bilagrid_tv_temp_bytes(N, L, GY, GX)) return GSR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned int* ticket = static_cast<unsigned int*>(temp);
    double* partials = reinterpret_cast<double*>(static_cast<unsigned char*>(temp) + 16);
    cudaError_t e = cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st);
    if (e != cudaSuccess) return (int)e;
    const long long M = 12LL * N, total = M * L * GY * GX;
    const double cz = (double)M * (L - 1) * GY * GX, cy = (double)M * L * (GY - 1) * GX,
                 cx = (double)M * L * GY * (GX - 1);
    k_bilagrid_tv_fwd<<<tv_blocks(total), TV_THREADS, 0, st>>>(total, L, GY, GX, grids, partials, ticket, out,
                                                               1.0 / cz, 1.0 / cy, 1.0 / cx);
    return (int)cudaGetLastError();
}

int gsr_bilagrid_tv_backward(int N, int L, int GY, int GX, const float* grids, const float* grad_tv,
                             float* grad_grids, void* stream) {
    if (!tv_grid_ok(N, L, GY, GX) || !grids || !grad_tv || !grad_grids) return GSR_ERR_BAD_ARG;
    const long long M = 12LL * N, total = M * L * GY * GX;
    const double cz = (double)M * (L - 1) * GY * GX, cy = (double)M * L * (GY - 1) * GX,
                 cx = (double)M * L * GY * (GX - 1);
    k_bilagrid_tv_bwd<<<(unsigned)((total + TV_THREADS - 1) / TV_THREADS), TV_THREADS, 0, (cudaStream_t)stream>>>(
        total, L, GY, GX, grids, grad_tv, grad_grids, (float)(2.0 / cz), (float)(2.0 / cy), (float)(2.0 / cx));
    return (int)cudaGetLastError();
}

}  // extern "C"
