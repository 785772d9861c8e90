// gsr_render_generic.cu — tile renderers for every (dtype, n_sh) the reference instantiates
// that is NOT the fp32 / precomputed-RGB training path: fp64 (the reference's gradcheck
// surface) and per-pixel spherical harmonics (use_sh_precompute=False), plus the depth
// renderer.  Same values as src/render.cu:101-188, src/render_backward.cu:120-284 and
// src/depth.cu:7-115; no staging tricks — each thread walks its tile's splat list through L1.
// Not on the measured path (SURVEY.md §8(f) rows 3-4).
#include "gsr_common.cuh"
#include "gsr_math.cuh"

namespace gsr {

template <typename T> struct IsF32 { static constexpr bool v = false; };
template <> struct IsF32<float> { static constexpr bool v = true; };

// CHUNK_SIZE table of the reference (src/render.cu:267-333, src/render_backward.cu:402-568);
// only its effect on the backward weight recurrence matters (SURVEY.md Q9)
template <typename T, int N_SH> struct RefChunk;
template <> struct RefChunk<float, 1> { static constexpr int v = 960; };
template <> struct RefChunk<float, 4> { static constexpr int v = 576; };
template <> struct RefChunk<float, 9> { static constexpr int v = 320; };
template <> struct RefChunk<float, 16> { static constexpr int v = 160; };
template <> struct RefChunk<double, 1> { static constexpr int v = 320; };
template <> struct RefChunk<double, 4> { static constexpr int v = 160; };
template <> struct RefChunk<double, 9> { static constexpr int v = 128; };
template <> struct RefChunk<double, 16> { static constexpr int v = 64; };

template <typename T> __device__ __forceinline__ T fast_or_exact_exp(T x);
template <> __device__ __forceinline__ float fast_or_exact_exp<float>(float x) { return __expf(x); }
template <> __device__ __forceinline__ double fast_or_exact_exp<double>(double x) { return exp(x); }

template <typename T, int N_SH>
__device__ __forceinline__ void pixel_basis(const T* __restrict__ view_dirs, int pix, T* __restrict__ Y) {
    if (N_SH == 1) {
        Y[0] = T(GSR_SH0);
    } else {
        sh_basis<T, N_SH>(view_dirs[pix * 3 + 0], view_dirs[pix * 3 + 1], view_dirs[pix * 3 + 2], Y);
    }
}

template <typename T, int N_SH>
__global__ void __launch_bounds__(TILE_PIXELS)
    k_render_fwd_generic(const T* __restrict__ uvs, const T* __restrict__ opacity, const T* __restrict__ rgb,
                         const T* __restrict__ conic, const T* __restrict__ view_dirs,
                         const int32_t* __restrict__ ranges, const int32_t* __restrict__ idx,
                         const T* __restrict__ background, int W, int H, int32_t* __restrict__ n_out,
                         T* __restrict__ w_out, T* __restrict__ image) {
    constexpr bool FAST = IsF32<T>::v;
    const int px = blockIdx.x * TILE + (threadIdx.x & 15);
    const int py = blockIdx.y * TILE + (threadIdx.x >> 4);
    if (px >= W || py >= H) return;
    const int tile = blockIdx.x + blockIdx.y * gridDim.x;
    const int start = ranges[tile], end = ranges[tile + 1];
    const int pix = py * W + px;
    T Y[N_SH];
    pixel_basis<T, N_SH>(view_dirs, pix, Y);
    T A = 0.0, wlast = 0.0, C[3] = {0.0, 0.0, 0.0};
    int n = 0;
    for (int p = start; p < end; ++p) {
        if (A > 0.9999) break;
        const int g = idx[p];
        const T du = T(px) - uvs[g * 2 + 0];
        const T dv = T(py) - uvs[g * 2 + 1];
        const T b = conic[g * 3 + 1] * 0.5;
        T a = conic[g * 3 + 0], c = conic[g * 3 + 2];
        if (FAST) {
            a = a + 0.25;
            c = c + 0.25;
        }
        const T det = a * c - b * b;
        T alpha = 0.0;
        const T mh = (c * du * du - (b + b) * du * dv + a * dv * dv) / det;
        if (mh > 0.0) alpha = opacity[g] * fast_or_exact_exp<T>(-0.5 * mh);
        if (FAST && alpha < 0.00392156862) {
            ++n;
            continue;
        }
        wlast = 1.0 - A;
        const T w = alpha * (1.0 - A);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            T col = Y[0] * rgb[(size_t)(g * 3 + ch) * N_SH];
#pragma unroll
            for (int k = 1; k < N_SH; ++k) col += Y[k] * rgb[(size_t)(g * 3 + ch) * N_SH + k];
            C[ch] += col * w;
        }
        A += w;
        ++n;
    }
    if (A < 0.999) {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) C[ch] += background[ch] * (1.0 - A);
    }
    n_out[pix] = n;
    w_out[pix] = wlast;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) image[pix * 3 + ch] = C[ch];
}

template <typename T>
__device__ __forceinline__ T warp_sum_t(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <typename T, int N_SH>
__global__ void __launch_bounds__(TILE_PIXELS)
    k_render_bwd_generic(const T* __restrict__ uvs, const T* __restrict__ opacity, const T* __restrict__ rgb,
                         const T* __restrict__ conic, const T* __restrict__ view_dirs,
                         const int32_t* __restrict__ ranges, const int32_t* __restrict__ idx,
                         const T* __restrict__ background, int W, int H, const int32_t* __restrict__ n_in,
                         const T* __restrict__ w_in, const T* __restrict__ grad_image, T* __restrict__ g_rgb,
                         T* __restrict__ g_opa, T* __restrict__ g_uv, T* __restrict__ g_conic) {
    constexpr bool FAST = IsF32<T>::v;
    constexpr int CHUNK = RefChunk<T, N_SH>::v;
    const int px = blockIdx.x * TILE + (threadIdx.x & 15);
    const int py = blockIdx.y * TILE + (threadIdx.x >> 4);
    const bool valid = (px < W) && (py < H);
    const int lane = threadIdx.x & 31;
    const int tile = blockIdx.x + blockIdx.y * gridDim.x;
    const int start = ranges[tile], end = ranges[tile + 1];
    const int pix = valid ? py * W + px : 0;
    T Y[N_SH];
    int n = 0;
    T weight = 0.0, dC[3] = {0.0, 0.0, 0.0}, acc[3] = {0.0, 0.0, 0.0};
    if (valid) {
        pixel_basis<T, N_SH>(view_dirs, pix, Y);
        n = n_in[pix];
        weight = w_in[pix];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) dC[ch] = grad_image[pix * 3 + ch];
    } else {
#pragma unroll
        for (int k = 0; k < N_SH; ++k) Y[k] = 0.0;
    }
    bool bg_init = false;
    for (int p = end - 1; p >= start; --p) {
        const int t_idx = p - start;
        const int g = idx[p];
        T gsh[3 * N_SH];
#pragma unroll
        for (int k = 0; k < 3 * N_SH; ++k) gsh[k] = 0.0;
        T go = 0.0, gu = 0.0, gv = 0.0, gc[3] = {0.0, 0.0, 0.0};
        bool contrib = false;
        if (valid && t_idx < n) {
            const T du = T(px) - uvs[g * 2 + 0];
            const T dv = T(py) - uvs[g * 2 + 1];
            const T b = conic[g * 3 + 1] * 0.5;
            T a = conic[g * 3 + 0], c = conic[g * 3 + 2];
            if (FAST) {
                a = a + 0.25;
                c = c + 0.25;
            }
            const T det = a * c - b * b;
            const T rdet = 1.0 / det;
            const T mh = (c * du * du - (b + b) * du * dv + a * dv * dv) * rdet;
            T prob = 0.0;
            if (mh > 0.0) prob = fast_or_exact_exp<T>(-0.5 * mh);
            const T opa = opacity[g];
            const T alpha = min(0.9999, opa * prob);
            if (alpha >= 0.00392156862 || !FAST) {
                contrib = true;
                if (!bg_init) {
                    const T bw = 1.0 - (alpha * weight + 1.0 - weight);
                    if (bw > 0.001) {
#pragma unroll
                        for (int ch = 0; ch < 3; ++ch) acc[ch] += background[ch] * bw;
                    }
                    bg_init = true;
                }
                const T r = 1.0 / (1.0 - alpha);
                if ((t_idx % CHUNK) < n - 1) weight = weight * r;
                T col[3], galpha = 0.0;
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    T cc = Y[0] * rgb[(size_t)(g * 3 + ch) * N_SH];
#pragma unroll
                    for (int k = 1; k < N_SH; ++k) cc += Y[k] * rgb[(size_t)(g * 3 + ch) * N_SH + k];
                    col[ch] = cc;
                    const T grgb = alpha * weight * dC[ch];
#pragma unroll
                    for (int k = 0; k < N_SH; ++k) gsh[ch * N_SH + k] = Y[k] * grgb;
                    galpha += (cc * weight - acc[ch] * r) * dC[ch];
                }
                go = prob * galpha;
                const T gprob = opa * galpha;
                const T gmh = -0.5 * prob * gprob;
                gu = -(-b * dv - b * dv + 2 * c * du) * rdet * gmh;
                gv = -(2 * a * dv - b * du - b * du) * rdet * gmh;
                const T cf = (a * dv * dv - b * du * dv - b * du * dv + c * du * du) * rdet * rdet;
                gc[0] = (-c * cf + dv * dv * rdet) * gmh;
                gc[1] = (b * cf - du * dv * rdet) * gmh;
                gc[2] = (-a * cf + du * du * rdet) * gmh;
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) acc[ch] += col[ch] * alpha * weight;
            }
        }
        if (__ballot_sync(0xffffffffu, contrib) == 0u) continue;
#pragma unroll
        for (int k = 0; k < 3 * N_SH; ++k) {
            const T v = warp_sum_t<T>(gsh[k]);
            if (lane == 0) atomicAdd(g_rgb + (size_t)g * 3 * N_SH + k, v);
        }
        go = warp_sum_t<T>(go);
        gu = warp_sum_t<T>(gu);
        gv = warp_sum_t<T>(gv);
#pragma unroll
        for (int k = 0; k < 3; ++k) gc[k] = warp_sum_t<T>(gc[k]);
        if (lane == 0) {
            atomicAdd(g_opa + g, go);
            atomicAdd(g_uv + g * 2 + 0, gu);
            atomicAdd(g_uv + g * 2 + 1, gv);
#pragma unroll
            for (int k = 0; k < 3; ++k) atomicAdd(g_conic + g * 3 + k, gc[k]);
        }
    }
}

// range to the first splat at which accumulated alpha exceeds the threshold.  Reference: src/depth.cu:57-113
__global__ void __launch_bounds__(TILE_PIXELS)
    k_render_depth(const float* __restrict__ xyz_cam, const float* __restrict__ uvs,
                   const float* __restrict__ opacity, const float* __restrict__ conic,
                   const int32_t* __restrict__ ranges, const int32_t* __restrict__ idx, float alpha_threshold,
                   int W, int H, float* __restrict__ depth) {
    const int px = blockIdx.x * TILE + (threadIdx.x & 15);
    const int py = blockIdx.y * TILE + (threadIdx.x >> 4);
    if (px >= W || py >= H) return;
    const int tile = blockIdx.x + blockIdx.y * gridDim.x;
    const int start = ranges[tile], end = ranges[tile + 1];
    float A = 0.0f;
    bool found = false;
    float out = 0.0f;
    for (int p = start; p < end && !found; ++p) {
        const int g = idx[p];
        const float du = float(px) - uvs[g * 2 + 0];
        const float dv = float(py) - uvs[g * 2 + 1];
        const float a = conic[g * 3 + 0] + 0.25f;
        const float b = conic[g * 3 + 1] / 2.0f;
        const float c = conic[g * 3 + 2] + 0.25f;
        const float det = a * c - b * b;
        const float mh = (c * du * du - (b + b) * du * dv + a * dv * dv) / det;
        float alpha = 0.0f;
        if (mh > 0.0f) alpha = opacity[g] * __expf(-0.5f * mh);
        // the reference forms the weight in double (its `1.0` literal) and rounds it once; an fp32 FMA differs
        const float w = (float)((1.0 - (double)A) * (double)alpha);
        A += w;
        if (A > alpha_threshold) {
            const float x = xyz_cam[g * 3 + 0], y = xyz_cam[g * 3 + 1], z = xyz_cam[g * 3 + 2];
            out = sqrtf(x * x + y * y + z * z);  // range, not z (src/depth.cu:102-105)
            found = true;
        }
    }
    if (found) depth[py * W + px] = out;
}

}  // namespace gsr

using namespace gsr;

#define GSR_RG_LAUNCH(KERNEL, T, NS, ...)                                                   \
    KERNEL<T, NS><<<grid, block, 0, (cudaStream_t)stream>>>(__VA_ARGS__)
#define GSR_RG_CASES(KERNEL, T, ...)                                                        \
    switch (n_sh) {                                                                         \
        case 1: GSR_RG_LAUNCH(KERNEL, T, 1, __VA_ARGS__); break;                            \
        case 4: GSR_RG_LAUNCH(KERNEL, T, 4, __VA_ARGS__); break;                            \
        case 9: GSR_RG_LAUNCH(KERNEL, T, 9, __VA_ARGS__); break;                            \
        case 16: GSR_RG_LAUNCH(KERNEL, T, 16, __VA_ARGS__); break;                          \
        default: return GSR_ERR_UNSUPPORTED;                                                \
    }

extern "C" {

int gsr_render_forward_generic(int dtype, int N, int n_sh, const void* uvs, const void* opacity,
                               const void* rgb, const void* conic, const void* view_dirs,
                               const int32_t* ranges, const int32_t* idx, const void* background, int H,
                               int W, int32_t* n_out, void* w_out, void* image, void* stream) {
    (void)N;
    if (H <= 0 || W <= 0) return GSR_ERR_BAD_ARG;
    const dim3 grid((W + TILE - 1) / TILE, (H + TILE - 1) / TILE), block(TILE_PIXELS);
    if (dtype == GSR_F32) {
        GSR_RG_CASES(k_render_fwd_generic, float, (const float*)uvs, (const float*)opacity, (const float*)rgb,
                     (const float*)conic, (const float*)view_dirs, ranges, idx, (const float*)background, W, H,
                     n_out, (float*)w_out, (float*)image)
    } else if (dtype == GSR_F64) {
        GSR_RG_CASES(k_render_fwd_generic, double, (const double*)uvs, (const double*)opacity,
                     (const double*)rgb, (const double*)conic, (const double*)view_dirs, ranges, idx,
                     (const double*)background, W, H, n_out, (double*)w_out, (double*)image)
    } else {
        return GSR_ERR_BAD_ARG;
    }
    return (int)cudaGetLastError();
}

int gsr_render_backward_generic(int dtype, int N, int n_sh, const void* uvs, const void* opacity,
                                const void* rgb, const void* conic, const void* view_dirs,
                                const int32_t* ranges, const int32_t* idx, const void* background, int H,
                                int W, const int32_t* n_in, const void* w_in, const void* grad_image,
                                void* g_rgb, void* g_opa, void* g_uv, void* g_conic, void* stream) {
    (void)N;
    if (H <= 0 || W <= 0) return GSR_ERR_BAD_ARG;
    const dim3 grid((W + TILE - 1) / TILE, (H + TILE - 1) / TILE), block(TILE_PIXELS);
    if (dtype == GSR_F32) {
        GSR_RG_CASES(k_render_bwd_generic, float, (const float*)uvs, (const float*)opacity, (const float*)rgb,
                     (const float*)conic, (const float*)view_dirs, ranges, idx, (const float*)background, W, H,
                     n_in, (const float*)w_in, (const float*)grad_image, (float*)g_rgb, (float*)g_opa,
                     (float*)g_uv, (float*)g_conic)
    } else if (dtype == GSR_F64) {
        GSR_RG_CASES(k_render_bwd_generic, double, (const double*)uvs, (const double*)opacity,
                     (const double*)rgb, (const double*)conic, (const double*)view_dirs, ranges, idx,
                     (const double*)background, W, H, n_in, (const double*)w_in, (const double*)grad_image,
                     (double*)g_rgb, (double*)g_opa, (double*)g_uv, (double*)g_conic)
    } else {
        return GSR_ERR_BAD_ARG;
    }
    return (int)cudaGetLastError();
}

int gsr_render_depth(int N, const float* xyz_cam, const float* uvs, const float* opacity, const float* conic,
                     const int32_t* ranges, const int32_t* idx, float alpha_threshold, int H, int W,
                     float* depth, void* stream) {
    (void)N;
    if (H <= 0 || W <= 0) return GSR_ERR_BAD_ARG;
    const dim3 grid((W + TILE - 1) / TILE, (H + TILE - 1) / TILE), block(TILE_PIXELS);
    k_render_depth<<<grid, block, 0, (cudaStream_t)stream>>>(xyz_cam, uvs, opacity, conic, ranges, idx,
                                                             alpha_threshold, W, H, depth);
    return (int)cudaGetLastError();
}

}  // extern "C"
