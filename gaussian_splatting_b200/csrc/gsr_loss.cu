// gsr_loss.cu — the training step's photometric loss, (1 - ssim_frac) * L1 + ssim_frac * (1 - SSIM), as two kernels.
//
// Contract (values): the SSIM of tools/e2e/shims/torchmetrics/image.py, which every training arm of tools/e2e uses
// for the reference trainer's loss (splat_py/trainer.py:363-374):
//   - 11-tap Gaussian window, sigma 1.5, formed in fp32 by the caller and passed in (window_host), applied
//     separably;
//   - moments mu_p, mu_t, E[p^2], E[t^2], E[pt] over every window lying fully inside the image: (H-10) x (W-10)
//     window origins per channel;
//   - S = (2 mu_p mu_t + C1)(2 s_pt + C2) / ((mu_p^2 + mu_t^2 + C1)(s_pp + s_tt + C2)), no clamping;
//     SSIM = mean of S over B*C*(H-10)*(W-10);
//   - L1 = mean |p - t| over all B*C*H*W elements, gradient sign(p - t) / numel with sign(0) = 0.
// loss = l1_weight * L1 + ssim_weight * (1 - SSIM).  Gradients flow to pred only.
//
// Forward: one CTA per 32x16 tile of window origins / pixels, all channels (staged LOSS_CG at a time).  The tile
// plus its 10-pixel halo to the right and below is staged in shared memory for pred and target, the five moments are
// blurred horizontally then vertically, S is summed over the CTA's valid origins and |p - t| over the CTA's own
// pixels (each pixel counts once).  Each CTA writes an fp64 (sum S, sum |p - t|) pair; the last CTA to finish (an
// atomic ticket) adds the pairs up in a fixed order and writes out[3] = {loss, L1, SSIM} on the device.  No host
// sync, no atomics on the result: bit-identical from run to run.
//
// Backward: recomputes instead of storing intermediate maps (an evaluation under no_grad pays for the forward
// only).  A 32x16 pixel tile needs dS/dmu_p, dS/dE[p^2], dS/dE[pt] at the window origins y in [x-10, x] (zero at
// origins outside the valid range), which need the images over [x-10, x+10]: that 52x36 region is staged, the
// moments and the three derivative maps are formed over the 42x26 origins, and the maps are blurred with the
// flipped window (separably) back onto the pixels:
//     grad(x) = g_out * (l1_weight / numel * sign(p - t) - ssim_weight / n_valid * (D_mu + 2 p D_pp + t D_pt)).
//
// Layouts: every image is a base pointer plus four element strides (B, C, H, W), so the rasterizer's [H,W,3] image,
// the trainer's image.unsqueeze(0).permute(0,3,1,2) view of it and a contiguous NCHW tensor go through the same code
// without a copy.  The strides only decide which thread loads / stores which element (loads and stores run along
// the smallest of the channel and column strides, so they are coalesced for HWC and for NCHW); every arithmetic
// operation reads shared memory in a fixed order, so all layouts give bit-identical values.
#include <cmath>
#include <cstdint>

#include "gsr_common.cuh"

namespace gsr {

constexpr int SSIM_TAPS = 11;
constexpr int SSIM_HALO = SSIM_TAPS - 1;
constexpr int LOSS_CG = 3;         // channels staged in shared memory per pass
constexpr int LOSS_TW = 32;        // tile width (pixels / window origins)
constexpr int LOSS_TH = 16;        // tile height
constexpr int LOSS_THREADS = 256;

template <typename T>
struct LossArgs {
    const T* pred;
    const T* target;
    long long ps[4], ts[4];  // element strides (B, C, H, W)
    int B, C, H, W;
    T w[SSIM_TAPS];
    T c1, c2;
};

// forward shared memory: pred + target [CG][TH+10][TW+10], horizontal moments [5][TH+10][TW]
constexpr int FWD_IH = LOSS_TH + SSIM_HALO, FWD_IW = LOSS_TW + SSIM_HALO;
template <typename T>
constexpr size_t fwd_smem_bytes() {
    return sizeof(T) * (2 * LOSS_CG * FWD_IH * FWD_IW + 5 * FWD_IH * LOSS_TW);
}
// backward shared memory: pred + target [CG][TH+20][TW+20], horizontal moments [5][TH+20][TW+10] (reused for the
// transposed horizontal pass [3][TH+10][TW]), derivative maps [3][TH+10][TW+10], gradient [CG][TH][TW]
constexpr int BWD_RH = LOSS_TH + 2 * SSIM_HALO, BWD_RW = LOSS_TW + 2 * SSIM_HALO;
constexpr int BWD_OH = LOSS_TH + SSIM_HALO, BWD_OW = LOSS_TW + SSIM_HALO;
template <typename T>
constexpr size_t bwd_smem_bytes() {
    return sizeof(T) * (2 * LOSS_CG * BWD_RH * BWD_RW + 5 * BWD_RH * BWD_OW + 3 * BWD_OH * BWD_OW +
                        LOSS_CG * LOSS_TH * LOSS_TW);
}

// Stage channels [c0, c0 + cg) of image b, rows [y0, y0 + nr), cols [x0, x0 + nc) into s[c][r][col]; zero outside
// the image.  The element each thread takes follows the smaller of the channel / column strides (coalescing only).
template <typename T>
__device__ __forceinline__ void stage_region(T* __restrict__ s, const T* __restrict__ src, const long long* st, int b,
                                             int c0, int cg, int y0, int x0, int nr, int nc, int H, int W) {
    const bool interleaved = st[1] < st[3];
    const long long base = (long long)b * st[0] + (long long)c0 * st[1];
    const int n = cg * nr * nc;
    for (int e = threadIdx.x; e < n; e += LOSS_THREADS) {
        int c, r, col;
        if (interleaved) {
            c = e % cg;
            const int rc = e / cg;
            col = rc % nc;
            r = rc / nc;
        } else {
            col = e % nc;
            const int rc = e / nc;
            r = rc % nr;
            c = rc / nr;
        }
        const int y = y0 + r, x = x0 + col;
        T v = T(0);
        if (y >= 0 && y < H && x >= 0 && x < W) v = src[base + c * st[1] + y * st[2] + x * st[3]];
        s[(c * nr + r) * nc + col] = v;
    }
}

// Five horizontal window sums of row r starting at column u: p, t, p^2, t^2, pt.
template <typename T>
__device__ __forceinline__ void hsum5(const T* __restrict__ p, const T* __restrict__ t, int off, const T* w, T& m0,
                                      T& m1, T& m2, T& m3, T& m4) {
    m0 = m1 = m2 = m3 = m4 = T(0);
#pragma unroll
    for (int k = 0; k < SSIM_TAPS; ++k) {
        const T a = p[off + k], c = t[off + k];
        m0 = fma(w[k], a, m0);
        m1 = fma(w[k], c, m1);
        m2 = fma(w[k], a * a, m2);
        m3 = fma(w[k], c * c, m3);
        m4 = fma(w[k], a * c, m4);
    }
}

// Vertical window sums of the five horizontal-moment planes (plane stride ps, row stride rs) at (row r, col j).
template <typename T>
__device__ __forceinline__ void vsum5(const T* __restrict__ hb, int ps, int rs, int r, int j, const T* w, T m[5]) {
#pragma unroll
    for (int q = 0; q < 5; ++q) {
        T s = T(0);
#pragma unroll
        for (int k = 0; k < SSIM_TAPS; ++k) s = fma(w[k], hb[q * ps + (r + k) * rs + j], s);
        m[q] = s;
    }
}

template <typename T>
struct SsimTerms {
    T a1, a2, b1, b2;
};

template <typename T>
__device__ __forceinline__ SsimTerms<T> ssim_terms(const T m[5], T c1, T c2) {
    const T mp = m[0], mt = m[1], mpt = mp * mt, mpp = mp * mp, mtt = mt * mt;
    SsimTerms<T> s;
    s.a1 = T(2) * mpt + c1;
    s.a2 = T(2) * (m[4] - mpt) + c2;
    s.b1 = mpp + mtt + c1;
    s.b2 = (m[2] - mpp) + (m[3] - mtt) + c2;
    return s;
}

// Deterministic CTA sum of two doubles (fixed shuffle tree, then the warps in order); result valid in thread 0.
__device__ __forceinline__ void block_sum2(double& a, double& b, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();  // red may still be read by a previous call
    if (lane == 0) {
        red[2 * warp] = a;
        red[2 * warp + 1] = b;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        a = red[0];
        b = red[1];
        for (int q = 1; q < LOSS_THREADS / 32; ++q) {
            a += red[2 * q];
            b += red[2 * q + 1];
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(LOSS_THREADS)
    k_photometric_loss_fwd(LossArgs<T> A, double2* __restrict__ partials, unsigned int* __restrict__ ticket,
                           T* __restrict__ out, double l1_weight, double ssim_weight) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* sp = reinterpret_cast<T*>(smem_raw);
    T* st = sp + LOSS_CG * FWD_IH * FWD_IW;
    T* hb = st + LOSS_CG * FWD_IH * FWD_IW;  // [5][IH][TW]
    __shared__ double red[2 * LOSS_THREADS / 32];
    __shared__ bool is_last;

    const int tx0 = blockIdx.x * LOSS_TW, ty0 = blockIdx.y * LOSS_TH, b = blockIdx.z;
    const int H = A.H, W = A.W;
    double acc_s = 0.0, acc_l1 = 0.0;
    for (int c0 = 0; c0 < A.C; c0 += LOSS_CG) {
        const int cg = min(LOSS_CG, A.C - c0);
        stage_region(sp, A.pred, A.ps, b, c0, cg, ty0, tx0, FWD_IH, FWD_IW, H, W);
        stage_region(st, A.target, A.ts, b, c0, cg, ty0, tx0, FWD_IH, FWD_IW, H, W);
        __syncthreads();
        for (int c = 0; c < cg; ++c) {
            const T* p = sp + c * FWD_IH * FWD_IW;
            const T* t = st + c * FWD_IH * FWD_IW;
            for (int e = threadIdx.x; e < FWD_IH * LOSS_TW; e += LOSS_THREADS) {
                const int r = e / LOSS_TW, j = e % LOSS_TW;
                T m0, m1, m2, m3, m4;
                hsum5(p, t, r * FWD_IW + j, A.w, m0, m1, m2, m3, m4);
                constexpr int PL = FWD_IH * LOSS_TW;
                hb[e] = m0;
                hb[PL + e] = m1;
                hb[2 * PL + e] = m2;
                hb[3 * PL + e] = m3;
                hb[4 * PL + e] = m4;
            }
            __syncthreads();
            for (int e = threadIdx.x; e < LOSS_TH * LOSS_TW; e += LOSS_THREADS) {
                const int i = e / LOSS_TW, j = e % LOSS_TW;
                const int y = ty0 + i, x = tx0 + j;
                if (y < H && x < W) acc_l1 += (double)fabs(p[i * FWD_IW + j] - t[i * FWD_IW + j]);
                if (y < H - SSIM_HALO && x < W - SSIM_HALO) {
                    T m[5];
                    vsum5(hb, FWD_IH * LOSS_TW, LOSS_TW, i, j, A.w, m);
                    const SsimTerms<T> s = ssim_terms(m, A.c1, A.c2);
                    acc_s += (double)((s.a1 * s.a2) / (s.b1 * s.b2));
                }
            }
            __syncthreads();  // hb / sp / st are rewritten next
        }
    }

    block_sum2(acc_s, acc_l1, red);
    const unsigned int n_blocks = gridDim.x * gridDim.y * gridDim.z;
    const unsigned int blk = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    if (threadIdx.x == 0) {
        partials[blk] = make_double2(acc_s, acc_l1);
        __threadfence();
        is_last = atomicAdd(ticket, 1u) == n_blocks - 1;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    double s = 0.0, l = 0.0;
    for (unsigned int q = threadIdx.x; q < n_blocks; q += LOSS_THREADS) {
        const double2 v = __ldcg(partials + q);
        s += v.x;
        l += v.y;
    }
    block_sum2(s, l, red);
    if (threadIdx.x == 0) {
        const double numel = (double)A.B * A.C * H * W;
        const double n_valid = (double)A.B * A.C * (H - SSIM_HALO) * (W - SSIM_HALO);
        const double l1 = l / numel, ssim = s / n_valid;
        out[0] = (T)(l1_weight * l1 + ssim_weight * (1.0 - ssim));
        out[1] = (T)l1;
        out[2] = (T)ssim;
        *ticket = 0u;  // ready for the next launch on the same buffer
    }
}

template <typename T>
__global__ void __launch_bounds__(LOSS_THREADS)
    k_photometric_loss_bwd(LossArgs<T> A, const T* __restrict__ grad_loss, T* __restrict__ grad, long long gs0,
                           long long gs1, long long gs2, long long gs3, T l1_scale, T ssim_scale) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* sp = reinterpret_cast<T*>(smem_raw);
    T* st = sp + LOSS_CG * BWD_RH * BWD_RW;
    T* hb = st + LOSS_CG * BWD_RH * BWD_RW;  // [5][RH][OW], then [3][OH][TW]
    T* db = hb + 5 * BWD_RH * BWD_OW;        // [3][OH][OW]
    T* gb = db + 3 * BWD_OH * BWD_OW;        // [CG][TH][TW]

    const int tx0 = blockIdx.x * LOSS_TW, ty0 = blockIdx.y * LOSS_TH, b = blockIdx.z;
    const int H = A.H, W = A.W;
    const int ry0 = ty0 - SSIM_HALO, rx0 = tx0 - SSIM_HALO;  // staged region / origin region start
    const T g = *grad_loss;
    const long long gs[4] = {gs0, gs1, gs2, gs3};
    for (int c0 = 0; c0 < A.C; c0 += LOSS_CG) {
        const int cg = min(LOSS_CG, A.C - c0);
        stage_region(sp, A.pred, A.ps, b, c0, cg, ry0, rx0, BWD_RH, BWD_RW, H, W);
        stage_region(st, A.target, A.ts, b, c0, cg, ry0, rx0, BWD_RH, BWD_RW, H, W);
        __syncthreads();
        for (int c = 0; c < cg; ++c) {
            const T* p = sp + c * BWD_RH * BWD_RW;
            const T* t = st + c * BWD_RH * BWD_RW;
            constexpr int PL = BWD_RH * BWD_OW;
            for (int e = threadIdx.x; e < PL; e += LOSS_THREADS) {
                const int r = e / BWD_OW, u = e % BWD_OW;
                T m0, m1, m2, m3, m4;
                hsum5(p, t, r * BWD_RW + u, A.w, m0, m1, m2, m3, m4);
                hb[e] = m0;
                hb[PL + e] = m1;
                hb[2 * PL + e] = m2;
                hb[3 * PL + e] = m3;
                hb[4 * PL + e] = m4;
            }
            __syncthreads();
            constexpr int DL = BWD_OH * BWD_OW;
            for (int e = threadIdx.x; e < DL; e += LOSS_THREADS) {
                const int v = e / BWD_OW, u = e % BWD_OW;
                const int oy = ry0 + v, ox = rx0 + u;
                T d_mu = T(0), d_pp = T(0), d_pt = T(0);
                if (oy >= 0 && oy < H - SSIM_HALO && ox >= 0 && ox < W - SSIM_HALO) {
                    T m[5];
                    vsum5(hb, PL, BWD_OW, v, u, A.w, m);
                    const SsimTerms<T> s = ssim_terms(m, A.c1, A.c2);
                    const T den = s.b1 * s.b2;
                    const T S = (s.a1 * s.a2) / den;
                    const T inv = T(1) / den;
                    d_mu = (T(2) * m[1] * (s.a2 - s.a1) - S * (T(2) * m[0] * (s.b2 - s.b1))) * inv;
                    d_pp = -S / s.b2;
                    d_pt = T(2) * s.a1 * inv;
                }
                db[e] = d_mu;
                db[DL + e] = d_pp;
                db[2 * DL + e] = d_pt;
            }
            __syncthreads();
            // transposed horizontal pass: pixel column j collects origins j + 10 - k (local origin coordinates)
            constexpr int TL = BWD_OH * LOSS_TW;
            for (int e = threadIdx.x; e < TL; e += LOSS_THREADS) {
                const int v = e / LOSS_TW, j = e % LOSS_TW;
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    T s = T(0);
#pragma unroll
                    for (int k = 0; k < SSIM_TAPS; ++k) s = fma(A.w[k], db[q * DL + v * BWD_OW + j + SSIM_HALO - k], s);
                    hb[q * TL + e] = s;
                }
            }
            __syncthreads();
            for (int e = threadIdx.x; e < LOSS_TH * LOSS_TW; e += LOSS_THREADS) {
                const int i = e / LOSS_TW, j = e % LOSS_TW;
                T dq[3];
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    T s = T(0);
#pragma unroll
                    for (int k = 0; k < SSIM_TAPS; ++k) s = fma(A.w[k], hb[q * TL + (i + SSIM_HALO - k) * LOSS_TW + j], s);
                    dq[q] = s;
                }
                const T pv = p[(i + SSIM_HALO) * BWD_RW + j + SSIM_HALO];
                const T tv = t[(i + SSIM_HALO) * BWD_RW + j + SSIM_HALO];
                const T diff = pv - tv;
                const T sgn = diff > T(0) ? T(1) : (diff < T(0) ? T(-1) : T(0));
                const T ssim_part = dq[0] + T(2) * pv * dq[1] + tv * dq[2];
                gb[c * LOSS_TH * LOSS_TW + e] = g * (l1_scale * sgn - ssim_scale * ssim_part);
            }
            __syncthreads();  // hb is rewritten by the next channel
        }
        // store the group's gradient in the caller's strides, along the smaller of the channel / column strides
        const bool interleaved = gs[1] < gs[3];
        const long long base = (long long)b * gs[0] + (long long)c0 * gs[1];
        const int n = cg * LOSS_TH * LOSS_TW;
        for (int e = threadIdx.x; e < n; e += LOSS_THREADS) {
            int c, i, j;
            if (interleaved) {
                c = e % cg;
                const int ij = e / cg;
                j = ij % LOSS_TW;
                i = ij / LOSS_TW;
            } else {
                j = e % LOSS_TW;
                const int ic = e / LOSS_TW;
                i = ic % LOSS_TH;
                c = ic / LOSS_TH;
            }
            const int y = ty0 + i, x = tx0 + j;
            if (y < H && x < W) grad[base + c * gs[1] + y * gs[2] + x * gs[3]] = gb[(c * LOSS_TH + i) * LOSS_TW + j];
        }
        __syncthreads();  // gb / sp / st are rewritten by the next channel group
    }
}

static dim3 loss_grid(int B, int H, int W) {
    return dim3((unsigned)((W + LOSS_TW - 1) / LOSS_TW), (unsigned)((H + LOSS_TH - 1) / LOSS_TH), (unsigned)B);
}

static bool loss_shape_ok(int B, int C, int H, int W) {
    return B >= 1 && B <= 65535 && C >= 1 && H >= SSIM_TAPS && W >= SSIM_TAPS && H <= (1 << 20) && W <= (1 << 24);
}

template <typename T>
static LossArgs<T> loss_args(int B, int C, int H, int W, const void* pred, const int64_t* ps, const void* target,
                             const int64_t* ts, const double* window, double c1, double c2) {
    LossArgs<T> A;
    A.pred = static_cast<const T*>(pred);
    A.target = static_cast<const T*>(target);
    for (int k = 0; k < 4; ++k) {
        A.ps[k] = ps[k];
        A.ts[k] = ts[k];
    }
    A.B = B;
    A.C = C;
    A.H = H;
    A.W = W;
    for (int k = 0; k < SSIM_TAPS; ++k) A.w[k] = (T)window[k];
    A.c1 = (T)c1;
    A.c2 = (T)c2;
    return A;
}

template <typename T>
static int launch_fwd(int B, int C, int H, int W, const void* pred, const int64_t* ps, const void* target,
                      const int64_t* ts, const double* window, double c1, double c2, double l1_weight,
                      double ssim_weight, void* out, void* temp, cudaStream_t stream) {
    const size_t smem = fwd_smem_bytes<T>();
    cudaError_t e = cudaFuncSetAttribute(k_photometric_loss_fwd<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return (int)e;
    unsigned int* ticket = static_cast<unsigned int*>(temp);
    double2* partials = reinterpret_cast<double2*>(static_cast<unsigned char*>(temp) + 16);
    e = cudaMemsetAsync(ticket, 0, sizeof(unsigned int), stream);
    if (e != cudaSuccess) return (int)e;
    k_photometric_loss_fwd<T><<<loss_grid(B, H, W), LOSS_THREADS, smem, stream>>>(
        loss_args<T>(B, C, H, W, pred, ps, target, ts, window, c1, c2), partials, ticket, static_cast<T*>(out),
        l1_weight, ssim_weight);
    return (int)cudaGetLastError();
}

template <typename T>
static int launch_bwd(int B, int C, int H, int W, const void* pred, const int64_t* ps, const void* target,
                      const int64_t* ts, const double* window, double c1, double c2, double l1_weight,
                      double ssim_weight, const void* grad_loss, void* grad_pred, const int64_t* gs,
                      cudaStream_t stream) {
    const size_t smem = bwd_smem_bytes<T>();
    cudaError_t e = cudaFuncSetAttribute(k_photometric_loss_bwd<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return (int)e;
    const double numel = (double)B * C * H * W;
    const double n_valid = (double)B * C * (H - SSIM_HALO) * (W - SSIM_HALO);
    k_photometric_loss_bwd<T><<<loss_grid(B, H, W), LOSS_THREADS, smem, stream>>>(
        loss_args<T>(B, C, H, W, pred, ps, target, ts, window, c1, c2), static_cast<const T*>(grad_loss),
        static_cast<T*>(grad_pred), gs[0], gs[1], gs[2], gs[3], (T)(l1_weight / numel), (T)(ssim_weight / n_valid));
    return (int)cudaGetLastError();
}

}  // namespace gsr

using namespace gsr;

extern "C" {

size_t gsr_photometric_loss_temp_bytes(int B, int C, int H, int W) {
    (void)C;
    if (B < 1 || H < 1 || W < 1) return 16;
    const dim3 g = loss_grid(B, H, W);
    return 16 + sizeof(double2) * (size_t)g.x * g.y * g.z;
}

int gsr_photometric_loss_forward(int dtype, int B, int C, int H, int W, const void* pred,
                                 const int64_t* pred_strides_host, const void* target,
                                 const int64_t* target_strides_host, const double* window_host, double c1, double c2,
                                 double l1_weight, double ssim_weight, void* out, void* temp, size_t temp_bytes,
                                 void* stream) {
    if (!loss_shape_ok(B, C, H, W) || (dtype != GSR_F32 && dtype != GSR_F64)) return GSR_ERR_BAD_ARG;
    if (!pred || !target || !out || !temp || !pred_strides_host || !target_strides_host || !window_host)
        return GSR_ERR_BAD_ARG;
    if (temp_bytes < gsr_photometric_loss_temp_bytes(B, C, H, W)) return GSR_ERR_BAD_ARG;
    if (dtype == GSR_F32)
        return launch_fwd<float>(B, C, H, W, pred, pred_strides_host, target, target_strides_host, window_host, c1,
                                 c2, l1_weight, ssim_weight, out, temp, (cudaStream_t)stream);
    return launch_fwd<double>(B, C, H, W, pred, pred_strides_host, target, target_strides_host, window_host, c1, c2,
                              l1_weight, ssim_weight, out, temp, (cudaStream_t)stream);
}

int gsr_photometric_loss_backward(int dtype, int B, int C, int H, int W, const void* pred,
                                  const int64_t* pred_strides_host, const void* target,
                                  const int64_t* target_strides_host, const double* window_host, double c1, double c2,
                                  double l1_weight, double ssim_weight, const void* grad_loss, void* grad_pred,
                                  const int64_t* grad_strides_host, void* stream) {
    if (!loss_shape_ok(B, C, H, W) || (dtype != GSR_F32 && dtype != GSR_F64)) return GSR_ERR_BAD_ARG;
    if (!pred || !target || !grad_loss || !grad_pred || !pred_strides_host || !target_strides_host ||
        !grad_strides_host || !window_host)
        return GSR_ERR_BAD_ARG;
    if (dtype == GSR_F32)
        return launch_bwd<float>(B, C, H, W, pred, pred_strides_host, target, target_strides_host, window_host, c1,
                                 c2, l1_weight, ssim_weight, grad_loss, grad_pred, grad_strides_host,
                                 (cudaStream_t)stream);
    return launch_bwd<double>(B, C, H, W, pred, pred_strides_host, target, target_strides_host, window_host, c1, c2,
                              l1_weight, ssim_weight, grad_loss, grad_pred, grad_strides_host, (cudaStream_t)stream);
}

}  // extern "C"
