// gsr_mcmc.cu — 3DGS-MCMC densification (Kheradmand et al. 2024, "3D Gaussian Splatting as Markov Chain Monte
// Carlo") on the FLAT parameter buffer and both Adam moments: the relocation formula, one pass that applies a
// relocation / growth plan, and the per-step SGLD position noise.
//
//   k_mcmc_relocation  per sampled row: the opacity and scale of N copies that render like the one source (fp64)
//   k_mcmc_apply       out row r <- in row src[r]; rows with set_row[r] >= 0 take the relocation's opacity / scale
//   k_mcmc_noise       xyz_i += scaler * w(o_i) * Sigma_i eps_i, in place, every optimizer step
#include <cstdint>

#include <curand_kernel.h>

#include "gsr_common.cuh"

namespace gsr {

// ---------------------------------------------------------------------------------------------------------------
// Relocation.  A Gaussian of opacity o and scale s is replaced by N copies of opacity o_hat and scale s', chosen so
// that N stacked copies have the source's total opacity and, at the centre, its rendered density:
//     1 - (1 - o_hat)^N = o                      ->  o_hat = 1 - (1 - o)^(1/N)
//     s' = s * o / D,   D = sum_{i=1..N} sum_{k=0..i-1} C(i-1, k) (-1)^k o_hat^(k+1) / sqrt(k+1)
// Hockey-stick identity sum_{i=k+1..N} C(i-1, k) = C(N, k+1) collapses D to one sum over j = k + 1:
//     D = sum_{j=1..N} C(N, j) (-1)^(j-1) o_hat^j / sqrt(j)
// (exactly the same value, N terms instead of N(N+1)/2).
//
// Why fp64.  The terms alternate in sign; their magnitudes add up to at most (1 + o_hat)^N - 1 < e^(N o_hat), while D
// itself is of the order of o.  For o near 1, N o_hat approaches -ln(1 - o) (about 16 at the clamp 1 - 2^-23), so the
// bound is e^16 ~ 9e6; at N = 51 and o = 1 - 2^-23 (o_hat = 0.268) the sum of |terms| is 5.8e4 against D = 1.98, a
// factor 2.9e4.  Summed in fp32 (2^-24 ~ 6e-8 per rounding) that leaves D, and the scale, wrong by 2e-4 relative
// (tests/mcmc_oracle.py restates it); in fp64 (2^-53 ~ 1.1e-16) the error stays below 1e-11.  The binomials are integers below 2^53 for N <= 51 (C(51, 25) ~ 2.5e14),
// and the recurrence C(N, j) = C(N, j-1) (N - j + 1) / j forms them exactly: the product before the division is
// below 51 * 2.5e14 < 2^53 and the quotient is an integer.  o_hat^j is a running product (relative error <= j ulp),
// and 1 - (1 - o)^(1/N) is formed as -expm1(log1p(-o) / N), which does not cancel for small o.
// o = 0: o_hat = 0 and D = 0; the limit o -> 0 of o / D is 1 (D ~ N o_hat ~ o), so the scale is kept.
// The opacity is rounded to fp32 and then clamped to [min_opacity, 1 - 2^-23]; the scale uses the unclamped o_hat.
__global__ void __launch_bounds__(256)
    k_mcmc_relocation(int n, const float* __restrict__ opacity, const float* __restrict__ scale,
                      const int32_t* __restrict__ ratio, int n_max, float min_opacity, float* __restrict__ new_opacity,
                      float* __restrict__ new_scale) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int N = min(max(ratio[r], 1), n_max);
    const double o = (double)opacity[r];
    const double oh = -expm1(log1p(-o) / (double)N);
    double D = 0.0, binom = 1.0, pw = 1.0;
    for (int j = 1; j <= N; ++j) {
        binom = binom * (double)(N - j + 1) / (double)j;
        pw *= oh;
        const double term = binom * pw / sqrt((double)j);
        D += (j & 1) ? term : -term;
    }
    const double coeff = (o > 0.0) ? o / D : 1.0;
    new_opacity[r] = fminf(fmaxf((float)oh, min_opacity), 1.0f - 0x1p-23f);
#pragma unroll
    for (int k = 0; k < 3; ++k) new_scale[3 * r + k] = (float)((double)scale[3 * r + k] * coeff);
}

// ---------------------------------------------------------------------------------------------------------------
// Apply: one pass over the flat layout, every output element written exactly once (like k_densify_apply, whose
// kernel is left as it is; the layout below is the same, gsr_densify.cu `densify_layout`).
//   out row r <- in row src[r]
//   set_row[r] >= 0: opacity <- logit(new_opacity[set_row[r]]) = logf(p / (1 - p)),  scale <- logf(new_scale[...])
//                    (one correctly rounded subtract and divide, then logf: the order torch.logit / torch.log use)
//   Adam moments: zero where set_row[r] >= 0 (the rows whose parameters the pass changes), else the source row's.
constexpr int MCMC_SECTIONS = 6;  // xyz 3 | quaternion 4 | scale 3 | opacity 1 | rgb 3 | sh 3K

struct McmcLayout {
    long long in_off[MCMC_SECTIONS + 1];
    long long out_off[MCMC_SECTIONS + 1];
    int width[MCMC_SECTIONS];
};

static void mcmc_layout(long long n, int n_sh_rest, long long* off, int* width) {
    const int w[MCMC_SECTIONS] = {3, 4, 3, 1, 3, 3 * n_sh_rest};
    off[0] = 0;
    for (int i = 0; i < MCMC_SECTIONS; ++i) {
        off[i + 1] = (off[i] + n * w[i] + 3) & ~3ll;
        if (width != nullptr) width[i] = w[i];
    }
}

__global__ void __launch_bounds__(256)
    k_mcmc_apply(int n_out, McmcLayout L, const float* __restrict__ p_in, const float* __restrict__ m_in,
                 const float* __restrict__ v_in, const int32_t* __restrict__ src, const int32_t* __restrict__ set_row,
                 const float* __restrict__ new_opacity, const float* __restrict__ new_scale, float* __restrict__ p_out,
                 float* __restrict__ m_out, float* __restrict__ v_out) {
    const int s = blockIdx.y;
    const int w = L.width[s];
    if (w == 0) return;
    const long long n_el = (long long)n_out * w;
    const long long padded = L.out_off[s + 1] - L.out_off[s];
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < padded; e += stride) {
        const long long o = L.out_off[s] + e;
        if (e >= n_el) {  // padding between sections
            p_out[o] = 0.0f;
            if (m_out != nullptr) { m_out[o] = 0.0f; v_out[o] = 0.0f; }
            continue;
        }
        const int r = (int)(e / w), k = (int)(e - (long long)r * w);
        const long long i = L.in_off[s] + (long long)src[r] * w + k;
        const int sr = set_row != nullptr ? set_row[r] : -1;
        float val;
        if (sr >= 0 && s == 2) {
            val = logf(new_scale[(size_t)sr * 3 + k]);
        } else if (sr >= 0 && s == 3) {
            const float q = new_opacity[sr];
            val = logf(__fdiv_rn(q, __fsub_rn(1.0f, q)));
        } else {
            val = p_in[i];
        }
        p_out[o] = val;
        if (m_out != nullptr) {
            m_out[o] = sr >= 0 ? 0.0f : m_in[i];
            v_out[o] = sr >= 0 ? 0.0f : v_in[i];
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Position noise (the SGLD step of 3DGS-MCMC), in place on the xyz section of the flat buffer, per Gaussian i:
//     o = sigmoid(opacity_i),  w = 1 / (1 + exp(-k ((1 - o) - x0))),  q = q_i / |q_i|,  R = R(q) (w, x, y, z)
//     d = R diag(exp(2 s_i)) R^T eps_i       (= Sigma_i eps_i, evaluated as R (exp(2 s) * (R^T eps)))
//     xyz_i <- fma(scaler * w, d, xyz_i)
// eps_i ~ N(0, I_3) from counter-based Philox4x32-10 keyed by (seed, subsequence i, offset): curand_normal4 of
// curand_init(seed, i, 4 * offset) — one 128-bit Philox block per Gaussian per offset, so offsets (steps) never share
// a block and a step's draws do not depend on the launch shape; its fourth normal is unused.  eps_in [N,3] replaces
// the draws; eps_out [N,3] records the draws used.  Reads 44 B and writes 12 B per Gaussian.
__global__ void __launch_bounds__(256)
    k_mcmc_noise(int n, long long off_q, long long off_s, long long off_o, float* __restrict__ p, float scaler,
                 float k_steep, float x0, unsigned long long seed, unsigned long long offset,
                 const float* __restrict__ eps_in, float* __restrict__ eps_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float e0, e1, e2;
    if (eps_in != nullptr) {
        e0 = eps_in[3 * i]; e1 = eps_in[3 * i + 1]; e2 = eps_in[3 * i + 2];
    } else {
        curandStatePhilox4_32_10_t st;
        curand_init(seed, (unsigned long long)i, 4ull * offset, &st);
        const float4 z = curand_normal4(&st);
        e0 = z.x; e1 = z.y; e2 = z.z;
    }
    if (eps_out != nullptr) {
        eps_out[3 * i] = e0; eps_out[3 * i + 1] = e1; eps_out[3 * i + 2] = e2;
    }
    const float4 q4 = reinterpret_cast<const float4*>(p + off_q)[i];
    const float op = 1.0f / (1.0f + expf(-p[off_o + i]));
    const float wgt = 1.0f / (1.0f + expf(-k_steep * ((1.0f - op) - x0)));
    const float inv = rsqrtf(q4.x * q4.x + q4.y * q4.y + q4.z * q4.z + q4.w * q4.w);
    const float w = q4.x * inv, x = q4.y * inv, y = q4.z * inv, z = q4.w * inv;
    const float R00 = 1.f - 2.f * (y * y + z * z), R01 = 2.f * (x * y - w * z), R02 = 2.f * (x * z + w * y);
    const float R10 = 2.f * (x * y + w * z), R11 = 1.f - 2.f * (x * x + z * z), R12 = 2.f * (y * z - w * x);
    const float R20 = 2.f * (x * z - w * y), R21 = 2.f * (y * z + w * x), R22 = 1.f - 2.f * (x * x + y * y);
    const float v0 = expf(2.f * p[off_s + 3 * i]), v1 = expf(2.f * p[off_s + 3 * i + 1]),
                v2 = expf(2.f * p[off_s + 3 * i + 2]);
    const float t0 = v0 * (R00 * e0 + R10 * e1 + R20 * e2);
    const float t1 = v1 * (R01 * e0 + R11 * e1 + R21 * e2);
    const float t2 = v2 * (R02 * e0 + R12 * e1 + R22 * e2);
    const float sw = scaler * wgt;
    p[3 * i] = __fmaf_rn(sw, R00 * t0 + R01 * t1 + R02 * t2, p[3 * i]);
    p[3 * i + 1] = __fmaf_rn(sw, R10 * t0 + R11 * t1 + R12 * t2, p[3 * i + 1]);
    p[3 * i + 2] = __fmaf_rn(sw, R20 * t0 + R21 * t1 + R22 * t2, p[3 * i + 2]);
}

// [a, a + na) and [b, b + nb) (in floats) share memory
static bool overlaps(const void* a, long long na, const void* b, long long nb) {
    if (a == nullptr || b == nullptr || na <= 0 || nb <= 0) return false;
    const char *pa = static_cast<const char*>(a), *pb = static_cast<const char*>(b);
    return pa < pb + nb * 4 && pb < pa + na * 4;
}

static int blocks_for(long long n) { return (int)((n + 255) / 256); }

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_mcmc_relocation(int n, const float* opacity, const float* scale, const int32_t* ratio, int n_max,
                        float min_opacity, float* new_opacity, float* new_scale, void* stream) {
    if (n < 0 || n_max < 1) return GSR_ERR_BAD_ARG;
    if (n == 0) return GSR_OK;
    if (!opacity || !scale || !ratio || !new_opacity || !new_scale) return GSR_ERR_BAD_ARG;
    const long long n1 = n, n3 = 3ll * n;
    if (overlaps(new_opacity, n1, new_scale, n3) || overlaps(new_opacity, n1, opacity, n1) ||
        overlaps(new_opacity, n1, scale, n3) || overlaps(new_opacity, n1, ratio, n1) ||
        overlaps(new_scale, n3, opacity, n1) || overlaps(new_scale, n3, scale, n3) ||
        overlaps(new_scale, n3, ratio, n1))
        return GSR_ERR_BAD_ARG;
    k_mcmc_relocation<<<blocks_for(n), 256, 0, (cudaStream_t)stream>>>(n, opacity, scale, ratio, n_max, min_opacity,
                                                                        new_opacity, new_scale);
    return (int)cudaGetLastError();
}

int gsr_mcmc_apply(int n_in, int n_out, int n_sh_rest, const float* p_in, const float* m_in, const float* v_in,
                   const int32_t* src, const int32_t* set_row, const float* new_opacity, const float* new_scale,
                   float* p_out, float* m_out, float* v_out, void* stream) {
    if (n_in < 0 || n_out < n_in || n_sh_rest < 0) return GSR_ERR_BAD_ARG;
    if ((m_in == nullptr) != (v_in == nullptr) || (m_out == nullptr) != (v_out == nullptr) ||
        (m_in == nullptr) != (m_out == nullptr))
        return GSR_ERR_BAD_ARG;
    if ((set_row == nullptr) != (new_opacity == nullptr) || (set_row == nullptr) != (new_scale == nullptr))
        return GSR_ERR_BAD_ARG;
    if (n_out == 0) return GSR_OK;
    if (p_in == nullptr || src == nullptr || p_out == nullptr) return GSR_ERR_BAD_ARG;
    McmcLayout L;
    mcmc_layout(n_in, n_sh_rest, L.in_off, L.width);
    mcmc_layout(n_out, n_sh_rest, L.out_off, nullptr);
    const long long ni = L.in_off[MCMC_SECTIONS], no = L.out_off[MCMC_SECTIONS];
    const void* outs[3] = {p_out, m_out, v_out};
    const void* ins[3] = {p_in, m_in, v_in};
    for (int a = 0; a < 3; ++a) {
        for (int b = 0; b < 3; ++b) {
            if (overlaps(outs[a], no, ins[b], ni)) return GSR_ERR_BAD_ARG;
            if (a < b && overlaps(outs[a], no, outs[b], no)) return GSR_ERR_BAD_ARG;
        }
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long widest = (long long)n_out * (n_sh_rest > 0 ? 3 * n_sh_rest : 4);
    long long bx = (widest + 255) / 256;
    const long long cap = (long long)sms * 8;
    if (bx > cap) bx = cap;
    if (bx < 1) bx = 1;
    const dim3 grid((unsigned)bx, MCMC_SECTIONS);
    k_mcmc_apply<<<grid, 256, 0, (cudaStream_t)stream>>>(n_out, L, p_in, m_in, v_in, src, set_row, new_opacity,
                                                          new_scale, p_out, m_out, v_out);
    return (int)cudaGetLastError();
}

int gsr_mcmc_noise(int n, int n_sh_rest, float* p, double scaler, double k, double x0, uint64_t seed,
                   uint64_t offset, const float* eps_in, float* eps_out, void* stream) {
    if (n < 0 || n_sh_rest < 0) return GSR_ERR_BAD_ARG;
    if (n == 0) return GSR_OK;
    if (p == nullptr) return GSR_ERR_BAD_ARG;
    long long off[MCMC_SECTIONS + 1];
    mcmc_layout(n, n_sh_rest, off, nullptr);
    const long long n3 = 3ll * n;
    if (overlaps(eps_out, n3, p, off[MCMC_SECTIONS]) || overlaps(eps_out, n3, eps_in, n3) ||
        overlaps(eps_in, n3, p, off[MCMC_SECTIONS]))
        return GSR_ERR_BAD_ARG;
    k_mcmc_noise<<<blocks_for(n), 256, 0, (cudaStream_t)stream>>>(n, off[1], off[2], off[3], p, (float)scaler,
                                                                   (float)k, (float)x0, seed, offset, eps_in, eps_out);
    return (int)cudaGetLastError();
}

}  // extern "C"
