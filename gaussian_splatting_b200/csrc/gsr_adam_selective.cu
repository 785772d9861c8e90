// gsr_adam_selective.cu — Adam on the flat parameter buffer, restricted to the rows a view saw
// (include/gsr_selective_adam.h; the sparse Adam of Taming 3DGS, gsplat's SelectiveAdam).
//
// The streaming float4 loop of k_adam (gsr_adam.cu) with two changes:
//   * each float4 finds its section, then the row of each of its 4 elements, (e - section_start) / width: one
//     64-bit multiply-high by a per-section ceil(2^64 / width) gives the first lane's row (exact for 32-bit offsets,
//     Lemire, Kaser & Kurz 2019), the other lanes add 0..3 by comparing the remainder with the width;
//   * when none of those rows is visible the float4 issues NO load of g, p, m or v — the HBM traffic of the rows
//     the view culled is the whole saving.  Otherwise every lane of a visible row gets adam_one, the other lanes
//     are stored back with their old values.
// Section padding lies past row n_rows - 1 of its section, so it is never visible and never written.
//
// Sharded form: the mask of a row is the OR of every rank's mask (peer loads, like the gradients); the gradient of
// a visible row is the rank-ordered mean, exactly as gsr_adam_step_sharded forms it, so the replicas stay
// bit-identical.
#include <cmath>
#include <cstdint>

#include "gsr_common.cuh"
#include "../../include/gsr_selective_adam.h"

namespace gsr {
namespace selective {

constexpr int SEL_MAX_SECTIONS = 8;
constexpr int SEL_MAX_PEERS = 16;
constexpr int FLAT_WIDTHS[6] = {3, 4, 3, 1, 3, 3};  // the sh width is 3 * n_sh_rest

struct SelSections {
    int n;
    long long end4[SEL_MAX_SECTIONS];             // exclusive end of each section, in float4 units
    long long start[SEL_MAX_SECTIONS];            // first element of each section
    unsigned long long magic[SEL_MAX_SECTIONS];   // ceil(2^64 / width); unused for width 1
    int width[SEL_MAX_SECTIONS];                  // floats per row
    float neg_step[SEL_MAX_SECTIONS];             // -lr / (1 - beta1^t)
};
struct SelPeers {
    int world;
    const float4* grad[SEL_MAX_PEERS];
    float4* param[SEL_MAX_PEERS];
    const uint8_t* vis[SEL_MAX_PEERS];
};

// gsr_adam.cu's per-element update, operation for operation (torch.optim.Adam's CUDA order; see there)
__device__ __forceinline__ float adam_one(float p, float g, float& m, float& v, float w1, float beta2, float w2,
                                          float inv_bias2_sqrt, float eps, float neg_step) {
    m = __fmaf_rn(w1, __fsub_rn(g, m), m);
    v = __fmaf_rn(__fmul_rn(w2, g), g, __fmul_rn(v, beta2));
    const float d = __fadd_rn(__fmul_rn(__fsqrt_rn(v), inv_bias2_sqrt), eps);
    return __fmaf_rn(neg_step, __fdiv_rn(m, d), p);
}

__device__ __forceinline__ float4 ld_peer(const float4* p) {  // peer memory changes between steps: never L1
    float4 v;
    asm volatile("ld.global.cv.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

__device__ __forceinline__ unsigned ld_peer_u8(const uint8_t* p) {
    unsigned short v;
    asm volatile("ld.global.cv.u8 %0, [%1];" : "=h"(v) : "l"(p));
    return v;
}

template <bool SHARDED>
__device__ __forceinline__ bool row_visible(const uint8_t* __restrict__ vis, const SelPeers& peers, unsigned r) {
    if (!SHARDED) return __ldg(vis + r) != 0;
    unsigned any = 0;
    for (int q = 0; q < peers.world; ++q) any |= ld_peer_u8(peers.vis[q] + r);
    return any != 0;
}

__device__ __forceinline__ void masked_update(float& p, float g, float& m, float& v, bool on, float w1, float beta2,
                                              float w2, float inv_bias2_sqrt, float eps, float ns) {
    if (on) p = adam_one(p, g, m, v, w1, beta2, w2, inv_bias2_sqrt, eps, ns);
}

// i4 indexes float4 elements of the flat buffer; m / v are indexed relative to lo4 (the shard).
template <bool SHARDED>
__global__ void __launch_bounds__(256)
    k_adam_selective(long long lo4, long long hi4, unsigned n_rows, float4* __restrict__ p,
                     const float4* __restrict__ g, float4* __restrict__ m, float4* __restrict__ v,
                     const uint8_t* __restrict__ vis, SelSections sec, SelPeers peers, float w1, float beta2, float w2,
                     float inv_bias2_sqrt, float eps, float inv_world) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = lo4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < hi4; i += stride) {
        int s = 0;
#pragma unroll
        for (int k = 0; k < SEL_MAX_SECTIONS - 1; ++k) s += (k < sec.n - 1 && i >= sec.end4[k]) ? 1 : 0;
        const int w = sec.width[s];
        const unsigned x0 = (unsigned)(4 * i - sec.start[s]);  // < 2^32: checked on the host
        const unsigned r0 = w == 1 ? x0 : (unsigned)__umul64hi((unsigned long long)x0, sec.magic[s]);
        const int rem = (int)(x0 - r0 * (unsigned)w);
        bool on[4];
        unsigned prev = 0xffffffffu;
        bool prev_on = false;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int t = rem + j;  // < w + 3: lane j lies 0..3 rows past r0
            const unsigned r = r0 + (t >= w) + (t >= 2 * w) + (t >= 3 * w);
            if (r != prev) {
                prev_on = r < n_rows && row_visible<SHARDED>(vis, peers, r);
                prev = r;
            }
            on[j] = prev_on;
        }
        if (!(on[0] || on[1] || on[2] || on[3])) continue;  // nothing of this float4 was seen: no traffic
        const float ns = sec.neg_step[s];
        float4 gg;
        if (SHARDED) {
            gg = ld_peer(peers.grad[0] + i);
            for (int q = 1; q < peers.world; ++q) {
                const float4 t = ld_peer(peers.grad[q] + i);
                gg.x += t.x; gg.y += t.y; gg.z += t.z; gg.w += t.w;
            }
            gg.x *= inv_world; gg.y *= inv_world; gg.z *= inv_world; gg.w *= inv_world;
        } else {
            gg = g[i];
        }
        float4 pp = p[i], mm = m[i - lo4], vv = v[i - lo4];
        masked_update(pp.x, gg.x, mm.x, vv.x, on[0], w1, beta2, w2, inv_bias2_sqrt, eps, ns);
        masked_update(pp.y, gg.y, mm.y, vv.y, on[1], w1, beta2, w2, inv_bias2_sqrt, eps, ns);
        masked_update(pp.z, gg.z, mm.z, vv.z, on[2], w1, beta2, w2, inv_bias2_sqrt, eps, ns);
        masked_update(pp.w, gg.w, mm.w, vv.w, on[3], w1, beta2, w2, inv_bias2_sqrt, eps, ns);
        m[i - lo4] = mm;
        v[i - lo4] = vv;
        if (SHARDED) {
            for (int q = 0; q < peers.world; ++q) peers.param[q][i] = pp;
        } else {
            p[i] = pp;
        }
    }
}

// The caller's sections must be exactly the flat layout of n_rows gaussians with n_sh_rest coefficients.
static int fill_sections(SelSections& sec, int64_t n_rows, int n_sh_rest, int n_sections,
                         const int64_t* section_end, const double* section_lr, double bias1, int64_t* numel) {
    if (n_rows < 0 || n_sh_rest < 0 || n_sections < 1 || n_sections > SEL_MAX_SECTIONS || section_end == nullptr ||
        section_lr == nullptr)
        return GSR_ERR_BAD_ARG;
    int k = 0;
    int64_t off = 0;
    for (int f = 0; f < 6; ++f) {
        const int64_t w = f == 5 ? 3 * (int64_t)n_sh_rest : FLAT_WIDTHS[f];
        if (w == 0) continue;
        if (n_rows > ((int64_t(1) << 32) - 4) / w) return GSR_ERR_BAD_ARG;  // rows come from 32-bit offsets
        const int64_t end = (off + n_rows * w + 3) & ~int64_t(3);
        if (k >= n_sections || section_end[k] != end) return GSR_ERR_BAD_ARG;
        sec.start[k] = off;
        sec.end4[k] = end / 4;
        sec.width[k] = (int)w;
        sec.magic[k] = w == 1 ? 0ull : ~0ull / (unsigned long long)w + 1ull;  // floor((2^64 - 1) / w) + 1 = ceil(2^64 / w)
        sec.neg_step[k] = (float)(-section_lr[k] / bias1);
        off = end;
        ++k;
    }
    if (k != n_sections) return GSR_ERR_BAD_ARG;
    sec.n = n_sections;
    for (int j = n_sections; j < SEL_MAX_SECTIONS; ++j) {
        sec.end4[j] = sec.end4[n_sections - 1];
        sec.start[j] = sec.start[n_sections - 1];
        sec.magic[j] = sec.magic[n_sections - 1];
        sec.width[j] = sec.width[n_sections - 1];
        sec.neg_step[j] = 0.0f;
    }
    *numel = off;
    return 0;
}

static int adam_grid(long long n4) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long want = (n4 + 255) / 256;
    const long long cap = (long long)sms * 8;  // 8 resident CTAs of 256 threads per SM
    return (int)(want < cap ? (want > 0 ? want : 1) : cap);
}

}  // namespace selective
}  // namespace gsr

using namespace gsr;
using namespace gsr::selective;

extern "C" {

int gsr_adam_step_selective(int64_t n_rows, int n_sh_rest, float* p, const float* g, float* m, float* v,
                            const uint8_t* visible, int n_sections, const int64_t* section_end,
                            const double* section_lr, double beta1, double beta2, double eps, int step, void* stream) {
    if (step < 1) return GSR_ERR_BAD_ARG;
    const double bias1 = 1.0 - pow(beta1, (double)step), bias2 = 1.0 - pow(beta2, (double)step);
    SelSections sec;
    int64_t n = 0;
    if (int rc = fill_sections(sec, n_rows, n_sh_rest, n_sections, section_end, section_lr, bias1, &n)) return rc;
    if (n_rows == 0) return 0;
    if (!p || !g || !m || !v || !visible) return GSR_ERR_BAD_ARG;
    SelPeers peers;
    peers.world = 1;
    const float inv_b2s = 1.0f / (float)sqrt(bias2);
    k_adam_selective<false><<<adam_grid(n / 4), 256, 0, (cudaStream_t)stream>>>(
        0, n / 4, (unsigned)n_rows, reinterpret_cast<float4*>(p), reinterpret_cast<const float4*>(g),
        reinterpret_cast<float4*>(m), reinterpret_cast<float4*>(v), visible, sec, peers, (float)(1.0 - beta1),
        (float)beta2, (float)(1.0 - beta2), inv_b2s, (float)eps, 1.0f);
    return (int)cudaGetLastError();
}

int gsr_adam_step_selective_sharded(int64_t lo, int64_t hi, int world, const float* const* peer_grads,
                                    float* const* peer_params, const uint8_t* const* peer_visible, int self_rank,
                                    float* m_shard, float* v_shard, int64_t n_rows, int n_sh_rest, int n_sections,
                                    const int64_t* section_end, const double* section_lr, double beta1, double beta2,
                                    double eps, int step, void* stream) {
    if (lo < 0 || hi < lo || lo % 4 != 0 || hi % 4 != 0 || step < 1 || world < 1 || world > SEL_MAX_PEERS ||
        self_rank < 0 || self_rank >= world)
        return GSR_ERR_BAD_ARG;
    const double bias1 = 1.0 - pow(beta1, (double)step), bias2 = 1.0 - pow(beta2, (double)step);
    SelSections sec;
    int64_t n = 0;
    if (int rc = fill_sections(sec, n_rows, n_sh_rest, n_sections, section_end, section_lr, bias1, &n)) return rc;
    if (hi > n) return GSR_ERR_BAD_ARG;
    if (n_rows == 0 || hi == lo) return 0;
    if (!peer_grads || !peer_params || !peer_visible || !m_shard || !v_shard) return GSR_ERR_BAD_ARG;
    SelPeers peers;
    peers.world = world;
    for (int q = 0; q < world; ++q) {
        if (!peer_grads[q] || !peer_params[q] || !peer_visible[q]) return GSR_ERR_BAD_ARG;
        peers.grad[q] = reinterpret_cast<const float4*>(peer_grads[q]);
        peers.param[q] = reinterpret_cast<float4*>(peer_params[q]);
        peers.vis[q] = peer_visible[q];
    }
    const float inv_b2s = 1.0f / (float)sqrt(bias2);
    k_adam_selective<true><<<adam_grid((hi - lo) / 4), 256, 0, (cudaStream_t)stream>>>(
        lo / 4, hi / 4, (unsigned)n_rows, reinterpret_cast<float4*>(peer_params[self_rank]), nullptr,
        reinterpret_cast<float4*>(m_shard), reinterpret_cast<float4*>(v_shard), nullptr, sec, peers,
        (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), inv_b2s, (float)eps, 1.0f / (float)world);
    return (int)cudaGetLastError();
}

}  // extern "C"
