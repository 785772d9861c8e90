// gsr_preprocess.cuh — the per-Gaussian backward of the fused path and the view constants it reads, shared by the
// single-view kernels (gsr_preprocess.cu, libgsr_b200.so) and the multi-view kernels (gsr_batch.cu,
// libgsr_batch.so).  GSR_PRE_BWD_VIEW is one view's VJP for one gaussian; the single-view kernels store its
// result, the batched kernels add it up over the views.
#pragma once
#include "gsr_common.cuh"
#include "gsr_math.cuh"
#include "gsr_math_bwd.cuh"
#include "gsr_record.cuh"

namespace gsr {

constexpr int PRE_THREADS = 128;  // gaussians per CTA; every per-gaussian array slice of a CTA is one contiguous,
                                  // 16-byte aligned run in HBM, moved by TMA bulk copies

struct ViewConsts {
    float T[16];
    float K[9];
    float cam[3];  // camera centre in world frame = inverse(camera_T_world)[:3, 3]
};

// Last column of inverse(T) with the bits torch.inverse / torch.linalg.inv_ex produce on this platform for one 4x4
// fp32 matrix (the reference's op, splat_py/rasterize.py:91-93).  torch runs cuSOLVER getrf + cuBLAS trsm x2 — 15
// micro-kernels; their arithmetic was pinned by tools/dev/inverse_probe2.py (600 of 600 random rigid and
// general matrices bit-identical, LU factors and solution separately):
//   LU, partial pivoting (first maximum):  l_ik = a_ik * (1 / a_kk)   [IEEE reciprocal, then a multiply]
//                                          a_ij = fma(-l_ik, a_kj, a_ij)
//   L y = P e_3 forward, fma accumulation;  U x = y by columns from the last one (right-looking: the terms of a row
//   are subtracted in DESCENDING column order), fma accumulation, then one IEEE division by the diagonal.
// One thread; ~100 flops.
__device__ void camera_centre(const float* __restrict__ T, float* __restrict__ cam) {
    float A[4][4];
    int perm[4] = {0, 1, 2, 3};
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) A[r][c] = T[r * 4 + c];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        int piv = k;
        float best = fabsf(A[k][k]);
#pragma unroll
        for (int r = k + 1; r < 4; ++r) {
            const float v = fabsf(A[r][k]);
            if (v > best) { best = v; piv = r; }
        }
#pragma unroll
        for (int r = k + 1; r < 4; ++r) {  // swap rows k and piv without dynamic indexing
            if (r == piv) {
#pragma unroll
                for (int c = 0; c < 4; ++c) { const float t = A[k][c]; A[k][c] = A[r][c]; A[r][c] = t; }
                const int tp = perm[k]; perm[k] = perm[r]; perm[r] = tp;
            }
        }
        const float rp = __frcp_rn(A[k][k]);
#pragma unroll
        for (int i = k + 1; i < 4; ++i) {
            const float l = __fmul_rn(A[i][k], rp);
            A[i][k] = l;
#pragma unroll
            for (int c = k + 1; c < 4; ++c) A[i][c] = __fmaf_rn(-l, A[k][c], A[i][c]);
        }
    }
    float y[4], x[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float acc = (perm[i] == 3) ? 1.0f : 0.0f;
#pragma unroll
        for (int c = 0; c < i; ++c) acc = __fmaf_rn(-A[i][c], y[c], acc);
        y[i] = acc;
    }
#pragma unroll
    for (int i = 3; i >= 0; --i) {
        float acc = y[i];
#pragma unroll
        for (int c = 3; c > i; --c) acc = __fmaf_rn(-A[i][c], x[c], acc);
        x[i] = __fdiv_rn(acc, A[i][i]);
    }
    cam[0] = x[0];
    cam[1] = x[1];
    cam[2] = x[2];
}

// Whole CTA: threads 0..27 fetch one constant each (one memory latency instead of 28 dependent-issue loads by a
// single thread); ends with a CTA barrier.  The camera centre is taken from `cam` when the caller supplies it,
// else derived from T by thread 0.
__device__ __forceinline__ void load_view_cta(const float* __restrict__ T, const float* __restrict__ K,
                                              const float* __restrict__ cam, ViewConsts& vc, bool need_centre) {
    const int t = threadIdx.x;
    if (t < 16) vc.T[t] = T[t];
    else if (t < 25) vc.K[t - 16] = K[t - 16];
    else if (t < 28 && cam != nullptr) vc.cam[t - 25] = cam[t - 25];
    __syncthreads();
    if (need_centre && cam == nullptr) {
        if (t == 0) camera_centre(vc.T, vc.cam);
        __syncthreads();
    }
}

// cooperative, coalesced smem <-> global copies for the last (partial) block, where TMA's 16-byte
// granularity does not hold
__device__ __forceinline__ void coop_copy(float* __restrict__ dst, const float* __restrict__ src, int n_floats) {
    for (int k = threadIdx.x; k < n_floats; k += PRE_THREADS) dst[k] = src[k];
}

// One view's fused VJP for one visible gaussian, as a statement block: it reads the view constants `vc`, the
// parameters x y z qw qx qy qz s0 s1 s2 opl (f: the 3-D filter) and the view's gradient row (grv rgb, gov opacity,
// guv uv, gcv conic, gzc camera-frame z; gov and gcv are modified) and assigns gx gq gs go gdc and the SH rest
// gradients my_sh[c * NR + k - 1].  A macro rather than a function so that the single-view kernels compile to
// exactly the instructions they had before the multi-view kernels shared this code.  Order of the chain: SURVEY.md
// Appendix A "Per-Gaussian backward".
// DEPTH: the interleaved rows carry the render backward's camera-frame z gradient in slot 9 (conic2 z pad2); it joins
// the z component of the camera-frame position gradient before grad_xyz = W^T grad_xyz_cam.
// ANTIALIAS: the rows' opacity slot is the gradient on the compensated opacity sigmoid(o) * rho of k_preprocess_fwd_aa;
// it is carried back to sigmoid(o) and, through rho, to the conic.
// FILTER3D: Sigma_world of the 3-D filtered variances (k_preprocess_fwd_f3d); the opacity slot (after rho) is the
// gradient on sigmoid(o) * coef, carried back to sigmoid(o) and, through coef, to the log-scales.  No gradient goes
// to the filter.
#define GSR_PRE_BWD_VIEW                                                                                                 \
    {                                                                                                                    \
        float px, py, pz;                                                                                                \
        transform_point<float>(vc.T, x, y, z, px, py, pz);                                                               \
        float S6[6], S9[9], J[6], W[9];                                                                                  \
        /* 3-D filter: the forward's variances and opacity factor, re-formed (gsr_record.cuh f3d_filter) */              \
        float e[3], v[3], vp[3], t[3], F = 0.f, coef = 1.f;                                                              \
        if (FILTER3D) {                                                                                                  \
            F = __fmul_rn(f, f);                                                                                         \
            e[0] = expf(s0); e[1] = expf(s1); e[2] = expf(s2);                                                           \
_Pragma("unroll")                                                                                                        \
            for (int k = 0; k < 3; ++k) v[k] = __fmul_rn(e[k], e[k]);                                                    \
            coef = f3d_filter(v, F, vp, t);                                                                              \
            sigma_world_var<float>(qw, qx, qy, qz, vp[0], vp[1], vp[2], S6);                                             \
        } else {                                                                                                         \
            sigma_world<float>(qw, qx, qy, qz, s0, s1, s2, S6);                                                          \
        }                                                                                                                \
        sym6_to_full(S6, S9);                                                                                            \
        proj_jacobian<float>(px, py, pz, vc.K[0], vc.K[4], J);                                                           \
        W[0] = vc.T[0]; W[1] = vc.T[1]; W[2] = vc.T[2];                                                                  \
        W[3] = vc.T[4]; W[4] = vc.T[5]; W[5] = vc.T[6];                                                                  \
        W[6] = vc.T[8]; W[7] = vc.T[9]; W[8] = vc.T[10];                                                                 \
                                                                                                                         \
        float rho = 1.0f;                                                                                                \
        if (ANTIALIAS) {                                                                                                 \
            /* The row's opacity slot is g' = dL/d(sigmoid(o) * rho).  With A = c0 + 1/4, C = c2 + 1/4, bh = c1 / 2, */  \
            /* det = A C - bh^2 and rho^2 = det0 / det, the cancellation-free forms of the conic derivatives are */      \
            /*   drho/dc0 = (c2 C + bh^2) / (8 rho det^2),  drho/dc2 = (c0 A + bh^2) / (8 rho det^2), */                 \
            /*   drho/dc1 = -bh (A + C - 1/4) / (8 rho det^2) */                                                         \
            /* (c2 - rho^2 C = (c2 C + bh^2) / (4 det), 1 - rho^2 = (A + C - 1/4) / (4 det)).  Where rho == 0 the */     \
            /* gradient is infinite but the splat never contributed (g' == 0): no gradient goes through rho there. */    \
            float cn[3];                                                                                                 \
            conic_from<float>(S9, J, W, cn, nullptr);                                                                    \
            rho = aa_rho(cn[0], cn[1], cn[2]);                                                                           \
            const float A = cn[0] + 0.25f, C = cn[2] + 0.25f, bh = 0.5f * cn[1];                                         \
            const float rd = 1.0f / (A * C - bh * bh);                                                                   \
            const float k =                                                                                              \
                (0.125f * gov * (FILTER3D ? __fmul_rn(sigmoid_torch(opl), coef) : sigmoid_torch(opl))) * rd / rho * rd;  \
            const float kr = rho > 0.0f ? k : 0.0f;                                                                      \
            gcv[0] += kr * (cn[2] * C + bh * bh);                                                                        \
            gcv[1] -= kr * bh * (A + C - 0.25f);                                                                         \
            gcv[2] += kr * (cn[0] * A + bh * bh);                                                                        \
        }                                                                                                                \
        const float gc[3] = {gcv[0], gcv[1], gcv[2]};                                                                    \
        float gS[9], gJ[6];                                                                                              \
        conic_bwd<float>(S9, J, W, gc, gS, gJ);                                                                          \
        if (FILTER3D) {                                                                                                  \
            sigma_world_bwd_f3d<float>(qw, qx, qy, qz, e, v, vp, F, gS, gq, gs);                                         \
        } else {                                                                                                         \
            sigma_world_bwd<float>(qw, qx, qy, qz, s0, s1, s2, gS, gq, gs);                                              \
        }                                                                                                                \
        float gp_j[3], gp_uv[3] = {0.f, 0.f, 0.f};                                                                       \
        proj_jacobian_bwd<float>(px, py, pz, vc.K[0], vc.K[4], gJ, gp_j);                                                \
        project_uv_bwd<float>(px, py, pz, vc.K[0], vc.K[4], guv[0], guv[1], gp_uv);                                      \
        float gp[3] = {gp_j[0] + gp_uv[0], gp_j[1] + gp_uv[1], gp_j[2] + gp_uv[2]};                                      \
        if (DEPTH) gp[2] += gzc;                                                                                         \
        /* xyz_cam = W xyz + t  =>  grad_xyz = W^T grad_xyz_cam */                                                       \
_Pragma("unroll")                                                                                                        \
        for (int k = 0; k < 3; ++k) gx[k] = W[0 + k] * gp[0] + W[3 + k] * gp[1] + W[6 + k] * gp[2];                      \
        const float sg = sigmoid_torch(opl);                                                                             \
        if (ANTIALIAS) gov *= rho;       /* gradient on sigmoid(o) (3-D filter: on sigmoid(o) * coef) */                 \
        if (FILTER3D) {                                                                                                  \
            /* d coef / d s_k = coef (1 - t_k), 1 - t_k = F / v'_k (no cancellation); 0 where F == 0.  Where coef == 0 */ \
            /* the splat never contributed: gov == 0 and every term here is an exact, finite 0. */                       \
            const float gc = gov * sg * coef;                                                                            \
_Pragma("unroll")                                                                                                        \
            for (int k = 0; k < 3; ++k) gs[k] += gc * (F == 0.0f ? 0.0f : F / vp[k]);                                    \
            gov *= coef;                                                                                                 \
        }                                                                                                                \
        go = gov * ((1.0f - sg) * sg);  /* torch sigmoid_backward: grad * (1 - y) * y */                                 \
                                                                                                                         \
        const float gr[3] = {grv[0], grv[1], grv[2]};                                                                    \
        if (HAS_SH) {                                                                                                    \
            /* src/precompute_sh.cu:96-109, split into the DC column and the rest */                                     \
            float dx, dy, dz, Y[N_SH];                                                                                   \
            view_dir<float>(x, y, z, vc.cam[0], vc.cam[1], vc.cam[2], dx, dy, dz);                                       \
            sh_basis<float, N_SH>(dx, dy, dz, Y);                                                                        \
_Pragma("unroll")                                                                                                        \
            for (int c = 0; c < 3; ++c) {                                                                                \
                const float g = gr[c] * GSR_RSH0;                                                                        \
                gdc[c] = g * Y[0];                                                                                       \
_Pragma("unroll")                                                                                                        \
                for (int k = 1; k < N_SH; ++k) my_sh[c * NR + (k - 1)] = g * Y[k];                                       \
            }                                                                                                            \
        } else {                                                                                                         \
_Pragma("unroll")                                                                                                        \
            for (int c = 0; c < 3; ++c) gdc[c] = gr[c];                                                                  \
        }                                                                                                                \
    }

// Fused VJP of one view.  g_rows are the per-Gaussian sums produced by the render backward, one interleaved row per
// original gaussian.
template <int N_SH, bool HAS_SH, bool DEPTH, bool ANTIALIAS, bool FILTER3D>
__device__ __forceinline__ void preprocess_bwd(int N, const float* __restrict__ xyz, const float* __restrict__ quat,
                     const float* __restrict__ scale, const float* __restrict__ opa_logit,
                     const float* __restrict__ Tdev, const float* __restrict__ Kdev,
                     const float* __restrict__ camdev, const uint8_t* __restrict__ visible,
                     const float* __restrict__ g_rows, int rows_uv,
                     const float* __restrict__ g_uv_compact,
                     const uint64_t* __restrict__ scan, float* __restrict__ o_xyz,
                     float* __restrict__ o_quat, float* __restrict__ o_scale, float* __restrict__ o_opa,
                     float* __restrict__ o_dc, float* __restrict__ o_sh, int use_tma,
                     const float* __restrict__ filter3d) {
    constexpr int NR = N_SH - 1;
    constexpr int NR3 = HAS_SH ? 3 * NR : 1;
    // all outputs of the CTA's 128 gaussians are staged in shared memory and leave as six bulk stores
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
    float gx[3] = {0.f, 0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f}, gs[3] = {0.f, 0.f, 0.f}, go = 0.f,
          gdc[3] = {0.f, 0.f, 0.f};
    float* my_sh = s_sh + tid * NR3;
    bool vis = false;
    if (i < N) vis = visible[i] != 0;
    // every thread fetches its gaussian's inputs before the view constants are fetched (cooperatively): the
    // memory latencies overlap instead of queueing up behind one thread's 28 loads
    float x = 0.f, y = 0.f, z = 0.f, qw = 1.f, qx = 0.f, qy = 0.f, qz = 0.f, s0 = 0.f, s1 = 0.f, s2 = 0.f, opl = 0.f,
          gcv[3] = {0.f, 0.f, 0.f}, guv[2] = {0.f, 0.f}, gov = 0.f, grv[3] = {0.f, 0.f, 0.f}, gzc = 0.f, f = 0.f;
    if (vis) {
        if (FILTER3D) f = filter3d[i];
        x = xyz[i * 3 + 0]; y = xyz[i * 3 + 1]; z = xyz[i * 3 + 2];
        qw = quat[i * 4 + 0]; qx = quat[i * 4 + 1]; qy = quat[i * 4 + 2]; qz = quat[i * 4 + 3];
        s0 = scale[i * 3 + 0]; s1 = scale[i * 3 + 1]; s2 = scale[i * 3 + 2];
        opl = opa_logit[i];
        // interleaved rows: rgb3 opa | uv2 conic0 conic1 | conic2 pad3
        const float4* row = reinterpret_cast<const float4*>(g_rows + (size_t)i * GSR_GRAD_ROW_FLOATS);
        const float4 r0 = row[0], r1 = row[1];
        grv[0] = r0.x; grv[1] = r0.y; grv[2] = r0.z; gov = r0.w;
        // gradient on the projected mean = the render backward's sum (the row's uv, unless rows_uv is 0) + whatever
        // arrives on the COMPACT uv rasterize returned (g_uv_compact [M,2]; row = rank among the visible gaussians,
        // read off the forward's packed inclusive scan)
        if (rows_uv) { guv[0] = r1.x; guv[1] = r1.y; }
        gcv[0] = r1.z; gcv[1] = r1.w;
        if (DEPTH) {
            const float2 r2 = *reinterpret_cast<const float2*>(g_rows + (size_t)i * GSR_GRAD_ROW_FLOATS + 8);
            gcv[2] = r2.x;
            gzc = r2.y;
        } else {
            gcv[2] = g_rows[(size_t)i * GSR_GRAD_ROW_FLOATS + 8];
        }
        if (g_uv_compact != nullptr) {
            const size_t r = (size_t)(scan[i] >> 32) - 1;
            const float2 t = *reinterpret_cast<const float2*>(g_uv_compact + r * 2);
            guv[0] = __fadd_rn(guv[0], t.x);
            guv[1] = __fadd_rn(guv[1], t.y);
        }
    }
    load_view_cta(Tdev, Kdev, camdev, vc, HAS_SH);
    if (vis) GSR_PRE_BWD_VIEW else if (HAS_SH) {
#pragma unroll
        for (int k = 0; k < NR3; ++k) my_sh[k] = 0.f;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) { s_xyz[tid * 3 + k] = gx[k]; s_scale[tid * 3 + k] = gs[k]; s_dc[tid * 3 + k] = gdc[k]; }
    *reinterpret_cast<float4*>(s_quat + tid * 4) = make_float4(gq[0], gq[1], gq[2], gq[3]);
    s_opa[tid] = go;
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

}  // namespace gsr
