// gsr_preprocess.cuh — the per-Gaussian stages of the fused path and the view constants they read, shared by the
// single-view kernels (gsr_preprocess.cu, libgsr_b200.so), the multi-view kernels (gsr_batch.cu, libgsr_batch.so)
// the lens kernels (gsr_lens.cu), the pose-gradient kernels (gsr_pose.cu) and the rolling-shutter kernels
// (gsr_shutter.cu).  GSR_PRE_BWD_VIEW is one view's VJP for one gaussian;
// the single-view kernels store its result, the batched kernels add it up over the views.  The camera model enters
// only through the GSR_PROJECT / GSR_JACOBIAN hooks below.
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

// Camera-model hooks.  The per-gaussian bodies below name the camera model only through these macros.  The pinhole
// defaults expand to exactly the calls the bodies made before the hooks existed, so every pinhole kernel keeps its
// instructions; a translation unit that defines GSR_PROJECTION_HOOKS (and the macros) before including this header
// compiles the same bodies for another model (the hook sets of gsr_fisheye.cuh and gsr_distortion.cuh).
//   GSR_VIEW_PARAM                       extra trailing parameters of the bodies
//   GSR_VIEW_DECL                        extra CTA-wide view constants, next to `vc`
//   GSR_LOAD_VIEW(T, K, cam, view)       fill `vc` (and the extra constants) for view index `view`; ends with a barrier
//   GSR_PROJECT(px, py, pz, u, v)        the projected mean
//   GSR_CULL_MORE                        extra `| (...)` terms of the forward's cull
//   GSR_JACOBIAN(px, py, pz, J)          J = d(u, v) / d(px, py, pz), 2x3 row-major
//   GSR_JACOBIAN_BWD(px, py, pz, gJ, g)  g = contraction of dJ / dp with the gradient on J
//   GSR_PROJECT_BWD(px, py, pz, gu, gv, g)  g = (d(u, v) / dp)^T (gu, gv); may read the body's `J`
#ifndef GSR_PROJECTION_HOOKS
#define GSR_VIEW_PARAM
#define GSR_VIEW_DECL
#define GSR_LOAD_VIEW(T, K, cam, view) load_view_cta(T, K, cam, vc, HAS_SH)
#define GSR_PROJECT(px, py, pz, u, v) project_uv<float>(px, py, pz, vc.K[0], vc.K[2], vc.K[4], vc.K[5], u, v)
#define GSR_CULL_MORE
#define GSR_JACOBIAN(px, py, pz, J) proj_jacobian<float>(px, py, pz, vc.K[0], vc.K[4], J)
#define GSR_JACOBIAN_BWD(px, py, pz, gJ, g) proj_jacobian_bwd<float>(px, py, pz, vc.K[0], vc.K[4], gJ, g)
#define GSR_PROJECT_BWD(px, py, pz, gu, gv, g) project_uv_bwd<float>(px, py, pz, vc.K[0], vc.K[4], gu, gv, g)
#endif

// Pose-gradient hooks, empty by default: every kernel that does not define GSR_POSE_HOOKS keeps its instructions.
// gsr_pose.cuh defines them (gsr_pose.cu, libgsr_pose.so).
//   GSR_POSE_PARAM          extra trailing parameters of the backward bodies
//   GSR_POSE_DECL           per-thread pose accumulators, zero (single view: once; batched: per view)
//   GSR_POSE_VIEW           inside GSR_PRE_BWD_VIEW once gp, the gradient on the camera-frame mean, is complete
//   GSR_POSE_REDUCE(view)   after the view's `if (vis)` block, reached by every thread of the CTA
#ifndef GSR_POSE_HOOKS
#define GSR_POSE_PARAM
#define GSR_POSE_DECL
#define GSR_POSE_VIEW
#define GSR_POSE_REDUCE(view)
#endif

// Rolling-shutter hooks, empty by default: every kernel that does not define GSR_SHUTTER_HOOKS keeps its instructions.
// gsr_shutter.cuh defines them (gsr_shutter.cu, libgsr_shutter.so).
//   GSR_SHUTTER_PARAM           extra trailing parameters of the bodies (after GSR_VIEW_PARAM)
//   GSR_SHUTTER_LOAD(view)      per-thread shutter constants of view `view`, after GSR_LOAD_VIEW
//   GSR_SHUTTER_POINT(px, py, pz)  replaces the camera-frame mean p0 by p(tau*), the mean at its own line's time
//   GSR_SHUTTER_CULL            extra `| (...)` terms of the forward's cull
//   GSR_SHUTTER_W(W)            W <- W(tau*), once W holds the rotation of camera_T_world
//   GSR_SHUTTER_JACOBIAN(J)     after GSR_JACOBIAN: forms the Jacobian the covariance uses, GSR_SHUTTER_J
//   GSR_SHUTTER_J               that Jacobian (J: the lens's)
//   GSR_SHUTTER_BWD_J(gJ)       after conic_bwd: gJ <- the gradient on the lens's J
//   GSR_SHUTTER_GP(gp)          once gp holds the gradient on p: adds the terms of the shutter time
#ifndef GSR_SHUTTER_HOOKS
#define GSR_SHUTTER_PARAM
#define GSR_SHUTTER_LOAD(view)
#define GSR_SHUTTER_POINT(px, py, pz)
#define GSR_SHUTTER_CULL
#define GSR_SHUTTER_W(W)
#define GSR_SHUTTER_JACOBIAN(J)
#define GSR_SHUTTER_J J
#define GSR_SHUTTER_BWD_J(gJ)
#define GSR_SHUTTER_GP(gp)
#endif

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
        GSR_SHUTTER_POINT(px, py, pz)                                                                                    \
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
        GSR_JACOBIAN(px, py, pz, J);                                                                                     \
        GSR_SHUTTER_JACOBIAN(J)                                                                                          \
        W[0] = vc.T[0]; W[1] = vc.T[1]; W[2] = vc.T[2];                                                                  \
        W[3] = vc.T[4]; W[4] = vc.T[5]; W[5] = vc.T[6];                                                                  \
        W[6] = vc.T[8]; W[7] = vc.T[9]; W[8] = vc.T[10];                                                                 \
        GSR_SHUTTER_W(W)                                                                                                 \
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
            conic_from<float>(S9, GSR_SHUTTER_J, W, cn, nullptr);                                                        \
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
        conic_bwd<float>(S9, GSR_SHUTTER_J, W, gc, gS, gJ);                                                              \
        GSR_SHUTTER_BWD_J(gJ)                                                                                            \
        if (FILTER3D) {                                                                                                  \
            sigma_world_bwd_f3d<float>(qw, qx, qy, qz, e, v, vp, F, gS, gq, gs);                                         \
        } else {                                                                                                         \
            sigma_world_bwd<float>(qw, qx, qy, qz, s0, s1, s2, gS, gq, gs);                                              \
        }                                                                                                                \
        float gp_j[3], gp_uv[3] = {0.f, 0.f, 0.f};                                                                       \
        GSR_JACOBIAN_BWD(px, py, pz, gJ, gp_j);                                                                          \
        GSR_PROJECT_BWD(px, py, pz, guv[0], guv[1], gp_uv);                                                              \
        float gp[3] = {gp_j[0] + gp_uv[0], gp_j[1] + gp_uv[1], gp_j[2] + gp_uv[2]};                                      \
        if (DEPTH) gp[2] += gzc;                                                                                         \
        GSR_SHUTTER_GP(gp)                                                                                               \
        GSR_POSE_VIEW                                                                                                    \
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
                     const float* __restrict__ filter3d GSR_VIEW_PARAM GSR_SHUTTER_PARAM GSR_POSE_PARAM) {
    constexpr int NR = N_SH - 1;
    constexpr int NR3 = HAS_SH ? 3 * NR : 1;
    // all outputs of the CTA's 128 gaussians are staged in shared memory and leave as six bulk stores
    __shared__ ViewConsts vc;
    GSR_VIEW_DECL
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
    GSR_POSE_DECL
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
    GSR_LOAD_VIEW(Tdev, Kdev, camdev, 0);
    GSR_SHUTTER_LOAD(0)
    if (vis) GSR_PRE_BWD_VIEW else if (HAS_SH) {
#pragma unroll
        for (int k = 0; k < NR3; ++k) my_sh[k] = 0.f;
    }
    GSR_POSE_REDUCE(0)
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

// SH -> RGB exactly as src/precompute_sh.cu:29-56 evaluates it on cat(rgb_dc, sh_rest)
template <int N_SH>
__device__ __forceinline__ void sh_rgb_fused(const float* __restrict__ dc, const float* __restrict__ rest,
                                             float px, float py, float pz, const float* cam,
                                             float* __restrict__ out) {
    if (N_SH == 1) {
        out[0] = dc[0]; out[1] = dc[1]; out[2] = dc[2];
        return;
    }
    float dx, dy, dz, Y[N_SH];
    view_dir<float>(px, py, pz, cam[0], cam[1], cam[2], dx, dy, dz);
    sh_basis<float, N_SH>(dx, dy, dz, Y);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float acc = __fmaf_rn(Y[0], dc[c], 0.0f);
#pragma unroll
        for (int k = 1; k < N_SH; ++k) acc = __fmaf_rn(Y[k], rest[c * (N_SH - 1) + (k - 1)], acc);
        out[c] = __fmul_rn(acc, GSR_RSH0);
    }
}

#define GSR_PRE_FWD_PARAMS                                                                                         \
    int N, const float* __restrict__ xyz, const float* __restrict__ xyz_cam, int cam_first,                        \
        const float* __restrict__ quat, const float* __restrict__ scale, const float* __restrict__ opa_logit,      \
        const float* __restrict__ rgb_dc, const float* __restrict__ sh_rest, const float* __restrict__ Tdev,       \
        const float* __restrict__ Kdev, const float* __restrict__ camdev, float width, float height, float near_t, \
        float far_t, float pad, float mh, int ntx, int nty, uint32_t depth_base, float* __restrict__ records,      \
        uint32_t* __restrict__ zkey, uint8_t* __restrict__ visible, uint64_t* __restrict__ packed,                 \
        uint64_t* __restrict__ tile_mask, uint32_t* __restrict__ tile_win, int use_tma
#define GSR_PRE_FWD_FORWARD                                                                                        \
    N, xyz, xyz_cam, cam_first, quat, scale, opa_logit, rgb_dc, sh_rest, Tdev, Kdev, camdev, width, height, near_t, \
        far_t, pad, mh, ntx, nty, depth_base, records, zkey, visible, packed, tile_mask, tile_win, use_tma
// The fused per-gaussian forward of one view (gsr_preprocess.cu).
// ANTIALIAS: the record's opacity is sigmoid(o) * aa_rho(conic) (gsr_record.cuh); the culling bound tau' is formed
// from that compensated opacity
// FILTER3D: Mip-Splatting's 3-D filter, f = filter3d[i]: Sigma_world is formed from the variances exp(s)^2 + f^2 and
// the opacity is multiplied by coef before rho (gsr_record.cuh f3d_filter)
template <int N_SH, bool HAS_SH, bool ANTIALIAS, bool FILTER3D>
__device__ __forceinline__ void preprocess_fwd(GSR_PRE_FWD_PARAMS, const float* __restrict__ filter3d GSR_VIEW_PARAM GSR_SHUTTER_PARAM) {
    constexpr int NR3 = HAS_SH ? 3 * (N_SH - 1) : 1;
    __shared__ ViewConsts vc;
    GSR_VIEW_DECL
    __shared__ __align__(128) float s_sh[PRE_THREADS * NR3];       // SH coefficients of the CTA's gaussians
    __shared__ __align__(128) float s_rec[PRE_THREADS * REC];      // output records
    __shared__ __align__(8) uint64_t s_bar;
    const int tid = threadIdx.x;
    const int i0 = blockIdx.x * PRE_THREADS;
    const int cnt = min(PRE_THREADS, N - i0);
    const bool tma = use_tma && cnt == PRE_THREADS;
    // Latencies overlap instead of queueing up: the SH slice's bulk copy is issued first, every thread then
    // fetches its own gaussian's parameters, and only then the view constants are fetched (cooperatively).
    if (tid == 0 && HAS_SH && tma) {
        mbar_init(&s_bar, 1);
        fence_mbar_init();
        const uint32_t bytes = (uint32_t)(PRE_THREADS * NR3 * sizeof(float));
        mbar_arrive_expect_tx(&s_bar, bytes);
        tma_load_1d(s_sh, sh_rest + (size_t)i0 * NR3, bytes, &s_bar);
    }
    if (HAS_SH && !tma) coop_copy(s_sh, sh_rest + (size_t)i0 * NR3, cnt * NR3);
    const int i = i0 + tid;
    float x = 0.f, y = 0.f, z = 0.f, q0 = 1.f, q1 = 0.f, q2 = 0.f, q3 = 0.f, sc0 = 0.f, sc1 = 0.f, sc2 = 0.f,
          opl = 0.f, dc0 = 0.f, dc1 = 0.f, dc2 = 0.f;
    if (i < N) {
        x = xyz[i * 3 + 0]; y = xyz[i * 3 + 1]; z = xyz[i * 3 + 2];
        q0 = quat[i * 4 + 0]; q1 = quat[i * 4 + 1]; q2 = quat[i * 4 + 2]; q3 = quat[i * 4 + 3];
        sc0 = scale[i * 3 + 0]; sc1 = scale[i * 3 + 1]; sc2 = scale[i * 3 + 2];
        opl = opa_logit[i];
        dc0 = rgb_dc[i * 3 + 0]; dc1 = rgb_dc[i * 3 + 1]; dc2 = rgb_dc[i * 3 + 2];
    }
    GSR_LOAD_VIEW(Tdev, Kdev, camdev, 0);
    GSR_SHUTTER_LOAD(0)
    float rec[REC];
#pragma unroll
    for (int k = 0; k < REC; ++k) rec[k] = 0.0f;
    if (i < N) {
        float px, py, pz, u, v;
        if (xyz_cam != nullptr && i >= cam_first) {
            const float* pc = xyz_cam + (size_t)(i - cam_first) * 3;
            px = pc[0]; py = pc[1]; pz = pc[2];
        } else {
            transform_point<float>(vc.T, x, y, z, px, py, pz);
        }
        GSR_SHUTTER_POINT(px, py, pz)
        GSR_PROJECT(px, py, pz, u, v);
        // splat_py/rasterize.py:38-49 (strict compares, fp32)
        const bool culled = (pz < near_t) | (pz > far_t) | (u < -pad) | (u > width + pad) | (v < -pad) |
                            (v > height + pad) GSR_CULL_MORE GSR_SHUTTER_CULL;
        // visible => pz >= near > 0: float bits are monotone, and relative to bits(near) only a few low
        // bits are significant (shorter radix sort)
        zkey[i] = depth_base ? (__float_as_uint(pz) - depth_base) : depth_key(pz);
        // NaN coordinates compare false everywhere and would survive; the reference aborts on them
        // (splat_py/tile_culling.py:15-18) — treat as culled instead.
        const bool vis = !culled && (pz == pz) && (u == u) && (v == v);
        visible[i] = vis ? 1 : 0;
        uint64_t pk = 0ull;
        if (vis) {
            float S6[6], S9[9], J[6], W[9], conic[3], coef = 1.0f;
            if (FILTER3D) {
                const float f = filter3d[i];
                const float F = __fmul_rn(f, f);
                const float e0 = expf(sc0), e1 = expf(sc1), e2 = expf(sc2);
                const float v[3] = {__fmul_rn(e0, e0), __fmul_rn(e1, e1), __fmul_rn(e2, e2)};
                float vp[3], t[3];
                coef = f3d_filter(v, F, vp, t);
                sigma_world_var<float>(q0, q1, q2, q3, vp[0], vp[1], vp[2], S6);
            } else {
                sigma_world<float>(q0, q1, q2, q3, sc0, sc1, sc2, S6);
            }
            sym6_to_full(S6, S9);
            GSR_JACOBIAN(px, py, pz, J);
            GSR_SHUTTER_JACOBIAN(J)
            W[0] = vc.T[0]; W[1] = vc.T[1]; W[2] = vc.T[2];
            W[3] = vc.T[4]; W[4] = vc.T[5]; W[5] = vc.T[6];
            W[6] = vc.T[8]; W[7] = vc.T[9]; W[8] = vc.T[10];
            GSR_SHUTTER_W(W)
            conic_from<float>(S9, GSR_SHUTTER_J, W, conic, nullptr);

            float opa = sigmoid_torch(opl);
            if (FILTER3D) opa = __fmul_rn(opa, coef);
            if (ANTIALIAS) opa = __fmul_rn(opa, aa_rho(conic[0], conic[1], conic[2]));
            float dc[3] = {dc0, dc1, dc2};
            float col[3];
            if (HAS_SH) {
                if (tma) mbar_wait(&s_bar, 0);
                sh_rgb_fused<N_SH>(dc, s_sh + tid * NR3, x, y, z, vc.cam, col);  // stride 3*(N_SH-1): odd, no conflicts
            } else {
                col[0] = dc[0]; col[1] = dc[1]; col[2] = dc[2];
            }
            make_record(u, v, conic[0], conic[1], conic[2], opa, col[0], col[1], col[2], rec);

            // tiles touched (src/tile_culling.cu:139-176)
            Obb ob;
            compute_obb(u, v, rec[R_A], __fmul_rn(rec[R_B2], 0.5f), rec[R_C], mh, ob);
            int x0, x1, y0, y1, c = 0;
            tile_window(u, v, ob.radius_tiles, ntx, nty, x0, x1, y0, y1);
            // The tiles hit are remembered as a bit mask over the window (bit = (tx - x0) * height + (ty - y0), the
            // enumeration order) when the window has at most 64 tiles — footprints up to 3 sigma = 48 px — so that
            // the pair emission does not repeat the OBB / separating-axis tests (gsr_binning.cu); larger windows
            // are flagged and re-tested there.
            const int wx = x1 - x0, wy = y1 - y0;
            const bool small = (wx * wy <= 64) & (x0 < 256) & (y0 < 256);
            uint64_t hits = 0ull;
            for (int tx = x0; tx < x1; ++tx) {
                const float left = __fmul_rn(__int2float_rn(tx), 16.0f);
                const float right = __fmul_rn(__int2float_rn(tx + 1), 16.0f);
                for (int ty = y0; ty < y1; ++ty) {
                    const float top = __fmul_rn(__int2float_rn(ty), 16.0f);
                    const float bottom = __fmul_rn(__int2float_rn(ty + 1), 16.0f);
                    if (obb_hits_tile(ob, left, right, top, bottom)) {
                        ++c;
                        if (small) hits |= 1ull << ((tx - x0) * wy + (ty - y0));
                    }
                }
            }
            if (tile_mask != nullptr) {
                tile_mask[i] = hits;
                tile_win[i] = small ? ((uint32_t)x0 | ((uint32_t)y0 << 8) | ((uint32_t)wx << 16) | ((uint32_t)wy << 24))
                                    : 0xffffffffu;
            }
            pk = (1ull << 32) | (uint64_t)(uint32_t)c;
        }
        packed[i] = pk;
    }
    // records leave through shared memory: one 6 KB bulk store per CTA instead of 48-byte strided stores
    float4* sr = reinterpret_cast<float4*>(s_rec + tid * REC);
    sr[0] = make_float4(rec[0], rec[1], rec[2], rec[3]);
    sr[1] = make_float4(rec[4], rec[5], rec[6], rec[7]);
    sr[2] = make_float4(rec[8], rec[9], rec[10], rec[11]);
    if (tma) {
        fence_proxy_async_smem();
        __syncthreads();
        if (tid == 0) {
            tma_store_1d(records + (size_t)i0 * REC, s_rec, (uint32_t)(PRE_THREADS * REC * sizeof(float)));
            tma_store_commit_and_wait();
        }
    } else {
        __syncthreads();
        coop_copy(records + (size_t)i0 * REC, s_rec, cnt * REC);
    }
    if (HAS_SH && tma && tid == 0) mbar_wait(&s_bar, 0);  // never exit with the SH load still in flight
}

// The per-gaussian backward of C views in one pass (gsr_batch.cu).  A CTA takes 128 gaussians, reads their parameters
// once and walks the views in order.  For every view that sees a gaussian it forms that view's VJP with the
// single-view kernel's own statement block (GSR_PRE_BWD_VIEW) and adds it to the running sums with one rounded fp32
// add, so the result is the view-order sum of the single-view gradients bit for bit (up to the sign of zero).  The
// sums of the SH rest coefficients live in the shared-memory staging the single-view kernel stores from; everything
// leaves once, by the same bulk stores.
template <int N_SH, bool HAS_SH, bool DEPTH, bool ANTIALIAS, bool FILTER3D>
__device__ __forceinline__ void batch_preprocess_bwd(
    int C, int N, const float* __restrict__ xyz, const float* __restrict__ quat, const float* __restrict__ scale,
    const float* __restrict__ opa_logit, const float* __restrict__ Tdev, const float* __restrict__ Kdev,
    const float* __restrict__ camdev, const uint8_t* __restrict__ visible, const float* __restrict__ g_rows,
    int rows_uv, const float* __restrict__ g_uv_compact, const uint64_t* __restrict__ scan, float* __restrict__ o_xyz,
    float* __restrict__ o_quat, float* __restrict__ o_scale, float* __restrict__ o_opa, float* __restrict__ o_dc,
    float* __restrict__ o_sh, int use_tma, const float* __restrict__ filter3d GSR_VIEW_PARAM GSR_SHUTTER_PARAM GSR_POSE_PARAM) {
    constexpr int NR = N_SH - 1;
    constexpr int NR3 = HAS_SH ? 3 * NR : 1;
    __shared__ ViewConsts vc;
    GSR_VIEW_DECL
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
        GSR_POSE_DECL
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
        GSR_LOAD_VIEW(Tdev + 16 * c, Kdev + 9 * c, camdev != nullptr ? camdev + 3 * c : nullptr, c);
        GSR_SHUTTER_LOAD(c)
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
        GSR_POSE_REDUCE(c)
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

}  // namespace gsr
