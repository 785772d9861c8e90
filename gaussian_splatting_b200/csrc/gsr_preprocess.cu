// gsr_preprocess.cu — the fused per-Gaussian stage behind rasterize().
//
// One kernel replaces, for every Gaussian of the scene, the reference's chain
//   transform_points_torch        splat_py/utils.py:60-72
//   CameraPointProjection         src/projection.cu:8-19
//   frustum cull + 8 mask gathers splat_py/rasterize.py:33-75
//   sigmoid(opacity)              splat_py/rasterize.py:60-62
//   ComputeSigmaWorld             src/projection.cu:56-109
//   ComputeProjectionJacobian     src/projection.cu:154-175
//   ComputeConic                  src/projection.cu:213-257
//   cat(rgb, sh) + PrecomputeRGBFromSH   splat_py/rasterize.py:89-93, src/precompute_sh.cu:7-58
//   compute_num_splats_kernel     src/tile_culling.cu:124-177
// and writes one 48-byte splat record, a depth key, a visibility flag and the
// tiles-touched count per Gaussian.  No Sigma_world / J intermediates reach HBM.
// The backward kernel is the fused VJP of the same chain (SURVEY.md Appendix A).
#include <cub/cub.cuh>

#include "gsr_preprocess.cuh"

namespace gsr {

__global__ void k_camera_centre(const float* __restrict__ T, float* __restrict__ cam) {
    if (threadIdx.x == 0 && blockIdx.x == 0) camera_centre(T, cam);
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
// ANTIALIAS: the record's opacity is sigmoid(o) * aa_rho(conic) (gsr_record.cuh); the culling bound tau' is formed
// from that compensated opacity
// FILTER3D: Mip-Splatting's 3-D filter, f = filter3d[i]: Sigma_world is formed from the variances exp(s)^2 + f^2 and
// the opacity is multiplied by coef before rho (gsr_record.cuh f3d_filter)
template <int N_SH, bool HAS_SH, bool ANTIALIAS, bool FILTER3D>
__device__ __forceinline__ void preprocess_fwd(GSR_PRE_FWD_PARAMS, const float* __restrict__ filter3d) {
    constexpr int NR3 = HAS_SH ? 3 * (N_SH - 1) : 1;
    __shared__ ViewConsts vc;
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
    load_view_cta(Tdev, Kdev, camdev, vc, HAS_SH);
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
        project_uv<float>(px, py, pz, vc.K[0], vc.K[2], vc.K[4], vc.K[5], u, v);
        // splat_py/rasterize.py:38-49 (strict compares, fp32)
        const bool culled = (pz < near_t) | (pz > far_t) | (u < -pad) | (u > width + pad) | (v < -pad) |
                            (v > height + pad);
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
            proj_jacobian<float>(px, py, pz, vc.K[0], vc.K[4], J);
            W[0] = vc.T[0]; W[1] = vc.T[1]; W[2] = vc.T[2];
            W[3] = vc.T[4]; W[4] = vc.T[5]; W[5] = vc.T[6];
            W[6] = vc.T[8]; W[7] = vc.T[9]; W[8] = vc.T[10];
            conic_from<float>(S9, J, W, conic, nullptr);

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

template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, 7) k_preprocess_fwd(GSR_PRE_FWD_PARAMS) {
    preprocess_fwd<N_SH, HAS_SH, false, false>(GSR_PRE_FWD_FORWARD, nullptr);
}
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, 7) k_preprocess_fwd_aa(GSR_PRE_FWD_PARAMS) {
    preprocess_fwd<N_SH, HAS_SH, true, false>(GSR_PRE_FWD_FORWARD, nullptr);
}
#ifndef GSR_PRE_FWD_F3D_MINB
#define GSR_PRE_FWD_F3D_MINB 7
#endif
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_FWD_F3D_MINB)
    k_preprocess_fwd_f3d(GSR_PRE_FWD_PARAMS, const float* __restrict__ filter3d) {
    preprocess_fwd<N_SH, HAS_SH, false, true>(GSR_PRE_FWD_FORWARD, filter3d);
}
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_FWD_F3D_MINB)
    k_preprocess_fwd_aa_f3d(GSR_PRE_FWD_PARAMS, const float* __restrict__ filter3d) {
    preprocess_fwd<N_SH, HAS_SH, true, true>(GSR_PRE_FWD_FORWARD, filter3d);
}
#undef GSR_PRE_FWD_PARAMS
#undef GSR_PRE_FWD_FORWARD

// Fused VJP (preprocess_bwd, gsr_preprocess.cuh).  g_rows are the per-Gaussian sums produced by the render
// backward, one interleaved row per original gaussian.
#ifndef GSR_PRE_BWD_MINB
#define GSR_PRE_BWD_MINB 6
#endif
// the anti-aliased backward re-forms the conic for rho's gradient: at 6 CTAs per SM (80 registers) that spills, at 5
// it does not
#ifndef GSR_PRE_BWD_AA_MINB
#define GSR_PRE_BWD_AA_MINB 5
#endif

#define GSR_PRE_BWD_PARAMS                                                                                          \
    int N, const float* __restrict__ xyz, const float* __restrict__ quat, const float* __restrict__ scale,          \
        const float* __restrict__ opa_logit, const float* __restrict__ Tdev, const float* __restrict__ Kdev,        \
        const float* __restrict__ camdev, const uint8_t* __restrict__ visible, const float* __restrict__ g_rows,    \
        int rows_uv, const float* __restrict__ g_uv_compact,                                                         \
        const uint64_t* __restrict__ scan, float* __restrict__ o_xyz, float* __restrict__ o_quat,                   \
        float* __restrict__ o_scale, float* __restrict__ o_opa, float* __restrict__ o_dc, float* __restrict__ o_sh, \
        int use_tma
#define GSR_PRE_BWD_FORWARD                                                                                      \
    N, xyz, quat, scale, opa_logit, Tdev, Kdev, camdev, visible, g_rows, rows_uv, g_uv_compact, scan, o_xyz, o_quat, \
        o_scale, o_opa, o_dc, o_sh, use_tma
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_BWD_MINB) k_preprocess_bwd(GSR_PRE_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, false, false, false>(GSR_PRE_BWD_FORWARD, nullptr);
}
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_BWD_MINB) k_preprocess_bwd_depth(GSR_PRE_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, true, false, false>(GSR_PRE_BWD_FORWARD, nullptr);
}
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_BWD_AA_MINB) k_preprocess_bwd_aa(GSR_PRE_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, false, true, false>(GSR_PRE_BWD_FORWARD, nullptr);
}
template <int N_SH, bool HAS_SH>
__global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_BWD_AA_MINB) k_preprocess_bwd_depth_aa(GSR_PRE_BWD_PARAMS) {
    preprocess_bwd<N_SH, HAS_SH, true, true, false>(GSR_PRE_BWD_FORWARD, nullptr);
}
#ifndef GSR_PRE_BWD_F3D_MINB
#define GSR_PRE_BWD_F3D_MINB 5
#endif
#define GSR_PRE_BWD_F3D_KERNEL(name, depth, aa)                                                                    \
    template <int N_SH, bool HAS_SH>                                                                             \
    __global__ void __launch_bounds__(PRE_THREADS, GSR_PRE_BWD_F3D_MINB)                                         \
        name(GSR_PRE_BWD_PARAMS, const float* __restrict__ filter3d) {                                           \
        preprocess_bwd<N_SH, HAS_SH, depth, aa, true>(GSR_PRE_BWD_FORWARD, filter3d);                            \
    }
GSR_PRE_BWD_F3D_KERNEL(k_preprocess_bwd_f3d, false, false)
GSR_PRE_BWD_F3D_KERNEL(k_preprocess_bwd_depth_f3d, true, false)
GSR_PRE_BWD_F3D_KERNEL(k_preprocess_bwd_aa_f3d, false, true)
GSR_PRE_BWD_F3D_KERNEL(k_preprocess_bwd_depth_aa_f3d, true, true)
#undef GSR_PRE_BWD_F3D_KERNEL
#undef GSR_PRE_BWD_PARAMS
#undef GSR_PRE_BWD_FORWARD

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// GSR_MODE_ABSGRAD only changes the render backward (row slots 10-11, which the per-gaussian backward does not read)
constexpr int KNOWN_MODES = GSR_MODE_DEPTH_ALPHA | GSR_MODE_ANTIALIASED | GSR_MODE_ABSGRAD | GSR_MODE_FILTER3D;

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_camera_centre(const float* camera_T_world, float* centre, void* stream) {
    if (camera_T_world == nullptr || centre == nullptr) return GSR_ERR_BAD_ARG;
    k_camera_centre<<<1, 32, 0, (cudaStream_t)stream>>>(camera_T_world, centre);
    return (int)cudaGetLastError();
}

size_t gsr_preprocess_temp_bytes(int N) {
    size_t b = 0;
    cub::DeviceScan::InclusiveSum((void*)nullptr, b, (uint64_t*)nullptr, (uint64_t*)nullptr, N > 0 ? N : 1);
    return align256(b) + align256(sizeof(uint64_t) * (size_t)(N > 0 ? N : 1));
}

int gsr_preprocess_forward(int mode, int N, int n_sh_rest, const float* xyz, const float* xyz_camera_frame,
                           int cam_first, const float* quaternion, const float* scale, const float* opacity_logit,
                           const float* filter3d, const float* rgb_dc, const float* sh_rest,
                           const float* camera_T_world, const float* K,
                           const float* camera_centre, int H, int W, float near_thresh, float far_thresh,
                           float cull_mask_padding, float mh_dist, uint32_t depth_base, float* records,
                           uint32_t* depth_key, uint8_t* visible, uint64_t* scan, uint64_t* tile_mask,
                           uint32_t* tile_win, void* temp, size_t temp_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if ((mode & ~KNOWN_MODES) != 0) return GSR_ERR_BAD_ARG;
    if (((mode & GSR_MODE_FILTER3D) != 0) != (filter3d != nullptr)) return GSR_ERR_BAD_ARG;
    if (N <= 0) return GSR_OK;
    if (temp_bytes < gsr_preprocess_temp_bytes(N)) return GSR_ERR_BAD_ARG;
    if ((tile_mask == nullptr) != (tile_win == nullptr)) return GSR_ERR_BAD_ARG;
    size_t scan_bytes = 0;
    cub::DeviceScan::InclusiveSum((void*)nullptr, scan_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, N);
    uint64_t* packed = reinterpret_cast<uint64_t*>((char*)temp + align256(scan_bytes));
    const int ntx = (W + TILE - 1) / TILE, nty = (H + TILE - 1) / TILE;
    const dim3 grid((N + PRE_THREADS - 1) / PRE_THREADS), block(PRE_THREADS);
    const int use_tma = (aligned16(records) && (sh_rest == nullptr || aligned16(sh_rest))) ? 1 : 0;
#define GSR_PRE_ARGS                                                                              \
    N, xyz, xyz_camera_frame, cam_first, quaternion, scale, opacity_logit, rgb_dc, sh_rest, camera_T_world, K, \
        camera_centre, (float)W, (float)H,                                                                 \
        near_thresh, far_thresh, cull_mask_padding, mh_dist, ntx, nty, depth_base, records, depth_key, visible, \
        packed, tile_mask, tile_win, use_tma
#define GSR_PRE_FWD_F3D_SWITCH(kernel)                                                                  \
    switch (n_sh_rest) {                                                                                \
        case 0: kernel<1, false><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;                \
        case 3: kernel<4, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;                 \
        case 8: kernel<9, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;                 \
        case 15: kernel<16, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;               \
        default: return GSR_ERR_UNSUPPORTED;                                                            \
    }
    if ((mode & GSR_MODE_FILTER3D) && (mode & GSR_MODE_ANTIALIASED)) {
        GSR_PRE_FWD_F3D_SWITCH(k_preprocess_fwd_aa_f3d)
    } else if (mode & GSR_MODE_FILTER3D) {
        GSR_PRE_FWD_F3D_SWITCH(k_preprocess_fwd_f3d)
    } else if (mode & GSR_MODE_ANTIALIASED) {
        switch (n_sh_rest) {
            case 0: k_preprocess_fwd_aa<1, false><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 3: k_preprocess_fwd_aa<4, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 8: k_preprocess_fwd_aa<9, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 15: k_preprocess_fwd_aa<16, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            default: return GSR_ERR_UNSUPPORTED;
        }
    } else {
        switch (n_sh_rest) {
            case 0: k_preprocess_fwd<1, false><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 3: k_preprocess_fwd<4, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 8: k_preprocess_fwd<9, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            case 15: k_preprocess_fwd<16, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;
            default: return GSR_ERR_UNSUPPORTED;
        }
    }
#undef GSR_PRE_FWD_F3D_SWITCH
#undef GSR_PRE_ARGS
    cudaError_t e = cub::DeviceScan::InclusiveSum(temp, scan_bytes, packed, scan, N, st);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

int gsr_preprocess_backward(int mode, int N, int n_sh_rest, const float* xyz, const float* quaternion,
                            const float* scale, const float* opacity_logit, const float* filter3d,
                            const float* camera_T_world,
                            const float* K, const float* camera_centre, const uint8_t* visible,
                            const float* grad_rows, int use_rows_uv, const float* grad_uv_compact, const uint64_t* scan,
                            float* g_xyz, float* g_quaternion, float* g_scale, float* g_opacity_logit, float* g_rgb_dc,
                            float* g_sh_rest, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if ((mode & ~KNOWN_MODES) != 0) return GSR_ERR_BAD_ARG;
    if (((mode & GSR_MODE_FILTER3D) != 0) != (filter3d != nullptr)) return GSR_ERR_BAD_ARG;
    if (N <= 0) return GSR_OK;
    if (grad_rows == nullptr || !aligned16(grad_rows)) return GSR_ERR_BAD_ARG;
    if (grad_uv_compact != nullptr && scan == nullptr) return GSR_ERR_BAD_ARG;
    const dim3 grid((N + PRE_THREADS - 1) / PRE_THREADS), block(PRE_THREADS);
    const int use_tma = (aligned16(g_xyz) && aligned16(g_quaternion) && aligned16(g_scale) &&
                         aligned16(g_opacity_logit) && aligned16(g_rgb_dc) &&
                         (g_sh_rest == nullptr || aligned16(g_sh_rest)))
                            ? 1
                            : 0;
#define GSR_PRE_ARGS                                                                                   \
    N, xyz, quaternion, scale, opacity_logit, camera_T_world, K, camera_centre, visible, grad_rows, use_rows_uv, \
        grad_uv_compact, scan, g_xyz, g_quaternion, g_scale, g_opacity_logit, g_rgb_dc, g_sh_rest, use_tma
#define GSR_PRE_BWD_SWITCH(kernel)                                                      \
    switch (n_sh_rest) {                                                                \
        case 0: kernel<1, false><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;          \
        case 3: kernel<4, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;           \
        case 8: kernel<9, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;           \
        case 15: kernel<16, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS); break;         \
        default: return GSR_ERR_UNSUPPORTED;                                            \
    }
    const bool depth = (mode & GSR_MODE_DEPTH_ALPHA) != 0, antialiased = (mode & GSR_MODE_ANTIALIASED) != 0;
    if (mode & GSR_MODE_FILTER3D) {
#define GSR_PRE_BWD_F3D_SWITCH(kernel)                                                      \
    switch (n_sh_rest) {                                                                    \
        case 0: kernel<1, false><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;    \
        case 3: kernel<4, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;     \
        case 8: kernel<9, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;     \
        case 15: kernel<16, true><<<grid, block, 0, st>>>(GSR_PRE_ARGS, filter3d); break;   \
        default: return GSR_ERR_UNSUPPORTED;                                                \
    }
        if (antialiased && depth) {
            GSR_PRE_BWD_F3D_SWITCH(k_preprocess_bwd_depth_aa_f3d)
        } else if (antialiased) {
            GSR_PRE_BWD_F3D_SWITCH(k_preprocess_bwd_aa_f3d)
        } else if (depth) {
            GSR_PRE_BWD_F3D_SWITCH(k_preprocess_bwd_depth_f3d)
        } else {
            GSR_PRE_BWD_F3D_SWITCH(k_preprocess_bwd_f3d)
        }
#undef GSR_PRE_BWD_F3D_SWITCH
    } else if (antialiased && depth) {
        GSR_PRE_BWD_SWITCH(k_preprocess_bwd_depth_aa)
    } else if (antialiased) {
        GSR_PRE_BWD_SWITCH(k_preprocess_bwd_aa)
    } else if (depth) {
        GSR_PRE_BWD_SWITCH(k_preprocess_bwd_depth)
    } else {
        GSR_PRE_BWD_SWITCH(k_preprocess_bwd)
    }
#undef GSR_PRE_BWD_SWITCH
#undef GSR_PRE_ARGS
    return (int)cudaGetLastError();
}

}  // extern "C"
