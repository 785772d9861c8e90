// gsr_surfels.cuh — the bodies of the 2-D Gaussian surfel kernels (DESIGN.md 3.25, 3.26), shared by the pinhole
// kernels of gsr_surfels.cu (libgsr_surfels.so) and the lens kernels of gsr_surfels_lens.cu (libgsr_surfels_lens.so).
//
// LENS 0 is the pinhole (M = K M', (u_c, v_c) the pinhole projection, pixel rays (x, y, 1)); LENS 1 / 2 the fisheye and
// OPENCV models of gsr_fisheye.cuh / gsr_distortion.cuh (the record holds M', (u_c, v_c) the lens projection, pixel
// rays from the ray map).  Every lens-dependent step is an `if constexpr`, so the pinhole instructions are the ones
// the pinhole kernels had before the lenses.
#pragma once
#include "gsr_common.cuh"
#include "gsr_distortion.cuh"
#include "gsr_fisheye.cuh"
#include "gsr_math.cuh"
#include "gsr_math_bwd.cuh"
#include "gsr_preprocess.cuh"
#include "gsr_surfels_lens.cuh"
#include "../../include/gsr_surfels.h"

namespace gsr {
namespace surfel {

constexpr int SF = GSR_SURFEL_REC_FLOATS;
constexpr int SG = GSR_SURFEL_GRAD_FLOATS;
// record slots
enum { S_U = 0, S_V = 1, S_OPA = 2, S_PZ = 3, S_M = 4, S_C = 13, S_N = 16 };
// gradient row slots
enum { G_M = 0, G_OPA = 9, G_C = 10, G_N = 13, G_UC = 16, G_PZ = 18 };
constexpr int PRE = 128;      // gaussians per CTA of the per-gaussian kernels
constexpr int PIX = 256;      // pixels (threads) per CTA of the tile kernels
constexpr int BATCH = 128;    // surfel records staged per batch
constexpr float ALPHA_MIN = 1.0f / 255.0f;
constexpr int LENS_CONSTS = 6;  // the larger of GSR_FISHEYE_CONSTS and GSR_DISTORTION_CONSTS

// One pixel's intersection with one surfel.  Every operation is pinned, so the forward and the backward (separate
// kernels) take the same skip decisions and get the same alpha for every (pixel, surfel).
struct Hit {
    float hx[3], hy[3];  // d_x M2 - d_z M0, d_y M2 - d_z M1 (pinhole: x M2 - M0, y M2 - M1)
    float c2, a, b;      // c = hx x hy; (a, b) = (c0, c1) / c2
    float dx, dy;        // (x, y) - (u_c, v_c)
    float G, alpha, z;   // exp(-rho / 2), min(0.99, opacity G), camera z of the intersection (or p_z)
    bool use3;           // rho = a^2 + b^2 (else the low-pass filter's 2 |d|^2)
};

// RAYS: the pixel's ray d from the ray map (a ray of d = 0 gives c2 = 0: no hit)
template <bool RAYS>
__device__ __forceinline__ bool intersect(const float* __restrict__ r, float x, float y, const float* d, float r2,
                                          Hit& h) {
    const float* M = r + S_M;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if constexpr (RAYS) {
            h.hx[k] = __fmaf_rn(d[0], M[6 + k], -__fmul_rn(d[2], M[k]));
            h.hy[k] = __fmaf_rn(d[1], M[6 + k], -__fmul_rn(d[2], M[3 + k]));
        } else {
            h.hx[k] = __fmaf_rn(x, M[6 + k], -M[k]);
            h.hy[k] = __fmaf_rn(y, M[6 + k], -M[3 + k]);
        }
    }
    const float c0 = __fmaf_rn(h.hx[1], h.hy[2], -__fmul_rn(h.hx[2], h.hy[1]));
    const float c1 = __fmaf_rn(h.hx[2], h.hy[0], -__fmul_rn(h.hx[0], h.hy[2]));
    h.c2 = __fmaf_rn(h.hx[0], h.hy[1], -__fmul_rn(h.hx[1], h.hy[0]));
    if (h.c2 == 0.0f) return false;
    const float ic = __frcp_rn(h.c2);
    h.a = __fmul_rn(c0, ic);
    h.b = __fmul_rn(c1, ic);
    const float rho3 = __fmaf_rn(h.a, h.a, __fmul_rn(h.b, h.b));
    h.dx = __fsub_rn(x, r[S_U]);
    h.dy = __fsub_rn(y, r[S_V]);
    const float rho2 = __fmul_rn(2.0f, __fmaf_rn(h.dx, h.dx, __fmul_rn(h.dy, h.dy)));
    h.use3 = rho3 <= rho2;
    const float rho = h.use3 ? rho3 : rho2;
    if (!(rho <= r2)) return false;
    h.G = __expf(__fmul_rn(-0.5f, rho));
    h.alpha = fminf(0.99f, __fmul_rn(r[S_OPA], h.G));
    if (h.alpha < ALPHA_MIN) return false;
    h.z = h.use3 ? __fmaf_rn(M[6], h.a, __fmaf_rn(M[7], h.b, M[8])) : r[S_PZ];
    return true;
}

// the distortion's normalised depth m = m_scale (1 - near / z)
__device__ __forceinline__ float ndc_depth(float z, float near_t, float ms) {
    return __fmul_rn(ms, __fsub_rn(1.0f, __fdiv_rn(near_t, z)));
}

__device__ __forceinline__ int pair_id(const uint64_t* __restrict__ keys, int id_bits, const int32_t* __restrict__ ids,
                                       int p) {
    return keys != nullptr ? (int)(keys[p] & ((1ull << id_bits) - 1ull)) : ids[p];
}

// Rc = W R (row-major), W the rotation of camera_T_world (row-major 4x4)
__device__ __forceinline__ void camera_rotation(const float* __restrict__ T, const float* __restrict__ R,
                                                float* __restrict__ Rc) {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            Rc[r * 3 + c] = __fmaf_rn(T[r * 4 + 2], R[6 + c], __fmaf_rn(T[r * 4 + 1], R[3 + c], __fmul_rn(T[r * 4], R[c])));
}

// the lens's projected centre and its fold cull (gsr_fisheye.cuh / gsr_distortion.cuh, as the lens preprocess does)
template <int LENS>
__device__ __forceinline__ bool lens_project(float px, float py, float pz, const float* K, const float* kc, float& u,
                                             float& v) {
    if constexpr (LENS == GSR_SURFEL_LENS_FISHEYE) {
        float theta;
        fisheye_project(px, py, pz, K[0], K[2], K[4], K[5], kc, u, v, theta);
        return theta >= kc[4];
    } else {
        float s;
        distortion_project(px, py, pz, K[0], K[2], K[4], K[5], kc, u, v, s);
        return s >= kc[5];
    }
}

// J = d(u, v) / dp of the lens at p (row-major 2x3)
template <int LENS>
__device__ __forceinline__ void lens_jacobian(float px, float py, float pz, const float* K, const float* kc, float* J) {
    if constexpr (LENS == GSR_SURFEL_LENS_FISHEYE) fisheye_jacobian(px, py, pz, K[0], K[4], kc, J);
    else distortion_jacobian(px, py, pz, K[0], K[4], kc, J);
}

// compute_obb(u, v, a, 0, c, mh, o) (gsr_math.cuh), operation for operation, with the box's angle (0 or pi/2) taken
// before cosf / sinf: each then folds to the constant gsr_emit_keys computes, and no argument-reduction path through
// local memory is left in the kernel (the lens kernels' fp64 binning bound keeps ptxas from removing it)
__device__ __forceinline__ void axis_obb(float u, float v, float a, float c, float mh_dist, Obb& o) {
    using A = Ar<float>;
    const float b = 0.0f;
    const float d = A::sub(a, c);
    const float disc = A::fma(b, b, A::mul(A::mul(d, d), 0.25f));
    const float right = A::sqrt(disc);
    const float s = A::add(a, c);
    const float l1 = A::fma(s, 0.5f, right);
    const float l2 = A::fma(s, 0.5f, -right);
    const float r_major = A::mul(A::sqrt(l1), mh_dist);
    const float r_minor = A::mul(A::sqrt(l2), mh_dist);
    const bool major_x = a >= c;
    const float ct = major_x ? cosf(0.0f) : cosf(1.5707963705062866211f);
    const float st = major_x ? sinf(0.0f) : sinf(1.5707963705062866211f);
    const float t_mc = A::mul(ct, r_minor);
    const float t_ms = A::mul(r_minor, st);
    o.c[0] = A::add(u, A::fma(ct, -r_major, t_ms));
    o.c[1] = A::add(v, A::fma(-r_major, st, -t_mc));
    o.c[2] = A::add(u, A::fma(ct, r_major, t_ms));
    o.c[3] = A::add(v, A::fma(r_major, st, -t_mc));
    o.c[4] = A::add(u, A::fma(ct, -r_major, -t_ms));
    o.c[5] = A::add(v, A::fma(-r_major, st, t_mc));
    o.c[6] = A::add(u, A::fma(ct, r_major, -t_ms));
    o.c[7] = A::add(v, A::fma(r_major, st, t_mc));
    o.radius_tiles = (int)A::add(ceilf(A::mul(r_major, 0.0625f)), 1.0f);
    o.min_x = fminf(fminf(o.c[0], o.c[2]), fminf(o.c[4], o.c[6]));
    o.max_x = fmaxf(fmaxf(o.c[0], o.c[2]), fmaxf(o.c[4], o.c[6]));
    o.min_y = fminf(fminf(o.c[1], o.c[3]), fminf(o.c[5], o.c[7]));
    o.max_y = fmaxf(fmaxf(o.c[1], o.c[3]), fmaxf(o.c[5], o.c[7]));
    o.ax = A::sub(o.c[2], o.c[0]);
    o.ay = A::sub(o.c[3], o.c[1]);
    const float pr = A::fma(o.c[2], o.ax, A::mul(o.c[3], o.ay));
    const float pl = A::fma(o.c[0], o.ax, A::mul(o.c[1], o.ay));
    o.amin = fminf(pr, pl);
    o.amax = fmaxf(pr, pl);
    o.mx = A::sub(o.c[2], o.c[6]);
    o.my = A::sub(o.c[3], o.c[7]);
    const float pt = A::fma(o.c[2], o.mx, A::mul(o.c[3], o.my));
    const float pb = A::fma(o.c[6], o.mx, A::mul(o.c[7], o.my));
    o.mmin = fminf(pt, pb);
    o.mmax = fmaxf(pt, pb);
}

// ---- per-gaussian forward ---------------------------------------------------------------------------------------------
// skc: the lens constants in shared memory (LENS > 0), filled by the caller before the body's barrier
template <int N_SH, int LENS>
__device__ __forceinline__ void surfel_fwd(int N, const float* __restrict__ xyz, const float* __restrict__ xyz_cam,
                                           int cam_first, const float* __restrict__ quat,
                                           const float* __restrict__ scale, const float* __restrict__ opa_logit,
                                           const float* __restrict__ rgb_dc, const float* __restrict__ sh_rest,
                                           const float* __restrict__ Tdev, const float* __restrict__ Kdev,
                                           const float* __restrict__ camdev, float width, float height, float near_t,
                                           float far_t, float pad, float mh, int ntx, int nty, uint32_t depth_base,
                                           float* __restrict__ surfels, float* __restrict__ bins,
                                           uint32_t* __restrict__ zkey, uint8_t* __restrict__ visible,
                                           uint64_t* __restrict__ packed, uint64_t* __restrict__ tile_mask,
                                           uint32_t* __restrict__ tile_win, const float* skc) {
    __shared__ float sT[16], sK[9], sc[3];
    const int t = threadIdx.x;
    if (t < 16) sT[t] = Tdev[t];
    else if (t < 25) sK[t - 16] = Kdev[t - 16];
    else if (t < 28 && N_SH > 1) sc[t - 25] = camdev[t - 25];
    __syncthreads();
    const int i = blockIdx.x * PRE + t;
    if (i >= N) return;
    const float x = xyz[i * 3 + 0], y = xyz[i * 3 + 1], z = xyz[i * 3 + 2];
    float px, py, pz, u, v;
    if (xyz_cam != nullptr && i >= cam_first) {
        const float* pc = xyz_cam + (size_t)(i - cam_first) * 3;
        px = pc[0]; py = pc[1]; pz = pc[2];
    } else {
        transform_point<float>(sT, x, y, z, px, py, pz);
    }
    // the centre, the depth key and the near / far / padding (/ fold) cull of the preprocess forward, bit for bit
    bool fold = false;
    if constexpr (LENS == 0) project_uv<float>(px, py, pz, sK[0], sK[2], sK[4], sK[5], u, v);
    else fold = lens_project<LENS>(px, py, pz, sK, skc, u, v);
    const bool culled = (pz < near_t) | (pz > far_t) | (u < -pad) | (u > width + pad) | (v < -pad) | (v > height + pad) |
                        fold;
    zkey[i] = depth_base ? (__float_as_uint(pz) - depth_base) : depth_key(pz);

    float R[9];
    quat_to_rot<float>(quat[i * 4 + 0], quat[i * 4 + 1], quat[i * 4 + 2], quat[i * 4 + 3], R);
    float Rc[9];
    camera_rotation(sT, R, Rc);
    const float su = expf(scale[i * 3 + 0]), sv = expf(scale[i * 3 + 1]);
    const float fx = sK[0], cx = sK[2], fy = sK[4], cy = sK[5];
    const float Tu[3] = {su * Rc[0], su * Rc[3], su * Rc[6]}, Tv[3] = {sv * Rc[1], sv * Rc[4], sv * Rc[7]};
    float M[9];
    if constexpr (LENS == 0) {
        M[0] = fmaf(fx, Tu[0], cx * Tu[2]); M[1] = fmaf(fx, Tv[0], cx * Tv[2]); M[2] = fmaf(fx, px, cx * pz);
        M[3] = fmaf(fy, Tu[1], cy * Tu[2]); M[4] = fmaf(fy, Tv[1], cy * Tv[2]); M[5] = fmaf(fy, py, cy * pz);
    } else {
        M[0] = Tu[0]; M[1] = Tv[0]; M[2] = px;
        M[3] = Tu[1]; M[4] = Tv[1]; M[5] = py;
    }
    M[6] = Tu[2]; M[7] = Tv[2]; M[8] = pz;
    const float r2 = mh * mh;
    // the cutoff disk a^2 + b^2 <= r^2 lies in front of the camera: min over the disk of M2 . (a, b, 1) > 0
    const bool front = (pz > 0.0f) && (r2 * (M[6] * M[6] + M[7] * M[7]) < pz * pz);
    const bool vis = !culled && front && (pz == pz) && (u == u) && (v == v);
    visible[i] = vis ? 1 : 0;

    float4* so = reinterpret_cast<float4*>(surfels + (size_t)i * SF);
    float4* bo = reinterpret_cast<float4*>(bins + (size_t)i * REC);
    if (!vis) {
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < 5; ++k) so[k] = z4;
        bo[0] = z4; bo[1] = z4; bo[2] = z4;
        packed[i] = 0ull;
        return;
    }
    float col[3];
    const float dc[3] = {rgb_dc[i * 3 + 0], rgb_dc[i * 3 + 1], rgb_dc[i * 3 + 2]};
    sh_rgb_fused<N_SH>(dc, sh_rest + (size_t)i * 3 * (N_SH - 1), x, y, z, sc, col);
    float n[3] = {Rc[2], Rc[5], Rc[8]};
    if (n[0] * px + n[1] * py + n[2] * pz > 0.0f) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
    so[0] = make_float4(u, v, sigmoid_torch(opa_logit[i]), pz);
    so[1] = make_float4(M[0], M[1], M[2], M[3]);
    so[2] = make_float4(M[4], M[5], M[6], M[7]);
    so[3] = make_float4(M[8], __fmul_rn(col[0], GSR_SH0), __fmul_rn(col[1], GSR_SH0), __fmul_rn(col[2], GSR_SH0));
    so[4] = make_float4(n[0], n[1], n[2], 0.f);

    // Binning ellipse, an axis-aligned ellipse around (u_c, v_c): the box of the disk's pixels (e_k: its largest
    // distance from the centre along axis k) lies inside the ellipse of semi-axes sqrt(2) e_k; the pixels of the
    // low-pass filter (2 |d|^2 <= r^2) lie inside the disk of radius r / sqrt(2).  Formed in fp64 and widened by
    // 2^-10 + 1/64 px against the fp32 rounding of the tile tests.
    float semi[2];
    if constexpr (LENS == 0) {
        // The pixels with a^2 + b^2 <= r^2 form the image of the disk, the conic whose dual is
        // D = M diag(r^2, r^2, -1) M^T; its bounding box has centre D_k2 / D_22 and half-width
        // sqrt(D_k2^2 - D_kk D_22) / |D_22| along axis k (D_22 < 0: the disk lies in front).
        const double R2 = (double)r2, cen[2] = {(double)u, (double)v};
        auto Dab = [&](int a, int b) {
            return R2 * ((double)M[a * 3] * M[b * 3] + (double)M[a * 3 + 1] * M[b * 3 + 1]) -
                   (double)M[a * 3 + 2] * M[b * 3 + 2];
        };
        const double D22 = Dab(2, 2);
        const float lim = fminf(2.0f * (width + height + 4.0f * pad) + 64.0f, 1e8f);
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const double Dk2 = Dab(k, 2), Dkk = Dab(k, k);
            const double half = sqrt(fmax(Dk2 * Dk2 - Dkk * D22, 0.0)) / -D22;
            const double e = fabs(Dk2 / D22 - cen[k]) + half;
            const double s = fmax(1.4142135623730951 * e, (double)mh * 0.7071067811865476) * (1.0 + 0x1p-10) + 1.0 / 64.0;
            semi[k] = s < (double)lim ? (float)s : lim;  // NaN and overflow: the limit, beyond every pixel of the image
        }
    } else {
        const float lim = fminf(2.0f * (width + height + 4.0f * pad) + 64.0f, 1e8f);
        // the box of surfel_lens_box (gsr_surfels_lens.cuh): the lens image of the disk's points with a valid ray
        double Md[9], u0 = u, u1 = u, v0 = v, v1 = v;
#pragma unroll
        for (int k = 0; k < 9; ++k) Md[k] = (double)M[k];
        const bool any = surfel_lens_box(LENS, Md, (double)r2, fx, fy, cx, cy, skc, u0, u1, v0, v1);
        const double e[2] = {any ? fmax(fabs(u0 - (double)u), fabs(u1 - (double)u)) : 0.0,
                             any ? fmax(fabs(v0 - (double)v), fabs(v1 - (double)v)) : 0.0};
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const double s = fmax(1.4142135623730951 * e[k], (double)mh * 0.7071067811865476) * (1.0 + 0x1p-10) + 1.0 / 64.0;
            // NaN and overflow: the limit, beyond every pixel of the image
            semi[k] = (e[k] == e[k] && s < (double)lim) ? (float)s : lim;
        }
    }
    const float A = __fdiv_rn(__fmul_rn(semi[0], semi[0]), r2), C = __fdiv_rn(__fmul_rn(semi[1], semi[1]), r2);
    bo[0] = make_float4(u, v, 0.f, 0.f);
    bo[1] = make_float4(A, 0.f, C, 0.f);
    bo[2] = make_float4(0.f, 0.f, 0.f, 0.f);

    // the tiles gsr_emit_keys will emit, enumerated exactly as gsr_preprocess_forward does
    Obb ob;
    if constexpr (LENS == 0) {
        compute_obb(u, v, A, 0.0f, C, mh, ob);
    } else {
        axis_obb(u, v, A, C, mh, ob);
    }
    int x0, x1, y0, y1, cnt = 0;
    tile_window(u, v, ob.radius_tiles, ntx, nty, x0, x1, y0, y1);
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
                ++cnt;
                if (small) hits |= 1ull << ((tx - x0) * wy + (ty - y0));
            }
        }
    }
    if (tile_mask != nullptr) {
        tile_mask[i] = hits;
        tile_win[i] = small ? ((uint32_t)x0 | ((uint32_t)y0 << 8) | ((uint32_t)wx << 16) | ((uint32_t)wy << 24))
                            : 0xffffffffu;
    }
    packed[i] = (1ull << 32) | (uint64_t)(uint32_t)cnt;
}

// ---- tile forward -----------------------------------------------------------------------------------------------------
__device__ __forceinline__ void stage_batch(float4* __restrict__ s_rec, const float* __restrict__ surfels,
                                            const uint64_t* __restrict__ keys, int id_bits,
                                            const int32_t* __restrict__ ids, int p0, int n) {
    for (int k = threadIdx.x; k < n * 5; k += PIX) {
        const int j = k / 5, q = k - j * 5;
        const int g = pair_id(keys, id_bits, ids, p0 + j);
        s_rec[k] = reinterpret_cast<const float4*>(surfels + (size_t)g * SF)[q];
    }
}

// RAYS: each pixel's ray from rays [H, W, 3] (the lens kernels), else (x, y, 1) in pixels (the pinhole)
template <bool RAYS>
__device__ __forceinline__ void surfel_render_fwd(const float* __restrict__ surfels, const uint64_t* __restrict__ keys,
                                                  int id_bits, const int32_t* __restrict__ ids,
                                                  const int32_t* __restrict__ ranges, const float* __restrict__ bg,
                                                  int H, int W, float near_t, float ms, float r2,
                                                  const float* __restrict__ rays, float* __restrict__ image,
                                                  float* __restrict__ depth, float* __restrict__ alpha,
                                                  float* __restrict__ normal, float* __restrict__ distortion,
                                                  int32_t* __restrict__ last, float* __restrict__ totals) {
    __shared__ float4 s_rec[BATCH * 5];
    const int ntx = (W + TILE - 1) / TILE;
    const int tile = blockIdx.x, tx = tile % ntx, ty = tile / ntx;
    const int px = tx * TILE + (threadIdx.x & 15), py = ty * TILE + (threadIdx.x >> 4);
    const bool inside = px < W && py < H;
    const float x = (float)px, y = (float)py;
    float d[3] = {0.f, 0.f, 0.f};
    if constexpr (RAYS) {
        if (inside) {
            const float* rp = rays + ((size_t)py * W + px) * 3;
            d[0] = rp[0]; d[1] = rp[1]; d[2] = rp[2];
        }
    }
    const int start = ranges[tile], end = ranges[tile + 1];
    // A: the accumulated alpha of the blend rules; Tp: the transmittance as a product, which the backward starts from
    // (1 - A cancels to a few significant bits in saturated pixels)
    float A = 0.f, Tp = 1.f, img[3] = {0.f, 0.f, 0.f}, dep = 0.f, nrm[3] = {0.f, 0.f, 0.f}, wm = 0.f, wm2 = 0.f,
          dist = 0.f;
    int lst = -1;
    bool done = !inside;
    for (int p0 = start; p0 < end; p0 += BATCH) {
        if (__syncthreads_and(done)) break;
        const int n = min(BATCH, end - p0);
        stage_batch(s_rec, surfels, keys, id_bits, ids, p0, n);
        __syncthreads();
        for (int j = 0; j < n && !done; ++j) {
            if (A > 0.9999f) {
                done = true;
                break;
            }
            const float* r = reinterpret_cast<const float*>(s_rec + j * 5);
            Hit h;
            if (!intersect<RAYS>(r, x, y, d, r2, h)) continue;
            const float w = h.alpha * (1.0f - A);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                img[c] = fmaf(w, r[S_C + c], img[c]);
                nrm[c] = fmaf(w, r[S_N + c], nrm[c]);
            }
            dep = fmaf(w, h.z, dep);
            const float m = ndc_depth(h.z, near_t, ms);
            dist = fmaf(w, fmaf(m, fmaf(m, A, -2.0f * wm), wm2), dist);
            wm = fmaf(w, m, wm);
            wm2 = fmaf(w * m, m, wm2);
            A += w;
            Tp *= 1.0f - h.alpha;
            lst = p0 + j;
        }
    }
    if (!inside) return;
    const size_t pix = (size_t)py * W + px;
    const float tb = A < 0.999f ? 1.0f - A : 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        image[pix * 3 + c] = fmaf(bg[c], tb, img[c]);
        normal[pix * 3 + c] = nrm[c];
    }
    depth[pix] = dep;
    alpha[pix] = A;
    distortion[pix] = dist;
    last[pix] = lst;
    totals[pix * 3 + 0] = Tp;
    totals[pix * 3 + 1] = wm;
    totals[pix * 3 + 2] = wm2;
}

// ---- tile backward ----------------------------------------------------------------------------------------------------
// The lens kernel's body.  The pinhole tile backward (gsr_surfels.cu) keeps its own copy of this walk with (x, y, 1) in
// place of the ray: shared through this body its instructions were scheduled differently.
__device__ __forceinline__ void surfel_render_bwd_rays(
    const float* __restrict__ surfels, const uint64_t* __restrict__ keys, int id_bits, const int32_t* __restrict__ ids,
    const int32_t* __restrict__ ranges, const float* __restrict__ bg, int H, int W, float near_t, float ms, float r2,
    const float* __restrict__ rays, const float* __restrict__ alpha, const int32_t* __restrict__ last,
    const float* __restrict__ totals, const float* __restrict__ g_img, const float* __restrict__ g_dep,
    const float* __restrict__ g_alp, const float* __restrict__ g_nrm, const float* __restrict__ g_dis,
    float* __restrict__ rows) {
    __shared__ float4 s_rec[BATCH * 5];
    __shared__ int s_id[BATCH];
    const int ntx = (W + TILE - 1) / TILE;
    const int tile = blockIdx.x, tx = tile % ntx, ty = tile / ntx;
    const int px = tx * TILE + (threadIdx.x & 15), py = ty * TILE + (threadIdx.x >> 4);
    const bool inside = px < W && py < H;
    const float x = (float)px, y = (float)py;
    const int start = ranges[tile], end = ranges[tile + 1];
    const int lane = threadIdx.x & 31;
    int lst = -1;
    float Wt = 0.f, WM = 0.f, WM2 = 0.f, T = 1.f, S = 0.f, Gi[3] = {0.f, 0.f, 0.f}, Gn[3] = {0.f, 0.f, 0.f}, Gd = 0.f,
          Ga = 0.f, Gx = 0.f;
    float d[3] = {0.f, 0.f, 0.f};
    if (inside) {
        const size_t pix = (size_t)py * W + px;
        d[0] = rays[pix * 3]; d[1] = rays[pix * 3 + 1]; d[2] = rays[pix * 3 + 2];
        lst = last[pix];
        Wt = alpha[pix];
        T = totals[pix * 3];
        WM = totals[pix * 3 + 1];
        WM2 = totals[pix * 3 + 2];
#pragma unroll
        for (int c = 0; c < 3; ++c) { Gi[c] = g_img[pix * 3 + c]; Gn[c] = g_nrm[pix * 3 + c]; }
        Gd = g_dep[pix];
        Ga = g_alp[pix];
        Gx = g_dis[pix];
        // d image / d alpha_i of the background term T_final bg (where it was added)
        if (Wt < 0.999f) S = T * (Gi[0] * bg[0] + Gi[1] * bg[1] + Gi[2] * bg[2]);
    }
    const int nb = (end - start + BATCH - 1) / BATCH;
    for (int bi = nb - 1; bi >= 0; --bi) {
        const int p0 = start + bi * BATCH;
        if (!__syncthreads_or(lst >= p0)) continue;
        const int n = min(BATCH, end - p0);
        stage_batch(s_rec, surfels, keys, id_bits, ids, p0, n);
        for (int k = threadIdx.x; k < n; k += PIX) s_id[k] = pair_id(keys, id_bits, ids, p0 + k);
        __syncthreads();
        for (int j = n - 1; j >= 0; --j) {
            const float* r = reinterpret_cast<const float*>(s_rec + j * 5);
            float g[SG - 1];
#pragma unroll
            for (int k = 0; k < SG - 1; ++k) g[k] = 0.f;
            Hit h;
            const bool on = p0 + j <= lst && intersect<true>(r, x, y, d, r2, h);
            if (on) {
                const float* M = r + S_M;
                const float om = 1.0f - h.alpha;
                T = T / om;  // T_i, the transmittance in front of this surfel
                const float w = T * h.alpha;
                const float m = ndc_depth(h.z, near_t, ms);
                const float e = fmaf(m, fmaf(m, Wt, -2.0f * WM), WM2);  // d distortion / d w_i
                const float gf = Gi[0] * r[S_C] + Gi[1] * r[S_C + 1] + Gi[2] * r[S_C + 2] + Gn[0] * r[S_N] +
                                 Gn[1] * r[S_N + 1] + Gn[2] * r[S_N + 2] + Gd * h.z + Ga + Gx * e;
                const float g_alpha = T * gf - S / om;
                S = fmaf(w, gf, S);
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    g[G_C + c] = w * Gi[c];
                    g[G_N + c] = w * Gn[c];
                }
                // depth and distortion through z: dm/dz = m_scale near / z^2
                const float gz = w * Gd + Gx * 2.0f * w * (m * Wt - WM) * (ms * near_t / (h.z * h.z));
                float grho = 0.f;
                if (__fmul_rn(r[S_OPA], h.G) < 0.99f) {  // not clamped
                    g[G_OPA] = g_alpha * h.G;
                    grho = -0.5f * h.alpha * g_alpha;
                }
                if (h.use3) {
                    const float ga = 2.0f * h.a * grho + gz * M[6], gb = 2.0f * h.b * grho + gz * M[7];
                    g[G_M + 6] += gz * h.a;
                    g[G_M + 7] += gz * h.b;
                    g[G_M + 8] += gz;
                    const float ic = 1.0f / h.c2;
                    const float gc[3] = {ga * ic, gb * ic, -(ga * h.a + gb * h.b) * ic};
                    // c = hx x hy: d/dhx = hy x gc, d/dhy = gc x hx
                    const float ghx[3] = {h.hy[1] * gc[2] - h.hy[2] * gc[1], h.hy[2] * gc[0] - h.hy[0] * gc[2],
                                          h.hy[0] * gc[1] - h.hy[1] * gc[0]};
                    const float ghy[3] = {gc[1] * h.hx[2] - gc[2] * h.hx[1], gc[2] * h.hx[0] - gc[0] * h.hx[2],
                                          gc[0] * h.hx[1] - gc[1] * h.hx[0]};
                    // hx = d_x M2 - d_z M0, hy = d_y M2 - d_z M1
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        g[G_M + k] = -d[2] * ghx[k];
                        g[G_M + 3 + k] = -d[2] * ghy[k];
                        g[G_M + 6 + k] += d[0] * ghx[k] + d[1] * ghy[k];
                    }
                } else {
                    // rho2 = 2 |(x, y) - (u_c, v_c)|^2
                    g[G_UC] = -4.0f * h.dx * grho;
                    g[G_UC + 1] = -4.0f * h.dy * grho;
                    g[G_PZ] = gz;
                }
            }
            // one atomic per warp and field
            if (__any_sync(0xffffffffu, on)) {
#pragma unroll
                for (int k = 0; k < SG - 1; ++k) {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) g[k] += __shfl_xor_sync(0xffffffffu, g[k], o);
                }
                if (lane == 0) {
                    float4* dst = reinterpret_cast<float4*>(rows + (size_t)s_id[j] * SG);
                    atomicAdd(dst + 0, make_float4(g[0], g[1], g[2], g[3]));
                    atomicAdd(dst + 1, make_float4(g[4], g[5], g[6], g[7]));
                    atomicAdd(dst + 2, make_float4(g[8], g[9], g[10], g[11]));
                    atomicAdd(dst + 3, make_float4(g[12], g[13], g[14], g[15]));
                    atomicAdd(dst + 4, make_float4(g[16], g[17], g[18], 0.f));
                }
            }
        }
        __syncthreads();
    }
}

// ---- per-gaussian backward --------------------------------------------------------------------------------------------
// uv.grad of one gaussian from its row and record (the same arithmetic for the uv.grad kernels and the backward).
// Pinhole: the gradient on a pixel translation of M.  Lens: J_n^-T g_n + g_c (gsr_surfels_lens.h), K and kc the camera
// and lens constants.
template <int LENS>
__device__ __forceinline__ float2 uv_grad_of(const float* __restrict__ r, const float* __restrict__ g, const float* K,
                                             const float* kc) {
    const float* M2 = r + S_M + 6;
    if constexpr (LENS == 0) {
        return make_float2(__fmaf_rn(g[2], M2[2], __fmaf_rn(g[1], M2[1], __fmaf_rn(g[0], M2[0], g[G_UC]))),
                           __fmaf_rn(g[5], M2[2], __fmaf_rn(g[4], M2[1], __fmaf_rn(g[3], M2[0], g[G_UC + 1]))));
    } else {
        const float gnx = __fmaf_rn(g[2], M2[2], __fmaf_rn(g[1], M2[1], __fmul_rn(g[0], M2[0])));
        const float gny = __fmaf_rn(g[5], M2[2], __fmaf_rn(g[4], M2[1], __fmul_rn(g[3], M2[0])));
        const float px = r[S_M + 2], py = r[S_M + 5], pz = r[S_M + 8];
        float J[6];
        lens_jacobian<LENS>(px, py, pz, K, kc, J);
        // J_n = p_z J[:, :2]; J_n^-T g_n = (j11 gx - j10 gy, j00 gy - j01 gx) / det
        const float j00 = pz * J[0], j01 = pz * J[1], j10 = pz * J[3], j11 = pz * J[4];
        const float idet = 1.0f / (j00 * j11 - j01 * j10);
        return make_float2(fmaf(j11 * gnx - j10 * gny, idet, g[G_UC]), fmaf(j00 * gny - j01 * gnx, idet, g[G_UC + 1]));
    }
}

template <int N_SH, int LENS>
__device__ __forceinline__ void surfel_bwd(int N, const float* __restrict__ xyz, const float* __restrict__ quat,
                                           const float* __restrict__ scale, const float* __restrict__ opa_logit,
                                           const float* __restrict__ Tdev, const float* __restrict__ Kdev,
                                           const float* __restrict__ camdev, const uint8_t* __restrict__ visible,
                                           const float* __restrict__ surfels, const float* __restrict__ rows,
                                           const float* __restrict__ g_uv_compact, const uint64_t* __restrict__ scan,
                                           int uv_emitted, float* __restrict__ o_xyz, float* __restrict__ o_quat,
                                           float* __restrict__ o_scale, float* __restrict__ o_opa,
                                           float* __restrict__ o_dc, float* __restrict__ o_sh, const float* skc) {
    constexpr int NR = N_SH - 1;
    __shared__ float sT[16], sK[9], sc[3];
    const int t = threadIdx.x;
    if (t < 16) sT[t] = Tdev[t];
    else if (t < 25) sK[t - 16] = Kdev[t - 16];
    else if (t < 28 && N_SH > 1) sc[t - 25] = camdev[t - 25];
    __syncthreads();
    const int i = blockIdx.x * PRE + t;
    if (i >= N) return;
    if (!visible[i]) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { o_xyz[i * 3 + k] = 0.f; o_scale[i * 3 + k] = 0.f; o_dc[i * 3 + k] = 0.f; }
#pragma unroll
        for (int k = 0; k < 4; ++k) o_quat[i * 4 + k] = 0.f;
        o_opa[i] = 0.f;
#pragma unroll
        for (int k = 0; k < 3 * NR; ++k) o_sh[(size_t)i * 3 * NR + k] = 0.f;
        return;
    }
    float g[SG];
    const float4* row = reinterpret_cast<const float4*>(rows + (size_t)i * SG);
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const float4 q = row[k];
        g[4 * k] = q.x; g[4 * k + 1] = q.y; g[4 * k + 2] = q.z; g[4 * k + 3] = q.w;
    }
    const float* rec = surfels + (size_t)i * SF;
    float guc = g[G_UC], gvc = g[G_UC + 1];
    if (g_uv_compact != nullptr) {
        // a gradient on the returned uv; the render's own part (uv_grad_of), when it was handed out, is already in
        // the rows, so only the caller's part moves the centre
        const float2 gin = reinterpret_cast<const float2*>(g_uv_compact)[(scan[i] >> 32) - 1];
        float2 own = make_float2(0.f, 0.f);
        if (uv_emitted) own = uv_grad_of<LENS>(rec, g, sK, skc);
        guc += gin.x - own.x;
        gvc += gin.y - own.y;
    }
    const float x = xyz[i * 3 + 0], y = xyz[i * 3 + 1], z = xyz[i * 3 + 2];
    const float qw = quat[i * 4 + 0], qx = quat[i * 4 + 1], qy = quat[i * 4 + 2], qz = quat[i * 4 + 3];
    float px, py, pz;
    transform_point<float>(sT, x, y, z, px, py, pz);
    float R[9];
    quat_to_rot<float>(qw, qx, qy, qz, R);
    float Wm[9], Rc[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) Wm[r * 3 + c] = sT[r * 4 + c];
    camera_rotation(sT, R, Rc);
    const float su = expf(scale[i * 3 + 0]), sv = expf(scale[i * 3 + 1]);
    const float fx = sK[0], cx = sK[2], fy = sK[4], cy = sK[5];
    // M[:, j] = K X_j, X = (s_u Rc[:,0], s_v Rc[:,1], p)  =>  g_X_j = K^T dM[:, j]  (lens: M = X, g_X_j = dM[:, j])
    float gX[3][3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        if constexpr (LENS == 0) {
            gX[j][0] = fx * g[G_M + j];
            gX[j][1] = fy * g[G_M + 3 + j];
            gX[j][2] = cx * g[G_M + j] + cy * g[G_M + 3 + j] + g[G_M + 6 + j];
        } else {
            gX[j][0] = g[G_M + j];
            gX[j][1] = g[G_M + 3 + j];
            gX[j][2] = g[G_M + 6 + j];
        }
    }
    float gp[3] = {gX[2][0], gX[2][1], gX[2][2] + g[G_PZ]};
    if constexpr (LENS == 0) {
        float gpc[3];
        if (project_uv_bwd<float>(px, py, pz, fx, fy, guc, gvc, gpc)) {
            gp[0] += gpc[0]; gp[1] += gpc[1]; gp[2] += gpc[2];
        }
    } else {
        float J[6];
        lens_jacobian<LENS>(px, py, pz, sK, skc, J);
#pragma unroll
        for (int k = 0; k < 3; ++k) gp[k] += J[k] * guc + J[3 + k] * gvc;
    }
    // the normal n = sign Rc[:,2] (no gradient through the orientation test)
    // the record's normal is +-Rc[:,2]: its sign is the forward's decision
    const float sgn = (rec[S_N] * Rc[2] + rec[S_N + 1] * Rc[5] + rec[S_N + 2] * Rc[8] < 0.0f) ? -1.0f : 1.0f;
    float gRc[9];  // row-major, like Rc
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        gRc[r * 3 + 0] = su * gX[0][r];
        gRc[r * 3 + 1] = sv * gX[1][r];
        gRc[r * 3 + 2] = sgn * g[G_N + r];
    }
    const float gsu = gX[0][0] * Rc[0] + gX[0][1] * Rc[3] + gX[0][2] * Rc[6];
    const float gsv = gX[1][0] * Rc[1] + gX[1][1] * Rc[4] + gX[1][2] * Rc[7];
    // Rc = W R  =>  g_R = W^T g_Rc;  p = W x + t  =>  g_x = W^T g_p
    float gR[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) gR[r * 3 + c] = Wm[r] * gRc[c] + Wm[3 + r] * gRc[3 + c] + Wm[6 + r] * gRc[6 + c];
#pragma unroll
    for (int k = 0; k < 3; ++k) o_xyz[i * 3 + k] = Wm[k] * gp[0] + Wm[3 + k] * gp[1] + Wm[6 + k] * gp[2];
    // R(q / |q|): the rotation's VJP (gsr_math_bwd.cuh sigma_world_bwd_e), then through the normalisation
    {
        const float nq = sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
        const float w = qw / nq, a = qx / nq, b = qy / nq, c = qz / nq;
        float gn[4];
        gn[0] = -2.f * c * gR[1] + 2.f * b * gR[2] + 2.f * c * gR[3] - 2.f * a * gR[5] - 2.f * b * gR[6] + 2.f * a * gR[7];
        gn[1] = 2.f * b * gR[1] + 2.f * c * gR[2] + 2.f * b * gR[3] - 4.f * a * gR[4] - 2.f * w * gR[5] + 2.f * c * gR[6] +
                2.f * w * gR[7] - 4.f * a * gR[8];
        gn[2] = -4.f * b * gR[0] + 2.f * a * gR[1] + 2.f * w * gR[2] + 2.f * a * gR[3] + 2.f * c * gR[5] - 2.f * w * gR[6] +
                2.f * c * gR[7] - 4.f * b * gR[8];
        gn[3] = -4.f * c * gR[0] - 2.f * w * gR[1] + 2.f * a * gR[2] + 2.f * w * gR[3] - 4.f * c * gR[4] + 2.f * b * gR[5] +
                2.f * a * gR[6] + 2.f * b * gR[7];
        const float q[4] = {qw, qx, qy, qz};
        const float dot = q[0] * gn[0] + q[1] * gn[1] + q[2] * gn[2] + q[3] * gn[3];
        const float n3 = nq * nq * nq;
#pragma unroll
        for (int k = 0; k < 4; ++k) o_quat[i * 4 + k] = gn[k] / nq - q[k] * dot / n3;
    }
    o_scale[i * 3 + 0] = gsu * su;
    o_scale[i * 3 + 1] = gsv * sv;
    o_scale[i * 3 + 2] = 0.f;
    const float sg = sigmoid_torch(opa_logit[i]);
    o_opa[i] = g[G_OPA] * ((1.0f - sg) * sg);
    // colour = SH0 * col, col = RSH0 sum_k Y_k coef_k (Y_0 = SH0): d colour / d coef_k = Y_k
    float Y[N_SH];
    if (N_SH > 1) {
        float dx, dy, dz;
        view_dir<float>(x, y, z, sc[0], sc[1], sc[2], dx, dy, dz);
        sh_basis<float, N_SH>(dx, dy, dz, Y);
    } else {
        Y[0] = GSR_SH0;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        o_dc[i * 3 + c] = g[G_C + c] * Y[0];
#pragma unroll
        for (int k = 1; k < N_SH; ++k) o_sh[(size_t)i * 3 * NR + c * NR + (k - 1)] = g[G_C + c] * Y[k];
    }
}

}  // namespace surfel
}  // namespace gsr
