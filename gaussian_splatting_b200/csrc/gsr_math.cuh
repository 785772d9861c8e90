// gsr_math.cuh — per-Gaussian projection math with pinned rounding order.
//
// Every function below states the value the reference computes
// (joeyan/gaussian_splatting, file:line cited per function) and pins the
// fp32 rounding sequence to the one the reference's nvcc build executes
// (multiply/add contraction into FMA was read off the reference's SASS, see
// DESIGN.md "Rounding contract").  Explicit __f*_rn intrinsics are used so that
// neither NVVM nor ptxas can re-associate or re-contract anything: uv, conic
// and the tile set must be bit-identical to the reference, because they feed
// discrete decisions (tile membership, the alpha < 1/255 skip, saturation).
//
// All functions are templated on T in {float,double}.  The double
// instantiation follows the same operation order (used by the fp64
// gradcheck surface; no bit contract there).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace gsr {

// ---------------------------------------------------------------------------
// rounding-pinned arithmetic
// ---------------------------------------------------------------------------
template <typename T> struct Ar;

template <> struct Ar<float> {
    static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
    static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
    static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
    static __device__ __forceinline__ float fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
    static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
    static __device__ __forceinline__ float sqrt(float a) { return __fsqrt_rn(a); }
    static __device__ __forceinline__ float exp(float a) { return expf(a); }
    static __device__ __forceinline__ float rsqrt(float a) { return rsqrtf(a); }
};

template <> struct Ar<double> {
    static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
    static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
    static __device__ __forceinline__ double sub(double a, double b) { return __dadd_rn(a, -b); }
    static __device__ __forceinline__ double fma(double a, double b, double c) { return __fma_rn(a, b, c); }
    static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
    static __device__ __forceinline__ double sqrt(double a) { return __dsqrt_rn(a); }
    static __device__ __forceinline__ double exp(double a) { return ::exp(a); }
    static __device__ __forceinline__ double rsqrt(double a) { return ::rsqrt(a); }
};

// ---------------------------------------------------------------------------
// world -> camera.  Reference: splat_py/utils.py:60-72, i.e. torch.matmul of the
// 4x4 with [x,y,z,1], which torch runs as a batched (4x4)@(4x1) product in cuBLAS.
// The rounding order of the cuBLAS kernel used for full 65535-matrix chunks (cuBLAS
// 12.8; identified by exhaustive search over evaluation trees against torch's output,
// tools/check_transform.py) is a 2-way split over k:
//     (x*m0 -> fma(y, m1, .))  +  (z*m2 -> fma(1, m3, .))
// Chunks of other sizes may go through a different cuBLAS kernel (on H100: roughly
// 16 K to 35 K matrices, and small ones); the host mirror hands such a last chunk to
// torch itself (gaussian_splatting_b200/rasterize.py) so the bits always match.
// ---------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void transform_point(const T* __restrict__ M /*4x4 row-major*/,
                                                T x, T y, T z, T& ox, T& oy, T& oz) {
    using A = Ar<T>;
    ox = A::add(A::fma(y, M[1], A::mul(x, M[0])), A::add(A::mul(z, M[2]), M[3]));
    oy = A::add(A::fma(y, M[5], A::mul(x, M[4])), A::add(A::mul(z, M[6]), M[7]));
    oz = A::add(A::fma(y, M[9], A::mul(x, M[8])), A::add(A::mul(z, M[10]), M[11]));
}

// ---------------------------------------------------------------------------
// pinhole projection.  Reference: src/projection.cu:16-18.
//   u = (fx*x)/z + cx ; v = (fy*y)/z + cy   (mul, IEEE div, add)
// ---------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void project_uv(T x, T y, T z, T fx, T cx, T fy, T cy, T& u, T& v) {
    using A = Ar<T>;
    u = A::add(A::div(A::mul(fx, x), z), cx);
    v = A::add(A::div(A::mul(fy, y), z), cy);
}

// ---------------------------------------------------------------------------
// Sigma_world = R(q/|q|) diag(exp(s))^2 R^T.  Reference: src/projection.cu:67-108.
// out[6] = {S00,S01,S02,S11,S12,S22}
// ---------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void quat_to_rot(T qw, T qx, T qy, T qz, T* __restrict__ R /*9*/) {
    using A = Ar<T>;
    const T n2 = A::fma(qw, qw, A::fma(qz, qz, A::fma(qx, qx, A::mul(qy, qy))));
    const T n = A::sqrt(n2);
    qx = A::div(qx, n);
    qy = A::div(qy, n);
    qz = A::div(qz, n);
    qw = A::div(qw, n);
    const T x2 = A::add(qx, qx), y2 = A::add(qy, qy), z2 = A::add(qz, qz);
    const T yw = A::mul(y2, qw), xw = A::mul(x2, qw), zw = A::mul(z2, qw);
    const T one = T(1);
    const T omx = A::fma(x2, -qx, one);  // 1 - 2x^2
    const T omy = A::fma(y2, -qy, one);  // 1 - 2y^2
    R[0] = A::fma(z2, -qz, omy);
    R[1] = A::fma(x2, qy, -zw);
    R[2] = A::fma(x2, qz, yw);
    R[3] = A::fma(x2, qy, zw);
    R[4] = A::fma(z2, -qz, omx);
    R[5] = A::fma(y2, qz, -xw);
    R[6] = A::fma(x2, qz, -yw);
    R[7] = A::fma(y2, qz, xw);
    R[8] = A::fma(y2, -qy, omx);
}

// Sigma_world = R diag(v) R^T from the rotation and the per-axis variances v_k
template <typename T>
__device__ __forceinline__ void sigma_from_rv(const T* __restrict__ R, T v0, T v1, T v2, T* __restrict__ S /*6*/) {
    using A = Ar<T>;
    // S_ab = fma(v2, Ra2*Rb2, fma(v0, Ra0*Rb0, v1*(Ra1*Rb1)))
#define GSR_SAB(a, b)                                                                        \
    A::fma(v2, A::mul(R[3 * a + 2], R[3 * b + 2]),                                           \
           A::fma(v0, A::mul(R[3 * a + 0], R[3 * b + 0]), A::mul(v1, A::mul(R[3 * a + 1], R[3 * b + 1]))))
    S[0] = GSR_SAB(0, 0);
    S[1] = GSR_SAB(0, 1);
    S[2] = GSR_SAB(0, 2);
    S[3] = GSR_SAB(1, 1);
    S[4] = GSR_SAB(1, 2);
    S[5] = GSR_SAB(2, 2);
#undef GSR_SAB
}

template <typename T>
__device__ __forceinline__ void sigma_world(T qw, T qx, T qy, T qz, T s0, T s1, T s2,
                                            T* __restrict__ S /*6*/) {
    using A = Ar<T>;
    T R[9];
    quat_to_rot<T>(qw, qx, qy, qz, R);
    const T e0 = A::exp(s0), e1 = A::exp(s1), e2 = A::exp(s2);
    sigma_from_rv<T>(R, A::mul(e0, e0), A::mul(e1, e1), A::mul(e2, e2), S);
}

// Sigma_world from given per-axis variances (the 3-D filter's exp(s)^2 + f^2, gsr_record.cuh f3d_filter)
template <typename T>
__device__ __forceinline__ void sigma_world_var(T qw, T qx, T qy, T qz, T v0, T v1, T v2, T* __restrict__ S /*6*/) {
    T R[9];
    quat_to_rot<T>(qw, qx, qy, qz, R);
    sigma_from_rv<T>(R, v0, v1, v2, S);
}

// ---------------------------------------------------------------------------
// projection Jacobian.  Reference: src/projection.cu:165-174.
//   J = [[fx/z, 0, (x*-fx)/(z*z)], [0, fy/z, (y*-fy)/(z*z)]]
// ---------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void proj_jacobian(T x, T y, T z, T fx, T fy, T* __restrict__ J /*6*/) {
    using A = Ar<T>;
    const T zz = A::mul(z, z);
    J[0] = A::div(fx, z);
    J[1] = T(0);
    J[2] = A::div(A::mul(x, -fx), zz);
    J[3] = T(0);
    J[4] = A::div(fy, z);
    J[5] = A::div(A::mul(y, -fy), zz);
}

// small dense product with the reference's accumulation order
// (src/matrix.cuh:15-30: sum = 0; sum += a*b  ->  FMA chain from +0)
template <typename T, int RA, int CA, int CB>
__device__ __forceinline__ void matmul_chain(const T* __restrict__ Am, const T* __restrict__ Bm,
                                             T* __restrict__ Cm) {
    using A = Ar<T>;
#pragma unroll
    for (int r = 0; r < RA; ++r) {
#pragma unroll
        for (int c = 0; c < CB; ++c) {
            T s = T(0);
#pragma unroll
            for (int k = 0; k < CA; ++k) s = A::fma(Am[r * CA + k], Bm[k * CB + c], s);
            Cm[r * CB + c] = s;
        }
    }
}

// ---------------------------------------------------------------------------
// 2-D covariance ("conic" in the reference's vocabulary).
// Reference: src/projection.cu:226-256.  S2 = (J W) Sigma (J W)^T,
// conic = [S2_00, S2_01 + S2_10, S2_11].  Sfull is the 3x3 row-major Sigma.
// ---------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void conic_from(const T* __restrict__ Sfull /*9*/,
                                           const T* __restrict__ J /*6*/,
                                           const T* __restrict__ W /*9*/, T* __restrict__ conic /*3*/,
                                           T* __restrict__ JW_out /*6 or null*/) {
    using A = Ar<T>;
    T JW[6], JWS[6], JWt[6], S2[4];
    matmul_chain<T, 2, 3, 3>(J, W, JW);
    matmul_chain<T, 2, 3, 3>(JW, Sfull, JWS);
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) JWt[c * 2 + r] = JW[r * 3 + c];
    matmul_chain<T, 2, 3, 2>(JWS, JWt, S2);
    conic[0] = S2[0];
    conic[1] = A::add(S2[1], S2[2]);
    conic[2] = S2[3];
    if (JW_out) {
#pragma unroll
        for (int i = 0; i < 6; ++i) JW_out[i] = JW[i];
    }
}

__device__ __forceinline__ void sym6_to_full(const float* S6, float* S9) {
    S9[0] = S6[0]; S9[1] = S6[1]; S9[2] = S6[2];
    S9[3] = S6[1]; S9[4] = S6[3]; S9[5] = S6[4];
    S9[6] = S6[2]; S9[7] = S6[4]; S9[8] = S6[5];
}
__device__ __forceinline__ void sym6_to_full(const double* S6, double* S9) {
    S9[0] = S6[0]; S9[1] = S6[1]; S9[2] = S6[2];
    S9[3] = S6[1]; S9[4] = S6[3]; S9[5] = S6[4];
    S9[6] = S6[2]; S9[7] = S6[4]; S9[8] = S6[5];
}

// ---------------------------------------------------------------------------
// real SH basis evaluated at a unit direction, and SH -> RGB.
// Reference: src/spherical_harmonics.cuh:4-96 (constants are float even in
// the fp64 instantiation; the "- 1.0"/"- 3.0" literals make bands 2/3 go
// through double arithmetic in the fp32 build, mirrored here).
// ---------------------------------------------------------------------------
#define GSR_SH0 0.28209479177387814f
#define GSR_RSH0 3.544907701811032f
#define GSR_SH1 0.4886025119029199f
#define GSR_SH2_0 1.0925484305920792f
#define GSR_SH2_2 0.31539156525252005f
#define GSR_SH2_4 0.5462742152960396f
#define GSR_SH3_0 0.5900435899266435f
#define GSR_SH3_1 2.890611442640554f
#define GSR_SH3_2 0.4570457994644658f
#define GSR_SH3_3 0.263875515352797f
#define GSR_SH3_5 1.445305721320277f

template <typename T, int N_SH>
__device__ __forceinline__ void sh_basis(T x, T y, T z, T* __restrict__ Y) {
    Y[0] = T(GSR_SH0);
    if (N_SH < 4) return;
    Y[1] = T(-GSR_SH1) * y;
    Y[2] = T(GSR_SH1) * z;
    Y[3] = T(-GSR_SH1) * x;
    if (N_SH < 9) return;
    const T xy = x * y, yz = y * z, xz = x * z, xx = x * x, yy = y * y, zz = z * z;
    Y[4] = T(GSR_SH2_0) * xy;
    Y[5] = T(-GSR_SH2_0) * yz;
    Y[6] = T(double(T(GSR_SH2_2)) * (double(T(3) * zz) - 1.0));
    Y[7] = T(-GSR_SH2_0) * xz;
    Y[8] = T(GSR_SH2_4) * (xx - yy);
    if (N_SH < 16) return;
    Y[9] = T(-GSR_SH3_0) * y * (T(3) * xx - yy);
    Y[10] = T(GSR_SH3_1) * xy * z;
    Y[11] = T(double(T(-GSR_SH3_2) * y) * (double(T(5) * zz) - 1.0));
    Y[12] = T(double(T(GSR_SH3_3) * z) * (double(T(5) * zz) - 3.0));
    Y[13] = T(double(T(-GSR_SH3_2) * x) * (double(T(5) * zz) - 1.0));
    Y[14] = T(GSR_SH3_5) * z * (xx - yy);
    Y[15] = T(-GSR_SH3_0) * x * (xx - T(3) * yy);
}

// view direction used by the SH precompute (src/precompute_sh.cu:26-37)
template <typename T>
__device__ __forceinline__ void view_dir(T px, T py, T pz, T cx, T cy, T cz, T& dx, T& dy, T& dz) {
    using A = Ar<T>;
    dx = px - cx;
    dy = py - cy;
    dz = pz - cz;
    const T r = A::rsqrt(dx * dx + dy * dy + dz * dz);
    dx *= r;
    dy *= r;
    dz *= r;
}

// ---------------------------------------------------------------------------
// tile footprint: oriented bounding box of the mh_dist-sigma ellipse and the
// separating-axis test against a 16x16 tile.  fp32 only, as in the reference.
// Reference: src/tile_culling.cu:8-122 (SAT :8-66, OBB :69-122).
// ---------------------------------------------------------------------------
struct Obb {
    float c[8];  // tl_x, tl_y, tr_x, tr_y, bl_x, bl_y, br_x, br_y
    // precomputed SAT terms
    float min_x, max_x, min_y, max_y;
    float ax, ay, amin, amax;  // major axis and obb extent on it
    float mx, my, mmin, mmax;  // minor axis and obb extent on it
    int radius_tiles;
};

// a = conic0 + 0.25, b = conic1 * 0.5, c = conic2 + 0.25 (src/tile_culling.cu:142-144)
__device__ __forceinline__ void compute_obb(float u, float v, float a, float b, float c, float mh_dist,
                                            Obb& o) {
    using A = Ar<float>;
    const float d = A::sub(a, c);
    const float disc = A::fma(b, b, A::mul(A::mul(d, d), 0.25f));
    const float right = A::sqrt(disc);
    const float s = A::add(a, c);
    const float l1 = A::fma(s, 0.5f, right);
    const float l2 = A::fma(s, 0.5f, -right);
    const float r_major = A::mul(A::sqrt(l1), mh_dist);
    const float r_minor = A::mul(A::sqrt(l2), mh_dist);
    float theta;
    if ((double)fabsf(b) < 1e-16) {
        theta = (a >= c) ? 0.0f : 1.5707963705062866211f;
    } else {
        theta = atan2f(A::sub(l1, a), b);
    }
    const float ct = cosf(theta);
    const float st = sinf(theta);
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

// true iff the OBB and the tile [left,right]x[top,bottom] overlap on all four axes
__device__ __forceinline__ bool obb_hits_tile(const Obb& o, float left, float right, float top,
                                              float bottom) {
    using A = Ar<float>;
    if (o.min_x > right || o.max_x < left) return false;
    if (o.min_y > bottom || o.max_y < top) return false;
    {
        const float xl = A::mul(o.ax, left), xr = A::mul(o.ax, right);
        const float tl = A::fma(o.ay, top, xl), tr = A::fma(o.ay, top, xr);
        const float bl = A::fma(o.ay, bottom, xl), br = A::fma(o.ay, bottom, xr);
        const float mn = fminf(fminf(tl, tr), fminf(bl, br));
        const float mxv = fmaxf(fmaxf(tl, tr), fmaxf(bl, br));
        if (mn > o.amax || mxv < o.amin) return false;
    }
    {
        const float xl = A::mul(o.mx, left), xr = A::mul(o.mx, right);
        const float tl = A::fma(o.my, top, xl), tr = A::fma(o.my, top, xr);
        const float bl = A::fma(o.my, bottom, xl), br = A::fma(o.my, bottom, xr);
        const float mn = fminf(fminf(tl, tr), fminf(bl, br));
        const float mxv = fmaxf(fmaxf(tl, tr), fmaxf(bl, br));
        if (mn > o.mmax || mxv < o.mmin) return false;
    }
    return true;
}

// half-open tile window [x0,x1) x [y0,y1) searched for one Gaussian
// (src/tile_culling.cu:149-155; int->float->int round trips kept)
__device__ __forceinline__ void tile_window(float u, float v, int radius_tiles, int ntx, int nty,
                                            int& x0, int& x1, int& y0, int& y1) {
    const int ptx = (int)floorf(__fmul_rn(u, 0.0625f));
    const int pty = (int)floorf(__fmul_rn(v, 0.0625f));
    x0 = (int)fmaxf(0.0f, (float)(ptx - radius_tiles));
    x1 = (int)fminf((float)ntx, (float)(ptx + radius_tiles));
    y0 = (int)fmaxf(0.0f, (float)(pty - radius_tiles));
    y1 = (int)fminf((float)nty, (float)(pty + radius_tiles));
}

// float depth -> order-preserving 32-bit key (identity on positive floats)
__device__ __forceinline__ uint32_t depth_key(float z) {
    const uint32_t b = __float_as_uint(z);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// sigmoid as torch evaluates it on CUDA: 1 / (1 + exp(-x))
__device__ __forceinline__ float sigmoid_torch(float x) {
    return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x)));
}

}  // namespace gsr
