/* filter3d_oracle.c — CPU oracle of Mip-Splatting's 3-D smoothing filter in the fused rasterizer
 * (rasterize(..., filter3d=f)) and of its sampling-rate pass (compute_filter3d).
 *
 * TEST INFRASTRUCTURE ONLY (tests/filter3d_oracle.py).  Compiled together with oracle/gsr_oracle.c, whose per-gaussian
 * helpers (rotation, jacobian, conic, transform_point) it reuses unchanged.
 *
 *   f3d_project_*   per visible gaussian: variances v_k = exp(s_k)^2, v'_k = v_k + f^2, t_k = v_k / v'_k (1 where
 *                   f^2 == 0), coef = sqrt((t0 t1) t2), the 2-D covariance of R diag(v') R^T — the operations of
 *                   gsr_record.cuh f3d_filter and gsr_math.cuh sigma_world_var in the fp32 instantiation; e_in (or
 *                   NULL): exp(s) supplied by the caller, e.g. the device's expf, which can differ from the host's by an ulp
 *   f3d_sample_f32  the sampling pass of csrc/gsr_filter3d.cu, operation for operation
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mfma -shared -fPIC -I<repo>/oracle filter3d_oracle.c -lm
 */
#include "gsr_oracle.c"

#define F3D_PROJECT(REAL, SUF, FMA_, SQRT_, EXP_)                                                                     \
    void SUF(f3d_project)(int N, const REAL* quat, const REAL* scale, const REAL* filter, const REAL* xyz_cam,        \
                          const REAL* K, const REAL* T, const unsigned char* visible, const REAL* e_in, REAL* conic,  \
                          REAL* coef, REAL* t_out) {                                                                  \
        for (int i = 0; i < N; ++i) {                                                                                 \
            if (!visible[i]) continue;                                                                                \
            const REAL F = filter[i] * filter[i];                                                                     \
            REAL v[3], vp[3], t[3];                                                                                   \
            for (int k = 0; k < 3; ++k) {                                                                             \
                const REAL e = e_in ? e_in[i * 3 + k] : EXP_(scale[i * 3 + k]);                                       \
                v[k] = e * e;                                                                                         \
                vp[k] = v[k] + F;                                                                                     \
                t[k] = F == (REAL)0 ? (REAL)1 : v[k] / vp[k];                                                         \
                t_out[i * 3 + k] = t[k];                                                                              \
            }                                                                                                         \
            coef[i] = SQRT_((t[0] * t[1]) * t[2]);                                                                    \
            REAL R[9], S[9], J[6];                                                                                    \
            SUF(rotation)(quat[i * 4], quat[i * 4 + 1], quat[i * 4 + 2], quat[i * 4 + 3], R);                         \
            for (int a = 0; a < 3; ++a)                                                                               \
                for (int b = 0; b < 3; ++b) {                                                                         \
                    REAL s = vp[1] * (R[3 * a + 1] * R[3 * b + 1]);                                                   \
                    s = FMA_(vp[0], R[3 * a + 0] * R[3 * b + 0], s);                                                  \
                    S[3 * a + b] = FMA_(vp[2], R[3 * a + 2] * R[3 * b + 2], s);                                       \
                }                                                                                                     \
            SUF(jacobian)(xyz_cam + i * 3, K[0], K[4], J);                                                            \
            SUF(conic)(S, J, T, conic + i * 3);                                                                       \
        }                                                                                                             \
    }

#define F32(x) x##_f32
#define F64(x) x##_f64
F3D_PROJECT(float, F32, fmaf, sqrtf, expf)
F3D_PROJECT(double, F64, fma, sqrt, exp)

/* filter [N] from C cameras: Ts [C,16], Ks [C,9], W / H [C] */
void f3d_sample_f32(int N, const float* xyz, int C, const float* Ts, const float* Ks, const int* W, const int* H,
                    float near_t, float margin, float variance, float* filter) {
    const float m1 = 1.0f + margin;
    float rmax = 0.0f;
    for (int i = 0; i < N; ++i) {
        float r = INFINITY;
        int seen = 0;
        for (int c = 0; c < C; ++c) {
            const float* T = Ts + (size_t)c * 16;
            const float* K = Ks + (size_t)c * 9;
            float p[3];
            transform_point_f32(T, xyz[i * 3], xyz[i * 3 + 1], xyz[i * 3 + 2], p);
            const float u = (K[0] * p[0]) / p[2] + K[2];
            const float v = (K[4] * p[1]) / p[2] + K[5];
            const float w = (float)W[c], h = (float)H[c];
            if (p[2] > near_t && u >= -(margin * w) && u <= m1 * w && v >= -(margin * h) && v <= m1 * h) {
                r = fminf(r, p[2] / fmaxf(K[0], K[4]));
                seen = 1;
            }
        }
        filter[i] = seen ? r : -1.0f;
        if (seen && r > rmax) rmax = r;
    }
    const float sv = sqrtf(variance);
    for (int i = 0; i < N; ++i) filter[i] = sv * (filter[i] < 0.0f ? rmax : filter[i]);
}
