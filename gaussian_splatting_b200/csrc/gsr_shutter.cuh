// gsr_shutter.cuh — rolling-shutter cameras: the shutter hooks of gsr_preprocess.cuh (gsr_shutter.cu,
// libgsr_shutter.so).  DESIGN.md 3.24 has the derivation.
//
// T = camera_T_world is the pose of the image's middle line.  xi = (rho, omega) is the camera's motion over the whole
// readout, applied on the left: T(tau) = se3_exp((tau - 1/2) xi) T, tau in [0, 1] the readout time.  An image point
// u = (u, v) is read at r(u) = r0 + e^T u (the readout direction, per view).  With p0 the camera-frame mean at the
// middle pose and s = tau - 1/2, the mean at time tau is p = p0 + delta, delta = (R_s - I) p0 + t_s, and the rotation
// W(tau) = R_s W0, formed as W0 + (R_s - I) W0: xi = 0 gives delta = 0 and W = W0 exactly.
//
// A gaussian's time tau* solves tau = clamp(r(u(tau)), 0, 1): SHUTTER_NEWTON_STEPS projected Newton steps from the
// line its middle-pose mean projects to, no data-dependent loop.  f = du/dtau = J p', p' = omega x p + rho, and the
// slope lambda = e^T f.  The covariance is the local affine map of x -> u at the gaussian's own time,
// du = A J W dx with A = I + f e^T / (1 - lambda) (A = I where tau* is clamped).  A gaussian with lambda >=
// SHUTTER_LAMBDA_MAX, or whose residual |tau* - clamp(r(u(tau*)))| exceeds SHUTTER_TOL, is culled.
#pragma once
#include "gsr_common.cuh"

namespace gsr {

constexpr int SHUTTER_NEWTON_STEPS = 4;
constexpr float SHUTTER_LAMBDA_MAX = 0.75f;
constexpr float SHUTTER_TOL = 9.5367431640625e-07f;  // 2^-20 of the readout
constexpr int SHUTTER_VALUES = 20;                   // a row: 12 pose values, 6 twist values, 2 zeros (float4 loads)
constexpr int SHUTTER_JL_TERMS = 11;                 // terms of the SE(3) left-Jacobian series

// one view's constants, per thread: the twist and the readout line r(u) = r0 + e0 u + e1 v
struct ShutterView {
    float rho[3], w[3], r0, e0, e1;
};

// a gaussian at its own time: s = tau* - 1/2, ph = s omega, the Rodrigues coefficients a, b of R_s, p' (pd), f,
// 1 / (1 - lambda), and whether tau* sits clamped at 0 or 1
struct ShutterPt {
    float s, a, b, ph[3], pd[3], f[2], kappa;
    bool clamped, ok;
};

__device__ __forceinline__ ShutterView load_shutter(const float* __restrict__ xi, float r0, float e0, float e1) {
    ShutterView v;
#pragma unroll
    for (int k = 0; k < 3; ++k) { v.rho[k] = xi[k]; v.w[k] = xi[3 + k]; }
    v.r0 = r0; v.e0 = e0; v.e1 = e1;
    return v;
}

__device__ __forceinline__ void cross3(const float* a, const float* b, float* o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

// sin(th)/th, (1 - cos th)/th^2, (th - sin th)/th^3 of th = |ph|.  Below th^2 = 1/2 (40 degrees of motion between the
// middle line and the gaussian's line) from their Taylor series through th^8 (truncation < 1e-9), which have no
// cancellation in fp32 and are exactly 1, 1/2, 1/6 at 0; above it the closed forms, written without cancellation
// where they have one.
__device__ __forceinline__ void so3_coefs(const float* ph, float& a, float& b, float& c) {
    const float t = ph[0] * ph[0] + ph[1] * ph[1] + ph[2] * ph[2];
    if (t < 0.5f) {
        a = fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.0f / 362880.0f, -1.0f / 5040.0f), 1.0f / 120.0f), -1.0f / 6.0f), 1.0f);
        b = fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.0f / 3628800.0f, -1.0f / 40320.0f), 1.0f / 720.0f), -1.0f / 24.0f), 0.5f);
        c = fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.0f / 39916800.0f, -1.0f / 362880.0f), 1.0f / 5040.0f), -1.0f / 120.0f),
                 1.0f / 6.0f);
    } else {
        // sinpif: its argument reduction is exact and needs no local memory (sinf's Payne-Hanek path does)
        const float th = sqrtf(t), x = th * 0.318309886183790672f;
        const float sn = sinpif(x), sh = sinpif(0.5f * x);
        a = sn / th;
        b = 2.0f * sh * sh / t;
        c = (th - sn) / (t * th);
    }
}

// p = p0 + delta at s; also ph = s omega and the coefficients of R_s
__device__ __forceinline__ void shutter_point(const ShutterView& sv, float s, const float* p0, float* p, float* ph,
                                              float& a, float& b) {
    float c;
#pragma unroll
    for (int k = 0; k < 3; ++k) ph[k] = s * sv.w[k];
    so3_coefs(ph, a, b, c);
    const float sr[3] = {s * sv.rho[0], s * sv.rho[1], s * sv.rho[2]};
    float c1[3], c2[3], d1[3], d2[3];
    cross3(ph, p0, c1);
    cross3(ph, c1, c2);
    cross3(ph, sr, d1);
    cross3(ph, d1, d2);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float delta = fmaf(a, c1[k], b * c2[k]) + (sr[k] + fmaf(b, d1[k], c * d2[k]));
        p[k] = p0[k] + delta;
    }
}

// v <- R_s v (sign +1) or R_s^T v (sign -1): v + sign a (ph x v) + b ph x (ph x v)
__device__ __forceinline__ void shutter_rotate(const ShutterPt& sp, float sign, float* v) {
    float c1[3], c2[3];
    cross3(sp.ph, v, c1);
    cross3(sp.ph, c1, c2);
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = v[k] + fmaf(sign * sp.a, c1[k], sp.b * c2[k]);
}

__device__ __forceinline__ float clamp01(float t) { return fminf(fmaxf(t, 0.0f), 1.0f); }

// tau* of a gaussian whose middle-pose camera-frame mean is (px, py, pz); replaces it by p(tau*).  eval(x, y, z, u, v,
// J) is the lens's projection and Jacobian.
template <class Eval>
__device__ __forceinline__ void shutter_solve(const ShutterView& sv, float& px, float& py, float& pz, Eval eval,
                                              ShutterPt& o) {
    const float p0[3] = {px, py, pz};
    float u, v, J[6], p[3], pd[3];
    eval(px, py, pz, u, v, J);
    float tau = clamp01(fmaf(sv.e1, v, fmaf(sv.e0, u, sv.r0)));
    float lam = 0.f, f0 = 0.f, f1 = 0.f, r = 0.f;
#pragma unroll
    for (int k = 0; k <= SHUTTER_NEWTON_STEPS; ++k) {
        o.s = tau - 0.5f;
        shutter_point(sv, o.s, p0, p, o.ph, o.a, o.b);
        eval(p[0], p[1], p[2], u, v, J);
        cross3(sv.w, p, pd);
#pragma unroll
        for (int j = 0; j < 3; ++j) pd[j] += sv.rho[j];
        f0 = fmaf(J[2], pd[2], fmaf(J[1], pd[1], J[0] * pd[0]));
        f1 = fmaf(J[5], pd[2], fmaf(J[4], pd[1], J[3] * pd[0]));
        lam = fmaf(sv.e1, f1, sv.e0 * f0);
        r = fmaf(sv.e1, v, fmaf(sv.e0, u, sv.r0));
        if (k == SHUTTER_NEWTON_STEPS) break;
        const float nt = clamp01(tau - (tau - r) / (1.0f - lam));
        tau = (lam < SHUTTER_LAMBDA_MAX && nt == nt) ? nt : tau;
    }
    px = p[0]; py = p[1]; pz = p[2];
#pragma unroll
    for (int j = 0; j < 3; ++j) o.pd[j] = pd[j];
    o.f[0] = f0; o.f[1] = f1;
    o.kappa = 1.0f / (1.0f - lam);
    o.clamped = !(r >= 0.0f && r <= 1.0f);
    o.ok = (lam < SHUTTER_LAMBDA_MAX) & (fabsf(tau - clamp01(r)) <= SHUTTER_TOL);
}

// Js = A J = J + kappa f (e^T J); Js = J where tau* is clamped or f = 0 (xi = 0: the global-shutter floats)
__device__ __forceinline__ void shutter_shear(const ShutterView& sv, const ShutterPt& sp, const float* J, float* Js) {
    const bool shear = !sp.clamped && (sp.f[0] != 0.0f || sp.f[1] != 0.0f);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float eJ = sp.kappa * fmaf(sv.e1, J[3 + j], sv.e0 * J[j]);
        Js[j] = shear ? fmaf(sp.f[0], eJ, J[j]) : J[j];
        Js[3 + j] = shear ? fmaf(sp.f[1], eJ, J[3 + j]) : J[3 + j];
    }
}

// the covariance's gradient on W(tau*): gW = Js^T (2 G M Sigma), M = Js W (gsr_pose.cuh pose_contribution), and
// v = vee of the skew part of gW W^T, the gradient on a rotation omega applied on the left of W
__device__ __forceinline__ void shutter_gw(const float* Js, const float* W, const float* S, const float* gc, float* gW,
                                           float* vw) {
    float M[6], MS[6], P[6];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) M[r * 3 + c] = fmaf(Js[r * 3 + 2], W[6 + c], fmaf(Js[r * 3 + 1], W[3 + c], Js[r * 3] * W[c]));
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) MS[r * 3 + c] = fmaf(M[r * 3 + 2], S[6 + c], fmaf(M[r * 3 + 1], S[3 + c], M[r * 3] * S[c]));
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        P[c] = 2.0f * fmaf(gc[1], MS[3 + c], gc[0] * MS[c]);
        P[3 + c] = 2.0f * fmaf(gc[2], MS[3 + c], gc[1] * MS[c]);
    }
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) gW[r * 3 + c] = fmaf(Js[3 + r], P[3 + c], Js[r] * P[c]);
    float N[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            N[r * 3 + c] = fmaf(gW[r * 3 + 2], W[c * 3 + 2], fmaf(gW[r * 3 + 1], W[c * 3 + 1], gW[r * 3] * W[c * 3]));
    vw[0] = N[7] - N[5];
    vw[1] = N[2] - N[6];
    vw[2] = N[3] - N[1];
}

// gJ (on Js) -> the gradient on the lens's J; gpd: the gradient on p' through f (0 where A = I)
__device__ __forceinline__ void shutter_bwd_j(const ShutterView& sv, const ShutterPt& sp, const float* J, float* gJ,
                                              float* gpd) {
    gpd[0] = gpd[1] = gpd[2] = 0.f;
    if (sp.clamped || (sp.f[0] == 0.0f && sp.f[1] == 0.0f)) return;
    const float e[2] = {sv.e0, sv.e1};
    float ga[2];  // (gJs J^T) e
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 2; ++k)
            acc = fmaf(e[k], fmaf(gJ[i * 3 + 2], J[k * 3 + 2], fmaf(gJ[i * 3 + 1], J[k * 3 + 1], gJ[i * 3] * J[k * 3])), acc);
        ga[i] = acc;
    }
    const float fa = fmaf(sp.f[1], ga[1], sp.f[0] * ga[0]);
    const float gf[2] = {sp.kappa * fmaf(sp.kappa * fa, e[0], ga[0]), sp.kappa * fmaf(sp.kappa * fa, e[1], ga[1])};
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float fg = sp.kappa * fmaf(sp.f[1], gJ[3 + j], sp.f[0] * gJ[j]);  // kappa f^T gJs, column j
        gJ[j] = fmaf(gf[0], sp.pd[j], fmaf(e[0], fg, gJ[j]));
        gJ[3 + j] = fmaf(gf[1], sp.pd[j], fmaf(e[1], fg, gJ[3 + j]));
        gpd[j] = fmaf(J[3 + j], gf[1], J[j] * gf[0]);
    }
}

// gp += gpd x omega (p' = omega x p + rho), then, unless tau* is clamped, the implicit time's term:
// g_tau = gp . p' + omega . vw,  gp += g_tau kappa J^T e
__device__ __forceinline__ void shutter_bwd_p(const ShutterView& sv, const ShutterPt& sp, const float* J,
                                              const float* gpd, const float* vw, float* gp) {
    float t[3];
    cross3(gpd, sv.w, t);
#pragma unroll
    for (int k = 0; k < 3; ++k) gp[k] += t[k];
    if (sp.clamped) return;
    const float gt = fmaf(gp[2], sp.pd[2], fmaf(gp[1], sp.pd[1], gp[0] * sp.pd[0])) +
                     fmaf(sv.w[2], vw[2], fmaf(sv.w[1], vw[1], sv.w[0] * vw[0]));
    const float k = gt * sp.kappa;
#pragma unroll
    for (int j = 0; j < 3; ++j) gp[j] = fmaf(k, fmaf(sv.e1, J[3 + j], sv.e0 * J[j]), gp[j]);
}

// The camera row of one gaussian: 12 pose values (d/dT[:3, :]) and 6 twist values.  p0 = W0 x + t0 and
// p = R_s p0 + t_s, W = R_s W0: dL/dW0 = (R_s^T gp) x^T + R_s^T gW, dL/dt0 = R_s^T gp.  The twist: a left
// perturbation eta of se3_exp(s xi) moves p by eta_rho + eta_omega x p and W by [eta_omega]x W, so
// g_eta = (gp, p x gp + vw); a change d xi perturbs se3_exp(s xi) by eta = s J_l(s xi) d xi, so
// g_xi = s J_l(s xi)^T g_eta, plus the direct terms of p' = omega x p + rho, (gpd, p x gpd).  J_l = sum_k ad^k / (k+1)! (truncated after SHUTTER_JL_TERMS
// terms: exact to fp32 for |omega| <= 2 rad over the readout, and exactly the identity at xi = 0).
__device__ __forceinline__ void shutter_contribution(const ShutterView& sv, const ShutterPt& sp, const float* p,
                                                     const float* gp, const float* gpd, const float* gW,
                                                     const float* vw, float x, float y, float z, float* acc) {
    float g0[3] = {gp[0], gp[1], gp[2]};
    shutter_rotate(sp, -1.0f, g0);
    const float xw[3] = {x, y, z};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float col[3] = {gW[c], gW[3 + c], gW[6 + c]};
        shutter_rotate(sp, -1.0f, col);
#pragma unroll
        for (int r = 0; r < 3; ++r) acc[r * 4 + c] += fmaf(g0[r], xw[c], col[r]);
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) acc[r * 4 + 3] += g0[r];
    float ge[6], pg[3];
    cross3(p, gp, pg);
#pragma unroll
    for (int k = 0; k < 3; ++k) { ge[k] = gp[k]; ge[3 + k] = pg[k] + vw[k]; }
    // Horner: h = sum_k (ad^T)^k g_eta / (k+1)!, ad^T (a, b) = (a x w', a x r' + b x w') at w' = s omega, r' = s rho
    const float rs[3] = {sp.s * sv.rho[0], sp.s * sv.rho[1], sp.s * sv.rho[2]};
    float inv = 1.0f;
#pragma unroll
    for (int k = 2; k <= SHUTTER_JL_TERMS; ++k) inv /= (float)k;
    float h[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) h[k] = ge[k] * inv;
#pragma unroll
    for (int n = SHUTTER_JL_TERMS - 1; n >= 1; --n) {
        inv *= (float)(n + 1);  // 1 / n!
        float a1[3], a2[3], b1[3];
        cross3(h, sp.ph, a1);
        cross3(h, rs, a2);
        cross3(h + 3, sp.ph, b1);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            h[k] = fmaf(ge[k], inv, a1[k]);
            h[3 + k] = fmaf(ge[3 + k], inv, a2[k] + b1[k]);
        }
    }
    float pq[3];
    cross3(p, gpd, pq);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        acc[12 + k] += fmaf(sp.s, h[k], gpd[k]);
        acc[15 + k] += fmaf(sp.s, h[3 + k], pq[k]);
    }
}

}  // namespace gsr

// The hooks (gsr_preprocess.cuh).  The bodies take the twists (6 floats per view), the readout line's constants and,
// the backward, the camera-row partials [C, grid, SHUTTER_VALUES] (NULL: no camera gradient).
#define GSR_SHUTTER_HOOKS
#define GSR_SHUTTER_PARAM , const float* __restrict__ shutter_xi, float sh_r0, float sh_e0, float sh_e1
#define GSR_SHUTTER_LOAD(view) const ShutterView sv = load_shutter(shutter_xi + 6 * (view), sh_r0, sh_e0, sh_e1);
#define GSR_SHUTTER_POINT(px, py, pz)                                                                         \
    ShutterPt sp;                                                                                             \
    shutter_solve(                                                                                            \
        sv, px, py, pz,                                                                                       \
        [&](float ex, float ey, float ez, float& eu, float& ev, float* eJ) {                                  \
            GSR_PROJECT(ex, ey, ez, eu, ev);                                                                  \
            GSR_JACOBIAN(ex, ey, ez, eJ);                                                                     \
        },                                                                                                    \
        sp);
#define GSR_SHUTTER_CULL | !sp.ok
#define GSR_SHUTTER_W(W)                                 \
    _Pragma("unroll") for (int wc = 0; wc < 3; ++wc) {   \
        float col[3] = {W[wc], W[3 + wc], W[6 + wc]};    \
        shutter_rotate(sp, 1.0f, col);                   \
        W[wc] = col[0]; W[3 + wc] = col[1]; W[6 + wc] = col[2]; \
    }
#define GSR_SHUTTER_JACOBIAN(J) \
    float Js[6];                \
    shutter_shear(sv, sp, J, Js);
#define GSR_SHUTTER_J Js
#define GSR_SHUTTER_BWD_J(gJ)             \
    float gpd[3], sgW[9], svw[3];         \
    shutter_gw(Js, W, S9, gc, sgW, svw);  \
    shutter_bwd_j(sv, sp, J, gJ, gpd);
#define GSR_SHUTTER_GP(gp) shutter_bwd_p(sv, sp, J, gpd, svw, gp);

#define GSR_POSE_HOOKS
#define GSR_POSE_PARAM , float* __restrict__ pose_partials
#define GSR_POSE_DECL float gpose[SHUTTER_VALUES] = {};
#define GSR_POSE_VIEW                                                                     \
    if (pose_partials != nullptr) {                                                       \
        const float pp[3] = {px, py, pz};                                                 \
        shutter_contribution(sv, sp, pp, gp, gpd, sgW, svw, x, y, z, gpose);              \
    }
#define GSR_POSE_REDUCE(view)                                                                                  \
    if (pose_partials != nullptr)                                                                              \
        pose_cta_reduce<SHUTTER_VALUES>(gpose,                                                                 \
                                        pose_partials + ((size_t)(view) * gridDim.x + blockIdx.x) * SHUTTER_VALUES);
