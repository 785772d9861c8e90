"""CPU restatements of the 3DGS-MCMC kernels (csrc/gsr_mcmc.cu), independent of the kernels' own formulation:

  relocation_mp    the paper's relocation with mpmath at 50 digits, the double sum exactly as written
  relocation_f64   the same double sum in numpy fp64 (vectorised over rows), the oracle the GPU kernel is held to
  relocation_f32   the same double sum accumulated in fp32 (shows why the kernel works in fp64)
  noise_weight     w = 1 / (1 + exp(-k ((1 - o) - x0)))
  noise_f64        xyz + scaler * w * R diag(exp(2 s)) R^T eps in fp64, given eps
"""
from __future__ import annotations

import math

import numpy as np

EPS32 = 2.0 ** -23


def relocation_mp(o, N, n_max=51, dps=50):
    """(o_hat, coeff = o / D) for one row, mpmath at `dps` digits: o_hat = 1 - (1 - o)^(1/N),
    D = sum_{i=1..N} sum_{k=0..i-1} C(i-1, k) (-1)^k o_hat^(k+1) / sqrt(k+1); N clamped to [1, n_max].  o is taken
    as the exact value of its float."""
    import mpmath

    with mpmath.workdps(dps):
        N = min(max(int(N), 1), n_max)
        o = mpmath.mpf(float(o))
        oh = 1 - (1 - o) ** (mpmath.mpf(1) / N)
        D = mpmath.mpf(0)
        for i in range(1, N + 1):
            for k in range(i):
                D += mpmath.binomial(i - 1, k) * (-1) ** k * oh ** (k + 1) / mpmath.sqrt(k + 1)
        return oh, (o / D if o > 0 else mpmath.mpf(1))


def _double_sum(oh, N, dtype):
    """The paper's double sum, accumulated in `dtype`, for rows of o_hat with per-row N."""
    oh = np.asarray(oh, dtype)
    D = np.zeros_like(oh)
    for i in range(1, int(N.max()) + 1):
        live = N >= i
        for k in range(i):
            term = dtype(math.comb(i - 1, k)) * dtype((-1) ** k) * oh ** dtype(k + 1) / dtype(math.sqrt(k + 1))
            D = np.where(live, (D + term).astype(dtype), D)
    return D


def relocation_f64(opacity, scale, ratio, n_max=51, min_opacity=0.005):
    """(new_opacity fp64 before rounding, clamped in fp32 like the kernel; new_scale fp64) for rows of sigmoid opacity
    [n], exp scale [n,3], ratio [n]."""
    o = np.asarray(opacity, np.float32).astype(np.float64)
    N = np.clip(np.asarray(ratio, np.int64), 1, n_max)
    oh = -np.expm1(np.log1p(-o) / N)
    D = _double_sum(oh, N, np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        coeff = np.where(o > 0, o / D, 1.0)
    new_o = np.clip(oh.astype(np.float32), np.float32(min_opacity), np.float32(1 - EPS32))
    return oh, new_o, np.asarray(scale, np.float32).astype(np.float64) * coeff[:, None]


def relocation_f32(opacity, ratio, n_max=51):
    """coeff = o / D with the double sum accumulated in fp32 (o_hat itself formed in fp64 and rounded, so that only
    the sum's cancellation shows)."""
    o = np.asarray(opacity, np.float32)
    N = np.clip(np.asarray(ratio, np.int64), 1, n_max)
    oh = (-np.expm1(np.log1p(-o.astype(np.float64)) / N)).astype(np.float32)
    D = _double_sum(oh, N, np.float32)
    return o / D


def noise_weight(o, k=100.0, x0=0.995):
    o = np.asarray(o, np.float64)
    return 1.0 / (1.0 + np.exp(-k * ((1.0 - o) - x0)))


def rotation(q):
    """[n,4] (w, x, y, z), normalised here -> [n,3,3]."""
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)


def noise_f64(xyz, quaternion, scale_log, opacity_logit, eps, scaler, k=100.0, x0=0.995):
    """xyz + scaler * w(sigmoid(opacity)) * R diag(exp(2 s)) R^T eps, all in fp64.  Also returns |Sigma eps| scaled
    the same way without cancellation (sum of absolute products), a bound for the fp32 rounding of the kernel."""
    R = rotation(quaternion)
    v = np.exp(2.0 * np.asarray(scale_log, np.float64))
    o = 1.0 / (1.0 + np.exp(-np.asarray(opacity_logit, np.float64).reshape(-1)))
    sw = scaler * noise_weight(o, k, x0)
    e = np.asarray(eps, np.float64)
    d = np.einsum("nij,nj->ni", R, v * np.einsum("nji,nj->ni", R, e))
    mag = np.einsum("nij,nj->ni", np.abs(R), v * np.einsum("nji,nj->ni", np.abs(R), np.abs(e)))
    return np.asarray(xyz, np.float64) + sw[:, None] * d, np.abs(sw)[:, None] * mag
