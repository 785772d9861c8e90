"""CPU oracle of the depth renderer's per-pixel walk (`render_depth_cuda`).  TEST INFRASTRUCTURE ONLY.

A pixel walks its tile's splats front to back, accumulating alpha, and reports the range sqrt(x^2 + y^2 + z^2) of
the first splat after which the accumulated alpha A exceeds the threshold (strictly), or -1 when none does.  The
alphas themselves come from the caller (on the GPU they are read back bit for bit); this module pins the
accumulation and the range, in explicit float32 / float64 roundings:

  reference order   w = (float)((1.0 - (double)A) * (double)alpha);  A = A + w        (fp32 add)
  fma order         A = fmaf(alpha, 1.0f - A, A)                                    (what a plain fp32
                                                                                      `A += alpha * (1.0f - A)`
                                                                                      compiles to)
  range             sqrtf(fmaf(z, z, fmaf(x, x, y * y)))                            (FMUL, FFMA, FFMA)

The two orders round differently in a few percent of the steps, which moves the first-surface index only when a
threshold falls between the two accumulated values; `separating_thresholds` finds such thresholds.
"""
from __future__ import annotations

import numpy as np

F32, F64 = np.float32, np.float64


def fma32(a, b, c):
    """fmaf(a, b, c) with one rounding.  a*b of two floats is exact in float64; the float64 sum s is exact up to
    the TwoSum residual e, and rounding s to float32 gives fmaf's answer unless s sits exactly on a float32
    rounding midpoint with e != 0 — then s is moved one float64 ulp towards the exact value first."""
    a, b, c = (np.asarray(v, F32).astype(F64) for v in (a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    e = (c - (s - bp)) + (p - bp)
    f = s.astype(F32)
    g = np.nextafter(f, np.where(s > f, F32(np.inf), F32(-np.inf)).astype(F32))
    mid = (f.astype(F64) + g.astype(F64)) * 0.5 == s
    s = np.where(mid & (e != 0), np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def splat_range(xyz):
    """[..., 3] float32 camera-frame positions -> float32 range, in the kernel's operation order."""
    xyz = np.asarray(xyz, F32)
    x, y, z = xyz[..., 0], xyz[..., 1], xyz[..., 2]
    return np.sqrt(fma32(z, z, fma32(x, x, y * y))).astype(F32)


def accumulate(alphas, order="reference"):
    """[P, K] float32 alphas in walk order -> [P, K] float32 accumulated alpha after each splat."""
    alphas = np.asarray(alphas, F32)
    A = np.zeros(alphas.shape[0], F32)
    out = np.empty_like(alphas)
    for k in range(alphas.shape[1]):
        a = alphas[:, k]
        if order == "reference":
            w = ((1.0 - A.astype(F64)) * a.astype(F64)).astype(F32)
            A = (A + w).astype(F32)
        elif order == "fma":
            A = fma32(a, F32(1.0) - A, A)
        else:
            raise ValueError(order)
        out[:, k] = A
    return out


def first_surface(alphas, xyz, threshold, order="reference"):
    """Depth of each pixel: alphas [P, K] float32, xyz [P, K, 3] float32 (the splat at each step) -> [P] float32
    range of the first splat with A > threshold, -1 where the threshold is never exceeded."""
    A = accumulate(alphas, order)
    if A.shape[1] == 0:  # empty tile
        return np.full(A.shape[0], -1.0, F32)
    hit = A > F32(threshold)
    k = np.argmax(hit, axis=1)
    rng = splat_range(np.asarray(xyz, F32)[np.arange(len(k)), k])
    return np.where(hit.any(axis=1), rng, F32(-1.0)).astype(F32)


def separating_thresholds(alphas, limit=8):
    """Thresholds at which the two orders report different first surfaces.

    For a pixel whose two accumulations first differ at step k (equal before), t = min of the two values at k
    makes exactly one order exceed t at k (the comparison is strict) while neither did before.  Returns up to
    `limit` distinct float32 thresholds, each with the pixel it was taken from: [(t, pixel, k), ...]."""
    ref, fma = accumulate(alphas, "reference"), accumulate(alphas, "fma")
    differ = ref != fma
    out, seen = [], set()
    for p in np.flatnonzero(differ.any(axis=1)):
        k = int(np.argmax(differ[p]))
        t = F32(min(ref[p, k], fma[p, k]))
        prev = ref[p, k - 1] if k else F32(0.0)
        if prev < t and float(t) not in seen:
            seen.add(float(t))
            out.append((t, int(p), k))
            if len(out) == limit:
                break
    return out
