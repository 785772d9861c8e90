"""Per-gaussian (row-by-row) comparison of gradients against the fp64 CPU oracle.

A global criterion max|mine - ref| / max|ref| never looks at a gaussian whose gradient is a small fraction of the
largest one: at 5e-4, a third to a half of the visible gaussians of a typical scene could have a zero, negated or
swapped gradient and still pass.  These checks bound every row by what its own arithmetic can explain:

  render-stage rows (the per-gaussian sums of the tile renderer's backward: rgb, opacity, uv, conic)
      |mine - ref| <= c * eps * mass      per entry, mass = sum over the (pixel, gaussian) terms the oracle added
                                          into that entry of the magnitudes of each term's parts
                                          (cpu_oracle.render_backward(mass=True))
  parameter rows (xyz, quaternion, scale, opacity, rgb, sh), fed the SAME render-stage rows
      |mine - ref| <= rtol * max|ref row| + floor * max|ref|

fp32 threshold flips: the oracle's exp2f and the GPU's ex2.approx can land on opposite sides of the 1/255 alpha
threshold for a few (pixel, gaussian) pairs.  In fp32, up to max(3, M / 10^4) rows may miss the row bound; each of those
must still pass the global criterion, and they are printed.  The fp64 branch has no threshold and allows none.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

EPS = {np.dtype(np.float32): 2.0 ** -24, np.dtype(np.float64): 2.0 ** -53}
GLOBAL_TOL = 5e-4  # the global criterion the oracle tests used before the per-row checks

# c of the render-stage bound, per field.  Worst row ratio |mine - ref| / (eps * mass) of the rows within the bound,
# measured on one H100 80GB HBM3 (400 W power limit) per scene of tests/test_gradient_rows_gpu.py:
#                                   rgb  opacity    uv  conic
#   64x64, SH 0-3 (fused, unfused)  1288     424  1275   1193
#   50x37                           3670     583  4735   4702
#   17x33, 1x64, 64x1                138      34   124    123
#   720p, 100k gaussians            6963    3539  4751   5063
#   deep stack (all four variants)    70      21    70     80
#   saturating stack                  63      19  7782   7553   (one row beyond the bound in uv and conic)
#   per-pixel SH, fp32                95       7    80     48
#   per-pixel SH, fp64                15       2    12     11   (RENDER_C_FP64)
RENDER_C = dict(rgb=16384.0, opacity=16384.0, uv=16384.0, conic=16384.0)
RENDER_C_FP64 = dict(rgb=64.0, opacity=64.0, uv=64.0, conic=64.0)
# parameter rows fed the same render-stage rows; measured worst row ratio at these values: 0.39 (quaternion, 720p)
PARAM_RTOL = 1e-4
PARAM_FLOOR = 1e-8


def as_rows(a):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)
    return a.astype(np.float64).reshape(a.shape[0], -1) if a.ndim else a.astype(np.float64).reshape(1, 1)


def global_rel(mine, ref):
    mine, ref = as_rows(mine), as_rows(ref)
    return float(np.abs(mine - ref).max() / max(np.abs(ref).max(), 1e-300)) if ref.size else 0.0


def flips_allowed(m, dtype=np.float32):
    """Rows allowed beyond their bound among m visible gaussians: threshold flips exist only in the fp32 branch."""
    return max(3, m // 10_000) if np.dtype(dtype) == np.float32 else 0


@dataclass
class RowResult:
    name: str
    worst: float                      # largest |mine - ref| / bound over the rows within the bound
    need: float                       # the smallest scale of the bound that leaves at most `allowed` rows beyond it
    bad: np.ndarray                   # rows beyond their bound
    allowed: int
    global_err: float                 # max |mine - ref| / max |ref| over the whole array
    bad_global: list = field(default_factory=list)   # bad rows that also fail the global criterion

    @property
    def ok(self):
        return len(self.bad) <= self.allowed and not self.bad_global

    def __str__(self):
        s = (f"{self.name}: worst row ratio {self.worst:.3g} (bound x{self.need:.3g} needed), {len(self.bad)} rows beyond the bound "
             f"(allowed {self.allowed}), global {self.global_err:.2e}")
        if len(self.bad):
            s += f", rows {self.bad[:10].tolist()}"
        if self.bad_global:
            s += f", failing the global criterion too: {self.bad_global[:10]}"
        return s


def compare_rows(name, mine, ref, bound, allowed):
    """Rows of mine / ref ([N, ...], any array type) against a per-entry bound (same shape, >= 0)."""
    mine, ref, bound = as_rows(mine), as_rows(ref), as_rows(bound)
    assert mine.shape == ref.shape == bound.shape, (name, mine.shape, ref.shape, bound.shape)
    err = np.abs(mine - ref)
    assert np.isfinite(err).all(), f"{name}: non-finite values"
    over = err > bound
    bad = np.flatnonzero(over.any(1))
    ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    ok_rows = np.ones(len(ratio), bool)
    ok_rows[bad] = False
    worst = float(ratio[ok_rows].max()) if ok_rows.any() and ratio.size else 0.0
    row_ratio = np.sort(ratio.max(1))[::-1] if ratio.size else np.zeros(1)
    need = float(row_ratio[allowed]) if allowed < len(row_ratio) else 0.0
    scale = max(float(np.abs(ref).max()), 1e-300) if ref.size else 1.0
    bad_global = [int(i) for i in bad if err[i].max() > GLOBAL_TOL * scale]
    return RowResult(name, worst, need, bad, allowed, float(err.max() / scale) if err.size else 0.0, bad_global)


def render_rows(name, mine, ref, mass, c, eps, allowed):
    """Render-stage sums: |mine - ref| <= c * eps * mass per entry."""
    return compare_rows(name, mine, ref, c * eps * as_rows(mass), allowed)


def param_rows(name, mine, ref, rtol, floor, allowed):
    """Parameter gradients: |mine - ref| <= rtol * max|ref row| + floor * max|ref| per entry."""
    ref2 = as_rows(ref)
    row_max = np.abs(ref2).max(1, keepdims=True) if ref2.size else ref2
    bound = rtol * np.broadcast_to(row_max, ref2.shape) + floor * (np.abs(ref2).max() if ref2.size else 0.0)
    return compare_rows(name, mine, ref2, bound, allowed)


def assert_all(results):
    """Print every result; fail with the ones that miss their bound."""
    for r in results:
        print(r)
    failed = [str(r) for r in results if not r.ok]
    assert not failed, "\n".join(failed)
