"""CPU oracle of rasterize(weight_stats=...): per-gaussian sum / max / count of the colour blend's weights.
TEST INFRASTRUCTURE.

Extends oracle/cpu_oracle.py with weight_stats_oracle.c, on the forward of any of the tests' oracles:

    o = depth_alpha_oracle.rasterize(sc_inputs...)     # or antialiased_oracle / filter3d_oracle .rasterize(...)
    r = weight_stats(o)                                 # r.sum (float64), r.max (float32), r.count (int64): [N] rows

r.* are indexed by gaussian row (zeros for culled gaussians); r.compact_* by compact (visible) index; r.alpha [H,W] is
the accumulated alpha of the same walk and r.nblend [H,W] its number of blends per pixel; r.uncertain [N] counts, per
gaussian, the pixels where an alpha near the 1/255 threshold earlier in the walk lets another exp implementation
decide differently (weight_stats_oracle.c).
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from pathlib import Path
from types import SimpleNamespace

import numpy as np

HERE = Path(__file__).resolve().parent
ORACLE = HERE.parent / "oracle"
_lib = None


def build() -> Path:
    """Compile into a per-user cache directory outside the tree (keyed by the sources' digest)."""
    srcs = [HERE / "weight_stats_oracle.c", ORACLE / "gsr_oracle.c", ORACLE / "gsr_oracle_body.inc"]
    digest = hashlib.sha256(b"".join(p.read_bytes() for p in srcs)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_weight_stats_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_weight_stats_oracle_{digest}.so"
    if not out.exists():
        tmp = out.with_suffix(f".{os.getpid()}.tmp")
        subprocess.run(["gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-mfma", "-shared", "-fPIC", f"-I{ORACLE}",
                        str(srcs[0]), "-o", str(tmp), "-lm"], check=True, capture_output=True)
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def compact_stats(uvs, opacity, conic, ranges, sorted_idx, H, W, dilated=False):
    """-> (sum float64 [M], max float32 [M], count int64 [M], alpha float32 [H,W], nblend int32 [H,W], uncertain
    int32 [M], see weight_stats_oracle.c); fp32 inputs
    indexed by the ids in sorted_idx, conic without the 0.25 dilation (the renderer adds it), or with it (dilated)."""
    f = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    M = int(np.asarray(uvs).shape[0])
    s, m, n = np.zeros(M), np.zeros(M, np.float32), np.zeros(M, np.int64)
    alpha, nblend, unc = np.zeros((H, W), np.float32), np.zeros((H, W), np.int32), np.zeros(M, np.int32)
    uvs, opacity, conic = f(uvs), f(opacity).reshape(-1), f(conic)
    ranges, sorted_idx = np.ascontiguousarray(ranges, np.int32), np.ascontiguousarray(sorted_idx, np.int32)
    lib().orc_weight_stats_f32(C.c_int(H), C.c_int(W), C.c_int(M), _p(uvs), _p(opacity), _p(conic), _p(ranges),
                               _p(sorted_idx), _p(s), _p(m), _p(n), _p(alpha), _p(nblend), _p(unc),
                               C.c_int(1 if dilated else 0))
    return s, m, n, alpha, nblend, unc


def weight_stats(o):
    """Statistics of an oracle forward o (fp32; its render_conic when present, and o.opacity, the opacity the renderer
    was fed), scattered to gaussian rows through o.keep."""
    H, W = o.n.shape
    s, m, n, alpha, nblend, unc = compact_stats(o.uv, o.opacity, getattr(o, "render_conic", o.conic), o.ranges,
                                           o.sorted_idx, H, W)
    N = int(o.keep.shape[0])
    r = SimpleNamespace(compact_sum=s, compact_max=m, compact_count=n, alpha=alpha, nblend=nblend)
    r.sum, r.max, r.count, r.uncertain = np.zeros(N), np.zeros(N, np.float32), np.zeros(N, np.int64), np.zeros(N, np.int32)
    r.sum[o.keep], r.max[o.keep], r.count[o.keep], r.uncertain[o.keep] = s, m, n, unc
    return r


def weight_stats_of_records(records, ranges, ids_sorted, H, W):
    """The same walk over the fused path's own render inputs: records [N,12] (u v tau opacity | a 2b c det | ...,
    dilation included), tile ranges and the sorted gaussian ids of the pairs.  This isolates the render stage: the
    per-gaussian stage's rounding (uv, conic, opacity within ~1e-6 of the host's) moves alpha at a pixel far from a
    sub-pixel splat's centre by much more than an ulp.  Rows are gaussian ids."""
    rec = np.asarray(records, np.float32).reshape(-1, 12)
    s, m, n, alpha, nblend, unc = compact_stats(rec[:, 0:2], rec[:, 3], rec[:, 4:7], ranges, ids_sorted, H, W,
                                                dilated=True)
    return SimpleNamespace(sum=s, max=m, count=n, uncertain=unc, alpha=alpha, nblend=nblend)
