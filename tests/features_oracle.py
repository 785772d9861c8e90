"""CPU oracle of rasterize(..., features=F): the feature map and its gradients.  TEST INFRASTRUCTURE.

Extends oracle/cpu_oracle.py (which it builds on and does not change) with features_oracle.c:

    o = orc.rasterize(...)                                   # compact gaussians, pair list, n / wlast per pixel
    fmap = render_forward(o, F[o.keep])                      # [H,W,D]
    d = rasterize_backward(o, F, G)                          # gradients of <G, feature_map>

d.F is the gradient on F [N,D], d.render the render-stage rows of the feature loss (opacity, uv, conic) over all N
gaussians and d.mass their masses, for tests/gradrows.py's per-row bounds.
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

from oracle import cpu_oracle as orc

HERE = Path(__file__).resolve().parent
ORACLE = HERE.parent / "oracle"
_lib = None


def build() -> Path:
    """Compile into a per-user cache directory outside the tree (keyed by the sources' digest)."""
    srcs = [HERE / "features_oracle.c", HERE / "features_oracle_body.inc", ORACLE / "gsr_oracle.c",
            ORACLE / "gsr_oracle_body.inc"]
    digest = hashlib.sha256(b"".join(p.read_bytes() for p in srcs)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_features_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_features_oracle_{digest}.so"
    if not out.exists():
        tmp = out.with_suffix(f".{os.getpid()}.tmp")
        subprocess.run(["gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-mfma", "-shared", "-fPIC", f"-I{ORACLE}",
                        f"-I{HERE}", str(srcs[0]), "-o", str(tmp), "-lm"], check=True, capture_output=True)
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _suffix(dt):
    return {np.dtype(np.float32): "_f32", np.dtype(np.float64): "_f64"}[np.dtype(dt)]


def forward(uvs, opacity, conic, F, ranges, sorted_idx, H, W):
    """feature_map [H,W,D] of the compact gaussians' features F [G,D] (dtype of uvs: fp32 walks like the GPU, fp64 is
    the exact function)."""
    dt = uvs.dtype
    c = lambda a: np.ascontiguousarray(a, dtype=dt)  # noqa: E731
    F = c(F)
    D = F.shape[1]
    fmap = np.zeros((H, W, D), dt)
    getattr(lib(), "orc_render_features_forward" + _suffix(dt))(
        C.c_int(H), C.c_int(W), C.c_int(D), _p(c(uvs)), _p(c(opacity).reshape(-1)), _p(c(conic)), _p(F),
        _p(np.ascontiguousarray(ranges, np.int32)), _p(np.ascontiguousarray(sorted_idx, np.int32)), _p(fmap))
    return fmap


def backward(uvs, opacity, conic, F, ranges, sorted_idx, n, wlast, G, chunk):
    """Gradients of <G, feature_map> (float64): F [G,D], opacity [G], uv [G,2], conic [G,3], and their masses."""
    dt = uvs.dtype
    c = lambda a: np.ascontiguousarray(a, dtype=dt)  # noqa: E731
    F = c(F)
    M, D = F.shape
    H, W = n.shape
    g = SimpleNamespace(F=np.zeros((M, D)), opacity=np.zeros(M), uv=np.zeros((M, 2)), conic=np.zeros((M, 3)))
    m = SimpleNamespace(**{k: np.zeros_like(v) for k, v in vars(g).items()})
    getattr(lib(), "orc_render_features_backward" + _suffix(dt))(
        C.c_int(H), C.c_int(W), C.c_int(D), C.c_int(chunk), _p(c(uvs)), _p(c(opacity).reshape(-1)), _p(c(conic)),
        _p(F), _p(np.ascontiguousarray(ranges, np.int32)), _p(np.ascontiguousarray(sorted_idx, np.int32)),
        _p(np.ascontiguousarray(n, np.int32)), _p(c(wlast)), _p(c(G)), _p(g.F), _p(g.opacity), _p(g.uv), _p(g.conic),
        _p(m.F), _p(m.opacity), _p(m.uv), _p(m.conic))
    return g, m


def render_forward(o, F_compact):
    """feature_map of an orc.rasterize result o for the compact gaussians' features."""
    H, W = o.n.shape
    return forward(o.uv, o.opacity, o.conic, F_compact, o.ranges, o.sorted_idx, H, W)


def rasterize_backward(o, F, G):
    """Gradients (float64) of <G, feature_map> for the features F [N,D] of all gaussians: d.F [N,D] (zero rows for
    culled ones); d.render / d.mass: render-stage rows (opacity, uv, conic) over all N gaussians and their masses;
    d.xyz, d.quaternion, d.scale, d.opacity, ... through cpu_oracle.project_backward."""
    N = o.inputs[0].shape[0]
    chunk = orc.REF_CHUNK[(np.dtype(o.dtype).type, 1)]
    g, m = backward(o.uv, o.opacity, o.conic, np.asarray(F)[o.keep], o.ranges, o.sorted_idx, o.n, o.wlast, G, chunk)

    def full(a):
        out = np.zeros((N,) + a.shape[1:], np.float64)
        out[o.keep] = a
        return out

    render = SimpleNamespace(**{k: full(v) for k, v in vars(g).items()})
    mass = SimpleNamespace(**{k: full(v) for k, v in vars(m).items()})
    d = orc.project_backward(o, np.zeros((N, 3)), render.opacity, render.uv, render.conic)
    d.F, d.uv, d.render, d.mass = render.F, g.uv, render, mass
    return d
