"""CPU oracle of rasterize(absgrad=True): per-gaussian sums of the per-pixel ABSOLUTE gradients on the projected means.
TEST INFRASTRUCTURE.

Extends oracle/cpu_oracle.py and tests/depth_alpha_oracle.py (which it builds on and does not change) with
absgrad_oracle.c:

    o = depth_alpha_oracle.rasterize(sc_inputs...)          # or antialiased_oracle.rasterize(...)
    r = uv_backward(o, G, G_depth=None, G_alpha=None)        # r.uv, r.mass, r.absgrad [M,2] (float64)

r.uv is the render stage's gradient on the compact uv for <G,image> (+ <Gd,depth> + <Ga,alpha>), r.mass its mass
(cpu_oracle.render_backward(mass=True)'s m_uv) and r.absgrad = sum_p |d <G_p, out_p> / d uv|.
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
    srcs = [HERE / "absgrad_oracle.c", HERE / "absgrad_oracle_body.inc", ORACLE / "gsr_oracle.c",
            ORACLE / "gsr_oracle_body.inc"]
    digest = hashlib.sha256(b"".join(p.read_bytes() for p in srcs)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_absgrad_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_absgrad_oracle_{digest}.so"
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


def uv_backward(o, grad_image, grad_depth=None, grad_alpha=None):
    """Render-stage sums over the compact gaussians of o (a depth_alpha_oracle / antialiased_oracle forward; its
    render_conic is used when present): uv [M,2], mass [M,2] and absgrad [M,2], float64."""
    dt = o.dtype
    c = lambda a: np.ascontiguousarray(a, dtype=dt)  # noqa: E731
    H, W = o.n.shape
    M = o.uv.shape[0]
    r = SimpleNamespace(uv=np.zeros((M, 2)), mass=np.zeros((M, 2)), absgrad=np.zeros((M, 2)))
    if (grad_depth is None) != (grad_alpha is None):
        grad_depth = np.zeros((H, W)) if grad_depth is None else grad_depth
        grad_alpha = np.zeros((H, W)) if grad_alpha is None else grad_alpha
    depth = grad_depth is not None
    chunk = orc.REF_CHUNK[(np.dtype(dt).type, 1)]
    fn = getattr(lib(), "orc_render_backward_abs" + {np.dtype(np.float32): "_f32", np.dtype(np.float64): "_f64"}[dt])
    fn(C.c_int(H), C.c_int(W), C.c_int(M), C.c_int(chunk), _p(c(o.uv)), _p(c(o.opacity).reshape(-1)), _p(c(o.rgb)),
       _p(c(getattr(o, "render_conic", o.conic))), _p(c(o.z)) if depth else None,
       _p(np.ascontiguousarray(o.ranges, np.int32)), _p(np.ascontiguousarray(o.sorted_idx, np.int32)),
       _p(c(o.background)), _p(np.ascontiguousarray(o.n, np.int32)), _p(c(o.wlast)), _p(c(grad_image)),
       _p(c(grad_depth)) if depth else None, _p(c(grad_alpha)) if depth else None, _p(r.uv), _p(r.mass),
       _p(r.absgrad))
    return r
