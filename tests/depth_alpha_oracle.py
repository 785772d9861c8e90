"""CPU oracle of rasterize(render_depth_alpha=True): depth and alpha maps and their gradients.  TEST INFRASTRUCTURE.

Extends oracle/cpu_oracle.py (which it builds on and does not change) with depth_alpha_oracle.c:

    o = rasterize(sc_inputs...)                       # cpu_oracle.rasterize + o.depth, o.alpha [H,W]
    d = rasterize_backward(o, G, G_depth, G_alpha)    # gradients of <G,image> + <Gd,depth> + <Ga,alpha>

d.render holds the render-stage per-gaussian sums (rgb, opacity, uv, conic and z, the gradient on camera-frame z) and
d.mass their masses (see orc_render_backward_da), for tests/gradrows.py's per-row bounds.
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
    srcs = [HERE / "depth_alpha_oracle.c", HERE / "depth_alpha_oracle_body.inc", ORACLE / "gsr_oracle.c",
            ORACLE / "gsr_oracle_body.inc"]
    digest = hashlib.sha256(b"".join(p.read_bytes() for p in srcs)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_depth_alpha_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_depth_alpha_oracle_{digest}.so"
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


def render_forward(uvs, opacity, rgb, conic, z, ranges, sorted_idx, background, H, W):
    """-> image [H,W,3], n [H,W] int32, wlast [H,W], depth [H,W], alpha [H,W] (precomputed colours rgb [G,3])."""
    dt = uvs.dtype
    c = lambda a: np.ascontiguousarray(a, dtype=dt)  # noqa: E731
    image, n, w = np.zeros((H, W, 3), dt), np.zeros((H, W), np.int32), np.zeros((H, W), dt)
    depth, alpha = np.zeros((H, W), dt), np.zeros((H, W), dt)
    getattr(lib(), "orc_render_forward_da" + _suffix(dt))(
        C.c_int(H), C.c_int(W), _p(c(uvs)), _p(c(opacity).reshape(-1)), _p(c(rgb)), _p(c(conic)), _p(c(z)),
        _p(np.ascontiguousarray(ranges, np.int32)), _p(np.ascontiguousarray(sorted_idx, np.int32)), _p(c(background)),
        _p(n), _p(w), _p(image), _p(depth), _p(alpha))
    return image, n, w, depth, alpha


def rasterize(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, near_thresh=0.3, far_thresh=500.0,
              cull_mask_padding=100.0, mh_dist=3.0, background=None):
    """cpu_oracle.rasterize (precomputed SH) + o.depth, o.alpha [H,W] and o.z, the compact camera-frame z."""
    o = orc.rasterize(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, near_thresh, far_thresh,
                      cull_mask_padding, mh_dist, background=background)
    o.z = np.ascontiguousarray(o.xyz_cam[:, 2])
    image, n, w, o.depth, o.alpha = render_forward(o.uv, o.opacity, o.rgb, o.conic, o.z, o.ranges, o.sorted_idx,
                                                   o.background, H, W)
    # the extended walk is the oracle's own: same image, counts and final weights
    assert np.array_equal(image, o.image) and np.array_equal(n, o.n) and np.array_equal(w, o.wlast)
    return o


def render_backward(o, grad_image, grad_depth, grad_alpha):
    """Render-stage sums over the compact gaussians (float64): rgb [M,3], opacity [M], uv [M,2], conic [M,3], z [M],
    their masses (same shapes) and near [H,W] (bool), as cpu_oracle.render_backward(mass=True)."""
    dt = o.dtype
    c = lambda a: np.ascontiguousarray(a, dtype=dt)  # noqa: E731
    H, W = o.n.shape
    M = o.uv.shape[0]
    g = SimpleNamespace(rgb=np.zeros((M, 3)), opacity=np.zeros(M), uv=np.zeros((M, 2)), conic=np.zeros((M, 3)),
                        z=np.zeros(M))
    m = SimpleNamespace(**{k: np.zeros_like(v) for k, v in vars(g).items()})
    near = np.zeros((H, W), np.uint8)
    chunk = orc.REF_CHUNK[(np.dtype(dt).type, 1)]
    getattr(lib(), "orc_render_backward_da" + _suffix(dt))(
        C.c_int(H), C.c_int(W), C.c_int(chunk), _p(c(o.uv)), _p(c(o.opacity).reshape(-1)), _p(c(o.rgb)),
        _p(c(o.conic)), _p(c(o.z)), _p(np.ascontiguousarray(o.ranges, np.int32)),
        _p(np.ascontiguousarray(o.sorted_idx, np.int32)), _p(c(o.background)), _p(np.ascontiguousarray(o.n, np.int32)),
        _p(c(o.wlast)), _p(c(grad_image)), _p(c(grad_depth)), _p(c(grad_alpha)), _p(g.rgb), _p(g.opacity), _p(g.uv),
        _p(g.conic), _p(g.z), _p(m.rgb), _p(m.opacity), _p(m.uv), _p(m.conic), _p(m.z), _p(near))
    return g, m, near.astype(bool)


def project_backward(o, g_rgb, g_opa, g_uv, g_conic, g_z):
    """cpu_oracle.project_backward with the gradient on camera-frame z (all [N, .] rows, float64): z = T[2,:3] . xyz
    + t_z, so grad_xyz += T[2,:3] * g_z; no gradient goes to the pose."""
    d = orc.project_backward(o, g_rgb, g_opa, g_uv, g_conic)
    T = np.asarray(o.inputs[6], np.float64)
    d.xyz = d.xyz + np.asarray(g_z, np.float64).reshape(-1, 1) * T[2, :3]
    return d


def rasterize_backward(o, grad_image, grad_depth, grad_alpha):
    """Gradients (float64) of xyz, quaternion, scale, opacity, rgb, sh and of the compact uv for the loss
    <G,image> + <Gd,depth> + <Ga,alpha>; d.render / d.mass: render-stage rows over all N gaussians (zero rows for
    culled ones) and their masses; d.near as in cpu_oracle.rasterize_backward."""
    N = o.inputs[0].shape[0]
    g, m, near = render_backward(o, grad_image, grad_depth, grad_alpha)

    def full(a):
        out = np.zeros((N,) + a.shape[1:], np.float64)
        out[o.keep] = a
        return out

    render = SimpleNamespace(**{k: full(v) for k, v in vars(g).items()})
    mass = SimpleNamespace(**{k: full(v) for k, v in vars(m).items()})
    d = project_backward(o, render.rgb, render.opacity, render.uv, render.conic, render.z)
    d.uv, d.render, d.mass, d.near = g.uv, render, mass, near
    return d
