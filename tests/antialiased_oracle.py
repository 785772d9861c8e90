"""CPU oracle of rasterize(antialiased=True).  TEST INFRASTRUCTURE.

The mode only changes the per-gaussian stage: each splat's opacity sigmoid(o) becomes sigmoid(o) * rho with
rho = sqrt(max(det0, 0) / det) (antialiased_oracle.c).  The render stage is the existing render oracle fed the
compensated opacities (depth_alpha_oracle's walk, which also gives the depth and alpha maps):

    o = rasterize(sc_inputs...)                      # o.rho, o.sigma, o.opacity = compensated; image, depth, alpha
    d = rasterize_backward(o, G, G_depth, G_alpha)   # gradients of <G,image> + <Gd,depth> + <Ga,alpha>

fp32 reproduces the production branch bit for bit (+0.25 dilation inside the renderer, fast exp, 1/255 skip).
fp64 is a smooth branch FOR FINITE DIFFERENCES WITH THE DILATION ON: the oracle's own fp64 renderer applies no
dilation (where rho would be 1 and a gradient check of the mode vacuous), so it is fed the dilated covariance
conic + (0.25, 0, 0.25) instead; exp, no 1/255 skip.  The dilation is a constant, so the render backward's conic
gradient is the same for the dilated and the undilated covariance.
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
from tests import depth_alpha_oracle as dao

HERE = Path(__file__).resolve().parent
DILATION = np.array([0.25, 0.0, 0.25])
_lib = None


def build() -> Path:
    """Compile into a per-user cache directory outside the tree (keyed by the source's digest)."""
    src = HERE / "antialiased_oracle.c"
    digest = hashlib.sha256(src.read_bytes()).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_antialiased_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_antialiased_oracle_{digest}.so"
    if not out.exists():
        tmp = out.with_suffix(f".{os.getpid()}.tmp")
        subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-mfma", "-shared", "-fPIC", str(src), "-o", str(tmp),
                        "-lm"], check=True, capture_output=True)
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
    return _lib


def compensate(conic, opacity):
    """-> (rho, opacity * rho), in the dtype of conic (fp32: the kernel's operations bit for bit)."""
    dt = np.dtype(conic.dtype)
    conic = np.ascontiguousarray(conic, dt).reshape(-1, 3)
    opacity = np.ascontiguousarray(opacity, dt).reshape(-1)
    rho, out = np.zeros(len(conic), dt), np.zeros(len(conic), dt)
    fn = getattr(lib(), "aa_compensate" + ("_f32" if dt == np.float32 else "_f64"))
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    fn(C.c_int(len(conic)), p(conic), p(opacity), p(rho), p(out))
    return rho, out


def rho_grad(conic, rho):
    """d rho / d (c0, c1, c2) [M,3] (float64) as derived over det, 0 where rho == 0 (no gradient goes through rho
    there).  With A = c0 + 1/4, C = c2 + 1/4, bh = c1 / 2, det = A C - bh^2:
        d rho/d c0 = (c2 - rho^2 C) / (2 rho det),  d rho/d c2 = (c0 - rho^2 A) / (2 rho det),
        d rho/d c1 = -bh (1 - rho^2) / (2 rho det)."""
    c0, c1, c2 = (np.asarray(conic, np.float64)[:, k] for k in range(3))
    r = np.asarray(rho, np.float64)
    A, Cc, bh = c0 + 0.25, c2 + 0.25, 0.5 * c1
    det = A * Cc - bh * bh
    live = r > 0
    k = np.where(live, 1.0 / (2.0 * np.where(live, r, 1.0) * det), 0.0)
    return np.stack([(c2 - r * r * Cc) * k, -bh * (1 - r * r) * k, (c0 - r * r * A) * k], 1)


def rasterize(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, near_thresh=0.3, far_thresh=500.0,
              cull_mask_padding=100.0, mh_dist=3.0, background=None):
    """cpu_oracle.rasterize (precomputed SH) in the anti-aliased mode.  Besides its fields: o.sigma (sigmoid(o)),
    o.rho, o.opacity = the compensated opacity the renderer was fed, o.z, o.depth and o.alpha [H,W]."""
    dt = np.dtype(xyz.dtype)
    if background is None:
        background = np.zeros(3, dt)
    pg = orc.project(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, near_thresh, far_thresh, cull_mask_padding)
    keep = pg.visible.astype(bool)
    o = SimpleNamespace(pg=pg, keep=keep, culling_mask=~keep, H=H, W=W, dtype=dt, background=np.asarray(background, dt),
                        inputs=(xyz, quaternion, scale, opacity, rgb, sh, T, K), per_pixel=False, view_dirs=None)
    o.uv, o.conic, o.xyz_cam, o.rgb = pg.uv[keep], pg.conic[keep], pg.xyz_cam[keep], pg.rgb[keep]
    o.sigma = pg.opacity[keep]
    o.rho, o.opacity = compensate(o.conic, o.sigma)
    o.z = np.ascontiguousarray(o.xyz_cam[:, 2])
    o.sorted_idx, o.ranges = orc.tile_lists(o.uv, o.xyz_cam, o.conic, (W + 15) // 16, (H + 15) // 16, mh_dist)
    o.render_conic = o.conic if dt == np.float32 else np.ascontiguousarray(o.conic + DILATION)
    o.image, o.n, o.wlast, o.depth, o.alpha = dao.render_forward(o.uv, o.opacity, o.rgb, o.render_conic, o.z, o.ranges,
                                                                 o.sorted_idx, o.background, H, W)
    return o


def project_backward(o, g_rgb, g_opa, g_uv, g_conic, g_z=None):
    """VJP of the anti-aliased per-gaussian stage from render-stage rows over all N gaussians (float64); g_opa is the
    gradient on the compensated opacity: sigmoid(o) receives g_opa * rho, the covariance g_opa * sigmoid(o) *
    grad(rho)."""
    N = o.inputs[0].shape[0]
    rho, sigma, conic = np.zeros(N), np.zeros(N), np.zeros((N, 3))
    rho[o.keep], sigma[o.keep], conic[o.keep] = o.rho, o.sigma, o.conic
    g_opa = np.asarray(g_opa, np.float64).reshape(-1)
    g_conic = np.asarray(g_conic, np.float64).reshape(N, 3) + (g_opa * sigma)[:, None] * rho_grad(conic, rho)
    return dao.project_backward(o, g_rgb, g_opa * rho, g_uv, g_conic, np.zeros(N) if g_z is None else g_z)


def rasterize_backward(o, grad_image, grad_depth=None, grad_alpha=None):
    """Gradients (float64) of every parameter and of the compact uv, with the render-stage rows d.render (opacity:
    the gradient on the compensated opacity), their masses d.mass and d.near, as depth_alpha_oracle's."""
    N = o.inputs[0].shape[0]
    H, W = o.n.shape
    grad_depth = np.zeros((H, W)) if grad_depth is None else grad_depth
    grad_alpha = np.zeros((H, W)) if grad_alpha is None else grad_alpha
    g, m, near = dao.render_backward(SimpleNamespace(**dict(vars(o), conic=o.render_conic)), grad_image, grad_depth,
                                     grad_alpha)

    def full(a):
        out = np.zeros((N,) + a.shape[1:], np.float64)
        out[o.keep] = a
        return out

    render = SimpleNamespace(**{k: full(v) for k, v in vars(g).items()})
    mass = SimpleNamespace(**{k: full(v) for k, v in vars(m).items()})
    d = project_backward(o, render.rgb, render.opacity, render.uv, render.conic, render.z)
    d.uv, d.render, d.mass, d.near = g.uv, render, mass, near
    return d
