"""CPU oracle of Mip-Splatting's 3-D filter: rasterize(..., filter3d=f) and compute_filter3d.  TEST INFRASTRUCTURE.

The filter only changes the per-gaussian stage: Sigma_world is formed from the variances v_k + f^2 (v_k = exp(s_k)^2)
and the opacity sigmoid(o) becomes sigmoid(o) * coef, coef = sqrt(prod_k v_k / (v_k + f^2)), before the anti-aliased
mode's rho (filter3d_oracle.c).  The render stage is the existing render oracle fed those (depth_alpha_oracle's walk,
which also gives the depth and alpha maps):

    o = rasterize(sc_inputs..., filter3d, antialiased)   # o.coef, o.t, o.sigma, o.rho, o.opacity; image, depth, alpha
    d = rasterize_backward(o, G, G_depth, G_alpha)        # gradients of <G,image> + <Gd,depth> + <Ga,alpha>
    f = sample(xyz, Ts, Ks, widths, heights)              # compute_filter3d, fp32 in kernel order

fp32 reproduces the production branch bit for bit (+0.25 dilation inside the renderer, fast exp, 1/255 skip).  fp64 is
the smooth branch for finite differences (with antialiased: the dilated covariance, as antialiased_oracle does).

Backward: Sigma = R diag(v + F) R^T is the plain Sigma at the filtered log-scale s' = 1/2 log(v + F), so the plain
oracle's VJP evaluated at s' gives the quaternion gradient and d/ds', and d s'_k / d s_k = t_k.  The opacity factor adds
d coef / d s_k = coef (1 - t_k), 1 - t_k = F / (v_k + F).
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
from tests import antialiased_oracle as aao
from tests import depth_alpha_oracle as dao

HERE = Path(__file__).resolve().parent
ORACLE = HERE.parent / "oracle"
_lib = None


def build() -> Path:
    """Compile into a per-user cache directory outside the tree (keyed by the sources' digest)."""
    srcs = [HERE / "filter3d_oracle.c", ORACLE / "gsr_oracle.c", ORACLE / "gsr_oracle_body.inc"]
    digest = hashlib.sha256(b"".join(p.read_bytes() for p in srcs)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_filter3d_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_filter3d_oracle_{digest}.so"
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
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _suffix(dt):
    return {np.dtype(np.float32): "_f32", np.dtype(np.float64): "_f64"}[np.dtype(dt)]


def filtered_conic(xyz_cam, quaternion, scale, filter3d, T, K, visible, e=None):
    """-> conic [N,3], coef [N], t [N,3] in the dtype of scale (rows of invisible gaussians 0; fp32: the kernel's
    operations bit for bit).  e: exp(scale) [N,3] to use instead of the host's exp (the device's expf can differ from
    it by an ulp)."""
    dt = np.dtype(scale.dtype)
    c = lambda a: np.ascontiguousarray(a, dt)  # noqa: E731
    N = scale.shape[0]
    conic, coef, t = np.zeros((N, 3), dt), np.zeros(N, dt), np.zeros((N, 3), dt)
    getattr(lib(), "f3d_project" + _suffix(dt))(
        C.c_int(N), _p(c(quaternion)), _p(c(scale)), _p(c(np.reshape(filter3d, -1))), _p(c(xyz_cam)), _p(c(K)),
        _p(c(T)), _p(np.ascontiguousarray(visible, np.uint8)), _p(None if e is None else c(e)), _p(conic), _p(coef),
        _p(t))
    return conic, coef, t


def sample(xyz, Ts, Ks, widths, heights, near=0.2, margin=0.15, variance=0.2):
    """compute_filter3d's result (float32 [N]) in the kernel's fp32 operations."""
    f32 = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    i32 = lambda a: np.ascontiguousarray(np.reshape(a, -1), np.int32)  # noqa: E731
    xyz, Ts, Ks = f32(xyz), f32(np.reshape(Ts, (-1, 16))), f32(np.reshape(Ks, (-1, 9)))
    out = np.zeros(xyz.shape[0], np.float32)
    lib().f3d_sample_f32(C.c_int(xyz.shape[0]), _p(xyz), C.c_int(Ts.shape[0]), _p(Ts), _p(Ks), _p(i32(widths)),
                         _p(i32(heights)), C.c_float(near), C.c_float(margin), C.c_float(variance), _p(out))
    return out


def mip_splatting_loop(xyz, Ts, Ks, widths, heights, near=0.2, margin=0.15, variance=0.2):
    """Mip-Splatting's published computation restated in float64 numpy: minimum camera-frame depth over the cameras
    that see a point and, separately, the maximum focal_x over all cameras; unseen points get the largest distance of
    the seen ones.  Agrees with `sample` when every camera has the same focal length (cx = W/2 there)."""
    xyz = np.asarray(xyz, np.float64)
    dist = np.full(len(xyz), 1e5)
    valid = np.zeros(len(xyz), bool)
    focal = 0.0
    for T, K, W, H in zip(Ts, Ks, widths, heights):
        T, K = np.asarray(T, np.float64), np.asarray(K, np.float64)
        p = xyz @ T[:3, :3].T + T[:3, 3]
        z = p[:, 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            x = p[:, 0] / z * K[0, 0] + W / 2.0
            y = p[:, 1] / z * K[1, 1] + H / 2.0
        ok = (z > near) & (x >= -margin * W) & (x <= (1 + margin) * W) & (y >= -margin * H) & (y <= (1 + margin) * H)
        dist[ok] = np.minimum(dist[ok], z[ok])
        valid |= ok
        focal = max(focal, float(K[0, 0]))
    if valid.any():
        dist[~valid] = dist[valid].max()
    else:
        dist[:] = 0.0
    return dist / focal * np.sqrt(variance)


def rasterize(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, filter3d, antialiased=False, near_thresh=0.3,
              far_thresh=500.0, cull_mask_padding=100.0, mh_dist=3.0, background=None, e=None, sigma=None):
    """cpu_oracle.rasterize (precomputed SH) with the 3-D filter.  Besides its fields: o.sigma (sigmoid(o)), o.coef,
    o.t [M,3], o.rho (1 without antialiased), o.opacity = the opacity the renderer was fed, o.z, o.depth, o.alpha.
    e: exp(scale) to use in the filtered stage instead of the host's exp (filtered_conic); sigma: sigmoid(opacity) [N]
    to use instead of the host's (the device's expf can differ from the host's by an ulp)."""
    dt = np.dtype(xyz.dtype)
    if background is None:
        background = np.zeros(3, dt)
    pg = orc.project(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, near_thresh, far_thresh, cull_mask_padding)
    keep = pg.visible.astype(bool)
    conic, coef, t = filtered_conic(pg.xyz_cam, quaternion, scale, np.asarray(filter3d, dt), T, K, pg.visible, e)
    o = SimpleNamespace(pg=pg, keep=keep, culling_mask=~keep, H=H, W=W, dtype=dt, background=np.asarray(background, dt),
                        inputs=(xyz, quaternion, scale, opacity, rgb, sh, T, K), per_pixel=False, view_dirs=None,
                        filter3d=np.asarray(filter3d, dt).reshape(-1), antialiased=antialiased)
    o.uv, o.conic, o.xyz_cam, o.rgb = pg.uv[keep], conic[keep], pg.xyz_cam[keep], pg.rgb[keep]
    o.sigma = pg.opacity[keep] if sigma is None else np.asarray(sigma, dt).reshape(-1)[keep]
    o.coef, o.t = coef[keep], t[keep]
    o.base = (o.sigma * o.coef).astype(dt)            # one rounding, as the kernel's __fmul_rn
    if antialiased:
        o.rho, o.opacity = aao.compensate(o.conic, o.base)
    else:
        o.rho, o.opacity = np.ones(len(o.base), dt), o.base
    o.z = np.ascontiguousarray(o.xyz_cam[:, 2])
    o.sorted_idx, o.ranges = orc.tile_lists(o.uv, o.xyz_cam, o.conic, (W + 15) // 16, (H + 15) // 16, mh_dist)
    o.render_conic = (np.ascontiguousarray(o.conic + aao.DILATION) if antialiased and dt == np.float64 else o.conic)
    o.image, o.n, o.wlast, o.depth, o.alpha = dao.render_forward(o.uv, o.opacity, o.rgb, o.render_conic, o.z, o.ranges,
                                                                 o.sorted_idx, o.background, H, W)
    return o


def filtered_scale(scale, filter3d):
    """(s' = 1/2 log(v + F), t = v / (v + F) or 1 where F == 0, 1 - t = F / (v + F)) in float64."""
    s = np.asarray(scale, np.float64)
    F = np.asarray(filter3d, np.float64).reshape(-1, 1) ** 2
    v = np.exp(2.0 * s)
    vp = v + F
    with np.errstate(divide="ignore", invalid="ignore"):
        sp = 0.5 * np.log(vp)
        t = np.where(F == 0, 1.0, v / vp)
        omt = np.where(F == 0, 0.0, F / vp)
    return sp, t, omt


def project_backward(o, g_rgb, g_opa, g_uv, g_conic, g_z=None):
    """VJP of the filtered per-gaussian stage from render-stage rows over all N gaussians (float64); g_opa is the
    gradient on the opacity the renderer was fed (sigmoid(o) * coef [* rho])."""
    N = o.inputs[0].shape[0]
    full = lambda a, shape=(): np.zeros((N,) + shape)  # noqa: E731
    rho, sigma, coef, conic = full(None), full(None), full(None), full(None, (3,))
    rho[o.keep], sigma[o.keep], coef[o.keep], conic[o.keep] = o.rho, o.sigma, o.coef, o.conic
    g_opa = np.asarray(g_opa, np.float64).reshape(-1)
    g_conic = np.asarray(g_conic, np.float64).reshape(N, 3)
    if o.antialiased:
        g_conic = g_conic + (g_opa * sigma * coef)[:, None] * aao.rho_grad(conic, rho)
        g_opa = g_opa * rho
    xyz, quaternion, scale, opacity, rgb, sh, T, K = o.inputs
    sp, t, omt = filtered_scale(scale, o.filter3d)
    o2 = SimpleNamespace(**vars(o))
    o2.inputs = (xyz, quaternion, sp.astype(o.dtype), opacity, rgb, sh, T, K)
    d = dao.project_backward(o2, g_rgb, g_opa * coef, g_uv, g_conic, np.zeros(N) if g_z is None else g_z)
    d.scale = d.scale * t + (g_opa * sigma * coef)[:, None] * omt
    return d


def rasterize_backward(o, grad_image, grad_depth=None, grad_alpha=None):
    """Gradients (float64) of every parameter and of the compact uv, with the render-stage rows d.render (opacity: the
    gradient on the opacity the renderer was fed), their masses d.mass and d.near, as depth_alpha_oracle's."""
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
