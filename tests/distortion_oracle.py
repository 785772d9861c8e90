"""CPU oracle of radial-tangential lens distortion: rasterize(..., distortion=k).  TEST INFRASTRUCTURE.

The lens only changes the per-gaussian stage: the projected mean, the Jacobian of the 2-D covariance and one cull
rule (s >= r2_max), all restated in fp64 by distortion_oracle.c.  The 3-D filter and the anti-aliased opacity act
on the result as in filter3d_oracle / antialiased_oracle, and the render stage is the existing render oracle
(depth_alpha_oracle's walk, which also gives the depth and alpha maps):

    o = rasterize(xyz, ..., T, K, H, W, k, antialiased=..., filter3d=...)   # fp64
    d = rasterize_backward(o, G, G_depth, G_alpha)
    r2_max(k)                                                                # numpy.roots, fp64
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
from tests import filter3d_oracle as fo

HERE = Path(__file__).resolve().parent
ORACLE = HERE.parent / "oracle"
_lib = None


def build() -> Path:
    """Compile into a per-user cache directory outside the tree (keyed by the sources' digest)."""
    srcs = [HERE / "distortion_oracle.c", ORACLE / "gsr_oracle.c", ORACLE / "gsr_oracle_body.inc"]
    digest = hashlib.sha256(b"".join(p.read_bytes() for p in srcs)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_distortion_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_distortion_oracle_{digest}.so"
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


def _d(a):
    return None if a is None else np.ascontiguousarray(a, np.float64)


def r2_max(k):
    """The smallest positive real root s of 1 + 3 k1 s + 5 k2 s^2 + 7 k3 s^3 (k = k1 k2 p1 p2 k3), by numpy.roots, in
    fp64 (+inf when there is none)."""
    k = np.asarray(k, np.float64)
    coeffs = [7 * k[4], 5 * k[1], 3 * k[0], 1.0]
    while coeffs and coeffs[0] == 0:
        coeffs.pop(0)
    best = np.inf
    if len(coeffs) > 1:
        for r in np.roots(coeffs):
            if abs(r.imag) <= 1e-9 * max(1.0, abs(r.real)) and r.real > 0:
                best = min(best, float(r.real))
    return best


def project_point(p, K, k):
    """((u, v), s) of one camera-frame point (distortion_oracle.c dt_project_point_f64)."""
    uv, s = np.zeros(2), np.zeros(1)
    lib().dt_project_point_f64(_p(_d(p)), _p(_d(K)), _p(_d(k)), _p(uv), _p(s))
    return uv, float(s[0])


def jacobian_vjp(p, fx, fy, k, gJ, guv):
    """(J [2,3], J^T guv + sum_ij gJ_ij dJ_ij / dp [3])."""
    J, g = np.zeros(6), np.zeros(3)
    lib().dt_jacobian_vjp_f64(_p(_d(p)), C.c_double(fx), C.c_double(fy), _p(_d(k)), _p(_d(np.reshape(gJ, 6))),
                              _p(_d(guv)), _p(J), _p(g))
    return J.reshape(2, 3), g


def project(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, kc, near_thresh, far_thresh, cull_mask_padding):
    """orc.project for the distorted camera (fp64, all N rows); kc = (k1, k2, p1, p2, k3, r2_max)."""
    N = xyz.shape[0]
    n_sh = 1 if sh is None else sh.shape[2] + 1
    cam = orc.camera_centre(T)
    out = SimpleNamespace(xyz_cam=np.zeros((N, 3)), uv=np.zeros((N, 2)), conic=np.zeros((N, 3)), opacity=np.zeros(N),
                          rgb=np.zeros((N, 3)), visible=np.zeros(N, np.uint8), s=np.zeros(N), cam_centre=cam,
                          n_sh=n_sh)
    lib().dt_project_f64(C.c_int(N), C.c_int(n_sh), _p(_d(xyz)), _p(_d(quaternion)), _p(_d(scale)),
                         _p(_d(np.reshape(opacity, -1))), _p(_d(rgb)), _p(_d(sh)), _p(_d(T)), _p(_d(K)), _p(cam),
                         _p(_d(kc)), C.c_double(W), C.c_double(H), C.c_double(near_thresh), C.c_double(far_thresh),
                         C.c_double(cull_mask_padding), _p(out.xyz_cam), _p(out.uv), _p(out.conic), _p(out.opacity),
                         _p(out.rgb), _p(out.visible), _p(out.s))
    return out


def rasterize(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, k, antialiased=False, filter3d=None,
              near_thresh=0.3, far_thresh=500.0, cull_mask_padding=100.0, mh_dist=3.0, background=None, smax=None):
    """The fp64 distorted forward.  Besides the render fields (image, depth, alpha, n, wlast): o.pg (all rows), o.keep,
    o.uv / o.conic / o.z (compact), o.sigma, o.coef, o.t, o.rho and o.opacity (the opacity the renderer was fed).
    smax: the cull limit to use (default: r2_max(k))."""
    xyz = np.asarray(xyz, np.float64)
    N = xyz.shape[0]
    if background is None:
        background = np.zeros(3)
    f = np.zeros(N) if filter3d is None else np.asarray(filter3d, np.float64).reshape(-1)
    sp, t, omt = fo.filtered_scale(scale, f)
    kc = np.append(np.asarray(k, np.float64), r2_max(k) if smax is None else smax)
    pg = project(xyz, quaternion, sp, opacity, rgb, sh, T, K, H, W, kc, near_thresh, far_thresh, cull_mask_padding)
    keep = pg.visible.astype(bool)
    o = SimpleNamespace(pg=pg, keep=keep, culling_mask=~keep, H=H, W=W, dtype=np.dtype(np.float64),
                        background=np.asarray(background, np.float64), kc=kc, antialiased=antialiased,
                        inputs=(xyz, quaternion, scale, opacity, rgb, sh, T, K), sp=sp, t_full=t, omt=omt,
                        coef_full=np.sqrt(np.prod(t, 1)))
    o.uv, o.conic, o.xyz_cam, o.rgb = pg.uv[keep], pg.conic[keep], pg.xyz_cam[keep], pg.rgb[keep]
    o.sigma, o.coef, o.t = pg.opacity[keep], o.coef_full[keep], t[keep]
    o.base = o.sigma * o.coef
    if antialiased:
        o.rho, o.opacity = aao.compensate(o.conic, o.base)
    else:
        o.rho, o.opacity = np.ones(len(o.base)), o.base
    o.z = np.ascontiguousarray(o.xyz_cam[:, 2])
    o.sorted_idx, o.ranges = orc.tile_lists(o.uv, o.xyz_cam, o.conic, (W + 15) // 16, (H + 15) // 16, mh_dist)
    o.render_conic = np.ascontiguousarray(o.conic + aao.DILATION) if antialiased else o.conic
    o.image, o.n, o.wlast, o.depth, o.alpha = dao.render_forward(o.uv, o.opacity, o.rgb, o.render_conic, o.z, o.ranges,
                                                                 o.sorted_idx, o.background, H, W)
    return o


def project_backward(o, g_rgb, g_opa, g_uv, g_conic, g_z=None):
    """VJP of the distorted per-gaussian stage from render-stage rows over all N gaussians (float64); g_opa is the
    gradient on the opacity the renderer was fed (sigmoid(o) * coef [* rho])."""
    xyz, quaternion, scale, opacity, rgb, sh, T, K = o.inputs
    N = xyz.shape[0]
    full = lambda shape=(): np.zeros((N,) + shape)  # noqa: E731
    rho, sigma, conic = full(), full(), full((3,))
    rho[o.keep], sigma[o.keep], conic[o.keep] = o.rho, o.sigma, o.conic
    coef = o.coef_full
    g_opa = np.asarray(g_opa, np.float64).reshape(-1)
    g_conic = np.asarray(g_conic, np.float64).reshape(N, 3)
    if o.antialiased:
        g_conic = g_conic + (g_opa * sigma * coef)[:, None] * aao.rho_grad(conic, rho)
        g_opa = g_opa * rho
    n_sh = o.pg.n_sh
    d = SimpleNamespace(xyz=np.zeros((N, 3)), quaternion=np.zeros((N, 4)), scale=np.zeros((N, 3)),
                        opacity=np.zeros((N, 1)), rgb=np.zeros((N, 3)),
                        sh=None if sh is None else np.zeros((N, 3, n_sh - 1)))
    g_z = np.zeros(N) if g_z is None else np.asarray(g_z, np.float64).reshape(-1)
    lib().dt_project_backward_f64(
        C.c_int(N), C.c_int(n_sh), _p(_d(xyz)), _p(_d(quaternion)), _p(_d(o.sp)), _p(_d(np.reshape(opacity, -1))),
        _p(_d(sh)), _p(_d(T)), _p(_d(K)), _p(o.pg.cam_centre), _p(o.kc), _p(np.ascontiguousarray(o.pg.visible)),
        _p(_d(np.reshape(g_rgb, (N, 3)))), _p(_d(g_opa * coef)), _p(_d(np.reshape(g_uv, (N, 2)))), _p(_d(g_conic)),
        _p(_d(g_z)), _p(d.xyz), _p(d.quaternion), _p(d.scale), _p(d.opacity), _p(d.rgb), _p(d.sh))
    d.scale = d.scale * o.t_full + (g_opa * sigma * coef)[:, None] * o.omt
    return d


def rasterize_backward(o, grad_image, grad_depth=None, grad_alpha=None):
    """Gradients (float64) of every parameter and of the compact uv, with the render-stage rows d.render and their
    masses d.mass, as filter3d_oracle.rasterize_backward."""
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
