"""ctypes front-end of the CPU oracle (oracle/gsr_oracle.c).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu-baseline leg import this module; the product
package gaussian_splatting_b200 never does.

    o = rasterize(params, T, K, H, W, ...)        # full forward of splat_py.rasterize.rasterize
    g = rasterize_backward(o, grad_image)          # gradients of every parameter

All arrays are numpy; dtype float32 selects the reference's production branch (dilation, fast exp,
1/255 skip), float64 its gradcheck branch.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
from pathlib import Path
from types import SimpleNamespace

import numpy as np

HERE = Path(__file__).resolve().parent
BUILD = HERE / "_build"
_lib = None

REF_CHUNK = {(np.float32, 1): 960, (np.float32, 4): 576, (np.float32, 9): 320, (np.float32, 16): 160,
             (np.float64, 1): 320, (np.float64, 4): 160, (np.float64, 9): 128, (np.float64, 16): 64}


def build(force: bool = False) -> Path:
    BUILD.mkdir(exist_ok=True)
    srcs = [HERE / "gsr_oracle.c", HERE / "gsr_oracle_body.inc"]
    digest = hashlib.sha256(b"".join(p.read_bytes() for p in srcs)).hexdigest()[:16]
    out = BUILD / "libgsr_oracle.so"
    stamp = BUILD / "oracle.sha"
    if force or not out.exists() or not stamp.exists() or stamp.read_text() != digest:
        cmd = ["gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-mfma", "-shared", "-fPIC", str(srcs[0]), "-o",
               str(out), "-lm"]
        subprocess.run(cmd, check=True, capture_output=True)
        stamp.write_text(digest)
    return out


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.orc_tile_lists.restype = C.c_int
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _suffix(dtype):
    return {np.dtype(np.float32): "_f32", np.dtype(np.float64): "_f64"}[np.dtype(dtype)]


def _real(dtype):
    return C.c_float if np.dtype(dtype) == np.float32 else C.c_double


def camera_centre(T):
    T64 = np.ascontiguousarray(T, dtype=np.float64)
    cam = np.zeros(3, dtype=np.float64)
    lib().orc_camera_centre(_p(T64), _p(cam))
    return cam


def project(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, near_thresh, far_thresh, cull_mask_padding):
    """Per-gaussian chain for all N gaussians (splat_py/rasterize.py:29-93)."""
    dt = xyz.dtype
    N = xyz.shape[0]
    n_sh = 1 if sh is None else sh.shape[2] + 1
    r = _real(dt)
    c = lambda a: None if a is None else np.ascontiguousarray(a, dtype=dt)  # noqa: E731
    xyz, quaternion, scale, rgb, sh, T, K = map(c, (xyz, quaternion, scale, rgb, sh, T, K))
    opacity = c(opacity).reshape(-1)
    cam = camera_centre(T).astype(dt)
    out = SimpleNamespace(
        xyz_cam=np.zeros((N, 3), dt), uv=np.zeros((N, 2), dt), conic=np.zeros((N, 3), dt),
        opacity=np.zeros(N, dt), rgb=np.zeros((N, 3), dt), visible=np.zeros(N, np.uint8), cam_centre=cam, n_sh=n_sh)
    fn = getattr(lib(), "orc_project" + _suffix(dt))
    fn(C.c_int(N), C.c_int(n_sh), _p(xyz), _p(quaternion), _p(scale), _p(opacity), _p(rgb), _p(sh), _p(T), _p(K),
       _p(cam), r(W), r(H), r(near_thresh), r(far_thresh), r(cull_mask_padding), _p(out.xyz_cam), _p(out.uv),
       _p(out.conic), _p(out.opacity), _p(out.rgb), _p(out.visible))
    return out


def tile_lists(uvs, xyz_cam, conic, n_tiles_x, n_tiles_y, mh_dist):
    """get_sorted_gaussian_list (src/tile_culling.cu:244-340): -> (sorted_idx int32 [P], ranges int32 [T+1])."""
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
    uvs, xyz_cam, conic = f(uvs), f(xyz_cam), f(conic)
    N = uvs.shape[0]
    P = lib().orc_tile_lists(C.c_int(N), _p(uvs), _p(xyz_cam), _p(conic), C.c_int(n_tiles_x), C.c_int(n_tiles_y),
                             C.c_float(mh_dist), None, None)
    sorted_idx = np.zeros(max(P, 1), np.int32)
    ranges = np.zeros(n_tiles_x * n_tiles_y + 1, np.int32)
    lib().orc_tile_lists(C.c_int(N), _p(uvs), _p(xyz_cam), _p(conic), C.c_int(n_tiles_x), C.c_int(n_tiles_y),
                         C.c_float(mh_dist), _p(sorted_idx), _p(ranges))
    return sorted_idx[:P], ranges


def render_forward(uvs, opacity, rgb, conic, view_dirs, ranges, sorted_idx, background, H, W, rows=None):
    """render_tiles_cuda (src/render.cu:191-422): -> (image [H,W,3], n [H,W] int32, wlast [H,W])."""
    dt = uvs.dtype
    c = lambda a: np.ascontiguousarray(a, dtype=dt)  # noqa: E731
    n_sh = rgb.shape[2] if rgb.ndim == 3 else 1
    image = np.zeros((H, W, 3), dt)
    n = np.zeros((H, W), np.int32)
    w = np.zeros((H, W), dt)
    vd = c(view_dirs) if n_sh > 1 else None
    r0, r1 = (0, H) if rows is None else rows
    fn = getattr(lib(), "orc_render_forward" + _suffix(dt))
    fn(C.c_int(H), C.c_int(W), C.c_int(n_sh), _p(c(uvs)), _p(c(opacity).reshape(-1)), _p(c(rgb)), _p(c(conic)), _p(vd),
       _p(np.ascontiguousarray(ranges, np.int32)), _p(np.ascontiguousarray(sorted_idx, np.int32)), _p(c(background)),
       C.c_int(r0), C.c_int(r1), _p(n), _p(w), _p(image))
    return image, n, w


def render_backward(uvs, opacity, rgb, conic, view_dirs, ranges, sorted_idx, background, n, w, grad_image, rows=None,
                    mass=False):
    """render_tiles_backward_cuda (src/render_backward.cu:287-595): float64 sums
    -> (g_rgb [G,3(,K)], g_opacity [G,1], g_uv [G,2], g_conic [G,3]).  mass=True appends a namespace of the same
    four shapes (rgb, opacity, uv, conic) holding, per entry, the sum over the terms added to it of the magnitudes
    of each term's parts (|term| for rgb; see orc_render_backward), and
    near (bool [H,W]): the pixels whose walk meets an alpha within a relative 3e-5 of the 1/255 skip threshold
    (fp32), where an implementation with another exp may skip a different set of splats."""
    dt = uvs.dtype
    c = lambda a: np.ascontiguousarray(a, dtype=dt)  # noqa: E731
    H, W = n.shape
    G = uvs.shape[0]
    n_sh = rgb.shape[2] if rgb.ndim == 3 else 1
    g_rgb = np.zeros(rgb.shape, np.float64)
    g_opa = np.zeros((G, 1), np.float64)
    g_uv = np.zeros((G, 2), np.float64)
    g_conic = np.zeros((G, 3), np.float64)
    m = SimpleNamespace(rgb=np.zeros_like(g_rgb), opacity=np.zeros_like(g_opa), uv=np.zeros_like(g_uv),
                        conic=np.zeros_like(g_conic), near=np.zeros((H, W), np.uint8)) if mass else None
    vd = c(view_dirs) if n_sh > 1 else None
    chunk = REF_CHUNK[(np.dtype(dt).type, n_sh)]
    r0, r1 = (0, H) if rows is None else rows
    fn = getattr(lib(), "orc_render_backward" + _suffix(dt))
    fn(C.c_int(H), C.c_int(W), C.c_int(n_sh), C.c_int(chunk), _p(c(uvs)), _p(c(opacity).reshape(-1)), _p(c(rgb)),
       _p(c(conic)), _p(vd), _p(np.ascontiguousarray(ranges, np.int32)), _p(np.ascontiguousarray(sorted_idx, np.int32)),
       _p(c(background)), C.c_int(r0), C.c_int(r1), _p(np.ascontiguousarray(n, np.int32)), _p(c(w)), _p(c(grad_image)),
       _p(g_rgb), _p(g_opa), _p(g_uv), _p(g_conic),
       *((_p(m.rgb), _p(m.opacity), _p(m.uv), _p(m.conic), _p(m.near)) if mass else (None,) * 5))
    if mass:
        m.near = m.near.astype(bool)
        return g_rgb, g_opa, g_uv, g_conic, m
    return g_rgb, g_opa, g_uv, g_conic


def rasterize(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, near_thresh=0.3, far_thresh=500.0,
              cull_mask_padding=100.0, mh_dist=3.0, background=None, use_sh_precompute=True, view_dirs=None):
    """splat_py.rasterize.rasterize.  Returns a namespace with every intermediate: per-gaussian stage `pg` (all N
    rows), keep (bool [N]), compact uv/conic/..., tile lists, image, n, wlast.  use_sh_precompute=False renders
    the SH coefficients per pixel (o.rgb = cat(rgb, sh) [M,3,n_sh]) along view_dirs [H,W,3], the per-pixel
    world-frame rays, which the caller supplies (splat_py/utils.py:112-123)."""
    dt = xyz.dtype
    if background is None:
        background = np.zeros(3, dt)
    per_pixel = sh is not None and not use_sh_precompute
    if per_pixel and view_dirs is None:
        raise ValueError("per-pixel SH needs the per-pixel view directions")
    pg = project(xyz, quaternion, scale, opacity, rgb, None if per_pixel else sh, T, K, H, W, near_thresh, far_thresh,
                 cull_mask_padding)
    keep = pg.visible.astype(bool)
    o = SimpleNamespace(pg=pg, keep=keep, culling_mask=~keep, H=H, W=W, dtype=dt, background=np.asarray(background, dt),
                        inputs=(xyz, quaternion, scale, opacity, rgb, sh, T, K), per_pixel=per_pixel,
                        view_dirs=np.ascontiguousarray(view_dirs, dt) if per_pixel else None)
    o.uv, o.conic, o.xyz_cam = pg.uv[keep], pg.conic[keep], pg.xyz_cam[keep]
    o.opacity, o.rgb = pg.opacity[keep], pg.rgb[keep]
    if per_pixel:
        o.rgb = np.ascontiguousarray(np.concatenate([np.asarray(rgb, dt)[keep][:, :, None], np.asarray(sh, dt)[keep]], 2))
    ntx, nty = (W + 15) // 16, (H + 15) // 16
    o.sorted_idx, o.ranges = tile_lists(o.uv, o.xyz_cam, o.conic, ntx, nty, mh_dist)
    o.image, o.n, o.wlast = render_forward(o.uv, o.opacity, o.rgb, o.conic, o.view_dirs, o.ranges, o.sorted_idx,
                                           o.background, H, W)
    return o


def project_backward(o, g_rgb, g_opa, g_uv, g_conic):
    """VJP of the per-gaussian chain from per-gaussian render-stage gradients (all [N, .] rows, float64; g_rgb is
    the gradient of the rendered colour, unused for per-pixel SH) -> namespace xyz, quaternion, scale, opacity, rgb,
    sh (float64)."""
    xyz, quaternion, scale, opacity, rgb, sh, T, K = o.inputs
    dt = o.dtype
    N = xyz.shape[0]
    n_sh = o.pg.n_sh
    c = lambda a: None if a is None else np.ascontiguousarray(a, dtype=dt)  # noqa: E731
    f = lambda a, cols: np.ascontiguousarray(np.asarray(a, np.float64).reshape(N, cols))  # noqa: E731
    d = SimpleNamespace(xyz=np.zeros((N, 3)), quaternion=np.zeros((N, 4)), scale=np.zeros((N, 3)), opacity=np.zeros((N, 1)),
                        rgb=np.zeros((N, 3)), sh=None if sh is None else np.zeros((N, 3, n_sh - 1)))
    fn = getattr(lib(), "orc_project_backward" + _suffix(dt))
    fn(C.c_int(N), C.c_int(n_sh), _p(c(xyz)), _p(c(quaternion)), _p(c(scale)), _p(c(opacity).reshape(-1)),
       _p(None if o.per_pixel else c(sh)), _p(c(T)), _p(c(K)), _p(o.pg.cam_centre.astype(dt)),
       _p(np.ascontiguousarray(o.pg.visible)), _p(f(g_rgb, 3)), _p(f(g_opa, 1)), _p(f(g_uv, 2)), _p(f(g_conic, 3)),
       _p(d.xyz), _p(d.quaternion), _p(d.scale), _p(d.opacity), _p(d.rgb), _p(d.sh))
    return d


def rasterize_backward(o, grad_image):
    """Gradients (float64) of xyz, quaternion, scale, opacity, rgb, sh and of the compact uv.  Also the render
    stage's per-gaussian sums d.render (rgb [N,3] — [N,3,n_sh] for per-pixel SH — opacity [N], uv [N,2], conic
    [N,3]; zero rows for culled gaussians), their masses d.mass and the near-threshold pixels d.near (see
    render_backward)."""
    N = o.inputs[0].shape[0]
    keep = o.keep
    g_rgb_c, g_opa_c, g_uv_c, g_conic_c, m = render_backward(o.uv, o.opacity, o.rgb, o.conic, o.view_dirs, o.ranges,
                                                             o.sorted_idx, o.background, o.n, o.wlast, grad_image,
                                                             mass=True)

    def full(a):
        out = np.zeros((N,) + a.shape[1:], np.float64)
        out[keep] = a
        return out

    render = SimpleNamespace(rgb=full(g_rgb_c), opacity=full(g_opa_c.reshape(-1)), uv=full(g_uv_c), conic=full(g_conic_c))
    mass = SimpleNamespace(rgb=full(m.rgb), opacity=full(m.opacity.reshape(-1)), uv=full(m.uv), conic=full(m.conic))
    if o.per_pixel:
        d = project_backward(o, np.zeros((N, 3)), render.opacity, render.uv, render.conic)
        d.rgb, d.sh = render.rgb[:, :, 0].copy(), render.rgb[:, :, 1:].copy()
    else:
        d = project_backward(o, render.rgb, render.opacity, render.uv, render.conic)
    d.uv, d.render, d.mass, d.near = g_uv_c, render, mass, m.near
    return d
