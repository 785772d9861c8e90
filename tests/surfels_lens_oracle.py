"""fp64 oracle of rasterize_surfels(..., fisheye=k / distortion=k) (tests/surfels_lens_oracle.c): every pixel's ray
against every visible surfel in depth order, no tiles, with the analytic backward.  TEST INFRASTRUCTURE.

    o = render(scene, bg, lens, kc)              # as tests/surfels_oracle.render (o.near, o.ill), plus o.rays [H,W,3]
    o = render(scene, bg, lens, kc, grads=G)     # + o.g, o.rows (dL/dM'), o.uv_grad, o.mass

lens: "fisheye" (kc = k1 k2 k3 k4) or "distortion" (kc = k1 k2 p1 p2 k3); the cull limit is appended here as the
kernels use it (rasterize.fisheye_theta_max / distortion_r2_max of the fp32 coefficients) unless `limit` is given.
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

from tests.surfels_oracle import _f64, _p, loss, sh_basis, view_dirs  # noqa: F401  (loss re-exported)

HERE = Path(__file__).resolve().parent
LENS_ID = {"fisheye": 1, "distortion": 2}
_lib = None


def build() -> Path:
    """Compile into a per-user cache directory outside the tree (keyed by the source's digest)."""
    src = HERE / "surfels_lens_oracle.c"
    digest = hashlib.sha256(src.read_bytes()).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_surfels_lens_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_surfels_lens_oracle_{digest}.so"
    if not out.exists():
        tmp = out.with_suffix(f".{os.getpid()}.tmp")
        subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", str(src), "-o", str(tmp), "-lm"],
                       check=True, capture_output=True)
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.surfel_lens_oracle.restype = C.c_int
    return _lib


def lens_constants(lens, kc, limit=None):
    """kc (fp32-rounded, as the kernels see it) and the cull limit, as fp64 [n+1]"""
    k = np.asarray(kc, np.float32).astype(np.float64)
    if limit is None:
        from gaussian_splatting_b200 import rasterize as R

        limit = (R.fisheye_theta_max if lens == "fisheye" else R.distortion_r2_max)(kc)
    return np.append(k, float(limit))


def render(scene, bg, lens, kc, grads=None, near=0.3, far=500.0, pad=100.0, mh=3.0, dirs=None, sort_z=None,
           limit=None):
    N, H, W = scene["xyz"].shape[0], int(scene["H"]), int(scene["W"])
    sh = scene.get("sh")
    n_sh = 1 if sh is None else 1 + sh.shape[2]
    coef = scene["rgb"].astype(np.float64)[:, :, None]
    if sh is not None:
        coef = np.concatenate([coef, sh.astype(np.float64)], 2)
    Y = sh_basis(view_dirs(scene) if dirs is None else dirs, n_sh)
    colour = _f64((coef * Y[:, None, :]).sum(2))
    o = SimpleNamespace(image=np.zeros((H, W, 3)), depth=np.zeros((H, W, 1)), alpha=np.zeros((H, W, 1)),
                        normal=np.zeros((H, W, 3)), dist=np.zeros((H, W, 1)), visible=np.zeros(N, np.uint8),
                        uv=np.zeros((N, 2)), colour=colour, rays=np.zeros((H, W, 3)))
    G = None
    if grads is not None:
        G = {k: _f64(grads.get(k, np.zeros((H, W, c)))) for k, c in
             (("image", 3), ("depth", 1), ("alpha", 1), ("normal", 3), ("dist", 1))}
        o.g = dict(xyz=np.zeros((N, 3)), quaternion=np.zeros((N, 4)), scale=np.zeros((N, 3)), opacity=np.zeros(N),
                   colour=np.zeros((N, 3)))
        o.rows, o.uv_grad, o.mass = np.zeros((N, 20)), np.zeros((N, 2)), np.zeros((N, 20))
    o.near = np.zeros((H, W), np.uint8)
    gp = (lambda k: None) if G is None else (lambda k: _p(G[k]))
    og = (lambda k: None) if G is None else (lambda k: _p(o.g[k]))
    zs = None if sort_z is None else _f64(sort_z)
    kcd = _f64(lens_constants(lens, kc, limit))
    keep = [_f64(scene["xyz"]), _f64(scene["quaternion"]), _f64(scene["scale"]), _f64(np.reshape(scene["opacity"], -1)),
            _f64(scene["T"]), _f64(scene["K"]), _f64(bg)]
    o.ill = np.zeros((H, W), np.uint8)
    lib().surfel_lens_oracle_ill(_p(o.ill))
    o.M = lib().surfel_lens_oracle(
        C.c_int(LENS_ID[lens]), _p(kcd), C.c_int(N), *[_p(a) for a in keep[:4]], _p(colour), _p(keep[4]),
        _p(keep[5]), C.c_int(H), C.c_int(W), C.c_double(near), C.c_double(far), C.c_double(pad), C.c_double(mh),
        _p(keep[6]), gp("image"), gp("depth"), gp("alpha"), gp("normal"), gp("dist"), _p(o.image), _p(o.depth),
        _p(o.alpha), _p(o.normal), _p(o.dist), _p(o.visible), _p(o.uv), og("xyz"), og("quaternion"), og("scale"),
        og("opacity"), og("colour"), None if G is None else _p(o.rows), None if G is None else _p(o.uv_grad),
        None if G is None else _p(o.mass), _p(o.near), _p(zs), _p(o.rays))
    lib().surfel_lens_oracle_ill(None)
    if G is not None:
        gc = o.g.pop("colour")
        gcoef = gc[:, :, None] * Y[:, None, :]
        o.g["rgb"] = gcoef[:, :, 0]
        o.g["sh"] = gcoef[:, :, 1:] if sh is not None else None
        o.g["opacity"] = o.g["opacity"].reshape(np.shape(scene["opacity"]))
    return o
