"""fp64 oracle of rasterize_surfels (tests/surfels_oracle.c): every pixel against every visible surfel in depth order,
no tiles, with the analytic backward.  TEST INFRASTRUCTURE.

    o = render(scene, bg)                        # o.image, o.depth, o.alpha, o.normal, o.dist, o.visible, o.uv
    o = render(scene, bg, grads=G)               # + o.g (xyz, quaternion, scale, opacity, rgb, sh), o.rows, o.uv_grad,
                                                 #   o.mass (per-pixel magnitudes summed into each row entry)
o.near [H,W]: pixels with a branch of the blend within 1e-4 of its threshold (surfels_oracle.c).

scene: dict of numpy arrays as tests/scenes.np_scene makes (xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W).
The SH colour is formed here at the centre's view direction; view_dirs [N,3] replaces that direction (held constant,
e.g. for central differences in xyz, which the kernels' gradient treats the same way).
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
_lib = None

SH_C = dict(c0=0.28209479177387814, c1=0.4886025119029199, c2=(1.0925484305920792, 0.31539156525252005,
                                                                0.5462742152960396),
            c3=(0.5900435899266435, 2.890611442640554, 0.4570457994644658, 0.263875515352797, 1.445305721320277))


def build() -> Path:
    """Compile into a per-user cache directory outside the tree (keyed by the source's digest)."""
    src = HERE / "surfels_oracle.c"
    digest = hashlib.sha256(src.read_bytes()).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_surfels_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_surfels_oracle_{digest}.so"
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
        _lib.surfel_oracle.restype = C.c_int
    return _lib


def sh_basis(d, n_sh):
    """Real SH basis [N, n_sh] at unit directions d [N,3] (gsr_math.cuh sh_basis, in fp64)."""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    Y = [np.full_like(x, SH_C["c0"])]
    if n_sh >= 4:
        Y += [-SH_C["c1"] * y, SH_C["c1"] * z, -SH_C["c1"] * x]
    if n_sh >= 9:
        a, b, c = SH_C["c2"]
        Y += [a * x * y, -a * y * z, b * (3 * z * z - 1), -a * x * z, c * (x * x - y * y)]
    if n_sh >= 16:
        a, b, c, e, f = SH_C["c3"]
        Y += [-a * y * (3 * x * x - y * y), b * x * y * z, -c * y * (5 * z * z - 1), e * z * (5 * z * z - 3),
              -c * x * (5 * z * z - 1), f * z * (x * x - y * y), -a * x * (x * x - 3 * y * y)]
    return np.stack(Y, 1)


def camera_centre(T):
    return np.linalg.inv(T.astype(np.float64))[:3, 3]


def view_dirs(scene):
    d = scene["xyz"].astype(np.float64) - camera_centre(scene["T"])
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def _f64(a):
    return np.ascontiguousarray(a, np.float64)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def render(scene, bg, grads=None, near=0.3, far=500.0, pad=100.0, mh=3.0, dirs=None, sort_z=None):
    """grads: None, or dict(image [H,W,3], depth [H,W,1], alpha [H,W,1], normal [H,W,3], dist [H,W,1]) (missing: 0).
    sort_z [N]: the depths the blend order sorts by (ties by index), e.g. the kernels' fp32 p_z; fp64 p_z when None."""
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
                        uv=np.zeros((N, 2)), colour=colour)
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
    keep = [_f64(scene["xyz"]), _f64(scene["quaternion"]), _f64(scene["scale"]), _f64(np.reshape(scene["opacity"], -1)),
            _f64(scene["T"]), _f64(scene["K"]), _f64(bg)]
    o.M = lib().surfel_oracle(
        C.c_int(N), *[_p(a) for a in keep[:4]], _p(colour), _p(keep[4]), _p(keep[5]), C.c_int(H), C.c_int(W),
        C.c_double(near), C.c_double(far), C.c_double(pad), C.c_double(mh), _p(keep[6]), gp("image"), gp("depth"),
        gp("alpha"), gp("normal"), gp("dist"), _p(o.image), _p(o.depth), _p(o.alpha), _p(o.normal), _p(o.dist),
        _p(o.visible), _p(o.uv), og("xyz"), og("quaternion"), og("scale"), og("opacity"), og("colour"),
        None if G is None else _p(o.rows), None if G is None else _p(o.uv_grad), None if G is None else _p(o.mass),
        _p(o.near), _p(zs))
    if G is not None:
        gc = o.g.pop("colour")
        gcoef = gc[:, :, None] * Y[:, None, :]   # colour = sum_k Y_k coef_k
        o.g["rgb"] = gcoef[:, :, 0]
        o.g["sh"] = gcoef[:, :, 1:] if sh is not None else None
        o.g["opacity"] = o.g["opacity"].reshape(np.shape(scene["opacity"]))
    return o


def loss(o, grads):
    """<G, outputs> of a forward, for central differences."""
    return sum(float((np.asarray(grads[k]) * getattr(o, k)).sum()) for k in grads)
